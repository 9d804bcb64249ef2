"""snarkjs / circom binary formats -> limb arrays (SURVEY 8f1).

Mirrors /root/reference/ark-circom/src/zkey.rs:53-387 (`read_zkey`: header, IC, coefficient section, the five
query sections), ark-circom/src/circom/r1cs_reader.rs:54-249 and the .wtns layout the reference consumes
through its witness calculator.  Pure byte shuffling with numpy -- no field arithmetic happens on the host:

  * curve points are stored by snarkjs in Montgomery form already (zkey.rs:340-345) and are returned as the
    (n, 8) / (n, 16) u64 limb arrays the C ABI takes; (0, 0) stays the infinity encoding (zkey.rs:353-373);
  * matrix coefficients are stored multiplied by R^2 (zkey.rs:333-338) and witness / r1cs values are
    canonical; they are returned raw together with the number of Montgomery reductions / conversions the
    device must apply (`Net.fr_convert`), which is how `groth16.qap.qap_from_zkey` feeds them to the GPU.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass

import numpy as np

FQ_MODULUS = 21888242871839275222246405745257275088696311157297823662689037894645226208583
FR_MODULUS = 21888242871839275222246405745257275088548364400416034343698204186575808495617


class FormatError(ValueError):
    pass


def _sections(buf: bytes, magic: bytes):
    if buf[:4] != magic:
        raise FormatError("bad magic %r (expected %r)" % (buf[:4], magic))
    _version, nsec = struct.unpack_from("<II", buf, 4)
    off = 12
    secs = {}
    for _ in range(nsec):
        sid, ln = struct.unpack_from("<IQ", buf, off)
        off += 12
        secs.setdefault(sid, []).append((off, ln))
        off += ln
    return secs


def _limbs(buf: bytes, off: int, count: int, width: int) -> np.ndarray:
    """count records of width u64 limbs starting at byte offset off."""
    return np.frombuffer(buf, dtype="<u8", count=count * width, offset=off).reshape(count, width).copy()


@dataclass
class ZKey:
    n_vars: int
    n_public: int
    domain_size: int
    alpha_g1: np.ndarray
    beta_g1: np.ndarray
    beta_g2: np.ndarray
    gamma_g2: np.ndarray
    delta_g1: np.ndarray
    delta_g2: np.ndarray
    ic: np.ndarray
    a_query: np.ndarray
    b_g1_query: np.ndarray
    b_g2_query: np.ndarray
    l_query: np.ndarray
    h_query: np.ndarray
    # coefficient section as COO triplets; values are value * R^2 mod r (raw file words)
    coef_matrix: np.ndarray
    coef_row: np.ndarray
    coef_col: np.ndarray
    coef_val_r2: np.ndarray

    @property
    def n_inputs(self) -> int:                 # num_instance_variables = n_public + 1 (zkey.rs:178)
        return self.n_public + 1

    @property
    def num_constraints(self) -> int:
        """zkey.rs:171: max constraint index - n_public (the appended public-input rows are dropped)."""
        return int(self.coef_row.max()) - self.n_public if self.coef_row.size else 0

    def vk_points(self) -> np.ndarray:
        """alpha_g1 beta_g1 delta_g1 beta_g2 delta_g2 -- the 56 limbs b200zk_pk_upload takes."""
        return np.concatenate([self.alpha_g1, self.beta_g1, self.delta_g1, self.beta_g2, self.delta_g2]).astype(np.uint64)


def read_zkey(buf: bytes) -> ZKey:
    secs = _sections(buf, b"zkey")
    for sid in (2, 3, 4, 5, 6, 7, 8, 9):
        if sid not in secs:
            raise FormatError("zkey section %d missing" % sid)
    off, _ = secs[2][0]
    n8q = struct.unpack_from("<I", buf, off)[0]
    off += 4
    q = int.from_bytes(buf[off:off + n8q], "little")
    off += n8q
    n8r = struct.unpack_from("<I", buf, off)[0]
    off += 4
    r = int.from_bytes(buf[off:off + n8r], "little")
    off += n8r
    if q != FQ_MODULUS or r != FR_MODULUS or n8q != 32 or n8r != 32:
        raise FormatError("zkey is not over BN254")
    n_vars, n_public, domain_size = struct.unpack_from("<III", buf, off)
    off += 12
    alpha_g1 = _limbs(buf, off, 1, 8)[0]; off += 64
    beta_g1 = _limbs(buf, off, 1, 8)[0]; off += 64
    beta_g2 = _limbs(buf, off, 1, 16)[0]; off += 128
    gamma_g2 = _limbs(buf, off, 1, 16)[0]; off += 128
    delta_g1 = _limbs(buf, off, 1, 8)[0]; off += 64
    delta_g2 = _limbs(buf, off, 1, 16)[0]; off += 128

    def sec(sid, count, width):
        o, ln = secs[sid][0]
        if ln < count * width * 8:
            raise FormatError("zkey section %d too short" % sid)
        return _limbs(buf, o, count, width)

    if n_vars == 0 or n_public + 1 > n_vars:
        raise FormatError("zkey header: n_public + 1 = %d variables are public but n_vars = %d" % (n_public + 1, n_vars))
    if domain_size == 0 or domain_size & (domain_size - 1):
        raise FormatError("zkey header: domain size %d is not a power of two" % domain_size)
    o4, l4 = secs[4][0]
    ncoef = struct.unpack_from("<I", buf, o4)[0]
    if l4 < 4 + ncoef * 44:
        raise FormatError("zkey coefficient section too short for %d records" % ncoef)
    rec = np.frombuffer(buf, dtype=np.dtype([("m", "<u4"), ("c", "<u4"), ("s", "<u4"), ("v", "<u8", (4,))]), count=ncoef,
                        offset=o4 + 4)
    # the device kernels index z[col] and the QAP rows with these values unchecked (csrc/qap.cu): reject what the reference
    # would panic on (index out of bounds) here, on the host
    if ncoef and (int(rec["m"].max()) > 1 or int(rec["s"].max()) >= n_vars or int(rec["c"].max()) >= domain_size):
        raise FormatError("zkey coefficient section: matrix index > 1, signal index >= n_vars or constraint index >= domain size")
    return ZKey(n_vars=n_vars, n_public=n_public, domain_size=domain_size, alpha_g1=alpha_g1, beta_g1=beta_g1,
                beta_g2=beta_g2, gamma_g2=gamma_g2, delta_g1=delta_g1, delta_g2=delta_g2,
                ic=sec(3, n_public + 1, 8), a_query=sec(5, n_vars, 8), b_g1_query=sec(6, n_vars, 8),
                b_g2_query=sec(7, n_vars, 16), l_query=sec(8, n_vars - n_public - 1, 8), h_query=sec(9, domain_size, 8),
                coef_matrix=rec["m"].copy(), coef_row=rec["c"].copy(), coef_col=rec["s"].copy(),
                coef_val_r2=rec["v"].copy())


_COEF = np.dtype([("m", "<u4"), ("c", "<u4"), ("s", "<u4"), ("v", "<u8", (4,))])
_ZKEY_ORDER = (1, 2, 4, 3, 9, 8, 5, 6, 7, 10)            # the section order snarkjs writes
_R2_LIMBS = np.array([((1 << 512) % FR_MODULUS >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)


def zkey_cir_power(n_constraints: int, n_public: int) -> int:
    """log2 of the zkey domain, ceil(log2(n_constraints + n_public + 1)): the constraints and the n_public + 1
    input-consistency rows must fit."""
    return (n_constraints + n_public).bit_length()


def zkey_coefficients(n_public: int, n_constraints: int, a, b):
    """The coefficient section (4) of a zkey as (matrix, constraint, signal, value * R^2) arrays, in snarkjs order: by
    constraint, A before B, then the input-consistency rows (0, n_constraints + j, j, 1) for j <= n_public.  a, b: (rows,
    cols, values already multiplied by R^2 as (n, 4) u64 limbs) of the r1cs A and B matrices.  Index work only."""
    m = [np.zeros(len(a[0]), np.uint32), np.ones(len(b[0]), np.uint32), np.zeros(n_public + 1, np.uint32)]
    c = [np.asarray(a[0], np.uint32), np.asarray(b[0], np.uint32), np.arange(n_constraints, n_constraints + n_public + 1, dtype=np.uint32)]
    s = [np.asarray(a[1], np.uint32), np.asarray(b[1], np.uint32), np.arange(n_public + 1, dtype=np.uint32)]
    v = [np.asarray(a[2], np.uint64).reshape(-1, 4), np.asarray(b[2], np.uint64).reshape(-1, 4), np.tile(_R2_LIMBS, (n_public + 1, 1))]
    m, c, s, v = (np.concatenate(x) for x in (m, c, s, v))
    order = np.argsort(c, kind="stable")
    return m[order], c[order], s[order], v[order]


def write_zkey(zk: ZKey, section10: bytes | None = None) -> bytes:
    """A Groth16 .zkey (snarkjs layout, the one read_zkey and ark-circom/src/zkey.rs read) with sections 1-10 in snarkjs
    order.  section10 defaults to a zero csHash (64 bytes) and zero phase-2 contributions: the real csHash hashes the
    ceremony's tau powers in snarkjs's order, which this writer does not compute, so `snarkjs zkey verify` rejects such a
    file while ark-circom's reader (and read_zkey) ignore the section."""
    hdr = struct.pack("<I", 32) + FQ_MODULUS.to_bytes(32, "little") + struct.pack("<I", 32) + FR_MODULUS.to_bytes(32, "little")
    hdr += struct.pack("<III", zk.n_vars, zk.n_public, zk.domain_size)
    pts = lambda a, w: np.ascontiguousarray(a, dtype="<u8").reshape(-1, w).tobytes()
    hdr += b"".join(pts(p, w) for p, w in ((zk.alpha_g1, 8), (zk.beta_g1, 8), (zk.beta_g2, 16), (zk.gamma_g2, 16),
                                            (zk.delta_g1, 8), (zk.delta_g2, 16)))
    rec = np.empty(len(zk.coef_matrix), dtype=_COEF)
    rec["m"], rec["c"], rec["s"], rec["v"] = zk.coef_matrix, zk.coef_row, zk.coef_col, np.asarray(zk.coef_val_r2).reshape(-1, 4)
    secs = {1: struct.pack("<I", 1), 2: hdr, 3: pts(zk.ic, 8), 4: struct.pack("<I", len(rec)) + rec.tobytes(),
            5: pts(zk.a_query, 8), 6: pts(zk.b_g1_query, 8), 7: pts(zk.b_g2_query, 16), 8: pts(zk.l_query, 8),
            9: pts(zk.h_query, 8), 10: bytes(64) + struct.pack("<I", 0) if section10 is None else bytes(section10)}
    return b"zkey" + struct.pack("<II", 1, len(_ZKEY_ORDER)) + b"".join(
        struct.pack("<IQ", sid, len(secs[sid])) + secs[sid] for sid in _ZKEY_ORDER)


class PTau:
    """A prepared Powers-of-Tau file (snarkjs `powersoftau prepare phase2`), memory-mapped: only the points a circuit needs
    are ever read (a 2^28 ceremony is hundreds of GB, a 2^20 circuit needs well under 1 GB of it).

    Layout (restated from snarkjs; points are Montgomery little-endian affine, infinity all-zero): section 1 = n8, q,
    power, ceremonyPower; 4 / 5 / 6 = alpha tau^i G1, beta tau^i G1, beta G2 (their first points are alpha_1, beta_1,
    beta_2); 12 / 13 / 14 / 15 = the Lagrange bases L G1, L G2, alpha L G1, beta L G1 of every domain 2^k, level k starting
    at point 2^k - 1 -- levels 0..power + 1 in section 12, 0..power in the others.

    prepared=False opens the output of a phase-1 ceremony instead (snarkjs `powersoftau prepare phase2` input): sections
    2-7 must be present and as long as the power requires (2 = tau^i G1, 2^(power+1) - 1 points; 3 = tau^i G2, 4, 5:
    2^power points each; 6: one point; 7 = the contribution records, any length), the power must be at most 27 (the top
    Lagrange level, power + 1, must fit the 2^28 domain of Fr), and sections 12-15 are neither required nor read."""

    _LAGRANGE = {12: 8, 13: 16, 14: 8, 15: 8}      # section -> u64 limbs per point
    MAX_UNPREPARED_POWER = 27

    def __init__(self, path: str, prepared: bool = True):
        import mmap
        self._prepared = prepared
        self._f = open(path, "rb")
        try:
            size = self._f.seek(0, 2)
            if size < 12:
                raise FormatError("ptau file too short (%d bytes)" % size)
            self._mm = mmap.mmap(self._f.fileno(), 0, access=mmap.ACCESS_READ)
            self._parse(size)
        except BaseException:
            self.close()
            raise

    def _parse(self, size: int):
        mm = self._mm
        if mm[:4] != b"ptau":
            raise FormatError("bad magic %r (expected b'ptau')" % mm[:4])
        _version, nsec = struct.unpack_from("<II", mm, 4)
        off, secs = 12, {}
        for _ in range(nsec):
            if off + 12 > size:
                raise FormatError("ptau section table runs past the end of the file")
            sid, ln = struct.unpack_from("<IQ", mm, off)
            off += 12
            if off + ln > size:
                raise FormatError("ptau section %d runs past the end of the file" % sid)
            secs.setdefault(sid, (off, ln))
            off += ln
        self._secs = secs
        if 1 not in secs or secs[1][1] < 4:
            raise FormatError("ptau header section 1 missing")
        o1, l1 = secs[1]
        n8 = struct.unpack_from("<I", mm, o1)[0]
        if n8 != 32 or l1 < 4 + n8 + 8:
            raise FormatError("ptau is not over BN254 (n8 = %d)" % n8)
        if int.from_bytes(mm[o1 + 4:o1 + 4 + n8], "little") != FQ_MODULUS:
            raise FormatError("ptau is not over BN254 (wrong q)")
        self.power, self.ceremony_power = struct.unpack_from("<II", mm, o1 + 4 + n8)
        if not self._prepared:
            if self.power > self.MAX_UNPREPARED_POWER:
                raise FormatError("ptau power %d above %d: its top Lagrange level (2^%d points) exceeds the 2^28 domain of Fr"
                                  % (self.power, self.MAX_UNPREPARED_POWER, self.power + 1))
            for sid, ln in self.tau_section_bytes(self.power).items():
                if sid not in secs:
                    raise FormatError("ptau section %d missing" % sid)
                if secs[sid][1] < ln:
                    raise FormatError("ptau section %d too short for power %d (%d < %d bytes)" % (sid, self.power, secs[sid][1], ln))
            return
        missing = [sid for sid in (12, 13, 14, 15) if sid not in secs]
        if missing:
            raise FormatError("ptau has no Lagrange sections %s: it is not prepared for phase 2 (run snarkjs powersoftau "
                              "prepare phase2 on it first)" % missing)
        need = {4: 64, 5: 64, 6: 128}
        for sid, w in self._LAGRANGE.items():
            need[sid] = ((1 << (self.power + (2 if sid == 12 else 1))) - 1) * w * 8
        for sid, ln in need.items():
            if sid not in secs:
                raise FormatError("ptau section %d missing" % sid)
            if secs[sid][1] < ln:
                raise FormatError("ptau section %d too short for power %d (%d < %d bytes)" % (sid, self.power, secs[sid][1], ln))

    @staticmethod
    def tau_section_bytes(power: int) -> dict:
        """Least length in bytes of sections 2-7 for a ceremony of this power."""
        n = 1 << power
        return {2: (2 * n - 1) * 64, 3: n * 128, 4: n * 64, 5: n * 64, 6: 128, 7: 0}

    @classmethod
    def lagrange_section_bytes(cls, power: int) -> dict:
        """Length in bytes of sections 12-15 of a prepared file of this power (levels 0..power + 1 in 12, 0..power in the
        others: 2^(top + 1) - 1 points)."""
        return {sid: ((1 << (power + (2 if sid == 12 else 1))) - 1) * w * 8 for sid, w in cls._LAGRANGE.items()}

    def section_span(self, sid: int):
        """(byte offset, length) of section sid in the file."""
        return self._secs[sid]

    def has_section(self, sid: int) -> bool:
        return sid in self._secs

    def section_chunks(self, sid: int, chunk: int = 1 << 26):
        """The bytes of section sid, in copies of at most `chunk` bytes."""
        off, ln = self._secs[sid]
        for lo in range(0, ln, chunk):
            yield self._mm[off + lo:off + min(ln, lo + chunk)]

    def points(self, sid: int, first: int, count: int, width: int) -> np.ndarray:
        """count points of section sid from point `first` as (count, width) u64 limbs (width 8: G1, 16: G2)."""
        return self._points(sid, first, count, width)

    def _points(self, sid: int, first: int, count: int, width: int) -> np.ndarray:
        off = self._secs[sid][0] + first * width * 8
        return np.frombuffer(self._mm, dtype="<u8", count=count * width, offset=off).reshape(count, width).copy()

    @property
    def alpha_g1(self) -> np.ndarray:
        return self._points(4, 0, 1, 8)[0]

    @property
    def beta_g1(self) -> np.ndarray:
        return self._points(5, 0, 1, 8)[0]

    @property
    def beta_g2(self) -> np.ndarray:
        return self._points(6, 0, 1, 16)[0]

    def lagrange(self, sid: int, level: int) -> np.ndarray:
        """Level `level` (2^level points) of Lagrange section sid (12, 13, 14 or 15) as (2^level, 8 | 16) u64 limbs."""
        top = self.power + (1 if sid == 12 else 0)
        if level > top:
            raise FormatError("the circuit needs Lagrange level %d of ptau section %d, the ceremony (power %d) has levels up "
                              "to %d: the circuit is too big for it" % (level, sid, self.power, top))
        return self._points(sid, (1 << level) - 1, 1 << level, self._LAGRANGE[sid])

    def close(self):
        mm, self._mm = getattr(self, "_mm", None), None
        if mm is not None:
            mm.close()
        f, self._f = getattr(self, "_f", None), None
        if f is not None:
            f.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def ptau_challenge_bytes(power: int) -> int:
    """Size of a snarkjs phase-1 challenge file of this power (n = 2^power): the 64-byte lastResponseHash, then the
    uncompressed sections 2 (2n - 1 G1), 3 (n G2), 4 and 5 (n G1 each) and 6 (1 G2): 384 n + 128 bytes."""
    return 384 * (1 << power) + 128


def ptau_response_bytes(power: int) -> int:
    """Size of a snarkjs phase-1 response file of this power: the 64-byte challenge hash, the compressed sections 2-6 and
    the 768-byte public key: 192 n + 864 bytes."""
    return 192 * (1 << power) + 864


def _power_of(size: int, per_power, what: str) -> int:
    for p in range(1, PTau.MAX_UNPREPARED_POWER + 1):
        if per_power(p) == size:
            return p
    raise FormatError("a %s file of %d bytes fits no power from 1 to %d" % (what, size, PTau.MAX_UNPREPARED_POWER))


def ptau_challenge_power(size: int) -> int:
    """The power whose challenge file is `size` bytes; FormatError when there is none in 1..27."""
    return _power_of(size, ptau_challenge_bytes, "challenge")


def ptau_response_power(size: int) -> int:
    """The power whose response file is `size` bytes; FormatError when there is none in 1..27."""
    return _power_of(size, ptau_response_bytes, "response")


def read_ptau(path: str) -> PTau:
    """Open a prepared .ptau (memory-mapped; see PTau).  Raises FormatError for a file that is not a BN254 ptau, is not
    prepared for phase 2 or whose sections are shorter than its stated power."""
    return PTau(path)


def ptau_preamble(n_sections: int, power: int) -> bytes:
    """The first bytes of every ptau file this package writes: magic, version 1, the section count and section 1 =
    (n8 = 32, q, power, ceremonyPower = power) -- what snarkjs' writePTauHeader(curve, power) writes as far as is known
    here (not checked against snarkjs)."""
    s1 = struct.pack("<I", 32) + FQ_MODULUS.to_bytes(32, "little") + struct.pack("<II", power, power)
    return b"ptau" + struct.pack("<II", 1, n_sections) + struct.pack("<IQ", 1, len(s1)) + s1


class PTauWriter:
    """Streams a phase-1 ceremony file (snarkjs `powersoftau new` / `contribute` / `beacon` output) of `power` (1..27) to
    `path`: sections 1-7 in that order.  Section 1 is ptau_preamble's; sections 2-6 are appended in chunks through
    write(sid, data) in file order, each exactly PTau.tau_section_bytes(power) long; section 7 (the contribution records,
    ptau_contributions_bytes) is written whole by write_contributions() once 2-6 are complete.  Every length is checked:
    close() raises ValueError for a file left short."""

    def __init__(self, path: str, power: int):
        if not 1 <= power <= PTau.MAX_UNPREPARED_POWER:
            raise ValueError("ptau power must be in 1..%d, got %d" % (PTau.MAX_UNPREPARED_POWER, power))
        self.power = power
        self._lengths = PTau.tau_section_bytes(power)
        self._sid, self._left = 1, 0              # section being written and bytes it still needs
        self.section_offsets = {}                 # section -> file offset of its first byte, once begun
        self._f = open(path, "wb")
        try:
            self._f.write(ptau_preamble(7, power))
        except BaseException:
            self._f.close()
            raise

    def write(self, sid: int, data) -> None:
        """Append `data` (bytes or a u64 array of points) to section sid (2..6); sections come in order, each complete
        before the next begins."""
        data = memoryview(np.ascontiguousarray(data) if isinstance(data, np.ndarray) else data).cast("B")
        if sid != self._sid:
            if self._left or sid != self._sid + 1 or not 2 <= sid <= 6:
                raise ValueError("ptau section %d out of order (section %d has %d bytes to go)" % (sid, self._sid, self._left))
            self._sid, self._left = sid, self._lengths[sid]
            self._f.write(struct.pack("<IQ", sid, self._left))
            self.section_offsets[sid] = self._f.tell()
        if data.nbytes > self._left:
            raise ValueError("ptau section %d: %d bytes more than its %d" % (sid, data.nbytes - self._left, self._lengths[sid]))
        self._f.write(data)
        self._left -= data.nbytes

    def flush(self) -> None:
        """Push what was written so far to the file, so that it can be read back while the writer stays open."""
        self._f.flush()

    def write_contributions(self, sec7: bytes) -> None:
        if self._sid != 6 or self._left:
            raise ValueError("ptau section 7 before sections 2-6 are complete")
        self._f.write(struct.pack("<IQ", 7, len(sec7)) + bytes(sec7))
        self._sid = 7

    def close(self) -> None:
        f, self._f = self._f, None
        if f is None:
            return
        f.close()
        if self._sid != 7:
            raise ValueError("ptau incomplete: stopped in section %d" % self._sid)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        f, self._f = self._f, None
        if f is not None:
            f.close()


class PreparedPTauWriter:
    """Streams the output of snarkjs `powersoftau prepare phase2` for an open ceremony `src` (a PTau, prepared or not) to
    `path`: 11 sections in the order 1, 2-7, 12-15.  Section 1 is restated as (n8, q, power, ceremonyPower = power) -- what
    snarkjs' writePTauHeader(curve, power) writes as far as is known here; sections 2-7 are copied byte for byte (section 7
    with any contribution records).  The Lagrange sections follow level by level through write_level(), in the order
    `levels()` lists, so the host holds one level at a time; every length is known in advance and checked."""

    def __init__(self, path: str, src: PTau):
        self.power = src.power
        self._lengths = PTau.lagrange_section_bytes(self.power)
        self._order = [(sid, k) for sid in (12, 13, 14, 15) for k in range(self.power + (2 if sid == 12 else 1))]
        self._next = 0
        self._f = open(path, "wb")
        try:
            self._f.write(ptau_preamble(11, self.power))
            for sid in (2, 3, 4, 5, 6, 7):
                self._f.write(struct.pack("<IQ", sid, src.section_span(sid)[1]))
                for part in src.section_chunks(sid):
                    self._f.write(part)
        except BaseException:
            self._f.close()
            raise

    def levels(self) -> list:
        """[(section, level)] in file order."""
        return list(self._order)

    def write_level(self, sid: int, level: int, data) -> None:
        """Level `level` of Lagrange section sid: 2^level points (8 or 16 u64 limbs each) as bytes or a u64 array."""
        if self._next >= len(self._order) or self._order[self._next] != (sid, level):
            raise ValueError("Lagrange level (%d, %d) out of order: expected %r" % (
                sid, level, self._order[self._next] if self._next < len(self._order) else None))
        data = memoryview(np.ascontiguousarray(data) if isinstance(data, np.ndarray) else data).cast("B")
        want = (1 << level) * PTau._LAGRANGE[sid] * 8
        if data.nbytes != want:
            raise ValueError("Lagrange level (%d, %d) has %d bytes, expected %d" % (sid, level, data.nbytes, want))
        if level == 0:
            self._f.write(struct.pack("<IQ", sid, self._lengths[sid]))
        self._f.write(data)
        self._next += 1

    def close(self) -> None:
        """Finish the file; raises ValueError (and leaves it truncated) if levels are missing."""
        f, self._f = self._f, None
        if f is None:
            return
        f.close()
        if self._next != len(self._order):
            raise ValueError("prepared ptau incomplete: %d of %d Lagrange levels written" % (self._next, len(self._order)))

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        f, self._f = self._f, None
        if f is not None:
            f.close()


@dataclass
class Contribution:
    """One phase-2 record of a zkey's section 10 (snarkjs `zkey contribute` / `zkey beacon`).  Points are Montgomery
    little-endian affine limb arrays like the other sections (G1 8, G2 16 u64 limbs; infinity all-zero)."""
    delta_after: np.ndarray        # delta_1 after this contribution
    g1_s: np.ndarray
    g1_sx: np.ndarray              # x g1_s
    g2_spx: np.ndarray             # x hashToG2(transcript)
    transcript: bytes              # 64 bytes
    type: int = 0                  # 0 = contribution, 1 = beacon
    name: str | None = None
    num_iterations_exp: int | None = None
    beacon_hash: bytes | None = None


@dataclass
class MPCParams:
    """Section 10 of a zkey: the circuit hash and the phase-2 contributions, oldest first."""
    cs_hash: bytes
    contributions: list


_MPC_NAME_MAX = 64


def parse_mpc_params(sec: bytes) -> MPCParams:
    """Section 10 bytes -> MPCParams.  Layout (restated from snarkjs zkey_utils read/writeMPCParams): csHash (64 bytes),
    u32 count, then per contribution deltaAfter, g1_s, g1_sx (G1), g2_spx (G2), transcript (64 bytes), u32 type, u32 byte
    length of a key / value stream: 1 = name (u8 length + UTF-8, at most 64 bytes), 2 = numIterationsExp (u8), 3 =
    beaconHash (u8 length + bytes).  Raises FormatError for a truncated section, a count that runs past it, an unknown
    parameter key or an over-long name."""
    sec = bytes(sec)

    def need(off, n, what):
        if off + n > len(sec):
            raise FormatError("zkey section 10 ends inside %s (%d + %d > %d bytes)" % (what, off, n, len(sec)))

    need(0, 68, "the csHash and contribution count")
    cs_hash, count = sec[:64], struct.unpack_from("<I", sec, 64)[0]
    rec = 3 * 64 + 128 + 64 + 8                     # fixed part of one contribution
    if 68 + count * rec > len(sec):
        raise FormatError("zkey section 10 claims %d contributions, more than its %d bytes hold" % (count, len(sec)))
    off, out = 68, []
    for i in range(count):
        need(off, rec, "contribution %d" % i)
        pts = np.frombuffer(sec, dtype="<u8", count=40, offset=off).copy()
        off += 320
        transcript = sec[off:off + 64]
        ctype, plen = struct.unpack_from("<II", sec, off + 64)
        off += 72
        need(off, plen, "the parameters of contribution %d" % i)
        p, end = off, off + plen
        c = Contribution(delta_after=pts[:8], g1_s=pts[8:16], g1_sx=pts[16:24], g2_spx=pts[24:40], transcript=transcript,
                         type=ctype)
        _read_params(sec, p, end, i, c)
        off = end
        out.append(c)
    return MPCParams(cs_hash=cs_hash, contributions=out)


def _read_params(sec: bytes, p: int, end: int, i: int, c) -> None:
    """The key / value parameters of contribution i in sec[p:end] into c.name, c.num_iterations_exp and c.beacon_hash
    (the same stream in a zkey's section 10 and a ptau's section 7)."""
    while p < end:
        key = sec[p]
        if key == 1:
            if p + 2 > end or p + 2 + sec[p + 1] > end:
                raise FormatError("contribution %d: name runs past its parameters" % i)
            ln = sec[p + 1]
            if ln > _MPC_NAME_MAX:
                raise FormatError("contribution %d: name of %d bytes (at most %d)" % (i, ln, _MPC_NAME_MAX))
            try:
                c.name = sec[p + 2:p + 2 + ln].decode("utf-8")
            except UnicodeDecodeError as e:
                raise FormatError("contribution %d: name is not UTF-8 (%s)" % (i, e)) from None
            p += 2 + ln
        elif key == 2:
            if p + 2 > end:
                raise FormatError("contribution %d: numIterationsExp runs past its parameters" % i)
            c.num_iterations_exp = sec[p + 1]
            p += 2
        elif key == 3:
            if p + 2 > end or p + 2 + sec[p + 1] > end:
                raise FormatError("contribution %d: beacon hash runs past its parameters" % i)
            c.beacon_hash = sec[p + 2:p + 2 + sec[p + 1]]
            p += 2 + sec[p + 1]
        else:
            raise FormatError("contribution %d: unknown parameter key %d" % (i, key))


def _params_bytes(c) -> bytes:
    """The parameter stream of a record (inverse of _read_params): name, then for a beacon (type 1) its parameters."""
    prm = b""
    if c.name:
        name = c.name.encode("utf-8")
        if len(name) > _MPC_NAME_MAX:
            raise FormatError("contribution name of %d bytes (at most %d)" % (len(name), _MPC_NAME_MAX))
        prm += bytes([1, len(name)]) + name
    if c.type == 1:
        if c.num_iterations_exp is None or c.beacon_hash is None or len(c.beacon_hash) > 255:
            raise FormatError("a beacon record needs numIterationsExp and a beacon hash of at most 255 bytes")
        prm += bytes([2, c.num_iterations_exp, 3, len(c.beacon_hash)]) + bytes(c.beacon_hash)
    return prm


@dataclass
class PTauContribution:
    """One phase-1 record of a ptau's section 7 (snarkjs `powersoftau contribute` / `beacon`).  Points are Montgomery
    little-endian affine limb arrays (G1 8, G2 16 u64 limbs; infinity all-zero).  key[name] for name in "tau", "alpha",
    "beta" holds the proof of knowledge of that secret x: g1_s, g1_sx = x g1_s (G1) and g2_spx = x g2_sp (G2), where g2_sp
    is hashed from the previous challenge and is not stored."""
    tau_g1: np.ndarray             # tau G1 after this contribution (point 1 of section 2)
    tau_g2: np.ndarray             # point 1 of section 3
    alpha_g1: np.ndarray           # point 0 of section 4
    beta_g1: np.ndarray            # point 0 of section 5
    beta_g2: np.ndarray            # the point of section 6
    key: dict                      # "tau" / "alpha" / "beta" -> {"g1_s", "g1_sx", "g2_spx"}
    partial_hash: bytes            # 216 bytes: the response hasher's state after the points (see csrc/blake2b.cuh)
    next_challenge: bytes          # 64 bytes
    type: int = 0                  # 0 = contribution, 1 = beacon
    name: str | None = None
    num_iterations_exp: int | None = None
    beacon_hash: bytes | None = None


_KEY_NAMES = ("tau", "alpha", "beta")
_PTAU_POINTS_U64 = (8 + 16 + 8 + 8 + 16) + 6 * 8 + 3 * 16          # record points, then the public key: 152 u64
_PTAU_REC = _PTAU_POINTS_U64 * 8 + 216 + 64 + 8                    # fixed part of one record: 1504 bytes


def parse_ptau_contributions(sec: bytes) -> list:
    """Section 7 bytes of a ptau -> [PTauContribution], oldest first.  Layout (restated from snarkjs powersoftau_utils
    writeContribution, NOT checked against a file snarkjs wrote): u32 count, then per record tauG1, tauG2, alphaG1,
    betaG1, betaG2, the public key tau.g1_s, tau.g1_sx, alpha.g1_s, alpha.g1_sx, beta.g1_s, beta.g1_sx, tau.g2_spx,
    alpha.g2_spx, beta.g2_spx (all Montgomery LE), partialHash (216 bytes), nextChallenge (64 bytes), u32 type, u32 byte
    length of the key / value parameters (as in a zkey's section 10: 1 = name, 2 = numIterationsExp, 3 = beacon hash).
    Raises FormatError for a truncated section, a count that runs past it, an unknown parameter key or an over-long
    name."""
    sec = bytes(sec)

    def need(off, n, what):
        if off + n > len(sec):
            raise FormatError("ptau section 7 ends inside %s (%d + %d > %d bytes)" % (what, off, n, len(sec)))

    need(0, 4, "the contribution count")
    count = struct.unpack_from("<I", sec, 0)[0]
    if 4 + count * _PTAU_REC > len(sec):
        raise FormatError("ptau section 7 claims %d contributions, more than its %d bytes hold" % (count, len(sec)))
    off, out = 4, []
    for i in range(count):
        need(off, _PTAU_REC, "contribution %d" % i)
        pts = np.frombuffer(sec, dtype="<u8", count=_PTAU_POINTS_U64, offset=off).copy()
        off += _PTAU_POINTS_U64 * 8
        g1s = [pts[56 + 8 * k:64 + 8 * k] for k in range(6)]
        g2s = [pts[104 + 16 * k:120 + 16 * k] for k in range(3)]
        key = {nm: {"g1_s": g1s[2 * k], "g1_sx": g1s[2 * k + 1], "g2_spx": g2s[k]} for k, nm in enumerate(_KEY_NAMES)}
        partial, nxt = sec[off:off + 216], sec[off + 216:off + 280]
        ctype, plen = struct.unpack_from("<II", sec, off + 280)
        off += 288
        need(off, plen, "the parameters of contribution %d" % i)
        c = PTauContribution(tau_g1=pts[0:8], tau_g2=pts[8:24], alpha_g1=pts[24:32], beta_g1=pts[32:40], beta_g2=pts[40:56],
                             key=key, partial_hash=partial, next_challenge=nxt, type=ctype)
        _read_params(sec, off, off + plen, i, c)
        off += plen
        out.append(c)
    return out


def ptau_contributions_bytes(contributions) -> bytes:
    """[PTauContribution] -> section 7 bytes (the inverse of parse_ptau_contributions)."""
    out = [struct.pack("<I", len(contributions))]
    for c in contributions:
        flat = lambda a: np.ascontiguousarray(a, dtype="<u8").reshape(-1)
        pts = [flat(a) for a in (c.tau_g1, c.tau_g2, c.alpha_g1, c.beta_g1, c.beta_g2)]
        pts += [flat(c.key[nm][f]) for nm in _KEY_NAMES for f in ("g1_s", "g1_sx")]
        pts += [flat(c.key[nm]["g2_spx"]) for nm in _KEY_NAMES]
        if [p.size for p in pts] != [8, 16, 8, 8, 16] + [8] * 6 + [16] * 3:
            raise FormatError("phase-1 record points must be G1 (8 limbs) and G2 (16 limbs) as the layout says")
        if len(c.partial_hash) != 216 or len(c.next_challenge) != 64:
            raise FormatError("partialHash must be 216 bytes and nextChallenge 64")
        prm = _params_bytes(c)
        out += [b"".join(p.tobytes() for p in pts), bytes(c.partial_hash), bytes(c.next_challenge),
                struct.pack("<II", c.type, len(prm)), prm]
    return b"".join(out)


def read_mpc_params(zkey_bytes: bytes) -> MPCParams:
    """The phase-2 parameters (section 10) of a zkey; see parse_mpc_params."""
    secs = _sections(zkey_bytes, b"zkey")
    if 10 not in secs:
        raise FormatError("zkey section 10 missing")
    off, ln = secs[10][0]
    if off + ln > len(zkey_bytes):
        raise FormatError("zkey section 10 runs past the end of the file")
    return parse_mpc_params(zkey_bytes[off:off + ln])


def mpc_params_bytes(params: MPCParams) -> bytes:
    """MPCParams -> section 10 bytes (the inverse of parse_mpc_params; feed them to write_zkey(zk, section10=...))."""
    if len(params.cs_hash) != 64:
        raise FormatError("csHash must be 64 bytes, got %d" % len(params.cs_hash))
    out = [bytes(params.cs_hash), struct.pack("<I", len(params.contributions))]
    for c in params.contributions:
        pts = [np.ascontiguousarray(a, dtype="<u8").reshape(-1) for a in (c.delta_after, c.g1_s, c.g1_sx, c.g2_spx)]
        if [p.size for p in pts] != [8, 8, 8, 16] or len(c.transcript) != 64:
            raise FormatError("contribution points must be 8, 8, 8 and 16 limbs and the transcript 64 bytes")
        prm = _params_bytes(c)
        out += [b"".join(p.tobytes() for p in pts), bytes(c.transcript), struct.pack("<II", c.type, len(prm)), prm]
    return b"".join(out)


# ---- bellman MPC params (snarkjs `zkey export bellman` / `zkey bellman contribute` / `zkey import bellman`) -------------
BELLMAN_HEADER = (("alpha_g1", 64), ("beta_g1", 64), ("beta_g2", 128), ("gamma_g2", 128), ("delta_g1", 64), ("delta_g2", 128))
BELLMAN_VECTORS = (("ic", 64), ("h", 64), ("l", 64), ("a", 64), ("b1", 64), ("b2", 128))
BELLMAN_RECORD = 384                              # U(deltaAfter) U(g1_s) U(g1_sx) U(g2_spx) transcript


@dataclass
class Bellman:
    """A parsed bellman MPC-params file.  spans[part] = (byte offset, byte length) for every part of BELLMAN_HEADER and
    BELLMAN_VECTORS (a vector's span excludes its count); counts[part] for the vectors; params_end = the offset of the
    csHash, so buf[:params_end] is what the circuit hash covers; records_offset = the offset of the first record."""
    counts: dict
    spans: dict
    params_end: int
    cs_hash: bytes
    records_offset: int
    contributions: list


def bellman_size(n_ic: int, n_h: int, n_l: int, n_vars: int, n_records: int = 0) -> int:
    """The byte size of a bellman MPC-params file: the 576-byte header points, six u32-counted vectors (IC, H, L, A, B1 of
    G1 points, B2 of G2 points, each of n_vars entries for A, B1 and B2), the csHash, a u32 record count and the records."""
    return 576 + 6 * 4 + 64 * (n_ic + n_h + n_l + 2 * n_vars) + 128 * n_vars + 64 + 4 + BELLMAN_RECORD * n_records


def _u_to_limbs(b: bytes, g2: bool, what: str) -> np.ndarray:
    """ffjavascript toRprUncompressed -> Montgomery limbs on the host (for the handful of record points).  Infinity is
    0x40 then zeros; otherwise the top two bits of byte 0 are clear and every coordinate is below q.  No curve check."""
    if b[0] & 0xC0:
        if b[0] != 0x40 or any(b[1:]):
            raise FormatError("%s: not an uncompressed point encoding (flag byte 0x%02x)" % (what, b[0]))
        return np.zeros(16 if g2 else 8, dtype=np.uint64)
    coords = [int.from_bytes(b[32 * k:32 * k + 32], "big") for k in range(len(b) // 32)]
    if any(v >= FQ_MODULUS for v in coords):
        raise FormatError("%s: a coordinate is not below q" % what)
    if g2:
        coords = [coords[k] for k in (1, 0, 3, 2)]          # x.c1 x.c0 y.c1 y.c0 -> x.c0 x.c1 y.c0 y.c1
    mont = [(v << 256) % FQ_MODULUS for v in coords]
    return np.array([(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for v in mont for i in range(4)], dtype=np.uint64)


def parse_bellman(buf: bytes) -> Bellman:
    """A bellman MPC-params file (as snarkjs `zkey export bellman` writes it) -> Bellman.  Byte shuffling only: points stay
    encoded except the records', which become formats.Contribution (type 0, no name; bellman carries neither).  Raises
    FormatError for a truncated file, a count that disagrees with the file's length and trailing bytes."""
    buf = bytes(buf)

    def need(off, n, what):
        if off + n > len(buf):
            raise FormatError("bellman params end inside %s (%d + %d > %d bytes)" % (what, off, n, len(buf)))

    spans, counts, off = {}, {}, 0
    for part, w in BELLMAN_HEADER:
        need(off, w, part)
        spans[part] = (off, w)
        off += w
    for part, w in BELLMAN_VECTORS:
        need(off, 4, "the count of %s" % part)
        cnt = struct.unpack_from(">I", buf, off)[0]
        off += 4
        if off + cnt * w > len(buf):
            raise FormatError("bellman params: %s claims %d points, more than the %d bytes left hold" % (part, cnt, len(buf) - off))
        counts[part], spans[part] = cnt, (off, cnt * w)
        off += cnt * w
    if not counts["a"] == counts["b1"] == counts["b2"]:
        raise FormatError("bellman params: A, B1 and B2 have %d, %d and %d points (one per variable each)"
                          % (counts["a"], counts["b1"], counts["b2"]))
    params_end = off
    need(off, 68, "the csHash and record count")
    cs_hash, k = buf[off:off + 64], struct.unpack_from(">I", buf, off + 64)[0]
    rec = off + 68
    if len(buf) != rec + BELLMAN_RECORD * k:
        raise FormatError("bellman params of %d bytes; its counts give %d (%d records)"
                          % (len(buf), bellman_size(counts["ic"], counts["h"], counts["l"], counts["a"], k), k))
    out = []
    for i in range(k):
        o = rec + BELLMAN_RECORD * i
        pt = lambda j, w, g2, nm: _u_to_limbs(buf[o + j:o + j + w], g2, "record %d %s" % (i, nm))
        out.append(Contribution(delta_after=pt(0, 64, False, "deltaAfter"), g1_s=pt(64, 64, False, "g1_s"),
                                g1_sx=pt(128, 64, False, "g1_sx"), g2_spx=pt(192, 128, True, "g2_spx"),
                                transcript=buf[o + 320:o + 384]))
    return Bellman(counts=counts, spans=spans, params_end=params_end, cs_hash=cs_hash, records_offset=rec, contributions=out)


def read_wtns(buf: bytes) -> np.ndarray:
    """(n, 4) u64 canonical (non-Montgomery) witness values."""
    secs = _sections(buf, b"wtns")
    off, _ = secs[1][0]
    n8 = struct.unpack_from("<I", buf, off)[0]
    prime = int.from_bytes(buf[off + 4:off + 4 + n8], "little")
    if n8 != 32 or prime != FR_MODULUS:
        raise FormatError("wtns is not over BN254 Fr")
    n = struct.unpack_from("<I", buf, off + 4 + n8)[0]
    o2, ln = secs[2][0]
    if ln < n * 32:
        raise FormatError("wtns data section too short")
    return _limbs(buf, o2, n, 4)


@dataclass
class R1CS:
    n_wires: int
    n_pub_out: int
    n_pub_in: int
    n_prv_in: int
    n_constraints: int
    # COO per matrix (A, B, C): rows, cols, canonical coefficient limbs
    rows: list
    cols: list
    vals: list


def read_r1cs(buf: bytes) -> R1CS:
    secs = _sections(buf, b"r1cs")
    off, _ = secs[1][0]
    fs = struct.unpack_from("<I", buf, off)[0]
    prime = int.from_bytes(buf[off + 4:off + 4 + fs], "little")
    if fs != 32 or prime != FR_MODULUS:                       # r1cs_reader.rs:180-188
        raise FormatError("r1cs is not over BN254 Fr")
    off += 4 + fs
    n_wires, n_pub_out, n_pub_in, n_prv_in = struct.unpack_from("<IIII", buf, off)
    off += 16 + 8
    n_constraints = struct.unpack_from("<I", buf, off)[0]
    off, l2 = secs[2][0]
    end2 = off + l2
    rows = [[], [], []]
    cols = [[], [], []]
    vals = [[], [], []]
    term = np.dtype([("w", "<u4"), ("v", "<u8", (4,))])
    for i in range(n_constraints):
        for k in range(3):
            if off + 4 > end2:
                raise FormatError("r1cs constraint section ends inside constraint %d" % i)
            nterm = struct.unpack_from("<I", buf, off)[0]
            off += 4
            if off + nterm * 36 > end2:
                raise FormatError("r1cs constraint section ends inside constraint %d" % i)
            t = np.frombuffer(buf, dtype=term, count=nterm, offset=off)
            off += nterm * 36
            if nterm and int(t["w"].max()) >= n_wires:
                raise FormatError("r1cs constraint %d names wire %d of %d" % (i, int(t["w"].max()), n_wires))
            rows[k].append(np.full(nterm, i, dtype=np.uint32))
            cols[k].append(t["w"].astype(np.uint32))
            vals[k].append(t["v"].astype(np.uint64).reshape(nterm, 4))
    cat = lambda parts, shape: np.concatenate(parts) if parts else np.zeros(shape, dtype=np.uint32)
    return R1CS(n_wires, n_pub_out, n_pub_in, n_prv_in, n_constraints,
                [cat(r, (0,)) for r in rows], [cat(c, (0,)) for c in cols],
                [np.concatenate(v) if v else np.zeros((0, 4), dtype=np.uint64) for v in vals])


def coo_to_csr(rows: np.ndarray, cols: np.ndarray, vals: np.ndarray, n_rows: int):
    """Stable sort by row -> (row_ptr[n_rows+1] u32, col u32, val (nnz,4) u64). Index-only host work."""
    keep = rows < n_rows
    rows, cols, vals = rows[keep], cols[keep], vals[keep]
    order = np.argsort(rows, kind="stable")
    counts = np.bincount(rows, minlength=n_rows).astype(np.uint64)
    row_ptr = np.zeros(n_rows + 1, dtype=np.uint32)
    row_ptr[1:] = np.cumsum(counts).astype(np.uint32)
    return row_ptr, np.ascontiguousarray(cols[order], dtype=np.uint32), np.ascontiguousarray(vals[order], dtype=np.uint64)


# ---- snarkjs's Groth16 JSON files: proof.json, public.json, verification_key.json ------------------------------------------
# Text only: points are coordinates as Python ints (G1 (x, y), G2 ((x.c0, x.c1), (y.c0, y.c1)), None = infinity); turning them
# into device points is groth16/snarkjs.py's job.  The writer reproduces snarkjs's JSON.stringify(obj, null, 1) byte for byte
# (one-space indent, one array item per line, no trailing newline); the reader takes decimal and 0x-hex strings, as
# ffjavascript's unstringifyBigInts does.

@dataclass
class SnarkjsProof:
    pi_a: tuple | None
    pi_b: tuple | None
    pi_c: tuple | None


@dataclass
class SnarkjsVerificationKey:
    n_public: int
    alpha_1: tuple | None
    beta_2: tuple | None
    gamma_2: tuple | None
    delta_2: tuple | None
    alphabeta_12: list          # 2 x 3 x 2 canonical Fq ints: [Fq6 c0, Fq6 c1], each [Fq2 a, b, c], each [c0, c1]
    ic: list                    # n_public + 1 G1 points


def _dumps(obj) -> str:
    import json
    return json.dumps(obj, indent=1)            # == JSON.stringify(obj, null, 1) for strings, ints, lists and dicts


def _g1_json(p) -> list:
    return ["0", "1", "0"] if p is None else [str(int(p[0])), str(int(p[1])), "1"]


def _g2_json(p) -> list:
    if p is None:
        return [["0", "0"], ["1", "0"], ["0", "0"]]
    return [[str(int(p[0][0])), str(int(p[0][1]))], [str(int(p[1][0])), str(int(p[1][1]))], ["1", "0"]]


def write_proof_json(proof: SnarkjsProof) -> str:
    return _dumps({"pi_a": _g1_json(proof.pi_a), "pi_b": _g2_json(proof.pi_b), "pi_c": _g1_json(proof.pi_c),
                   "protocol": "groth16", "curve": "bn128"})


def write_public_json(values) -> str:
    return _dumps([str(int(v)) for v in values])


def write_vk_json(vk: SnarkjsVerificationKey) -> str:
    ab = [[[str(int(vk.alphabeta_12[h][k][j])) for j in range(2)] for k in range(3)] for h in range(2)]
    return _dumps({"protocol": "groth16", "curve": "bn128", "nPublic": int(vk.n_public), "vk_alpha_1": _g1_json(vk.alpha_1),
                   "vk_beta_2": _g2_json(vk.beta_2), "vk_gamma_2": _g2_json(vk.gamma_2), "vk_delta_2": _g2_json(vk.delta_2),
                   "vk_alphabeta_12": ab, "IC": [_g1_json(p) for p in vk.ic]})


def _json_load(text, what: str):
    import json
    try:
        return json.loads(text)
    except (ValueError, TypeError) as e:
        raise FormatError("%s is not JSON: %s" % (what, e)) from None


def _json_object(text, what: str, keys) -> dict:
    obj = _json_load(text, what)
    if not isinstance(obj, dict):
        raise FormatError("%s: expected a JSON object" % what)
    for k in keys:
        if k not in obj:
            raise FormatError("%s: missing key %r" % (what, k))
    for k, want in (("protocol", "groth16"), ("curve", "bn128")):
        if k in obj and obj[k] != want:
            raise FormatError("%s: %s is %r, only %r is supported" % (what, k, obj[k], want))
    return obj


def _json_int(v, field: str, bound: int | None = None) -> int:
    """A decimal or 0x-hex string -> int; bound: the value must be below it (FQ_MODULUS for coordinates)."""
    import re
    if not isinstance(v, str) or not (re.fullmatch(r"[0-9]+", v) or re.fullmatch(r"0x[0-9a-fA-F]+", v)):
        raise FormatError("%s: %r is not a decimal or 0x-hex number string" % (field, v))
    x = int(v, 0) if v.startswith("0x") else int(v)
    if bound is not None and x >= bound:
        raise FormatError("%s: %d is not below the base-field modulus q" % (field, x))
    return x


def _json_list(v, n: int, field: str) -> list:
    if not isinstance(v, list) or len(v) != n:
        raise FormatError("%s: expected a list of %d items" % (field, n))
    return v


def _json_g1(v, field: str):
    x, y, z = (_json_int(c, "%s[%d]" % (field, i), FQ_MODULUS) for i, c in enumerate(_json_list(v, 3, field)))
    if z == 0:
        return None
    if z != 1:
        raise FormatError("%s: z = %d; only affine points (z = 1) and infinity (z = 0) are read" % (field, z))
    return (x, y)


def _json_fq2(v, field: str) -> tuple:
    return tuple(_json_int(c, "%s[%d]" % (field, i), FQ_MODULUS) for i, c in enumerate(_json_list(v, 2, field)))


def _json_g2(v, field: str):
    x, y, z = (_json_fq2(c, "%s[%d]" % (field, i)) for i, c in enumerate(_json_list(v, 3, field)))
    if z == (0, 0):
        return None
    if z != (1, 0):
        raise FormatError("%s: z = %s; only affine points (z = [1, 0]) and infinity (z = [0, 0]) are read" % (field, z))
    return (x, y)


def read_proof_json(text) -> SnarkjsProof:
    obj = _json_object(text, "proof.json", ("pi_a", "pi_b", "pi_c", "protocol", "curve"))
    return SnarkjsProof(_json_g1(obj["pi_a"], "pi_a"), _json_g2(obj["pi_b"], "pi_b"), _json_g1(obj["pi_c"], "pi_c"))


def read_public_json(text) -> list:
    """-> the public signals as ints (not reduced: a value >= r is the verifier's to reject)."""
    arr = _json_load(text, "public.json")
    if not isinstance(arr, list):
        raise FormatError("public.json: expected a JSON array")
    return [_json_int(v, "public[%d]" % i) for i, v in enumerate(arr)]


def read_vk_json(text) -> SnarkjsVerificationKey:
    obj = _json_object(text, "verification_key.json", ("protocol", "curve", "nPublic", "vk_alpha_1", "vk_beta_2", "vk_gamma_2",
                                                       "vk_delta_2", "vk_alphabeta_12", "IC"))
    n = obj["nPublic"]
    if isinstance(n, bool) or not isinstance(n, int) or n < 0:
        raise FormatError("nPublic: %r is not a non-negative integer" % (n,))
    ic = obj["IC"]
    if not isinstance(ic, list) or len(ic) != n + 1:
        raise FormatError("IC: %s points for nPublic = %d (expected %d)" % (len(ic) if isinstance(ic, list) else "no list of",
                                                                           n, n + 1))
    ab = [[_json_fq2(c, "vk_alphabeta_12[%d][%d]" % (h, k)) for k, c in enumerate(_json_list(half, 3, "vk_alphabeta_12[%d]" % h))]
          for h, half in enumerate(_json_list(obj["vk_alphabeta_12"], 2, "vk_alphabeta_12"))]
    return SnarkjsVerificationKey(n, _json_g1(obj["vk_alpha_1"], "vk_alpha_1"), _json_g2(obj["vk_beta_2"], "vk_beta_2"),
                                  _json_g2(obj["vk_gamma_2"], "vk_gamma_2"), _json_g2(obj["vk_delta_2"], "vk_delta_2"), ab,
                                  [_json_g1(p, "IC[%d]" % i) for i, p in enumerate(ic)])
