"""Test-side writer of prepared Powers-of-Tau files from a known (tau, alpha, beta), so that the ptau reader and the setup
from a ceremony can be exercised without a ceremony file.  The layout is the one distributed_groth16_b200.formats.PTau
reads (restated from snarkjs).  Every section is consistent: tau^i G1 (2^(power+1) - 1 points), tau^i G2, alpha tau^i G1,
beta tau^i G1 (2^power each), beta G2, zero contributions (section 7) and the Lagrange levels 12-15.  Level k is the
inverse NTT of the first 2^k powers, powers beyond the tau G1 section taken as zero -- which only touches the top level
(power + 1) of section 12.

`sections_oracle` computes everything with the pure-Python oracle (tiny powers only); `sections_gpu` uses the pinned GPU
building blocks (fr_powers, inverse NTT, fixed-base multiplication of the generators)."""
import struct

from artefact_writer import Q, container

ORDER = (1, 2, 3, 4, 5, 6, 7, 12, 13, 14, 15)


def _assemble(power, s2, s3, s4, s5, s6, s12, s13, s14, s15) -> dict:
    s1 = struct.pack("<I", 32) + Q.to_bytes(32, "little") + struct.pack("<II", power, power)
    return {1: s1, 2: s2, 3: s3, 4: s4, 5: s5, 6: s6, 7: struct.pack("<I", 0), 12: s12, 13: s13, 14: s14, 15: s15}


def sections_oracle(tau: int, alpha: int, beta: int, power: int) -> dict:
    from oracle import bn254 as o, layout
    n1, n = (1 << (power + 1)) - 1, 1 << power
    pw = lambda scale, cnt: [scale * pow(tau, i, o.R) % o.R for i in range(cnt)]
    g1 = lambda sc: layout.g1_to_arr([o.G1.mul(o.G1_GEN, s) for s in sc]).tobytes()
    g2 = lambda sc: layout.g2_to_arr([o.G2.mul(o.G2_GEN, s) for s in sc]).tobytes()

    def lag(scale, top):
        out = []
        for k in range(top + 1):
            out += o.intt([x if i < n1 else 0 for i, x in enumerate(pw(scale, 1 << k))])
        return out

    return _assemble(power, g1(pw(1, n1)), g2(pw(1, n)), g1(pw(alpha, n)), g1(pw(beta, n)), g2([beta]),
                     g1(lag(1, power + 1)), g2(lag(1, power)), g1(lag(alpha, power)), g1(lag(beta, power)))


def sections_gpu(net, tau: int, alpha: int, beta: int, power: int) -> dict:
    import torch
    from distributed_groth16_b200.groth16.setup import _fixed_base, _powers
    n1, n = (1 << (power + 1)) - 1, 1 << power
    pts = lambda sc, g2=False: _fixed_base(net, sc.contiguous(), g2).cpu().numpy().tobytes()

    def lag(scale, top):
        parts = []
        for k in range(top + 1):
            v = _powers(net, tau, scale, 1 << k)
            v[n1:] = 0
            parts.append(net.ntt_dev(v, inverse=True))
        return torch.cat(parts)

    return _assemble(power, pts(_powers(net, tau, 1, n1)), pts(_powers(net, tau, 1, n), True), pts(_powers(net, tau, alpha, n)),
                     pts(_powers(net, tau, beta, n)), pts(_powers(net, tau, beta, 1), True), pts(lag(1, power + 1)),
                     pts(lag(1, power), True), pts(lag(alpha, power)), pts(lag(beta, power)))


def ptau_bytes(secs: dict, magic: bytes = b"ptau") -> bytes:
    return container(magic, [(sid, secs[sid]) for sid in ORDER if sid in secs])


def write_ptau(path, secs: dict, magic: bytes = b"ptau"):
    with open(path, "wb") as f:
        f.write(ptau_bytes(secs, magic))
    return path
