"""The sharding kernels at every rank's parameters of worlds 1, 2, 4 and 8, against exact answers, on one GPU.

parallel.py's torch.distributed flows cannot run more than one rank per GPU (NCCL refuses two ranks on one device, and a CUDA
IPC handle cannot be opened in the process that made it), so the kernels they call are driven here one rank at a time with
the arguments rank g of P would pass:
  - b200zk_ntt_fr_batched_post_dev with every tuple of parallel.sharded_ntt / group.cu's sharded_ntt: the column step
    (b0 = g cg, alpha = 1) forward and inverse, and the shifted row step (b0 = g rl, beta = 1, gamma = rows, base_is_shift).
    Expected: mgpu_common.OracleBackend (the backend the gloo test runs parallel.py's host logic on) up to 2^9, the CPU twin
    it is pinned to (tests/test_oracle_batched_post.py) above;
  - b200zk_ntt_fr_fourstep_cols_p2p_dev, the column step fused with the exchange: all P ranks' kernels one after another,
    each storing into every rank's receive buffer (plain device buffers with a guard row on each side).  Each buffer must
    equal the exact four-step intermediate and the unfused path (batched post + the permute of parallel.sharded_ntt), and no
    guard word may change;
  - b200zk_msm_exchange_sum_dev, the peer-mailbox MSM exchange.  Before rank r's launch the test has already put every other
    rank's partial into rank r's mailbox and raised all 16 of its flags to `seq`, so the kernel never waits: its spin on
    the flags is NOT exercised here (that needs two kernels resident at once, i.e. real peers).  What is checked: the sum,
    the parity slot it reads, and that it writes its own partial and flag into slot [seq & 1][r] of every mailbox and
    nothing else;
  - b200zk_xyzz_sum_dev and b200zk_g1_sum_dev / b200zk_g2_sum_dev over count 0..8 and strides 1, 3, 6 (the prover's layout;
    xyzz_sum_dev refuses count 0).
Device outputs start as all-ones words, so an element no kernel writes cannot pass.  Then the input guards of the NTT entry
points: each refusal comes before any launch and leaves the context usable."""
import ctypes
import random

import numpy as np
import pytest
import torch

import arith_oracle as ao
from mgpu_common import OracleBackend
from oracle import bn254 as o

pytestmark = pytest.mark.gpu

ERR_DOMAIN, ERR_ARG = 2, 4
WORLDS = (1, 2, 4, 8)
M64 = (1 << 64) - 1


def _c_vp(x):
    from distributed_groth16_b200._native import c_vp
    return c_vp(x.data_ptr() if isinstance(x, torch.Tensor) else x)


def _dev(net, arr):
    return torch.from_numpy(np.ascontiguousarray(arr, dtype=np.uint64).view(np.int64)).to(net._dev())


def _host(t) -> np.ndarray:
    return t.cpu().numpy().view(np.uint64)


def _ones(net, n_words):
    return torch.full((n_words,), -1, dtype=torch.int64, device=net._dev())


def _batched_post(net, x, log_t, batch, inverse, log_base, shift, b0, alpha, beta, gamma):
    out = _ones(net, (batch << log_t) * 4)
    net.check(net._lib.b200zk_ntt_fr_batched_post_dev(net._h, 0, _c_vp(x), _c_vp(out), log_t, batch, int(inverse), log_base, int(shift),
                                                      b0, alpha, beta, gamma))
    return out


def _expect_post(cref, x, log_t, batch, inverse, log_base, shift, b0, alpha, beta, gamma):
    if (batch << log_t) <= 1 << 9:
        return OracleBackend().batched_ntt_post(torch.from_numpy(x.view(np.int64)), log_t, batch, inverse, log_base=log_base, shift=shift,
                                                b0=b0, alpha=alpha, beta=beta, gamma=gamma).numpy().view(np.uint64).reshape(-1, 4)
    return cref.ntt_batched_post(x, log_t, batch, inverse, log_base, shift, b0, alpha, beta, gamma)


# ---- batched post at every rank's tuple ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_m", [4, 9, 16, 17, 18])
def test_batched_post_at_every_ranks_sharded_ntt_tuples(net, cref, log_m):
    log_rows, log_cols = (log_m + 1) // 2, log_m // 2
    rows, cols = 1 << log_rows, 1 << log_cols
    for P in WORLDS:
        if cols < P:
            continue
        cg, rl = cols // P, rows // P
        for g in range(P):
            what = "log_m=%d P=%d g=%d" % (log_m, P, g)
            steps = [(log_rows, cg, inv, log_m, False, g * cg, 1, 0, 0) for inv in (False, True)]          # column step
            steps.append((log_cols, rl, True, log_m + 1, True, g * rl, 0, 1, rows))                        # shifted row step (h)
            for args in steps:
                x = cref.fr_generate(0x5EA0 + 131 * log_m + 17 * P + g, args[1] << args[0])
                got = _host(_batched_post(net, _dev(net, x), *args)).reshape(-1, 4)
                assert (got == _expect_post(cref, x, *args)).all(), (what, args)


# ---- the fused exchange ---------------------------------------------------------------------------------------------------------
# (log_rows, log_cols): one- and two-pass column transforms (log_rows > 8), rows >= cols (the inverse of h) and rows < cols (its
# forward), cols / P = 1, 2 (untiled remote stores) and >= 4 (batch-tiled)
P2P_GEOMETRY = [(3, 3), (5, 5), (4, 9), (9, 3), (9, 8), (10, 4)]


@pytest.mark.parametrize("inverse", [False, True], ids=["fwd", "inv"])
@pytest.mark.parametrize("geom", P2P_GEOMETRY, ids=lambda g: "rows2^%d_cols2^%d" % g)
def test_fourstep_cols_p2p_every_rank_into_guarded_buffers(net, cref, geom, inverse):
    from distributed_groth16_b200._native import c_vp
    log_rows, log_cols = geom
    log_n = log_rows + log_cols
    rows, cols = 1 << log_rows, 1 << log_cols
    X = cref.fr_generate(0xF5 + 7 * log_n + inverse, cols * rows)           # column n2 = X[n2 * rows : (n2 + 1) * rows]
    # the exact intermediate: Y[n2][k1] = NTT_rows(column n2)[k1] w_N^(+-n2 k1) (inverse: also 1 / rows)
    Y = cref.ntt_batched_post(X, log_rows, cols, inverse, log_n, False, 0, 1, 0, 0).reshape(cols, rows, 4)
    for P in WORLDS:
        if cols < P or rows < P:
            continue
        cg, rl = cols // P, rows // P
        body, guard = rl * cols * 4, cols * 4                              # words: rl rows of cols elements, one row each side
        bufs = [_ones(net, body + 2 * guard) for _ in range(P)]
        for b in bufs:
            b[guard + body:] = 0x5A5A5A5A5A5A5A5A                           # the two guard zones differ from each other and the fill
            b[:guard] = 0x0123456789ABCDEF
        guard_before = [(_host(b[:guard]).copy(), _host(b[guard + body:]).copy()) for b in bufs]
        ptrs = (c_vp * P)(*[c_vp(b.data_ptr() + guard * 8) for b in bufs])
        ins = [_dev(net, X[g * cg * rows:(g + 1) * cg * rows]) for g in range(P)]
        for g in range(P):
            net.check(net._lib.b200zk_ntt_fr_fourstep_cols_p2p_dev(net._h, 0, _c_vp(ins[g]), ptrs, P, log_rows, cg.bit_length() - 1, log_n,
                                                                   g * cg, int(inverse)))
        # the unfused path: batched post per rank, then parallel.sharded_ntt's all-to-all permute
        ys = [_batched_post(net, ins[g], log_rows, cg, inverse, log_n, False, g * cg, 1, 0, 0) for g in range(P)]
        sends = [y.reshape(cg, P, rl, 4).permute(1, 0, 2, 3) for y in ys]
        for g in range(P):
            what = "P=%d g=%d" % (P, g)
            got = _host(bufs[g][guard:guard + body]).reshape(rl, cols, 4)
            assert (got == Y[:, g * rl:(g + 1) * rl].transpose(1, 0, 2)).all(), what
            unfused = torch.stack([sends[q][g] for q in range(P)]).permute(2, 0, 1, 3).reshape(rl, cols, 4)
            assert (got == _host(unfused).reshape(rl, cols, 4)).all(), what
            lo, hi = guard_before[g]
            assert (_host(bufs[g][:guard]) == lo).all() and (_host(bufs[g][guard + body:]) == hi).all(), what + ": guard zone written"


# ---- the mailbox exchange ---------------------------------------------------------------------------------------------------------
SLOT, MAXP, BOX = 256, 8, 8192
FLAGS = 2 * MAXP * SLOT                      # byte offset of the [2][8] u64 flags


def _pts(G, k, seed):
    rnd = random.Random(seed)
    return [G.c.mul(G.gen, rnd.randrange(1, o.R)) for _ in range(k)]


def _lam(G, rnd):
    if G is ao.G1:
        return rnd.randrange(2, o.P)
    return (rnd.randrange(o.P), rnd.randrange(1, o.P))


def _xyzz_bytes(G, pt, rnd) -> bytes:
    """pt (None = identity) as a non-normalised XYZZ record: (x l^2, y l^3, l^2, l^3) for a random l."""
    return np.array(G.xyzz_w(pt, _lam(G, rnd)), dtype=np.uint64).tobytes()


def _sum(G, pts):
    acc = None
    for p in pts:
        acc = G.c.add(acc, p)
    return acc


def _partials(G, P, seq):
    """P partials with two equal ones, a cancelling pair and the identity (as far as P allows)."""
    A, B, C, D, E = _pts(G, 5, 0xE8 + seq)
    odd = [A, A, B, G.c.neg(B), None, C, D, E]
    even = [B, G.c.neg(B), None, A, A, C, D, E]
    return (odd if seq & 1 else even)[:P]


@pytest.mark.parametrize("seq", [5, 6], ids=["seq_odd", "seq_even"])
@pytest.mark.parametrize("g2", [False, True], ids=["G1", "G2"])
def test_msm_exchange_sum_every_rank(net, g2, seq):
    G = ao.G2 if g2 else ao.G1
    W = 16 if g2 else 8
    par = seq & 1
    rnd = random.Random(0xB0C5 + seq + 2 * g2)
    other_parity = _pts(G, 1, 0xF00 + seq)[0]
    for P in WORLDS:
        parts = _partials(G, P, seq)
        recs = [_xyzz_bytes(G, p, rnd) for p in parts]
        want = G.pt_view(_sum(G, parts))
        for r in range(P):
            what = "P=%d rank=%d" % (P, r)
            boxes = []
            for q in range(P):
                raw = bytearray(rnd.randbytes(BOX))                   # every byte the kernel must leave alone is random
                for g in range(MAXP):
                    off = ((1 - par) * MAXP + g) * SLOT
                    raw[off:off + len(recs[0])] = _xyzz_bytes(G, other_parity, rnd)    # the other parity: a valid, wrong point
                if q == r:
                    for g in range(P):
                        if g != r:
                            off = (par * MAXP + g) * SLOT
                            raw[off:off + len(recs[g])] = recs[g]
                    raw[FLAGS:FLAGS + 16 * 8] = np.full(16, seq, dtype=np.uint64).tobytes()   # no flag the kernel can read is < seq
                boxes.append(bytes(raw))
            dboxes = [torch.from_numpy(np.frombuffer(b, dtype=np.uint8).copy()).to(net._dev()) for b in boxes]
            part = torch.from_numpy(np.frombuffer(recs[r], dtype=np.uint8).copy()).to(net._dev())
            out = _ones(net, W + 1)
            ptrs = (ctypes.c_void_p * P)(*[b.data_ptr() for b in dboxes])
            net.check(net._lib.b200zk_msm_exchange_sum_dev(net._h, 0, int(g2), _c_vp(part), ptrs, P, r, seq, _c_vp(out)))
            res = [int(w) for w in _host(out)]
            assert res[W] == (1 if want == ("inf",) else 0), what
            assert G.aff_view(res[:W]) == want, what
            for q in range(P):
                after = bytearray(_host(dboxes[q].view(torch.int64)).tobytes())
                exp = bytearray(boxes[q])
                off = (par * MAXP + r) * SLOT
                exp[off:off + len(recs[r])] = recs[r]
                exp[FLAGS + (par * MAXP + r) * 8:FLAGS + (par * MAXP + r + 1) * 8] = int(seq).to_bytes(8, "little")
                assert after == exp, what + ": mailbox %d" % q


# ---- point sums at every count and stride ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("g2", [False, True], ids=["G1", "G2"])
def test_xyzz_and_point_sums_every_count_and_stride(net, g2):
    G = ao.G2 if g2 else ao.G1
    W = 16 if g2 else 8
    rnd = random.Random(0x5C + g2)
    A, B, C, D = _pts(G, 4, 0x5D + g2)
    filler = _pts(G, 1, 0x5E + g2)[0]
    pool = [A, A, B, G.c.neg(B), None, C, D, G.c.neg(A)]           # P + P, P - P, an identity, and -A cancelling the A + A
    for count in range(9):
        for stride in (1, 3, 6):
            pts = [pool[(i + count) % len(pool)] for i in range(count)]
            recs = [_xyzz_bytes(G, filler, rnd) for _ in range(max(count * stride, 1))]   # the skipped records: valid, wrong points
            for i, p in enumerate(pts):
                recs[i * stride] = _xyzz_bytes(G, p, rnd)
            d_in = torch.from_numpy(np.frombuffer(b"".join(recs), dtype=np.uint8).copy()).to(net._dev())
            want = G.pt_view(_sum(G, pts))
            out = _ones(net, 2 * W)
            rc = net._lib.b200zk_xyzz_sum_dev(net._h, 0, int(g2), _c_vp(d_in), count, stride, _c_vp(out))
            if count == 0:                                          # an empty sum is refused; the output stays untouched
                assert rc == ERR_ARG and (_host(out) == np.uint64(M64)).all()
            else:
                net.check(rc)
                view = G.xyzz_view([int(w) for w in _host(out)])
                assert view == want, (count, stride, view[0])
            if stride == 1:
                aff, inf = net.sum_points_dev(d_in, count, g2=g2)
                assert inf == (want == ("inf",)) and G.aff_view([int(w) for w in aff]) == want, (count, "sum_dev")


# ---- input guards of the NTT entry points -----------------------------------------------------------------------------------
def _refused(net, call, code, text):
    before = net.launch_count()
    assert call() == code
    assert text in net._lib.b200zk_last_error(net._h).decode()
    assert net.launch_count() == before


def _still_works(net, cref):
    x = cref.fr_generate(0x57, 1 << 10)
    assert (_host(net.ntt_dev(_dev(net, x).reshape(-1, 4))).reshape(-1, 4) == cref.ntt(x)).all()


def test_batched_post_refusals_before_any_launch(net, cref):
    buf = _ones(net, 4 << 12)
    p = _c_vp(buf)
    f = net._lib.b200zk_ntt_fr_batched_post_dev
    # base_is_shift with log_base = 0 has no shift table (it would ask for the plan of log_n = -1)
    _refused(net, lambda: f(net._h, 0, p, p, 4, 1, 1, 0, 1, 0, 0, 1, 0), ERR_DOMAIN, "log_base >= 1")
    # largest exponent (batch - 1 + b0)(alpha k_max + beta) + gamma k_max must be below 2^log_base (shift: 2^(log_base - 1))
    for args in [(4, 19, 0, 8, 0, 0, 1, 0, 0),                 # 18 x 15 = 270 >= 2^8
                 (4, 1, 0, 8, 0, 18, 1, 0, 0),                 # the same through b0
                 (4, 2, 1, 9, 1, 15, 0, 1, 16),                # shift table of 2^8: 16 x 1 + 16 x 15 = 256
                 (3, 1, 0, 5, 0, 1 << 63, 1, 0, 0),            # b0 near 2^64
                 (3, 4, 0, 5, 0, 0, 1 << 62, 0, 0),            # alpha near 2^64
                 (3, 1, 0, 5, 0, 0, 0, 0, (1 << 64) - 1),      # gamma = 2^64 - 1
                 (3, 1, 0, 5, 0, (1 << 64) - 1, 0, 1 << 63, 0)]:   # (b0)(beta) past 2^127
        _refused(net, lambda: f(net._h, 0, p, p, *args), ERR_ARG, "exceeds the table")
    # the edges themselves run: largest exponent 2^log_base - 1 = 17 x 15, and 2^(log_base - 1) - 1 = 16 + 15 x 15 for the shift
    x = cref.fr_generate(0x58, 18 << 4)
    for args in [(4, 18, False, 8, False, 0, 1, 0, 0), (4, 2, True, 9, True, 15, 0, 1, 15)]:
        got = _host(_batched_post(net, _dev(net, x[:args[1] << 4]), *args)).reshape(-1, 4)
        assert (got == cref.ntt_batched_post(x[:args[1] << 4], *args)).all(), args
    _still_works(net, cref)


def test_fourstep_cols_p2p_refusals_before_any_launch(net, cref):
    from distributed_groth16_b200._native import c_vp
    buf = _ones(net, 4 << 12)
    ptrs = (c_vp * 2)(_c_vp(buf), _c_vp(buf))
    f = net._lib.b200zk_ntt_fr_fourstep_cols_p2p_dev
    # log_n < log_rows: no column at all (log_n - log_rows would wrap)
    _refused(net, lambda: f(net._h, 0, _c_vp(buf), ptrs, 2, 5, 0, 4, 0, 0), ERR_ARG, "log_n < log_rows")
    # columns [col0, col0 + 2^log_cols_local) past the 2^(log_n - log_rows) columns of a receive row
    for log_cols_local, col0 in ((2, 1), (3, 0), (0, 4), (0, (1 << 64) - 1), (40, 0)):
        _refused(net, lambda: f(net._h, 0, _c_vp(buf), ptrs, 2, 4, log_cols_local, 6, col0, 0), ERR_ARG, "run past the receive rows")
    _still_works(net, cref)
