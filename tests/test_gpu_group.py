"""`b200zk_group_*` (csrc/group.cu): the sharded hot path behind single C calls, vs the oracle and vs the single-GPU calls.

Worlds:
  - world1: one context on GPU 0.  Every rank-dependent quantity is 0 or 1 there, so a wrong offset cannot show.
  - emu2 / emu4 / emu8: `Group([0] * P)`, P independent contexts on GPU 0.  `b200zk_group_create` skips peer enabling for
    repeated device ids, so all of group.cu's index arithmetic (shard cuts, column offsets, gather offsets), the fused remote
    stores of the four-step transform (same-device stores here), the cross-context event barriers and the double-buffered
    receive buffers run at P ranks.  Not covered: NVLink transport and event ordering across real devices.
  - all: every GPU of the box (2, 4 or 8); skips on a single-GPU box.

Expected values are the CPU twin's (`cref`), computed once per input and shared by the worlds."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ERR_DOMAIN, ERR_ARG = 2, 4
_memo = {}


def _cached(key, fn):
    if key not in _memo:
        _memo[key] = fn()
    return _memo[key]


def _worlds():
    import torch
    n = torch.cuda.device_count()
    out = [1]
    w = 2
    while w <= min(n, 8):
        out.append(w)
        w *= 2
    return out


@pytest.fixture(scope="module", params=["world1", "emu2", "emu4", "emu8", "all"])
def group(request):
    from distributed_groth16_b200.group import Group
    if request.param == "all":
        worlds = _worlds()
        if worlds[-1] == 1:
            pytest.skip("needs >= 2 GPUs (run with gpurun --gpus N)")
        devices = list(range(worlds[-1]))
    elif request.param == "world1":
        devices = [0]
    else:
        devices = [0] * int(request.param[3:])
    g = Group(devices)
    yield g
    g.close()


def _launches(grp) -> int:
    lib = grp._lib
    return sum(int(lib.b200zk_launch_count(lib.b200zk_group_ctx(grp._h, r))) for r in range(grp.size()))


def _refused(grp, fn, code, text):
    """fn() must return `code` with `text` in the group's last error, before any kernel launch on any rank."""
    before = _launches(grp)
    rc = fn()
    assert rc == code, (rc, code)
    assert text in grp._lib.b200zk_group_last_error(grp._h).decode()
    assert _launches(grp) == before


def _neg_fr(s):
    from oracle import layout
    return layout.fr_to_arr([-v for v in layout.arr_to_fr(s)])


# ---- d_msm ----------------------------------------------------------------------------------------------------------------
def _msm_inputs(g2, n, P, kind):
    """kind 'plain': random, with a zero scalar, an infinity base and a duplicate base from n >= 5 on;
    'equal': every shard of P holds the same pairs (all partials equal: the gather-and-sum doubles);
    'cancel': shard 2k + 1 holds shard 2k's bases with negated scalars (partials cancel in pairs: the sum is infinity)."""
    from oracle import cref
    gen = cref.g2_generate if g2 else cref.g1_generate
    if kind == "plain":
        if n >= (1 << 18):        # distinct bases up to 2^14, tiled: the twin's MSM does not care, generation stays cheap
            bases = np.tile(gen(0xB2000011, 1 << 14), (n // (1 << 14) + 1, 1))[:n].copy()
        else:
            bases = gen(0xB2000001 + g2, n)
        scalars = cref.fr_generate(0xB2000002 + n, n)
        if n >= 5:
            scalars[0] = 0
            bases[1] = 0
            bases[3] = bases[2]
        return bases, scalars
    k = n // P
    b, s = gen(0xB2000021 + g2, k), cref.fr_generate(0xB2000022, k)
    if kind == "equal":
        return np.tile(b, (P, 1)), np.tile(s, (P, 1))
    return np.tile(b, (P, 1)), np.concatenate([s if g % 2 == 0 else _neg_fr(s) for g in range(P)])


def _msm_expect(g2, n, P, kind):
    from oracle import cref
    def f():
        bases, scalars = _msm_inputs(g2, n, P, kind)
        return (cref.msm_g2 if g2 else cref.msm_g1)(bases, scalars)
    return _cached(("msm", g2, n, P if kind != "plain" else 0, kind), f)


def test_group_d_msm_matches_oracle(group):
    """G1 and G2, n in {0, 1, P - 1, P, P + 1, 1000, 2^14}: shards of length 0 (n < P) and uneven cuts; for G1 also 2^21 + 3, where
    every shard of up to 8 ranks has at least 2^18 pairs and stages in five parts.  Then all-equal and pairwise-cancelling
    shard partials."""
    for g2 in (False, True):
        _check_d_msm(group, g2)


def _check_d_msm(group, g2):
    P = group.size()
    sizes = sorted({0, 1, P - 1, P, P + 1, 1000, 1 << 14} | (set() if g2 else {(1 << 21) + 3}))
    w = 16 if g2 else 8
    for n in sizes:
        if n == 0:
            got = group.d_msm(np.zeros((0, w), dtype=np.uint64), np.zeros((0, 4), dtype=np.uint64), g2=g2)
            assert got.infinity
            continue
        bases, scalars = _msm_inputs(g2, n, P, "plain")
        exp, inf = _msm_expect(g2, n, P, "plain")
        got = group.d_msm(bases, scalars, g2=g2)
        assert got.infinity == inf and (got.infinity or (got.limbs == exp).all()), n
    for kind in ("equal", "cancel"):
        n = 40 * P
        bases, scalars = _msm_inputs(g2, n, P, kind)
        exp, inf = _msm_expect(g2, n, P, kind)
        assert inf == (kind == "cancel" and P > 1)
        got = group.d_msm(bases, scalars, g2=g2)
        assert got.infinity == inf and (got.infinity or (got.limbs == exp).all()), kind


def test_group_d_msm_length_mismatch_is_the_reference_error(group, cref):
    from distributed_groth16_b200 import MpcNetError
    with pytest.raises(MpcNetError) as e:
        group.d_msm(cref.g1_generate(1, 7), cref.fr_generate(1, 5))
    assert e.value.kind == "Generic" and e.value.message == "5"          # arkworks Err(min_len) through `?`, dmsm/mod.rs:82


# ---- d_fft / d_ifft -------------------------------------------------------------------------------------------------------
def _ntt_expect(log_n, inverse):
    from oracle import cref
    return _cached(("ntt", log_n, inverse), lambda: cref.ntt(cref.fr_generate(0xB2000003 + log_n, 1 << log_n), inverse=inverse))


# log_rows = ceil(log_n / 2) > 8 (log_n >= 17) makes the column transform two-pass, and its inverse plan folds 1/N into the
# first pass; cols / P = 1 or 2 takes the untiled remote stores, >= 4 the batch-tiled ones
FFT_LOGS = (1, 2, 3, 6, 7, 16, 17, 18, 20, 22)


def test_group_d_fft_and_d_ifft_match_oracle(group, cref):
    P = group.size()
    for log_n in FFT_LOGS:
        x = cref.fr_generate(0xB2000003 + log_n, 1 << log_n)
        if (1 << (log_n // 2)) < P:
            for inverse in (0, 1):
                buf = x.copy()
                _refused(group, lambda: group._lib.b200zk_group_ntt_fr(group._h, buf.ctypes.data, log_n, inverse), ERR_ARG,
                         "transform too small for this many GPUs")
                assert (buf == x).all()
            continue
        assert (group.d_fft(x) == _ntt_expect(log_n, False)).all(), log_n
        assert (group.d_ifft(x) == _ntt_expect(log_n, True)).all(), log_n


# ---- h ----------------------------------------------------------------------------------------------------------------
H_LOGS = (2, 6, 11, 17, 18, 20)


def _h_inputs(log_m):
    from oracle import cref
    return tuple(cref.fr_generate(s + log_m, 1 << log_m) for s in (21, 22, 23))


def test_group_h_matches_oracle(group, cref):
    P = group.size()
    for log_m in H_LOGS:
        a, b, c = _h_inputs(log_m)
        if (1 << (log_m // 2)) < P:
            out = np.zeros_like(a)
            _refused(group, lambda: group._lib.b200zk_group_h_circom(group._h, a.ctypes.data, b.ctypes.data, c.ctypes.data, log_m,
                                                                      out.ctypes.data), ERR_ARG, "domain too small for this many GPUs")
            continue
        want = _cached(("h", log_m), lambda: cref.h_circom(a, b, c))
        assert (group.h(a, b, c) == want).all(), log_m


def test_group_h_refuses_a_domain_past_2_to_the_27(group):
    """2m must fit the 2^28 subgroup; the refusal comes before the inputs are read, so 1-element buffers stand in."""
    one = np.zeros((1, 4), dtype=np.uint64)
    for log_m in (28, 40):
        _refused(group, lambda: group._lib.b200zk_group_h_circom(group._h, one.ctypes.data, one.ctypes.data, one.ctypes.data, log_m,
                                                                  one.ctypes.data), ERR_DOMAIN, "2m exceeds the 2^28 subgroup")
    assert (group.d_fft(np.tile(one, (64, 1))) == 0).all()


# ---- the group prover -------------------------------------------------------------------------------------------------------
# (name, m, n_vars, n_inputs): n_vars not divisible by 2, 4 or 8; n_inputs above one shard; n_inputs = n_vars (no L query: every
# L shard has length 0); 100 L rows (shards below 64 rows: generic MSM) next to 500 a / b rows (tables); m = 2^18 (two-pass
# column transforms in the h pipeline)
PROVE_CASES = [
    ("m4096_nvars3001", 1 << 12, 3001, 3),
    ("inputs_past_one_shard", 1 << 12, 1003, 700),
    ("no_l_query", 1 << 12, 300, 300),
    ("small_and_table_shards", 1 << 12, 600, 500),
    ("m2^18", 1 << 18, 5003, 5),
]


def _instance(m, n_vars, n_inputs):
    from oracle import cref
    from distributed_groth16_b200._constants import FR_ONE_MONT
    def f():
        sd = n_vars * 7 + m
        aq, b1, hq = cref.g1_generate(sd + 1, n_vars), cref.g1_generate(sd + 2, n_vars), cref.g1_generate(sd + 5, m)
        lq = cref.g1_generate(sd + 4, n_vars - n_inputs)
        b2, vk1, vk2 = cref.g2_generate(sd + 3, n_vars), cref.g1_generate(sd + 6, 3), cref.g2_generate(sd + 7, 2)
        z = cref.fr_generate(sd + 8, n_vars)
        z[0] = np.array(FR_ONE_MONT, dtype=np.uint64)
        a, b, c = (cref.fr_generate(sd + k, m) for k in (9, 10, 11))
        return dict(aq=aq, b1=b1, b2=b2, lq=lq, hq=hq, vk1=vk1, vk2=vk2, z=z, a=a, b=b, c=c, n_inputs=n_inputs)
    return _cached(("inst", m, n_vars, n_inputs), f)


def _rs(rs):
    from oracle import layout
    return tuple(layout.fr_to_arr([v])[0] for v in rs)


def _want_proof(net, m, n_vars, n_inputs, rs):
    """The CPU twin's proof bytes; the single-GPU prover is checked against them once per instance."""
    from oracle import cref
    from distributed_groth16_b200.groth16 import ProvingKey, prove
    def f():
        I = _instance(m, n_vars, n_inputs)
        r, s = _rs(rs)
        vk = np.concatenate([I["vk1"].reshape(-1), I["vk2"].reshape(-1)])
        h = _cached(("h_inst", m, n_vars, n_inputs), lambda: cref.h_circom(I["a"], I["b"], I["c"]))
        want = cref.groth16_prove(I["aq"], I["b1"], I["b2"], I["lq"], I["hq"], vk, n_inputs, I["z"], h, r, s, mirror_bg1=False)
        pk = ProvingKey(net, I["aq"], I["b1"], I["b2"], I["lq"], I["hq"], n_inputs, I["vk1"][0], I["vk1"][1], I["vk1"][2], I["vk2"][0],
                        I["vk2"][1])
        single = prove.create_proof(pk, I["z"], I["a"], I["b"], I["c"], r, s)
        pk.free()
        assert single == want, "single-GPU prover"
        return want
    return _cached(("proof", m, n_vars, n_inputs, rs), f)


def _group_prove(group, m, n_vars, n_inputs, rs):
    from distributed_groth16_b200.group import GroupProvingKey
    I = _instance(m, n_vars, n_inputs)
    gpk = GroupProvingKey(group, I["aq"], I["b1"], I["b2"], I["lq"], I["hq"], n_inputs, I["vk1"][0], I["vk1"][1], I["vk1"][2], I["vk2"][0],
                          I["vk2"][1])
    try:
        return gpk.create_proof(I["z"], I["a"], I["b"], I["c"], *_rs(rs)), gpk.table_bytes
    finally:
        gpk.free()


@pytest.mark.parametrize("rs", [(0, 0), (777, 999)])
def test_group_prove_equals_single_gpu_prover_and_oracle(group, net, rs):
    _check_prove(group, net, PROVE_CASES[0], rs)


@pytest.mark.parametrize("rs", [(0, 0), (777, 999)], ids=["rs0", "rs"])
@pytest.mark.parametrize("case", PROVE_CASES[1:], ids=[c[0] for c in PROVE_CASES[1:]])
def test_group_prove_shard_shapes_equal_single_gpu_prover_and_oracle(group, net, case, rs):
    _check_prove(group, net, case, rs)


def _check_prove(group, net, case, rs):
    _, m, n_vars, n_inputs = case
    want = _want_proof(net, m, n_vars, n_inputs, rs)
    got, table_bytes = _group_prove(group, m, n_vars, n_inputs, rs)
    assert table_bytes > 0
    assert got == want


def test_group_prove_without_tables(group, net, monkeypatch):
    """B200ZK_PK_TABLES=0 (read by every upload): every shard runs the generic MSM, same bytes."""
    monkeypatch.setenv("B200ZK_PK_TABLES", "0")
    for case in PROVE_CASES[:2]:
        _, m, n_vars, n_inputs = case
        got, table_bytes = _group_prove(group, m, n_vars, n_inputs, (777, 999))
        assert table_bytes == 0
        assert got == _want_proof(net, m, n_vars, n_inputs, (777, 999)), case[0]


def test_group_repeated_calls_on_one_group(group, net, cref):
    """One fresh group: transforms of 2^6, 2^20, 2^6, 2^20 (the receive buffers grow, then alternate), an h (six transforms), a
    proof and a transform again, each checked."""
    from distributed_groth16_b200.group import Group
    P = group.size()
    g = Group(group.devices)
    try:
        for log_n in (6, 20, 6, 20):
            x = cref.fr_generate(0xB2000003 + log_n, 1 << log_n)
            assert (g.d_fft(x) == _ntt_expect(log_n, False)).all(), log_n
        a, b, c = _h_inputs(11)
        assert (g.h(a, b, c) == _cached(("h", 11), lambda: cref.h_circom(a, b, c))).all()
        _, m, n_vars, n_inputs = PROVE_CASES[0]
        assert _group_prove(g, m, n_vars, n_inputs, (777, 999))[0] == _want_proof(net, m, n_vars, n_inputs, (777, 999))
        x = cref.fr_generate(0xB2000003 + 16, 1 << 16)
        assert (g.d_ifft(x) == _ntt_expect(16, True)).all()
        assert g.size() == P
    finally:
        g.close()


# ---- refusals -----------------------------------------------------------------------------------------------------------------
def test_group_create_refuses_bad_sizes():
    from distributed_groth16_b200 import _native
    from distributed_groth16_b200._native import c_vp
    lib = _native.lib()
    for n in (0, 3, 9, 16):
        devs = (ctypes.c_int * max(n, 1))(*([0] * max(n, 1)))
        h = c_vp()
        assert lib.b200zk_group_create(devs, n, ctypes.byref(h)) == ERR_ARG, n
        assert not h.value, n


def test_group_prove_refuses_a_key_sharded_for_another_group(net):
    from distributed_groth16_b200.group import Group, GroupProvingKey
    _, m, n_vars, n_inputs = PROVE_CASES[0]
    I = _instance(m, n_vars, n_inputs)
    g2, g4 = Group([0, 0]), Group([0] * 4)
    try:
        gpk = GroupProvingKey(g2, I["aq"], I["b1"], I["b2"], I["lq"], I["hq"], n_inputs, I["vk1"][0], I["vk1"][1], I["vk1"][2],
                              I["vk2"][0], I["vk2"][1])
        r, s = _rs((777, 999))
        out = (ctypes.c_uint8 * 128)()
        p = lambda v: v.ctypes.data
        _refused(g4, lambda: g4._lib.b200zk_group_groth16_prove(g4._h, gpk._h, p(I["z"]), p(I["a"]), p(I["b"]), p(I["c"]), p(r), p(s), out),
                 ERR_ARG, "proving key was sharded for a different group")
        assert bytes(out) == bytes(128)
        x = np.asarray(_instance(m, n_vars, n_inputs)["a"])
        from oracle import cref
        assert (g4.d_fft(x) == cref.ntt(x)).all()                     # the refused group still works
        assert gpk.create_proof(I["z"], I["a"], I["b"], I["c"], r, s) == _want_proof(net, m, n_vars, n_inputs, (777, 999))
        gpk.free()
    finally:
        g4.close()
        g2.close()
