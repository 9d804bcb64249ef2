"""Powers-of-Tau files for phase 2 on the GPU: snarkjs `powersoftau prepare phase2` and the Lagrange part of
`powersoftau verify`.

`zkey new` (circom.zkey_new) reads a circuit's query points from the Lagrange sections 12-15 of a prepared ceremony file.
A phase-1 ceremony ends with the tau-power sections only; preparing it computes, for every domain 2^k the file supports,
the Lagrange basis in the exponent: level k of section 12 / 13 / 14 / 15 is the inverse NTT of the first 2^k points of
section 2 / 3 / 4 / 5 (tau^i G1, tau^i G2, alpha tau^i G1, beta tau^i G1), levels 0..power + 1 in section 12 (the missing
last tau power of its top level taken as infinity) and 0..power in the others.  Each level is one call of
b200zk_points_intt_dev: an FFT whose elements are curve points, so every twiddle product is a full scalar multiplication
-- the whole cost of the step.

The check needs no toxic waste: for random 128-bit rho, sum_j rho_j tau-points_j == sum_i NTT(rho)_i L_i exactly when L is
the inverse NTT of the tau points (up to a chance of about 2^-128), evaluated with the existing MSM and field NTT."""
from __future__ import annotations

import os
from dataclasses import dataclass, field

import numpy as np

from .. import formats
from .._native import c_vp

# Lagrange section -> (tau section, G2?, levels above power)
_SECTIONS = {12: (2, False, 1), 13: (3, True, 0), 14: (4, False, 0), 15: (5, False, 0)}


def points_intt(net, points, g2: bool = False, out=None):
    """out[i] = n^-1 sum_j w_n^(-i j) points[j] on the device (b200zk_points_intt_dev); points: CUDA int64 (2^k, 8 | 16)
    affine Montgomery limbs.  out may be points."""
    import torch
    points = points.contiguous()
    n = int(points.shape[0])
    log_n = n.bit_length() - 1
    if n == 0 or (1 << log_n) != n:
        raise ValueError("points_intt: the number of points must be a power of two, got %d" % n)
    if out is None:
        out = torch.empty_like(points)
    net.check(net._lib.b200zk_points_intt_dev(net._h, 0, int(g2), c_vp(points.data_ptr()), log_n, c_vp(out.data_ptr())))
    return out


def points_ntt(net, points, g2: bool = False, out=None):
    """out[i] = sum_j w_n^(i j) points[j] on the device (b200zk_points_ntt_dev), the unscaled forward transform of
    points_intt; points: CUDA int64 (2^k, 8 | 16) affine Montgomery limbs.  out may be points."""
    import torch
    points = points.contiguous()
    n = int(points.shape[0])
    log_n = n.bit_length() - 1
    if n == 0 or (1 << log_n) != n:
        raise ValueError("points_ntt: the number of points must be a power of two, got %d" % n)
    if out is None:
        out = torch.empty_like(points)
    net.check(net._lib.b200zk_points_ntt_dev(net._h, 0, int(g2), c_vp(points.data_ptr()), log_n, c_vp(out.data_ptr())))
    return out


def _tau_level(pt: formats.PTau, sid: int, level: int) -> np.ndarray:
    """The first 2^level points of the tau section behind Lagrange section sid, infinity (all-zero) past its end."""
    src, g2, _ = _SECTIONS[sid]
    w, n = 16 if g2 else 8, 1 << level
    have = min(n, (2 << pt.power) - 1)            # short of n only at the top level of section 12
    pts = pt.points(src, 0, have, w)
    if have < n:
        pts = np.concatenate([pts, np.zeros((n - have, w), dtype=np.uint64)])
    return pts


def prepare_phase2(net, src_path: str, dst_path: str, timings: dict | None = None) -> None:
    """snarkjs `powersoftau prepare phase2 <src> <dst>` on the GPU: write to dst_path the prepared ceremony file of
    src_path (formats.PreparedPTauWriter: sections 1-7 restated / copied, Lagrange sections 12-15 appended level by level
    as the device produces them).  src_path may already be prepared: its sections 12-15 are ignored and recomputed.
    dst_path must not be src_path (the input is memory-mapped while the output is written).  `timings`, if given,
    receives seconds spent in the transform (device), in transfers and in file writes."""
    import time
    if os.path.exists(dst_path) and os.path.samefile(src_path, dst_path):
        raise ValueError("prepare_phase2: the output %r is the input file" % dst_path)
    t = {"intt_s": 0.0, "transfer_s": 0.0, "write_s": 0.0}
    with formats.PTau(src_path, prepared=False) as pt:
        t0 = time.perf_counter()
        w = formats.PreparedPTauWriter(dst_path, pt)
        t["write_s"] += time.perf_counter() - t0
        try:
            for sid, level in w.levels():
                t0 = time.perf_counter()
                d = net.to_device(_tau_level(pt, sid, level))
                net.sync(0)
                t1 = time.perf_counter()
                points_intt(net, d, _SECTIONS[sid][1], out=d)
                net.sync(0)
                t2 = time.perf_counter()
                host = d.cpu().numpy()
                t3 = time.perf_counter()
                w.write_level(sid, level, host)
                t4 = time.perf_counter()
                t["transfer_s"] += (t1 - t0) + (t3 - t2)
                t["intt_s"] += t2 - t1
                t["write_s"] += t4 - t3
            t0 = time.perf_counter()
            w.close()
            t["write_s"] += time.perf_counter() - t0
        except BaseException:
            w.__exit__(None, None, None)
            os.unlink(dst_path)
            raise
    if timings is not None:
        timings.update(t)


@dataclass
class LagrangeReport:
    ok: bool
    failures: list = field(default_factory=list)          # one line per (section, level) that does not check


def _msm(net, pts, scalars, g2: bool) -> np.ndarray:
    xyzz = net.msm_dev(pts, scalars, g2=g2)
    out, inf = net.sum_points_dev(xyzz, 1, g2=g2)
    return np.zeros(16 if g2 else 8, dtype=np.uint64) if inf else out


def check_lagrange(net, ptau_path: str) -> LagrangeReport:
    """The Lagrange part of snarkjs `powersoftau verify` on the GPU: for every section 12-15 and level k, with fresh
    128-bit random rho, MSM(tau-points[:2^k], rho) == MSM(L_k, NTT(rho)).  At the top level of section 12 only the
    2^(power+1) - 1 existing tau points enter.  Needs a prepared file (formats.read_ptau)."""
    from .phase2 import _random_scalars
    rep = LagrangeReport(ok=False)
    try:
        pt = formats.read_ptau(ptau_path)
    except formats.FormatError as e:
        rep.failures.append("not a prepared ptau: %s" % e)
        return rep
    with pt:
        for sid, (src, g2, extra) in _SECTIONS.items():
            w = 16 if g2 else 8
            for k in range(pt.power + extra + 1):
                n = 1 << k
                m = min(n, (2 << pt.power) - 1)
                rho = _random_scalars(net, n)
                lhs = _msm(net, net.to_device(pt.points(src, 0, m, w)), rho[:m].contiguous(), g2)
                rhs = _msm(net, net.to_device(pt.lagrange(sid, k)), net.ntt_dev(rho), g2)
                if not (lhs == rhs).all():
                    rep.failures.append("section %d level %d: the Lagrange points are not the inverse NTT of the first %d "
                                        "points of section %d" % (sid, k, n, src))
    rep.ok = not rep.failures
    return rep
