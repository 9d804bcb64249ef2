// msm_window_pairs.cuh -- EXPERIMENT (not compiled into libb200zk.so): the window sums of the segment pairs (R_s, A_s) as
// a weighted tree, where msm.cu now uses plain per-bit sums (k_msm_window_bits).
//
// With segments of L buckets, R_s = sum_{j<L} b_{sL+j} and A_s = sum_{j<L} (j+1) b_{sL+j}, the window sum is
//   S_w = sum_s A_s + L * sum_s s R_s.
// msm.cu's segment kernel writes (R_s, A_s); k_msm_window_pairs forms the weighted sum in two passes of one tree each (chunks
// of up to 128 segments, then one block per set), and the powers of two L and C are doublings once per block.
//
// Outcome on an H100 80GB HBM3 (700 W, 1980 MHz), G1 2^20 step of bench.py: BIT-EXACT (the exact MSM window sweeps, the
// table sweeps at c = 2..24, the size ladder to 2^22, and segment sums designed to make the trees add P + (-P) and P + P)
// but SLOWER.
// msm_reduce fell from 0.50 to 0.29 ms (184 registers, 256 B stack, against 208 and 384 B); the two tree passes took
// 0.50 ms against 0.12 ms for the plain window sum of the time, and the step went from 4.70-4.96 ms to 4.94-5.09 ms.  The trees are about
// 60 dependent point operations deep on one or two warps per SM, against 16 for the plain sum.  The 2^24 and 2^26 generic
// MSMs, whose tails overlap the next window group's bucket kernel, gained 4.3 and 3.5 ms (separate sessions).  Next step if this is taken up
// again: run the tree levels on quads (quad_ops) and keep the doublings off the critical path.  See DESIGN.md section 7.
//
// Host side as measured (msm_dev_impl, when !quad_reduce): partials sized 2 * WB * nseg, chunks 2 * WB * nchunk, and
//   pt = min(nseg, T); pm = nseg / pt > 128 ? nseg / pt / 128 : 1; nchunk = nseg / (pt * pm); ct = min(nchunk, T);
//   cm = nchunk / ct   (T = 128 on G1, 64 on G2: three shared arrays of T points = 48 KB)
//   k_msm_reduce_segments        <<<(nsets * nseg + 127) / 128, 128>>>(buckets, nsets, B, L, pairs)   (as in msm.cu)
//   k_msm_window_pairs<F, T>     <<<nsets * nchunk, pt>>>(pairs, nseg, pm, log2 L, chunks, chunks + 1, 2)
//   k_msm_window_pairs<F, T>     <<<nsets, ct>>>(chunks, nchunk, cm, log2 L + log2 (pt * pm), nullptr, wsum, 1)
// with the segment length rounded down to a power of two.
#pragma once

namespace b200zk {

// Items i = 0..n-1 of a set are pairs (P_i, X_i), item i standing for u consecutive buckets: P_i = their sum, X_i = their
// running-sum total.  Block (set w, chunk q) of T threads covers the items [q C, (q + 1) C), C = T m, and writes
//   P = sum P_i,   X = sum X_i + u * Z,   Z = sum_i (i - q C) P_i.
// Thread t takes the items q C + t + j T, so Z = sum_t t rho_t + T sum_t omega_t (rho_t = sum_j P, omega_t = sum_j j P).
// At stride s of the tree the thread pairs (i, i + s) differ in bit log2 s alone, so Z_i <- 2 (Z_i + Z_{i+s}) + P_{i+s}
// keeps Z_i = sum over t = i mod s of ((t - i) / s) rho_t + (T / s) omega_t, and Z_0 = Z at s = 1.  The left thread of a
// pair runs the Z chain while the right one adds P and X.
template <class F, int THREADS>
__global__ void __launch_bounds__(THREADS) k_msm_window_pairs(const xyzz_t<F>* items, uint32_t n, uint32_t m, uint32_t log2u,
                                                              xyzz_t<F>* out_p, xyzz_t<F>* out_x, uint32_t out_stride) {
    typedef xyzz_t<F> X;
    __shared__ X shp[THREADS], shz[THREADS], shx[THREADS];
    const uint32_t T = blockDim.x, C = T * m, K = n / C, i = threadIdx.x;      // T, m, C, n: powers of two, C <= n
    const uint32_t w = blockIdx.x / K, q = blockIdx.x % K;
    const X* it = items + 2 * ((size_t)w * n + (size_t)q * C + i);
    X p = X::identity(), z = X::identity(), x = X::identity();
    for (uint32_t j = m; j-- > 0;) {
        const X* e = it + 2 * (size_t)j * T;
        p = X::add_ilp(p, ld16(e));
        x = X::add_ilp(x, ld16(e + 1));
        if (j) z = X::add_ilp(z, p);
    }
    shp[i] = p; shz[i] = z; shx[i] = x;
    __syncthreads();
    for (uint32_t s = T / 2; s > 0; s >>= 1) {
        if (i < s) {
            z = X::add_ilp(X::dbl_ilp(X::add_ilp(z, shz[i + s])), shp[i + s]);
            shz[i] = z;
        } else if (i < 2 * s) {
            shp[i - s] = X::add_ilp(shp[i - s], shp[i]);
            shx[i - s] = X::add_ilp(shx[i - s], shx[i]);
        }
        __syncthreads();
    }
    if (i != 0) return;
    for (uint32_t k = 0; k < log2u; ++k) z = X::dbl_ilp(z);
    if (out_p) st16(out_p + (size_t)blockIdx.x * out_stride, shp[0]);
    st16(out_x + (size_t)blockIdx.x * out_stride, X::add_ilp(shx[0], z));
}

}  // namespace b200zk
