// setup.cu -- kernels for a circuit-specific Groth16 setup on the device (SURVEY 8f3): fixed-base scalar
// multiplication of the G1 / G2 generators, power vectors, generic CSR mat-vec and the linear combinations that turn
// QAP evaluations at tau into query scalars.  Mirrors what `Groth16::circuit_specific_setup` does in the reference's
// drivers (/root/reference/groth16/examples/sha256.rs:133-137, mpc-api/src/main.rs:148-152) with the CircomReduction
// h-query of ark-circom/src/circom/qap.rs:94-110; orchestration in distributed_groth16_b200/groth16/setup.py.
#include <algorithm>

#include "common.cuh"
#include "glv.cuh"

namespace b200zk {

// table[w * 15 + (d - 1)] = d * 16^w * G,  w < 64, d in 1..15 (affine).  64 threads: thread w first walks to 16^w G.
template <class F>
__global__ void k_fixed_base_table(affine_t<F>* table) {
    uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= 64) return;
    xyzz_t<F> base = xyzz_t<F>::from_affine(curve_generator<F>());
    for (uint32_t k = 0; k < 4 * w; ++k) base = xyzz_t<F>::dbl(base);
    affine_t<F> b = xyzz_t<F>::to_affine(base);
    xyzz_t<F> acc = xyzz_t<F>::identity();
    for (uint32_t d = 1; d <= 15; ++d) {
        xyzz_t<F>::madd(acc, b, false);
        st16(table + w * 15 + (d - 1), xyzz_t<F>::to_affine(acc));
    }
}

// out[i] = scalars[i] * G  (scalars Montgomery); 64 mixed additions, no doublings
template <class F>
__global__ void __launch_bounds__(128) k_fixed_base_mul(const affine_t<F>* table, const Fr* scalars, size_t n, affine_t<F>* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr k = Fr::from_mont(ld16(scalars + i));
    xyzz_t<F> acc = xyzz_t<F>::identity();
    for (uint32_t w = 0; w < 64; ++w) {
        uint32_t d = (k.l[w >> 3] >> ((w & 7) * 4)) & 15;
        if (d) xyzz_t<F>::madd(acc, ld16(table + w * 15 + (d - 1)), false);
    }
    st16(out + i, xyzz_t<F>::to_affine(acc));
}

// out[i] = scale * base^i
__global__ void k_fr_powers(const Fr* consts /* base, scale */, size_t n, Fr* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    st16(out + i, Fr::pow_u64(consts[0], i, consts[1]));
}

// out[r] = sum_k val[k] * x[idx[k]],  k in [ptr[r], ptr[r+1])
__global__ void k_spmv(const uint32_t* ptr, const uint32_t* idx, const Fr* val, const Fr* x, size_t n_rows, Fr* out) {
    size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rows) return;
    Fr acc = Fr::zero();
    for (uint32_t k = ptr[r], e = ptr[r + 1]; k < e; ++k) acc = Fr::add(acc, Fr::mul(ld16(val + k), ld16(x + idx[k])));
    st16(out + r, acc);
}

// ---- CSR product over points: out[r] = sum_k val[k] * points[idx[k]]  (snarkjs `zkey new`) -----------------------
// The rows are very skewed (the constant wire's column of A holds 17 896 of the sha256 circuit's 106 808 non-zeros, every
// other column <= 64), so the work is split per non-zero: one variable-base scalar multiplication per thread into a
// product array, then a per-row sum over it.  Rows longer than SPMV_MSM_ROW go through the MSM instead, which bounds the
// per-row sum at SPMV_MSM_ROW additions -- about the cost of one scalar multiplication.
// A 64-bit signed path for short coefficients (v or r - v below 2^64, e.g. -1) was measured and dropped: a warp runs as
// long as its longest scalar and nearly every warp holds a full-width one, so the products kernel took the same time
// (2^20-constraint synthetic circuit on an H100 80GB HBM3 at 400 W: 1787 ms with it, 1766 ms without).
constexpr uint32_t SPMV_MSM_ROW = 256;

template <class F>
__global__ void __launch_bounds__(128) k_points_spmv_products(const uint32_t* idx, const Fr* val, const affine_t<F>* points,
                                                              size_t lo, size_t hi, xyzz_t<F>* prod) {
    size_t k = lo + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= hi) return;
    const Fr v = Fr::from_mont(ld16(val + k));
    int top = 7;
    while (top >= 0 && v.l[top] == 0) --top;
    xyzz_t<F> acc = xyzz_t<F>::identity();
    if (top >= 0) {
        const affine_t<F> p = ld16(points + idx[k]);
        for (int bit = 32 * top + 31 - __clz(v.l[top]); bit >= 0; --bit) {     // double-and-add from the top set bit
            acc = xyzz_t<F>::dbl(acc);
            if ((v.l[bit >> 5] >> (bit & 31)) & 1) xyzz_t<F>::madd(acc, p, false);
        }
    }
    st16(prod + k, acc);
}

// rows of at most SPMV_MSM_ROW entries: sum of their products, normalised; longer rows are left to the MSM path
template <class F>
__global__ void __launch_bounds__(128) k_points_spmv_sum(const uint32_t* ptr, const xyzz_t<F>* prod, size_t n_rows, affine_t<F>* out) {
    size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rows) return;
    const uint32_t b = ptr[r], e = ptr[r + 1];
    if (e - b > SPMV_MSM_ROW) return;
    xyzz_t<F> acc = xyzz_t<F>::identity();
    for (uint32_t k = b; k < e; ++k) acc = xyzz_t<F>::add(acc, ld16(prod + k));
    st16(out + r, xyzz_t<F>::to_affine(acc));
}

template <class F>
__global__ void k_points_gather(const uint32_t* idx, const affine_t<F>* points, size_t n, affine_t<F>* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) st16(out + i, ld16(points + idx[i]));
}

template <class F>
__global__ void k_xyzz_to_affine_one(const xyzz_t<F>* in, affine_t<F>* out) {
    if (threadIdx.x == 0) st16(out, xyzz_t<F>::to_affine(ld16(in)));
}

template <class F>
static int points_spmv_impl(b200zk_ctx* ctx, Slot& sl, const uint32_t* d_ptr, const uint32_t* d_idx, const Fr* d_val,
                            const affine_t<F>* d_points, size_t n_rows, affine_t<F>* d_out) {
    cudaStream_t st = sl.stream;
    // the row pointers decide which rows take the MSM path: read them once on the host (index work only)
    std::vector<uint32_t> ptr(n_rows + 1);
    B2_CUDA_OK(ctx, cudaMemcpyAsync(ptr.data(), d_ptr, (n_rows + 1) * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(st));
    const size_t nnz = ptr[n_rows];
    std::vector<size_t> long_rows;
    for (size_t r = 0; r < n_rows; ++r) {
        if (ptr[r + 1] < ptr[r]) return set_error(ctx, B200ZK_ERR_ARG, "points_spmv: row pointers decrease");
        if (ptr[r + 1] - ptr[r] > SPMV_MSM_ROW) long_rows.push_back(r);
    }
    xyzz_t<F>* prod = nullptr;
    affine_t<F>* gathered = nullptr;
    void* msm_out = nullptr;
    size_t longest = 0;
    for (size_t r : long_rows) longest = std::max(longest, (size_t)(ptr[r + 1] - ptr[r]));
    int rc = B200ZK_OK;
    auto run = [&]() -> int {
        B2_CUDA_OK(ctx, cudaMalloc(&prod, (nnz ? nnz : 1) * sizeof(xyzz_t<F>)));
        // products of every non-zero outside the long rows: one launch per gap between them
        size_t lo = 0;
        for (size_t i = 0; i <= long_rows.size(); ++i) {
            const size_t hi = i < long_rows.size() ? ptr[long_rows[i]] : nnz;
            if (hi > lo) {
                LaunchScope ls(ctx, st, "points_spmv_products");
                k_points_spmv_products<F><<<(unsigned)((hi - lo + 127) / 128), 128, 0, st>>>(d_idx, d_val, d_points, lo, hi, prod);
            }
            B2_TRY(check_launch(ctx, "k_points_spmv_products"));
            if (i < long_rows.size()) lo = ptr[long_rows[i] + 1];
        }
        {
            LaunchScope ls(ctx, st, "points_spmv_sum");
            k_points_spmv_sum<F><<<(unsigned)((n_rows + 127) / 128), 128, 0, st>>>(d_ptr, prod, n_rows, d_out);
        }
        B2_TRY(check_launch(ctx, "k_points_spmv_sum"));
        if (long_rows.empty()) return B200ZK_OK;
        B2_CUDA_OK(ctx, cudaMalloc(&gathered, longest * sizeof(affine_t<F>)));
        B2_CUDA_OK(ctx, cudaMalloc(&msm_out, sizeof(xyzz_t<F>)));
        for (size_t r : long_rows) {
            const size_t b = ptr[r], len = ptr[r + 1] - ptr[r];
            {
                LaunchScope ls(ctx, st, "points_gather");
                k_points_gather<F><<<(unsigned)((len + 255) / 256), 256, 0, st>>>(d_idx + b, d_points, len, gathered);
            }
            B2_TRY(check_launch(ctx, "k_points_gather"));
            B2_TRY(sizeof(F) > 32 ? msm_g2_dev(ctx, sl, gathered, d_val + b, len, msm_out)
                                  : msm_g1_dev(ctx, sl, gathered, d_val + b, len, msm_out));
            {
                LaunchScope ls(ctx, st, "xyzz_to_affine");
                k_xyzz_to_affine_one<F><<<1, 32, 0, st>>>(reinterpret_cast<const xyzz_t<F>*>(msm_out), d_out + r);
            }
            B2_TRY(check_launch(ctx, "k_xyzz_to_affine_one"));
        }
        return B200ZK_OK;
    };
    rc = run();
    cudaError_t e = cudaStreamSynchronize(st);        // the temporaries are freed below
    cudaFree(prod);
    cudaFree(gathered);
    cudaFree(msm_out);
    if (rc != B200ZK_OK) return rc;
    B2_CUDA_OK(ctx, e);
    return B200ZK_OK;
}

int points_spmv_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* ptr, const void* idx, const void* val, const void* points,
                    size_t n_rows, void* out) {
    if (n_rows == 0) return B200ZK_OK;
    return g2 ? points_spmv_impl<Fq2>(ctx, sl, (const uint32_t*)ptr, (const uint32_t*)idx, (const Fr*)val,
                                      (const affine_t<Fq2>*)points, n_rows, (affine_t<Fq2>*)out)
              : points_spmv_impl<Fq>(ctx, sl, (const uint32_t*)ptr, (const uint32_t*)idx, (const Fr*)val,
                                     (const affine_t<Fq>*)points, n_rows, (affine_t<Fq>*)out);
}

// out[i] = (a[i] * s[0] + b[i] * s[1] + c[i] * s[2]) * s[3]
__global__ void k_fr_lincomb(const Fr* a, const Fr* b, const Fr* c, const Fr* s, size_t n, Fr* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr v = Fr::add(Fr::add(Fr::mul(ld16(a + i), s[0]), Fr::mul(ld16(b + i), s[1])), Fr::mul(ld16(c + i), s[2]));
    st16(out + i, Fr::mul(v, s[3]));
}

template <class F>
static int fixed_base_impl(b200zk_ctx* ctx, Slot& sl, void** table_slot, const void* d_scalars, size_t n, void* d_out) {
    cudaStream_t st = sl.stream;
    if (!*table_slot) {
        B2_CUDA_OK(ctx, cudaMalloc(table_slot, 64 * 15 * sizeof(affine_t<F>)));
        {
            LaunchScope ls(ctx, st, "fixed_base_table");
            k_fixed_base_table<F><<<2, 32, 0, st>>>(reinterpret_cast<affine_t<F>*>(*table_slot));
        }
        B2_TRY(check_launch(ctx, "k_fixed_base_table"));
        B2_CUDA_OK(ctx, cudaStreamSynchronize(st));
    }
    if (n == 0) return B200ZK_OK;
    {
        LaunchScope ls(ctx, st, "fixed_base_mul");
        k_fixed_base_mul<F><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(reinterpret_cast<const affine_t<F>*>(*table_slot),
                                                                           reinterpret_cast<const Fr*>(d_scalars), n,
                                                                           reinterpret_cast<affine_t<F>*>(d_out));
    }
    return check_launch(ctx, "k_fixed_base_mul");
}

int fixed_base_mul_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_scalars, size_t n, void* d_out) {
    std::lock_guard<std::mutex> g(ctx->plan_mu);
    return g2 ? fixed_base_impl<Fq2>(ctx, sl, &ctx->fb_table_g2, d_scalars, n, d_out)
              : fixed_base_impl<Fq>(ctx, sl, &ctx->fb_table_g1, d_scalars, n, d_out);
}

int fr_powers_dev(b200zk_ctx* ctx, Slot& sl, const uint64_t base[4], const uint64_t scale[4], size_t n, void* d_out) {
    if (n == 0) return B200ZK_OK;
    B2_CUDA_OK(ctx, sl.small.reserve(1024));
    uint64_t h[8];
    memcpy(h, base, 32); memcpy(h + 4, scale, 32);
    B2_CUDA_OK(ctx, cudaMemcpyAsync(reinterpret_cast<char*>(sl.small.p) + 896, h, 64, cudaMemcpyHostToDevice, sl.stream));
    {
        LaunchScope ls(ctx, sl.stream, "fr_powers");
        k_fr_powers<<<(unsigned)((n + 255) / 256), 256, 0, sl.stream>>>(reinterpret_cast<const Fr*>(reinterpret_cast<char*>(sl.small.p) + 896), n,
                                                                         reinterpret_cast<Fr*>(d_out));
    }
    B2_TRY(check_launch(ctx, "k_fr_powers"));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(sl.stream));      // the staging words are reused by the next call
    return B200ZK_OK;
}

int spmv_dev(b200zk_ctx* ctx, Slot& sl, const void* ptr, const void* idx, const void* val, const void* x, size_t n_rows, void* out) {
    if (n_rows == 0) return B200ZK_OK;
    {
        LaunchScope ls(ctx, sl.stream, "spmv");
        k_spmv<<<(unsigned)((n_rows + 127) / 128), 128, 0, sl.stream>>>((const uint32_t*)ptr, (const uint32_t*)idx, (const Fr*)val,
                                                                         (const Fr*)x, n_rows, (Fr*)out);
    }
    return check_launch(ctx, "k_spmv");
}

int fr_lincomb_dev(b200zk_ctx* ctx, Slot& sl, const void* a, const void* b, const void* c, const uint64_t s[16], size_t n, void* out) {
    if (n == 0) return B200ZK_OK;
    B2_CUDA_OK(ctx, sl.small.reserve(1024));
    char* stage = reinterpret_cast<char*>(sl.small.p) + 768;
    B2_CUDA_OK(ctx, cudaMemcpyAsync(stage, s, 128, cudaMemcpyHostToDevice, sl.stream));
    {
        LaunchScope ls(ctx, sl.stream, "fr_lincomb");
        k_fr_lincomb<<<(unsigned)((n + 255) / 256), 256, 0, sl.stream>>>((const Fr*)a, (const Fr*)b, (const Fr*)c,
                                                                          reinterpret_cast<const Fr*>(stage), n, (Fr*)out);
    }
    B2_TRY(check_launch(ctx, "k_fr_lincomb"));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(sl.stream));
    return B200ZK_OK;
}

// ---- one scalar times many points: out[i] = k * points[i]  (snarkjs `zkey contribute`: L and H times delta^-1) ------
// The phase-2 step the reference's scripts/phase2_proving_key.sh runs after `zkey new`; orchestration in groth16/phase2.py.
// G1: k is reduced mod r and split once per launch, k = k1 + k2 lambda (glv.cuh), and both halves are recoded on the
// host into width-5 NAF digits (odd, |d| <= 15, at least four zeros after each non-zero).  The digits travel as a kernel
// parameter and are the same for every thread, so the digit loop (glv_table_mul, shared with the point iNTT below) has
// no divergence: per point about 128 doublings and
// ~43 mixed additions from a per-thread table of the odd multiples P, 3P, .., 15P (phi(jP) = (beta x, y) is applied on
// the fly).  The table entries and the results are normalised to affine with block-batched inversions (Montgomery's
// trick over a block-wide prefix / suffix product): 8 field inversions per block of 64 points, not one per point.
constexpr int SCALE_BLOCK = 64;
constexpr int SCALE_NAF = 130;            // |k1|, |k2| < 2^127: at most 128 NAF digits
constexpr int SCALE_TAB = 8;              // P, 3P, .., 15P

struct ScaleDigits {
    int8_t d[2][SCALE_NAF];               // d[h][i]: digit i (weight 2^i) of k1 (h = 0) / k2 (h = 1) as a table position
                                          // (glv_table_mul): NAF digit v -> +-(|v| + 1) / 2, signs folded in
    int top;                              // highest index with a non-zero digit in either half; -1: k = 0 mod r
};

// a^-1 for every thread's a (a != 0) of the block, with one F::inv: inclusive prefix and suffix products
// (Hillis-Steele, log2(B) steps), then a_t^-1 = (a_0 .. a_{B-1})^-1 * prefix_{t-1} * suffix_{t+1}.  All threads call it.
template <class F, int B>
__device__ F block_batch_inv(const F& a, F* pre, F* suf, F* tot) {
    const int t = threadIdx.x;
    F p = a, s = a;
    pre[t] = p;
    suf[t] = s;
    __syncthreads();
#pragma unroll 1
    for (int off = 1; off < B; off <<= 1) {
        F pp = t >= off ? pre[t - off] : F::one();
        F ss = t + off < B ? suf[t + off] : F::one();
        __syncthreads();
        if (t >= off) p = F::mul(p, pp);
        if (t + off < B) s = F::mul(s, ss);
        pre[t] = p;
        suf[t] = s;
        __syncthreads();
    }
    if (t == 0) *tot = F::inv(pre[B - 1]);
    __syncthreads();
    F r = *tot;
    if (t > 0) r = F::mul(r, pre[t - 1]);
    if (t < B - 1) r = F::mul(r, suf[t + 1]);
    __syncthreads();                      // pre / suf / tot are reused by the next call
    return r;
}

// every thread's a in affine form with one block_batch_inv over their ZZZ; finite = !a.is_inf(), passed in because the
// caller often knows it more cheaply (a thread with finite = false gets infinity).  All threads call it.
template <class F, int B>
__device__ __forceinline__ affine_t<F> block_to_affine(const xyzz_t<F>& a, bool finite, F* pre, F* suf, F* tot) {
    const F izzz = block_batch_inv<F, B>(finite ? a.zzz : F::one(), pre, suf, tot);
    return finite ? xyzz_t<F>::to_affine(a, izzz) : affine_t<F>::infinity();
}

// table entry j of this thread, stored as C = sizeof(point) / 16 uint4 per point, [entry][chunk][thread]: conflict-free
// shared accesses for a block of B threads
template <class F, int B>
__device__ __forceinline__ void tab_put(uint4* tab, int j, const affine_t<F>& p) {
    constexpr int C = sizeof(affine_t<F>) / 16;
    const uint4* s = reinterpret_cast<const uint4*>(&p);
#pragma unroll
    for (int c = 0; c < C; ++c) tab[(j * C + c) * B + threadIdx.x] = s[c];
}
template <class F, int B>
__device__ __forceinline__ affine_t<F> tab_get(const uint4* tab, int j) {
    constexpr int C = sizeof(affine_t<F>) / 16;
    affine_t<F> p;
    uint4* d = reinterpret_cast<uint4*>(&p);
#pragma unroll
    for (int c = 0; c < C; ++c) d[c] = tab[(j * C + c) * B + threadIdx.x];
    return p;
}

// acc = 2^(DOUBLINGS (top + 1)) acc + sum_{q <= top} 2^(DOUBLINGS q) (d1[q] + d2[q] lambda) P by Horner from q = top, over
// this thread's table of multiples of P: a digit is a signed table position, +-(j + 1) adds +-(entry j), 0 adds nothing;
// the d2 entries go through phi (glv_phi_x).
template <class F, int B, int DOUBLINGS>
__device__ __forceinline__ void glv_table_mul(xyzz_t<F>& acc, const uint4* tab, const int8_t* d1, const int8_t* d2, int top) {
#pragma unroll 1
    for (int q = top; q >= 0; --q) {
#pragma unroll
        for (int k = 0; k < DOUBLINGS; ++k) acc = xyzz_t<F>::dbl(acc);
        const int a = d1[q], b = d2[q];
        if (a) xyzz_t<F>::madd(acc, tab_get<F, B>(tab, (a < 0 ? -a : a) - 1), a < 0);
        if (b) {
            affine_t<F> p = tab_get<F, B>(tab, (b < 0 ? -b : b) - 1);
            glv_phi_x(p.x);
            xyzz_t<F>::madd(acc, p, b < 0);
        }
    }
}

__global__ void __launch_bounds__(SCALE_BLOCK) k_points_scale_g1(const __grid_constant__ ScaleDigits dg,
                                                                  const affine_t<Fq>* points, size_t n, affine_t<Fq>* out) {
    __shared__ uint4 tab[SCALE_TAB * 4 * SCALE_BLOCK];
    __shared__ Fq pre[SCALE_BLOCK], suf[SCALE_BLOCK], tot;
    const size_t i = (size_t)blockIdx.x * SCALE_BLOCK + threadIdx.x;
    const affine_t<Fq> P = i < n ? ld16(points + i) : affine_t<Fq>::infinity();
    const bool inf = P.is_inf();
    // the odd multiples, (2j + 1) P = (2j - 1) P + 2P in XYZZ, each normalised as it is made (one block-batched
    // inverse per entry: only the running entry and 2P are live)
    tab_put<Fq, SCALE_BLOCK>(tab, 0, P);
    {
        const xyzz_t<Fq> two = inf ? xyzz_t<Fq>::identity() : xyzz_t<Fq>::dbl_affine(P.x, P.y);
        xyzz_t<Fq> odd = xyzz_t<Fq>::from_affine(P);
#pragma unroll 1
        for (int j = 1; j < SCALE_TAB; ++j) {
            odd = xyzz_t<Fq>::add(odd, two);
            tab_put<Fq, SCALE_BLOCK>(tab, j, block_to_affine<Fq, SCALE_BLOCK>(odd, !inf, pre, suf, &tot));
        }
    }
    xyzz_t<Fq> acc = xyzz_t<Fq>::identity();
    if (!inf) glv_table_mul<Fq, SCALE_BLOCK, 1>(acc, tab, dg.d[0], dg.d[1], dg.top);
    const affine_t<Fq> r = block_to_affine<Fq, SCALE_BLOCK>(acc, !acc.is_inf(), pre, suf, &tot);
    if (i < n) st16(out + i, r);
}

// G2 (single points: delta_2, g2_spx, the cofactor of hash-to-G2): the plain 256-bit ladder, no reduction mod r, so that
// it is right for twist points outside the order-r subgroup too
struct ScaleK { uint32_t k[8]; };

__global__ void __launch_bounds__(128) k_points_scale_g2_ladder(const __grid_constant__ ScaleK k, const affine_t<Fq2>* points,
                                                                size_t n, affine_t<Fq2>* out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const affine_t<Fq2> p = ld16(points + i);
    st16(out + i, xyzz_t<Fq2>::to_affine(xyzz_t<Fq2>::mul_scalar(xyzz_t<Fq2>::from_affine(p), k.k)));
}

// width-5 NAF of a non-negative k < 2^127 into d (digits odd in [-15, 15]); returns the highest non-zero index or -1
static int naf5(unsigned __int128 k, int8_t* d) {
    int top = -1;
    for (int i = 0; i < SCALE_NAF; ++i) {
        int v = 0;
        if (k & 1) {
            v = (int)(k & 31);
            if (v >= 16) v -= 32;
            if (v > 0) k -= (unsigned)v;
            else k += (unsigned)(-v);
            top = i;
        }
        d[i] = (int8_t)v;
        k >>= 1;
    }
    return top;
}

// 4 u64 limbs of a plain integer < 2^256 -> 8 u32 limbs of it mod r (k < 2^256 < 6 r)
static void reduce_mod_r(const uint64_t k64[4], uint32_t k[8]) {
    for (int i = 0; i < 4; ++i) { k[2 * i] = (uint32_t)k64[i]; k[2 * i + 1] = (uint32_t)(k64[i] >> 32); }
    for (;;) {
        bool ge = true;
        for (int i = 7; i >= 0; --i) {
            if (k[i] != FrParams::mod(i)) { ge = k[i] > FrParams::mod(i); break; }
        }
        if (!ge) break;
        int64_t br = 0;
        for (int i = 0; i < 8; ++i) {
            int64_t v = (int64_t)k[i] - (int64_t)FrParams::mod(i) + br;
            k[i] = (uint32_t)v;
            br = v >> 32;
        }
    }
}

int points_scale_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_points, size_t n, const uint64_t k64[4], void* d_out) {
    if (n == 0) return B200ZK_OK;
    uint32_t k[8];
    if (g2) {
        for (int i = 0; i < 4; ++i) { k[2 * i] = (uint32_t)k64[i]; k[2 * i + 1] = (uint32_t)(k64[i] >> 32); }
        ScaleK sk;
        memcpy(sk.k, k, sizeof(k));
        {
            LaunchScope ls(ctx, sl.stream, "points_scale_g2");
            k_points_scale_g2_ladder<<<(unsigned)((n + 127) / 128), 128, 0, sl.stream>>>(
                sk, reinterpret_cast<const affine_t<Fq2>*>(d_points), n, reinterpret_cast<affine_t<Fq2>*>(d_out));
        }
        return check_launch(ctx, "k_points_scale_g2");
    }
    reduce_mod_r(k64, k);
    const GlvSplit sp = glv_decompose(k);
    ScaleDigits dg;
    int top = -1;
    for (int h = 0; h < 2; ++h) {
        const uint32_t* w = h ? sp.k2 : sp.k1;
        unsigned __int128 v = 0;
        for (int i = 3; i >= 0; --i) v = (v << 32) | w[i];
        const int t = naf5(v, dg.d[h]);
        const bool neg = h ? sp.neg2 : sp.neg1;
        for (int i = 0; i < SCALE_NAF; ++i) {          // the table holds P, 3P, .., 15P: |v| P is entry (|v| - 1) / 2
            const int v = neg ? -dg.d[h][i] : dg.d[h][i];
            dg.d[h][i] = (int8_t)(v < 0 ? -((1 - v) / 2) : (v + 1) / 2);
        }
        top = t > top ? t : top;
    }
    dg.top = top;
    if (n >= ((size_t)1 << 31) * SCALE_BLOCK) return set_error(ctx, B200ZK_ERR_ARG, "points_scale: too many points");
    {
        LaunchScope ls(ctx, sl.stream, "points_scale_g1");
        k_points_scale_g1<<<(unsigned)((n + SCALE_BLOCK - 1) / SCALE_BLOCK), SCALE_BLOCK, 0, sl.stream>>>(
            dg, reinterpret_cast<const affine_t<Fq>*>(d_points), n, reinterpret_cast<affine_t<Fq>*>(d_out));
    }
    return check_launch(ctx, "k_points_scale_g1");
}

// ---- NTT over points: out[i] = sum_j w_n^(i j) in[j], and the inverse n^-1 sum_j w_n^(-i j) in[j] -----------------------
// The inverse makes the Lagrange levels of a prepared Powers-of-Tau file (snarkjs `powersoftau prepare phase2`,
// orchestration in groth16/ptau.py); the forward one moves a zkey's H query into the tau basis of a bellman MPC-params
// file (snarkjs `zkey export bellman`, groth16/bellman.py).  Radix-2 decimation in time: one bit-reversal pass, then
// log_n in-place butterfly passes over global memory, then, for the inverse only, n^-1 by points_scale_dev.  Each
// butterfly costs one full scalar multiplication (w^-j P) against a handful of point additions, so the passes are plain
// and the work per thread is made uniform instead:
//   * the twiddles w_n^-+i, i < n / 2, are computed once per transform on the device, split with GLV (glv.cuh; on G2
//     phi = (beta^2 x, y), right for points of the order-r subgroup) and recoded into 32 signed 4-bit windows per half,
//     digits in [-7, 8] (|k1|, |k2| < 2^127 leave no carry out of the top window).  Every thread runs the same
//     32 x (4 doublings + 2 mixed additions) from a per-thread table P, 2P, .., 8P in shared memory (normalised with
//     block-batched inversions like points_scale);
//   * butterflies are numbered twiddle-major, so consecutive threads share a twiddle whenever a pass has >= 32
//     butterflies per twiddle: a warp reads one digit string, and the blocks whose twiddle is w^0 skip the product;
//   * U + wP and U - wP share one block-batched inversion (of the product of their ZZZ).
constexpr int INTT_WINDOWS = 32;
constexpr int INTT_TAB = 8;               // P, 2P, .., 8P
constexpr int INTT_BLOCK_G1 = 64;
constexpr int INTT_BLOCK_G2 = 32;         // the G2 table (8 x 128 B per thread) fills 32 KB of shared memory at 32 threads

// the scalar of one product of the point iNTT (a twiddle) or of points_mul_powers (first ratio^i) in the form
// glv_table_mul<F, B, 4> takes
struct __align__(16) TwiddleDigits {
    int8_t d[2][INTT_WINDOWS];            // d[h][w]: window w (weight 16^w) of k1 (h = 0) / k2 (h = 1), signs folded in
};

// k (canonical, < r) -> GLV halves, each recoded into 32 signed 4-bit windows in [-7, 8] (a window above 8 borrows 16 from
// the next one; |k1|, |k2| < 2^127 leave no carry out of the top window)
__device__ __forceinline__ TwiddleDigits glv_window_digits(const Fr& k) {
    const GlvSplit sp = glv_decompose(k.l);
    TwiddleDigits dg;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const uint32_t* w = h ? sp.k2 : sp.k1;
        const bool neg = h ? sp.neg2 : sp.neg1;
        int carry = 0;
#pragma unroll
        for (int q = 0; q < INTT_WINDOWS; ++q) {
            int v = (int)((w[q >> 3] >> ((q & 7) * 4)) & 15) + carry;
            carry = v > 8;
            if (carry) v -= 16;
            dg.d[h][q] = (int8_t)(neg ? -v : v);
        }
    }
    return dg;
}

// digits of w_n^-i (inverse) or w_n^i for i < count
__global__ void k_intt_twiddle_digits(unsigned log_n, bool inverse, size_t count, TwiddleDigits* out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    st16(out + i, glv_window_digits(Fr::from_mont(Fr::pow_u64(fr_root_of_unity(log_n, inverse), i))));
}

// out[i] = in[bitrev(i)]; each pair is handled by one thread that reads both before writing, so out may equal in
template <class F>
__global__ void k_points_bitrev(const affine_t<F>* in, affine_t<F>* out, unsigned log_n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >> log_n) return;
    const size_t r = log_n ? (size_t)(__brevll((unsigned long long)i) >> (64 - log_n)) : 0;
    if (r < i) return;
    const affine_t<F> x = ld16(in + i), y = ld16(in + r);
    st16(out + i, y);
    if (r != i) st16(out + r, x);
}

// this thread's table P, 2P, .., 8P for glv_table_mul<F, B, 4>, normalised with block-batched inversions; mul = false
// leaves entries 1..7 at infinity (P is not multiplied).  The table is built from shared memory copies only: P and the
// products stay out of registers during the loop.  All threads call it.
template <class F, int B>
__device__ __forceinline__ void build_mul_table(uint4* tab, const affine_t<F>& P, bool mul, F* pre, F* suf, F* tot) {
    tab_put<F, B>(tab, 0, P);
    xyzz_t<F> run = xyzz_t<F>::identity();
#pragma unroll 1
    for (int e = 1; e < INTT_TAB; ++e) {                                 // (e + 1) P
        if (mul) {
            const affine_t<F> Q = tab_get<F, B>(tab, 0);
            if (e == 1) run = xyzz_t<F>::dbl_affine(Q.x, Q.y);
            else xyzz_t<F>::madd(run, Q, false);
        }
        tab_put<F, B>(tab, e, block_to_affine<F, B>(run, mul, pre, suf, tot));
    }
}

// pass with half-size m = 2^log_m: butterfly t = (j, g), j = t >> lg, g = t mod 2^lg (lg = log2(n / 2m)), on the
// elements g 2m + j and g 2m + j + m with twiddle w_2m^-+j = w_n^-+(j << lg) (the sign is the transform's direction)
template <class F, int B>
__global__ void __launch_bounds__(B) k_points_intt_pass(affine_t<F>* a, const TwiddleDigits* __restrict__ tw, unsigned log_n,
                                                        unsigned log_m) {
    constexpr int C = sizeof(affine_t<F>) / 16;
    __shared__ uint4 tab[INTT_TAB * C * B];
    __shared__ F pre[B], suf[B], tot;
    const unsigned lg = log_n - 1 - log_m;
    const size_t t = (size_t)blockIdx.x * B + threadIdx.x;
    const bool live = (t >> (log_n - 1)) == 0;
    const size_t j = t >> lg;
    const size_t ia = ((t & (((size_t)1 << lg) - 1)) << (log_m + 1)) + j, ib = ia + ((size_t)1 << log_m);
    bool mul = false;
    if (!__syncthreads_and(!live || j == 0)) {                           // block-uniform
        const affine_t<F> P = live ? ld16(a + ib) : affine_t<F>::infinity();
        mul = live && j != 0 && !P.is_inf();
        build_mul_table<F, B>(tab, P, mul, pre, suf, &tot);
    }
    xyzz_t<F> prod = xyzz_t<F>::identity();
    if (mul) glv_table_mul<F, B, 4>(prod, tab, tw[j << lg].d[0], tw[j << lg].d[1], INTT_WINDOWS - 1);
    else prod = xyzz_t<F>::from_affine(live ? ld16(a + ib) : affine_t<F>::infinity());      // w^0 P, or P = infinity
    // T = w P in affine form, then U + T and U - T as affine additions that share one inverse: the denominator is
    // x_T - x_U, or 2 y_U when T = +-U (then one result is infinity and the other 2U), or 1 when T or U is infinity
    const affine_t<F> T = block_to_affine<F, B>(prod, !prod.is_inf(), pre, suf, &tot);
    const affine_t<F> U = live ? ld16(a + ia) : affine_t<F>::infinity();
    const bool edge = T.is_inf() || U.is_inf();
    const F dx = F::sub(T.x, U.x);
    const bool dbl = !edge && dx.is_zero();
    const F inv = block_batch_inv<F, B>(edge ? F::one() : dbl ? F::dbl(U.y) : dx, pre, suf, &tot);
    if (!live) return;
    affine_t<F> s, df;
    if (T.is_inf()) {
        s = U;
        df = U;
    } else if (U.is_inf()) {
        s = T;
        df = T;
        df.y = F::neg(T.y);
    } else {
        auto finish = [&](const F& lam, const F& x_other) {                  // U + Q from the slope, x_Q = x_other
            affine_t<F> r;
            r.x = F::sub(F::sub(F::sqr(lam), U.x), x_other);
            r.y = F::sub(F::mul(lam, F::sub(U.x, r.x)), U.y);
            return r;
        };
        if (dbl) {                                                           // T = U or T = -U
            const F x2 = F::sqr(U.x);
            const affine_t<F> two = finish(F::mul(F::add(F::dbl(x2), x2), inv), U.x);
            const bool same = F::sub(T.y, U.y).is_zero();
            s = same ? two : affine_t<F>::infinity();
            df = same ? affine_t<F>::infinity() : two;
        } else {
            s = finish(F::mul(F::sub(T.y, U.y), inv), T.x);
            df = finish(F::mul(F::neg(F::add(T.y, U.y)), inv), T.x);
        }
    }
    st16(a + ia, s);
    st16(a + ib, df);
}

template <class F, int B>
static int points_intt_impl(b200zk_ctx* ctx, Slot& sl, int g2, bool inverse, const affine_t<F>* d_in, unsigned log_n,
                            affine_t<F>* d_out) {
    const char* what = inverse ? "points_intt" : "points_ntt";
    cudaStream_t st = sl.stream;
    const size_t n = (size_t)1 << log_n, half = n >> 1;
    TwiddleDigits* tw = nullptr;
    if (half) {
        const cudaError_t e = cudaMalloc(&tw, half * sizeof(TwiddleDigits));
        if (e != cudaSuccess) {
            cudaGetLastError();                                           // nothing was launched: leave no error behind
            char b[256];
            snprintf(b, sizeof(b), "%s: the twiddle digits of 2^%u points (%zu MB of device memory) do not fit: %s",
                     what, log_n, half * sizeof(TwiddleDigits) >> 20, cudaGetErrorString(e));
            return set_error(ctx, e == cudaErrorMemoryAllocation ? B200ZK_ERR_OOM : B200ZK_ERR_CUDA, b);
        }
    }
    auto run = [&]() -> int {
        {
            LaunchScope ls(ctx, st, "points_intt_bitrev");
            k_points_bitrev<F><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_in, d_out, log_n);
        }
        B2_TRY(check_launch(ctx, "k_points_bitrev"));
        if (!half) return B200ZK_OK;
        {
            LaunchScope ls(ctx, st, "points_intt_twiddles");
            k_intt_twiddle_digits<<<(unsigned)((half + 255) / 256), 256, 0, st>>>(log_n, inverse, half, tw);
        }
        B2_TRY(check_launch(ctx, "k_intt_twiddle_digits"));
        for (unsigned log_m = 0; log_m < log_n; ++log_m) {
            {
                LaunchScope ls(ctx, st, g2 ? "points_intt_pass_g2" : "points_intt_pass_g1");
                k_points_intt_pass<F, B><<<(unsigned)((half + B - 1) / B), B, 0, st>>>(d_out, tw, log_n, log_m);
            }
            B2_TRY(check_launch(ctx, "k_points_intt_pass"));
        }
        if (!inverse) return B200ZK_OK;
        // n^-1 mod r = r - (r - 1) / n  (n divides r - 1)
        uint32_t q[8], ninv32[8];
        for (int i = 0; i < 8; ++i) q[i] = FrParams::mod(i) & (i ? ~0u : ~1u);
        for (int i = 0; i < 8; ++i) {
            const uint64_t hi = i < 7 ? (uint64_t)q[i + 1] : 0;
            q[i] = (uint32_t)((((hi << 32) | q[i]) >> log_n));
        }
        int64_t br = 0;
        for (int i = 0; i < 8; ++i) {
            const int64_t v = (int64_t)FrParams::mod(i) - (int64_t)q[i] + br;
            ninv32[i] = (uint32_t)v;
            br = v >> 32;
        }
        uint64_t ninv[4];
        for (int i = 0; i < 4; ++i) ninv[i] = (uint64_t)ninv32[2 * i] | ((uint64_t)ninv32[2 * i + 1] << 32);
        return points_scale_dev(ctx, sl, g2, d_out, n, ninv, d_out);
    };
    const int rc = run();
    const cudaError_t e = cudaStreamSynchronize(st);                     // the twiddle digits are freed below
    cudaFree(tw);
    if (rc != B200ZK_OK) return rc;
    B2_CUDA_OK(ctx, e);
    return B200ZK_OK;
}

static int points_transform(b200zk_ctx* ctx, Slot& sl, int g2, bool inverse, const void* d_in, unsigned log_n, void* d_out) {
    return g2 ? points_intt_impl<Fq2, INTT_BLOCK_G2>(ctx, sl, 1, inverse, (const affine_t<Fq2>*)d_in, log_n,
                                                     (affine_t<Fq2>*)d_out)
              : points_intt_impl<Fq, INTT_BLOCK_G1>(ctx, sl, 0, inverse, (const affine_t<Fq>*)d_in, log_n,
                                                    (affine_t<Fq>*)d_out);
}

int points_intt_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_in, unsigned log_n, void* d_out) {
    return points_transform(ctx, sl, g2, true, d_in, log_n, d_out);
}

int points_ntt_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_in, unsigned log_n, void* d_out) {
    return points_transform(ctx, sl, g2, false, d_in, log_n, d_out);
}

// ---- each point times its own term of a geometric sequence: out[i] = (first ratio^i) points[i]  (snarkjs `powersoftau
// contribute`, ffjavascript G.batchApplyKey) -------------------------------------------------------------------------------
// The whole cost of a phase-1 contribution; orchestration in groth16/phase1.py.  The scalars differ per point, so the
// point iNTT's product is reused as it stands: a digit kernel makes first ratio^i on the device and recodes it with
// glv_window_digits into a workspace (64 bytes per point), then every thread runs the same 32 x (4 doublings + 2 mixed
// additions) over its table P..8P.  The digits are read straight from the workspace: a thread's 64 bytes sit in one cache
// line, and the reads are two bytes per 4 doublings + 2 additions.
struct PowersConsts { Fr first, ratio; };        // canonical (reduced mod r), turned into Montgomery form on the device

__global__ void k_powers_digits(const __grid_constant__ PowersConsts c, size_t count, TwiddleDigits* out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    st16(out + i, glv_window_digits(Fr::from_mont(Fr::pow_u64(Fr::to_mont(c.ratio), i, Fr::to_mont(c.first)))));
}

template <class F, int B>
__global__ void __launch_bounds__(B) k_points_mul_powers(const affine_t<F>* points, const TwiddleDigits* __restrict__ dg,
                                                         size_t n, affine_t<F>* out) {
    constexpr int C = sizeof(affine_t<F>) / 16;
    __shared__ uint4 tab[INTT_TAB * C * B];
    __shared__ F pre[B], suf[B], tot;
    const size_t i = (size_t)blockIdx.x * B + threadIdx.x;
    bool mul;
    {
        const affine_t<F> P = i < n ? ld16(points + i) : affine_t<F>::infinity();
        mul = !P.is_inf();
        build_mul_table<F, B>(tab, P, mul, pre, suf, &tot);
    }
    xyzz_t<F> prod = xyzz_t<F>::identity();
    if (mul) glv_table_mul<F, B, 4>(prod, tab, dg[i].d[0], dg[i].d[1], INTT_WINDOWS - 1);
    const affine_t<F> r = block_to_affine<F, B>(prod, !prod.is_inf(), pre, suf, &tot);
    if (i < n) st16(out + i, r);
}

template <class F, int B>
static int points_mul_powers_impl(b200zk_ctx* ctx, Slot& sl, const affine_t<F>* d_points, size_t n, const uint64_t first[4],
                                  const uint64_t ratio[4], affine_t<F>* d_out) {
    if (n == 0) return B200ZK_OK;
    if (n >= ((size_t)1 << 31) * B) return set_error(ctx, B200ZK_ERR_ARG, "points_mul_powers: too many points");
    cudaStream_t st = sl.stream;
    PowersConsts c;
    reduce_mod_r(first, c.first.l);
    reduce_mod_r(ratio, c.ratio.l);
    TwiddleDigits* dg = nullptr;
    {
        const cudaError_t e = cudaMalloc(&dg, n * sizeof(TwiddleDigits));
        if (e != cudaSuccess) {
            cudaGetLastError();                                           // nothing was launched: leave no error behind
            char b[256];
            snprintf(b, sizeof(b), "points_mul_powers: the scalar digits of %zu points (%zu MB of device memory) do not fit: %s",
                     n, n * sizeof(TwiddleDigits) >> 20, cudaGetErrorString(e));
            return set_error(ctx, e == cudaErrorMemoryAllocation ? B200ZK_ERR_OOM : B200ZK_ERR_CUDA, b);
        }
    }
    auto run = [&]() -> int {
        {
            LaunchScope ls(ctx, st, "powers_digits");
            k_powers_digits<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, n, dg);
        }
        B2_TRY(check_launch(ctx, "k_powers_digits"));
        {
            LaunchScope ls(ctx, st, sizeof(F) > 32 ? "points_mul_powers_g2" : "points_mul_powers_g1");
            k_points_mul_powers<F, B><<<(unsigned)((n + B - 1) / B), B, 0, st>>>(d_points, dg, n, d_out);
        }
        return check_launch(ctx, "k_points_mul_powers");
    };
    const int rc = run();
    const cudaError_t e = cudaStreamSynchronize(st);                     // the digits are freed below
    cudaFree(dg);
    if (rc != B200ZK_OK) return rc;
    B2_CUDA_OK(ctx, e);
    return B200ZK_OK;
}

int points_mul_powers_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_points, size_t n, const uint64_t first[4],
                          const uint64_t ratio[4], void* d_out) {
    return g2 ? points_mul_powers_impl<Fq2, INTT_BLOCK_G2>(ctx, sl, (const affine_t<Fq2>*)d_points, n, first, ratio,
                                                           (affine_t<Fq2>*)d_out)
              : points_mul_powers_impl<Fq, INTT_BLOCK_G1>(ctx, sl, (const affine_t<Fq>*)d_points, n, first, ratio,
                                                          (affine_t<Fq>*)d_out);
}

// ---- pointwise difference: out[i] = a[i] - b[i]  (snarkjs `zkey new`: the circuit hash's H points tau^(n+i) G1 - tau^i G1)
// One mixed addition per point (madd handles a = +-b and either side at infinity), normalised with one block-batched
// inversion per block.  Each thread reads its a[i] and b[i] before the block's first barrier and writes only out[i], so
// out may equal a or b.
constexpr int SUB_BLOCK = 128;

template <class F>
__global__ void __launch_bounds__(SUB_BLOCK) k_points_sub(const affine_t<F>* a, const affine_t<F>* b, size_t n, affine_t<F>* out) {
    __shared__ F pre[SUB_BLOCK], suf[SUB_BLOCK], tot;
    const size_t i = (size_t)blockIdx.x * SUB_BLOCK + threadIdx.x;
    xyzz_t<F> d = xyzz_t<F>::identity();
    if (i < n) {
        d = xyzz_t<F>::from_affine(ld16(a + i));
        xyzz_t<F>::madd(d, ld16(b + i), true);
    }
    const affine_t<F> r = block_to_affine<F, SUB_BLOCK>(d, !d.is_inf(), pre, suf, &tot);
    if (i < n) st16(out + i, r);
}

int points_sub_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_a, const void* d_b, size_t n, void* d_out) {
    if (n == 0) return B200ZK_OK;
    if (n >= ((size_t)1 << 31) * SUB_BLOCK) return set_error(ctx, B200ZK_ERR_ARG, "points_sub: too many points");
    const unsigned grid = (unsigned)((n + SUB_BLOCK - 1) / SUB_BLOCK);
    {
        LaunchScope ls(ctx, sl.stream, g2 ? "points_sub_g2" : "points_sub_g1");
        if (g2) k_points_sub<Fq2><<<grid, SUB_BLOCK, 0, sl.stream>>>((const affine_t<Fq2>*)d_a, (const affine_t<Fq2>*)d_b, n,
                                                                     (affine_t<Fq2>*)d_out);
        else k_points_sub<Fq><<<grid, SUB_BLOCK, 0, sl.stream>>>((const affine_t<Fq>*)d_a, (const affine_t<Fq>*)d_b, n,
                                                                 (affine_t<Fq>*)d_out);
    }
    return check_launch(ctx, "k_points_sub");
}

}  // namespace b200zk
