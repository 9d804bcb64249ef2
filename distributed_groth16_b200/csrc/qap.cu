// qap.cu -- R1CS x witness -> QAP evaluation vectors on the device (SURVEY 8f2), plus the Montgomery
// conversions the file readers need.
//
// Replaces `qap::qap` (/root/reference/groth16/src/qap.rs:44-91; identical logic in
// ark-circom/src/circom/qap.rs:38-62): a_i = <A_i, z>, b_i = <B_i, z> for i < num_constraints (rayon
// `evaluate_constraint` per row, qap.rs:60-67), a[num_constraints + j] = z[j] for j < num_inputs (:69-73),
// c_i = a_i * b_i (:75-81), everything zero-padded to the domain size m.  The same mat-vec, with C as a third matrix, checks
// a witness against its circuit (r1cs_check_dev, snarkjs `wtns check`).
// HBM-bound sparse mat-vec: per non-zero 4 B column index + 32 B coefficient + a 32 B gather from z.
#include "common.cuh"

namespace b200zk {

__global__ void k_fr_convert(const Fr* in, Fr* out, size_t n, int to_mont, int times) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr v = ld16(in + i);
    for (int t = 0; t < times; ++t) v = to_mont ? Fr::to_mont(v) : Fr::from_mont(v);
    st16(out + i, v);
}

__device__ __forceinline__ Fr row_dot(const uint32_t* ptr, const uint32_t* col, const Fr* val, const Fr* z, uint32_t i) {
    Fr acc = Fr::zero();
    for (uint32_t k = ptr[i], e = ptr[i + 1]; k < e; ++k) acc = Fr::add(acc, Fr::mul(ld16(val + k), ld16(z + col[k])));
    return acc;
}

__global__ void k_qap(const uint32_t* a_ptr, const uint32_t* a_col, const Fr* a_val, const uint32_t* b_ptr, const uint32_t* b_col,
                      const Fr* b_val, const Fr* z, uint32_t nc, uint32_t n_inputs, uint32_t m, Fr* a, Fr* b, Fr* c) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    Fr va = Fr::zero(), vb = Fr::zero(), vc = Fr::zero();
    if (i < nc) {
        va = row_dot(a_ptr, a_col, a_val, z, i);
        vb = row_dot(b_ptr, b_col, b_val, z, i);
        vc = Fr::mul(va, vb);
    } else if (i < nc + n_inputs) {
        va = ld16(z + (i - nc));
    }
    st16(a + i, va); st16(b + i, vb); st16(c + i, vc);
}

// One warp per row: the lanes stride over the row's non-zeros and the partial sums meet in a shuffle tree.  Small circuits have
// far fewer rows than the machine has lanes and a few long rows (the reference's sha256 circuit: 30 134 rows, the longest row
// is a long serial chain for one thread); field addition is exact, so the order of summation does not change the result.
__device__ __forceinline__ Fr warp_sum(Fr v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        Fr o;
#pragma unroll
        for (int i = 0; i < 8; ++i) o.l[i] = __shfl_down_sync(0xFFFFFFFFu, v.l[i], d);
        v = Fr::add(v, o);
    }
    return v;
}
__device__ __forceinline__ Fr row_dot_warp(const uint32_t* ptr, const uint32_t* col, const Fr* val, const Fr* z, uint32_t i, uint32_t lane) {
    Fr acc = Fr::zero();
    for (uint32_t k = ptr[i] + lane, e = ptr[i + 1]; k < e; k += 32) acc = Fr::add(acc, Fr::mul(ld16(val + k), ld16(z + col[k])));
    return warp_sum(acc);
}
__global__ void __launch_bounds__(256) k_qap_warp(const uint32_t* a_ptr, const uint32_t* a_col, const Fr* a_val, const uint32_t* b_ptr,
                                                  const uint32_t* b_col, const Fr* b_val, const Fr* z, uint32_t nc, uint32_t n_inputs,
                                                  uint32_t m, Fr* a, Fr* b, Fr* c) {
    const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (i >= m) return;
    Fr va = Fr::zero(), vb = Fr::zero(), vc = Fr::zero();
    if (i < nc) {
        va = row_dot_warp(a_ptr, a_col, a_val, z, i, lane);
        vb = row_dot_warp(b_ptr, b_col, b_val, z, i, lane);
        vc = Fr::mul(va, vb);
    } else if (i < nc + n_inputs) {
        va = ld16(z + (i - nc));
    }
    if (lane == 0) { st16(a + i, va); st16(b + i, vb); st16(c + i, vc); }
}

int fr_convert_dev(b200zk_ctx* ctx, Slot& sl, const void* d_in, void* d_out, size_t n, int to_mont, int times) {
    if (n == 0) return B200ZK_OK;
    {
        LaunchScope ls(ctx, sl.stream, "fr_convert");
        k_fr_convert<<<(unsigned)((n + 255) / 256), 256, 0, sl.stream>>>((const Fr*)d_in, (Fr*)d_out, n, to_mont, times);
    }
    return check_launch(ctx, "k_fr_convert");
}

int qap_dev(b200zk_ctx* ctx, Slot& sl, const void* a_ptr, const void* a_col, const void* a_val, const void* b_ptr,
            const void* b_col, const void* b_val, size_t nc, size_t n_inputs, const void* d_z, unsigned log_m, void* d_a,
            void* d_b, void* d_c) {
    if (log_m > 28) return set_error(ctx, B200ZK_ERR_DOMAIN, "domain too large (PolynomialDegreeTooLarge)");
    size_t m = (size_t)1 << log_m;
    if (nc + n_inputs > m) return set_error(ctx, B200ZK_ERR_DOMAIN, "num_constraints + num_inputs exceeds the domain size");
    {
        LaunchScope ls(ctx, sl.stream, "qap_matvec");
        const uint32_t *ap = (const uint32_t*)a_ptr, *ac = (const uint32_t*)a_col, *bp = (const uint32_t*)b_ptr, *bc = (const uint32_t*)b_col;
        if (m <= ((size_t)1 << 18))          // warp per row while rows x 32 lanes still fit a few waves
            k_qap_warp<<<(unsigned)((m * 32 + 255) / 256), 256, 0, sl.stream>>>(ap, ac, (const Fr*)a_val, bp, bc, (const Fr*)b_val, (const Fr*)d_z,
                                                                                (uint32_t)nc, (uint32_t)n_inputs, (uint32_t)m, (Fr*)d_a, (Fr*)d_b, (Fr*)d_c);
        else
            k_qap<<<(unsigned)((m + 127) / 128), 128, 0, sl.stream>>>(ap, ac, (const Fr*)a_val, bp, bc, (const Fr*)b_val, (const Fr*)d_z,
                                                                       (uint32_t)nc, (uint32_t)n_inputs, (uint32_t)m, (Fr*)d_a, (Fr*)d_b, (Fr*)d_c);
    }
    return check_launch(ctx, "k_qap");
}

// R1CS satisfaction (snarkjs `wtns check`): constraint i holds iff <A_i, w> <B_i, w> = <C_i, w>.  The same mat-vec as k_qap
// with C as a third matrix; a failing row bumps bad[0] and lowers bad[1] to its index.
struct CsrRows {
    const uint32_t* ptr;
    const uint32_t* col;
    const Fr* val;
};

__device__ __forceinline__ void r1cs_flag(const Fr& a, const Fr& b, const Fr& c, uint32_t i, unsigned long long* bad) {
    if (Fr::mul(a, b) != c) {
        atomicAdd(&bad[0], 1ull);
        atomicMin(&bad[1], (unsigned long long)i);
    }
}

__global__ void __launch_bounds__(128) k_r1cs_check(CsrRows A, CsrRows B, CsrRows C, const Fr* w, uint32_t nc, unsigned long long* bad) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nc) return;
    r1cs_flag(row_dot(A.ptr, A.col, A.val, w, i), row_dot(B.ptr, B.col, B.val, w, i), row_dot(C.ptr, C.col, C.val, w, i), i, bad);
}

__global__ void __launch_bounds__(256) k_r1cs_check_warp(CsrRows A, CsrRows B, CsrRows C, const Fr* w, uint32_t nc,
                                                         unsigned long long* bad) {
    const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (i >= nc) return;                       // whole warps: nc x 32 lanes, so a warp never straddles the end
    const Fr a = row_dot_warp(A.ptr, A.col, A.val, w, i, lane);
    const Fr b = row_dot_warp(B.ptr, B.col, B.val, w, i, lane);
    const Fr c = row_dot_warp(C.ptr, C.col, C.val, w, i, lane);
    if (lane == 0) r1cs_flag(a, b, c, i, bad);
}

int r1cs_check_dev(b200zk_ctx* ctx, Slot& sl, const void* const ptr[3], const void* const col[3], const void* const val[3], size_t nc,
                   const void* d_w, uint64_t* n_failed, uint64_t* first_failed) {
    *n_failed = 0;
    *first_failed = nc;
    if (nc == 0) return B200ZK_OK;
    if (nc >= ((size_t)1 << 32)) return set_error(ctx, B200ZK_ERR_ARG, "r1cs_check: more than 2^32 - 1 constraints");
    CsrRows m[3];
    for (int k = 0; k < 3; ++k) m[k] = {(const uint32_t*)ptr[k], (const uint32_t*)col[k], (const Fr*)val[k]};
    B2_CUDA_OK(ctx, sl.small.reserve(1024));
    unsigned long long* bad = reinterpret_cast<unsigned long long*>(sl.small.p);
    B2_CUDA_OK(ctx, cudaMemsetAsync(bad, 0, 8, sl.stream));
    B2_CUDA_OK(ctx, cudaMemsetAsync(bad + 1, 0xFF, 8, sl.stream));
    {
        LaunchScope ls(ctx, sl.stream, "r1cs_check");
        if (nc <= ((size_t)1 << 18))           // the warp-per-row rule of qap_dev
            k_r1cs_check_warp<<<(unsigned)((nc * 32 + 255) / 256), 256, 0, sl.stream>>>(m[0], m[1], m[2], (const Fr*)d_w, (uint32_t)nc, bad);
        else
            k_r1cs_check<<<(unsigned)((nc + 127) / 128), 128, 0, sl.stream>>>(m[0], m[1], m[2], (const Fr*)d_w, (uint32_t)nc, bad);
    }
    B2_TRY(check_launch(ctx, "k_r1cs_check"));
    unsigned long long h_bad[2] = {0, 0};
    B2_CUDA_OK(ctx, cudaMemcpyAsync(h_bad, bad, 16, cudaMemcpyDeviceToHost, sl.stream));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(sl.stream));
    *n_failed = h_bad[0];
    if (h_bad[0]) *first_failed = h_bad[1];
    return B200ZK_OK;
}

}  // namespace b200zk
