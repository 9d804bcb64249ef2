// packexp.cu -- packed secret sharing "in the exponent" for whole vectors of curve points.
//
// `packexp_from_public` (/root/reference/dist-primitives/src/dmsm/mod.rs:50-68) maps l group elements to n = 4l shares by
// an inverse FFT over the `secret` coset followed by an FFT over the `share` domain; both are linear, so a chunk's shares
// are M * chunk for one fixed n x l matrix M of scalars (M = pack applied to the unit vectors).  The reference applies it
// chunk by chunk to every query vector of the proving key (groth16/src/proving_key.rs:35-110 -- its per-circuit CRS
// preprocessing); here all chunks of a vector are done in one launch, one thread per (chunk, share):
//   out[k * rows + j] = sum_i M[j][i] * points[k * l + i].
// The same kernel with the unpack matrix inverts it (`unpackexp`, dmsm/mod.rs:7-48).
#include "common.cuh"

namespace b200zk {

template <class F>
__global__ void __launch_bounds__(128) k_points_matmul(const affine_t<F>* points, uint32_t n_chunks, uint32_t l, const Fr* matrix,
                                                       uint32_t rows, affine_t<F>* out) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_chunks * rows) return;
    uint32_t k = t / rows, j = t % rows;
    xyzz_t<F> acc = xyzz_t<F>::identity();
    for (uint32_t i = 0; i < l; ++i) {
        affine_t<F> p = points[(size_t)k * l + i];
        if (p.is_inf()) continue;
        Fr s = Fr::from_mont(matrix[(size_t)j * l + i]);
        acc = xyzz_t<F>::add(acc, xyzz_t<F>::mul_scalar(xyzz_t<F>::from_affine(p), s.l));
    }
    out[t] = xyzz_t<F>::to_affine(acc);
}

int points_matmul_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_points, size_t n_chunks, size_t l, const void* d_matrix,
                      size_t rows, void* d_out) {
    if (n_chunks == 0 || rows == 0) return B200ZK_OK;
    if (l == 0 || l > 1024 || rows > 4096 || n_chunks * rows >= (1ull << 32))
        return set_error(ctx, B200ZK_ERR_ARG, "points_matmul: need 1 <= l <= 1024, rows <= 4096, n_chunks * rows < 2^32");
    unsigned grid = (unsigned)((n_chunks * rows + 127) / 128);
    if (g2)
        return launch(ctx, sl.stream, "points_matmul", k_points_matmul<Fq2>, grid, 128, 0, reinterpret_cast<const affine_t<Fq2>*>(d_points),
                      (uint32_t)n_chunks, (uint32_t)l, reinterpret_cast<const Fr*>(d_matrix), (uint32_t)rows,
                      reinterpret_cast<affine_t<Fq2>*>(d_out));
    return launch(ctx, sl.stream, "points_matmul", k_points_matmul<Fq>, grid, 128, 0, reinterpret_cast<const affine_t<Fq>*>(d_points),
                  (uint32_t)n_chunks, (uint32_t)l, reinterpret_cast<const Fr*>(d_matrix), (uint32_t)rows,
                  reinterpret_cast<affine_t<Fq>*>(d_out));
}

}  // namespace b200zk
