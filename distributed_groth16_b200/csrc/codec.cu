// codec.cu -- batch (de)compression of BN254 points in ark-serialize `Compress::Yes` form.
//
// The reference moves every proving / verifying key and proof through `CanonicalSerialize` with compression
// (/root/reference/common/src/utils/serializer.rs:20-49; `proving_key.bin` written at mpc-api/src/main.rs:161-165,
// proofs at zk-cli/src/main.rs:130-136).  Encoding (SURVEY 8c, pinned on zk-cli/test-circuits/sha256/proof.bin):
//   G1: x as 32 little-endian bytes; top two bits of the last byte are flags: 0x80 = y is the larger of (y, -y),
//       0x40 = point at infinity (all other bits zero).
//   G2: x.c0 then x.c1 (32 bytes each), flags in the last byte of x.c1; Fq2 order compares c1 first, then c0.
// Decompression needs one square root per point (p = 3 mod 4: a^((p+1)/4), 253 squarings + ~127 products), which
// for a 2^20-constraint key is ~5 * 2^20 independent exponentiations: a data-parallel kernel, one thread per point.
#include "common.cuh"
#include "codec.cuh"

namespace b200zk {

__global__ void __launch_bounds__(128) k_g1_compress(const affine_t<Fq>* in, uint32_t n, uint8_t* out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    __align__(16) uint8_t b[32];
    g1_encode(in[i], b);
    uint4* o = reinterpret_cast<uint4*>(out + (size_t)i * 32);
    o[0] = *reinterpret_cast<uint4*>(b);
    o[1] = *reinterpret_cast<uint4*>(b + 16);
}

__global__ void __launch_bounds__(128) k_g2_compress(const affine_t<Fq2>* in, uint32_t n, uint8_t* out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    __align__(16) uint8_t b[64];
    g2_encode(in[i], b);
    uint4* o = reinterpret_cast<uint4*>(out + (size_t)i * 64);
    for (int k = 0; k < 4; ++k) o[k] = *reinterpret_cast<uint4*>(b + 16 * k);
}

// bad[0] += 1 for every encoding that is not a point (x >= p, x not on the curve, infinity flag with other bits set,
// or -- G2 with check_subgroup -- a twist point outside the order-r subgroup); its slot is left as infinity.
__global__ void __launch_bounds__(128) k_g1_decompress(const uint8_t* in, uint32_t n, affine_t<Fq>* out, uint32_t* bad) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    affine_t<Fq> p;
    if (!g1_decode(in + (size_t)i * 32, &p)) atomicAdd(bad, 1u);
    out[i] = p;
}

__global__ void __launch_bounds__(128) k_g2_decompress(const uint8_t* in, uint32_t n, int check_subgroup, affine_t<Fq2>* out,
                                                       uint32_t* bad) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    affine_t<Fq2> p;
    if (!g2_decode(in + (size_t)i * 64, check_subgroup != 0, &p)) atomicAdd(bad, 1u);
    out[i] = p;
}

int points_compress_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_affine, size_t n, void* d_bytes) {
    if (n == 0) return B200ZK_OK;
    if (n >= (1ull << 32)) return set_error(ctx, B200ZK_ERR_ARG, "too many points");
    const unsigned grid = (unsigned)((n + 127) / 128);
    if (g2)
        return launch(ctx, sl.stream, "points_compress", k_g2_compress, grid, 128, 0, reinterpret_cast<const affine_t<Fq2>*>(d_affine),
                      (uint32_t)n, (uint8_t*)d_bytes);
    return launch(ctx, sl.stream, "points_compress", k_g1_compress, grid, 128, 0, reinterpret_cast<const affine_t<Fq>*>(d_affine),
                  (uint32_t)n, (uint8_t*)d_bytes);
}

// ffjavascript encodings (codec.cuh ffjs_encode): the bytes a phase-1 contribution hashes, about 2.4 GB at power 22 --
// one thread per point, since leaving Montgomery form is a field product per coordinate
template <class F, bool COMPRESSED>
__global__ void __launch_bounds__(128) k_points_encode(const affine_t<F>* in, size_t n, uint8_t* out) {
    constexpr int LEN = (COMPRESSED ? 1 : 2) * (int)sizeof(F);
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    __align__(16) uint8_t b[LEN];
    ffjs_encode<F, COMPRESSED>(ld16(in + i), b);
    uint4* o = reinterpret_cast<uint4*>(out + i * LEN);
#pragma unroll
    for (int k = 0; k < LEN / 16; ++k) o[k] = *reinterpret_cast<const uint4*>(b + 16 * k);
}

int points_encode_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_affine, size_t n, int fmt, void* d_bytes) {
    if (fmt != 0 && fmt != 1) return set_error(ctx, B200ZK_ERR_ARG, "points_encode: fmt must be 0 (uncompressed) or 1 (compressed)");
    if (n == 0) return B200ZK_OK;
    if (n >= ((size_t)1 << 31) * 128) return set_error(ctx, B200ZK_ERR_ARG, "points_encode: too many points");
    const unsigned grid = (unsigned)((n + 127) / 128);
    uint8_t* out = (uint8_t*)d_bytes;
    if (g2) {
        const affine_t<Fq2>* in = reinterpret_cast<const affine_t<Fq2>*>(d_affine);
        return launch(ctx, sl.stream, "points_encode", fmt ? k_points_encode<Fq2, true> : k_points_encode<Fq2, false>, grid, 128, 0, in, n,
                      out);
    }
    const affine_t<Fq>* in = reinterpret_cast<const affine_t<Fq>*>(d_affine);
    return launch(ctx, sl.stream, "points_encode", fmt ? k_points_encode<Fq, true> : k_points_encode<Fq, false>, grid, 128, 0, in, n, out);
}

// The inverse (codec.cuh ffjs_decode): one square root per compressed point, one curve-equation check per uncompressed
// one, and with check_subgroup a 254-bit ladder per G2 point.  bad[0] counts the invalid encodings, bad[1] keeps the
// lowest invalid index; an invalid slot is left at infinity.
template <class F, bool COMPRESSED>
__global__ void __launch_bounds__(128) k_points_decode(const uint8_t* in, size_t n, int check_subgroup, affine_t<F>* out,
                                                       unsigned long long* bad) {
    constexpr int LEN = (COMPRESSED ? 1 : 2) * (int)sizeof(F);
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    __align__(16) uint8_t b[LEN];
    const uint4* s = reinterpret_cast<const uint4*>(in + i * LEN);
#pragma unroll
    for (int k = 0; k < LEN / 16; ++k) *reinterpret_cast<uint4*>(b + 16 * k) = s[k];
    affine_t<F> p;
    if (!ffjs_decode<F, COMPRESSED>(b, check_subgroup != 0, &p)) {
        atomicAdd(&bad[0], 1ull);
        atomicMin(&bad[1], (unsigned long long)i);
    }
    st16(out + i, p);
}

int points_decode_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_bytes, size_t n, int fmt, int check_subgroup,
                      void* d_affine, size_t* n_invalid, size_t* first_invalid) {
    if (n_invalid) *n_invalid = 0;
    if (first_invalid) *first_invalid = n;
    if (fmt != 0 && fmt != 1) return set_error(ctx, B200ZK_ERR_ARG, "points_decode: fmt must be 0 (uncompressed) or 1 (compressed)");
    if (n == 0) return B200ZK_OK;
    if (n >= ((size_t)1 << 31) * 128) return set_error(ctx, B200ZK_ERR_ARG, "points_decode: too many points");
    if (((uintptr_t)d_bytes | (uintptr_t)d_affine) & 15)
        return set_error(ctx, B200ZK_ERR_ARG, "points_decode: the encodings and the points must be 16-byte aligned");
    B2_CUDA_OK(ctx, sl.small.reserve(1024));
    unsigned long long* bad = reinterpret_cast<unsigned long long*>(sl.small.p);
    B2_CUDA_OK(ctx, cudaMemsetAsync(bad, 0, 8, sl.stream));
    B2_CUDA_OK(ctx, cudaMemsetAsync(bad + 1, 0xFF, 8, sl.stream));
    const unsigned grid = (unsigned)((n + 127) / 128);
    const uint8_t* in = (const uint8_t*)d_bytes;
    if (g2)
        B2_TRY(launch(ctx, sl.stream, "points_decode", fmt ? k_points_decode<Fq2, true> : k_points_decode<Fq2, false>, grid, 128, 0, in, n,
                      check_subgroup, reinterpret_cast<affine_t<Fq2>*>(d_affine), bad));
    else
        B2_TRY(launch(ctx, sl.stream, "points_decode", fmt ? k_points_decode<Fq, true> : k_points_decode<Fq, false>, grid, 128, 0, in, n,
                      check_subgroup, reinterpret_cast<affine_t<Fq>*>(d_affine), bad));
    unsigned long long h_bad[2] = {0, 0};
    B2_CUDA_OK(ctx, cudaMemcpyAsync(h_bad, bad, 16, cudaMemcpyDeviceToHost, sl.stream));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(sl.stream));
    if (n_invalid) *n_invalid = (size_t)h_bad[0];
    if (h_bad[0]) {
        if (first_invalid) *first_invalid = (size_t)h_bad[1];
        char msg[128];
        snprintf(msg, sizeof(msg), "points_decode: %llu of %zu encodings are not valid points, the first at index %llu", h_bad[0],
                 n, h_bad[1]);
        return set_error(ctx, B200ZK_ERR_ARG, msg);
    }
    return B200ZK_OK;
}

int points_decompress_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_bytes, size_t n, int check_subgroup, void* d_affine,
                          size_t* n_invalid) {
    if (n_invalid) *n_invalid = 0;
    if (n == 0) return B200ZK_OK;
    if (n >= (1ull << 32)) return set_error(ctx, B200ZK_ERR_ARG, "too many points");
    B2_CUDA_OK(ctx, sl.small.reserve(1024));
    uint32_t* bad = reinterpret_cast<uint32_t*>(sl.small.p);
    B2_CUDA_OK(ctx, cudaMemsetAsync(bad, 0, 4, sl.stream));
    const unsigned grid = (unsigned)((n + 127) / 128);
    if (g2)
        B2_TRY(launch(ctx, sl.stream, "points_decompress", k_g2_decompress, grid, 128, 0, (const uint8_t*)d_bytes, (uint32_t)n,
                      check_subgroup, reinterpret_cast<affine_t<Fq2>*>(d_affine), bad));
    else
        B2_TRY(launch(ctx, sl.stream, "points_decompress", k_g1_decompress, grid, 128, 0, (const uint8_t*)d_bytes, (uint32_t)n,
                      reinterpret_cast<affine_t<Fq>*>(d_affine), bad));
    uint32_t h_bad = 0;
    B2_CUDA_OK(ctx, cudaMemcpyAsync(&h_bad, bad, 4, cudaMemcpyDeviceToHost, sl.stream));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(sl.stream));
    if (n_invalid) *n_invalid = h_bad;
    if (h_bad) {
        char msg[96];
        snprintf(msg, sizeof(msg), "%u of %zu encodings are not valid curve points", h_bad, n);
        return set_error(ctx, B200ZK_ERR_ARG, msg);
    }
    return B200ZK_OK;
}

}  // namespace b200zk
