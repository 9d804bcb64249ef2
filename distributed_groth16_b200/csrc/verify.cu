// verify.cu -- Groth16 verification on the device: e(A, B) == e(alpha, beta) e(sum_i x_i IC_i, gamma) e(C, delta).
//
// Replaces `Groth16::verify_with_processed_vk` as the reference calls it after every proof
// (/root/reference/groth16/examples/sha256.rs:229-254, mpc-api/src/main.rs:187-247).  One proof = four Miller loops and
// one final exponentiation (csrc/pairing.cuh): a latency-bound scalar computation, so the kernel is four warps with one
// active lane each for the Miller loops, and the first then multiplies them and runs the final exponentiation.
#include "common.cuh"
#include "pairing.cuh"

namespace b200zk {

struct VerifyArgs {
    const affine_t<Fq>* alpha_g1;
    const affine_t<Fq2>* beta_g2;
    const affine_t<Fq2>* gamma_g2;
    const affine_t<Fq2>* delta_g2;
    const affine_t<Fq>* ic;            // n_public + 1 points
    const Fr* x;                       // n_public public inputs (Montgomery)
    uint32_t n_public;
    const affine_t<Fq>* a;
    const affine_t<Fq2>* b;
    const affine_t<Fq>* c;
    uint32_t* result;                  // 1 = accept, 0 = reject
};

__global__ void __launch_bounds__(128) k_groth16_verify(VerifyArgs v) {
    __shared__ Fq12 ml[4];
    const int role = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
        affine_t<Fq> P;
        affine_t<Fq2> Q;
        if (role == 0) { P = *v.a; Q = *v.b; }
        else if (role == 1) { P = *v.alpha_g1; P.y = Fq::neg(P.y); Q = *v.beta_g2; }
        else if (role == 2) {
            xyzz_t<Fq> acc = xyzz_t<Fq>::from_affine(v.ic[0]);
            for (uint32_t i = 0; i < v.n_public; ++i) {
                Fr k = Fr::from_mont(v.x[i]);
                acc = xyzz_t<Fq>::add(acc, xyzz_t<Fq>::mul_scalar(xyzz_t<Fq>::from_affine(v.ic[i + 1]), k.l));
            }
            P = xyzz_t<Fq>::to_affine(acc);
            P.y = Fq::neg(P.y);
            Q = *v.gamma_g2;
        } else { P = *v.c; P.y = Fq::neg(P.y); Q = *v.delta_g2; }
        if (P.is_inf()) P = affine_t<Fq>::infinity();          // -(0,0) must stay the identity
        ml[role] = miller_loop(P, Q);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        Fq12 f = Fq12::mul(Fq12::mul(ml[0], ml[1]), Fq12::mul(ml[2], ml[3]));
        *v.result = final_exponentiation(f) == Fq12::one() ? 1u : 0u;
    }
}

int groth16_verify_dev(b200zk_ctx* ctx, Slot& sl, const uint64_t* alpha_g1, const uint64_t* beta_g2, const uint64_t* gamma_g2,
                       const uint64_t* delta_g2, const uint64_t* gamma_abc_g1, size_t n_public, const uint64_t* public_inputs,
                       const uint64_t* proof_a, const uint64_t* proof_b, const uint64_t* proof_c, int* is_valid) {
    if (n_public >= (1u << 20)) return set_error(ctx, B200ZK_ERR_ARG, "too many public inputs");
    cudaStream_t st = sl.stream;
    // staging block: alpha 64 | beta 128 | gamma 128 | delta 128 | A 64 | B 128 | C 64 | result 64 | ic | x
    const size_t o_alpha = 0, o_beta = 64, o_gamma = 192, o_delta = 320, o_a = 448, o_b = 512, o_c = 640, o_res = 704, o_ic = 768;
    const size_t o_x = o_ic + (n_public + 1) * 64;
    B2_CUDA_OK(ctx, sl.io_b.reserve(o_x + n_public * 32 + 64));
    char* d = reinterpret_cast<char*>(sl.io_b.p);
    auto up = [&](size_t off, const void* src, size_t bytes) { return cudaMemcpyAsync(d + off, src, bytes, cudaMemcpyHostToDevice, st); };
    B2_CUDA_OK(ctx, up(o_alpha, alpha_g1, 64));
    B2_CUDA_OK(ctx, up(o_beta, beta_g2, 128));
    B2_CUDA_OK(ctx, up(o_gamma, gamma_g2, 128));
    B2_CUDA_OK(ctx, up(o_delta, delta_g2, 128));
    B2_CUDA_OK(ctx, up(o_a, proof_a, 64));
    B2_CUDA_OK(ctx, up(o_b, proof_b, 128));
    B2_CUDA_OK(ctx, up(o_c, proof_c, 64));
    B2_CUDA_OK(ctx, up(o_ic, gamma_abc_g1, (n_public + 1) * 64));
    if (n_public) B2_CUDA_OK(ctx, up(o_x, public_inputs, n_public * 32));
    VerifyArgs v;
    v.alpha_g1 = reinterpret_cast<const affine_t<Fq>*>(d + o_alpha);
    v.beta_g2 = reinterpret_cast<const affine_t<Fq2>*>(d + o_beta);
    v.gamma_g2 = reinterpret_cast<const affine_t<Fq2>*>(d + o_gamma);
    v.delta_g2 = reinterpret_cast<const affine_t<Fq2>*>(d + o_delta);
    v.ic = reinterpret_cast<const affine_t<Fq>*>(d + o_ic);
    v.x = reinterpret_cast<const Fr*>(d + o_x);
    v.n_public = (uint32_t)n_public;
    v.a = reinterpret_cast<const affine_t<Fq>*>(d + o_a);
    v.b = reinterpret_cast<const affine_t<Fq2>*>(d + o_b);
    v.c = reinterpret_cast<const affine_t<Fq>*>(d + o_c);
    v.result = reinterpret_cast<uint32_t*>(d + o_res);
    {
        LaunchScope ls(ctx, st, "groth16_verify");
        k_groth16_verify<<<1, 128, 0, st>>>(v);
    }
    B2_TRY(check_launch(ctx, "k_groth16_verify"));
    uint32_t res = 0;
    B2_CUDA_OK(ctx, cudaMemcpyAsync(&res, d + o_res, 4, cudaMemcpyDeviceToHost, st));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(st));
    *is_valid = res ? 1 : 0;
    return B200ZK_OK;
}

// snarkjs's vk_alphabeta_12.  ffjavascript's final exponentiation computes the hard part with the Fuentes-Castaneda chain,
// which raises to m (p^4 - p^2 + 1)/r with m = 2u(6u^2 + 3u + 1), so snarkjs's e(alpha, beta) is the plain pairing of
// pairing.cuh raised to m.  m is 190 bits; SNARKJS_M holds it little-endian.
__constant__ uint64_t SNARKJS_M[3] = {0x2e5d4e223ddedaf4ull, 0x1ea96b02d9d9e38dull, 0x3bec47df15e307c8ull};
constexpr int SNARKJS_M_BITS = 190;

// One scalar computation: one thread.  out: the 12 Fq coefficients in snarkjs's nesting (c0.a, c0.b, c0.c, c1.a, c1.b,
// c1.c, each Fq2 as c0, c1), canonical.
__global__ void k_vk_alphabeta_12(const affine_t<Fq>* alpha, const affine_t<Fq2>* beta, Fq* out) {
    const Fq12 e = final_exponentiation(miller_loop(*alpha, *beta));
    Fq12 r = Fq12::one();
    for (int bit = SNARKJS_M_BITS - 1; bit >= 0; --bit) {
        r = Fq12::mul(r, r);
        if ((SNARKJS_M[bit >> 6] >> (bit & 63)) & 1) r = Fq12::mul(r, e);
    }
    const Fq2* c[6] = {&r.c0.a, &r.c0.b, &r.c0.c, &r.c1.a, &r.c1.b, &r.c1.c};
    for (int k = 0; k < 6; ++k) {
        out[2 * k] = Fq::from_mont(c[k]->c0);
        out[2 * k + 1] = Fq::from_mont(c[k]->c1);
    }
}

int vk_alphabeta_12_dev(b200zk_ctx* ctx, Slot& sl, const uint64_t* alpha_g1, const uint64_t* beta_g2, uint64_t* out) {
    cudaStream_t st = sl.stream;
    // staging block: alpha 64 | beta 128 | out 384
    B2_CUDA_OK(ctx, sl.io_b.reserve(576));
    char* d = reinterpret_cast<char*>(sl.io_b.p);
    B2_CUDA_OK(ctx, cudaMemcpyAsync(d, alpha_g1, 64, cudaMemcpyHostToDevice, st));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(d + 64, beta_g2, 128, cudaMemcpyHostToDevice, st));
    {
        LaunchScope ls(ctx, st, "vk_alphabeta_12");
        k_vk_alphabeta_12<<<1, 1, 0, st>>>(reinterpret_cast<const affine_t<Fq>*>(d), reinterpret_cast<const affine_t<Fq2>*>(d + 64),
                                            reinterpret_cast<Fq*>(d + 192));
    }
    B2_TRY(check_launch(ctx, "k_vk_alphabeta_12"));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(out, d + 192, 384, cudaMemcpyDeviceToHost, st));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(st));
    return B200ZK_OK;
}

}  // namespace b200zk
