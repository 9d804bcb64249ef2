// selftest.cu -- b200zk_test_arith: the device field, tower and group primitives one element at a time, for the exact tests
// (tests/test_gpu_arith_exact.py against Python big integers, tests/arith_oracle.py).
//
// Every op reads a fixed record of u64 words per element and writes a fixed record (table below and in include/b200zk.h).
// Field elements are the raw Montgomery limbs the product kernels hold (4 words; Fq2 8, Fq6 24, Fq12 48), points are
// affine_t (G1 8 words, G2 16) or xyzz_t (G1 16, G2 32).  Each op's body is one host+device function arith_apply<OP>, so
// tests/host/arith_host_test.cpp runs the same bodies through g++ (PTX carry chain emulated); the kernels run them on the
// device, one small kernel per op so that each keeps the register allocation of its own body.  Device only: the root of
// unity (fr_root_of_unity) and the quad-cooperative group law (quad_ops).
#include <type_traits>

#include "codec.cuh"
#include "glv.cuh"
#include "pairing.cuh"
#ifdef __CUDACC__
#include "common.cuh"
#endif

namespace b200zk {

// op numbers.  Fp ops: ARITH_FQ + s on Fq, ARITH_FR + s on Fr.
enum {
    ARITH_FQ = 0, ARITH_FR = 32,
    FP_ADD = 0, FP_SUB, FP_NEG, FP_DBL, FP_MUL, FP_MUL_NI, FP_SQR, FP_MUL_ANY, FP_MUL_K2, FP_MUL_K3, FP_MUL_K4,
    FP_MUL_WIDE_REDC1, FP_REDC2, FP_INV, FP_INV_FERMAT, FP_TO_MONT, FP_FROM_MONT, FP_FROM_U32, FP_POW_U64,
    ARITH_FR_ROOT = 64,
    ARITH_FQ2_MUL = 70, ARITH_FQ2_SQR, ARITH_FQ2_INV, ARITH_FQ2_MUL_GROUP1, ARITH_FQ2_MUL_GROUP2, ARITH_FQ2_MUL_GROUP3,
    ARITH_FQ2_MUL_GROUP4, ARITH_FQ2_MUL_XI, ARITH_FQ2_CONJ, ARITH_GLV_PHI_G1, ARITH_GLV_PHI_G2,
    ARITH_FQ_POW_P1_4 = 84, ARITH_FQ_SQRT, ARITH_FQ2_SQRT, ARITH_FQ_HALF, ARITH_FQ_IS_LARGER, ARITH_FQ2_IS_LARGER,
    ARITH_FQ_FROM_BYTES,
    ARITH_FQ6_MUL = 96, ARITH_FQ6_INV, ARITH_FQ6_MUL_V, ARITH_FQ12_MUL, ARITH_FQ12_INV, ARITH_FQ12_CONJ, ARITH_FQ12_FROB2,
    ARITH_FINAL_EXP, ARITH_PAIRING, ARITH_G2_FROBENIUS_TWIST,
    ARITH_GLV_DECOMPOSE = 108,
    // group law: ARITH_G1 + s on G1, ARITH_G2 + s on G2
    ARITH_G1 = 112, ARITH_G2 = 128,
    EC_DBL = 0, EC_ADD, EC_DBL_ILP, EC_ADD_ILP, EC_MADD, EC_DBL_AFFINE, EC_TO_AFFINE, EC_MUL_SCALAR,
    EC_QUAD_ADD, EC_QUAD_DBL, EC_QUAD_ADD_FULLWARP, EC_QUAD_DBL_FULLWARP,
};

// record sizes in u64 words: X(op, in, out) for the ops with a host+device body
#define B2_ARITH_FP_OPS(X, B)                                                                                             \
    X(B + FP_ADD, 8, 4) X(B + FP_SUB, 8, 4) X(B + FP_NEG, 4, 4) X(B + FP_DBL, 4, 4) X(B + FP_MUL, 8, 4)                   \
    X(B + FP_MUL_NI, 8, 4) X(B + FP_SQR, 4, 4) X(B + FP_MUL_ANY, 8, 4) X(B + FP_MUL_K2, 16, 8) X(B + FP_MUL_K3, 24, 12)   \
    X(B + FP_MUL_K4, 32, 16) X(B + FP_MUL_WIDE_REDC1, 8, 12) X(B + FP_REDC2, 8, 4) X(B + FP_INV, 4, 4)                   \
    X(B + FP_INV_FERMAT, 4, 4) X(B + FP_TO_MONT, 4, 4) X(B + FP_FROM_MONT, 4, 4) X(B + FP_FROM_U32, 1, 4)                \
    X(B + FP_POW_U64, 5, 4)
#define B2_ARITH_EC_OPS(X, B, W)                                                                                          \
    X(B + EC_DBL, 4 * W, 4 * W) X(B + EC_ADD, 8 * W, 4 * W) X(B + EC_DBL_ILP, 4 * W, 4 * W) X(B + EC_ADD_ILP, 8 * W, 4 * W) \
    X(B + EC_MADD, 6 * W + 1, 4 * W) X(B + EC_DBL_AFFINE, 2 * W, 4 * W) X(B + EC_TO_AFFINE, 4 * W, 2 * W)                \
    X(B + EC_MUL_SCALAR, 4 * W + 4, 4 * W)
#define B2_ARITH_OPS(X)                                                                                                   \
    B2_ARITH_FP_OPS(X, ARITH_FQ) B2_ARITH_FP_OPS(X, ARITH_FR)                                                             \
    X(ARITH_FQ2_MUL, 16, 8) X(ARITH_FQ2_SQR, 8, 8) X(ARITH_FQ2_INV, 8, 8) X(ARITH_FQ2_MUL_GROUP1, 16, 8)                  \
    X(ARITH_FQ2_MUL_GROUP2, 32, 16) X(ARITH_FQ2_MUL_GROUP3, 48, 24) X(ARITH_FQ2_MUL_GROUP4, 64, 32)                      \
    X(ARITH_FQ2_MUL_XI, 8, 8) X(ARITH_FQ2_CONJ, 8, 8) X(ARITH_GLV_PHI_G1, 4, 4) X(ARITH_GLV_PHI_G2, 8, 8)                 \
    X(ARITH_FQ_POW_P1_4, 4, 4) X(ARITH_FQ_SQRT, 4, 5) X(ARITH_FQ2_SQRT, 8, 9) X(ARITH_FQ_HALF, 4, 4)                      \
    X(ARITH_FQ_IS_LARGER, 4, 1) X(ARITH_FQ2_IS_LARGER, 8, 1) X(ARITH_FQ_FROM_BYTES, 5, 5)                                \
    X(ARITH_FQ6_MUL, 48, 24) X(ARITH_FQ6_INV, 24, 24) X(ARITH_FQ6_MUL_V, 24, 24) X(ARITH_FQ12_MUL, 96, 48)                \
    X(ARITH_FQ12_INV, 48, 48) X(ARITH_FQ12_CONJ, 48, 48) X(ARITH_FQ12_FROB2, 48, 48) X(ARITH_FINAL_EXP, 48, 48)           \
    X(ARITH_PAIRING, 24, 48) X(ARITH_G2_FROBENIUS_TWIST, 16, 16) X(ARITH_GLV_DECOMPOSE, 4, 6)                            \
    B2_ARITH_EC_OPS(X, ARITH_G1, 4) B2_ARITH_EC_OPS(X, ARITH_G2, 8)
// device only: X(op, in, out)
#define B2_ARITH_DEVICE_OPS(X)                                                                                            \
    X(ARITH_FR_ROOT, 1, 4)                                                                                                \
    X(ARITH_G1 + EC_QUAD_ADD, 32, 16) X(ARITH_G1 + EC_QUAD_DBL, 16, 16) X(ARITH_G1 + EC_QUAD_ADD_FULLWARP, 32, 16)       \
    X(ARITH_G1 + EC_QUAD_DBL_FULLWARP, 16, 16) X(ARITH_G2 + EC_QUAD_ADD, 64, 32) X(ARITH_G2 + EC_QUAD_DBL, 32, 32)       \
    X(ARITH_G2 + EC_QUAD_ADD_FULLWARP, 64, 32) X(ARITH_G2 + EC_QUAD_DBL_FULLWARP, 32, 32)

// (in, out) words of `op`; (0, 0) when there is no such op
B2_HD void arith_words(int op, int* in, int* out) {
    *in = 0; *out = 0;
    switch (op) {
#define B2_ARITH_WORDS(OP, IN, OUT) case OP: *in = IN; *out = OUT; break;
        B2_ARITH_OPS(B2_ARITH_WORDS)
        B2_ARITH_DEVICE_OPS(B2_ARITH_WORDS)
#undef B2_ARITH_WORDS
        default: break;
    }
}

// a field element / point / tower element <-> its u64 words (the memory image of the 32-bit limbs)
template <class T>
B2_HD T arith_ld(const uint64_t* w) {
    T r;
    uint32_t* d = reinterpret_cast<uint32_t*>(&r);
    for (int i = 0; i < (int)(sizeof(T) / 4); ++i) d[i] = (uint32_t)(w[i >> 1] >> (32 * (i & 1)));
    return r;
}
template <class T>
B2_HD void arith_st(uint64_t* w, const T& v) {
    const uint32_t* s = reinterpret_cast<const uint32_t*>(&v);
    for (int i = 0; i < (int)(sizeof(T) / 8); ++i) w[i] = (uint64_t)s[2 * i] | (uint64_t)s[2 * i + 1] << 32;
}
B2_HD void arith_st_limbs(uint64_t* w, const uint32_t* l, int n32) {
    for (int i = 0; i < n32 / 2; ++i) w[i] = (uint64_t)l[2 * i] | (uint64_t)l[2 * i + 1] << 32;
}

template <class F, int S>
B2_HD void arith_fp(const uint64_t* in, uint64_t* out) {
    if constexpr (S == FP_ADD) arith_st(out, F::add(arith_ld<F>(in), arith_ld<F>(in + 4)));
    else if constexpr (S == FP_SUB) arith_st(out, F::sub(arith_ld<F>(in), arith_ld<F>(in + 4)));
    else if constexpr (S == FP_NEG) arith_st(out, F::neg(arith_ld<F>(in)));
    else if constexpr (S == FP_DBL) arith_st(out, F::dbl(arith_ld<F>(in)));
    else if constexpr (S == FP_MUL || S == FP_MUL_ANY) arith_st(out, F::mul(arith_ld<F>(in), arith_ld<F>(in + 4)));
    else if constexpr (S == FP_MUL_NI) arith_st(out, F::mul_ni(arith_ld<F>(in), arith_ld<F>(in + 4)));
    else if constexpr (S == FP_SQR) arith_st(out, F::sqr(arith_ld<F>(in)));
    else if constexpr (S == FP_MUL_K2 || S == FP_MUL_K3 || S == FP_MUL_K4) {
        constexpr int K = S - FP_MUL_K2 + 2;                // K (a, b) pairs in, K products out
        F a[K], b[K], r[K];
        for (int k = 0; k < K; ++k) { a[k] = arith_ld<F>(in + 8 * k); b[k] = arith_ld<F>(in + 8 * k + 4); }
        F::template mul_k<K>(r, a, b);
        for (int k = 0; k < K; ++k) arith_st(out + 4 * k, r[k]);
    } else if constexpr (S == FP_MUL_WIDE_REDC1) {          // out: the 512-bit product, then its reduction
        const F a = arith_ld<F>(in), b = arith_ld<F>(in + 4);
        uint32_t t[16];
        F::mul_wide(t, a.l, b.l);
        F r;
        F::template redc<1>(r, t);
        arith_st_limbs(out, t, 16);
        arith_st(out + 8, r);
    } else if constexpr (S == FP_REDC2) {                   // in: a 512-bit t < 2 p 2^256
        uint32_t t[16];
        for (int i = 0; i < 16; ++i) t[i] = (uint32_t)(in[i >> 1] >> (32 * (i & 1)));
        F r;
        F::template redc<2>(r, t);
        arith_st(out, r);
    } else if constexpr (S == FP_INV) arith_st(out, F::inv(arith_ld<F>(in)));
    else if constexpr (S == FP_INV_FERMAT) arith_st(out, F::inv_fermat(arith_ld<F>(in)));
    else if constexpr (S == FP_TO_MONT) arith_st(out, F::to_mont(arith_ld<F>(in)));
    else if constexpr (S == FP_FROM_MONT) arith_st(out, F::from_mont(arith_ld<F>(in)));
    else if constexpr (S == FP_FROM_U32) arith_st(out, F::from_u32((uint32_t)in[0]));
    else if constexpr (S == FP_POW_U64) arith_st(out, F::pow_u64(arith_ld<F>(in), in[4]));
    else static_assert(S < 0, "no such Fp op");
}

template <class F, int S>
B2_HD void arith_ec(const uint64_t* in, uint64_t* out) {
    typedef xyzz_t<F> X;
    typedef affine_t<F> A;
    constexpr int XW = (int)sizeof(X) / 8, AW = (int)sizeof(A) / 8;
    if constexpr (S == EC_DBL) arith_st(out, X::dbl(arith_ld<X>(in)));
    else if constexpr (S == EC_ADD) arith_st(out, X::add(arith_ld<X>(in), arith_ld<X>(in + XW)));
    else if constexpr (S == EC_DBL_ILP) arith_st(out, X::dbl_ilp(arith_ld<X>(in)));
    else if constexpr (S == EC_ADD_ILP) arith_st(out, X::add_ilp(arith_ld<X>(in), arith_ld<X>(in + XW)));
    else if constexpr (S == EC_MADD) {                      // in: acc, p, negate
        X acc = arith_ld<X>(in);
        X::madd(acc, arith_ld<A>(in + XW), in[XW + AW] != 0);
        arith_st(out, acc);
    } else if constexpr (S == EC_DBL_AFFINE) {
        const A p = arith_ld<A>(in);
        arith_st(out, X::dbl_affine(p.x, p.y));
    } else if constexpr (S == EC_TO_AFFINE) arith_st(out, X::to_affine(arith_ld<X>(in)));
    else if constexpr (S == EC_MUL_SCALAR) {                // in: p, then k as 4 canonical words (any value < 2^256)
        uint32_t k[8];
        for (int i = 0; i < 8; ++i) k[i] = (uint32_t)(in[XW + (i >> 1)] >> (32 * (i & 1)));
        arith_st(out, X::mul_scalar(arith_ld<X>(in), k));
    } else static_assert(S < 0, "no such group op");
}

template <class T>
B2_HD void arith_st_flag(uint64_t* out, bool flag, const T& v) {
    out[0] = flag ? 1 : 0;
    arith_st(out + 1, v);
}

template <int OP>
B2_HD void arith_apply(const uint64_t* in, uint64_t* out) {
    if constexpr (OP < ARITH_FR) arith_fp<Fq, OP - ARITH_FQ>(in, out);
    else if constexpr (OP < ARITH_FR_ROOT) arith_fp<Fr, OP - ARITH_FR>(in, out);
    else if constexpr (OP == ARITH_FQ2_MUL) arith_st(out, Fq2::mul(arith_ld<Fq2>(in), arith_ld<Fq2>(in + 8)));
    else if constexpr (OP == ARITH_FQ2_SQR) arith_st(out, Fq2::sqr(arith_ld<Fq2>(in)));
    else if constexpr (OP == ARITH_FQ2_INV) arith_st(out, Fq2::inv(arith_ld<Fq2>(in)));
    else if constexpr (OP >= ARITH_FQ2_MUL_GROUP1 && OP <= ARITH_FQ2_MUL_GROUP4) {
        constexpr int K = OP - ARITH_FQ2_MUL_GROUP1 + 1;    // K (a, b) pairs in, K products out
        Fq2 a[K], b[K], r[K];
        for (int k = 0; k < K; ++k) { a[k] = arith_ld<Fq2>(in + 16 * k); b[k] = arith_ld<Fq2>(in + 16 * k + 8); }
        Fq2::mul_group<K>(r, a, b);
        for (int k = 0; k < K; ++k) arith_st(out + 8 * k, r[k]);
    } else if constexpr (OP == ARITH_FQ2_MUL_XI) arith_st(out, fq2_mul_xi(arith_ld<Fq2>(in)));
    else if constexpr (OP == ARITH_FQ2_CONJ) arith_st(out, fq2_conj(arith_ld<Fq2>(in)));
    else if constexpr (OP == ARITH_GLV_PHI_G1) { Fq x = arith_ld<Fq>(in); glv_phi_x(x); arith_st(out, x); }
    else if constexpr (OP == ARITH_GLV_PHI_G2) { Fq2 x = arith_ld<Fq2>(in); glv_phi_x(x); arith_st(out, x); }
    else if constexpr (OP == ARITH_FQ_POW_P1_4) arith_st(out, fq_pow_p1_4(arith_ld<Fq>(in)));
    else if constexpr (OP == ARITH_FQ_SQRT) {                // out: flag, root
        Fq s = Fq::zero();
        const bool ok = fq_sqrt(arith_ld<Fq>(in), &s);
        arith_st_flag(out, ok, s);
    } else if constexpr (OP == ARITH_FQ2_SQRT) {             // out: flag, root (zero where fq2_sqrt leaves it untouched)
        Fq2 s = Fq2::zero();
        const bool ok = fq2_sqrt(arith_ld<Fq2>(in), &s);
        arith_st_flag(out, ok, s);
    } else if constexpr (OP == ARITH_FQ_HALF) arith_st(out, fq_half(arith_ld<Fq>(in)));
    else if constexpr (OP == ARITH_FQ_IS_LARGER) out[0] = fq_is_larger(arith_ld<Fq>(in)) ? 1 : 0;
    else if constexpr (OP == ARITH_FQ2_IS_LARGER) out[0] = fq2_is_larger(arith_ld<Fq2>(in)) ? 1 : 0;
    else if constexpr (OP == ARITH_FQ_FROM_BYTES) {          // in: 32 little-endian bytes, top_mask; out: flag, value
        uint8_t b[32];
        for (int i = 0; i < 32; ++i) b[i] = (uint8_t)(in[i >> 3] >> (8 * (i & 7)));
        Fq x;
        const bool ok = fq_from_bytes(b, (uint8_t)in[4], &x);
        arith_st_flag(out, ok, x);
    } else if constexpr (OP == ARITH_FQ6_MUL) arith_st(out, Fq6::mul(arith_ld<Fq6>(in), arith_ld<Fq6>(in + 24)));
    else if constexpr (OP == ARITH_FQ6_INV) arith_st(out, Fq6::inv(arith_ld<Fq6>(in)));
    else if constexpr (OP == ARITH_FQ6_MUL_V) arith_st(out, Fq6::mul_v(arith_ld<Fq6>(in)));
    else if constexpr (OP == ARITH_FQ12_MUL) arith_st(out, Fq12::mul(arith_ld<Fq12>(in), arith_ld<Fq12>(in + 48)));
    else if constexpr (OP == ARITH_FQ12_INV) arith_st(out, Fq12::inv(arith_ld<Fq12>(in)));
    else if constexpr (OP == ARITH_FQ12_CONJ) arith_st(out, Fq12::conj(arith_ld<Fq12>(in)));
    else if constexpr (OP == ARITH_FQ12_FROB2) arith_st(out, Fq12::frob2(arith_ld<Fq12>(in)));
    else if constexpr (OP == ARITH_FINAL_EXP) arith_st(out, final_exponentiation(arith_ld<Fq12>(in)));
    else if constexpr (OP == ARITH_PAIRING)                  // in: P (G1 affine), Q (G2 affine)
        arith_st(out, final_exponentiation(miller_loop(arith_ld<affine_t<Fq>>(in), arith_ld<affine_t<Fq2>>(in + 8))));
    else if constexpr (OP == ARITH_G2_FROBENIUS_TWIST) arith_st(out, g2_frobenius_twist(arith_ld<affine_t<Fq2>>(in)));
    else if constexpr (OP == ARITH_GLV_DECOMPOSE) {          // in: canonical k < r; out: |k1| (2 words), neg1, |k2|, neg2
        uint32_t k[8];
        for (int i = 0; i < 8; ++i) k[i] = (uint32_t)(in[i >> 1] >> (32 * (i & 1)));
        const GlvSplit s = glv_decompose(k);
        arith_st_limbs(out, s.k1, 4);
        out[2] = s.neg1 ? 1 : 0;
        arith_st_limbs(out + 3, s.k2, 4);
        out[5] = s.neg2 ? 1 : 0;
    } else if constexpr (OP >= ARITH_G1 && OP < ARITH_G2) arith_ec<Fq, OP - ARITH_G1>(in, out);
    else if constexpr (OP >= ARITH_G2) arith_ec<Fq2, OP - ARITH_G2>(in, out);
    else static_assert(OP < 0, "no such op");
}

#ifdef __CUDACC__
constexpr int ARITH_BLOCK = 128;

template <int OP>
__global__ void __launch_bounds__(ARITH_BLOCK) k_arith(const uint64_t* in, uint64_t* out, size_t n, int in_w, int out_w) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    arith_apply<OP>(in + i * in_w, out + i * out_w);
}

__global__ void __launch_bounds__(ARITH_BLOCK) k_arith_fr_root(const uint64_t* in, uint64_t* out, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;                                       // in: log_n | inverse << 8
    arith_st(out + 4 * i, fr_root_of_unity((unsigned)(in[i] & 0xFF), ((in[i] >> 8) & 1) != 0));
}

// quad_ops<F, false>: element i on the quad of threads 4 i .. 4 i + 3; quad_ops<F, true>: element i on warp i, all 32 lanes
// with the same operands.  Each quad has its own exchange area; lane 0 of the quad / warp writes the result.
template <class F, bool FULLWARP, bool DBL>
__global__ void __launch_bounds__(ARITH_BLOCK) k_arith_quad(const uint64_t* in, uint64_t* out, size_t n) {
    typedef quad_ops<F, FULLWARP> Q;
    typedef xyzz_t<F> X;
    constexpr int XW = (int)sizeof(X) / 8;
    __shared__ __align__(16) typename Q::xch_t xch[ARITH_BLOCK / 4];
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t i = FULLWARP ? t >> 5 : t >> 2;
    if (i >= n) return;                                       // uniform over the quad / warp
    typename Q::xch_t* x = &xch[threadIdx.x >> 2];
    const uint64_t* r = in + i * (DBL ? XW : 2 * XW);
    const X res = DBL ? Q::dbl(x, arith_ld<X>(r)) : Q::add(x, arith_ld<X>(r), arith_ld<X>(r + XW));
    if ((threadIdx.x & (FULLWARP ? 31u : 3u)) == 0) arith_st(out + i * XW, res);
}

static int arith_launch(b200zk_ctx* ctx, Slot& sl, int op, const uint64_t* d_in, uint64_t* d_out, size_t n, int in_w,
                        int out_w) {
    const unsigned grid1 = (unsigned)((n + ARITH_BLOCK - 1) / ARITH_BLOCK);
    const unsigned grid4 = (unsigned)((4 * n + ARITH_BLOCK - 1) / ARITH_BLOCK);
    const unsigned grid32 = (unsigned)((32 * n + ARITH_BLOCK - 1) / ARITH_BLOCK);
    LaunchScope ls(ctx, sl.stream, "arith");
    switch (op) {
#define B2_ARITH_CASE(OP, IN, OUT) \
        case OP: k_arith<OP><<<grid1, ARITH_BLOCK, 0, sl.stream>>>(d_in, d_out, n, in_w, out_w); break;
        B2_ARITH_OPS(B2_ARITH_CASE)
#undef B2_ARITH_CASE
        case ARITH_FR_ROOT: k_arith_fr_root<<<grid1, ARITH_BLOCK, 0, sl.stream>>>(d_in, d_out, n); break;
        case ARITH_G1 + EC_QUAD_ADD: k_arith_quad<Fq, false, false><<<grid4, ARITH_BLOCK, 0, sl.stream>>>(d_in, d_out, n); break;
        case ARITH_G1 + EC_QUAD_DBL: k_arith_quad<Fq, false, true><<<grid4, ARITH_BLOCK, 0, sl.stream>>>(d_in, d_out, n); break;
        case ARITH_G1 + EC_QUAD_ADD_FULLWARP: k_arith_quad<Fq, true, false><<<grid32, ARITH_BLOCK, 0, sl.stream>>>(d_in, d_out, n); break;
        case ARITH_G1 + EC_QUAD_DBL_FULLWARP: k_arith_quad<Fq, true, true><<<grid32, ARITH_BLOCK, 0, sl.stream>>>(d_in, d_out, n); break;
        case ARITH_G2 + EC_QUAD_ADD: k_arith_quad<Fq2, false, false><<<grid4, ARITH_BLOCK, 0, sl.stream>>>(d_in, d_out, n); break;
        case ARITH_G2 + EC_QUAD_DBL: k_arith_quad<Fq2, false, true><<<grid4, ARITH_BLOCK, 0, sl.stream>>>(d_in, d_out, n); break;
        case ARITH_G2 + EC_QUAD_ADD_FULLWARP: k_arith_quad<Fq2, true, false><<<grid32, ARITH_BLOCK, 0, sl.stream>>>(d_in, d_out, n); break;
        case ARITH_G2 + EC_QUAD_DBL_FULLWARP: k_arith_quad<Fq2, true, true><<<grid32, ARITH_BLOCK, 0, sl.stream>>>(d_in, d_out, n); break;
        default: return set_error(ctx, B200ZK_ERR_ARG, "b200zk_test_arith: no such op");
    }
    return check_launch(ctx, "k_arith");
}
#endif  // __CUDACC__

}  // namespace b200zk

#ifdef __CUDACC__
using namespace b200zk;

extern "C" int b200zk_test_arith(b200zk_ctx* ctx, int op, const uint64_t* in, size_t n, uint64_t* out) {
    int in_w, out_w;
    arith_words(op, &in_w, &out_w);
    if (!ctx || in_w == 0) return set_error(ctx, B200ZK_ERR_ARG, "b200zk_test_arith: no such op");
    if (n == 0) return B200ZK_OK;
    if (!in || !out) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[0];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    const size_t in_bytes = n * in_w * 8, out_bytes = n * out_w * 8;
    B2_CUDA_OK(ctx, sl.io_a.reserve(in_bytes + out_bytes + 64));
    uint64_t* d_in = reinterpret_cast<uint64_t*>(sl.io_a.p);
    uint64_t* d_out = d_in + n * in_w;
    B2_CUDA_OK(ctx, cudaMemcpyAsync(d_in, in, in_bytes, cudaMemcpyHostToDevice, sl.stream));
    B2_CUDA_OK(ctx, cudaMemsetAsync(d_out, 0xFF, out_bytes, sl.stream));    // a record the kernel never writes cannot read as 0
    B2_TRY(arith_launch(ctx, sl, op, d_in, d_out, n, in_w, out_w));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(out, d_out, out_bytes, cudaMemcpyDeviceToHost, sl.stream));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(sl.stream));
    return B200ZK_OK;
}
#endif  // __CUDACC__
