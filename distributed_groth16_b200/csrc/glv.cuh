// glv.cuh -- Gallant-Lambert-Vanstone scalar split for BN254 G1 (and, with beta^2 in place of beta, for G2 on the twist:
// the same lambda acts there as (x, y) -> (beta^2 x, y); tools/gen_constants.py checks both).
//
// phi(x, y) = (beta x, y) acts on G1 as multiplication by lambda (lambda^2 + lambda + 1 = 0 mod r), so
//   k P = k1 P + k2 phi(P),  k = k1 + k2 lambda (mod r),  |k1|, |k2| < 2^127.
// The MSM uses it only to halve the Horner chain at the end: sum_i k2_i phi(P_i) = phi(sum_i k2_i P_i), so the
// digits of k2 simply go to a second group of windows over the SAME points and phi is applied once to that group's
// result.  Same group element as the reference's `G::msm` (dist-primitives/src/dmsm/mod.rs:82).
//
// k1 = k - c1 a1 - c2 a2, k2 = c1 |b1| - c2 b2 with c_i = round(k g_i / 2^256) (constants: GlvParams, derived by
// tools/gen_constants.py from the lattice {(a, b): a + b lambda = 0 mod r}).  Plain C: unit-tested on the host.
#pragma once
#include "fp.cuh"

namespace b200zk {

// out[0..na+nb) = a * b  (little-endian u32 limbs)
template <int NA, int NB>
B2_HD void mul_limbs(uint32_t* out, const uint32_t* a, const uint32_t* b) {
#pragma unroll
    for (int i = 0; i < NA + NB; ++i) out[i] = 0;
#pragma unroll
    for (int i = 0; i < NA; ++i) {
        uint64_t carry = 0;
#pragma unroll
        for (int j = 0; j < NB; ++j) {
            uint64_t t = (uint64_t)a[i] * b[j] + out[i + j] + carry;
            out[i + j] = (uint32_t)t;
            carry = t >> 32;
        }
        out[i + NB] = (uint32_t)carry;
    }
}

struct GlvSplit {
    uint32_t k1[4], k2[4];   // absolute values, < 2^127
    bool neg1, neg2;
};

// k: canonical (non-Montgomery) scalar < r, 8 limbs
B2_HD GlvSplit glv_decompose(const uint32_t k[8]) {
    uint32_t g1[3], g2[5], a1[2], a2[4], nb1[4], b2[2];
#pragma unroll
    for (int i = 0; i < 3; ++i) g1[i] = GlvParams::g1(i);
#pragma unroll
    for (int i = 0; i < 5; ++i) g2[i] = GlvParams::g2(i);
#pragma unroll
    for (int i = 0; i < 2; ++i) { a1[i] = GlvParams::a1(i); b2[i] = GlvParams::b2(i); }
#pragma unroll
    for (int i = 0; i < 4; ++i) { a2[i] = GlvParams::a2(i); nb1[i] = GlvParams::nb1(i); }
    // c1 = (k g1 + 2^255) >> 256 (fits 3 limbs), c2 = (k g2 + 2^255) >> 256 (fits 5 limbs)
    uint32_t t1[11], t2[13], c1[3], c2[5];
    mul_limbs<8, 3>(t1, k, g1);
    mul_limbs<8, 5>(t2, k, g2);
    {
        uint64_t cy = (uint64_t)t1[7] + 0x80000000u;
        cy >>= 32;
#pragma unroll
        for (int i = 0; i < 3; ++i) { uint64_t v = (uint64_t)t1[8 + i] + cy; c1[i] = (uint32_t)v; cy = v >> 32; }
        cy = ((uint64_t)t2[7] + 0x80000000u) >> 32;
#pragma unroll
        for (int i = 0; i < 5; ++i) { uint64_t v = (uint64_t)t2[8 + i] + cy; c2[i] = (uint32_t)v; cy = v >> 32; }
    }
    // all arithmetic below modulo 2^256 (two's complement); the true results are < 2^127 in magnitude
    uint32_t p1[5], p2[9], p3[7], p4[7];
    mul_limbs<3, 2>(p1, c1, a1);       // c1 a1
    mul_limbs<5, 4>(p2, c2, a2);       // c2 a2
    mul_limbs<3, 4>(p3, c1, nb1);      // c1 |b1|
    mul_limbs<5, 2>(p4, c2, b2);       // c2 b2
    uint32_t k1[8], k2[8];
    {
        int64_t br = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            int64_t v = (int64_t)k[i] - (i < 5 ? (int64_t)p1[i] : 0) - (int64_t)p2[i] + br;
            k1[i] = (uint32_t)v;
            br = v >> 32;                      // arithmetic shift: borrow propagates as a negative carry
        }
        br = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            int64_t v = (i < 7 ? (int64_t)p3[i] : 0) - (i < 7 ? (int64_t)p4[i] : 0) + br;
            k2[i] = (uint32_t)v;
            br = v >> 32;
        }
    }
    GlvSplit s;
    s.neg1 = (k1[7] >> 31) != 0;
    s.neg2 = (k2[7] >> 31) != 0;
    {   // absolute values
        uint64_t c = 1;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            uint32_t w = s.neg1 ? ~k1[i] : k1[i];
            if (s.neg1) { uint64_t v = (uint64_t)w + c; w = (uint32_t)v; c = v >> 32; }
            if (i < 4) s.k1[i] = w;
        }
        c = 1;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            uint32_t w = s.neg2 ? ~k2[i] : k2[i];
            if (s.neg2) { uint64_t v = (uint64_t)w + c; w = (uint32_t)v; c = v >> 32; }
            if (i < 4) s.k2[i] = w;
        }
    }
    return s;
}

// the x coordinate of phi(P): beta x on G1, beta^2 x on the twist (the same lambda; tools/gen_constants.py checks both).
// phi leaves y and the XYZZ denominators alone, so it applies to affine and XYZZ points alike.
B2_HD void glv_phi_x(Fq& x) {
    Fq beta;
#pragma unroll
    for (int i = 0; i < 8; ++i) beta.l[i] = GlvParams::beta(i);
    x = Fq::mul(x, beta);
}
B2_HD void glv_phi_x(Fq2& x) {
    Fq beta;
#pragma unroll
    for (int i = 0; i < 8; ++i) beta.l[i] = GlvParams::beta_g2(i);
    x.c0 = Fq::mul(x.c0, beta);
    x.c1 = Fq::mul(x.c1, beta);
}

}  // namespace b200zk
