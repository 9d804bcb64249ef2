// ec.cuh -- short-Weierstrass (a = 0) group arithmetic for BN254 G1 (over Fq) and G2 (over Fq2).
//
// Replaces arkworks' `short_weierstrass::{Affine,Projective}` (un-vendored) as used by `G::msm`
// (/root/reference/dist-primitives/src/dmsm/mod.rs:82) and the proof assembly
// (/root/reference/groth16/src/prove.rs:36-44,75-83,128-134).
//
// Accumulators use extended Jacobian "XYZZ" coordinates (x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2):
// a mixed add costs 8M+2S and needs no field inversion, which is what the bucket kernels want.
// Infinity: affine (0,0) (the zkey convention, ark-circom/src/zkey.rs:353-373); XYZZ with ZZ = 0.
// Results only ever leave the library as canonical affine coordinates, so they are bit-identical
// to arkworks' regardless of the internal coordinate system.
#pragma once
#include "fp.cuh"

namespace b200zk {

template <class F>
struct affine_t {
    F x, y;
    B2_HD bool is_inf() const { return x.is_zero() && y.is_zero(); }
    B2_HD static affine_t infinity() { affine_t r; r.x = F::zero(); r.y = F::zero(); return r; }
};

template <class F>
struct xyzz_t {
    F x, y, zz, zzz;

    B2_HD static xyzz_t identity() {
        xyzz_t r; r.x = F::zero(); r.y = F::zero(); r.zz = F::zero(); r.zzz = F::zero(); return r;
    }
    B2_HD bool is_inf() const { return zz.is_zero(); }

    B2_HD static xyzz_t from_affine(const affine_t<F>& p) {
        if (p.is_inf()) return identity();
        xyzz_t r; r.x = p.x; r.y = p.y; r.zz = F::one(); r.zzz = F::one(); return r;
    }

    // 2*p for an affine p (mdbl-2008-s-1)
    B2_HD_NI static xyzz_t dbl_affine(const F& px, const F& py) {
        F U = F::dbl(py);
        F V = F::sqr(U);
        F W = F::mul(U, V);
        F S = F::mul(px, V);
        F X2 = F::sqr(px);
        F M = F::add(F::dbl(X2), X2);
        xyzz_t r;
        r.x = F::sub(F::sqr(M), F::dbl(S));
        r.y = F::sub(F::mul(M, F::sub(S, r.x)), F::mul(W, py));
        r.zz = V;
        r.zzz = W;
        return r;
    }

    B2_HD_NI static xyzz_t dbl(const xyzz_t& p) { return dbl_inl(p); }
    B2_HD_NI static xyzz_t add(const xyzz_t& a, const xyzz_t& b) { return add_inl(a, b); }

    // dbl-2008-s-1
    B2_HD static xyzz_t dbl_inl(const xyzz_t& p) {
        if (p.is_inf()) return p;
        F U = F::dbl(p.y);
        F V = F::sqr(U);
        F W = F::mul(U, V);
        F S = F::mul(p.x, V);
        F X2 = F::sqr(p.x);
        F M = F::add(F::dbl(X2), X2);
        xyzz_t r;
        r.x = F::sub(F::sqr(M), F::dbl(S));
        r.y = F::sub(F::mul(M, F::sub(S, r.x)), F::mul(W, p.y));
        r.zz = F::mul(V, p.zz);
        r.zzz = F::mul(W, p.zzz);
        return r;
    }

    // acc += (negate ? -p : p), p affine (madd-2008-s); handles p = inf, acc = inf, acc = +-p.  The G2 bucket loop keeps
    // its Fq2 products out of line (DESIGN §7): inlined they save the call / argument traffic at ~3x the code.
    B2_HD static void madd(xyzz_t& acc, const affine_t<F>& p, bool negate) {
        if (p.is_inf()) return;
        F py = negate ? F::neg(p.y) : p.y;
        if (acc.is_inf()) {
            acc.x = p.x; acc.y = py; acc.zz = F::one(); acc.zzz = F::one();
            return;
        }
        F U2 = F::mul(p.x, acc.zz);
        F S2 = F::mul(py, acc.zzz);
        F Pp = F::sub(U2, acc.x);
        F R = F::sub(S2, acc.y);
        if (Pp.is_zero()) {
            if (R.is_zero()) acc = dbl_affine(p.x, py);
            else acc = identity();
            return;
        }
        F PP = F::sqr(Pp);
        F PPP = F::mul(Pp, PP);
        F Q = F::mul(acc.x, PP);
        F X3 = F::sub(F::sub(F::sqr(R), PPP), F::dbl(Q));
        F Y3 = F::sub(F::mul(R, F::sub(Q, X3)), F::mul(acc.y, PPP));
        acc.x = X3;
        acc.y = Y3;
        acc.zz = F::mul(acc.zz, PP);
        acc.zzz = F::mul(acc.zzz, PPP);
    }

    // add-2008-s
    B2_HD static xyzz_t add_inl(const xyzz_t& a, const xyzz_t& b) {
        if (a.is_inf()) return b;
        if (b.is_inf()) return a;
        F U1 = F::mul(a.x, b.zz);
        F U2 = F::mul(b.x, a.zz);
        F S1 = F::mul(a.y, b.zzz);
        F S2 = F::mul(b.y, a.zzz);
        F Pp = F::sub(U2, U1);
        F R = F::sub(S2, S1);
        if (Pp.is_zero()) {
            if (R.is_zero()) return dbl(a);      // rare: out-of-line
            return identity();
        }
        F PP = F::sqr(Pp);
        F PPP = F::mul(Pp, PP);
        F Q = F::mul(U1, PP);
        xyzz_t r;
        r.x = F::sub(F::sub(F::sqr(R), PPP), F::dbl(Q));
        r.y = F::sub(F::mul(R, F::sub(Q, r.x)), F::mul(S1, PPP));
        r.zz = F::mul(F::mul(a.zz, b.zz), PP);
        r.zzz = F::mul(F::mul(a.zzz, b.zzz), PPP);
        return r;
    }

    // ---- latency-optimised variants: the independent products of each dependency level are issued as one
    //      row-interleaved group (F::mul_group), 3 levels per doubling and 4 per addition -------------------
    B2_HD static xyzz_t dbl_ilp(const xyzz_t& p) {
        if (p.is_inf()) return p;
        F U = F::dbl(p.y);
        F a1[2] = {U, p.x}, b1[2] = {U, p.x}, r1[2];
        F::template mul_group<2>(r1, a1, b1);                       // V = U^2, X2 = X^2
        F V = r1[0];
        F M = F::add(F::dbl(r1[1]), r1[1]);
        F a2[4] = {U, p.x, V, M}, b2[4] = {V, V, p.zz, M}, r2[4];
        F::template mul_group<4>(r2, a2, b2);                       // W, S, ZZ3, M^2
        xyzz_t r;
        r.x = F::sub(r2[3], F::dbl(r2[1]));
        F a3[3] = {M, r2[0], r2[0]}, b3[3] = {F::sub(r2[1], r.x), p.y, p.zzz}, r3[3];
        F::template mul_group<3>(r3, a3, b3);                       // M(S - X3), W Y, W ZZZ
        r.y = F::sub(r3[0], r3[1]);
        r.zz = r2[2];
        r.zzz = r3[2];
        return r;
    }
    B2_HD static xyzz_t add_ilp(const xyzz_t& a, const xyzz_t& b) {
        if (a.is_inf()) return b;
        if (b.is_inf()) return a;
        F a1[4] = {a.x, b.x, a.y, b.y}, b1[4] = {b.zz, a.zz, b.zzz, a.zzz}, r1[4];
        F::template mul_group<4>(r1, a1, b1);                       // U1, U2, S1, S2
        F Pp = F::sub(r1[1], r1[0]), R = F::sub(r1[3], r1[2]);
        if (Pp.is_zero()) {
            if (R.is_zero()) return dbl(a);
            return identity();
        }
        F a2[4] = {Pp, R, a.zz, a.zzz}, b2[4] = {Pp, R, b.zz, b.zzz}, r2[4];
        F::template mul_group<4>(r2, a2, b2);                       // PP, R^2, ZZ1 ZZ2, ZZZ1 ZZZ2
        F a3[3] = {Pp, r1[0], r2[2]}, b3[3] = {r2[0], r2[0], r2[0]}, r3[3];
        F::template mul_group<3>(r3, a3, b3);                       // PPP, Q, ZZ3
        xyzz_t r;
        r.x = F::sub(F::sub(r2[1], r3[0]), F::dbl(r3[1]));
        F a4[3] = {R, r1[2], r2[3]}, b4[3] = {F::sub(r3[1], r.x), r3[0], r3[0]}, r4[3];
        F::template mul_group<3>(r4, a4, b4);                       // R(Q - X3), S1 PPP, ZZZ3
        r.y = F::sub(r4[0], r4[1]);
        r.zz = r3[2];
        r.zzz = r4[2];
        return r;
    }

    B2_HD_NI static xyzz_t dbl_ilp_ni(const xyzz_t& p) { return dbl_ilp(p); }
    B2_HD_NI static xyzz_t add_ilp_ni(const xyzz_t& a, const xyzz_t& b) { return add_ilp(a, b); }

    B2_HD static xyzz_t neg(const xyzz_t& a) { xyzz_t r = a; r.y = F::neg(a.y); return r; }

    // canonical affine (x = X/ZZ, y = Y/ZZZ) of a finite a from a known izzz = 1/ZZZ
    B2_HD static affine_t<F> to_affine(const xyzz_t& a, const F& izzz) {
        F izz = F::sqr(F::mul(izzz, a.zz));          // ZZ^3 = ZZZ^2  =>  1/ZZ = (ZZ/ZZZ)^2
        affine_t<F> r;
        r.x = F::mul(a.x, izz);
        r.y = F::mul(a.y, izzz);
        return r;
    }
    // the same with its own inversion; infinity -> (0,0)
    B2_HD_NI static affine_t<F> to_affine(const xyzz_t& a) {
        if (a.is_inf()) return affine_t<F>::infinity();
        return to_affine(a, F::inv(a.zzz));
    }

    // k * p for a 256-bit canonical (non-Montgomery) scalar k given as 8 x u32
    B2_HD_NI static xyzz_t mul_scalar(const xyzz_t& p, const uint32_t k[8]) {
        xyzz_t acc = identity();
        for (int bit = 255; bit >= 0; --bit) {
            acc = dbl(acc);
            if ((k[bit >> 5] >> (bit & 31)) & 1) acc = add(acc, p);
        }
        return acc;
    }
};

// the fixed generator of G1 (F = Fq) or G2 (F = Fq2), Montgomery form
template <class F> B2_HD affine_t<F> curve_generator();
template <> B2_HD affine_t<Fq> curve_generator<Fq>() {
    affine_t<Fq> g;
    for (int i = 0; i < 8; ++i) { g.x.l[i] = CurveConst::g1_gen_x(i); g.y.l[i] = CurveConst::g1_gen_y(i); }
    return g;
}
template <> B2_HD affine_t<Fq2> curve_generator<Fq2>() {
    affine_t<Fq2> g;
    for (int i = 0; i < 8; ++i) {
        g.x.c0.l[i] = CurveConst::g2_gen_x0(i); g.x.c1.l[i] = CurveConst::g2_gen_x1(i);
        g.y.c0.l[i] = CurveConst::g2_gen_y0(i); g.y.c1.l[i] = CurveConst::g2_gen_y1(i);
    }
    return g;
}

#ifdef __CUDACC__
// ---------------------------------------------------------------------------------------------
// quad-cooperative group law (device only)
//
// The serial tails of an MSM (bucket running sums, window trees, the final Horner) are chains of
// dependent point operations, i.e. latency-bound: one warp alone retires a 256-bit Montgomery product
// in ~0.4 us (tools/microbench.cu).  Here four adjacent lanes hold identical copies of the operands,
// each computes one of the (up to four) independent field products of a dependency level and the
// results are exchanged with quad-wide shuffles: an XYZZ addition becomes 4 product-latencies instead
// of 14, a doubling 3 instead of 9.  All lanes of a quad must call with identical arguments.
// ---------------------------------------------------------------------------------------------
// FULLWARP = true: every lane of the warp executes the same call sequence (e.g. one warp doing one chain
// redundantly in its 8 quads), so the shuffles can use the full mask -- with a runtime quad mask the compiler
// wraps every SHFL in a WARPSYNC/collective sequence, which more than doubles the latency of an operation.
template <class F, bool FULLWARP = false>
struct quad_ops {
    static constexpr int WORDS = sizeof(F) / 4;

    __device__ __forceinline__ static unsigned quad_mask() { return FULLWARP ? 0xFFFFFFFFu : (0xFu << (threadIdx.x & 28u)); }
    __device__ __forceinline__ static int quad_lane() { return threadIdx.x & 3; }

    // exchange area in shared memory: 2 buffers x 4 products per quad (double-buffered: one __syncwarp per level).
    // Shuffles were measured slower here: with data-dependent branches upstream every SHFL gets wrapped in a
    // WARPSYNC/collective sequence (576 SHFL + 320 WARPSYNC per doubling+addition in SASS).
    struct xch_t { F p[2][4]; };
    __device__ __forceinline__ static F sel(int q, const F& a0, const F& a1, const F& a2, const F& a3) {
        F r;
        const uint32_t* p0 = reinterpret_cast<const uint32_t*>(&a0);
        const uint32_t* p1 = reinterpret_cast<const uint32_t*>(&a1);
        const uint32_t* p2 = reinterpret_cast<const uint32_t*>(&a2);
        const uint32_t* p3 = reinterpret_cast<const uint32_t*>(&a3);
        uint32_t* pr = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
        for (int i = 0; i < WORDS; ++i) pr[i] = q == 0 ? p0[i] : q == 1 ? p1[i] : q == 2 ? p2[i] : p3[i];
        return r;
    }
    // p_k = a_k * b_k, lane k computing product k; every lane receives all four through `x` (buffer `buf`)
    __device__ __forceinline__ static void mul4(xch_t* x, int buf, const F& a0, const F& b0, const F& a1, const F& b1,
                                                const F& a2, const F& b2, const F& a3, const F& b3, F& p0, F& p1, F& p2, F& p3) {
        const int q = quad_lane();
        F a = sel(q, a0, a1, a2, a3), b = sel(q, b0, b1, b2, b3);
        F p = F::mul(a, b);
        st16(&x->p[buf][q], p);
        __syncwarp(quad_mask());
        p0 = ld16(&x->p[buf][0]); p1 = ld16(&x->p[buf][1]); p2 = ld16(&x->p[buf][2]); p3 = ld16(&x->p[buf][3]);
    }

    __device__ static xyzz_t<F> dbl(xch_t* x, const xyzz_t<F>& p) {
        if (p.is_inf()) return p;
        F U = F::dbl(p.y);
        F V, X2, d0, d1;
        mul4(x, 0, U, U, p.x, p.x, U, U, U, U, V, X2, d0, d1);
        F M = F::add(F::dbl(X2), X2);
        F W, S, ZZ3, MM;
        mul4(x, 1, U, V, p.x, V, V, p.zz, M, M, W, S, ZZ3, MM);
        xyzz_t<F> r;
        r.x = F::sub(MM, F::dbl(S));
        F T1, T2, ZZZ3;
        mul4(x, 0, M, F::sub(S, r.x), W, p.y, W, p.zzz, W, W, T1, T2, ZZZ3, d0);
        r.y = F::sub(T1, T2);
        r.zz = ZZ3;
        r.zzz = ZZZ3;
        __syncwarp(quad_mask());          // buffer 1 is reused by the next operation's second level
        return r;
    }

    __device__ static xyzz_t<F> add(xch_t* x, const xyzz_t<F>& a, const xyzz_t<F>& b) {
        if (a.is_inf()) return b;
        if (b.is_inf()) return a;
        F U1, U2, S1, S2;
        mul4(x, 0, a.x, b.zz, b.x, a.zz, a.y, b.zzz, b.y, a.zzz, U1, U2, S1, S2);
        F Pp = F::sub(U2, U1), R = F::sub(S2, S1);
        if (Pp.is_zero()) {
            __syncwarp(quad_mask());
            if (R.is_zero()) return dbl(x, a);
            return xyzz_t<F>::identity();
        }
        F PP, RR, ZZ12, ZZZ12;
        mul4(x, 1, Pp, Pp, R, R, a.zz, b.zz, a.zzz, b.zzz, PP, RR, ZZ12, ZZZ12);
        F PPP, Q, ZZ3, d0;
        mul4(x, 0, Pp, PP, U1, PP, ZZ12, PP, PP, PP, PPP, Q, ZZ3, d0);
        xyzz_t<F> r;
        r.x = F::sub(F::sub(RR, PPP), F::dbl(Q));
        F T1, T2, ZZZ3;
        mul4(x, 1, R, F::sub(Q, r.x), S1, PPP, ZZZ12, PPP, PPP, PPP, T1, T2, ZZZ3, d0);
        r.y = F::sub(T1, T2);
        r.zz = ZZ3;
        r.zzz = ZZZ3;
        __syncwarp(quad_mask());
        return r;
    }
};
#endif  // __CUDACC__

struct G1Curve {
    typedef Fq F;
    static constexpr int LIMBS64 = 8;     // u64 limbs per affine point
};
struct G2Curve {
    typedef Fq2 F;
    static constexpr int LIMBS64 = 16;
};

}  // namespace b200zk
