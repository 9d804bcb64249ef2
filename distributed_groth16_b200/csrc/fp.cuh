// fp.cuh -- 256-bit Montgomery prime-field arithmetic for sm_90a (BN254 Fq and Fr).
//
// Replaces arkworks' `Fp256<MontBackend<..,4>>` (un-vendored dependency of the reference; used at
// every hot-path site, e.g. /root/reference/dist-primitives/src/dfft/mod.rs:128-131 butterflies and
// inside `G::msm` at dist-primitives/src/dmsm/mod.rs:82).
//
// Representation: 8 x 32-bit little-endian limbs, Montgomery form with R = 2^256, value always
// canonical (< p) between operations.  The memory image of one element (32 bytes) is identical to
// arkworks' 4 x u64 `BigInt` limbs, which is what crosses the C ABI (include/b200zk.h).
//
// The multiplier is a row-interleaved Montgomery product built from PTX carry-chain multiply-adds
// (mad.lo.cc / madc.hi.cc); two accumulators hold the products of the even- and odd-indexed limbs
// of `a` so that every 64-bit partial product lands on an aligned (lo,hi) register pair and ptxas
// can emit IMAD.WIDE with carry.  There are no tensor cores anywhere: the arithmetic is wide-integer.
//
// Every primitive has a plain-C emulation behind `#ifndef __CUDA_ARCH__` so the exact same limb
// schedule is unit-tested on the CPU (tests/host/fp_host_test.cpp) -- this is a test seam, not a CPU
// fallback: no product entry point runs the host branch.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B2_HD __host__ __device__ __forceinline__
// inline: only the linkage (the free functions of codec.cuh / pairing.cuh are defined in every translation unit that
// includes them); __noinline__ still keeps each one a single out-of-line copy per unit
#define B2_HD_NI __host__ __device__ __noinline__ inline
#else
#define B2_HD inline __attribute__((always_inline))
#define B2_HD_NI inline
#endif

namespace b200zk {

// ---------------------------------------------------------------------------------------------
// carry-chain primitives
// ---------------------------------------------------------------------------------------------
namespace cc {
#ifdef __CUDA_ARCH__
#define B2_ASM asm volatile
B2_HD uint32_t add_cc(uint32_t a, uint32_t b) { uint32_t r; B2_ASM("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2_HD uint32_t addc_cc(uint32_t a, uint32_t b) { uint32_t r; B2_ASM("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2_HD uint32_t addc(uint32_t a, uint32_t b) { uint32_t r; B2_ASM("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2_HD uint32_t sub_cc(uint32_t a, uint32_t b) { uint32_t r; B2_ASM("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2_HD uint32_t subc_cc(uint32_t a, uint32_t b) { uint32_t r; B2_ASM("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2_HD uint32_t subc(uint32_t a, uint32_t b) { uint32_t r; B2_ASM("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2_HD uint32_t mul_lo(uint32_t a, uint32_t b) { uint32_t r; B2_ASM("mul.lo.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2_HD uint32_t mul_hi(uint32_t a, uint32_t b) { uint32_t r; B2_ASM("mul.hi.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2_HD uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; B2_ASM("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
B2_HD uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; B2_ASM("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
B2_HD uint32_t mad_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; B2_ASM("mad.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
B2_HD uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; B2_ASM("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
B2_HD uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; B2_ASM("madc.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
B2_HD uint32_t madc_lo(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; B2_ASM("madc.lo.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
#undef B2_ASM
#else
// host emulation of the PTX condition-code register (test seam only)
static thread_local uint32_t CF = 0;
B2_HD uint32_t add_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b; CF = (uint32_t)(t >> 32); return (uint32_t)t; }
B2_HD uint32_t addc_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b + CF; CF = (uint32_t)(t >> 32); return (uint32_t)t; }
B2_HD uint32_t addc(uint32_t a, uint32_t b) { return a + b + CF; }
B2_HD uint32_t sub_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b; CF = (uint32_t)(t >> 32) & 1; return (uint32_t)t; }
B2_HD uint32_t subc_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b - CF; CF = (uint32_t)(t >> 32) & 1; return (uint32_t)t; }
B2_HD uint32_t subc(uint32_t a, uint32_t b) { return a - b - CF; }
B2_HD uint32_t mul_lo(uint32_t a, uint32_t b) { return a * b; }
B2_HD uint32_t mul_hi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
B2_HD uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t t = (uint64_t)(uint32_t)(a * b) + c; CF = (uint32_t)(t >> 32); return (uint32_t)t; }
B2_HD uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t t = (uint64_t)(uint32_t)(a * b) + c + CF; CF = (uint32_t)(t >> 32); return (uint32_t)t; }
B2_HD uint32_t mad_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t t = (((uint64_t)a * b) >> 32) + c; CF = (uint32_t)(t >> 32); return (uint32_t)t; }
B2_HD uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t t = (((uint64_t)a * b) >> 32) + c + CF; CF = (uint32_t)(t >> 32); return (uint32_t)t; }
B2_HD uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { return (uint32_t)((((uint64_t)a * b) >> 32) + c + CF); }
B2_HD uint32_t madc_lo(uint32_t a, uint32_t b, uint32_t c) { return a * b + c + CF; }
#endif
}  // namespace cc

// ---------------------------------------------------------------------------------------------
// field parameters (BN254).  MOD = p, INV = -p^{-1} mod 2^32, R1 = 2^256 mod p, R2 = 2^512 mod p.
// Values are generated by tools/gen_constants.py from oracle/bn254.py and re-checked by
// tests/test_constants.py; they are compile-time so ptxas can fold them into immediates.
// ---------------------------------------------------------------------------------------------
#include "bn254_constants.inc"

template <class P>
struct Fp {
    uint32_t l[8];

    B2_HD static Fp zero() { Fp r; for (int i = 0; i < 8; ++i) r.l[i] = 0; return r; }
    B2_HD static Fp one() { Fp r; for (int i = 0; i < 8; ++i) r.l[i] = P::r1(i); return r; }
    B2_HD static Fp r2() { Fp r; for (int i = 0; i < 8; ++i) r.l[i] = P::r2(i); return r; }
    B2_HD bool is_zero() const {
        uint32_t o = 0;
        for (int i = 0; i < 8; ++i) o |= l[i];
        return o == 0;
    }
    B2_HD bool operator==(const Fp& b) const {
        uint32_t o = 0;
        for (int i = 0; i < 8; ++i) o |= l[i] ^ b.l[i];
        return o == 0;
    }
    B2_HD bool operator!=(const Fp& b) const { return !(*this == b); }

    // r = t - p if t >= p else t   (t < 2p)
    B2_HD static void final_sub(Fp& r, const uint32_t t[8]) {
        uint32_t d[8];
        d[0] = cc::sub_cc(t[0], P::mod(0));
#pragma unroll
        for (int i = 1; i < 8; ++i) d[i] = cc::subc_cc(t[i], P::mod(i));
        uint32_t borrow = cc::subc(0, 0);       // 0xffffffff when t < p
#pragma unroll
        for (int i = 0; i < 8; ++i) r.l[i] = borrow ? t[i] : d[i];
    }

    B2_HD static Fp add(const Fp& a, const Fp& b) {
        uint32_t t[8];
        t[0] = cc::add_cc(a.l[0], b.l[0]);
#pragma unroll
        for (int i = 1; i < 7; ++i) t[i] = cc::addc_cc(a.l[i], b.l[i]);
        t[7] = cc::addc(a.l[7], b.l[7]);        // a+b < 2p < 2^255: no carry out
        Fp r; final_sub(r, t); return r;
    }
    B2_HD static Fp sub(const Fp& a, const Fp& b) {
        uint32_t t[8];
        t[0] = cc::sub_cc(a.l[0], b.l[0]);
#pragma unroll
        for (int i = 1; i < 8; ++i) t[i] = cc::subc_cc(a.l[i], b.l[i]);
        uint32_t borrow = cc::subc(0, 0);       // all ones when a < b
        Fp r;
        r.l[0] = cc::add_cc(t[0], P::mod(0) & borrow);
#pragma unroll
        for (int i = 1; i < 7; ++i) r.l[i] = cc::addc_cc(t[i], P::mod(i) & borrow);
        r.l[7] = cc::addc(t[7], P::mod(7) & borrow);
        return r;
    }
    B2_HD static Fp neg(const Fp& a) { return sub(zero(), a); }
    B2_HD static Fp dbl(const Fp& a) { return add(a, a); }

    // ---- Montgomery product --------------------------------------------------------------
    // acc[j], acc[j+1] = a[j]*bi for even j (no carries)
    B2_HD static void mul_n(uint32_t* acc, const uint32_t* a, uint32_t bi) {
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
            acc[j] = cc::mul_lo(a[j], bi);
            acc[j + 1] = cc::mul_hi(a[j], bi);
        }
    }
    // acc += sum_{even j} a[j]*bi * 2^(32 j); carry-out left in CC
    B2_HD static void cmad_n(uint32_t* acc, const uint32_t* a, uint32_t bi) {
        acc[0] = cc::mad_lo_cc(a[0], bi, acc[0]);
        acc[1] = cc::madc_hi_cc(a[0], bi, acc[1]);
#pragma unroll
        for (int j = 2; j < 8; j += 2) {
            acc[j] = cc::madc_lo_cc(a[j], bi, acc[j]);
            acc[j + 1] = cc::madc_hi_cc(a[j], bi, acc[j + 1]);
        }
    }
    // acc += sum_{even j} p[j+OFF]*mi * 2^(32 j); carry-out left in CC
    template <int OFF>
    B2_HD static void cmad_mod(uint32_t* acc, uint32_t mi) {
        acc[0] = cc::mad_lo_cc(P::mod(OFF), mi, acc[0]);
        acc[1] = cc::madc_hi_cc(P::mod(OFF), mi, acc[1]);
#pragma unroll
        for (int j = 2; j < 8; j += 2) {
            acc[j] = cc::madc_lo_cc(P::mod(j + OFF), mi, acc[j]);
            acc[j + 1] = cc::madc_hi_cc(P::mod(j + OFF), mi, acc[j + 1]);
        }
    }
    // acc = (acc >> 64) + sum_{even j} a[j]*bi * 2^(32 j) + CC  (top product < 2^62: no carry out)
    B2_HD static void madc_n_rshift(uint32_t* acc, const uint32_t* a, uint32_t bi) {
#pragma unroll
        for (int j = 0; j < 6; j += 2) {
            acc[j] = cc::madc_lo_cc(a[j], bi, acc[j + 2]);
            acc[j + 1] = cc::madc_hi_cc(a[j], bi, acc[j + 3]);
        }
        acc[6] = cc::madc_lo_cc(a[6], bi, 0);
        acc[7] = cc::madc_hi(a[6], bi, 0);
    }
    // one row: (ev + 2^32 od) <- (ev + 2^32 od + a*bi + m*p) / 2^32, roles of ev/od swap for the next row
    B2_HD static void mad_row(uint32_t* ev, uint32_t* od, const uint32_t* a, uint32_t bi, bool first) {
        if (first) {
            mul_n(od, a + 1, bi);
            mul_n(ev, a, bi);
        } else {
            ev[0] = cc::add_cc(ev[0], od[1]);
            madc_n_rshift(od, a + 1, bi);
            cmad_n(ev, a, bi);
            od[7] = cc::addc(od[7], 0);
        }
        uint32_t mi = ev[0] * P::INV;
        cmad_mod<1>(od, mi);
        cmad_mod<0>(ev, mi);
        od[7] = cc::addc(od[7], 0);
    }
    B2_HD static Fp mul(const Fp& a, const Fp& b) {
        uint32_t ev[8], od[8];
#pragma unroll
        for (int i = 0; i < 8; i += 2) {
            mad_row(ev, od, a.l, b.l[i], i == 0);
            mad_row(od, ev, a.l, b.l[i + 1], false);
        }
        ev[0] = cc::add_cc(ev[0], od[1]);
#pragma unroll
        for (int i = 1; i < 7; ++i) ev[i] = cc::addc_cc(ev[i], od[i + 1]);
        ev[7] = cc::addc(ev[7], 0);
        Fp r; final_sub(r, ev); return r;
    }
    // a dedicated squaring (36 + 72 wide multiply-adds instead of 136) was measured 3% SLOWER in the G1 bucket kernel
    // (126 vs 120 registers, doubling shifts)
    B2_HD static Fp sqr(const Fp& a) { return mul(a, a); }

    // ---- unreduced 512-bit products and a separate Montgomery reduction ----------------------------------------------------
    // Column-wise (product scanning) with a three-word column accumulator (c0, c1, c2): every partial product is one fused
    // (mad.lo.cc, madc.hi.cc) pair = one wide multiply-add, plus an addc for the third word on the ALU pipe.  They exist for
    // what the row-interleaved product above cannot do: Fq2 products that reduce two sums of products instead of three
    // products (Fq2::mul).
    B2_HD static void col_mad(uint32_t& c0, uint32_t& c1, uint32_t& c2, uint32_t x, uint32_t y) {
        c0 = cc::mad_lo_cc(x, y, c0);
        c1 = cc::madc_hi_cc(x, y, c1);
        c2 = cc::addc(c2, 0);
    }
    // t[0..16) = a * b
    B2_HD static void mul_wide(uint32_t* t, const uint32_t* a, const uint32_t* b) {
        uint32_t c0 = 0, c1 = 0, c2 = 0;
#pragma unroll
        for (int k = 0; k < 15; ++k) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int j = k - i;
                if (j >= 0 && j < 8) col_mad(c0, c1, c2, a[i], b[j]);
            }
            t[k] = c0; c0 = c1; c1 = c2; c2 = 0;
        }
        t[15] = c0;
    }
    // r = t / 2^256 mod p for t < SUBS * p * 2^256 (SUBS = 1: products of canonical values; 2: a lazy sum of two of them):
    // column-wise Montgomery reduction, then SUBS conditional subtractions.  Clobbers nothing outside r.
    template <int SUBS>
    B2_HD static void redc(Fp& r, const uint32_t* t) {
        uint32_t m[8], u[8];
        uint32_t c0 = 0, c1 = 0, c2 = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
#pragma unroll
            for (int i = 0; i < k; ++i) col_mad(c0, c1, c2, m[i], P::mod(k - i));
            c0 = cc::add_cc(c0, t[k]); c1 = cc::addc_cc(c1, 0); c2 = cc::addc(c2, 0);
            m[k] = c0 * P::INV;
            col_mad(c0, c1, c2, m[k], P::mod(0));           // c0 becomes 0
            c0 = c1; c1 = c2; c2 = 0;
        }
#pragma unroll
        for (int k = 8; k < 16; ++k) {
#pragma unroll
            for (int i = k - 7; i < 8; ++i) col_mad(c0, c1, c2, m[i], P::mod(k - i));
            c0 = cc::add_cc(c0, t[k]); c1 = cc::addc_cc(c1, 0); c2 = cc::addc(c2, 0);
            u[k - 8] = c0; c0 = c1; c1 = c2; c2 = 0;
        }
        // value = u + c0 * 2^256 < (SUBS + 1) p: subtract p while >= p (c0 can only be set when SUBS > 1)
        uint32_t top = c0;
#pragma unroll
        for (int sidx = 0; sidx < SUBS; ++sidx) {
            uint32_t d[8];
            d[0] = cc::sub_cc(u[0], P::mod(0));
#pragma unroll
            for (int i = 1; i < 8; ++i) d[i] = cc::subc_cc(u[i], P::mod(i));
            const uint32_t dtop = cc::subc(top, 0);
            const bool ge = (int32_t)dtop >= 0;                 // no borrow out of the 288-bit subtraction
#pragma unroll
            for (int i = 0; i < 8; ++i) u[i] = ge ? d[i] : u[i];
            top = ge ? dtop : top;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) r.l[i] = u[i];
    }
    // 512-bit helpers for lazy sums: x += y (no overflow by the callers' bounds), x -= y (x >= y)
    B2_HD static void add_wide(uint32_t* x, const uint32_t* y) {
        x[0] = cc::add_cc(x[0], y[0]);
#pragma unroll
        for (int i = 1; i < 15; ++i) x[i] = cc::addc_cc(x[i], y[i]);
        x[15] = cc::addc(x[15], y[15]);
    }
    B2_HD static void sub_wide(uint32_t* x, const uint32_t* y) {
        x[0] = cc::sub_cc(x[0], y[0]);
#pragma unroll
        for (int i = 1; i < 15; ++i) x[i] = cc::subc_cc(x[i], y[i]);
        x[15] = cc::subc(x[15], y[15]);
    }
    // x += p * 2^256 (keeps a difference of two products non-negative)
    B2_HD static void add_mod_hi(uint32_t* x) {
        x[8] = cc::add_cc(x[8], P::mod(0));
#pragma unroll
        for (int i = 1; i < 7; ++i) x[8 + i] = cc::addc_cc(x[8 + i], P::mod(i));
        x[15] = cc::addc(x[15], P::mod(7));
    }

    // K independent products with their rows interleaved in program order.  One warp alone retires a single
    // product in ~0.42 us because each row waits on the previous one (carry chains + the m_i dependency);
    // the serial tails of an MSM (bucket running sums, Horner) are exactly that regime.  Interleaving the rows
    // of K independent products gives the scheduler K independent chains and hides most of that latency.
    template <int K>
    B2_HD static void mul_k(Fp* r, const Fp* a, const Fp* b) {
        uint32_t ev[K][8], od[K][8];
#pragma unroll
        for (int i = 0; i < 8; i += 2) {
#pragma unroll
            for (int k = 0; k < K; ++k) mad_row(ev[k], od[k], a[k].l, b[k].l[i], i == 0);
#pragma unroll
            for (int k = 0; k < K; ++k) mad_row(od[k], ev[k], a[k].l, b[k].l[i + 1], false);
        }
#pragma unroll
        for (int k = 0; k < K; ++k) {
            ev[k][0] = cc::add_cc(ev[k][0], od[k][1]);
#pragma unroll
            for (int i = 1; i < 7; ++i) ev[k][i] = cc::addc_cc(ev[k][i], od[k][i + 1]);
            ev[k][7] = cc::addc(ev[k][7], 0);
            final_sub(r[k], ev[k]);
        }
    }
    // generic entry used by the group law: K <= 4 products at once
    template <int K>
    B2_HD static void mul_group(Fp* r, const Fp* a, const Fp* b) { mul_k<K>(r, a, b); }
    // out-of-line copy for the cold / very large kernels (G2, reductions): keeps code size and
    // compile time bounded; the G1 bucket loop uses the inlined `mul`.
    B2_HD_NI static Fp mul_ni(const Fp& a, const Fp& b) { return mul(a, b); }

    B2_HD static Fp to_mont(const Fp& a) { return mul(a, r2()); }
    B2_HD static Fp from_mont(const Fp& a) {
        Fp o = zero(); o.l[0] = 1;
        return mul(a, o);
    }
    // a^(p-2) (Fermat) -- kept as the slow cross-check of inv()
    B2_HD_NI static Fp inv_fermat(const Fp& a) {
        Fp res = one();
        for (int i = 255; i >= 0; --i) {
            res = mul_ni(res, res);
            uint32_t w = 0;
#pragma unroll
            for (int k = 0; k < 8; ++k) if ((i >> 5) == k) w = P::mod_m2(k);
            if ((w >> (i & 31)) & 1) res = mul_ni(res, a);
        }
        return res;
    }

    // Montgomery inverse by the binary extended Euclid ("almost inverse", Kaliski): ~2*254 shift/subtract
    // steps on 256-bit integers instead of ~380 dependent field multiplications -- the affine normalisation
    // is a single-thread latency chain at the end of every MSM (about 10x shorter than Fermat).
    // Input/outputs in Montgomery form; inv(0) = 0.
    B2_HD_NI static Fp inv(const Fp& a) {
        if (a.is_zero()) return a;
        uint32_t u[8], v[8], r[8], s[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) { u[i] = P::mod(i); v[i] = a.l[i]; r[i] = 0; s[i] = 0; }
        s[0] = 1;
        int k = 0;
        for (;;) {
            uint32_t vz = 0;
#pragma unroll
            for (int i = 0; i < 8; ++i) vz |= v[i];
            if (vz == 0) break;
            if ((u[0] & 1) == 0) { shr1(u); shl1(s); }
            else if ((v[0] & 1) == 0) { shr1(v); shl1(r); }
            else if (gt(u, v)) { sub_n(u, v); shr1(u); add_n(r, s); shl1(s); }
            else { sub_n(v, u); shr1(v); add_n(s, r); shl1(r); }
            ++k;
        }
        // r < 2p; r = p - (r mod p) = (aR)^-1 * 2^k
        Fp t;
        final_sub(t, r);
        t = neg(t);
        // t*R^2*R^-1 = a^-1 * 2^k, then * 2^(512-k) * R^-1 = a^-1 * R
        t = mul_ni(t, r2());
        int j = 512 - k;                         // k in [254, 508]
        if (j >= 256) {
            for (int d = 0; d < j - 256; ++d) t = dbl(t);
            return t;
        }
        Fp pw = zero();
#pragma unroll
        for (int i = 0; i < 8; ++i) if ((j >> 5) == i) pw.l[i] = 1u << (j & 31);
        return mul_ni(t, pw);                    // second operand may exceed p: only the rows use it (see mul)
    }
    B2_HD static void shr1(uint32_t* x) {
#pragma unroll
        for (int i = 0; i < 7; ++i) x[i] = (x[i] >> 1) | (x[i + 1] << 31);
        x[7] >>= 1;
    }
    B2_HD static void shl1(uint32_t* x) {
#pragma unroll
        for (int i = 7; i > 0; --i) x[i] = (x[i] << 1) | (x[i - 1] >> 31);
        x[0] <<= 1;
    }
    B2_HD static bool gt(const uint32_t* x, const uint32_t* y) {
#pragma unroll
        for (int i = 7; i >= 0; --i) {
            if (x[i] > y[i]) return true;
            if (x[i] < y[i]) return false;
        }
        return false;
    }
    B2_HD static void sub_n(uint32_t* x, const uint32_t* y) {          // x -= y (x >= y)
        x[0] = cc::sub_cc(x[0], y[0]);
#pragma unroll
        for (int i = 1; i < 7; ++i) x[i] = cc::subc_cc(x[i], y[i]);
        x[7] = cc::subc(x[7], y[7]);
    }
    B2_HD static void add_n(uint32_t* x, const uint32_t* y) {          // x += y (no overflow: < 2^256)
        x[0] = cc::add_cc(x[0], y[0]);
#pragma unroll
        for (int i = 1; i < 7; ++i) x[i] = cc::addc_cc(x[i], y[i]);
        x[7] = cc::addc(x[7], y[7]);
    }
    B2_HD static Fp from_u32(uint32_t v) { Fp o = zero(); o.l[0] = v; return to_mont(o); }
    // start * base^e by square-and-multiply
    B2_HD static Fp pow_u64(Fp base, uint64_t e, Fp start = one()) {
        while (e) {
            if (e & 1) start = mul(start, base);
            base = sqr(base);
            e >>= 1;
        }
        return start;
    }
};

typedef Fp<FqParams> Fq;
typedef Fp<FrParams> Fr;

// ---------------------------------------------------------------------------------------------
// Fq2 = Fq[u]/(u^2 + 1)   (arkworks Fq2Config for BN254: NONRESIDUE = -1)
// ---------------------------------------------------------------------------------------------
struct Fq2 {
    Fq c0, c1;
    B2_HD static Fq2 zero() { Fq2 r; r.c0 = Fq::zero(); r.c1 = Fq::zero(); return r; }
    B2_HD static Fq2 one() { Fq2 r; r.c0 = Fq::one(); r.c1 = Fq::zero(); return r; }
    B2_HD bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
    B2_HD bool operator==(const Fq2& b) const { return c0 == b.c0 && c1 == b.c1; }
    B2_HD bool operator!=(const Fq2& b) const { return !(*this == b); }
    B2_HD static Fq2 add(const Fq2& a, const Fq2& b) { Fq2 r; r.c0 = Fq::add(a.c0, b.c0); r.c1 = Fq::add(a.c1, b.c1); return r; }
    B2_HD static Fq2 sub(const Fq2& a, const Fq2& b) { Fq2 r; r.c0 = Fq::sub(a.c0, b.c0); r.c1 = Fq::sub(a.c1, b.c1); return r; }
    B2_HD static Fq2 neg(const Fq2& a) { Fq2 r; r.c0 = Fq::neg(a.c0); r.c1 = Fq::neg(a.c1); return r; }
    B2_HD static Fq2 dbl(const Fq2& a) { return add(a, a); }
    // one out-of-line unit per Fq2 product (3 inlined Fq products): 10 calls per mixed add instead of 28.  Three
    // unreduced products and two reductions (336 wide multiply-adds) beat three full products (384).
    B2_HD_NI static Fq2 mul(const Fq2 a, const Fq2 b) {
        // c0 = a0 b0 - a1 b1, c1 = (a0 + a1)(b0 + b1) - a0 b0 - a1 b1, reduced once each.  Bounds: the products of canonical
        // values are < p^2; sa, sb = a0 + a1, b0 + b1 < 2p (no reduction: < 2^255), so sa sb < 4 p^2 < 2^512 and
        // c1's integer = a0 b1 + a1 b0 < 2 p^2 < 2 p 2^256; c0's = a0 b0 - a1 b1 + p 2^256 in (0, 2 p 2^256).
        uint32_t t0[16], t1[16], t2[16], sa[8], sb[8];
        Fq::mul_wide(t0, a.c0.l, b.c0.l);
        Fq::mul_wide(t1, a.c1.l, b.c1.l);
        sa[0] = cc::add_cc(a.c0.l[0], a.c1.l[0]);
#pragma unroll
        for (int i = 1; i < 7; ++i) sa[i] = cc::addc_cc(a.c0.l[i], a.c1.l[i]);
        sa[7] = cc::addc(a.c0.l[7], a.c1.l[7]);
        sb[0] = cc::add_cc(b.c0.l[0], b.c1.l[0]);
#pragma unroll
        for (int i = 1; i < 7; ++i) sb[i] = cc::addc_cc(b.c0.l[i], b.c1.l[i]);
        sb[7] = cc::addc(b.c0.l[7], b.c1.l[7]);
        Fq::mul_wide(t2, sa, sb);
        Fq::sub_wide(t2, t0);
        Fq::sub_wide(t2, t1);                                   // a0 b1 + a1 b0
        Fq::add_mod_hi(t0);
        Fq::sub_wide(t0, t1);                                   // a0 b0 - a1 b1 + p 2^256
        Fq2 r;
        Fq::template redc<2>(r.c0, t0);
        Fq::template redc<2>(r.c1, t2);
        return r;
    }
    B2_HD_NI static Fq2 sqr(const Fq2 a) {
        Fq t = Fq::mul(Fq::add(a.c0, a.c1), Fq::sub(a.c0, a.c1));
        Fq u = Fq::mul(a.c0, a.c1);
        Fq2 r; r.c0 = t; r.c1 = Fq::dbl(u); return r;
    }
    // K Fq2 products, each as 3 row-interleaved Fq products (see Fp::mul_k)
    template <int K>
    B2_HD static void mul_group(Fq2* r, const Fq2* a, const Fq2* b) {
#pragma unroll
        for (int k = 0; k < K; ++k) {
            Fq x[3], y[3], p[3];
            x[0] = a[k].c0; y[0] = b[k].c0;
            x[1] = a[k].c1; y[1] = b[k].c1;
            x[2] = Fq::add(a[k].c0, a[k].c1); y[2] = Fq::add(b[k].c0, b[k].c1);
            Fq::template mul_k<3>(p, x, y);
            r[k].c0 = Fq::sub(p[0], p[1]);
            r[k].c1 = Fq::sub(Fq::sub(p[2], p[0]), p[1]);
        }
    }
    B2_HD_NI static Fq2 inv(const Fq2& a) {
        Fq n = Fq::inv(Fq::add(Fq::sqr(a.c0), Fq::sqr(a.c1)));
        Fq2 r; r.c0 = Fq::mul(a.c0, n); r.c1 = Fq::neg(Fq::mul(a.c1, n)); return r;
    }
};

#ifdef __CUDACC__
// 16-byte vector load / store of a field element, a point or any other T whose size is a multiple of 16 bytes
template <class T>
__device__ __forceinline__ T ld16(const T* p) {
    static_assert(sizeof(T) % 16 == 0, "16-byte multiple");
    T r;
    const uint4* s = reinterpret_cast<const uint4*>(p);
    uint4* d = reinterpret_cast<uint4*>(&r);
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 16); ++i) d[i] = s[i];
    return r;
}
// the same at an untyped (16-byte aligned) address, e.g. a byte offset into a packed record
template <class T>
__device__ __forceinline__ T ld16(const void* p) { return ld16(static_cast<const T*>(p)); }
template <class T>
__device__ __forceinline__ void st16(T* p, const T& v) {
    static_assert(sizeof(T) % 16 == 0, "16-byte multiple");
    const uint4* s = reinterpret_cast<const uint4*>(&v);
    uint4* d = reinterpret_cast<uint4*>(p);
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 16); ++i) d[i] = s[i];
}

// w_n, the primitive 2^log_n-th root of unity of the field NTT (its inverse if `inverse`), log_n <= 28
__device__ __forceinline__ Fr fr_root_of_unity(unsigned log_n, bool inverse) {
    Fr w;
#pragma unroll
    for (int i = 0; i < 8; ++i) w.l[i] = inverse ? FrParams::root28_inv(i) : FrParams::root28(i);
    for (unsigned k = log_n; k < 28; ++k) w = Fr::sqr(w);
    return w;
}
#endif  // __CUDACC__

}  // namespace b200zk
