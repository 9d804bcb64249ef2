// codec.cuh -- field / point helpers of the ark-serialize Compress::Yes codec (see codec.cu), host + device so that
// tests/host/codec_host_test.cpp checks the square roots and the (de)compression rules against the oracle without a GPU.
#pragma once
#include "ec.cuh"

namespace b200zk {

// a^((p+1)/4) in Fq
B2_HD_NI Fq fq_pow_p1_4(const Fq& a) {
    // e = (p + 1) / 4, from the modulus limbs
    uint32_t e[8];
    uint32_t carry = 1;
    for (int i = 0; i < 8; ++i) {
        uint64_t t = (uint64_t)FqParams::mod(i) + carry;
        e[i] = (uint32_t)t;
        carry = (uint32_t)(t >> 32);
    }
    for (int i = 0; i < 8; ++i) e[i] = (e[i] >> 2) | (i < 7 ? e[i + 1] << 30 : 0);
    Fq res = Fq::one();
    for (int i = 253; i >= 0; --i) {
        res = Fq::mul_ni(res, res);
        if ((e[i >> 5] >> (i & 31)) & 1) res = Fq::mul_ni(res, a);
    }
    return res;
}

B2_HD_NI bool fq_sqrt(const Fq& a, Fq* out) {
    Fq s = fq_pow_p1_4(a);
    *out = s;
    return Fq::mul_ni(s, s) == a;
}

// x / 2 (works on Montgomery representatives as on plain ones: the map is linear)
B2_HD Fq fq_half(const Fq& a) {
    uint32_t t[9];
    for (int i = 0; i < 8; ++i) t[i] = a.l[i];
    t[8] = 0;
    if (a.l[0] & 1) {
        uint32_t carry = 0;
        for (int i = 0; i < 8; ++i) {
            uint64_t s = (uint64_t)t[i] + FqParams::mod(i) + carry;
            t[i] = (uint32_t)s;
            carry = (uint32_t)(s >> 32);
        }
        t[8] = carry;
    }
    Fq r;
    for (int i = 0; i < 8; ++i) r.l[i] = (t[i] >> 1) | (t[i + 1] << 31);
    return r;
}

// square root in Fq2 = Fq[u]/(u^2+1), "complex method": sqrt(a0 + a1 u) = x0 + x1 u with
// x0^2 = (a0 +- |a|) / 2, x1 = a1 / (2 x0), |a| = sqrt(a0^2 + a1^2)
B2_HD_NI bool fq2_sqrt(const Fq2& a, Fq2* out) {
    if (a.is_zero()) { *out = Fq2::zero(); return true; }
    if (a.c1.is_zero()) {
        Fq s;
        if (fq_sqrt(a.c0, &s)) { out->c0 = s; out->c1 = Fq::zero(); return true; }
        if (!fq_sqrt(Fq::neg(a.c0), &s)) return false;       // cannot happen: -1 is a non-residue
        out->c0 = Fq::zero(); out->c1 = s;
        return true;
    }
    Fq norm = Fq::add(Fq::mul_ni(a.c0, a.c0), Fq::mul_ni(a.c1, a.c1));
    Fq alpha;
    if (!fq_sqrt(norm, &alpha)) return false;
    Fq delta = fq_half(Fq::add(a.c0, alpha));
    Fq x0;
    if (!fq_sqrt(delta, &x0)) {
        delta = fq_half(Fq::sub(a.c0, alpha));
        if (!fq_sqrt(delta, &x0)) return false;
    }
    Fq x1 = Fq::mul_ni(a.c1, Fq::inv(Fq::dbl(x0)));
    out->c0 = x0; out->c1 = x1;
    return Fq2::sqr(*out) == a;
}

B2_HD bool fq_is_larger(const Fq& y) {       // arkworks: y > -y as canonical integers
    Fq a = Fq::from_mont(y), b = Fq::from_mont(Fq::neg(y));
    for (int i = 7; i >= 0; --i) {
        if (a.l[i] > b.l[i]) return true;
        if (a.l[i] < b.l[i]) return false;
    }
    return false;
}
B2_HD bool fq2_is_larger(const Fq2& y) { return y.c1.is_zero() ? fq_is_larger(y.c0) : fq_is_larger(y.c1); }

// 32 little-endian bytes (flags already masked off) -> canonical limbs; false when >= p
B2_HD bool fq_from_bytes(const uint8_t* in, uint8_t top_mask, Fq* out) {
    Fq x;
    for (int i = 0; i < 8; ++i) {
        uint32_t w = 0;
        for (int b = 0; b < 4; ++b) {
            uint32_t byte = in[4 * i + b];
            if (4 * i + b == 31) byte &= top_mask;
            w |= byte << (8 * b);
        }
        x.l[i] = w;
    }
    bool lt = false;                                   // x < p ?
    for (int i = 7; i >= 0; --i) {
        if (x.l[i] < FqParams::mod(i)) { lt = true; break; }
        if (x.l[i] > FqParams::mod(i)) break;
    }
    *out = Fq::to_mont(x);
    return lt;
}
B2_HD void fq_to_bytes(const Fq& xm, uint8_t* out) {
    Fq x = Fq::from_mont(xm);
    for (int i = 0; i < 32; ++i) out[i] = (uint8_t)(x.l[i >> 2] >> (8 * (i & 3)));
}

B2_HD bool is_larger(const Fq& y) { return fq_is_larger(y); }
B2_HD bool is_larger(const Fq2& y) { return fq2_is_larger(y); }

// ---- the curve equation, y from x and a sign, and the order-r subgroup test, for ffjs_decode ----------------------------
// g1_decode / g2_decode below keep their own inline copies: built on these helpers, k_g1_decompress went from 68 to 56
// registers and k_g2_decompress from 246 to 252 (sm_90a), and those kernels are left as they were.
B2_HD Fq curve_rhs(const Fq& x) {                // x^3 + b on G1
    Fq bb;
    for (int k = 0; k < 8; ++k) bb.l[k] = CurveConst::g1_b(k);
    return Fq::add(Fq::mul_ni(Fq::mul_ni(x, x), x), bb);
}
B2_HD Fq2 curve_rhs(const Fq2& x) {              // x^3 + b' on the twist
    Fq2 bb;
    for (int k = 0; k < 8; ++k) { bb.c0.l[k] = CurveConst::g2_b_c0(k); bb.c1.l[k] = CurveConst::g2_b_c1(k); }
    return Fq2::add(Fq2::mul(Fq2::sqr(x), x), bb);
}
B2_HD Fq field_sqr(const Fq& a) { return Fq::mul_ni(a, a); }
B2_HD Fq2 field_sqr(const Fq2& a) { return Fq2::sqr(a); }
B2_HD bool field_sqrt(const Fq& a, Fq* out) { return fq_sqrt(a, out); }
B2_HD bool field_sqrt(const Fq2& a, Fq2* out) { return fq2_sqrt(a, out); }

// the y of x's curve point that is_larger(y) == larger; false when x^3 + b is not a square (no point has that x)
template <class F>
B2_HD bool curve_y(const F& x, bool larger, F* y) {
    if (!field_sqrt(curve_rhs(x), y)) return false;
    if (is_larger(*y) != larger) *y = F::neg(*y);
    return true;
}

// [r] P == O.  G1 has cofactor 1, so every G1 point passes; the twist has a large cofactor.
B2_HD bool in_subgroup(const affine_t<Fq>&) { return true; }
B2_HD bool in_subgroup(const affine_t<Fq2>& p) {
    uint32_t r[8];
    for (int k = 0; k < 8; ++k) r[k] = FrParams::mod(k);
    return xyzz_t<Fq2>::mul_scalar(xyzz_t<Fq2>::from_affine(p), r).is_inf();
}

// one G1 / G2 encoding -> affine point; false when it is not a valid encoding (the point is then left at infinity)
B2_HD_NI bool g1_decode(const uint8_t* b, affine_t<Fq>* out) {
    *out = affine_t<Fq>::infinity();
    uint8_t flags = b[31] & 0xC0;
    if (flags & 0x40) {
        for (int k = 0; k < 32; ++k) if ((k == 31 ? (b[k] & 0x3F) : b[k]) != 0) return false;
        return (flags & 0x80) == 0;
    }
    Fq x;
    if (!fq_from_bytes(b, 0x3F, &x)) return false;
    Fq bb;
    for (int k = 0; k < 8; ++k) bb.l[k] = CurveConst::g1_b(k);
    Fq y2 = Fq::add(Fq::mul_ni(Fq::mul_ni(x, x), x), bb), y;
    if (!fq_sqrt(y2, &y)) return false;
    if (fq_is_larger(y) != ((flags & 0x80) != 0)) y = Fq::neg(y);
    out->x = x; out->y = y;
    return true;
}

B2_HD_NI bool g2_decode(const uint8_t* b, bool check_subgroup, affine_t<Fq2>* out) {
    *out = affine_t<Fq2>::infinity();
    uint8_t flags = b[63] & 0xC0;
    if (flags & 0x40) {
        for (int k = 0; k < 64; ++k) if ((k == 63 ? (b[k] & 0x3F) : b[k]) != 0) return false;
        return (flags & 0x80) == 0;
    }
    Fq2 x;
    bool ok = fq_from_bytes(b, 0xFF, &x.c0);
    ok = fq_from_bytes(b + 32, 0x3F, &x.c1) && ok;
    if (!ok) return false;
    Fq2 bb;
    for (int k = 0; k < 8; ++k) { bb.c0.l[k] = CurveConst::g2_b_c0(k); bb.c1.l[k] = CurveConst::g2_b_c1(k); }
    Fq2 y2 = Fq2::add(Fq2::mul(Fq2::sqr(x), x), bb), y;
    if (!fq2_sqrt(y2, &y)) return false;
    if (fq2_is_larger(y) != ((flags & 0x80) != 0)) y = Fq2::neg(y);
    affine_t<Fq2> p;
    p.x = x; p.y = y;
    if (check_subgroup) {                       // [r] P == O  (the twist has a large cofactor)
        uint32_t r[8];
        for (int k = 0; k < 8; ++k) r[k] = FrParams::mod(k);
        if (!xyzz_t<Fq2>::mul_scalar(xyzz_t<Fq2>::from_affine(p), r).is_inf()) return false;
    }
    *out = p;
    return true;
}

B2_HD void g1_encode(const affine_t<Fq>& p, uint8_t* b) {
    if (p.is_inf()) {
        for (int k = 0; k < 32; ++k) b[k] = 0;
        b[31] = 0x40;
        return;
    }
    fq_to_bytes(p.x, b);
    if (fq_is_larger(p.y)) b[31] |= 0x80;
}

// ---- ffjavascript's encodings (toRprUncompressed / toRprCompressed), the bytes snarkjs hashes in a phase-1 ceremony -----
// canonical big-endian; an Fq2 element as c1 then c0
B2_HD void ffjs_put(const Fq& am, uint8_t* out) {
    const Fq a = Fq::from_mont(am);
    for (int i = 0; i < 32; ++i) out[31 - i] = (uint8_t)(a.l[i >> 2] >> (8 * (i & 3)));
}
B2_HD void ffjs_put(const Fq2& a, uint8_t* out) {
    ffjs_put(a.c1, out);
    ffjs_put(a.c0, out + 32);
}
// the inverse: canonical big-endian bytes (byte 0 ANDed with top_mask) -> Montgomery form; false when the value is >= q
B2_HD bool ffjs_get(const uint8_t* in, Fq* out, uint8_t top_mask = 0xFF) {
    uint8_t le[32];
    for (int i = 0; i < 32; ++i) le[i] = in[31 - i];
    return fq_from_bytes(le, top_mask, out);
}
B2_HD bool ffjs_get(const uint8_t* in, Fq2* out, uint8_t top_mask = 0xFF) {
    const bool ok1 = ffjs_get(in, &out->c1, top_mask);
    const bool ok0 = ffjs_get(in + 32, &out->c0);
    return ok1 && ok0;
}

// COMPRESSED = false: x || y (64 / 128 bytes); true: x with 0x80 in byte 0 when y is the larger of (y, -y) (32 / 64
// bytes).  Infinity: 0x40 then zeros in both.
template <class F, bool COMPRESSED>
B2_HD void ffjs_encode(const affine_t<F>& p, uint8_t* b) {
    constexpr int FB = (int)sizeof(F), LEN = COMPRESSED ? FB : 2 * FB;
    if (p.is_inf()) {
        for (int k = 0; k < LEN; ++k) b[k] = 0;
        b[0] = 0x40;
        return;
    }
    ffjs_put(p.x, b);
    if (COMPRESSED) {
        if (is_larger(p.y)) b[0] |= 0x80;
    } else {
        ffjs_put(p.y, b + FB);
    }
}

// The inverse of ffjs_encode: one encoding -> affine point; false when it is not a valid encoding (the point is then
// left at infinity).  Valid: infinity is 0x40 then zeros; uncompressed is x || y, both < q, byte 0's top bits clear and
// y^2 = x^3 + b; compressed is x < q (0x80 masked off) with a curve point, y the root whose is_larger matches 0x80.
// check_subgroup also requires [r] P == O (G2 only: G1 has cofactor 1).
template <class F, bool COMPRESSED>
B2_HD bool ffjs_decode(const uint8_t* b, bool check_subgroup, affine_t<F>* out) {
    constexpr int FB = (int)sizeof(F), LEN = COMPRESSED ? FB : 2 * FB;
    *out = affine_t<F>::infinity();
    if (b[0] & 0x40) {
        for (int k = 1; k < LEN; ++k) if (b[k] != 0) return false;
        return b[0] == 0x40;
    }
    if (!COMPRESSED && (b[0] & 0x80)) return false;
    affine_t<F> p;
    if (!ffjs_get(b, &p.x, 0x3F)) return false;
    if (COMPRESSED) {
        if (!curve_y(p.x, (b[0] & 0x80) != 0, &p.y)) return false;
    } else {
        if (!ffjs_get(b + FB, &p.y)) return false;
        if (!(field_sqr(p.y) == curve_rhs(p.x))) return false;
    }
    if (check_subgroup && !in_subgroup(p)) return false;
    *out = p;
    return true;
}

B2_HD void g2_encode(const affine_t<Fq2>& p, uint8_t* b) {
    if (p.is_inf()) {
        for (int k = 0; k < 64; ++k) b[k] = 0;
        b[63] = 0x40;
        return;
    }
    fq_to_bytes(p.x.c0, b);
    fq_to_bytes(p.x.c1, b + 32);
    if (fq2_is_larger(p.y)) b[63] |= 0x80;
}

}  // namespace b200zk
