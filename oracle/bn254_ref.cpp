// oracle/bn254_ref.cpp -- CPU twin of the reference's arkworks path (TEST INFRASTRUCTURE ONLY).
//
// Nothing under distributed_groth16_b200/ may link, load or call this file.  It exists so that
//   (1) tests/ can check the CUDA path bit-for-bit at sizes pure Python cannot reach, and
//   (2) bench.py's cpu_baseline / `--impl reference` leg has a CPU arm to time ("kind": "port").
//
// It restates, for BN254, what the reference obtains from the un-vendored, unpinned arkworks 0.4
// crates (ark-ff / ark-ec / ark-poly / ark-groth16 fork; /root/reference/.gitignore:2 ignores
// Cargo.lock), following the reference's own call sites:
//   * G::msm                      dist-primitives/src/dmsm/mod.rs:82      -> orc_msm_g1 / orc_msm_g2
//       (ark-ec VariableBaseMSM::msm_bigint_wnaf: window c = ln(n)+2 (3 if n<32), signed digits,
//        windows processed in parallel [rayon <-> OpenMP], running-sum bucket reduction)
//   * dom.fft / dom.ifft          dist-primitives/src/dfft/mod.rs:17-95   -> orc_ntt
//   * qap mat-vec                 groth16/src/qap.rs:60-67                -> orc_fr_spmv
//   * CircomReduction h           ark-circom/src/circom/qap.rs:64-89      -> orc_h_circom
//   * prove::{A,B,C} + assembly   groth16/src/prove.rs:21-136,
//                                 groth16/examples/sha256.rs:208-212      -> orc_groth16_prove
//   * Compress::Yes encoding      zk-cli/src/main.rs:130-136              -> (inside orc_groth16_prove)
// Parity pin: tests/test_oracle_*.py check every entry point against oracle/bn254.py, which is
// itself pinned on the reference's golden vectors (see its header).
//
// Data layout (same as include/b200zk.h): field element = 4 x u64 little-endian limbs in
// Montgomery form (R = 2^256) -- arkworks' in-memory Fp256<MontBackend>; G1 affine = x||y (8 limbs),
// G2 affine = x.c0||x.c1||y.c0||y.c1 (16 limbs); the all-zero encoding is the point at infinity
// (ark-circom/src/zkey.rs:353-373).
#include <cstdint>
#include <cstring>
#include <cstdlib>
#include <vector>
#include <algorithm>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef uint64_t u64;
typedef unsigned __int128 u128;

// ----------------------------------------------------------------------------------------------
// Prime fields
// ----------------------------------------------------------------------------------------------
struct FieldConst {
    u64 mod[4];
    u64 inv;      // -mod^{-1} mod 2^64
    u64 r1[4];    // R mod p   (Montgomery one)
    u64 r2[4];    // R^2 mod p
};

static inline int geq4(const u64* a, const u64* b) {
    for (int i = 3; i >= 0; --i) {
        if (a[i] > b[i]) return 1;
        if (a[i] < b[i]) return 0;
    }
    return 1;
}
static inline u64 add4(u64* r, const u64* a, const u64* b) {
    u128 c = 0;
    for (int i = 0; i < 4; ++i) { c += (u128)a[i] + b[i]; r[i] = (u64)c; c >>= 64; }
    return (u64)c;
}
static inline u64 sub4(u64* r, const u64* a, const u64* b) {
    u64 br = 0;
    for (int i = 0; i < 4; ++i) {
        u128 t = (u128)a[i] - b[i] - br;
        r[i] = (u64)t; br = (u64)(t >> 64) & 1;
    }
    return br;
}

static void field_const_init(FieldConst& fc, const u64 mod[4]) {
    memcpy(fc.mod, mod, 32);
    u64 x = 1;                                   // Newton: x = mod^{-1} mod 2^64
    for (int i = 0; i < 6; ++i) x *= 2 - mod[0] * x;
    fc.inv = (u64)0 - x;
    u64 t[4] = {1, 0, 0, 0};                     // 2^k mod p by repeated doubling
    for (int k = 0; k < 512; ++k) {
        u64 c = add4(t, t, t);
        if (c || geq4(t, mod)) sub4(t, t, mod);
        if (k == 255) memcpy(fc.r1, t, 32);
    }
    memcpy(fc.r2, t, 32);
}

// BN254 moduli (mathematical constants; cross-checked against oracle/bn254.py in tests)
static const u64 FQ_MOD[4] = {0x3c208c16d87cfd47ULL, 0x97816a916871ca8dULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL};
static const u64 FR_MOD[4] = {0x43e1f593f0000001ULL, 0x2833e84879b97091ULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL};
static FieldConst FQC, FRC;

template <const FieldConst* FC>
struct Fp {
    u64 l[4];
    static Fp zero() { Fp r; memset(r.l, 0, 32); return r; }
    static Fp one() { Fp r; memcpy(r.l, FC->r1, 32); return r; }
    bool is_zero() const { return (l[0] | l[1] | l[2] | l[3]) == 0; }
    bool operator==(const Fp& o) const { return memcmp(l, o.l, 32) == 0; }
    bool operator!=(const Fp& o) const { return !(*this == o); }
    Fp operator+(const Fp& o) const {
        Fp r; u64 c = add4(r.l, l, o.l);
        if (c || geq4(r.l, FC->mod)) sub4(r.l, r.l, FC->mod);
        return r;
    }
    Fp operator-(const Fp& o) const {
        Fp r; u64 b = sub4(r.l, l, o.l);
        if (b) add4(r.l, r.l, FC->mod);
        return r;
    }
    Fp neg() const { if (is_zero()) return *this; Fp r; sub4(r.l, FC->mod, l); return r; }
    Fp dbl() const { return *this + *this; }
    static inline void mont_mul(u64* out, const u64* a, const u64* b) {
        u64 t[6] = {0, 0, 0, 0, 0, 0};
        for (int i = 0; i < 4; ++i) {
            u128 c = 0;
            for (int j = 0; j < 4; ++j) {
                c += (u128)a[j] * b[i] + t[j];
                t[j] = (u64)c; c >>= 64;
            }
            c += t[4]; t[4] = (u64)c; t[5] = (u64)(c >> 64);
            u64 m = t[0] * FC->inv;
            c = (u128)m * FC->mod[0] + t[0]; c >>= 64;
            for (int j = 1; j < 4; ++j) {
                c += (u128)m * FC->mod[j] + t[j];
                t[j - 1] = (u64)c; c >>= 64;
            }
            c += t[4]; t[3] = (u64)c; t[4] = t[5] + (u64)(c >> 64);
        }
        if (t[4] || geq4(t, FC->mod)) sub4(t, t, FC->mod);
        memcpy(out, t, 32);
    }
    Fp operator*(const Fp& o) const { Fp r; mont_mul(r.l, l, o.l); return r; }
    Fp sqr() const { return *this * *this; }
    Fp to_mont() const { Fp r; mont_mul(r.l, l, FC->r2); return r; }      // canonical -> Montgomery
    Fp from_mont() const { u64 o1[4] = {1, 0, 0, 0}; Fp r; mont_mul(r.l, l, o1); return r; }
    Fp pow(const u64* e, int nlimbs) const {
        Fp res = one();
        for (int i = nlimbs * 64 - 1; i >= 0; --i) {
            res = res.sqr();
            if ((e[i / 64] >> (i % 64)) & 1) res = res * *this;
        }
        return res;
    }
    Fp inv() const {                                        // Fermat: a^(p-2)
        u64 e[4]; u64 two[4] = {2, 0, 0, 0};
        sub4(e, FC->mod, two);
        return pow(e, 4);
    }
    static Fp from_u64(u64 v) { Fp r = zero(); r.l[0] = v; return r.to_mont(); }
};

typedef Fp<&FQC> Fq;
typedef Fp<&FRC> Fr;

struct Fq2 {
    Fq c0, c1;
    static Fq2 zero() { return {Fq::zero(), Fq::zero()}; }
    static Fq2 one() { return {Fq::one(), Fq::zero()}; }
    bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
    bool operator==(const Fq2& o) const { return c0 == o.c0 && c1 == o.c1; }
    bool operator!=(const Fq2& o) const { return !(*this == o); }
    Fq2 operator+(const Fq2& o) const { return {c0 + o.c0, c1 + o.c1}; }
    Fq2 operator-(const Fq2& o) const { return {c0 - o.c0, c1 - o.c1}; }
    Fq2 neg() const { return {c0.neg(), c1.neg()}; }
    Fq2 dbl() const { return {c0.dbl(), c1.dbl()}; }
    Fq2 operator*(const Fq2& o) const {                     // u^2 = -1
        Fq a = c0 * o.c0, b = c1 * o.c1;
        Fq c = (c0 + c1) * (o.c0 + o.c1);
        return {a - b, c - a - b};
    }
    Fq2 sqr() const {
        Fq a = (c0 + c1) * (c0 - c1);
        Fq b = (c0 * c1).dbl();
        return {a, b};
    }
    Fq2 inv() const {
        Fq n = (c0.sqr() + c1.sqr()).inv();
        return {c0 * n, (c1 * n).neg()};
    }
};

// ----------------------------------------------------------------------------------------------
// Short-Weierstrass curves y^2 = x^3 + b, Jacobian coordinates (a = 0)
// ----------------------------------------------------------------------------------------------
template <class F>
struct Aff { F x, y; bool inf; };
template <class F>
struct Jac {
    F X, Y, Z;
    static Jac identity() { return {F::one(), F::one(), F::zero()}; }
    bool is_inf() const { return Z.is_zero(); }
};

template <class F>
static Jac<F> jac_double(const Jac<F>& p) {
    if (p.is_inf()) return p;
    F A = p.X.sqr(), B = p.Y.sqr(), C = B.sqr();
    F t = (p.X + B).sqr() - A - C;
    F D = t.dbl();
    F E = A.dbl() + A;
    F Fv = E.sqr();
    F X3 = Fv - D.dbl();
    F C8 = C.dbl().dbl().dbl();
    F Y3 = E * (D - X3) - C8;
    F Z3 = (p.Y * p.Z).dbl();
    return {X3, Y3, Z3};
}

template <class F>
static Jac<F> jac_add(const Jac<F>& p, const Jac<F>& q) {
    if (p.is_inf()) return q;
    if (q.is_inf()) return p;
    F Z1Z1 = p.Z.sqr(), Z2Z2 = q.Z.sqr();
    F U1 = p.X * Z2Z2, U2 = q.X * Z1Z1;
    F S1 = p.Y * q.Z * Z2Z2, S2 = q.Y * p.Z * Z1Z1;
    if (U1 == U2) {
        if (S1 == S2) return jac_double(p);
        return Jac<F>::identity();
    }
    F H = U2 - U1, Rr = S2 - S1;
    F HH = H.sqr(), HHH = H * HH, V = U1 * HH;
    F X3 = Rr.sqr() - HHH - V.dbl();
    F Y3 = Rr * (V - X3) - S1 * HHH;
    F Z3 = p.Z * q.Z * H;
    return {X3, Y3, Z3};
}

template <class F>
static Jac<F> jac_add_mixed(const Jac<F>& p, const Aff<F>& q, bool negate = false) {
    if (q.inf) return p;
    F qy = negate ? q.y.neg() : q.y;
    if (p.is_inf()) return {q.x, qy, F::one()};
    F Z1Z1 = p.Z.sqr();
    F U2 = q.x * Z1Z1;
    F S2 = qy * p.Z * Z1Z1;
    if (p.X == U2) {
        if (p.Y == S2) return jac_double(p);
        return Jac<F>::identity();
    }
    F H = U2 - p.X, Rr = S2 - p.Y;
    F HH = H.sqr(), HHH = H * HH, V = p.X * HH;
    F X3 = Rr.sqr() - HHH - V.dbl();
    F Y3 = Rr * (V - X3) - p.Y * HHH;
    F Z3 = p.Z * H;
    return {X3, Y3, Z3};
}

template <class F>
static Aff<F> jac_to_affine(const Jac<F>& p) {
    if (p.is_inf()) return {F::zero(), F::zero(), true};
    F zi = p.Z.inv(), zi2 = zi.sqr();
    return {p.X * zi2, p.Y * zi2 * zi, false};
}

template <class F>
static Jac<F> jac_mul_bits(const Jac<F>& p, const u64* k, int nbits) {
    Jac<F> acc = Jac<F>::identity();
    for (int i = nbits - 1; i >= 0; --i) {
        acc = jac_double(acc);
        if ((k[i / 64] >> (i % 64)) & 1) acc = jac_add(acc, p);
    }
    return acc;
}

template <class F> struct Limbs;
template <> struct Limbs<Fq> {
    static const int N = 4;
    static Fq load(const u64* p) { Fq r; memcpy(r.l, p, 32); return r; }
    static void store(u64* p, const Fq& v) { memcpy(p, v.l, 32); }
};
template <> struct Limbs<Fq2> {
    static const int N = 8;
    static Fq2 load(const u64* p) { return {Limbs<Fq>::load(p), Limbs<Fq>::load(p + 4)}; }
    static void store(u64* p, const Fq2& v) { Limbs<Fq>::store(p, v.c0); Limbs<Fq>::store(p + 4, v.c1); }
};

template <class F>
static Aff<F> load_affine(const u64* p) {
    Aff<F> a;
    a.x = Limbs<F>::load(p);
    a.y = Limbs<F>::load(p + Limbs<F>::N);
    a.inf = a.x.is_zero() && a.y.is_zero();
    return a;
}
template <class F>
static void store_affine(u64* p, const Aff<F>& a) {
    if (a.inf) { memset(p, 0, 16 * Limbs<F>::N); return; }
    Limbs<F>::store(p, a.x);
    Limbs<F>::store(p + Limbs<F>::N, a.y);
}

// ----------------------------------------------------------------------------------------------
// MSM -- restatement of ark-ec 0.4 VariableBaseMSM::msm_bigint_wnaf
// ----------------------------------------------------------------------------------------------
static inline unsigned ark_log2(size_t x) {                 // ark_std::log2 = ceil(log2 x)
    if (x <= 1) return 0;
    unsigned fl = 63 - __builtin_clzll((unsigned long long)x);
    return (x & (x - 1)) ? fl + 1 : fl;
}
static inline unsigned ark_window(size_t n) {               // ln_without_floats(n) + 2
    return n < 32 ? 3 : (ark_log2(n) * 69 / 100) + 2;
}

static void make_digits(const u64 s[4], unsigned w, unsigned num_bits, std::vector<int64_t>& out, size_t off, size_t stride) {
    const u64 radix = 1ULL << w, mask = radix - 1;
    unsigned digits = (num_bits + w - 1) / w;
    u64 carry = 0;
    for (unsigned i = 0; i < digits; ++i) {
        unsigned bit_off = i * w, idx = bit_off / 64, bit = bit_off % 64;
        u64 buf;
        if (bit < 64 - w || idx == 3) buf = s[idx] >> bit;
        else buf = (s[idx] >> bit) | (s[idx + 1] << (64 - bit));
        u64 coef = carry + (buf & mask);
        carry = (coef + radix / 2) >> w;
        int64_t d = (int64_t)coef - (int64_t)(carry << w);
        if (i == digits - 1) d += (int64_t)(carry << w);
        out[off + i * stride] = d;
    }
}

template <class F>
static Jac<F> msm_pippenger(const u64* bases, const u64* scalars, size_t n, int nthreads) {
    const int PL = 2 * Limbs<F>::N;
    if (n == 0) return Jac<F>::identity();
    unsigned c = ark_window(n);
    const unsigned num_bits = 254;
    unsigned nwin = (num_bits + c - 1) / c;
    // scalars: Montgomery -> canonical bigint (arkworks into_bigint), then signed digits
    std::vector<int64_t> digits((size_t)nwin * n);
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (long long i = 0; i < (long long)n; ++i) {
        Fr s; memcpy(s.l, scalars + 4 * i, 32);
        Fr cs = s.from_mont();
        make_digits(cs.l, c, num_bits, digits, (size_t)i, n);     // digits[w*n + i]
    }
    std::vector<Jac<F>> wsum(nwin);
#pragma omp parallel for num_threads(nthreads) schedule(dynamic, 1)
    for (int w = 0; w < (int)nwin; ++w) {
        std::vector<Jac<F>> buckets((size_t)1 << (c - 1), Jac<F>::identity());
        const int64_t* dg = digits.data() + (size_t)w * n;
        for (size_t i = 0; i < n; ++i) {
            int64_t d = dg[i];
            if (d == 0) continue;
            Aff<F> b = load_affine<F>(bases + (size_t)PL * i);
            if (d > 0) buckets[d - 1] = jac_add_mixed(buckets[d - 1], b, false);
            else buckets[-d - 1] = jac_add_mixed(buckets[-d - 1], b, true);
        }
        Jac<F> run = Jac<F>::identity(), res = Jac<F>::identity();
        for (size_t k = buckets.size(); k-- > 0;) {
            run = jac_add(run, buckets[k]);
            res = jac_add(res, run);
        }
        wsum[w] = res;
    }
    Jac<F> total = Jac<F>::identity();
    for (int w = (int)nwin - 1; w >= 1; --w) {
        total = jac_add(total, wsum[w]);
        for (unsigned k = 0; k < c; ++k) total = jac_double(total);
    }
    return jac_add(total, wsum[0]);
}

// ----------------------------------------------------------------------------------------------
// NTT over Fr (arkworks Radix2EvaluationDomain semantics: natural order in and out)
// ----------------------------------------------------------------------------------------------
static Fr fr_pow_u64(Fr b, u64 e) { u64 ee[1] = {e}; return b.pow(ee, 1); }

static Fr fr_root_of_unity(unsigned log_n) {                // 5^((r-1)/2^log_n)
    u64 e[4]; u64 one[4] = {1, 0, 0, 0};
    sub4(e, FR_MOD, one);
    for (unsigned k = 0; k < log_n; ++k) {                  // e >>= 1
        for (int i = 0; i < 4; ++i) e[i] = (e[i] >> 1) | (i < 3 ? (e[i + 1] << 63) : 0);
    }
    return Fr::from_u64(5).pow(e, 4);
}

static void bitrev_permute(Fr* a, unsigned log_n) {
    size_t n = (size_t)1 << log_n;
    for (size_t i = 0; i < n; ++i) {
        size_t j = 0;
        for (unsigned b = 0; b < log_n; ++b) j |= ((i >> b) & 1) << (log_n - 1 - b);
        if (j > i) std::swap(a[i], a[j]);
    }
}

static void ntt_core(Fr* a, unsigned log_n, bool inverse, int nthreads) {
    size_t n = (size_t)1 << log_n;
    if (n == 1) return;
    Fr omega = fr_root_of_unity(log_n);
    if (inverse) omega = omega.inv();
    std::vector<Fr> tw(n / 2);
    tw[0] = Fr::one();
    for (size_t i = 1; i < n / 2; ++i) tw[i] = tw[i - 1] * omega;
    bitrev_permute(a, log_n);
    for (unsigned s = 1; s <= log_n; ++s) {
        size_t len = (size_t)1 << s, half = len >> 1, step = n >> s;
#pragma omp parallel for num_threads(nthreads) schedule(static)
        for (long long bf = 0; bf < (long long)(n / 2); ++bf) {
            size_t blk = (size_t)bf / half, j = (size_t)bf % half;
            size_t i0 = blk * len + j, i1 = i0 + half;
            Fr u = a[i0], v = a[i1] * tw[j * step];
            a[i0] = u + v; a[i1] = u - v;
        }
    }
}

static void ntt_full(Fr* a, unsigned log_n, bool inverse, bool coset, int nthreads) {
    size_t n = (size_t)1 << log_n;
    Fr g = Fr::from_u64(5);
    if (coset && !inverse) {                                 // a[j] *= g^j
        Fr x = Fr::one();
        for (size_t j = 0; j < n; ++j) { a[j] = a[j] * x; x = x * g; }
    }
    ntt_core(a, log_n, inverse, nthreads);
    if (inverse) {
        Fr ninv = Fr::from_u64((u64)n).inv();
        Fr gi = g.inv(), x = ninv;
        for (size_t j = 0; j < n; ++j) {
            a[j] = a[j] * x;
            if (coset) x = x * gi;
        }
    }
}

// CircomReduction::witness_map_from_matrices after the mat-vec (ark-circom/src/circom/qap.rs:64-89)
static void h_circom(const Fr* a, const Fr* b, const Fr* c, unsigned log_m, Fr* h, int nthreads) {
    size_t m = (size_t)1 << log_m;
    Fr w2m = fr_root_of_unity(log_m + 1);
    std::vector<Fr> buf[3];
    const Fr* src[3] = {a, b, c};
    for (int k = 0; k < 3; ++k) {
        buf[k].assign(src[k], src[k] + m);
        ntt_full(buf[k].data(), log_m, true, false, nthreads);
        Fr x = Fr::one();
        for (size_t j = 0; j < m; ++j) { buf[k][j] = buf[k][j] * x; x = x * w2m; }   // distribute_powers
        ntt_full(buf[k].data(), log_m, false, false, nthreads);
    }
    for (size_t i = 0; i < m; ++i) h[i] = buf[0][i] * buf[1][i] - buf[2][i];
}

// ----------------------------------------------------------------------------------------------
// ark-serialize Compress::Yes
// ----------------------------------------------------------------------------------------------
static bool fq_gt_half(const Fq& y_mont) {                   // y > -y  <=>  y > (p-1)/2
    Fq y = y_mont.from_mont(), ny = y_mont.neg().from_mont();
    return geq4(y.l, ny.l) && !(y == ny);
}
static void compress_g1(const Aff<Fq>& p, uint8_t out[32]) {
    memset(out, 0, 32);
    if (p.inf) { out[31] |= 0x40; return; }
    Fq x = p.x.from_mont();
    memcpy(out, x.l, 32);
    if (fq_gt_half(p.y)) out[31] |= 0x80;
}
static void compress_g2(const Aff<Fq2>& p, uint8_t out[64]) {
    memset(out, 0, 64);
    if (p.inf) { out[63] |= 0x40; return; }
    Fq x0 = p.x.c0.from_mont(), x1 = p.x.c1.from_mont();
    memcpy(out, x0.l, 32); memcpy(out + 32, x1.l, 32);
    bool neg = p.y.c1.is_zero() ? fq_gt_half(p.y.c0) : fq_gt_half(p.y.c1);   // compare c1 first, then c0
    if (neg) out[63] |= 0x80;
}

// ----------------------------------------------------------------------------------------------
// deterministic dummy points: P_i = k_i * G, k_i = splitmix64(seed, i)   (mirrors the reference's
// dummy-CRS benches: groth16/examples/local_groth_bench.rs:21-52, groth16/src/proving_key.rs:112-155)
// ----------------------------------------------------------------------------------------------
static inline u64 splitmix64(u64 x) {
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}

static bool g_init_done = false;
static Aff<Fq> G1GEN;
static Aff<Fq2> G2GEN;

static Fq fq_from_dec(const char* s) {
    Fq acc = Fq::zero(), ten = Fq::from_u64(10);
    for (; *s; ++s) acc = acc * ten + Fq::from_u64((u64)(*s - '0'));
    return acc;
}

static void ensure_init() {
    if (g_init_done) return;
    field_const_init(FQC, FQ_MOD);
    field_const_init(FRC, FR_MOD);
    G1GEN = {Fq::from_u64(1), Fq::from_u64(2), false};
    // G2 generator, decimal coordinates as printed in ark-circom/src/zkey.rs:466-486 (test data)
    G2GEN.x = {fq_from_dec("10857046999023057135944570762232829481370756359578518086990519993285655852781"),
               fq_from_dec("11559732032986387107991004021392285783925812861821192530917403151452391805634")};
    G2GEN.y = {fq_from_dec("8495653923123431417604973247489272438418190587263600148770280649306958101930"),
               fq_from_dec("4082367875863433681332203403145435568316851327593401208105741076214120093531")};
    G2GEN.inf = false;
    g_init_done = true;
}

static int resolve_threads(int nthreads) {
#ifdef _OPENMP
    if (nthreads <= 0) nthreads = omp_get_max_threads();
#else
    nthreads = 1;
#endif
    return nthreads;
}

template <class F>
static void gen_points(const Aff<F>& gen, u64 seed, size_t n, u64* out, int nthreads) {
    const int PL = 2 * Limbs<F>::N;
    Jac<F> g = {gen.x, gen.y, F::one()};
#pragma omp parallel for num_threads(nthreads) schedule(static)
    for (long long i = 0; i < (long long)n; ++i) {
        u64 k = splitmix64(seed + (u64)i) | 1ULL;
        Aff<F> a = jac_to_affine(jac_mul_bits(g, &k, 64));
        store_affine<F>(out + (size_t)PL * i, a);
    }
}

template <class F>
static void msm_entry(const u64* bases, const u64* scalars, size_t n, u64* out_affine, int* out_is_inf, int nthreads) {
    Aff<F> r = jac_to_affine(msm_pippenger<F>(bases, scalars, n, nthreads));
    store_affine<F>(out_affine, r);
    *out_is_inf = r.inf ? 1 : 0;
}

template <class F>
static Jac<F> jac_mul_fr(const Jac<F>& p, const u64* k_mont) {
    Fr k; memcpy(k.l, k_mont, 32);
    Fr kc = k.from_mont();
    return jac_mul_bits(p, kc.l, 256);
}
template <class F>
static Jac<F> aff_to_jac(const Aff<F>& a) {
    if (a.inf) return Jac<F>::identity();
    return {a.x, a.y, F::one()};
}

// out[i] = scalars[i] * base (affine, Montgomery limbs): what `FixedBase::msm(.., g1_table, scalars)` yields in
// ark-groth16's generator (third-party; restated from its contract) -- used to rebuild the reference's proving key from
// the regenerated toxic waste (oracle/ark_rand.py).  Plain double-and-add per scalar, OpenMP over the scalars.
template <class F>
static void fixed_base_mul(const u64* base, const u64* scalars, size_t n, u64* out, int nthreads) {
    const int PL = 2 * Limbs<F>::N;
    Jac<F> g = aff_to_jac(load_affine<F>(base));
#pragma omp parallel for num_threads(nthreads) schedule(dynamic, 64)
    for (long long i = 0; i < (long long)n; ++i) {
        Aff<F> a = jac_to_affine(jac_mul_fr(g, scalars + 4 * (size_t)i));
        store_affine<F>(out + (size_t)PL * i, a);
    }
}

extern "C" {

int orc_num_threads(void) { return resolve_threads(0); }

// mod_q[4], mod_r[4], inv_q, inv_r, r1_q[4], r1_r[4], r2_q[4], r2_r[4]  (26 limbs)
void orc_constants(u64* out) {
    ensure_init();
    memcpy(out, FQC.mod, 32); memcpy(out + 4, FRC.mod, 32);
    out[8] = FQC.inv; out[9] = FRC.inv;
    memcpy(out + 10, FQC.r1, 32); memcpy(out + 14, FRC.r1, 32);
    memcpy(out + 18, FQC.r2, 32); memcpy(out + 22, FRC.r2, 32);
}

// op: 0 mul, 1 add, 2 sub, 3 inv(a), 4 to_mont(a), 5 from_mont(a); field: 0 Fq, 1 Fr
void orc_field_op(int field, int op, const u64* a, const u64* b, u64* out) {
    ensure_init();
    if (field == 0) {
        Fq x, y, r; memcpy(x.l, a, 32); if (b) memcpy(y.l, b, 32);
        switch (op) { case 0: r = x * y; break; case 1: r = x + y; break; case 2: r = x - y; break;
                      case 3: r = x.inv(); break; case 4: r = x.to_mont(); break; default: r = x.from_mont(); }
        memcpy(out, r.l, 32);
    } else {
        Fr x, y, r; memcpy(x.l, a, 32); if (b) memcpy(y.l, b, 32);
        switch (op) { case 0: r = x * y; break; case 1: r = x + y; break; case 2: r = x - y; break;
                      case 3: r = x.inv(); break; case 4: r = x.to_mont(); break; default: r = x.from_mont(); }
        memcpy(out, r.l, 32);
    }
}

void orc_g1_fixed_base_mul(const u64* base, const u64* scalars, size_t n, u64* out, int nthreads) {
    ensure_init(); fixed_base_mul<Fq>(base, scalars, n, out, resolve_threads(nthreads));
}
void orc_g2_fixed_base_mul(const u64* base, const u64* scalars, size_t n, u64* out, int nthreads) {
    ensure_init(); fixed_base_mul<Fq2>(base, scalars, n, out, resolve_threads(nthreads));
}

void orc_g1_generate(u64 seed, size_t n, u64* out, int nthreads) { ensure_init(); gen_points<Fq>(G1GEN, seed, n, out, resolve_threads(nthreads)); }
void orc_g2_generate(u64 seed, size_t n, u64* out, int nthreads) { ensure_init(); gen_points<Fq2>(G2GEN, seed, n, out, resolve_threads(nthreads)); }

// uniform Fr elements in Montgomery form: canonical value = (4 splitmix words) mod r (top bits masked, retry-free
// reduction by conditional subtraction: mask to 254 bits then subtract r up to 1x).
void orc_fr_generate(u64 seed, size_t n, u64* out) {
    ensure_init();
    for (size_t i = 0; i < n; ++i) {
        Fr v;
        for (int k = 0; k < 4; ++k) v.l[k] = splitmix64(seed * 0x100000001B3ULL + 4 * (u64)i + k);
        v.l[3] &= 0x3FFFFFFFFFFFFFFFULL;
        if (geq4(v.l, FR_MOD)) sub4(v.l, v.l, FR_MOD);
        // the 256-bit pattern is used directly as the Montgomery representation (still uniform)
        memcpy(out + 4 * i, v.l, 32);
    }
}

int orc_msm_g1(const u64* bases, const u64* scalars, size_t n, u64* out_affine, int* out_is_inf, int nthreads) {
    ensure_init(); msm_entry<Fq>(bases, scalars, n, out_affine, out_is_inf, resolve_threads(nthreads)); return 0;
}
int orc_msm_g2(const u64* bases, const u64* scalars, size_t n, u64* out_affine, int* out_is_inf, int nthreads) {
    ensure_init(); msm_entry<Fq2>(bases, scalars, n, out_affine, out_is_inf, resolve_threads(nthreads)); return 0;
}

// naive sum_i s_i * P_i by double-and-add (independent of the Pippenger code above)
int orc_msm_g1_naive(const u64* bases, const u64* scalars, size_t n, u64* out_affine, int* out_is_inf) {
    ensure_init();
    Jac<Fq> acc = Jac<Fq>::identity();
    for (size_t i = 0; i < n; ++i) acc = jac_add(acc, jac_mul_fr(aff_to_jac(load_affine<Fq>(bases + 8 * i)), scalars + 4 * i));
    Aff<Fq> r = jac_to_affine(acc); store_affine<Fq>(out_affine, r); *out_is_inf = r.inf; return 0;
}
int orc_msm_g2_naive(const u64* bases, const u64* scalars, size_t n, u64* out_affine, int* out_is_inf) {
    ensure_init();
    Jac<Fq2> acc = Jac<Fq2>::identity();
    for (size_t i = 0; i < n; ++i) acc = jac_add(acc, jac_mul_fr(aff_to_jac(load_affine<Fq2>(bases + 16 * i)), scalars + 4 * i));
    Aff<Fq2> r = jac_to_affine(acc); store_affine<Fq2>(out_affine, r); *out_is_inf = r.inf; return 0;
}

// 1 if every point is on its curve (or infinity)
int orc_g1_on_curve(const u64* pts, size_t n) {
    ensure_init();
    Fq b = Fq::from_u64(3);
    for (size_t i = 0; i < n; ++i) {
        Aff<Fq> a = load_affine<Fq>(pts + 8 * i);
        if (a.inf) continue;
        if (a.y.sqr() != a.x.sqr() * a.x + b) return 0;
    }
    return 1;
}
int orc_g2_on_curve(const u64* pts, size_t n) {
    ensure_init();
    Fq2 xi = {Fq::from_u64(9), Fq::from_u64(1)};
    Fq2 three = {Fq::from_u64(3), Fq::zero()};
    Fq2 b = three * xi.inv();
    for (size_t i = 0; i < n; ++i) {
        Aff<Fq2> a = load_affine<Fq2>(pts + 16 * i);
        if (a.inf) continue;
        if (a.y.sqr() != a.x.sqr() * a.x + b) return 0;
    }
    return 1;
}

// in-place NTT: data n x 4 limbs (Montgomery). inverse: 0/1. coset: 0/1 (offset = generator 5).
int orc_ntt(u64* data, unsigned log_n, int inverse, int coset, int nthreads) {
    ensure_init();
    if (log_n > 28) return 2;
    ntt_full(reinterpret_cast<Fr*>(data), log_n, inverse != 0, coset != 0, resolve_threads(nthreads));
    return 0;
}

void orc_bitrev(u64* data, unsigned log_n) { ensure_init(); bitrev_permute(reinterpret_cast<Fr*>(data), log_n); }

// `batch` contiguous transforms of 2^log_t elements (in place), then output k of transform b times base^e with
// e = (b + b0)(alpha k + beta) + gamma k and base = w_{2^log_base}, inverted for an inverse transform unless `shift`: the
// semantics of b200zk_ntt_fr_batched_post_dev.  e is reduced modulo the order of base, so any e gives the exact value.
int orc_ntt_batched_post(u64* data, unsigned log_t, size_t batch, int inverse, unsigned log_base, int shift, u64 b0, u64 alpha,
                         u64 beta, u64 gamma, int nthreads) {
    ensure_init();
    if (log_t > 28 || log_base > 28) return 2;
    nthreads = resolve_threads(nthreads);
    const size_t t = (size_t)1 << log_t;
    Fr* a = reinterpret_cast<Fr*>(data);
    Fr base = fr_root_of_unity(log_base);
    if (inverse && !shift) base = base.inv();
    const unsigned __int128 mask = ((unsigned __int128)1 << log_base) - 1;
#pragma omp parallel for num_threads(nthreads) schedule(dynamic, 1)
    for (long long b = 0; b < (long long)batch; ++b) {
        ntt_full(a + b * t, log_t, inverse != 0, false, 1);
        for (size_t k = 0; k < t; ++k) {
            // wraps modulo 2^128, a multiple of the order 2^log_base
            const unsigned __int128 e = ((unsigned __int128)(u64)b + b0) * ((unsigned __int128)alpha * k + beta) + (unsigned __int128)gamma * k;
            a[b * t + k] = a[b * t + k] * fr_pow_u64(base, (u64)(e & mask));
        }
    }
    return 0;
}

// CSR mat-vec over Fr: out[r] = sum_k val[k] * x[idx[k]], k in [ptr[r], ptr[r+1]) -- the per-row evaluation of qap.rs:60-67
// (`evaluate_constraint`), with the conventions of b200zk.h (u32 row pointers and column indices, Montgomery values).
void orc_fr_spmv(const uint32_t* ptr, const uint32_t* idx, const u64* val, const u64* x, size_t n_rows, u64* out,
                 int nthreads) {
    ensure_init();
    const Fr* v = reinterpret_cast<const Fr*>(val);
    const Fr* xs = reinterpret_cast<const Fr*>(x);
    Fr* o = reinterpret_cast<Fr*>(out);
#pragma omp parallel for num_threads(resolve_threads(nthreads)) schedule(dynamic, 4096)
    for (long long r = 0; r < (long long)n_rows; ++r) {
        Fr acc = Fr::zero();
        for (uint32_t k = ptr[r]; k < ptr[r + 1]; ++k) acc = acc + v[k] * xs[idx[k]];
        o[r] = acc;
    }
}

int orc_h_circom(const u64* a, const u64* b, const u64* c, unsigned log_m, u64* h_out, int nthreads) {
    ensure_init();
    h_circom(reinterpret_cast<const Fr*>(a), reinterpret_cast<const Fr*>(b), reinterpret_cast<const Fr*>(c), log_m,
             reinterpret_cast<Fr*>(h_out), resolve_threads(nthreads));
    return 0;
}

// Groth16 prove (formulas: see oracle/bn254.py::groth16_prove).  All points affine Montgomery limbs.
//   a_query, b_g1_query, b_g2_query: n_vars points; l_query: n_vars - n_inputs; h_query: m
//   z: n_vars scalars (z[0] = 1); h: m scalars; r, s: 4 limbs Montgomery
//   vk_pts: alpha_g1(8) beta_g1(8) delta_g1(8) beta_g2(16) delta_g2(16)  = 56 limbs
//   mirror_bg1: also compute MSM(b_g1_query[1..], z[1..]) when r == 0, as groth16/src/prove.rs:123 does
int orc_groth16_prove(const u64* a_query, const u64* b_g1_query, const u64* b_g2_query, const u64* l_query,
                      const u64* h_query, size_t n_vars, size_t n_inputs, size_t m, const u64* vk_pts,
                      const u64* z, const u64* h, const u64* r, const u64* s, int mirror_bg1,
                      uint8_t proof_out[128], int nthreads) {
    ensure_init();
    nthreads = resolve_threads(nthreads);
    Aff<Fq> alpha = load_affine<Fq>(vk_pts), beta1 = load_affine<Fq>(vk_pts + 8), delta1 = load_affine<Fq>(vk_pts + 16);
    Aff<Fq2> beta2 = load_affine<Fq2>(vk_pts + 24), delta2 = load_affine<Fq2>(vk_pts + 40);
    Fr rr, ss; memcpy(rr.l, r, 32); memcpy(ss.l, s, 32);

    Jac<Fq> A = msm_pippenger<Fq>(a_query + 8, z + 4, n_vars - 1, nthreads);
    A = jac_add_mixed(A, load_affine<Fq>(a_query));
    A = jac_add_mixed(A, alpha);
    A = jac_add(A, jac_mul_fr(aff_to_jac(delta1), r));

    Jac<Fq2> B = msm_pippenger<Fq2>(b_g2_query + 16, z + 4, n_vars - 1, nthreads);
    B = jac_add_mixed(B, load_affine<Fq2>(b_g2_query));
    B = jac_add_mixed(B, beta2);
    B = jac_add(B, jac_mul_fr(aff_to_jac(delta2), s));

    Jac<Fq> C = msm_pippenger<Fq>(l_query, z + 4 * n_inputs, n_vars - n_inputs, nthreads);
    C = jac_add(C, msm_pippenger<Fq>(h_query, h, m, nthreads));
    C = jac_add(C, jac_mul_fr(A, s));
    if (!rr.is_zero() || mirror_bg1) {
        Jac<Fq> B1 = msm_pippenger<Fq>(b_g1_query + 8, z + 4, n_vars - 1, nthreads);
        B1 = jac_add_mixed(B1, load_affine<Fq>(b_g1_query));
        B1 = jac_add_mixed(B1, beta1);
        B1 = jac_add(B1, jac_mul_fr(aff_to_jac(delta1), s));
        C = jac_add(C, jac_mul_fr(B1, r));
        Fr rs = rr * ss;
        Jac<Fq> t = jac_mul_fr(aff_to_jac(delta1), rs.l);
        t.Y = t.Y.neg();
        C = jac_add(C, t);
    }
    compress_g1(jac_to_affine(A), proof_out);
    compress_g2(jac_to_affine(B), proof_out + 32);
    compress_g1(jac_to_affine(C), proof_out + 96);
    return 0;
}

}  // extern "C"
