// ntt.cu -- radix-2 Cooley-Tukey NTT / iNTT over BN254 Fr as Stockham passes through shared memory.
//
// Replaces `d_fft` / `d_ifft` (/root/reference/dist-primitives/src/dfft/mod.rs:17-95: fft1 butterflies
// :122-135, king-side fft2 :161-175, size_inv scaling :78) whose contract, once the protocol's own
// bit-reverse/stride packing and `rotate_right(1)` are accounted for, is the natural-order
// `Radix2EvaluationDomain::{fft,ifft}` (asserted at dfft/mod.rs:304,373,384,458), and the
// h-polynomial pipeline `ext_wit::h` (groth16/src/ext_wit.rs:16-101) ==
// `CircomReduction::witness_map_from_matrices` (ark-circom/src/circom/qap.rs:64-89).
//
// Decomposition N = R_1 R_2 .. R_p (R_s = 2^k, k <= MAX_LOG_R).  Pass s, with L = R_1..R_{s-1} and
// M = N / (L R_s), views its input as T_s[j][n_s][n''] (j < L, n_s < R_s, n'' < M), performs the R_s-point
// DIT NTT along n_s in shared memory (root w_N^(N/R_s)), multiplies output k_s by w_N^(L n'' k_s) and
// writes T_{s+1}[j + L k_s][n''].  After the last pass the array is X in natural order, so no separate
// bit-reversal pass over HBM is needed (the reference's `fft_in_place_rearrange`, dfft/mod.rs:258-271,
// is folded into the shared-memory placement).  A block owns G consecutive columns, so every global
// access is a run of G x 32 B.
#include "common.cuh"

namespace b200zk {

static const unsigned MAX_LOG_R = 8;
static const unsigned LOG_G = 2;

struct PowTab {
    const Fr* lo;
    const Fr* hi;
    uint32_t lo_bits;
};

struct NttPlan {
    unsigned log_n = 0;
    bool inverse = false;
    unsigned npass = 0;
    unsigned logR[8];
    Fr* twR[8];          // per pass: w_R^i, i < R/2
    Fr* consts = nullptr;  // [0] w_N (direction applied) [1] n^-1 [2] coset generator (g or g^-1) [3] w_2N (forward)
    PowTab tw;           // powers of consts[0]
    PowTab tw_pass[8];   // middle passes: single-level table of w_N^(L i), i < N/L (one product less per element)
    bool has_tw_pass[8];
    PowTab coset;        // powers of consts[2]   (lazy)
    PowTab shift;        // powers of consts[3]   (lazy; used by h)
    bool scale_folded = false;   // inverse plans: tw_pass[0] carries the 1/N of the inverse transform
    std::vector<void*> allocs;
};

__device__ __forceinline__ Fr powtab_get(const PowTab& t, uint64_t e) {
    Fr lo = ld16(t.lo + (e & ((1ull << t.lo_bits) - 1)));
    uint64_t hi_i = e >> t.lo_bits;
    if (hi_i == 0) return lo;
    return Fr::mul(lo, ld16(t.hi + hi_i));
}

// consts[0] = w_N (or its inverse), [1] = N^-1, [2] = g (or g^-1), [3] = w_2N (forward; one if log_n = 28)
__global__ void k_plan_consts(unsigned log_n, int inverse, Fr* consts) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    Fr g;
    for (int i = 0; i < 8; ++i) g.l[i] = inverse ? FrParams::gen_inv(i) : FrParams::gen(i);
    consts[0] = fr_root_of_unity(log_n, inverse);
    Fr two = Fr::add(Fr::one(), Fr::one());
    Fr n = Fr::one();
    for (unsigned k = 0; k < log_n; ++k) n = Fr::mul(n, two);
    consts[1] = Fr::inv(n);
    consts[2] = g;
    consts[3] = log_n < 28 ? fr_root_of_unity(log_n + 1, false) : Fr::one();
}

// out[i] = base^(i << shift) (* scale, if given)
__global__ void k_build_pow(const Fr* base_ptr, Fr* out, uint32_t count, uint32_t shift, const Fr* scale = nullptr) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    Fr v = Fr::pow_u64(*base_ptr, (uint64_t)i << shift);
    if (scale) v = Fr::mul(v, *scale);
    st16(out + i, v);
}

struct PassParams {
    const Fr* in;
    Fr* out;
    uint32_t log_n, logL, logR, logM, logG;
    uint32_t tw_shift;           // exponent of the inter-pass twiddle = (n'' k_s) << tw_shift
    const Fr* twR;
    PowTab tw;
    PowTab pre;
    PowTab post;
    const Fr* post_const;
    int apply_tw, apply_pre, apply_post, apply_post_const;
    // post exponent = (batch + post_b0) * (post_alpha * k + post_beta) + post_gamma * k   (k = output index);
    // the single-GPU transforms use (alpha, beta, gamma) = (0, 0, 1); the four-step column twiddle
    // w_N^(col * k1) uses (1, 0, 0) and the distributed coefficient shift w_2m^(k1 + N1 k2) uses (0, 1, N1).
    uint64_t post_b0, post_alpha, post_beta, post_gamma;
    size_t batch_stride;
    // fused four-step exchange: the last pass stores output k of batch element (= matrix column) c straight into
    // the row-major receive buffer of the rank that owns row k, over NVLink peer mappings (no pack / all-to-all /
    // unpack passes): dst = peer_out[k >> log_rl] + ((k & (rl-1)) << log_cols_total) + col0 + c
    Fr* peer_out[8];
    uint32_t p2p, log_rl, log_cols_total;
    uint64_t col0;
    // last pass only: the G columns of a block are G consecutive BATCH elements (same sub-problem j = blockIdx.x) instead
    // of G consecutive j of one batch element, so that the remote stores of the fused exchange are runs of G x 32 B
    uint32_t batch_tile;
};

static const unsigned NTT_MINBLOCKS = 2;   // 64 registers: four 256-thread tiles per SM (76 registers uncapped = three)
__global__ void __launch_bounds__(512, NTT_MINBLOCKS) k_ntt_pass(PassParams p) {
    extern __shared__ uint4 smem[];
    const uint32_t R = 1u << p.logR, G = 1u << p.logG;
    const uint32_t RG = R << p.logG;
    uint4* s_lo = smem;                 // [G][R]
    uint4* s_hi = smem + RG;
    uint4* s_tw = smem + 2 * RG;        // [R/2][2]
    const uint32_t tid = threadIdx.x, nt = blockDim.x;
    const uint64_t q0 = p.batch_tile ? (uint64_t)blockIdx.x : ((uint64_t)blockIdx.x << p.logG);
    const uint32_t b0 = p.batch_tile ? (blockIdx.y << p.logG) : blockIdx.y;
    const uint64_t Mmask = (1ull << p.logM) - 1;

    for (uint32_t i = tid; i < R / 2; i += nt) {
        const uint4* t = reinterpret_cast<const uint4*>(p.twR + i);
        s_tw[2 * i] = t[0];
        s_tw[2 * i + 1] = t[1];
    }
    for (uint32_t idx = tid; idx < RG; idx += nt) {
        uint32_t c = idx & (G - 1), ns = idx >> p.logG;
        uint64_t q = p.batch_tile ? q0 : q0 + c, j = q >> p.logM, n2 = q & Mmask;
        uint64_t addr = (j << (p.logR + p.logM)) + ((uint64_t)ns << p.logM) + n2;
        const Fr* in = p.in + (size_t)(p.batch_tile ? b0 + c : b0) * p.batch_stride;
        Fr v = ld16(in + addr);
        if (p.apply_pre) v = Fr::mul(v, powtab_get(p.pre, addr));
        uint32_t slot = p.logR ? (__brev(ns) >> (32 - p.logR)) : 0;
        uint32_t e = c * R + slot;
        s_lo[e] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
        s_hi[e] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
    }
    __syncthreads();

    // Butterfly stages, two at a time: a thread loads the four elements {e, e + h, e + 2h, e + 3h} of a radix-4 unit
    // (h = 2^(s-1)), runs stage s on (e, e+h), (e+2h, e+3h) and stage s + 1 on (e, e+2h), (e+h, e+3h) in registers and
    // stores them back: the same 4 twiddle products as two radix-2 stages (a prime field has no free multiplication by i),
    // but one shared-memory round trip and one barrier instead of two, and four independent products in flight per thread.
    // An odd number of stages starts with the single unit-twiddle stage s = 1.
    auto ld_split = [&](uint32_t i) {
        uint4 lo = s_lo[i], hi = s_hi[i];
        Fr v;
        v.l[0] = lo.x; v.l[1] = lo.y; v.l[2] = lo.z; v.l[3] = lo.w; v.l[4] = hi.x; v.l[5] = hi.y; v.l[6] = hi.z; v.l[7] = hi.w;
        return v;
    };
    auto st_split = [&](uint32_t i, const Fr& v) {
        s_lo[i] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
        s_hi[i] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
    };
    auto twd = [&](uint32_t ti) {
        uint4 tl = s_tw[2 * ti], th = s_tw[2 * ti + 1];
        Fr t;
        t.l[0] = tl.x; t.l[1] = tl.y; t.l[2] = tl.z; t.l[3] = tl.w; t.l[4] = th.x; t.l[5] = th.y; t.l[6] = th.z; t.l[7] = th.w;
        return t;
    };
    uint32_t s = 1;
    if (p.logR & 1) {                       // stage 1 alone: (x, y) -> (x + y, x - y)
        const uint32_t nbf = RG >> 1;
        for (uint32_t b = tid; b < nbf; b += nt) {
            const uint32_t c = b >> (p.logR - 1), bb = b & (R / 2 - 1);
            const uint32_t i0 = c * R + (bb << 1), i1 = i0 + 1;
            const Fr u = ld_split(i0), v = ld_split(i1);
            st_split(i0, Fr::add(u, v));
            st_split(i1, Fr::sub(u, v));
        }
        __syncthreads();
        s = 2;
    }
    const uint32_t nq = RG >> 2;            // radix-4 units per tile
    for (; s < p.logR + 1; s += 2) {        // stages s and s + 1 (logR - s + 1 is even here)
        const uint32_t half = 1u << (s - 1);
        for (uint32_t b = tid; b < nq; b += nt) {
            const uint32_t c = b >> (p.logR - 2), bb = b & (R / 4 - 1);
            const uint32_t jj = bb & (half - 1);
            const uint32_t e0 = c * R + (((bb >> (s - 1)) << (s + 1)) | jj);
            Fr x0 = ld_split(e0), x1 = ld_split(e0 + half), x2 = ld_split(e0 + 2 * half), x3 = ld_split(e0 + 3 * half);
            if (s > 1) {                    // stage s twiddle w_R^(jj 2^(logR - s)), the same for both pairs
                const Fr t = twd(jj << (p.logR - s));
                x1 = Fr::mul(x1, t);
                x3 = Fr::mul(x3, t);
            }
            Fr y0 = Fr::add(x0, x1), y1 = Fr::sub(x0, x1), y2 = Fr::add(x2, x3), y3 = Fr::sub(x2, x3);
            // stage s + 1: pairs (y0, y2) at index jj and (y1, y3) at index jj + half of a 2^s-point group
            if (s > 1) y2 = Fr::mul(y2, twd(jj << (p.logR - s - 1)));      // s = 1: jj = 0, unit twiddle
            y3 = Fr::mul(y3, twd((jj + half) << (p.logR - s - 1)));
            st_split(e0, Fr::add(y0, y2));
            st_split(e0 + 2 * half, Fr::sub(y0, y2));
            st_split(e0 + half, Fr::add(y1, y3));
            st_split(e0 + 3 * half, Fr::sub(y1, y3));
        }
        __syncthreads();
    }

    for (uint32_t idx = tid; idx < RG; idx += nt) {
        uint32_t c = idx & (G - 1), ks = idx >> p.logG;
        uint64_t q = p.batch_tile ? q0 : q0 + c, j = q >> p.logM, n2 = q & Mmask;
        const uint32_t bidx = p.batch_tile ? b0 + c : b0;
        Fr* out = p.out + (size_t)bidx * p.batch_stride;
        uint32_t e = c * R + ks;
        uint4 a = s_lo[e], bq = s_hi[e];
        Fr v;
        v.l[0] = a.x; v.l[1] = a.y; v.l[2] = a.z; v.l[3] = a.w; v.l[4] = bq.x; v.l[5] = bq.y; v.l[6] = bq.z; v.l[7] = bq.w;
        if (p.apply_tw) {
            uint64_t ex = (n2 * ks) << p.tw_shift;
            if (ex || p.apply_tw == 2) v = Fr::mul(v, powtab_get(p.tw, ex));
        }
        uint64_t oaddr = ((j + ((uint64_t)ks << p.logL)) << p.logM) + n2;
        if (p.apply_post) {
            uint64_t ex = (bidx + p.post_b0) * (p.post_alpha * oaddr + p.post_beta) + p.post_gamma * oaddr;
            if (ex) v = Fr::mul(v, powtab_get(p.post, ex));
        }
        if (p.apply_post_const) v = Fr::mul(v, ld16(p.post_const));
        if (p.p2p) {
            Fr* dst = p.peer_out[oaddr >> p.log_rl] + ((oaddr & ((1ull << p.log_rl) - 1)) << p.log_cols_total) + p.col0 + bidx;
            st16(dst, v);
        } else {
            st16(out + oaddr, v);
        }
    }
}

__global__ void k_bitrev(const Fr* in, Fr* out, unsigned log_n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ((size_t)1 << log_n)) return;
    size_t j = log_n ? (size_t)(__brevll((unsigned long long)i) >> (64 - log_n)) : 0;
    st16(out + j, ld16(in + i));
}

// h[i] = a[i]*b[i] - c[i]
__global__ void k_h_pointwise(const Fr* a, const Fr* b, const Fr* c, Fr* h, size_t m) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    st16(h + i, Fr::sub(Fr::mul(ld16(a + i), ld16(b + i)), ld16(c + i)));
}

static int build_powtab(b200zk_ctx* ctx, cudaStream_t st, NttPlan* pl, const Fr* base, unsigned log_range, PowTab* out) {
    unsigned lo_bits = (log_range + 1) / 2, hi_bits = log_range - lo_bits;
    Fr *lo = nullptr, *hi = nullptr;
    B2_CUDA_OK(ctx, cudaMalloc(&lo, sizeof(Fr) << lo_bits));
    pl->allocs.push_back(lo);
    B2_CUDA_OK(ctx, cudaMalloc(&hi, sizeof(Fr) << hi_bits));
    pl->allocs.push_back(hi);
    const uint32_t n_lo = 1u << lo_bits, n_hi = 1u << hi_bits;
    B2_TRY(launch(ctx, st, "ntt_build_tables", k_build_pow, (n_lo + 127) / 128, 128, 0, base, lo, n_lo, 0u, nullptr));
    B2_TRY(launch(ctx, st, "ntt_build_tables", k_build_pow, (n_hi + 127) / 128, 128, 0, base, hi, n_hi, lo_bits, nullptr));
    out->lo = lo; out->hi = hi; out->lo_bits = lo_bits;
    return B200ZK_OK;
}

static int get_plan(b200zk_ctx* ctx, cudaStream_t st, unsigned log_n, bool inverse, NttPlan** out) {
    std::lock_guard<std::mutex> g(ctx->plan_mu);
    uint32_t key = (log_n << 1) | (inverse ? 1u : 0u);
    auto it = ctx->plans.find(key);
    if (it != ctx->plans.end()) { *out = it->second; return B200ZK_OK; }
    NttPlan* pl = new NttPlan();
    pl->log_n = log_n; pl->inverse = inverse;
    pl->coset.lo = nullptr; pl->shift.lo = nullptr;
    pl->npass = log_n == 0 ? 0 : (log_n + MAX_LOG_R - 1) / MAX_LOG_R;
    for (unsigned i = 0; i < pl->npass; ++i) {
        pl->logR[i] = log_n / pl->npass + (i < log_n % pl->npass ? 1 : 0);
    }
    B2_CUDA_OK(ctx, cudaMalloc(&pl->consts, 4 * sizeof(Fr)));
    pl->allocs.push_back(pl->consts);
    B2_TRY(launch(ctx, st, "ntt_build_tables", k_plan_consts, 1, 1, 0, log_n, inverse ? 1 : 0, pl->consts));
    for (unsigned i = 0; i < pl->npass; ++i) {
        uint32_t cnt = 1u << (pl->logR[i] - 1);
        B2_CUDA_OK(ctx, cudaMalloc(&pl->twR[i], sizeof(Fr) * cnt));
        pl->allocs.push_back(pl->twR[i]);
        B2_TRY(launch(ctx, st, "ntt_build_tables", k_build_pow, (cnt + 127) / 128, 128, 0, pl->consts, pl->twR[i], cnt,
                      log_n - pl->logR[i], nullptr));
    }
    B2_TRY(build_powtab(ctx, st, pl, pl->consts, log_n, &pl->tw));
    {
        unsigned logL = 0;
        for (unsigned i = 0; i < pl->npass; ++i) {
            pl->has_tw_pass[i] = false;
            unsigned range = log_n - logL;                      // exponents n'' k_s < N / L
            // first boundary (range = log_n): one table of N entries (128 MB at 2^22) read once per transform -- 32 B gathers the
            // otherwise idle HBM serves -- instead of a second product through the two-level table; an inverse plan's table also
            // carries the 1/N every inverse transform ends with.  B200ZK_NTT_BIGTAB = largest log_n that gets one (default 24:
            // 512 MB per direction), 0 = never
            static const unsigned bigtab = getenv("B200ZK_NTT_BIGTAB") ? (unsigned)atoi(getenv("B200ZK_NTT_BIGTAB")) : 24u;
            const bool first_big = i == 0 && pl->npass > 1 && range <= bigtab;
            if ((i > 0 && i + 1 < pl->npass && range <= 16) || first_big) {
                Fr* t = nullptr;
                if (cudaMalloc(&t, sizeof(Fr) << range) != cudaSuccess) {
                    cudaGetLastError();
                    if (!first_big) return set_error(ctx, B200ZK_ERR_OOM, "cudaMalloc failed for an NTT twiddle table");
                    logL += pl->logR[i];                        // no room for the big table: the two-level one serves this boundary
                    continue;
                }
                pl->allocs.push_back(t);
                const uint32_t cnt = 1u << range;
                const bool fold_scale = first_big && inverse;
                B2_TRY(launch(ctx, st, "ntt_build_tables", k_build_pow, (cnt + 127) / 128, 128, 0, pl->consts, t, cnt, logL,
                              fold_scale ? pl->consts + 1 : nullptr));
                if (fold_scale) pl->scale_folded = true;
                pl->tw_pass[i].lo = t; pl->tw_pass[i].hi = t; pl->tw_pass[i].lo_bits = range;
                pl->has_tw_pass[i] = true;
            }
            logL += pl->logR[i];
        }
    }
    // tables are built on `st`; other slots may use the plan later, so finish construction here
    B2_CUDA_OK(ctx, cudaStreamSynchronize(st));
    ctx->plans[key] = pl;
    *out = pl;
    return B200ZK_OK;
}

static int plan_lazy_tab(b200zk_ctx* ctx, cudaStream_t st, NttPlan* pl, int which, PowTab** out) {
    std::lock_guard<std::mutex> g(ctx->plan_mu);
    PowTab* t = which == 2 ? &pl->coset : &pl->shift;
    if (!t->lo) {
        // exponents < N.  One level (one product per element instead of two) up to B200ZK_NTT_BIGTAB, like the first pass boundary
        static const unsigned bigtab = getenv("B200ZK_NTT_BIGTAB") ? (unsigned)atoi(getenv("B200ZK_NTT_BIGTAB")) : 24u;
        Fr* tab = nullptr;
        if (pl->log_n <= bigtab && cudaMalloc(&tab, sizeof(Fr) << pl->log_n) != cudaSuccess) { cudaGetLastError(); tab = nullptr; }
        if (tab) {
            pl->allocs.push_back(tab);
            const uint32_t cnt = 1u << pl->log_n;
            B2_TRY(launch(ctx, st, "ntt_build_tables", k_build_pow, (cnt + 127) / 128, 128, 0, pl->consts + which, tab, cnt, 0u, nullptr));
            t->hi = tab; t->lo_bits = pl->log_n; t->lo = tab;
        } else {
            B2_TRY(build_powtab(ctx, st, pl, pl->consts + which, pl->log_n, t));
        }
        B2_CUDA_OK(ctx, cudaStreamSynchronize(st));
    }
    *out = t;
    return B200ZK_OK;
}

void ntt_free_plans(b200zk_ctx* ctx) {
    for (auto& kv : ctx->plans) {
        for (void* p : kv.second->allocs) cudaFree(p);
        delete kv.second;
    }
    ctx->plans.clear();
}

// Runs all passes.  pre / post may be null.  post_const: device pointer or null.
struct PostExp { uint64_t b0, alpha, beta, gamma; };
static const PostExp POST_PLAIN = {0, 0, 0, 1};
struct P2PStore { Fr* peer[8]; unsigned n_peers, log_rl, log_cols_total; uint64_t col0; };

static int ntt_run(b200zk_ctx* ctx, Slot& sl, NttPlan* pl, const Fr* d_in, Fr* d_out, unsigned batch,
                   const PowTab* pre, const PowTab* post, const Fr* post_const, PostExp pe = POST_PLAIN,
                   const P2PStore* p2p = nullptr) {
    cudaStream_t st = sl.stream;
    const size_t N = (size_t)1 << pl->log_n;
    if (pl->npass == 0) {   // N == 1: X[0] = x[0] (all scale factors are 1)
        if (d_in != d_out) B2_CUDA_OK(ctx, cudaMemcpyAsync(d_out, d_in, sizeof(Fr) * batch, cudaMemcpyDeviceToDevice, st));
        return B200ZK_OK;
    }
    const size_t bytes = sizeof(Fr) * N * batch;
    B2_CUDA_OK(ctx, sl.ws_ntt.reserve(2 * bytes));
    Fr* scratch[2] = {reinterpret_cast<Fr*>(sl.ws_ntt.p), reinterpret_cast<Fr*>(sl.ws_ntt.p) + N * batch};
    const Fr* cur = d_in;
    unsigned logL = 0;
    for (unsigned i = 0; i < pl->npass; ++i) {
        bool last = (i + 1 == pl->npass);
        Fr* dst = last ? d_out : scratch[(i + 1) & 1];
        bool bounce = last && (cur == d_out);     // only when npass == 1 and in-place
        if (bounce) dst = scratch[0];
        PassParams p;
        memset(&p, 0, sizeof(p));
        p.in = cur; p.out = dst;
        p.log_n = pl->log_n; p.logL = logL; p.logR = pl->logR[i];
        p.logM = pl->log_n - logL - pl->logR[i];
        unsigned log_cols = pl->log_n - pl->logR[i];
        p.logG = log_cols < LOG_G ? log_cols : LOG_G;
        p.twR = pl->twR[i];
        p.tw = pl->tw;
        p.tw_shift = logL;
        if (pl->has_tw_pass[i]) { p.tw = pl->tw_pass[i]; p.tw_shift = 0; }
        p.apply_tw = last ? 0 : (i == 0 && pl->scale_folded ? 2 : 1);          // 2: the table entry for exponent 0 is 1/N, not 1
        if (i == 0 && pre) { p.pre = *pre; p.apply_pre = 1; }
        if (last && post) {
            p.post = *post; p.apply_post = 1;
            p.post_b0 = pe.b0; p.post_alpha = pe.alpha; p.post_beta = pe.beta; p.post_gamma = pe.gamma;
        }
        if (last && post_const && !pl->scale_folded) { p.post_const = post_const; p.apply_post_const = 1; }
        p.batch_stride = N;
        if (last && p2p) {
            for (unsigned g = 0; g < 8; ++g) p.peer_out[g] = g < p2p->n_peers ? p2p->peer[g] : nullptr;
            p.p2p = 1; p.log_rl = p2p->log_rl; p.log_cols_total = p2p->log_cols_total; p.col0 = p2p->col0;
        }
        uint32_t RG = 1u << (p.logR + p.logG);
        // threads = tile / tdiv: tdiv / 4 radix-4 units per thread per stage pair.  Measured on an earlier GPU: 4 wins at
        // 2^20, the two tie at 2^22, 8 wins at 2^24 -> 8 from 2^23 up
        const unsigned tdiv = pl->log_n >= 23 ? 8u : 4u;
        uint32_t threads = RG / tdiv < 32 ? 32 : RG / tdiv;
        size_t smem = (size_t)(2 * RG + (1u << p.logR)) * sizeof(uint4);
        dim3 grid((unsigned)(((size_t)1 << log_cols) >> p.logG), batch);
        if (last && p2p && p.logM == 0 && batch >= (1u << LOG_G) && batch % (1u << LOG_G) == 0) {
            p.batch_tile = 1;
            p.logG = LOG_G;
            RG = 1u << (p.logR + p.logG);
            threads = RG / tdiv < 32 ? 32 : RG / tdiv;
            smem = (size_t)(2 * RG + (1u << p.logR)) * sizeof(uint4);
            grid = dim3((unsigned)((size_t)1 << log_cols), batch >> LOG_G);
        }
        B2_TRY(launch(ctx, st, "ntt_pass", k_ntt_pass, grid, threads, smem, p));
        if (bounce) B2_CUDA_OK(ctx, cudaMemcpyAsync(d_out, dst, bytes, cudaMemcpyDeviceToDevice, st));
        cur = dst;
        logL += pl->logR[i];
    }
    return B200ZK_OK;
}

int ntt_dev(b200zk_ctx* ctx, Slot& sl, const Fr* d_in, Fr* d_out, unsigned log_n, bool inverse, bool coset,
            unsigned batch) {
    if (log_n > 28) return set_error(ctx, B200ZK_ERR_DOMAIN, "log_n > 28 exceeds the two-adicity of BN254 Fr");
    NttPlan* pl;
    B2_TRY(get_plan(ctx, sl.stream, log_n, inverse, &pl));
    PowTab* ct = nullptr;
    if (coset && log_n > 0) B2_TRY(plan_lazy_tab(ctx, sl.stream, pl, 2, &ct));
    if (!inverse) return ntt_run(ctx, sl, pl, d_in, d_out, batch, ct, nullptr, nullptr);
    return ntt_run(ctx, sl, pl, d_in, d_out, batch, nullptr, ct, log_n > 0 ? pl->consts + 1 : nullptr);
}

int bitrev_dev(b200zk_ctx* ctx, Slot& sl, const Fr* d_in, Fr* d_out, unsigned log_n) {
    size_t n = (size_t)1 << log_n;
    return launch(ctx, sl.stream, "bitrev", k_bitrev, (unsigned)((n + 255) / 256), 256, 0, d_in, d_out, log_n);
}

// h = (NTT(shift(iNTT a)) * NTT(shift(iNTT b))) - NTT(shift(iNTT c)),  shift: coeff j *= w_2m^j
// d_a, d_b, d_c may be separate buffers; they are staged into one [3][m] batch.
int h_circom_dev(b200zk_ctx* ctx, Slot& sl, const Fr* d_a, const Fr* d_b, const Fr* d_c, unsigned log_m, Fr* d_h) {
    if (log_m + 1 > 28) return set_error(ctx, B200ZK_ERR_DOMAIN, "2m exceeds the 2^28 subgroup (PolynomialDegreeTooLarge)");
    cudaStream_t st = sl.stream;
    const size_t m = (size_t)1 << log_m;
    B2_CUDA_OK(ctx, sl.io_b.reserve(2 * 3 * m * sizeof(Fr)));
    Fr* buf0 = reinterpret_cast<Fr*>(sl.io_b.p);
    Fr* buf1 = buf0 + 3 * m;
    B2_CUDA_OK(ctx, cudaMemcpyAsync(buf0, d_a, m * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(buf0 + m, d_b, m * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(buf0 + 2 * m, d_c, m * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
    NttPlan *inv, *fwd;
    B2_TRY(get_plan(ctx, st, log_m, true, &inv));
    B2_TRY(get_plan(ctx, st, log_m, false, &fwd));
    if (log_m == 0) {
        // m = 1: iNTT and NTT are the identity and the shift multiplies coefficient 0 by 1
        buf1 = buf0;
    } else {
        PowTab* shift;
        B2_TRY(plan_lazy_tab(ctx, st, inv, 3, &shift));
        B2_TRY(ntt_run(ctx, sl, inv, buf0, buf1, 3, nullptr, shift, inv->consts + 1));
        B2_TRY(ntt_run(ctx, sl, fwd, buf1, buf1, 3, nullptr, nullptr, nullptr));
    }
    return launch(ctx, st, "h_pointwise", k_h_pointwise, (unsigned)((m + 255) / 256), 256, 0, buf1, buf1 + m, buf1 + 2 * m, d_h, m);
}

// Batched transform of size 2^log_t over `batch` contiguous vectors with a per-batch post factor
// base^((b + b0)(alpha k + beta) + gamma k), base = w_{2^log_base} (forward root, or its inverse when
// `inverse`); the inverse transform also scales by 2^-log_t.  Building block of the multi-GPU four-step
// NTT and of the distributed h pipeline (dist_primitives/dfft_sharded.py).
int ntt_batched_post_dev(b200zk_ctx* ctx, Slot& sl, const Fr* d_in, Fr* d_out, unsigned log_t, unsigned batch, bool inverse,
                         unsigned log_base, bool base_is_shift, uint64_t b0, uint64_t alpha, uint64_t beta, uint64_t gamma) {
    if (log_t > 28 || log_base > 28 || log_t == 0) return set_error(ctx, B200ZK_ERR_DOMAIN, "bad transform size for batched NTT");
    if (base_is_shift && log_base == 0) return set_error(ctx, B200ZK_ERR_DOMAIN, "the shift table needs log_base >= 1");
    // the post table holds base^e for e < 2^log_base (shift: e < 2^(log_base - 1)); exponents are not reduced, so the largest
    // one, (batch - 1 + b0)(alpha k_max + beta) + gamma k_max with k_max = 2^log_t - 1, must lie below that bound
    {
        typedef unsigned __int128 u128;
        const u128 bound = (u128)1 << (base_is_shift ? log_base - 1 : log_base);
        const u128 k_max = ((u128)1 << log_t) - 1;
        const u128 per_b = (u128)alpha * k_max + beta, b_max = (u128)(batch - 1) + b0;
        if ((b_max && per_b >= bound) || b_max * per_b + (u128)gamma * k_max >= bound)     // no overflow: per_b < 2^28 or b_max = 0
            return set_error(ctx, B200ZK_ERR_ARG, "post-factor exponent (batch - 1 + b0)(alpha k + beta) + gamma k exceeds the table of "
                                                  "base powers");
    }
    NttPlan *pl, *base_plan;
    B2_TRY(get_plan(ctx, sl.stream, log_t, inverse, &pl));
    const PowTab* tab = nullptr;
    if (base_is_shift) {
        // powers of the FORWARD root w_{2^(log_base)} = consts[3] of the (log_base - 1) plan
        B2_TRY(get_plan(ctx, sl.stream, log_base - 1, true, &base_plan));
        PowTab* t;
        B2_TRY(plan_lazy_tab(ctx, sl.stream, base_plan, 3, &t));
        tab = t;
        // the shift table covers exponents < 2^(log_base-1); callers keep (k1 + N1 k2) < m = 2^(log_base-1)
    } else {
        B2_TRY(get_plan(ctx, sl.stream, log_base, inverse, &base_plan));
        tab = &base_plan->tw;
    }
    PostExp pe = {b0, alpha, beta, gamma};
    return ntt_run(ctx, sl, pl, d_in, d_out, batch, nullptr, tab, inverse ? pl->consts + 1 : nullptr, pe);
}

int fourstep_cols_dev(b200zk_ctx* ctx, Slot& sl, const Fr* d_in, Fr* d_out, unsigned log_rows, unsigned log_cols_local,
                      unsigned log_n, uint64_t global_col0, bool inverse) {
    if (log_cols_local > 28) return set_error(ctx, B200ZK_ERR_DOMAIN, "bad four-step geometry");
    return ntt_batched_post_dev(ctx, sl, d_in, d_out, log_rows, 1u << log_cols_local, inverse, log_n, false, global_col0, 1, 0, 0);
}

// Column step of the four-step NTT fused with the exchange: the transformed, twiddled columns are written directly
// into the peers' row-major receive buffers (P2P stores over NVLink) -- the compute kernel IS the all-to-all.
int fourstep_cols_p2p_dev(b200zk_ctx* ctx, Slot& sl, const Fr* d_in, void* const* peer_out, unsigned n_peers, unsigned log_rows,
                          unsigned log_cols_local, unsigned log_n, uint64_t global_col0, bool inverse) {
    if (n_peers == 0 || n_peers > 8 || (n_peers & (n_peers - 1))) return set_error(ctx, B200ZK_ERR_ARG, "peer count must be 1, 2, 4 or 8");
    if (log_rows == 0 || log_rows > 28 || log_n > 28) return set_error(ctx, B200ZK_ERR_DOMAIN, "bad four-step geometry");
    unsigned log_p = ceil_log2(n_peers);
    if (log_rows < log_p) return set_error(ctx, B200ZK_ERR_ARG, "fewer rows than peers");
    if (log_n < log_rows) return set_error(ctx, B200ZK_ERR_ARG, "log_n < log_rows: the transform has fewer elements than one column");
    // the remote stores write columns [global_col0, global_col0 + 2^log_cols_local) of rows 2^(log_n - log_rows) wide
    const uint64_t cols_total = (uint64_t)1 << (log_n - log_rows);
    if (log_cols_local > log_n - log_rows || global_col0 > cols_total - ((uint64_t)1 << log_cols_local))
        return set_error(ctx, B200ZK_ERR_ARG, "columns [global_col0, global_col0 + 2^log_cols_local) run past the receive rows");
    NttPlan *pl, *base_plan;
    B2_TRY(get_plan(ctx, sl.stream, log_rows, inverse, &pl));
    B2_TRY(get_plan(ctx, sl.stream, log_n, inverse, &base_plan));
    P2PStore ps;
    for (unsigned g = 0; g < 8; ++g) ps.peer[g] = g < n_peers ? reinterpret_cast<Fr*>(peer_out[g]) : nullptr;
    ps.n_peers = n_peers;
    ps.log_rl = log_rows - log_p;
    ps.log_cols_total = log_n - log_rows;
    ps.col0 = global_col0;
    PostExp pe = {global_col0, 1, 0, 0};
    // d_out is only used by the earlier passes' scratch chain; the last pass stores remotely
    Fr* dummy_out = reinterpret_cast<Fr*>(peer_out[0]);
    return ntt_run(ctx, sl, pl, d_in, dummy_out, 1u << log_cols_local, nullptr, &base_plan->tw, inverse ? pl->consts + 1 : nullptr, pe, &ps);
}

// out[i] = a[i]*b[i] - c[i]   (ext_wit.rs:88-92 on device-resident vectors)
int mul_sub_dev(b200zk_ctx* ctx, Slot& sl, const Fr* a, const Fr* b, const Fr* c, Fr* out, size_t n) {
    if (n == 0) return B200ZK_OK;
    return launch(ctx, sl.stream, "h_pointwise", k_h_pointwise, (unsigned)((n + 255) / 256), 256, 0, a, b, c, out, n);
}

}  // namespace b200zk
