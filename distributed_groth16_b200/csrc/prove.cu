// prove.cu -- Groth16 proof assembly on the device.
//
// Replaces `prove::{A,B,C}::compute` (/root/reference/groth16/src/prove.rs:21-46,62-85,106-136) plus the
// final assembly of groth16/examples/sha256.rs:208-212,240-244 (== mpc-api/src/main.rs:600-616) and the
// `Proof::serialize_with_mode(Compress::Yes)` of zk-cli/src/main.rs:130-136.  With the PSS layer gone
// (single box, no secret sharing) the formulas are the single-node ones of the zkHubHQ ark-groth16 fork
// (SURVEY 3.2):
//   A  = alpha_g1 + a_query[0] + r*delta_g1 + MSM(a_query[1..], z[1..])
//   B  = beta_g2  + b_g2_query[0] + s*delta_g2 + MSM_G2(b_g2_query[1..], z[1..])
//   B1 = beta_g1  + b_g1_query[0] + s*delta_g1 + MSM(b_g1_query[1..], z[1..])      (only enters C times r)
//   C  = MSM(l_query, z[n_inputs..]) + MSM(h_query, h) + s*A + r*B1 - r*s*delta_g1
#include "common.cuh"

namespace b200zk {

__device__ bool fq_is_neg(const Fq& y) {       // arkworks: y > -y  (canonical integers)
    Fq a = Fq::from_mont(y), b = Fq::from_mont(Fq::neg(y));
    for (int i = 7; i >= 0; --i) {
        if (a.l[i] > b.l[i]) return true;
        if (a.l[i] < b.l[i]) return false;
    }
    return false;
}

__device__ void compress_g1(const xyzz_t<Fq>& p, uint8_t* out) {
    for (int i = 0; i < 32; ++i) out[i] = 0;
    if (p.is_inf()) { out[31] = 0x40; return; }
    affine_t<Fq> a = xyzz_t<Fq>::to_affine(p);
    Fq x = Fq::from_mont(a.x);
    for (int i = 0; i < 32; ++i) out[i] = (uint8_t)(x.l[i >> 2] >> (8 * (i & 3)));
    if (fq_is_neg(a.y)) out[31] |= 0x80;
}

__device__ void compress_g2(const xyzz_t<Fq2>& p, uint8_t* out) {
    for (int i = 0; i < 64; ++i) out[i] = 0;
    if (p.is_inf()) { out[63] = 0x40; return; }
    affine_t<Fq2> a = xyzz_t<Fq2>::to_affine(p);
    Fq x0 = Fq::from_mont(a.x.c0), x1 = Fq::from_mont(a.x.c1);
    for (int i = 0; i < 32; ++i) {
        out[i] = (uint8_t)(x0.l[i >> 2] >> (8 * (i & 3)));
        out[32 + i] = (uint8_t)(x1.l[i >> 2] >> (8 * (i & 3)));
    }
    // Fq2 ordering: c1 first, then c0
    bool neg = a.y.c1.is_zero() ? fq_is_neg(a.y.c0) : fq_is_neg(a.y.c1);
    if (neg) out[63] |= 0x80;
}

struct FinalizeArgs {
    const void *msm_a, *msm_b2, *msm_l, *msm_h, *msm_b1;   // XYZZ partials (msm_b1 may be null)
    const void *a0, *b1_0, *b2_0;                            // query[0] points (affine)
    const void* vk;                                          // alpha_g1 beta_g1 delta_g1 | beta_g2 delta_g2
    const Fr* rs;                                            // r, s (Montgomery)
    uint8_t* out;
    int add_zero_terms;                                      // 0: the MSMs already covered index 0 (z[0] = 1)
};

// Three warps, one active lane each: warp 0 -> A, warp 1 -> B (G2), warp 2 -> C (recomputes the A it needs for s * A).
// The three normalisations (one field inversion each) used to run back to back at the very end of the proof.
__global__ void __launch_bounds__(96) k_prove_finalize(FinalizeArgs f) {
    if ((threadIdx.x & 31) != 0 || blockIdx.x != 0) return;
    const int role = threadIdx.x >> 5;
    const char* vk = reinterpret_cast<const char*>(f.vk);
    Fr r = Fr::from_mont(f.rs[0]), s = Fr::from_mont(f.rs[1]);
    bool r_zero = r.is_zero(), s_zero = s.is_zero();

    if (role == 1) {
        affine_t<Fq2> beta2 = ld16<affine_t<Fq2>>(vk + 192), delta2 = ld16<affine_t<Fq2>>(vk + 320);
        xyzz_t<Fq2> Bp = ld16<xyzz_t<Fq2>>(f.msm_b2);
        if (f.add_zero_terms) xyzz_t<Fq2>::madd(Bp, ld16<affine_t<Fq2>>(f.b2_0), false);
        xyzz_t<Fq2>::madd(Bp, beta2, false);
        if (!s_zero) Bp = xyzz_t<Fq2>::add(Bp, xyzz_t<Fq2>::mul_scalar(xyzz_t<Fq2>::from_affine(delta2), s.l));
        compress_g2(Bp, f.out + 32);
        return;
    }
    affine_t<Fq> alpha = ld16<affine_t<Fq>>(vk), beta1 = ld16<affine_t<Fq>>(vk + 64), delta1 = ld16<affine_t<Fq>>(vk + 128);
    xyzz_t<Fq> d1 = xyzz_t<Fq>::from_affine(delta1);
    xyzz_t<Fq> A = xyzz_t<Fq>::identity();
    if (role == 0 || !s_zero) {
        A = ld16<xyzz_t<Fq>>(f.msm_a);
        if (f.add_zero_terms) xyzz_t<Fq>::madd(A, ld16<affine_t<Fq>>(f.a0), false);
        xyzz_t<Fq>::madd(A, alpha, false);
        if (!r_zero) A = xyzz_t<Fq>::add(A, xyzz_t<Fq>::mul_scalar(d1, r.l));
    }
    if (role == 0) {
        compress_g1(A, f.out);
        return;
    }
    Fr rs = Fr::from_mont(Fr::mul(f.rs[0], f.rs[1]));
    xyzz_t<Fq> C = xyzz_t<Fq>::add(ld16<xyzz_t<Fq>>(f.msm_l), ld16<xyzz_t<Fq>>(f.msm_h));
    if (!s_zero) C = xyzz_t<Fq>::add(C, xyzz_t<Fq>::mul_scalar(A, s.l));
    if (!r_zero) {
        xyzz_t<Fq> B1 = ld16<xyzz_t<Fq>>(f.msm_b1);
        if (f.add_zero_terms) xyzz_t<Fq>::madd(B1, ld16<affine_t<Fq>>(f.b1_0), false);
        xyzz_t<Fq>::madd(B1, beta1, false);
        if (!s_zero) B1 = xyzz_t<Fq>::add(B1, xyzz_t<Fq>::mul_scalar(d1, s.l));
        C = xyzz_t<Fq>::add(C, xyzz_t<Fq>::mul_scalar(B1, r.l));
        C = xyzz_t<Fq>::add(C, xyzz_t<Fq>::neg(xyzz_t<Fq>::mul_scalar(d1, rs.l)));
    }
    compress_g1(C, f.out + 96);
}

static void free_tables(void* tab[5], unsigned tab_c[5], size_t* bytes) {
    for (int k = 0; k < 5; ++k) {
        if (tab[k]) cudaFree(tab[k]);
        tab[k] = nullptr;
        tab_c[k] = 0;
    }
    *bytes = 0;
}

void pk_free_tables(b200zk_pk* pk) { free_tables(pk->tab, pk->tab_c, &pk->tab_bytes); }

bool pk_tables_enabled() {
    const char* env = getenv("B200ZK_PK_TABLES");
    return !(env && env[0] == '0');
}

int pk_tables_build(b200zk_ctx* ctx, Slot& sl, const void* const src[5], const size_t cnt[5], unsigned c_req, void* tab[5],
                    unsigned tab_c[5], size_t* bytes) {
    for (int k = 0; k < 5; ++k) { tab[k] = nullptr; tab_c[k] = 0; }
    *bytes = 0;
    // budget: B200ZK_PK_TABLE_MAX_GB, else 60% of the HBM that is free right now (2^24 constraints: 84 GB of tables)
    double max_gb = 48.0;
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess) max_gb = 0.6 * (double)free_b / 1073741824.0;
    if (const char* env = getenv("B200ZK_PK_TABLE_MAX_GB")) max_gb = atof(env);
    unsigned cs[5];
    size_t size[5], total = 0;
    for (int k = 0; k < 5; ++k) {
        cs[k] = c_req ? c_req : msm_table_auto_window(cnt[k]);
        const uint64_t entries = (uint64_t)msm_table_windows(cs[k]) * cnt[k];
        if (entries >= (1ull << 31)) return B200ZK_OK;                    // generic path keeps working
        size[k] = (size_t)entries * (k == 2 ? 128 : 64);
        total += size[k];
    }
    if ((double)total > max_gb * 1073741824.0) return B200ZK_OK;
    for (int k = 0; k < 5; ++k) {
        if (cnt[k] < 64) continue;                   // tiny query: nothing to gain
        if (cudaMalloc(&tab[k], size[k]) != cudaSuccess) {
            cudaGetLastError();
            tab[k] = nullptr;
            free_tables(tab, tab_c, bytes);
            return B200ZK_OK;
        }
        const int rc = msm_table_build_dev(ctx, sl, k == 2, src[k], cnt[k], cs[k], tab[k]);
        if (rc) { free_tables(tab, tab_c, bytes); return rc; }
        tab_c[k] = cs[k];
        *bytes += size[k];
    }
    return B200ZK_OK;
}

int query_msm(b200zk_ctx* ctx, Slot& sl, int k, const void* query, void* const tab[5], const unsigned tab_c[5], const Fr* scalars,
              size_t n, void* out, unsigned seg) {
    if (tab_c[k]) return msm_table_dev(ctx, sl, k == 2, tab[k], scalars, n, tab_c[k], out, seg);
    return k == 2 ? msm_g2_dev(ctx, sl, query, scalars, n, out, seg) : msm_g1_dev(ctx, sl, query, scalars, n, out, seg);
}

// c = 0: msm_table_auto_window(n) per query (B200ZK_PK_TABLE_WINDOW overrides)
int pk_precompute_dev(b200zk_ctx* ctx, b200zk_pk* pk, unsigned c_req) {
    pk_free_tables(pk);
    Slot& sl = ctx->slots[0];
    const size_t n1 = pk->n_vars - 1;
    const void* src[5] = {(const char*)pk->a_query + 64, (const char*)pk->b_g1_query + 64, (const char*)pk->b_g2_query + 128,
                          pk->l_query, pk->h_query};
    const size_t cnt[5] = {n1, n1, n1, pk->n_vars - pk->n_inputs, pk->m};
    if (const char* env = getenv("B200ZK_PK_TABLE_WINDOW")) { int v = atoi(env); if (v >= 2 && v <= 24) c_req = (unsigned)v; }
    B2_TRY(pk_tables_build(ctx, sl, src, cnt, c_req, pk->tab, pk->tab_c, &pk->tab_bytes));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(sl.stream));
    return B200ZK_OK;
}

// Slot::small of prove_dev and assemble_dev: r, s (Montgomery) at SMALL_RS, uploaded by the caller; the proof at SMALL_PROOF
static const size_t SMALL_RS = 768, SMALL_PROOF = 832;

// k_prove_finalize over the five MSM partials (msm_b1 may be null) and the key's query[0] points and vk on sl's stream, then
// the 128 proof bytes to the host
static int finalize_dev(b200zk_ctx* ctx, Slot& sl, const b200zk_pk* pk, const void* msm_a, const void* msm_b2, const void* msm_l,
                        const void* msm_h, const void* msm_b1, int add_zero_terms, uint8_t proof_out[128]) {
    char* sm = reinterpret_cast<char*>(sl.small.p);
    FinalizeArgs f;
    f.msm_a = msm_a; f.msm_b2 = msm_b2; f.msm_l = msm_l; f.msm_h = msm_h; f.msm_b1 = msm_b1;
    f.a0 = pk->a_query; f.b1_0 = pk->b_g1_query; f.b2_0 = pk->b_g2_query;
    f.vk = pk->vk;
    f.rs = reinterpret_cast<const Fr*>(sm + SMALL_RS);
    f.out = reinterpret_cast<uint8_t*>(sm + SMALL_PROOF);
    f.add_zero_terms = add_zero_terms;
    B2_TRY(launch(ctx, sl.stream, "prove_finalize", k_prove_finalize, 1, 96, 0, f));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(proof_out, sm + SMALL_PROOF, 128, cudaMemcpyDeviceToHost, sl.stream));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(sl.stream));
    return B200ZK_OK;
}

int prove_dev(b200zk_ctx* ctx, const b200zk_pk* pk, const Fr* d_z, const Fr* d_a, const Fr* d_b, const Fr* d_c,
              const uint64_t r[4], const uint64_t s[4], int mirror_bg1, uint8_t proof_out[128]) {
    Slot& s0 = ctx->slots[0];
    Slot& s1 = ctx->slots[1];
    Slot& s2 = ctx->slots[2];
    std::lock_guard<std::mutex> g1(s1.mu);
    std::lock_guard<std::mutex> g2(s2.mu);
    cudaStream_t st = s0.stream;
    const size_t n1 = pk->n_vars - 1, n_aux = pk->n_vars - pk->n_inputs, m = pk->m;
    unsigned log_m = ceil_log2(m);
    if (((size_t)1 << log_m) != m) return set_error(ctx, B200ZK_ERR_DOMAIN, "h_query length must be a power of two");
    bool r_nonzero = (r[0] | r[1] | r[2] | r[3]) != 0;
    bool need_b1 = r_nonzero || mirror_bg1;

    // small device block: 5 partials (3 G1 + 1 G2 + 1 G1) + r,s + 128-byte proof, then the h vector
    const size_t o_a = 0, o_l = 128, o_h = 256, o_b1 = 384, o_b2 = 512, o_hvec = 1024;
    B2_CUDA_OK(ctx, s0.small.reserve(o_hvec + m * sizeof(Fr)));
    char* sm = reinterpret_cast<char*>(s0.small.p);
    Fr* d_h = reinterpret_cast<Fr*>(sm + o_hvec);
    uint64_t rs_host[8];
    memcpy(rs_host, r, 32); memcpy(rs_host + 4, s, 32);
    B2_CUDA_OK(ctx, cudaMemcpyAsync(sm + SMALL_RS, rs_host, 64, cudaMemcpyHostToDevice, st));

    // inputs (z, a, b, c) were produced on slot 0's stream: the other slots wait for them
    cudaEvent_t ev_in, ev1, ev2;
    B2_CUDA_OK(ctx, cudaEventCreateWithFlags(&ev_in, cudaEventDisableTiming));
    B2_CUDA_OK(ctx, cudaEventCreateWithFlags(&ev1, cudaEventDisableTiming));
    B2_CUDA_OK(ctx, cudaEventCreateWithFlags(&ev2, cudaEventDisableTiming));
    B2_CUDA_OK(ctx, cudaEventRecord(ev_in, st));
    B2_CUDA_OK(ctx, cudaStreamWaitEvent(s1.stream, ev_in, 0));
    B2_CUDA_OK(ctx, cudaStreamWaitEvent(s2.stream, ev_in, 0));

    const char* aq = reinterpret_cast<const char*>(pk->a_query);
    const char* b1q = reinterpret_cast<const char*>(pk->b_g1_query);
    const char* b2q = reinterpret_cast<const char*>(pk->b_g2_query);
    // Query k runs over its fixed-base table when pk_precompute_dev built one, else as the generic MSM on the query.
    // Default schedule ("slots"): the five MSMs are spread over the three stream slots, as the reference runs C's
    // three d_msm on mux streams 0/1/2 (prove.rs:119-125): slot 1 = the G2 MSM (issued first: longest bucket kernel and
    // longest latency-bound tail), slot 2 = MSM(a_query), MSM(l_query), (MSM(b_g1_query)), slot 0 = h pipeline then
    // MSM(h_query, h).  The tails of one MSM then overlap the bucket kernels of another.
    // One stream pair per MSM with bucket kernels at the lowest priority and the h pipeline at the highest was measured
    // and lost at 2^20: it removes the idle stretches of this schedule, but the proof is bound by total multiplier work
    // and the reductions then compete with the bucket kernels (tools/prove_timeline.py).
    const unsigned seg = 32;           // bucket reduction in 32-bucket segments: 21% fewer group operations than 16, and
                                       // its longer dependency chains are hidden by the concurrent MSMs
    int rc = query_msm(ctx, s1, 2, b2q + 128, pk->tab, pk->tab_c, d_z + 1, n1, sm + o_b2, seg);
    if (!rc) rc = query_msm(ctx, s2, 0, aq + 64, pk->tab, pk->tab_c, d_z + 1, n1, sm + o_a, seg);
    if (!rc) rc = query_msm(ctx, s2, 3, pk->l_query, pk->tab, pk->tab_c, d_z + pk->n_inputs, n_aux, sm + o_l, seg);
    if (!rc && need_b1) rc = query_msm(ctx, s2, 1, b1q + 64, pk->tab, pk->tab_c, d_z + 1, n1, sm + o_b1, seg);
    if (!rc) rc = h_circom_dev(ctx, s0, d_a, d_b, d_c, log_m, d_h);
    if (!rc) rc = query_msm(ctx, s0, 4, pk->h_query, pk->tab, pk->tab_c, d_h, m, sm + o_h, seg);
    cudaEventRecord(ev1, s1.stream);
    cudaEventRecord(ev2, s2.stream);
    cudaStreamWaitEvent(st, ev1, 0);
    cudaStreamWaitEvent(st, ev2, 0);
    if (!rc) rc = finalize_dev(ctx, s0, pk, sm + o_a, sm + o_b2, sm + o_l, sm + o_h, need_b1 ? sm + o_b1 : nullptr, 1, proof_out);
    if (rc) cudaStreamSynchronize(st);
    cudaEventDestroy(ev_in); cudaEventDestroy(ev1); cudaEventDestroy(ev2);
    return rc;
}

// Final assembly from externally combined MSM results (multi-GPU prove: every rank contributes partial sums,
// parallel.sharded_prove all-gathers and adds them).  include_zero_terms = 0 when the sharded MSMs ran over
// index 0 as well (z[0] = 1 makes a_query[0] * z[0] the same term the driver adds, sha256.rs:208-212).
int assemble_dev(b200zk_ctx* ctx, Slot& sl, const b200zk_pk* pk, const void* msm_a, const void* msm_b2, const void* msm_l,
                 const void* msm_h, const void* msm_b1, const uint64_t r[4], const uint64_t s[4], int include_zero_terms,
                 uint8_t proof_out[128]) {
    bool r_nonzero = (r[0] | r[1] | r[2] | r[3]) != 0;
    if (r_nonzero && !msm_b1) return set_error(ctx, B200ZK_ERR_ARG, "r != 0 needs the b_g1_query MSM");
    B2_CUDA_OK(ctx, sl.small.reserve(1024));
    uint64_t rs_host[8];
    memcpy(rs_host, r, 32); memcpy(rs_host + 4, s, 32);
    B2_CUDA_OK(ctx, cudaMemcpyAsync(reinterpret_cast<char*>(sl.small.p) + SMALL_RS, rs_host, 64, cudaMemcpyHostToDevice, sl.stream));
    return finalize_dev(ctx, sl, pk, msm_a, msm_b2, msm_l, msm_h, msm_b1, include_zero_terms, proof_out);
}

}  // namespace b200zk
