// common.cuh -- context, error handling, workspace and per-kernel event profiling shared by the
// translation units of libb200zk.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "../../include/b200zk.h"
#include "ec.cuh"

namespace b200zk {

struct ProfEntry {
    const char* name;
    cudaEvent_t start, stop;
};

struct NttPlan;   // ntt.cu

// grow-only device buffer
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

struct Slot {                 // one per MultiplexedStreamID
    cudaStream_t stream = nullptr;
    bool owns_stream = false;
    std::mutex mu;            // same-slot calls are serialised
    DevBuf ws_msm;            // MSM workspace
    DevBuf ws_ntt;            // NTT ping-pong
    DevBuf io_a, io_b;        // staging for host-buffer entry points
    DevBuf small;             // results
    cudaStream_t copy_stream = nullptr;   // second stream for overlapped H2D staging (host-buffer entry points)
    cudaEvent_t copy_done = nullptr;      // host-staged MSM: earlier work on `stream` is done with io_a (the copy stream waits)
    cudaEvent_t rebind = nullptr;         // b200zk_ctx_set_stream: work queued on the old stream, waited on by the new one
    cudaEvent_t stage_ev[32] = {};        // host-staged MSM: arrival of part p's scalars [2 p] / bases [2 p + 1]
};

}  // namespace b200zk

struct b200zk_ctx {
    int device = 0;
    int sm_count = 132;
    b200zk::Slot slots[3];
    std::string last_error;
    std::mutex err_mu;
    // profiling
    bool prof_on = false;
    std::mutex prof_mu;
    std::vector<b200zk::ProfEntry> prof_pending;
    std::map<std::string, std::pair<uint64_t, double>> prof_acc;   // name -> (launches, ms)
    // B200ZK_PROFILE_TIMELINE=1: (name, start, end) in ms since the first profiled launch (scheduling diagnostics)
    cudaEvent_t prof_base = nullptr;
    std::vector<std::tuple<std::string, float, float>> prof_timeline;
    std::atomic<uint64_t> launches{0};     // kernels launched (slots may be driven from different host threads)
    // NTT plans keyed by (log_n << 1 | inverse)
    std::mutex plan_mu;
    std::map<uint32_t, b200zk::NttPlan*> plans;
    void *fb_table_g1 = nullptr, *fb_table_g2 = nullptr;     // fixed-base window tables of the generators (setup.cu)
    // MSM window-group pipeline (msm.cu), one per slot: msm_side[i], a high-priority helper stream that runs the sort phases
    // and the reduction / Horner tail of one window group while the bucket kernel of the next group occupies the SMs;
    // msm_events[i], the event pool of slot i's MSMs (grown on demand, only ever touched under the slot's mutex).
    cudaStream_t msm_side[3] = {nullptr, nullptr, nullptr};
    std::vector<cudaEvent_t> msm_events[3];
};

struct b200zk_pk {
    size_t n_vars = 0, n_inputs = 0, m = 0;
    void *a_query = nullptr, *b_g1_query = nullptr, *b_g2_query = nullptr, *l_query = nullptr, *h_query = nullptr;
    void* vk = nullptr;       // device copy of the 56 vk limbs
    // fixed-base window tables (msm.cu section 7) over a_query[1..], b_g1_query[1..], b_g2_query[1..], l_query, h_query;
    // tab_c[k] == 0: no table, the generic MSM runs on the query itself
    void* tab[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    unsigned tab_c[5] = {0, 0, 0, 0, 0};
    size_t tab_bytes = 0;
};

// A snarkjs Groth16 zkey resident in HBM (zkey.cu): the proving key and A, B in CSR form.  row_ptr holds 2 nc + 1 entries, A's
// row i at entry i and B's row i at entry nc + i, both indexing col / val (val Montgomery), so b200zk_qap_dev runs on
// (row_ptr, col, val) and (row_ptr + nc, col, val).
struct b200zk_zkey {
    b200zk_pk* pk = nullptr;
    size_t n_vars = 0, n_public = 0, domain_size = 0, num_constraints = 0;
    void* csr = nullptr;                  // one allocation behind row_ptr, val and col
    uint32_t* row_ptr = nullptr;
    uint32_t* col = nullptr;
    b200zk::Fr* val = nullptr;
};

namespace b200zk {

inline int set_error(b200zk_ctx* ctx, int code, const std::string& msg) {
    if (ctx) {
        std::lock_guard<std::mutex> g(ctx->err_mu);
        ctx->last_error = msg;
    }
    return code;
}

#define B2_CUDA_OK(ctx, expr)                                                                         \
    do {                                                                                              \
        cudaError_t _e = (expr);                                                                      \
        if (_e != cudaSuccess) {                                                                      \
            char _b[512];                                                                             \
            snprintf(_b, sizeof(_b), "CUDA error %s at %s:%d (%s)", cudaGetErrorString(_e), __FILE__, \
                     __LINE__, #expr);                                                                \
            return set_error((ctx), _e == cudaErrorMemoryAllocation ? B200ZK_ERR_OOM : B200ZK_ERR_CUDA, _b); \
        }                                                                                             \
    } while (0)

#define B2_TRY(expr)                 \
    do {                             \
        int _rc = (expr);            \
        if (_rc != B200ZK_OK) return _rc; \
    } while (0)

// RAII kernel-launch bracket: counts launches and, when profiling is on, records an event pair.
struct LaunchScope {
    b200zk_ctx* ctx;
    cudaStream_t st;
    ProfEntry e;
    bool active;
    LaunchScope(b200zk_ctx* c, cudaStream_t s, const char* name) : ctx(c), st(s), active(false) {
        ctx->launches++;
        if (ctx->prof_on) {
            e.name = name;
            cudaEventCreate(&e.start);
            cudaEventCreate(&e.stop);
            cudaEventRecord(e.start, st);
            active = true;
        }
    }
    ~LaunchScope() {
        if (active) {
            cudaEventRecord(e.stop, st);
            std::lock_guard<std::mutex> g(ctx->prof_mu);
            ctx->prof_pending.push_back(e);
        }
    }
};

inline int check_launch(b200zk_ctx* ctx, const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        char b[256];
        snprintf(b, sizeof(b), "kernel launch failed (%s): %s", what, cudaGetErrorString(e));
        return set_error(ctx, B200ZK_ERR_CUDA, b);
    }
    return B200ZK_OK;
}

// Every kernel launch of the library: counted, timed under the profile name `name` while profiling is on, and checked.
// Arguments convert to the kernel's parameter types as in a direct launch; default arguments do not apply.
template <class... P, class... A>
int launch(b200zk_ctx* ctx, cudaStream_t st, const char* name, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem,
           A&&... args) {
    {
        LaunchScope ls(ctx, st, name);
        kernel<<<grid, block, smem, st>>>(std::forward<A>(args)...);
    }
    return check_launch(ctx, name);
}

static inline unsigned ceil_log2(size_t n) {
    unsigned l = 0;
    while (((size_t)1 << l) < n) ++l;
    return l;
}

// The column layout of a 2^(log_rows + log_cols) vector over P = 2^(log_cols - log_cg) GPUs (group.cu): GPU g keeps the
// cg = 2^log_cg columns [g cg, (g+1) cg), its local slot c rows + r holding global row r cols + g cg + c.  The one definition
// of the map in both directions, for the host (slot_row, the sharded row_ptr) and the device (the group zkey's sort key).
struct ColumnLayout {
    uint32_t log_rows, log_cols, log_cg;
    __host__ __device__ __forceinline__ size_t row(uint32_t g, size_t j) const {           // slot j of GPU g -> global row
        return ((j & (((size_t)1 << log_rows) - 1)) << log_cols) + ((size_t)g << log_cg) + (j >> log_rows);
    }
    __host__ __device__ __forceinline__ uint32_t owner(uint32_t R) const {                 // global row -> its GPU
        return (R & ((1u << log_cols) - 1)) >> log_cg;
    }
    __host__ __device__ __forceinline__ uint32_t slot(uint32_t R) const {                  // global row -> its owner's slot
        return ((R & ((1u << log_cg) - 1)) << log_rows) + (R >> log_cols);
    }
};

// ---- entry points implemented across translation units -------------------------------------
// ntt.cu
int ntt_dev(b200zk_ctx* ctx, Slot& sl, const Fr* d_in, Fr* d_out, unsigned log_n, bool inverse, bool coset,
            unsigned batch);
int h_circom_dev(b200zk_ctx* ctx, Slot& sl, const Fr* d_a, const Fr* d_b, const Fr* d_c, unsigned log_m, Fr* d_h);
int bitrev_dev(b200zk_ctx* ctx, Slot& sl, const Fr* d_in, Fr* d_out, unsigned log_n);
int fourstep_cols_dev(b200zk_ctx* ctx, Slot& sl, const Fr* d_in, Fr* d_out, unsigned log_rows,
                      unsigned log_cols_local, unsigned log_n, uint64_t global_col0, bool inverse);
int ntt_batched_post_dev(b200zk_ctx* ctx, Slot& sl, const Fr* d_in, Fr* d_out, unsigned log_t, unsigned batch, bool inverse,
                         unsigned log_base, bool base_is_shift, uint64_t b0, uint64_t alpha, uint64_t beta, uint64_t gamma);
int fourstep_cols_p2p_dev(b200zk_ctx* ctx, Slot& sl, const Fr* d_in, void* const* peer_out, unsigned n_peers, unsigned log_rows,
                          unsigned log_cols_local, unsigned log_n, uint64_t global_col0, bool inverse);
int mul_sub_dev(b200zk_ctx* ctx, Slot& sl, const Fr* a, const Fr* b, const Fr* c, Fr* out, size_t n);
void ntt_free_plans(b200zk_ctx* ctx);
// msm.cu
// seg: buckets per segment of the bucket reduction; 0, or more than one window's buckets, keeps the default of 16 (small bucket
// sets take 8 whatever seg says)
int msm_g1_dev(b200zk_ctx* ctx, Slot& sl, const void* d_bases, const void* d_scalars, size_t n, void* d_out_xyzz, unsigned seg);
int msm_g2_dev(b200zk_ctx* ctx, Slot& sl, const void* d_bases, const void* d_scalars, size_t n, void* d_out_xyzz, unsigned seg);
int msm_parts_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_bases, const void* d_scalars, const size_t* cnt, unsigned nparts,
                  const cudaEvent_t* ev_scalars, const cudaEvent_t* ev_bases, void* d_out_xyzz);
// api.cu: host buffers -> device partial, staged in parts
int msm_staged_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* bases, const void* scalars, size_t n, void* d_out, bool wait_copies);
unsigned msm_table_windows(unsigned c);
unsigned msm_table_auto_window(size_t n);
// exclusive prefix sum of n u32 (n < 2^32); sums: scratch of ceil(n / 2048) u32
int exclusive_scan(b200zk_ctx* ctx, cudaStream_t st, const uint32_t* in, uint32_t* out, uint32_t* sums, uint32_t n);
int msm_table_build_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_bases, size_t n, unsigned c, void* d_table);
int msm_table_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_table, const void* d_scalars, size_t n, unsigned c,
                  void* d_out_xyzz, unsigned seg);
int g1_sum_dev(b200zk_ctx* ctx, Slot& sl, const void* d_xyzz, size_t count, void* d_out_affine);
int g2_sum_dev(b200zk_ctx* ctx, Slot& sl, const void* d_xyzz, size_t count, void* d_out_affine);
int xyzz_sum_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_in, size_t count, size_t stride, void* d_out);
int msm_exchange_sum_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_partial, void* const* peer_boxes, unsigned n_peers, unsigned rank,
                         uint64_t seq, void* d_out_affine);
int generate_points_dev(b200zk_ctx* ctx, Slot& sl, int g2, uint64_t seed, size_t n, void* d_out);
int generate_fr_dev(b200zk_ctx* ctx, Slot& sl, uint64_t seed, size_t n, void* d_out);
int field_op_dev(b200zk_ctx* ctx, Slot& sl, int field, int op, const void* d_a, const void* d_b, void* d_out, size_t n);
// qap.cu
int fr_convert_dev(b200zk_ctx* ctx, Slot& sl, const void* d_in, void* d_out, size_t n, int to_mont, int times);
int qap_dev(b200zk_ctx* ctx, Slot& sl, const void* a_ptr, const void* a_col, const void* a_val, const void* b_ptr,
            const void* b_col, const void* b_val, size_t nc, size_t n_inputs, const void* d_z, unsigned log_m, void* d_a,
            void* d_b, void* d_c);
// The same mat-vec over n_slots output slots of a column-layout slice (qap.cu, QapSlots): slot j holds global row
// (j mod 2^log_rows) 2^log_cols + c0 + j div 2^log_rows, the matrices' CSR row j holds that row's terms.  The caller checks
// the domain.
int qap_slots_dev(b200zk_ctx* ctx, Slot& sl, const void* a_ptr, const void* a_col, const void* a_val, const void* b_ptr,
                  const void* b_col, const void* b_val, size_t nc, size_t n_inputs, const void* d_z, unsigned log_rows,
                  unsigned log_cols, size_t c0, size_t n_slots, void* d_a, void* d_b, void* d_c);
int r1cs_check_dev(b200zk_ctx* ctx, Slot& sl, const void* const ptr[3], const void* const col[3], const void* const val[3], size_t nc,
                   const void* d_w, uint64_t* n_failed, uint64_t* first_failed);
// setup.cu
int fixed_base_mul_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_scalars, size_t n, void* d_out);
int fr_powers_dev(b200zk_ctx* ctx, Slot& sl, const uint64_t base[4], const uint64_t scale[4], size_t n, void* d_out);
int spmv_dev(b200zk_ctx* ctx, Slot& sl, const void* ptr, const void* idx, const void* val, const void* x, size_t n_rows, void* out);
int points_spmv_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* ptr, const void* idx, const void* val, const void* points,
                    size_t n_rows, void* out);
int points_scale_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_points, size_t n, const uint64_t k[4], void* d_out);
int points_intt_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_in, unsigned log_n, void* d_out);
int points_ntt_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_in, unsigned log_n, void* d_out);
int points_mul_powers_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_points, size_t n, const uint64_t first[4],
                          const uint64_t ratio[4], void* d_out);
int points_sub_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_a, const void* d_b, size_t n, void* d_out);
int fr_lincomb_dev(b200zk_ctx* ctx, Slot& sl, const void* a, const void* b, const void* c, const uint64_t s[16], size_t n, void* out);
// codec.cu
int points_compress_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_affine, size_t n, void* d_bytes);
int points_encode_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_affine, size_t n, int fmt, void* d_bytes);
int points_decode_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_bytes, size_t n, int fmt, int check_subgroup,
                      void* d_affine, size_t* n_invalid, size_t* first_invalid);
int points_decompress_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_bytes, size_t n, int check_subgroup, void* d_affine,
                          size_t* n_invalid);
// packexp.cu
int points_matmul_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_points, size_t n_chunks, size_t l, const void* d_matrix,
                      size_t rows, void* d_out);
// verify.cu
int groth16_verify_dev(b200zk_ctx* ctx, Slot& sl, const uint64_t* alpha_g1, const uint64_t* beta_g2, const uint64_t* gamma_g2,
                       const uint64_t* delta_g2, const uint64_t* gamma_abc_g1, size_t n_public, const uint64_t* public_inputs,
                       const uint64_t* proof_a, const uint64_t* proof_b, const uint64_t* proof_c, int* is_valid);
int vk_alphabeta_12_dev(b200zk_ctx* ctx, Slot& sl, const uint64_t* alpha_g1, const uint64_t* beta_g2, uint64_t* out);
// prove.cu
int assemble_dev(b200zk_ctx* ctx, Slot& sl, const b200zk_pk* pk, const void* msm_a, const void* msm_b2, const void* msm_l,
                 const void* msm_h, const void* msm_b1, const uint64_t r[4], const uint64_t s[4], int include_zero_terms,
                 uint8_t proof_out[128]);
int pk_precompute_dev(b200zk_ctx* ctx, b200zk_pk* pk, unsigned c);
void pk_free_tables(b200zk_pk* pk);
// false when B200ZK_PK_TABLES=0: proving keys are then uploaded without fixed-base tables
bool pk_tables_enabled();
// The fixed-base window tables (msm.cu section 7) of a proving key's five queries src[k] of cnt[k] points (a, b_g1, b_g2, l, h;
// k = 2 is the G2 one), built on sl's stream with window c_req, or msm_table_auto_window(cnt[k]) per query for c_req = 0.
// Queries under 64 points get none.  All or nothing: when a table would reach 2^31 entries, when the tables would exceed
// B200ZK_PK_TABLE_MAX_GB (default: 60% of the HBM free right now) or when an allocation fails, none is kept and the generic MSM
// runs on the queries.  tab / tab_c / *bytes: what was built (tab_c[k] = 0: no table).
int pk_tables_build(b200zk_ctx* ctx, Slot& sl, const void* const src[5], const size_t cnt[5], unsigned c_req, void* tab[5],
                    unsigned tab_c[5], size_t* bytes);
// MSM over query k (numbered as for pk_tables_build): over tab[k] when tab_c[k] != 0, else the generic MSM on `query`;
// seg as for msm_g1_dev
int query_msm(b200zk_ctx* ctx, Slot& sl, int k, const void* query, void* const tab[5], const unsigned tab_c[5], const Fr* scalars,
              size_t n, void* out, unsigned seg);
int prove_dev(b200zk_ctx* ctx, const b200zk_pk* pk, const Fr* d_z, const Fr* d_a, const Fr* d_b, const Fr* d_c,
              const uint64_t r[4], const uint64_t s[4], int mirror_bg1, uint8_t proof_out[128]);
// zkey.cu (the header fields come from snarkjs_files.h's parse_zkey)
namespace sjf { struct Zkey; }
// parse_zkey and the 2^27 domain limit of every zkey load: B200ZK_OK, or the code with *err
int zkey_header(const uint8_t* file, size_t len, sjf::Zkey* h, std::string* err);
// the 56 vk limbs of b200zk_pk_upload from the header's points
void zkey_vk_points(const uint8_t* file, const sjf::Zkey& h, uint64_t vk[56]);
int zkey_matrices_dev(b200zk_ctx* ctx, Slot& sl, const uint8_t* file, const sjf::Zkey& h, b200zk_zkey* zk);
// The group load's sort on one device: the checked records keyed owner-major over the layout cl, in one allocation `csr` (the
// caller frees it): row_ptr of 2 m + 1 entries, GPU g's A rows at [2 g loc, (2 g + 1) loc] and B rows at [(2 g + 1) loc,
// 2 (g + 1) loc] (loc = m / P), indexing col / val
struct ZkeyCsr {
    void* csr = nullptr;
    uint32_t* row_ptr = nullptr;
    uint32_t* col = nullptr;
    Fr* val = nullptr;
    uint32_t nc = 0;
};
int zkey_group_matrices_dev(b200zk_ctx* ctx, Slot& sl, const uint8_t* file, const sjf::Zkey& h, const ColumnLayout& cl, ZkeyCsr* out);
// p[i] -= base, i < n, on the slot's stream
int rebase_dev(b200zk_ctx* ctx, Slot& sl, uint32_t* p, size_t n, uint32_t base);
// The host side of a prove from a .wtns, before any launch: parse, entry count, JSON buffer sizes (both lengths set when one
// is short), r and s (drawn from getrandom when null).  B200ZK_OK, or the code with *err.
struct WtnsJob {
    const uint8_t* z = nullptr;          // n_vars canonical values in the caller's bytes
    std::string pub;                     // public.json
    uint64_t r[4], s[4];
};
int wtns_prologue(const uint8_t* wtns, size_t wtns_len, size_t n_vars, size_t n_public, const uint64_t* r_in, const uint64_t* s_in,
                  const char* proof_json, size_t* proof_json_len, const char* public_json, size_t* public_json_len, WtnsJob* job,
                  std::string* err);
// the nv canonical values z -> Montgomery at d_z (refused, with a context error, when an entry is not below r)
int witness_to_device(b200zk_ctx* ctx, Slot& sl, const uint8_t* z, size_t nv, Fr* d_z);
// the scratch in sl.io_a that zkey_outputs_dev uses
static const size_t JSON_SCRATCH = 768;
// proof bytes and texts to the caller: proof_out, public.json, and proof.json from the points' encodings made on sl
int zkey_outputs_dev(b200zk_ctx* ctx, Slot& sl, const uint8_t proof[128], const WtnsJob& job, uint8_t* proof_out, char* proof_json,
                     size_t* proof_json_len, char* public_json, size_t* public_json_len);
int zkey_prove_dev(b200zk_ctx* ctx, Slot& sl, const b200zk_zkey* zk, const uint8_t* wtns, size_t wtns_len, const uint64_t* r,
                   const uint64_t* s, uint8_t* proof_out, char* proof_json, size_t* proof_json_len, char* public_json,
                   size_t* public_json_len);

}  // namespace b200zk
