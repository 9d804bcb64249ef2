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
    cudaEvent_t copy_done = nullptr;
    cudaStream_t aux_stream = nullptr;    // second compute stream + workspace: host-staged MSMs run as two halves
    DevBuf ws_msm_aux;
    cudaEvent_t aux_done = nullptr;
    cudaEvent_t stage_ev[32] = {};        // host-staged MSM: arrival of part p's scalars [2 p] / bases [2 p + 1]
};

}  // namespace b200zk

struct b200zk_ctx {
    int device = 0;
    int sm_count = 132;
    b200zk::Slot slots[3];
    unsigned msm_seg_hint = 0;      // set by prove_dev around its MSM launches (it holds every slot lock): reduction segment length
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
    // MSM channels (msm.cu, window-group pipeline): 0..5 = slot i's main / aux workspace (2 i + aux).
    // msm_side[ch]: high-priority helper stream that runs the sort phases and the reduction / Horner tail of one window
    // group while the bucket kernel of the next group occupies the SMs; msm_events[ch]: its event pool (grown on demand,
    // only ever touched under the owning slot's mutex).
    cudaStream_t msm_side[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    std::vector<cudaEvent_t> msm_events[6];
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

static inline unsigned ceil_log2(size_t n) {
    unsigned l = 0;
    while (((size_t)1 << l) < n) ++l;
    return l;
}

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
// aux != 0: run on the slot's second compute stream / workspace (aux_stream, ws_msm_aux)
int msm_g1_dev(b200zk_ctx* ctx, Slot& sl, const void* d_bases, const void* d_scalars, size_t n, void* d_out_xyzz,
               cudaEvent_t bases_ready = nullptr, int aux = 0);
int msm_g2_dev(b200zk_ctx* ctx, Slot& sl, const void* d_bases, const void* d_scalars, size_t n, void* d_out_xyzz,
               cudaEvent_t bases_ready = nullptr, int aux = 0);
int msm_parts_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_bases, const void* d_scalars, const size_t* cnt, unsigned nparts,
                  const cudaEvent_t* ev_scalars, const cudaEvent_t* ev_bases, void* d_out_xyzz);
// api.cu: host buffers -> device partial, staged in parts
int msm_staged_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* bases, const void* scalars, size_t n, void* d_out, bool wait_copies);
unsigned msm_table_windows(unsigned c);
unsigned msm_table_auto_window(size_t n);
int msm_table_build_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_bases, size_t n, unsigned c, void* d_table);
int msm_table_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_table, const void* d_scalars, size_t n, unsigned c,
                  void* d_out_xyzz, int aux = 0);
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
int prove_dev(b200zk_ctx* ctx, const b200zk_pk* pk, const Fr* d_z, const Fr* d_a, const Fr* d_b, const Fr* d_c,
              const uint64_t r[4], const uint64_t s[4], int mirror_bg1, uint8_t proof_out[128]);

}  // namespace b200zk
