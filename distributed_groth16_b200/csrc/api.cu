// api.cu -- the extern "C" surface declared in include/b200zk.h.
#include <sstream>

#include "blake2b.cuh"
#include "common.cuh"

using namespace b200zk;

static const char* kVersion = "b200zk 0.1 (sm_90a)";

static bool valid_slot(int s) { return s >= 0 && s < 3; }

extern "C" {

const char* b200zk_version(void) { return kVersion; }

int b200zk_ctx_create(int device, b200zk_ctx** out) {
    if (!out) return B200ZK_ERR_ARG;
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0 || device < 0 || device >= count) return B200ZK_ERR_CUDA;   // no CPU fallback
    if (cudaSetDevice(device) != cudaSuccess) return B200ZK_ERR_CUDA;
    b200zk_ctx* ctx = new b200zk_ctx();
    ctx->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) ctx->sm_count = prop.multiProcessorCount;
    for (int i = 0; i < 3; ++i) {
        if (cudaStreamCreateWithFlags(&ctx->slots[i].stream, cudaStreamNonBlocking) != cudaSuccess) {
            delete ctx;
            return B200ZK_ERR_CUDA;
        }
        ctx->slots[i].owns_stream = true;
        bool ok = cudaStreamCreateWithFlags(&ctx->slots[i].copy_stream, cudaStreamNonBlocking) == cudaSuccess &&
                  cudaStreamCreateWithFlags(&ctx->slots[i].aux_stream, cudaStreamNonBlocking) == cudaSuccess &&
                  cudaEventCreateWithFlags(&ctx->slots[i].copy_done, cudaEventDisableTiming) == cudaSuccess &&
                  cudaEventCreateWithFlags(&ctx->slots[i].aux_done, cudaEventDisableTiming) == cudaSuccess;
        for (int k = 0; ok && k < 32; ++k) ok = cudaEventCreateWithFlags(&ctx->slots[i].stage_ev[k], cudaEventDisableTiming) == cudaSuccess;
        if (!ok) {
            delete ctx;
            return B200ZK_ERR_CUDA;
        }
    }
    {
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        bool ok = true;
        for (int k = 0; ok && k < 6; ++k) ok = cudaStreamCreateWithPriority(&ctx->msm_side[k], cudaStreamNonBlocking, hi) == cudaSuccess;
        if (!ok) { b200zk_ctx_destroy(ctx); return B200ZK_ERR_CUDA; }
    }
    *out = ctx;
    return B200ZK_OK;
}

void b200zk_ctx_destroy(b200zk_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    ntt_free_plans(ctx);
    if (ctx->fb_table_g1) cudaFree(ctx->fb_table_g1);
    if (ctx->fb_table_g2) cudaFree(ctx->fb_table_g2);
    for (int i = 0; i < 3; ++i) {
        Slot& s = ctx->slots[i];
        s.ws_msm.release(); s.ws_ntt.release(); s.io_a.release(); s.io_b.release(); s.small.release();
        if (s.owns_stream && s.stream) cudaStreamDestroy(s.stream);
        s.ws_msm_aux.release();
        if (s.copy_stream) cudaStreamDestroy(s.copy_stream);
        if (s.aux_stream) cudaStreamDestroy(s.aux_stream);
        if (s.copy_done) cudaEventDestroy(s.copy_done);
        if (s.aux_done) cudaEventDestroy(s.aux_done);
        for (int k = 0; k < 32; ++k) if (s.stage_ev[k]) cudaEventDestroy(s.stage_ev[k]);
    }
    for (int k = 0; k < 6; ++k) if (ctx->msm_side[k]) cudaStreamDestroy(ctx->msm_side[k]);
    for (auto& v : ctx->msm_events) for (cudaEvent_t e : v) cudaEventDestroy(e);
    for (auto& e : ctx->prof_pending) { cudaEventDestroy(e.start); cudaEventDestroy(e.stop); }
    delete ctx;
}

const char* b200zk_last_error(const b200zk_ctx* ctx) { return ctx ? ctx->last_error.c_str() : "null context"; }

int b200zk_ctx_set_stream(b200zk_ctx* ctx, int stream, void* cuda_stream) {
    if (!ctx || !valid_slot(stream)) return B200ZK_ERR_ARG;
    Slot& s = ctx->slots[stream];
    std::lock_guard<std::mutex> g(s.mu);
    if (s.owns_stream && s.stream) { cudaStreamSynchronize(s.stream); cudaStreamDestroy(s.stream); }
    s.stream = reinterpret_cast<cudaStream_t>(cuda_stream);
    s.owns_stream = false;
    return B200ZK_OK;
}

int b200zk_ctx_sync(b200zk_ctx* ctx, int stream) {
    if (!ctx || !valid_slot(stream)) return B200ZK_ERR_ARG;
    B2_CUDA_OK(ctx, cudaStreamSynchronize(ctx->slots[stream].stream));
    return B200ZK_OK;
}

int b200zk_profile_enable(b200zk_ctx* ctx, int on) {
    if (!ctx) return B200ZK_ERR_ARG;
    ctx->prof_on = on != 0;
    return B200ZK_OK;
}

static void prof_drain(b200zk_ctx* ctx) {
    std::lock_guard<std::mutex> g(ctx->prof_mu);
    static const bool timeline = getenv("B200ZK_PROFILE_TIMELINE") && getenv("B200ZK_PROFILE_TIMELINE")[0] == '1';
    for (auto& e : ctx->prof_pending) {
        cudaEventSynchronize(e.stop);
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, e.start, e.stop) == cudaSuccess) {
            auto& acc = ctx->prof_acc[e.name];
            acc.first += 1;
            acc.second += ms;
        }
        bool keep = false;
        if (timeline) {
            if (!ctx->prof_base) { ctx->prof_base = e.start; keep = true; }
            float t0 = 0.f, t1 = 0.f;
            cudaEventElapsedTime(&t0, ctx->prof_base, e.start);
            cudaEventElapsedTime(&t1, ctx->prof_base, e.stop);
            ctx->prof_timeline.emplace_back(e.name, t0, t1);
        }
        if (!keep) cudaEventDestroy(e.start);
        cudaEventDestroy(e.stop);
    }
    ctx->prof_pending.clear();
}

int b200zk_profile_reset(b200zk_ctx* ctx) {
    if (!ctx) return B200ZK_ERR_ARG;
    prof_drain(ctx);
    std::lock_guard<std::mutex> g(ctx->prof_mu);
    ctx->prof_acc.clear();
    ctx->prof_timeline.clear();
    if (ctx->prof_base) { cudaEventDestroy(ctx->prof_base); ctx->prof_base = nullptr; }
    ctx->launches = 0;
    return B200ZK_OK;
}

int b200zk_profile_json(b200zk_ctx* ctx, char* buf, size_t buf_len) {
    if (!ctx || !buf || buf_len == 0) return B200ZK_ERR_ARG;
    prof_drain(ctx);
    std::ostringstream os;
    os << "{";
    bool first = true;
    {
        std::lock_guard<std::mutex> g(ctx->prof_mu);
        for (auto& kv : ctx->prof_acc) {
            if (!first) os << ", ";
            first = false;
            os << "\"" << kv.first << "\": {\"launches\": " << kv.second.first << ", \"ms\": " << kv.second.second << "}";
        }
        if (!ctx->prof_timeline.empty()) {
            os << (first ? "" : ", ") << "\"_timeline\": [";
            for (size_t i = 0; i < ctx->prof_timeline.size(); ++i) {
                auto& t = ctx->prof_timeline[i];
                os << (i ? ", " : "") << "[\"" << std::get<0>(t) << "\", " << std::get<1>(t) << ", " << std::get<2>(t) << "]";
            }
            os << "]";
        }
    }
    os << "}";
    std::string s = os.str();
    if (s.size() + 1 > buf_len) return B200ZK_ERR_ARG;
    memcpy(buf, s.c_str(), s.size() + 1);
    return B200ZK_OK;
}

uint64_t b200zk_launch_count(const b200zk_ctx* ctx) { return ctx ? ctx->launches.load() : 0; }

}  // extern "C"

// ---- MSM ---------------------------------------------------------------------------------------
// Host buffers -> this device's XYZZ partial in d_out (device memory), stream-ordered on the slot's stream.  Large inputs travel
// in parts on the copy stream (scalars of part p, bases of part p, scalars of part p + 1, ...): the sort phases of a part start when
// its scalars are there, its bucket kernel when its bases are, and every part adds into the same bucket set -- the PCIe transfer of
// part p + 1 hides behind the bucket kernel of part p (msm.cu, msm_dev_impl).  The host buffers may be reused once the copy stream
// has drained, which `wait_copies` does before returning.  Caller holds the slot mutex and has made the device current.
namespace b200zk {
int msm_staged_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* bases, const void* scalars, size_t n, void* d_out, bool wait_copies) {
    const size_t PB = g2 ? 128 : 64;
    B2_CUDA_OK(ctx, sl.io_a.reserve(n * PB + n * 32 + 64));
    char* d_bases = reinterpret_cast<char*>(sl.io_a.p);
    char* d_scalars = d_bases + n * PB;
    // Part sizes: a smaller first part shortens the time the GPU waits for its first bases, a smaller last part the bucket work
    // left when the last byte has arrived.  Weights 2,3,4,4,3 beat four equal parts, other weightings and seven parts at
    // 2^20 / 2^22 -- every part costs a sort, a bucket kernel with its drain and a merge.  Below 2^18 one part.
    static const unsigned staged_weights[5] = {2, 3, 4, 4, 3}, one_weight[1] = {1};
    const unsigned nparts = n >= ((size_t)1 << 18) ? 5 : 1;
    const unsigned* weights = nparts > 1 ? staged_weights : one_weight;
    unsigned wsum = 0;
    for (unsigned p = 0; p < nparts; ++p) wsum += weights[p];
    const char* hb = reinterpret_cast<const char*>(bases);
    const char* hs = reinterpret_cast<const char*>(scalars);
    cudaStream_t cs = sl.copy_stream;
    size_t cnt[5];
    cudaEvent_t ev_s[5], ev_b[5];
    size_t lo = 0;
    unsigned wcum = 0;
    for (unsigned p = 0; p < nparts; ++p) {
        wcum += weights[p];
        const size_t hi = (size_t)(((unsigned __int128)n * wcum) / wsum);
        cnt[p] = hi - lo;
        ev_s[p] = ev_b[p] = nullptr;
        if (cnt[p]) {
            B2_CUDA_OK(ctx, cudaMemcpyAsync(d_scalars + lo * 32, hs + lo * 32, cnt[p] * 32, cudaMemcpyHostToDevice, cs));
            B2_CUDA_OK(ctx, cudaEventRecord(sl.stage_ev[2 * p], cs));
            B2_CUDA_OK(ctx, cudaMemcpyAsync(d_bases + lo * PB, hb + lo * PB, cnt[p] * PB, cudaMemcpyHostToDevice, cs));
            B2_CUDA_OK(ctx, cudaEventRecord(sl.stage_ev[2 * p + 1], cs));
            ev_s[p] = sl.stage_ev[2 * p];
            ev_b[p] = sl.stage_ev[2 * p + 1];
        }
        lo = hi;
    }
    B2_TRY(msm_parts_dev(ctx, sl, g2, d_bases, d_scalars, cnt, nparts, ev_s, ev_b, d_out));
    if (wait_copies) B2_CUDA_OK(ctx, cudaStreamSynchronize(cs));
    return B200ZK_OK;
}
}  // namespace b200zk

template <int G2>
static int msm_host(b200zk_ctx* ctx, int stream, const uint64_t* bases, size_t n_bases, const uint64_t* scalars,
                    size_t n_scalars, uint64_t* out_affine, int* out_is_inf) {
    if (!ctx || !valid_slot(stream) || !out_affine || !out_is_inf) return B200ZK_ERR_ARG;
    if (n_bases != n_scalars) {
        // arkworks: `Err(min(bases.len(), scalars.len()))`, turned into MpcNetError::Generic(min_len.to_string())
        return set_error(ctx, B200ZK_ERR_LENGTH, std::to_string(n_bases < n_scalars ? n_bases : n_scalars));
    }
    const size_t n = n_bases;
    if (n && (!bases || !scalars)) return B200ZK_ERR_ARG;
    const size_t PB = G2 ? 128 : 64, XB = G2 ? 256 : 128;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    B2_CUDA_OK(ctx, sl.small.reserve(1024));
    char* sm = reinterpret_cast<char*>(sl.small.p);
    B2_TRY(msm_staged_dev(ctx, sl, G2, bases, scalars, n, sm, false));
    B2_TRY(G2 ? g2_sum_dev(ctx, sl, sm, 1, sm + XB) : g1_sum_dev(ctx, sl, sm, 1, sm + XB));
    uint64_t host[17];
    B2_CUDA_OK(ctx, cudaMemcpyAsync(host, sm + XB, PB + 8, cudaMemcpyDeviceToHost, sl.stream));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(sl.stream));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(sl.copy_stream));
    memcpy(out_affine, host, PB);
    *out_is_inf = (int)host[PB / 8];
    return B200ZK_OK;
}

template <int G2>
static int sum_host(b200zk_ctx* ctx, int stream, const void* d_xyzz, size_t count, uint64_t* out_affine, int* out_is_inf) {
    if (!ctx || !valid_slot(stream) || !out_affine || !out_is_inf) return B200ZK_ERR_ARG;
    const size_t PB = G2 ? 128 : 64;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    B2_CUDA_OK(ctx, sl.small.reserve(1024));
    char* sm = reinterpret_cast<char*>(sl.small.p);
    B2_TRY(G2 ? g2_sum_dev(ctx, sl, d_xyzz, count, sm) : g1_sum_dev(ctx, sl, d_xyzz, count, sm));
    uint64_t host[17];
    B2_CUDA_OK(ctx, cudaMemcpyAsync(host, sm, PB + 8, cudaMemcpyDeviceToHost, sl.stream));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(sl.stream));
    memcpy(out_affine, host, PB);
    *out_is_inf = (int)host[PB / 8];
    return B200ZK_OK;
}

extern "C" {

int b200zk_msm_g1(b200zk_ctx* ctx, int stream, const uint64_t* bases, size_t n_bases, const uint64_t* scalars,
                  size_t n_scalars, uint64_t out_affine[8], int* out_is_inf) {
    return msm_host<0>(ctx, stream, bases, n_bases, scalars, n_scalars, out_affine, out_is_inf);
}
int b200zk_msm_g2(b200zk_ctx* ctx, int stream, const uint64_t* bases, size_t n_bases, const uint64_t* scalars,
                  size_t n_scalars, uint64_t out_affine[16], int* out_is_inf) {
    return msm_host<1>(ctx, stream, bases, n_bases, scalars, n_scalars, out_affine, out_is_inf);
}

int b200zk_msm_staged_dev(b200zk_ctx* ctx, int stream, int g2, const uint64_t* bases, size_t n_bases, const uint64_t* scalars,
                          size_t n_scalars, void* d_out_xyzz) {
    if (!ctx || !valid_slot(stream) || !d_out_xyzz) return B200ZK_ERR_ARG;
    if (n_bases != n_scalars) return set_error(ctx, B200ZK_ERR_LENGTH, std::to_string(n_bases < n_scalars ? n_bases : n_scalars));
    if (n_bases && (!bases || !scalars)) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    return msm_staged_dev(ctx, sl, g2, bases, scalars, n_bases, d_out_xyzz, true);
}

int b200zk_msm_g1_dev(b200zk_ctx* ctx, int stream, const void* d_bases, const void* d_scalars, size_t n, void* d_out) {
    if (!ctx || !valid_slot(stream) || !d_out) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return msm_g1_dev(ctx, sl, d_bases, d_scalars, n, d_out);
}
int b200zk_msm_g2_dev(b200zk_ctx* ctx, int stream, const void* d_bases, const void* d_scalars, size_t n, void* d_out) {
    if (!ctx || !valid_slot(stream) || !d_out) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return msm_g2_dev(ctx, sl, d_bases, d_scalars, n, d_out);
}

unsigned b200zk_msm_table_windows(unsigned c) { return c ? msm_table_windows(c) : 0; }
unsigned b200zk_msm_table_auto_window(size_t n) { return msm_table_auto_window(n); }
int b200zk_msm_table_build_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_bases, size_t n, unsigned c, void* d_table) {
    if (!ctx || !valid_slot(stream) || (n && (!d_bases || !d_table))) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return msm_table_build_dev(ctx, sl, g2, d_bases, n, c, d_table);
}
int b200zk_msm_table_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_table, const void* d_scalars, size_t n, unsigned c,
                         void* d_out) {
    if (!ctx || !valid_slot(stream) || !d_out) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return msm_table_dev(ctx, sl, g2, d_table, d_scalars, n, c, d_out);
}

int b200zk_g1_sum_dev(b200zk_ctx* ctx, int stream, const void* d, size_t count, uint64_t out[8], int* inf) {
    return sum_host<0>(ctx, stream, d, count, out, inf);
}
int b200zk_g2_sum_dev(b200zk_ctx* ctx, int stream, const void* d, size_t count, uint64_t out[16], int* inf) {
    return sum_host<1>(ctx, stream, d, count, out, inf);
}

// ---- NTT ---------------------------------------------------------------------------------------
int b200zk_ntt_fr(b200zk_ctx* ctx, int stream, uint64_t* data, unsigned log_n, int inverse, int coset, int bitrev_in,
                  int bitrev_out, unsigned pad) {
    if (!ctx || !valid_slot(stream) || !data) return B200ZK_ERR_ARG;
    if (log_n > 28) return set_error(ctx, B200ZK_ERR_DOMAIN, "log_n > 28 exceeds the two-adicity of BN254 Fr");
    if (pad == 0) pad = 1;
    if (pad & (pad - 1)) return set_error(ctx, B200ZK_ERR_ARG, "pad must be a power of two");
    const size_t n = (size_t)1 << log_n, n_out = n * pad;
    unsigned log_out = log_n + ceil_log2(pad);
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    B2_CUDA_OK(ctx, sl.io_a.reserve(2 * n_out * sizeof(Fr)));
    Fr* b0 = reinterpret_cast<Fr*>(sl.io_a.p);
    Fr* b1 = b0 + n_out;
    B2_CUDA_OK(ctx, cudaMemcpyAsync(b0, data, n * sizeof(Fr), cudaMemcpyHostToDevice, sl.stream));
    Fr* cur = b0; Fr* other = b1;
    if (bitrev_in) { B2_TRY(bitrev_dev(ctx, sl, cur, other, log_n)); std::swap(cur, other); }
    B2_TRY(ntt_dev(ctx, sl, cur, other, log_n, inverse != 0, coset != 0, 1));
    std::swap(cur, other);
    if (pad > 1) B2_CUDA_OK(ctx, cudaMemsetAsync(cur + n, 0, (n_out - n) * sizeof(Fr), sl.stream));
    if (bitrev_out) { B2_TRY(bitrev_dev(ctx, sl, cur, other, log_out)); std::swap(cur, other); }
    B2_CUDA_OK(ctx, cudaMemcpyAsync(data, cur, n_out * sizeof(Fr), cudaMemcpyDeviceToHost, sl.stream));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(sl.stream));
    return B200ZK_OK;
}

int b200zk_ntt_fr_dev(b200zk_ctx* ctx, int stream, const void* d_in, void* d_out, unsigned log_n, int inverse, int coset,
                      unsigned batch) {
    if (!ctx || !valid_slot(stream) || !d_in || !d_out || batch == 0) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return ntt_dev(ctx, sl, reinterpret_cast<const Fr*>(d_in), reinterpret_cast<Fr*>(d_out), log_n, inverse != 0,
                   coset != 0, batch);
}

int b200zk_ntt_fr_fourstep_cols_dev(b200zk_ctx* ctx, int stream, const void* d_in, void* d_out, unsigned log_rows,
                                    unsigned log_cols_local, unsigned log_n, uint64_t global_col0, int inverse) {
    if (!ctx || !valid_slot(stream)) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return fourstep_cols_dev(ctx, sl, reinterpret_cast<const Fr*>(d_in), reinterpret_cast<Fr*>(d_out), log_rows,
                             log_cols_local, log_n, global_col0, inverse != 0);
}

int b200zk_ntt_fr_fourstep_cols_p2p_dev(b200zk_ctx* ctx, int stream, const void* d_in, void* const* peer_out, unsigned n_peers,
                                        unsigned log_rows, unsigned log_cols_local, unsigned log_n, uint64_t global_col0,
                                        int inverse) {
    if (!ctx || !valid_slot(stream) || !d_in || !peer_out) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return fourstep_cols_p2p_dev(ctx, sl, reinterpret_cast<const Fr*>(d_in), peer_out, n_peers, log_rows, log_cols_local, log_n,
                                 global_col0, inverse != 0);
}

int b200zk_peer_alloc(b200zk_ctx* ctx, size_t bytes, void** d_ptr, uint8_t handle_out[64]) {
    if (!ctx || !d_ptr || !handle_out || bytes == 0) return B200ZK_ERR_ARG;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    B2_CUDA_OK(ctx, cudaMalloc(d_ptr, bytes));
    B2_CUDA_OK(ctx, cudaMemset(*d_ptr, 0, bytes));      // mailboxes (b200zk_msm_exchange_sum_dev) start with sequence flags = 0
    B2_CUDA_OK(ctx, cudaDeviceSynchronize());
    cudaIpcMemHandle_t h;
    B2_CUDA_OK(ctx, cudaIpcGetMemHandle(&h, *d_ptr));
    memcpy(handle_out, &h, 64);
    return B200ZK_OK;
}
int b200zk_peer_open(b200zk_ctx* ctx, const uint8_t handle[64], void** d_ptr) {
    if (!ctx || !d_ptr || !handle) return B200ZK_ERR_ARG;
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    B2_CUDA_OK(ctx, cudaIpcOpenMemHandle(d_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return B200ZK_OK;
}
int b200zk_peer_close(b200zk_ctx* ctx, void* d_ptr) {
    if (!ctx || !d_ptr) return B200ZK_ERR_ARG;
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    B2_CUDA_OK(ctx, cudaIpcCloseMemHandle(d_ptr));
    return B200ZK_OK;
}
int b200zk_peer_free(b200zk_ctx* ctx, void* d_ptr) {
    if (!ctx || !d_ptr) return B200ZK_ERR_ARG;
    B2_CUDA_OK(ctx, cudaFree(d_ptr));
    return B200ZK_OK;
}

int b200zk_msm_exchange_sum_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_partial, void* const* peer_mailboxes, unsigned n_peers,
                                unsigned rank, uint64_t seq, void* d_out_affine) {
    if (!ctx || !valid_slot(stream) || !d_partial || !peer_mailboxes || !d_out_affine) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    return msm_exchange_sum_dev(ctx, sl, g2, d_partial, peer_mailboxes, n_peers, rank, seq, d_out_affine);
}

int b200zk_ntt_fr_batched_post_dev(b200zk_ctx* ctx, int stream, const void* d_in, void* d_out, unsigned log_t, unsigned batch,
                                   int inverse, unsigned log_base, int base_is_shift, uint64_t b0, uint64_t alpha,
                                   uint64_t beta, uint64_t gamma) {
    if (!ctx || !valid_slot(stream) || !d_in || !d_out || batch == 0) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return ntt_batched_post_dev(ctx, sl, reinterpret_cast<const Fr*>(d_in), reinterpret_cast<Fr*>(d_out), log_t, batch,
                                inverse != 0, log_base, base_is_shift != 0, b0, alpha, beta, gamma);
}

int b200zk_fr_mul_sub_dev(b200zk_ctx* ctx, int stream, const void* d_a, const void* d_b, const void* d_c, void* d_out, size_t n) {
    if (!ctx || !valid_slot(stream) || (n && (!d_a || !d_b || !d_c || !d_out))) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return mul_sub_dev(ctx, sl, (const Fr*)d_a, (const Fr*)d_b, (const Fr*)d_c, (Fr*)d_out, n);
}

// ---- h -----------------------------------------------------------------------------------------
int b200zk_h_circom_dev(b200zk_ctx* ctx, const void* d_a, const void* d_b, const void* d_c, unsigned log_m, void* d_h) {
    if (!ctx || !d_a || !d_b || !d_c || !d_h) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[0];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return h_circom_dev(ctx, sl, (const Fr*)d_a, (const Fr*)d_b, (const Fr*)d_c, log_m, (Fr*)d_h);
}

int b200zk_h_circom(b200zk_ctx* ctx, const uint64_t* a, const uint64_t* b, const uint64_t* c, unsigned log_m, uint64_t* h_out) {
    if (!ctx || !a || !b || !c || !h_out) return B200ZK_ERR_ARG;
    if (log_m + 1 > 28) return set_error(ctx, B200ZK_ERR_DOMAIN, "2m exceeds the 2^28 subgroup (PolynomialDegreeTooLarge)");
    const size_t m = (size_t)1 << log_m;
    Slot& sl = ctx->slots[0];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    B2_CUDA_OK(ctx, sl.io_a.reserve(4 * m * sizeof(Fr)));
    Fr* d = reinterpret_cast<Fr*>(sl.io_a.p);
    B2_CUDA_OK(ctx, cudaMemcpyAsync(d, a, m * sizeof(Fr), cudaMemcpyHostToDevice, sl.stream));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(d + m, b, m * sizeof(Fr), cudaMemcpyHostToDevice, sl.stream));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(d + 2 * m, c, m * sizeof(Fr), cudaMemcpyHostToDevice, sl.stream));
    B2_TRY(h_circom_dev(ctx, sl, d, d + m, d + 2 * m, log_m, d + 3 * m));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(h_out, d + 3 * m, m * sizeof(Fr), cudaMemcpyDeviceToHost, sl.stream));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(sl.stream));
    return B200ZK_OK;
}

// ---- qap / conversions -------------------------------------------------------------------------
int b200zk_qap_dev(b200zk_ctx* ctx, int stream, const void* a_ptr, const void* a_col, const void* a_val, const void* b_ptr,
                   const void* b_col, const void* b_val, size_t nc, size_t n_inputs, const void* d_z, unsigned log_m, void* d_a,
                   void* d_b, void* d_c) {
    if (!ctx || !valid_slot(stream) || !a_ptr || !b_ptr || !d_z || !d_a || !d_b || !d_c) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return qap_dev(ctx, sl, a_ptr, a_col, a_val, b_ptr, b_col, b_val, nc, n_inputs, d_z, log_m, d_a, d_b, d_c);
}
int b200zk_fr_convert_dev(b200zk_ctx* ctx, int stream, const void* d_in, void* d_out, size_t n, int to_mont, int times) {
    if (!ctx || !valid_slot(stream) || (n && (!d_in || !d_out)) || times < 0) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return fr_convert_dev(ctx, sl, d_in, d_out, n, to_mont, times);
}
int b200zk_r1cs_check_dev(b200zk_ctx* ctx, int stream, const void* a_ptr, const void* a_col, const void* a_val, const void* b_ptr,
                          const void* b_col, const void* b_val, const void* c_ptr, const void* c_col, const void* c_val, size_t nc,
                          const void* d_w, uint64_t* n_failed, uint64_t* first_failed) {
    if (!ctx) return B200ZK_ERR_ARG;
    if (nc == 0) {
        if (n_failed) *n_failed = 0;
        if (first_failed) *first_failed = 0;
        return B200ZK_OK;
    }
    if (!valid_slot(stream) || !a_ptr || !b_ptr || !c_ptr || !d_w || !n_failed || !first_failed)
        return set_error(ctx, B200ZK_ERR_ARG, "r1cs_check: null pointer or bad stream slot");
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    const void* ptr[3] = {a_ptr, b_ptr, c_ptr};
    const void* col[3] = {a_col, b_col, c_col};
    const void* val[3] = {a_val, b_val, c_val};
    return r1cs_check_dev(ctx, sl, ptr, col, val, nc, d_w, n_failed, first_failed);
}

// ---- proving key + prove -----------------------------------------------------------------------
static int upload(b200zk_ctx* ctx, void** dst, const void* src, size_t bytes, cudaMemcpyKind kind = cudaMemcpyHostToDevice) {
    *dst = nullptr;
    size_t alloc = bytes == 0 ? 16 : bytes;
    B2_CUDA_OK(ctx, cudaMalloc(dst, alloc + 16));
    // the caller's device buffers were written on slot 0's stream (the stream the library hands results back on), so the
    // copy is ordered there; pk_build synchronises that stream before any other slot touches the key
    if (src && bytes) B2_CUDA_OK(ctx, cudaMemcpyAsync(*dst, src, bytes, kind, ctx->slots[0].stream));
    return B200ZK_OK;
}

static int pk_build(b200zk_ctx* ctx, const void* a_query, const void* b_g1_query, const void* b_g2_query, const void* l_query,
                    const void* h_query, size_t n_vars, size_t n_inputs, size_t m, const uint64_t* vk_points,
                    cudaMemcpyKind kind, b200zk_pk** out) {
    if (!ctx || !out || !a_query || !b_g1_query || !b_g2_query || !h_query || !vk_points) return B200ZK_ERR_ARG;
    if (n_vars == 0 || n_inputs == 0 || n_inputs > n_vars) return set_error(ctx, B200ZK_ERR_ARG, "need 1 <= n_inputs <= n_vars");
    if (m == 0 || (m & (m - 1))) return set_error(ctx, B200ZK_ERR_DOMAIN, "h_query length must be a power of two");
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    b200zk_pk* pk = new b200zk_pk();
    pk->n_vars = n_vars; pk->n_inputs = n_inputs; pk->m = m;
    int rc = upload(ctx, &pk->a_query, a_query, n_vars * 64, kind);
    if (!rc) rc = upload(ctx, &pk->b_g1_query, b_g1_query, n_vars * 64, kind);
    if (!rc) rc = upload(ctx, &pk->b_g2_query, b_g2_query, n_vars * 128, kind);
    if (!rc) rc = upload(ctx, &pk->l_query, l_query, (n_vars - n_inputs) * 64, kind);
    if (!rc) rc = upload(ctx, &pk->h_query, h_query, m * 64, kind);
    if (!rc) rc = upload(ctx, &pk->vk, vk_points, 56 * 8);
    if (!rc && cudaStreamSynchronize(ctx->slots[0].stream) != cudaSuccess) rc = set_error(ctx, B200ZK_ERR_CUDA, "proving-key upload failed");
    if (rc) { b200zk_pk_free(ctx, pk); return rc; }
    const char* env = getenv("B200ZK_PK_TABLES");
    if (!(env && env[0] == '0')) {
        std::lock_guard<std::mutex> g(ctx->slots[0].mu);
        B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
        rc = pk_precompute_dev(ctx, pk, 0);
        if (rc) { b200zk_pk_free(ctx, pk); return rc; }
    }
    *out = pk;
    return B200ZK_OK;
}

int b200zk_pk_upload(b200zk_ctx* ctx, const uint64_t* a_query, const uint64_t* b_g1_query, const uint64_t* b_g2_query,
                     const uint64_t* l_query, const uint64_t* h_query, size_t n_vars, size_t n_inputs, size_t m,
                     const uint64_t* vk_points, b200zk_pk** out) {
    return pk_build(ctx, a_query, b_g1_query, b_g2_query, l_query, h_query, n_vars, n_inputs, m, vk_points,
                    cudaMemcpyHostToDevice, out);
}
int b200zk_pk_upload_dev(b200zk_ctx* ctx, const void* a_query, const void* b_g1_query, const void* b_g2_query,
                         const void* l_query, const void* h_query, size_t n_vars, size_t n_inputs, size_t m,
                         const uint64_t* vk_points, b200zk_pk** out) {
    return pk_build(ctx, a_query, b_g1_query, b_g2_query, l_query, h_query, n_vars, n_inputs, m, vk_points,
                    cudaMemcpyDeviceToDevice, out);
}

void b200zk_pk_free(b200zk_ctx* ctx, b200zk_pk* pk) {
    if (!pk) return;
    if (ctx) cudaSetDevice(ctx->device);
    void* ptrs[6] = {pk->a_query, pk->b_g1_query, pk->b_g2_query, pk->l_query, pk->h_query, pk->vk};
    for (void* p : ptrs) if (p) cudaFree(p);
    pk_free_tables(pk);
    delete pk;
}

int b200zk_pk_precompute(b200zk_ctx* ctx, b200zk_pk* pk, unsigned c) {
    if (!ctx || !pk) return B200ZK_ERR_ARG;
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> g(ctx->slots[0].mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    if (c == 0xFFFFFFFFu) { pk_free_tables(pk); return B200ZK_OK; }
    return pk_precompute_dev(ctx, pk, c);
}
size_t b200zk_pk_table_bytes(const b200zk_pk* pk) { return pk ? pk->tab_bytes : 0; }

int b200zk_groth16_prove(b200zk_ctx* ctx, const b200zk_pk* pk, const uint64_t* z, const uint64_t* a, const uint64_t* b,
                         const uint64_t* c, const uint64_t r[4], const uint64_t s[4], int mirror_bg1, uint8_t proof_out[128]) {
    if (!ctx || !pk || !z || !a || !b || !c || !r || !s || !proof_out) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[0];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    const size_t m = pk->m, nv = pk->n_vars;
    B2_CUDA_OK(ctx, sl.io_a.reserve((nv + 3 * m) * sizeof(Fr)));
    Fr* d_z = reinterpret_cast<Fr*>(sl.io_a.p);
    Fr* d_abc = d_z + nv;
    B2_CUDA_OK(ctx, cudaMemcpyAsync(d_z, z, nv * sizeof(Fr), cudaMemcpyHostToDevice, sl.stream));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(d_abc, a, m * sizeof(Fr), cudaMemcpyHostToDevice, sl.stream));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(d_abc + m, b, m * sizeof(Fr), cudaMemcpyHostToDevice, sl.stream));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(d_abc + 2 * m, c, m * sizeof(Fr), cudaMemcpyHostToDevice, sl.stream));
    return prove_dev(ctx, pk, d_z, d_abc, d_abc + m, d_abc + 2 * m, r, s, mirror_bg1, proof_out);
}

int b200zk_groth16_prove_dev(b200zk_ctx* ctx, const b200zk_pk* pk, const void* d_z, const void* d_a, const void* d_b,
                             const void* d_c, const uint64_t r[4], const uint64_t s[4], int mirror_bg1, uint8_t proof_out[128]) {
    if (!ctx || !pk || !d_z || !d_a || !d_b || !d_c || !r || !s || !proof_out) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[0];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    return prove_dev(ctx, pk, (const Fr*)d_z, (const Fr*)d_a, (const Fr*)d_b, (const Fr*)d_c, r, s, mirror_bg1, proof_out);
}

int b200zk_points_compress_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_affine, size_t n, void* d_bytes) {
    if (!ctx || !valid_slot(stream) || (n && (!d_affine || !d_bytes))) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return points_compress_dev(ctx, sl, g2, d_affine, n, d_bytes);
}
int b200zk_points_decompress_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_bytes, size_t n, int check_subgroup,
                                 void* d_affine, size_t* n_invalid) {
    if (!ctx || !valid_slot(stream) || (n && (!d_affine || !d_bytes))) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return points_decompress_dev(ctx, sl, g2, d_bytes, n, check_subgroup, d_affine, n_invalid);
}

int b200zk_points_matmul_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_points, size_t n_chunks, size_t l,
                             const void* d_matrix, size_t rows, void* d_out) {
    if (!ctx || !valid_slot(stream) || (n_chunks && rows && (!d_points || !d_matrix || !d_out))) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return points_matmul_dev(ctx, sl, g2, d_points, n_chunks, l, d_matrix, rows, d_out);
}

int b200zk_groth16_verify(b200zk_ctx* ctx, const uint64_t* alpha_g1, const uint64_t* beta_g2, const uint64_t* gamma_g2,
                          const uint64_t* delta_g2, const uint64_t* gamma_abc_g1, size_t n_public, const uint64_t* public_inputs,
                          const uint64_t* proof_a, const uint64_t* proof_b, const uint64_t* proof_c, int* is_valid) {
    if (!ctx || !alpha_g1 || !beta_g2 || !gamma_g2 || !delta_g2 || !gamma_abc_g1 || (n_public && !public_inputs) || !proof_a ||
        !proof_b || !proof_c || !is_valid)
        return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[0];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    return groth16_verify_dev(ctx, sl, alpha_g1, beta_g2, gamma_g2, delta_g2, gamma_abc_g1, n_public, public_inputs, proof_a, proof_b,
                              proof_c, is_valid);
}
int b200zk_vk_alphabeta_12(b200zk_ctx* ctx, const uint64_t alpha_g1[8], const uint64_t beta_g2[16], uint64_t out[48]) {
    if (!ctx || !alpha_g1 || !beta_g2 || !out) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[0];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    return vk_alphabeta_12_dev(ctx, sl, alpha_g1, beta_g2, out);
}

int b200zk_xyzz_sum_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_in, size_t count, size_t stride, void* d_out) {
    if (!ctx || !valid_slot(stream) || !d_in || !d_out || count == 0) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return xyzz_sum_dev(ctx, sl, g2, d_in, count, stride, d_out);
}
int b200zk_groth16_assemble_dev(b200zk_ctx* ctx, const b200zk_pk* pk, const void* d_msm_a, const void* d_msm_b2,
                                const void* d_msm_l, const void* d_msm_h, const void* d_msm_b1, const uint64_t r[4],
                                const uint64_t s[4], int include_zero_terms, uint8_t proof_out[128]) {
    if (!ctx || !pk || !d_msm_a || !d_msm_b2 || !d_msm_l || !d_msm_h || !r || !s || !proof_out) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[0];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return assemble_dev(ctx, sl, pk, d_msm_a, d_msm_b2, d_msm_l, d_msm_h, d_msm_b1, r, s, include_zero_terms, proof_out);
}

// ---- setup building blocks -----------------------------------------------------------------------
int b200zk_fixed_base_mul_dev(b200zk_ctx* ctx, int g2, const void* d_scalars, size_t n, void* d_out) {
    if (!ctx || (n && (!d_scalars || !d_out))) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[0];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    return fixed_base_mul_dev(ctx, sl, g2, d_scalars, n, d_out);
}
int b200zk_fr_powers_dev(b200zk_ctx* ctx, const uint64_t base[4], const uint64_t scale[4], size_t n, void* d_out) {
    if (!ctx || !base || !scale || (n && !d_out)) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[0];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return fr_powers_dev(ctx, sl, base, scale, n, d_out);
}
int b200zk_fr_spmv_dev(b200zk_ctx* ctx, const void* d_ptr, const void* d_idx, const void* d_val, const void* d_x, size_t n_rows,
                       void* d_out) {
    if (!ctx || !d_ptr || !d_x || (n_rows && !d_out)) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[0];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return spmv_dev(ctx, sl, d_ptr, d_idx, d_val, d_x, n_rows, d_out);
}
int b200zk_points_spmv_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_ptr, const void* d_idx, const void* d_val,
                           const void* d_points, size_t n_rows, void* d_out) {
    if (!ctx || !valid_slot(stream) || (n_rows && (!d_ptr || !d_idx || !d_val || !d_points || !d_out))) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return points_spmv_dev(ctx, sl, g2, d_ptr, d_idx, d_val, d_points, n_rows, d_out);
}
int b200zk_points_scale_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_points, size_t n, const uint64_t k[4],
                            void* d_out) {
    if (!ctx || !k || !valid_slot(stream) || (n && (!d_points || !d_out))) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return points_scale_dev(ctx, sl, g2, d_points, n, k, d_out);
}
int b200zk_points_intt_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_in, unsigned log_n, void* d_out) {
    if (!ctx) return B200ZK_ERR_ARG;
    if (!valid_slot(stream) || !d_in || !d_out) return set_error(ctx, B200ZK_ERR_ARG, "points_intt: null pointer or bad stream slot");
    if (log_n > 28) return set_error(ctx, B200ZK_ERR_DOMAIN, "points_intt: log_n > 28 (the two-adicity of Fr)");
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return points_intt_dev(ctx, sl, g2, d_in, log_n, d_out);
}
int b200zk_points_ntt_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_in, unsigned log_n, void* d_out) {
    if (!ctx) return B200ZK_ERR_ARG;
    if (!valid_slot(stream) || !d_in || !d_out) return set_error(ctx, B200ZK_ERR_ARG, "points_ntt: null pointer or bad stream slot");
    if (log_n > 28) return set_error(ctx, B200ZK_ERR_DOMAIN, "points_ntt: log_n > 28 (the two-adicity of Fr)");
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    return points_ntt_dev(ctx, sl, g2, d_in, log_n, d_out);
}
int b200zk_points_mul_powers_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_points, size_t n, const uint64_t first[4],
                                 const uint64_t ratio[4], void* d_out) {
    if (!ctx) return B200ZK_ERR_ARG;
    if (!valid_slot(stream) || !first || !ratio || (n && (!d_points || !d_out)))
        return set_error(ctx, B200ZK_ERR_ARG, "points_mul_powers: null pointer or bad stream slot");
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return points_mul_powers_dev(ctx, sl, g2, d_points, n, first, ratio, d_out);
}
int b200zk_points_sub_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_a, const void* d_b, size_t n, void* d_out) {
    if (!ctx) return B200ZK_ERR_ARG;
    if (!valid_slot(stream) || (n && (!d_a || !d_b || !d_out)))
        return set_error(ctx, B200ZK_ERR_ARG, "points_sub: null pointer or bad stream slot");
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return points_sub_dev(ctx, sl, g2, d_a, d_b, n, d_out);
}
int b200zk_points_encode_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_affine, size_t n, int fmt, void* d_bytes) {
    if (!ctx) return B200ZK_ERR_ARG;
    if (!valid_slot(stream) || (n && (!d_affine || !d_bytes)))
        return set_error(ctx, B200ZK_ERR_ARG, "points_encode: null pointer or bad stream slot");
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return points_encode_dev(ctx, sl, g2, d_affine, n, fmt, d_bytes);
}
int b200zk_points_decode_dev(b200zk_ctx* ctx, int stream, int g2, const void* d_bytes, size_t n, int fmt, int check_subgroup,
                             void* d_affine, size_t* n_invalid, size_t* first_invalid) {
    if (!ctx) return B200ZK_ERR_ARG;
    if (!valid_slot(stream) || (n && (!d_bytes || !d_affine)))
        return set_error(ctx, B200ZK_ERR_ARG, "points_decode: null pointer or bad stream slot");
    Slot& sl = ctx->slots[stream];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return points_decode_dev(ctx, sl, g2, d_bytes, n, fmt, check_subgroup, d_affine, n_invalid, first_invalid);
}

// ---- Blake2b-512 with an exported state (csrc/blake2b.cuh): host only, no context --------------------------------------
int b200zk_blake2b512_init(uint8_t state[216]) {
    if (!state) return B200ZK_ERR_ARG;
    blake2b_ctx c;
    blake2b_init(&c, 64);
    blake2b_export(&c, state);
    return B200ZK_OK;
}
int b200zk_blake2b512_update(uint8_t state[216], const void* data, size_t len) {
    if (!state || (len && !data)) return B200ZK_ERR_ARG;
    blake2b_ctx c;
    if (!blake2b_import(&c, state)) return B200ZK_ERR_ARG;
    blake2b_update(&c, data, len);
    blake2b_export(&c, state);
    return B200ZK_OK;
}
int b200zk_blake2b512_final(const uint8_t state[216], uint8_t out[64]) {
    if (!state || !out) return B200ZK_ERR_ARG;
    blake2b_ctx c;
    if (!blake2b_import(&c, state) || c.outlen != 64) return B200ZK_ERR_ARG;
    blake2b_final(&c, out);
    return B200ZK_OK;
}

int b200zk_fr_lincomb_dev(b200zk_ctx* ctx, const void* d_a, const void* d_b, const void* d_c, const uint64_t s[16], size_t n,
                          void* d_out) {
    if (!ctx || !s || (n && (!d_a || !d_b || !d_c || !d_out))) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[0];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return fr_lincomb_dev(ctx, sl, d_a, d_b, d_c, s, n, d_out);
}

// ---- generators / self-test --------------------------------------------------------------------
int b200zk_g1_generate_dev(b200zk_ctx* ctx, uint64_t seed, size_t n, void* d_out) {
    if (!ctx || (n && !d_out)) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[0];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return generate_points_dev(ctx, sl, 0, seed, n, d_out);
}
int b200zk_g2_generate_dev(b200zk_ctx* ctx, uint64_t seed, size_t n, void* d_out) {
    if (!ctx || (n && !d_out)) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[0];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return generate_points_dev(ctx, sl, 1, seed, n, d_out);
}
int b200zk_fr_generate_dev(b200zk_ctx* ctx, uint64_t seed, size_t n, void* d_out) {
    if (!ctx || (n && !d_out)) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[0];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));     // the caller may have made another device current (multi-GPU groups)
    return generate_fr_dev(ctx, sl, seed, n, d_out);
}

int b200zk_fr_op(b200zk_ctx* ctx, int op, const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n) {
    if (op < 0 || op > 2) return B200ZK_ERR_ARG;
    return b200zk_test_field_op(ctx, 1, op, a, b, out, n);
}

int b200zk_test_field_op(b200zk_ctx* ctx, int field, int op, const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n) {
    if (!ctx || !a || !b || !out) return B200ZK_ERR_ARG;
    Slot& sl = ctx->slots[0];
    std::lock_guard<std::mutex> g(sl.mu);
    B2_CUDA_OK(ctx, cudaSetDevice(ctx->device));
    B2_CUDA_OK(ctx, sl.io_a.reserve(3 * n * 32 + 64));
    char* d = reinterpret_cast<char*>(sl.io_a.p);
    B2_CUDA_OK(ctx, cudaMemcpyAsync(d, a, n * 32, cudaMemcpyHostToDevice, sl.stream));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(d + n * 32, b, n * 32, cudaMemcpyHostToDevice, sl.stream));
    B2_TRY(field_op_dev(ctx, sl, field, op, d, d + n * 32, d + 2 * n * 32, n));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(out, d + 2 * n * 32, n * 32, cudaMemcpyDeviceToHost, sl.stream));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(sl.stream));
    return B200ZK_OK;
}

}  // extern "C"
