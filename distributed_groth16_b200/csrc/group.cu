// group.cu -- the multi-GPU hot path behind the C ABI: one host process, one b200zk_ctx per device, NVLink peer access.
//
// Replaces, for the single-box setting, the reference's king/client star (/root/reference/mpc-net/src/lib.rs:61-139 used
// through dist-primitives/src/channel/mod.rs:8-56) under the very calls the Rust prover makes:
//   d_msm   dist-primitives/src/dmsm/mod.rs:70-98      -> b200zk_group_msm_g1 / _g2   (bases / scalars split by index range,
//                                                          one XYZZ partial per GPU, peer copies to GPU 0, point sum)
//   d_fft / d_ifft  dist-primitives/src/dfft/mod.rs:17-95 -> b200zk_group_ntt_fr        (four-step transform: column NTTs whose last
//                                                          pass stores straight into the owning peer's memory -- the kernel IS
//                                                          the all-to-all -- then row NTTs)
//   ext_wit::h      groth16/src/ext_wit.rs:16-101         -> b200zk_group_h_circom      (3 inverse + 3 forward sharded transforms)
//   prove::{A,B,C}  groth16/src/prove.rs:21-136 + sha256.rs:208-212 -> b200zk_group_groth16_prove (BASELINE config 5)
//   qap::qap + prove  groth16/src/qap.rs:44-91 + the above       -> b200zk_group_groth16_prove_r1cs_dev (the R1CS sharded by
//                                                          output slot: each GPU computes its column-layout slice of a, b, c)
// It is the C++ port of distributed_groth16_b200/parallel.py (the torch.distributed orchestration used by bench.py under
// torchrun): same layouts, same kernels (ntt.cu / msm.cu / prove.cu entry points), the NCCL collectives replaced by peer
// stores and cross-device events because everything lives in one address space.  The host thread only enqueues: all
// devices run concurrently, ordered by events; the only host synchronisation is the final read of the result.
//
// Distributed vectors use the "column layout" of parallel.py: for a length-N vector seen as rows x cols (row-major),
// GPU g of P owns columns [g cols/P, (g+1) cols/P), each stored contiguously: local[c][r] = x[r cols + g cols/P + c].
// A transform with (rows, cols) maps layout(cols) to layout(rows), so iNTT -> NTT chains need no redistribution.
#include "common.cuh"
#include "snarkjs_files.h"

#include <algorithm>

using namespace b200zk;

struct b200zk_group {
    int n = 0;
    std::vector<b200zk_ctx*> ctx;
    void* recv[2][8] = {};            // four-step receive buffers (2 alternate) on every device
    size_t recv_bytes = 0;
    int turn = 0;
    std::vector<cudaEvent_t> ev_col, ev_done;   // per device
    std::string last_error;
};

struct b200zk_group_pk {
    int n = 0;
    size_t n_vars = 0, n_inputs = 0, m = 0;
    unsigned log_m = 0;
    // per device: slices of the five queries (a / b_g1 / b_g2 rows [lo_g, hi_g) of n_vars; l rows of n_vars - n_inputs;
    // h in the column layout) and their fixed-base tables
    struct Shard {
        size_t v0 = 0, v1 = 0, l0 = 0, l1 = 0, hn = 0;
        void* q[5] = {};              // a, b_g1, b_g2, l, h
        void* tab[5] = {};
        unsigned tab_c[5] = {};
    };
    std::vector<Shard> shard;
    b200zk_pk* pk0 = nullptr;         // device 0: vk points for the final assembly
    size_t table_bytes = 0;
    const b200zk_group* owner = nullptr;
};

struct b200zk_group_r1cs {
    const b200zk_group* owner = nullptr;
    size_t nc = 0, n_inputs = 0, n_vars = 0, m = 0;
    unsigned log_m = 0;
    // per device: A and B (k = 0, 1) in CSR form over the m / P output slots of its column-layout slice, Montgomery values
    struct Shard {
        void* ptr[2] = {};
        void* col[2] = {};
        void* val[2] = {};
    };
    std::vector<Shard> shard;
};

// A snarkjs Groth16 zkey resident on a group (b200zk_group_zkey_load): the sharded proving key, and per device one allocation
// csr[g] behind A and B of its column-layout slice, row_ptr (2 loc + 1 entries: A's rows at [0, loc], B's at [loc, 2 loc])
// then val then col, exactly b200zk_zkey's layout.  mats[g] views it as b200zk_group_r1cs shards (which own nothing here).
struct b200zk_group_zkey {
    const b200zk_group* owner = nullptr;
    b200zk_group_pk* pk = nullptr;
    size_t n_vars = 0, n_public = 0, domain_size = 0, num_constraints = 0;
    std::vector<void*> csr;
    std::vector<b200zk_group_r1cs::Shard> mats;
};

namespace {

// the group calls hop between devices; the caller's current device (which frameworks such as torch cache) is restored on exit
struct DeviceGuard {
    int prev = -1;
    DeviceGuard() { if (cudaGetDevice(&prev) != cudaSuccess) prev = -1; }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

int gerr(b200zk_group* g, int code, const std::string& msg) {
    if (g) g->last_error = msg;
    return code;
}
int gfrom(b200zk_group* g, int rank, int rc) {
    if (rc != B200ZK_OK && g) g->last_error = "device " + std::to_string(g->ctx[rank]->device) + ": " + g->ctx[rank]->last_error;
    return rc;
}

// The prologue of every b200zk_group_* entry that works on the devices: a null group is refused, the caller's current device
// is restored on return, and slot 0 of every device is held for the whole call, taken in rank order (the same order
// everywhere: no deadlock).
template <class Body>
int with_group(b200zk_group* grp, Body&& body) {
    DeviceGuard dev_guard;
    if (!grp) return B200ZK_ERR_ARG;
    std::vector<std::unique_lock<std::mutex>> locks;
    for (int g = 0; g < grp->n; ++g) locks.emplace_back(grp->ctx[g]->slots[0].mu);
    return body();
}

// body(ctx, slot 0) of rank g with its device current.  body's errors are context errors (the message in ctx->last_error)
// and reach the group as "device N: <message>".
template <class Body>
int on_device(b200zk_group* grp, int g, Body&& body) {
    b200zk_ctx* ctx = grp->ctx[g];
    const cudaError_t e = cudaSetDevice(ctx->device);
    if (e != cudaSuccess) {
        char b[512];
        snprintf(b, sizeof(b), "CUDA error %s at %s:%d (cudaSetDevice(ctx->device))", cudaGetErrorString(e), __FILE__, __LINE__);
        return gerr(grp, e == cudaErrorMemoryAllocation ? B200ZK_ERR_OOM : B200ZK_ERR_CUDA, b);
    }
    return gfrom(grp, g, body(ctx, ctx->slots[0]));
}

// body(g, ctx, slot 0) on every rank in order, up to the first failure
template <class Body>
int each_device(b200zk_group* grp, Body&& body) {
    for (int g = 0; g < grp->n; ++g) {
        const int rc = on_device(grp, g, [&](b200zk_ctx* ctx, Slot& sl) { return body(g, ctx, sl); });
        if (rc) return rc;
    }
    return B200ZK_OK;
}

// out[c][r] = in[r][c] for an R x C matrix of T (Fr: 32 B, G1 point: 64 B, G2 point: 128 B)
template <class T>
__global__ void k_transpose(const T* in, T* out, uint32_t R, uint32_t C) {
    __shared__ T tile[16][17];
    const uint32_t c = blockIdx.x * 16 + threadIdx.x, r = blockIdx.y * 16 + threadIdx.y;
    if (r < R && c < C) tile[threadIdx.y][threadIdx.x] = in[(size_t)r * C + c];
    __syncthreads();
    const uint32_t oc = blockIdx.x * 16 + threadIdx.y, orow = blockIdx.y * 16 + threadIdx.x;   // out is C x R
    if (oc < C && orow < R) out[(size_t)oc * R + orow] = tile[threadIdx.x][threadIdx.y];
}
struct Blob32 { uint4 v[2]; };
struct Blob64 { uint4 v[4]; };
struct Blob128 { uint4 v[8]; };

template <class T>
int transpose_dev(b200zk_ctx* ctx, cudaStream_t st, const void* in, void* out, size_t R, size_t C) {
    return launch(ctx, st, "transpose", k_transpose<T>, dim3((unsigned)((C + 15) / 16), (unsigned)((R + 15) / 16)), dim3(16, 16), 0,
                  reinterpret_cast<const T*>(in), reinterpret_cast<T*>(out), (uint32_t)R, (uint32_t)C);
}

void split_log(unsigned log_n, unsigned* log_rows, unsigned* log_cols) {
    *log_rows = (log_n + 1) / 2;
    *log_cols = log_n / 2;
}

// every device's stream waits until all devices have passed `ev[g]` (recorded on their streams just before)
int cross_barrier(b200zk_group* grp, std::vector<cudaEvent_t>& ev) {
    int rc = each_device(grp, [&](int g, b200zk_ctx* ctx, Slot& sl) -> int {
        B2_CUDA_OK(ctx, cudaEventRecord(ev[g], sl.stream));
        return B200ZK_OK;
    });
    if (rc) return rc;
    return each_device(grp, [&](int g, b200zk_ctx* ctx, Slot& sl) -> int {
        for (int o = 0; o < grp->n; ++o)
            if (o != g) B2_CUDA_OK(ctx, cudaStreamWaitEvent(sl.stream, ev[o], 0));
        return B200ZK_OK;
    });
}

int ensure_recv(b200zk_group* grp, size_t bytes) {
    if (bytes <= grp->recv_bytes) return B200ZK_OK;
    int rc = each_device(grp, [&](int g, b200zk_ctx* ctx, Slot&) -> int {
        B2_CUDA_OK(ctx, cudaDeviceSynchronize());
        for (int b = 0; b < 2; ++b) {
            if (grp->recv[b][g]) cudaFree(grp->recv[b][g]);
            grp->recv[b][g] = nullptr;
            B2_CUDA_OK(ctx, cudaMalloc(&grp->recv[b][g], bytes));
        }
        return B200ZK_OK;
    });
    if (rc) return rc;
    grp->recv_bytes = bytes;
    return B200ZK_OK;
}

// One sharded four-step transform (parallel.sharded_ntt_p2p).  in[g]: (cols / P) x rows on device g; out[g]: (rows / P) x cols.
// shift_log_m != 0 (inverse transforms of the h pipeline): output coefficient j is also multiplied by w_2m^j.
int sharded_ntt(b200zk_group* grp, Fr* const* in, Fr* const* out, unsigned log_rows, unsigned log_cols, bool inverse, unsigned shift_log_m) {
    const int P = grp->n;
    const size_t rows = (size_t)1 << log_rows, cols = (size_t)1 << log_cols;
    if (rows % P || cols % P) return gerr(grp, B200ZK_ERR_ARG, "rows and cols of the four-step split must be divisible by the number of GPUs");
    const size_t cg = cols / P, rl = rows / P;
    int rc = ensure_recv(grp, rl * cols * sizeof(Fr));
    if (rc) return rc;
    const int b = grp->turn;
    grp->turn ^= 1;
    rc = each_device(grp, [&](int g, b200zk_ctx* ctx, Slot& sl) {
        return fourstep_cols_p2p_dev(ctx, sl, in[g], grp->recv[b], (unsigned)P, log_rows, ceil_log2(cg), log_rows + log_cols, (uint64_t)g * cg,
                                     inverse);
    });
    if (rc) return rc;
    rc = cross_barrier(grp, grp->ev_col);          // all column kernels (= all peer stores) are complete
    if (rc) return rc;
    return each_device(grp, [&](int g, b200zk_ctx* ctx, Slot& sl) {
        const Fr* rows_in = reinterpret_cast<const Fr*>(grp->recv[b][g]);
        if (!shift_log_m) return ntt_dev(ctx, sl, rows_in, out[g], log_cols, inverse, false, (unsigned)rl);
        return ntt_batched_post_dev(ctx, sl, rows_in, out[g], log_cols, (unsigned)rl, inverse, shift_log_m + 1, true, (uint64_t)g * rl, 0, 1, rows);
    });
}

// host vector (natural order, N = rows x cols row-major) -> column layout on the devices: a strided H2D copy of the
// device's column slab (rows x cg) followed by an on-device transpose to cg x rows
int scatter_columns(b200zk_group* grp, const void* host, size_t rows, size_t cols, Fr* const* d_tmp, Fr* const* d_out) {
    const size_t cg = cols / grp->n;
    return each_device(grp, [&](int g, b200zk_ctx* ctx, Slot& sl) -> int {
        B2_CUDA_OK(ctx, cudaMemcpy2DAsync(d_tmp[g], cg * sizeof(Fr), reinterpret_cast<const char*>(host) + g * cg * sizeof(Fr), cols * sizeof(Fr),
                                          cg * sizeof(Fr), rows, cudaMemcpyHostToDevice, sl.stream));
        return transpose_dev<Blob32>(ctx, sl.stream, d_tmp[g], d_out[g], rows, cg);
    });
}
// column layout (cg x rows per device) -> host natural order
int gather_columns(b200zk_group* grp, void* host, size_t rows, size_t cols, Fr* const* d_in, Fr* const* d_tmp) {
    const size_t cg = cols / grp->n;
    return each_device(grp, [&](int g, b200zk_ctx* ctx, Slot& sl) -> int {
        B2_TRY(transpose_dev<Blob32>(ctx, sl.stream, d_in[g], d_tmp[g], cg, rows));
        B2_CUDA_OK(ctx, cudaMemcpy2DAsync(reinterpret_cast<char*>(host) + g * cg * sizeof(Fr), cols * sizeof(Fr), d_tmp[g], cg * sizeof(Fr),
                                          cg * sizeof(Fr), rows, cudaMemcpyDeviceToHost, sl.stream));
        return B200ZK_OK;
    });
}

int sync_all(b200zk_group* grp) {
    return each_device(grp, [&](int, b200zk_ctx* ctx, Slot& sl) -> int {
        B2_CUDA_OK(ctx, cudaStreamSynchronize(sl.stream));
        return B200ZK_OK;
    });
}

// Device 0's slot-0 stream copies the first `bytes` of every rank g's slot-0 result buffer (`small`) to dst + g * bytes,
// behind ev_done[g], which rank g recorded once it wrote them.  Device 0 is current.
int gather_on_device0(b200zk_group* grp, size_t bytes, char* dst) {
    b200zk_ctx* c0 = grp->ctx[0];
    cudaStream_t st = c0->slots[0].stream;
    for (int g = 0; g < grp->n; ++g) {
        if (g) B2_CUDA_OK(c0, cudaStreamWaitEvent(st, grp->ev_done[g], 0));
        B2_CUDA_OK(c0, cudaMemcpyPeerAsync(dst + g * bytes, c0->device, grp->ctx[g]->slots[0].small.p, grp->ctx[g]->device, bytes, st));
    }
    return B200ZK_OK;
}

// balanced index-range split
size_t cut(size_t n, int g, int P) { return (size_t)(((unsigned __int128)n * (unsigned)g) / (unsigned)P); }

template <int G2>
int group_msm(b200zk_group* grp, const uint64_t* bases, size_t n_bases, const uint64_t* scalars, size_t n_scalars, uint64_t* out_affine,
              int* out_is_inf) {
    return with_group(grp, [&]() -> int {
        if (!out_affine || !out_is_inf) return B200ZK_ERR_ARG;
        if (n_bases != n_scalars) return gerr(grp, B200ZK_ERR_LENGTH, std::to_string(n_bases < n_scalars ? n_bases : n_scalars));
        const size_t n = n_bases;
        if (n && (!bases || !scalars)) return gerr(grp, B200ZK_ERR_ARG, "null input");
        const size_t PB = G2 ? 128 : 64, XB = G2 ? 256 : 128;
        const int P = grp->n;
        // every device: stage its slice (scalars on the compute stream, bases on the copy stream behind the sort phases), MSM
        int rc = each_device(grp, [&](int g, b200zk_ctx* ctx, Slot& sl) -> int {
            const size_t lo = cut(n, g, P), cnt = cut(n, g + 1, P) - lo;
            B2_CUDA_OK(ctx, sl.small.reserve(4096));
            // this device's index range, staged in parts behind its own bucket kernels (api.cu, msm_staged_dev)
            B2_TRY(msm_staged_dev(ctx, sl, G2, reinterpret_cast<const char*>(bases) + lo * PB, reinterpret_cast<const char*>(scalars) + lo * 32,
                                  cnt, sl.small.p, false));
            B2_CUDA_OK(ctx, cudaEventRecord(grp->ev_done[g], sl.stream));
            return B200ZK_OK;
        });
        if (rc) return rc;
        // partials -> device 0 (peer copies), sum, normalise
        uint64_t host[17];
        rc = on_device(grp, 0, [&](b200zk_ctx* c0, Slot& s0) -> int {
            char* sm = reinterpret_cast<char*>(s0.small.p);
            char* gathered = sm + 1024;                               // P x XB <= 2 KB
            B2_TRY(gather_on_device0(grp, XB, gathered));
            B2_TRY(G2 ? g2_sum_dev(c0, s0, gathered, P, sm + 3584) : g1_sum_dev(c0, s0, gathered, P, sm + 3584));
            B2_CUDA_OK(c0, cudaMemcpyAsync(host, sm + 3584, PB + 8, cudaMemcpyDeviceToHost, s0.stream));
            B2_CUDA_OK(c0, cudaStreamSynchronize(s0.stream));
            return B200ZK_OK;
        });
        if (!rc) rc = sync_all(grp);
        // the host buffers are free again once every copy stream drained
        if (!rc) rc = each_device(grp, [&](int, b200zk_ctx* ctx, Slot& sl) -> int {
            B2_CUDA_OK(ctx, cudaStreamSynchronize(sl.copy_stream));
            return B200ZK_OK;
        });
        if (rc) return rc;
        memcpy(out_affine, host, PB);
        *out_is_inf = (int)host[PB / 8];
        return B200ZK_OK;
    });
}

// The column-layout workspace of an h or proof computation, carved from slot 0's io_a on every device g: a, b, c and the
// temporaries t1, t2 (t2 ends up holding h), loc Fr each, then the caller's tail of z at z[g].
struct Columns {
    std::vector<Fr*> a, b, c, t1, t2, z;
    explicit Columns(int P) : a(P), b(P), c(P), t1(P), t2(P), z(P) {}
};

// tail(g): the Fr that follow the five vectors on device g
template <class Tail>
int carve_columns(b200zk_group* grp, size_t loc, Tail&& tail, Columns& w) {
    return each_device(grp, [&](int g, b200zk_ctx* ctx, Slot& sl) -> int {
        B2_CUDA_OK(ctx, sl.io_a.reserve((5 * loc + tail(g)) * sizeof(Fr)));
        Fr* p = reinterpret_cast<Fr*>(sl.io_a.p);
        w.a[g] = p; w.b[g] = p + loc; w.c[g] = p + 2 * loc; w.t1[g] = p + 3 * loc; w.t2[g] = p + 4 * loc; w.z[g] = p + 5 * loc;
        return B200ZK_OK;
    });
}

// the h pipeline on w.a, w.b, w.c, already in the column layout ((cols / P) x rows per device); h lands in w.t2
int sharded_h(b200zk_group* grp, const Columns& w, unsigned log_m) {
    unsigned log_rows, log_cols;
    split_log(log_m, &log_rows, &log_cols);
    // a, b, c are transformed in place (through t1): coef = iNTT + shift, ev = NTT
    for (const std::vector<Fr*>* v : {&w.a, &w.b, &w.c}) {
        int rc = sharded_ntt(grp, v->data(), w.t1.data(), log_rows, log_cols, true, log_m);
        if (rc) return rc;
        rc = sharded_ntt(grp, w.t1.data(), v->data(), log_cols, log_rows, false, 0);
        if (rc) return rc;
    }
    const size_t local = ((size_t)1 << log_m) / grp->n;
    return each_device(grp, [&](int g, b200zk_ctx* ctx, Slot& sl) { return mul_sub_dev(ctx, sl, w.a[g], w.b[g], w.c[g], w.t2[g], local); });
}

// Slot j of GPU g's column-layout slice holds global row (j mod rows) cols + g cols / P + j div rows (local[c rows + r] =
// x[r cols + g cg + c]); qap.cu's global_row is the device twin
size_t slot_row(size_t j, unsigned log_rows, unsigned log_cols, int P, int g) {
    return ColumnLayout{log_rows, log_cols, log_cols - ceil_log2((size_t)P)}.row((uint32_t)g, j);
}

// The m / P + 1 entries of GPU g's slice CSR row_ptr from the global one (num_constraints + 1 entries; global rows >=
// num_constraints have no terms).  Host only.
void fill_local_row_ptr(const uint32_t* row_ptr, size_t nc, unsigned log_rows, unsigned log_cols, int P, int g, uint32_t* lptr) {
    const size_t n = ((size_t)1 << (log_rows + log_cols)) / P;
    lptr[0] = 0;
    for (size_t j = 0; j < n; ++j) {
        const size_t i = slot_row(j, log_rows, log_cols, P, g);
        lptr[j + 1] = lptr[j] + (i < nc ? row_ptr[i + 1] - row_ptr[i] : 0);
    }
}

// A CSR matrix from outside the program: row_ptr starts at 0 and never decreases, every column is < n_vars (the QAP kernel
// gathers z[col] unchecked)
int check_csr(b200zk_group* grp, const char* name, const uint32_t* row_ptr, const uint32_t* col, const uint64_t* val, size_t nc,
              size_t n_vars) {
    if (row_ptr[0] != 0) return gerr(grp, B200ZK_ERR_ARG, std::string("matrix ") + name + ": row_ptr[0] is " + std::to_string(row_ptr[0]) + ", not 0");
    for (size_t i = 0; i < nc; ++i)
        if (row_ptr[i + 1] < row_ptr[i])
            return gerr(grp, B200ZK_ERR_ARG, std::string("matrix ") + name + ": row_ptr decreases at constraint " + std::to_string(i));
    const size_t nnz = row_ptr[nc];
    if (nnz && (!col || !val)) return gerr(grp, B200ZK_ERR_ARG, std::string("matrix ") + name + ": null col or val with terms");
    for (size_t i = 0; i < nc; ++i)
        for (size_t k = row_ptr[i]; k < row_ptr[i + 1]; ++k)
            if (col[k] >= n_vars)
                return gerr(grp, B200ZK_ERR_ARG, std::string("matrix ") + name + ": term " + std::to_string(k) + " (constraint " + std::to_string(i) +
                                                     ") has column " + std::to_string(col[k]) + " >= n_vars " + std::to_string(n_vars));
    return B200ZK_OK;
}

// The prover from a, b, c already in w's column layout on the devices: sharded h, five partial MSMs per device, peer copies
// of the partials to device 0, sums and assembly there.  zq[g] = z[v0, v1) and zl[g] = z[n_inputs + l0, n_inputs + l1) of
// device g's key shard.  The caller holds the slot locks and has reserved every device's small buffer (4 KB).
int prove_columns(b200zk_group* grp, const b200zk_group_pk* pk, const Columns& w, const Fr* const* zq, const Fr* const* zl, const uint64_t r[4],
                  const uint64_t s[4], uint8_t proof_out[128]) {
    const int P = grp->n;
    const bool need_b1 = (r[0] | r[1] | r[2] | r[3]) != 0;
    int rc = sharded_h(grp, w, pk->log_m);
    if (rc) return rc;
    // partial MSMs: small[0..16) A, [16..32) L, [32..48) H, [48..64) B1 (u64 words), [64..96) B2
    rc = each_device(grp, [&](int g, b200zk_ctx* ctx, Slot& sl) -> int {
        const b200zk_group_pk::Shard& S = pk->shard[g];
        char* sm = reinterpret_cast<char*>(sl.small.p);
        auto msm = [&](int k, const Fr* scalars, size_t n, void* out) {
            return query_msm(ctx, sl, k, S.q[k], S.tab, S.tab_c, scalars, n, out, 0);
        };
        B2_TRY(msm(2, zq[g], S.v1 - S.v0, sm + 512));                    // the G2 MSM first: the longest
        B2_TRY(msm(0, zq[g], S.v1 - S.v0, sm + 0));
        B2_TRY(msm(3, zl[g], S.l1 - S.l0, sm + 128));
        B2_TRY(msm(4, w.t2[g], S.hn, sm + 256));
        if (need_b1) B2_TRY(msm(1, zq[g], S.v1 - S.v0, sm + 384));
        else B2_CUDA_OK(ctx, cudaMemsetAsync(sm + 384, 0, 128, sl.stream));
        B2_CUDA_OK(ctx, cudaEventRecord(grp->ev_done[g], sl.stream));
        return B200ZK_OK;
    });
    if (rc) return rc;
    // gather on device 0, add up, assemble (the sharded MSMs ran over index 0 too: z[0] = 1 makes a_query[0] z[0] the term the
    // reference's driver adds, sha256.rs:208-212 -> include_zero_terms = 0)
    rc = on_device(grp, 0, [&](b200zk_ctx* c0, Slot& s0) -> int {
        B2_CUDA_OK(c0, s0.io_b.reserve((size_t)(P + 1) * 768));
        char* gathered = reinterpret_cast<char*>(s0.io_b.p);
        char* tot = gathered + (size_t)P * 768;
        B2_TRY(gather_on_device0(grp, 768, gathered));
        for (int k = 0; k < 4; ++k) B2_TRY(xyzz_sum_dev(c0, s0, 0, gathered + k * 128, P, 6, tot + k * 128));      // stride: 768 B = 6 G1 XYZZ
        B2_TRY(xyzz_sum_dev(c0, s0, 1, gathered + 512, P, 3, tot + 512));                                          // 3 G2 XYZZ
        return assemble_dev(c0, s0, pk->pk0, tot, tot + 512, tot + 128, tot + 256, need_b1 ? tot + 384 : nullptr, r, s, 0, proof_out);
    });
    if (rc) return rc;
    return sync_all(grp);
}

// b200zk_group_groth16_prove_r1cs_dev after its checks, on A and B sharded as mats[g] (b200zk_group_r1cs's layout): the full
// witness on device 0 is peer-copied to every other device, each device computes its column-layout slice of a, b, c, then
// prove_columns.  z0(c0, s0, tail, &z) gives device 0's witness on its slot-0 stream: the caller's, or one it writes into
// `tail`, n_vars Fr that are reserved on device 0 only when z0_in_tail.
template <class Z0>
int prove_r1cs_columns(b200zk_group* grp, const b200zk_group_pk* pk, const std::vector<b200zk_group_r1cs::Shard>& mats, size_t nc,
                       size_t n_inputs, bool z0_in_tail, Z0&& z0, const uint64_t r[4], const uint64_t s[4], uint8_t proof_out[128]) {
    const int P = grp->n;
    unsigned log_rows, log_cols;
    split_log(pk->log_m, &log_rows, &log_cols);
    const size_t cg = ((size_t)1 << log_cols) / P, loc = pk->m / P, zbytes = pk->n_vars * sizeof(Fr);
    // the tail (devices >= 1, and device 0 for z0_in_tail): a copy of z.  a, b, c are written by the mat-vec.
    Columns w(P);
    int rc = carve_columns(grp, loc, [&](int g) { return g || z0_in_tail ? pk->n_vars : 0; }, w);
    // every other device's copy of z waits for the point where device 0's stream holds it
    const Fr* z0p = nullptr;
    if (!rc) rc = on_device(grp, 0, [&](b200zk_ctx* c0, Slot& s0) -> int {
        B2_TRY(z0(c0, s0, w.z[0], &z0p));
        B2_CUDA_OK(c0, cudaEventRecord(grp->ev_done[0], s0.stream));
        return B200ZK_OK;
    });
    std::vector<const Fr*> zq(P), zl(P);
    if (!rc) rc = each_device(grp, [&](int g, b200zk_ctx* ctx, Slot& sl) -> int {
        const b200zk_group_pk::Shard& S = pk->shard[g];
        const b200zk_group_r1cs::Shard& Q = mats[g];
        B2_CUDA_OK(ctx, sl.small.reserve(4096));
        const Fr* z = z0p;
        if (g) {
            B2_CUDA_OK(ctx, cudaStreamWaitEvent(sl.stream, grp->ev_done[0], 0));
            B2_CUDA_OK(ctx, cudaMemcpyPeerAsync(w.z[g], ctx->device, z0p, grp->ctx[0]->device, zbytes, sl.stream));
            z = w.z[g];
        }
        zq[g] = z + S.v0;
        zl[g] = z + n_inputs + S.l0;
        return qap_slots_dev(ctx, sl, Q.ptr[0], Q.col[0], Q.val[0], Q.ptr[1], Q.col[1], Q.val[1], nc, n_inputs, z, log_rows, log_cols,
                             (size_t)g * cg, loc, w.a[g], w.b[g], w.c[g]);
    });
    if (rc) return rc;
    return prove_columns(grp, pk, w, zq.data(), zl.data(), r, s, proof_out);
}

// The body of b200zk_group_pk_upload (the caller holds the slot locks), with the table window of b200zk_zkey_load: 0 = the
// automatic policy, 0xFFFFFFFF = no tables, else c on every shard.  The queries are host bytes.
int group_pk_build(b200zk_group* grp, const void* a_query, const void* b_g1_query, const void* b_g2_query, const void* l_query,
                   const void* h_query, size_t n_vars, size_t n_inputs, size_t m, const uint64_t* vk_points, unsigned table_window,
                   b200zk_group_pk** out) {
    if (n_vars == 0 || n_inputs == 0 || n_inputs > n_vars) return gerr(grp, B200ZK_ERR_ARG, "need 1 <= n_inputs <= n_vars");
    if (m == 0 || (m & (m - 1))) return gerr(grp, B200ZK_ERR_DOMAIN, "h_query length must be a power of two");
    const int P = grp->n;
    const unsigned log_m = ceil_log2(m);
    unsigned log_rows, log_cols;
    split_log(log_m, &log_rows, &log_cols);
    const size_t rows = (size_t)1 << log_rows, cols = (size_t)1 << log_cols;
    if (cols < (size_t)P) return gerr(grp, B200ZK_ERR_ARG, "domain too small for this many GPUs");
    b200zk_group_pk* pk = new b200zk_group_pk();
    pk->n = P; pk->n_vars = n_vars; pk->n_inputs = n_inputs; pk->m = m; pk->log_m = log_m; pk->owner = grp;
    pk->shard.resize(P);
    const size_t n_aux = n_vars - n_inputs;
    // table_window as b200zk_pk_precompute's c: 0 is the automatic policy, which B200ZK_PK_TABLES=0 turns off
    const bool want_tables = table_window != 0xFFFFFFFFu && (table_window != 0 || pk_tables_enabled());
    int rc = each_device(grp, [&](int g, b200zk_ctx* ctx, Slot& sl) -> int {
        b200zk_group_pk::Shard& S = pk->shard[g];
        S.v0 = cut(n_vars, g, P); S.v1 = cut(n_vars, g + 1, P);
        S.l0 = cut(n_aux, g, P); S.l1 = cut(n_aux, g + 1, P);
        S.hn = m / P;
        const size_t cnt[5] = {S.v1 - S.v0, S.v1 - S.v0, S.v1 - S.v0, S.l1 - S.l0, S.hn};
        const size_t psz[5] = {64, 64, 128, 64, 64};
        const void* src[4] = {reinterpret_cast<const char*>(a_query) + S.v0 * 64, reinterpret_cast<const char*>(b_g1_query) + S.v0 * 64,
                              reinterpret_cast<const char*>(b_g2_query) + S.v0 * 128,
                              l_query ? reinterpret_cast<const char*>(l_query) + S.l0 * 64 : nullptr};
        for (int k = 0; k < 5; ++k) {
            if (cudaMalloc(&S.q[k], cnt[k] * psz[k] + 16) != cudaSuccess) return set_error(ctx, B200ZK_ERR_OOM, "proving-key shard allocation failed");
            if (k < 4 && cnt[k] && cudaMemcpyAsync(S.q[k], src[k], cnt[k] * psz[k], cudaMemcpyHostToDevice, sl.stream) != cudaSuccess)
                return set_error(ctx, B200ZK_ERR_CUDA, "proving-key upload failed");
        }
        {   // h_query in the column layout of the h this device will compute: local[c][r] = h_query[r cols + g cg + c]
            const size_t cg = cols / P;
            if (sl.io_a.reserve(S.hn * 64) != cudaSuccess) return set_error(ctx, B200ZK_ERR_OOM, "staging allocation failed");
            if (cudaMemcpy2DAsync(sl.io_a.p, cg * 64, reinterpret_cast<const char*>(h_query) + g * cg * 64, cols * 64, cg * 64, rows,
                                  cudaMemcpyHostToDevice, sl.stream) != cudaSuccess)
                return set_error(ctx, B200ZK_ERR_CUDA, "h_query upload failed");
            B2_TRY(transpose_dev<Blob64>(ctx, sl.stream, sl.io_a.p, S.q[4], rows, cg));
        }
        if (want_tables) {          // B200ZK_PK_TABLE_WINDOW is not read here
            size_t bytes = 0;
            B2_TRY(pk_tables_build(ctx, sl, S.q, cnt, table_window, S.tab, S.tab_c, &bytes));
            pk->table_bytes += bytes;
        }
        return B200ZK_OK;
    });
    // device 0 keeps the vk points for the final assembly (queries of the tiny pk object are never read: include_zero_terms = 0)
    if (!rc) rc = on_device(grp, 0, [&](b200zk_ctx* c0, Slot& s0) -> int {
        pk->pk0 = new b200zk_pk();
        pk->pk0->n_vars = n_vars; pk->pk0->n_inputs = n_inputs; pk->pk0->m = m;
        if (cudaMalloc(&pk->pk0->vk, 56 * 8) != cudaSuccess || cudaMemcpyAsync(pk->pk0->vk, vk_points, 56 * 8, cudaMemcpyHostToDevice, s0.stream) != cudaSuccess)
            return set_error(c0, B200ZK_ERR_CUDA, "vk upload failed");
        return B200ZK_OK;
    });
    if (!rc) rc = sync_all(grp);
    if (rc) {
        b200zk_group_pk_free(grp, pk);
        return rc;
    }
    *out = pk;
    return B200ZK_OK;
}

}  // namespace

extern "C" {

int b200zk_group_create(const int* device_ids, int n_dev, b200zk_group** out) {
    DeviceGuard dev_guard;
    if (!device_ids || !out || n_dev < 1 || n_dev > 8 || (n_dev & (n_dev - 1))) return B200ZK_ERR_ARG;
    b200zk_group* grp = new b200zk_group();
    grp->n = n_dev;
    for (int g = 0; g < n_dev; ++g) {
        b200zk_ctx* c = nullptr;
        int rc = b200zk_ctx_create(device_ids[g], &c);
        if (rc) { b200zk_group_destroy(grp); return rc; }
        grp->ctx.push_back(c);
    }
    for (int g = 0; g < n_dev; ++g) {
        cudaSetDevice(device_ids[g]);
        for (int o = 0; o < n_dev; ++o) {
            if (o == g || device_ids[o] == device_ids[g]) continue;
            int can = 0;
            cudaDeviceCanAccessPeer(&can, device_ids[g], device_ids[o]);
            if (!can) { b200zk_group_destroy(grp); return B200ZK_ERR_CUDA; }
            cudaError_t e = cudaDeviceEnablePeerAccess(device_ids[o], 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { b200zk_group_destroy(grp); return B200ZK_ERR_CUDA; }
            cudaGetLastError();
        }
        cudaEvent_t e1 = nullptr, e2 = nullptr;
        if (cudaEventCreateWithFlags(&e1, cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&e2, cudaEventDisableTiming) != cudaSuccess) {
            b200zk_group_destroy(grp);
            return B200ZK_ERR_CUDA;
        }
        grp->ev_col.push_back(e1);
        grp->ev_done.push_back(e2);
    }
    *out = grp;
    return B200ZK_OK;
}

void b200zk_group_destroy(b200zk_group* grp) {
    DeviceGuard dev_guard;
    if (!grp) return;
    for (size_t g = 0; g < grp->ctx.size(); ++g) {
        cudaSetDevice(grp->ctx[g]->device);
        cudaDeviceSynchronize();
        for (int b = 0; b < 2; ++b) if (grp->recv[b][g]) cudaFree(grp->recv[b][g]);
        if (g < grp->ev_col.size()) cudaEventDestroy(grp->ev_col[g]);
        if (g < grp->ev_done.size()) cudaEventDestroy(grp->ev_done[g]);
    }
    for (b200zk_ctx* c : grp->ctx) b200zk_ctx_destroy(c);
    delete grp;
}

int b200zk_group_size(const b200zk_group* grp) { return grp ? grp->n : 0; }
b200zk_ctx* b200zk_group_ctx(b200zk_group* grp, int rank) { return grp && rank >= 0 && rank < grp->n ? grp->ctx[rank] : nullptr; }
const char* b200zk_group_last_error(const b200zk_group* grp) { return grp ? grp->last_error.c_str() : "null group"; }

int b200zk_group_msm_g1(b200zk_group* grp, const uint64_t* bases, size_t n_bases, const uint64_t* scalars, size_t n_scalars,
                        uint64_t out_affine[8], int* out_is_inf) {
    return group_msm<0>(grp, bases, n_bases, scalars, n_scalars, out_affine, out_is_inf);
}
int b200zk_group_msm_g2(b200zk_group* grp, const uint64_t* bases, size_t n_bases, const uint64_t* scalars, size_t n_scalars,
                        uint64_t out_affine[16], int* out_is_inf) {
    return group_msm<1>(grp, bases, n_bases, scalars, n_scalars, out_affine, out_is_inf);
}

int b200zk_group_ntt_fr(b200zk_group* grp, uint64_t* data, unsigned log_n, int inverse) {
    return with_group(grp, [&]() -> int {
        if (!data) return B200ZK_ERR_ARG;
        if (log_n > 28) return gerr(grp, B200ZK_ERR_DOMAIN, "log n > 28");
        const int P = grp->n;
        unsigned log_rows, log_cols;
        split_log(log_n, &log_rows, &log_cols);
        const size_t rows = (size_t)1 << log_rows, cols = (size_t)1 << log_cols, N = (size_t)1 << log_n;
        if (cols < (size_t)P) return gerr(grp, B200ZK_ERR_ARG, "transform too small for this many GPUs");
        std::vector<Fr*> bufA(P), bufB(P);
        int rc = each_device(grp, [&](int g, b200zk_ctx* ctx, Slot& sl) -> int {
            B2_CUDA_OK(ctx, sl.io_a.reserve(2 * (N / P) * sizeof(Fr)));
            bufA[g] = reinterpret_cast<Fr*>(sl.io_a.p);
            bufB[g] = bufA[g] + N / P;
            return B200ZK_OK;
        });
        if (!rc) rc = scatter_columns(grp, data, rows, cols, bufB.data(), bufA.data());                    // layout(cols) in A
        if (!rc) rc = sharded_ntt(grp, bufA.data(), bufB.data(), log_rows, log_cols, inverse != 0, 0);     // layout(rows) in B: (rows / P) x cols
        // X[k1 + rows k2] sits at bufB[g][k1 local][k2]: as a cols x rows row-major matrix X[k2][k1] the device owns columns k1
        if (!rc) rc = gather_columns(grp, data, cols, rows, bufB.data(), bufA.data());
        if (rc) return rc;
        return sync_all(grp);
    });
}

int b200zk_group_h_circom(b200zk_group* grp, const uint64_t* a, const uint64_t* b, const uint64_t* c, unsigned log_m, uint64_t* h_out) {
    return with_group(grp, [&]() -> int {
        if (!a || !b || !c || !h_out) return B200ZK_ERR_ARG;
        if (log_m + 1 > 28) return gerr(grp, B200ZK_ERR_DOMAIN, "2m exceeds the 2^28 subgroup (PolynomialDegreeTooLarge)");
        const int P = grp->n;
        unsigned log_rows, log_cols;
        split_log(log_m, &log_rows, &log_cols);
        const size_t rows = (size_t)1 << log_rows, cols = (size_t)1 << log_cols, m = (size_t)1 << log_m, loc = m / P;
        if (cols < (size_t)P) return gerr(grp, B200ZK_ERR_ARG, "domain too small for this many GPUs");
        Columns w(P);
        int rc = carve_columns(grp, loc, [](int) { return (size_t)0; }, w);
        if (!rc) rc = scatter_columns(grp, a, rows, cols, w.t1.data(), w.a.data());
        if (!rc) rc = scatter_columns(grp, b, rows, cols, w.t1.data(), w.b.data());
        if (!rc) rc = scatter_columns(grp, c, rows, cols, w.t1.data(), w.c.data());
        if (!rc) rc = sharded_h(grp, w, log_m);
        if (!rc) rc = gather_columns(grp, h_out, rows, cols, w.t2.data(), w.t1.data());
        if (rc) return rc;
        return sync_all(grp);
    });
}

// ---- sharded proving key + prove (BASELINE config 5) ------------------------------------------------------------------------
void b200zk_group_pk_free(b200zk_group* grp, b200zk_group_pk* pk) {
    DeviceGuard dev_guard;
    if (!pk) return;
    for (size_t g = 0; g < pk->shard.size(); ++g) {
        if (grp && g < grp->ctx.size()) cudaSetDevice(grp->ctx[g]->device);
        for (int k = 0; k < 5; ++k) {
            if (pk->shard[g].q[k]) cudaFree(pk->shard[g].q[k]);
            if (pk->shard[g].tab[k]) cudaFree(pk->shard[g].tab[k]);
        }
    }
    if (pk->pk0) b200zk_pk_free(grp ? grp->ctx[0] : nullptr, pk->pk0);
    delete pk;
}

int b200zk_group_pk_upload(b200zk_group* grp, const uint64_t* a_query, const uint64_t* b_g1_query, const uint64_t* b_g2_query,
                           const uint64_t* l_query, const uint64_t* h_query, size_t n_vars, size_t n_inputs, size_t m,
                           const uint64_t* vk_points, b200zk_group_pk** out) {
    return with_group(grp, [&]() -> int {
        if (!out || !a_query || !b_g1_query || !b_g2_query || !h_query || !vk_points) return B200ZK_ERR_ARG;
        return group_pk_build(grp, a_query, b_g1_query, b_g2_query, l_query, h_query, n_vars, n_inputs, m, vk_points, 0, out);
    });
}

size_t b200zk_group_pk_table_bytes(const b200zk_group_pk* pk) { return pk ? pk->table_bytes : 0; }

int b200zk_group_groth16_prove(b200zk_group* grp, const b200zk_group_pk* pk, const uint64_t* z, const uint64_t* a, const uint64_t* b,
                               const uint64_t* c, const uint64_t r[4], const uint64_t s[4], uint8_t proof_out[128]) {
    return with_group(grp, [&]() -> int {
        if (!pk || !z || !a || !b || !c || !r || !s || !proof_out) return B200ZK_ERR_ARG;
        if (pk->n != grp->n) return gerr(grp, B200ZK_ERR_ARG, "proving key was sharded for a different group");
        const int P = grp->n;
        unsigned log_rows, log_cols;
        split_log(pk->log_m, &log_rows, &log_cols);
        const size_t rows = (size_t)1 << log_rows, cols = (size_t)1 << log_cols, loc = pk->m / P;
        // the tail: this device's rows of z, z[v0, v1) then z[n_inputs + l0, n_inputs + l1), and as many Fr again as the longer of the two
        Columns w(P);
        int rc = carve_columns(grp, loc, [&](int g) {
            const b200zk_group_pk::Shard& S = pk->shard[g];
            return (S.v1 - S.v0) + (S.l1 - S.l0) + std::max(S.v1 - S.v0, S.l1 - S.l0);
        }, w);
        std::vector<const Fr*> zq(P), zl(P);
        if (!rc) rc = each_device(grp, [&](int g, b200zk_ctx* ctx, Slot& sl) -> int {
            const b200zk_group_pk::Shard& S = pk->shard[g];
            B2_CUDA_OK(ctx, sl.small.reserve(4096));
            zq[g] = w.z[g];
            zl[g] = w.z[g] + (S.v1 - S.v0);
            B2_CUDA_OK(ctx, cudaMemcpyAsync(w.z[g], reinterpret_cast<const char*>(z) + S.v0 * 32, (S.v1 - S.v0) * 32, cudaMemcpyHostToDevice, sl.stream));
            B2_CUDA_OK(ctx, cudaMemcpyAsync(w.z[g] + (S.v1 - S.v0), reinterpret_cast<const char*>(z) + (pk->n_inputs + S.l0) * 32, (S.l1 - S.l0) * 32,
                                            cudaMemcpyHostToDevice, sl.stream));
            return B200ZK_OK;
        });
        if (!rc) rc = scatter_columns(grp, a, rows, cols, w.t1.data(), w.a.data());
        if (!rc) rc = scatter_columns(grp, b, rows, cols, w.t1.data(), w.b.data());
        if (!rc) rc = scatter_columns(grp, c, rows, cols, w.t1.data(), w.c.data());
        if (rc) return rc;
        return prove_columns(grp, pk, w, zq.data(), zl.data(), r, s, proof_out);
    });
}

// ---- R1CS sharded by output slot + prove from the witness on device 0 ---------------------------------------------------------
int b200zk_group_r1cs_local_row_ptr(const uint32_t* row_ptr, size_t num_constraints, unsigned log_m, int n_gpus, int rank,
                                    uint32_t* local_row_ptr) {
    if (!row_ptr || !local_row_ptr || n_gpus < 1 || n_gpus > 8 || (n_gpus & (n_gpus - 1)) || rank < 0 || rank >= n_gpus) return B200ZK_ERR_ARG;
    if (log_m > 27 || num_constraints > ((size_t)1 << log_m)) return B200ZK_ERR_DOMAIN;
    unsigned log_rows, log_cols;
    split_log(log_m, &log_rows, &log_cols);
    if (((size_t)1 << log_cols) < (size_t)n_gpus) return B200ZK_ERR_ARG;
    fill_local_row_ptr(row_ptr, num_constraints, log_rows, log_cols, n_gpus, rank, local_row_ptr);
    return B200ZK_OK;
}
void b200zk_group_r1cs_free(b200zk_group* grp, b200zk_group_r1cs* q) {
    DeviceGuard dev_guard;
    if (!q) return;
    for (size_t g = 0; g < q->shard.size(); ++g) {
        if (grp && g < grp->ctx.size()) cudaSetDevice(grp->ctx[g]->device);
        for (int k = 0; k < 2; ++k) {
            if (q->shard[g].ptr[k]) cudaFree(q->shard[g].ptr[k]);
            if (q->shard[g].col[k]) cudaFree(q->shard[g].col[k]);
            if (q->shard[g].val[k]) cudaFree(q->shard[g].val[k]);
        }
    }
    delete q;
}

int b200zk_group_r1cs_upload(b200zk_group* grp, const uint32_t* a_row_ptr, const uint32_t* a_col, const uint64_t* a_val,
                             const uint32_t* b_row_ptr, const uint32_t* b_col, const uint64_t* b_val, size_t num_constraints,
                             size_t num_inputs, size_t n_vars, unsigned log_m, int values_montgomery_depth, b200zk_group_r1cs** out) {
    return with_group(grp, [&]() -> int {
        if (!out || !a_row_ptr || !b_row_ptr) return B200ZK_ERR_ARG;
        *out = nullptr;
        if (log_m > 27) return gerr(grp, B200ZK_ERR_DOMAIN, "log_m > 27: 2m exceeds the 2^28 subgroup (PolynomialDegreeTooLarge)");
        const size_t m = (size_t)1 << log_m, nc = num_constraints;
        if (nc + num_inputs > m) return gerr(grp, B200ZK_ERR_DOMAIN, "num_constraints + num_inputs exceeds the domain size");
        if (num_inputs == 0 || num_inputs > n_vars) return gerr(grp, B200ZK_ERR_ARG, "need 1 <= num_inputs <= n_vars");
        const int P = grp->n;
        unsigned log_rows, log_cols;
        split_log(log_m, &log_rows, &log_cols);
        if (((size_t)1 << log_cols) < (size_t)P) return gerr(grp, B200ZK_ERR_ARG, "domain too small for this many GPUs");
        const uint32_t* row_ptr[2] = {a_row_ptr, b_row_ptr};
        const uint32_t* col[2] = {a_col, b_col};
        const uint64_t* val[2] = {a_val, b_val};
        for (int k = 0; k < 2; ++k) {
            int rc = check_csr(grp, k ? "B" : "A", row_ptr[k], col[k], val[k], nc, n_vars);
            if (rc) return rc;
        }
        b200zk_group_r1cs* q = new b200zk_group_r1cs();
        q->owner = grp; q->nc = nc; q->n_inputs = num_inputs; q->n_vars = n_vars; q->m = m; q->log_m = log_m;
        q->shard.resize(P);
        const size_t loc = m / P;
        std::vector<uint32_t> lptr(loc + 1), lcol;
        std::vector<uint64_t> lval;
        int rc = each_device(grp, [&](int g, b200zk_ctx* ctx, Slot& sl) -> int {
            b200zk_group_r1cs::Shard& S = q->shard[g];
            for (int k = 0; k < 2; ++k) {
                // the slice's rows in slot order, gathered once on the host (index and word copies only)
                fill_local_row_ptr(row_ptr[k], nc, log_rows, log_cols, P, g, lptr.data());
                const size_t nnz = lptr[loc];
                lcol.resize(nnz);
                lval.resize(nnz * 4);
                for (size_t j = 0; j < loc; ++j) {
                    const size_t i = slot_row(j, log_rows, log_cols, P, g);
                    if (i >= nc || row_ptr[k][i + 1] == row_ptr[k][i]) continue;
                    const size_t lo = row_ptr[k][i], n = row_ptr[k][i + 1] - lo;
                    memcpy(lcol.data() + lptr[j], col[k] + lo, n * sizeof(uint32_t));
                    memcpy(lval.data() + (size_t)lptr[j] * 4, val[k] + lo * 4, n * 32);
                }
                if (cudaMalloc(&S.ptr[k], (loc + 1) * sizeof(uint32_t)) != cudaSuccess || cudaMalloc(&S.col[k], nnz * sizeof(uint32_t) + 16) != cudaSuccess ||
                    cudaMalloc(&S.val[k], nnz * 32 + 16) != cudaSuccess)
                    return set_error(ctx, B200ZK_ERR_OOM, "constraint-matrix shard allocation failed");
                // pageable sources: each copy has consumed its source when the call returns, so the host vectors can be refilled
                if (cudaMemcpyAsync(S.ptr[k], lptr.data(), (loc + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, sl.stream) != cudaSuccess ||
                    (nnz && cudaMemcpyAsync(S.col[k], lcol.data(), nnz * sizeof(uint32_t), cudaMemcpyHostToDevice, sl.stream) != cudaSuccess) ||
                    (nnz && cudaMemcpyAsync(S.val[k], lval.data(), nnz * 32, cudaMemcpyHostToDevice, sl.stream) != cudaSuccess))
                    return set_error(ctx, B200ZK_ERR_CUDA, "constraint-matrix upload failed");
                if (values_montgomery_depth != 0) {
                    const int to_mont = values_montgomery_depth < 0, times = to_mont ? -values_montgomery_depth : values_montgomery_depth;
                    B2_TRY(fr_convert_dev(ctx, sl, S.val[k], S.val[k], nnz, to_mont, times));
                }
            }
            return B200ZK_OK;
        });
        if (!rc) rc = sync_all(grp);
        if (rc) {
            b200zk_group_r1cs_free(grp, q);
            return rc;
        }
        *out = q;
        return B200ZK_OK;
    });
}

int b200zk_group_groth16_prove_r1cs_dev(b200zk_group* grp, const b200zk_group_pk* pk, const b200zk_group_r1cs* q, const void* d_z,
                                        const uint64_t r[4], const uint64_t s[4], uint8_t proof_out[128]) {
    return with_group(grp, [&]() -> int {
        if (!pk || !q || !d_z || !r || !s || !proof_out) return B200ZK_ERR_ARG;
        if (pk->owner != grp) return gerr(grp, B200ZK_ERR_ARG, "proving key was uploaded to a different group");
        if (q->owner != grp) return gerr(grp, B200ZK_ERR_ARG, "constraint matrices were uploaded to a different group");
        if (q->m != pk->m)
            return gerr(grp, B200ZK_ERR_DOMAIN, "constraint matrices of domain " + std::to_string(q->m) + ", proving key of domain " + std::to_string(pk->m));
        if (q->n_inputs != pk->n_inputs)
            return gerr(grp, B200ZK_ERR_ARG, "constraint matrices with " + std::to_string(q->n_inputs) + " inputs, proving key with " + std::to_string(pk->n_inputs));
        if (q->n_vars != pk->n_vars)
            return gerr(grp, B200ZK_ERR_ARG, "constraint matrices over " + std::to_string(q->n_vars) + " variables, proving key over " + std::to_string(pk->n_vars));
        return prove_r1cs_columns(grp, pk, q->shard, q->nc, q->n_inputs, false, [&](b200zk_ctx*, Slot&, Fr*, const Fr** z) {
            *z = reinterpret_cast<const Fr*>(d_z);         // the caller wrote it on device 0's slot-0 stream
            return B200ZK_OK;
        }, r, s, proof_out);
    });
}

// ---- a snarkjs zkey resident on the group (the group twin of b200zk_zkey_*, zkey.cu) -------------------------------------------
void b200zk_group_zkey_free(b200zk_group* grp, b200zk_group_zkey* zk) {
    DeviceGuard dev_guard;
    if (!zk) return;
    for (size_t g = 0; g < zk->csr.size(); ++g) {
        if (grp && g < grp->ctx.size()) cudaSetDevice(grp->ctx[g]->device);
        if (zk->csr[g]) cudaFree(zk->csr[g]);
    }
    b200zk_group_pk_free(grp, zk->pk);
    delete zk;
}

int b200zk_group_zkey_load(b200zk_group* grp, const void* zkey, size_t zkey_len, unsigned table_window, b200zk_group_zkey** out) {
    return with_group(grp, [&]() -> int {
        if (!zkey || !out) return gerr(grp, B200ZK_ERR_ARG, "zkey_load: null pointer");
        *out = nullptr;
        const uint8_t* file = reinterpret_cast<const uint8_t*>(zkey);
        sjf::Zkey h;
        std::string err;
        const int hrc = zkey_header(file, zkey_len, &h, &err);
        if (hrc) return gerr(grp, hrc, err);
        const int P = grp->n;
        const size_t m = h.domain_size;
        unsigned log_rows, log_cols;
        split_log(ceil_log2(m), &log_rows, &log_cols);
        if (((size_t)1 << log_cols) < (size_t)P) return gerr(grp, B200ZK_ERR_ARG, "domain too small for this many GPUs");
        const ColumnLayout cl{log_rows, log_cols, log_cols - ceil_log2((size_t)P)};
        const size_t loc = m / P, L = 2 * loc + 1, ptr_bytes = (L * 4 + 15) & ~(size_t)15;
        b200zk_group_zkey* zk = new b200zk_group_zkey();
        zk->owner = grp; zk->n_vars = h.n_vars; zk->n_public = h.n_public; zk->domain_size = m;
        zk->csr.assign(P, nullptr);
        zk->mats.resize(P);
        // the sort on device 0, keyed owner-major: GPU g's A and B are entries [2 g loc, 2 (g + 1) loc] of its row_ptr
        ZkeyCsr all;
        std::vector<uint32_t> start(P + 1);
        int rc = on_device(grp, 0, [&](b200zk_ctx* c0, Slot& s0) -> int {
            B2_TRY(zkey_group_matrices_dev(c0, s0, file, h, cl, &all));
            B2_CUDA_OK(c0, cudaMemcpy2DAsync(start.data(), 4, all.row_ptr, 2 * loc * 4, 4, P + 1, cudaMemcpyDeviceToHost, s0.stream));
            B2_CUDA_OK(c0, cudaStreamSynchronize(s0.stream));
            return B200ZK_OK;
        });
        zk->num_constraints = all.nc;
        // every GPU's slice into one allocation of its own, row_ptr rebased to start at 0
        if (!rc) rc = each_device(grp, [&](int g, b200zk_ctx* ctx, Slot& sl) -> int {
            const size_t nnz = start[g + 1] - start[g];
            B2_CUDA_OK(ctx, cudaMalloc(&zk->csr[g], ptr_bytes + nnz * 36 + 16));
            uint32_t* row_ptr = reinterpret_cast<uint32_t*>(zk->csr[g]);
            Fr* val = reinterpret_cast<Fr*>(reinterpret_cast<char*>(zk->csr[g]) + ptr_bytes);
            uint32_t* col = reinterpret_cast<uint32_t*>(val + nnz);
            const int d0 = grp->ctx[0]->device;
            B2_CUDA_OK(ctx, cudaMemcpyPeerAsync(row_ptr, ctx->device, all.row_ptr + (size_t)g * 2 * loc, d0, L * 4, sl.stream));
            if (nnz) {
                B2_CUDA_OK(ctx, cudaMemcpyPeerAsync(val, ctx->device, all.val + start[g], d0, nnz * sizeof(Fr), sl.stream));
                B2_CUDA_OK(ctx, cudaMemcpyPeerAsync(col, ctx->device, all.col + start[g], d0, nnz * 4, sl.stream));
            }
            B2_TRY(rebase_dev(ctx, sl, row_ptr, L, start[g]));
            b200zk_group_r1cs::Shard& Q = zk->mats[g];
            Q.ptr[0] = row_ptr; Q.ptr[1] = row_ptr + loc;
            Q.col[0] = Q.col[1] = col;
            Q.val[0] = Q.val[1] = val;
            return B200ZK_OK;
        });
        if (!rc) rc = sync_all(grp);
        if (all.csr) {                                  // device 0 keeps only its own share
            cudaSetDevice(grp->ctx[0]->device);
            cudaFree(all.csr);
        }
        if (!rc) {
            uint64_t vk[56];
            zkey_vk_points(file, h, vk);
            rc = group_pk_build(grp, file + h.a, file + h.b1, file + h.b2, file + h.l, file + h.h, h.n_vars, (size_t)h.n_public + 1, m, vk,
                                table_window, &zk->pk);
        }
        if (rc) {
            b200zk_group_zkey_free(grp, zk);
            return rc;
        }
        *out = zk;
        return B200ZK_OK;
    });
}

int b200zk_group_zkey_info(const b200zk_group_zkey* zk, size_t* n_vars, size_t* n_public, size_t* domain_size, size_t* num_constraints) {
    if (!zk) return B200ZK_ERR_ARG;
    if (n_vars) *n_vars = zk->n_vars;
    if (n_public) *n_public = zk->n_public;
    if (domain_size) *domain_size = zk->domain_size;
    if (num_constraints) *num_constraints = zk->num_constraints;
    return B200ZK_OK;
}

size_t b200zk_group_zkey_table_bytes(const b200zk_group_zkey* zk) { return zk && zk->pk ? zk->pk->table_bytes : 0; }

int b200zk_group_zkey_prove(b200zk_group* grp, const b200zk_group_zkey* zk, const void* wtns, size_t wtns_len, const uint64_t r[4],
                            const uint64_t s[4], uint8_t proof_out[128], char* proof_json, size_t* proof_json_len, char* public_json,
                            size_t* public_json_len) {
    return with_group(grp, [&]() -> int {
        if (!zk || !wtns || (proof_json && !proof_json_len) || (public_json && !public_json_len))
            return gerr(grp, B200ZK_ERR_ARG, "zkey_prove: null key or witness, or a JSON buffer without its length");
        if (zk->owner != grp) return gerr(grp, B200ZK_ERR_ARG, "zkey was loaded on a different group");
        WtnsJob job;
        std::string err;
        const int prc = wtns_prologue(reinterpret_cast<const uint8_t*>(wtns), wtns_len, zk->n_vars, zk->n_public, r, s, proof_json,
                                      proof_json_len, public_json, public_json_len, &job, &err);
        if (prc) return gerr(grp, prc, err);
        uint8_t proof[128];
        int rc = prove_r1cs_columns(grp, zk->pk, zk->mats, zk->num_constraints, zk->n_public + 1, true,
                                    [&](b200zk_ctx* c0, Slot& s0, Fr* tail, const Fr** z) {
            *z = tail;
            return witness_to_device(c0, s0, job.z, zk->n_vars, tail);
        }, job.r, job.s, proof);
        if (rc) return rc;
        return on_device(grp, 0, [&](b200zk_ctx* c0, Slot& s0) {
            return zkey_outputs_dev(c0, s0, proof, job, proof_out, proof_json, proof_json_len, public_json, public_json_len);
        });
    });
}

}  // extern "C"
