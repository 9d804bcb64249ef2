// zkey.cu -- a snarkjs Groth16 .zkey resident in HBM and the prove call on its bytes (b200zk_zkey_*, the C side of what
// formats.read_zkey + circom.load_zkey + circom.groth16_prove do in Python), and the device sort of the group twin
// (b200zk_group_zkey_*, group.cu).
//
// Load: api.cu parses the header on the host (snarkjs_files.h) and uploads the point sections through pk_build; here the
// coefficient section (section 4: n records of m, c, s u32 and value R^2 as 32 bytes, 44 bytes each, so the values are only
// 4-byte aligned) becomes the CSR matrices of ConstraintMatrices on the device:
//   1. k_zkey_coef_check: every record has m <= 1, s < n_vars, c < domain size (count + lowest bad index), and the largest c;
//      num_constraints = largest c - n_public, as ZKey.num_constraints
//   2. k_zkey_coef_hist: terms per key for rows below num_constraints -- the public-input rows snarkjs appends are dropped,
//      as coo_to_csr does.  The key of one GPU (RowKey) is (matrix, row); that of a group (SlotKey) is owner-major (owner
//      GPU, matrix, slot of the owner's column-layout slice), so each GPU's A and B are one contiguous slice of the result
//   3. exclusive scan (msm.cu) of the L = keys + 1 counts: for one GPU, A's row_ptr is entries [0, nc], B's row_ptr entries
//      [nc, 2 nc] of the same array, and both matrices index one col / val array (b200zk_qap_dev reads ptr[i] .. ptr[i + 1]
//      as absolute positions, so B's row_ptr need not start at 0); a group's GPU g finds the same layout in entries
//      [2 g loc, 2 (g + 1) loc] once they are rebased to start at 0 (loc = m / P)
//   4. k_zkey_coef_scatter: columns and values into place, with the one Montgomery reduction of ConstraintMatrices
//      (fr_convert(to_mont = 0, times = 1)) fused; the order of terms within a row is that of the atomics, which the mat-vec
//      does not see (field addition is exact)
// Peak device memory of the load: 44 n bytes of raw records + 36 n + 4 L bytes of CSR + 4 L bytes of counters while the
// matrices are built; the raw records and counters are freed before the proving key is uploaded (its queries, plus the
// fixed-base tables the table policy builds).
//
// Prove: the witness (section 2 of the .wtns: n_vars canonical 32-byte values) is uploaded and k_wtns_to_mont checks every
// entry is below r and converts it; then qap_dev and prove_dev as circom.prove_zkey_wtns runs them, and the proof's points
// reach the host as ffjavascript encodings (points_decompress_dev -> points_encode_dev fmt 0) for the JSON writer.
#include <errno.h>
#include <algorithm>
#include <sys/random.h>

#include "common.cuh"
#include "snarkjs_files.h"

namespace b200zk {

static const uint32_t COEF_WORDS = 11;           // 44-byte records

// The sort keys of a kept record (matrix mat, constraint R < nc)
struct RowKey {                                  // one GPU: A's rows, then B's
    uint32_t nc;
    __device__ __forceinline__ uint32_t operator()(uint32_t mat, uint32_t R) const { return mat * nc + R; }
};
struct SlotKey {                                 // a group: owner GPU, then matrix, then the slot of the owner's slice
    ColumnLayout cl;
    uint32_t loc;                                // slots per GPU
    __device__ __forceinline__ uint32_t operator()(uint32_t mat, uint32_t R) const {
        return (cl.owner(R) * 2 + mat) * loc + cl.slot(R);
    }
};

__global__ void k_zkey_coef_check(const uint32_t* rec, uint32_t n, uint32_t n_vars, uint32_t domain_size, unsigned long long* bad,
                                  uint32_t* max_c) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t c = 0;
    if (i < n) {
        const uint32_t* w = rec + (size_t)i * COEF_WORDS;
        c = w[1];
        if (!sjf::coef_record_ok(w[0], c, w[2], n_vars, domain_size)) {
            atomicAdd(&bad[0], 1ull);
            atomicMin(&bad[1], (unsigned long long)i);
            c = 0;
        }
    }
    c = __reduce_max_sync(0xFFFFFFFFu, c);
    if ((threadIdx.x & 31) == 0 && c) atomicMax(max_c, c);
}

template <class Key>
__global__ void k_zkey_coef_hist(const uint32_t* rec, uint32_t n, uint32_t nc, Key key, uint32_t* counts) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t* w = rec + (size_t)i * COEF_WORDS;
    if (w[1] < nc) atomicAdd(&counts[key(w[0], w[1])], 1u);
}

template <class Key>
__global__ void k_zkey_coef_scatter(const uint32_t* rec, uint32_t n, uint32_t nc, Key key, uint32_t* cursor, uint32_t* col, Fr* val) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t* w = rec + (size_t)i * COEF_WORDS;
    if (w[1] >= nc) return;
    const uint32_t pos = atomicAdd(&cursor[key(w[0], w[1])], 1u);
    Fr v;
#pragma unroll
    for (int k = 0; k < 8; ++k) v.l[k] = w[3 + k];
    col[pos] = w[2];
    st16(val + pos, Fr::from_mont(v));            // value R^2 -> value R (Montgomery)
}

__device__ __forceinline__ bool fr_below_modulus(const Fr& v) {
#pragma unroll
    for (int k = 7; k >= 0; --k)
        if (v.l[k] != FrParams::mod(k)) return v.l[k] < FrParams::mod(k);
    return false;
}

// canonical witness values -> Montgomery in place; an entry >= r bumps bad[0], lowers bad[1] to its index and becomes 0
__global__ void k_wtns_to_mont(Fr* z, size_t n, unsigned long long* bad) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr v = ld16(z + i);
    if (!fr_below_modulus(v)) {
        atomicAdd(&bad[0], 1ull);
        atomicMin(&bad[1], (unsigned long long)i);
        v = Fr::zero();
    }
    st16(z + i, Fr::to_mont(v));
}

namespace {
struct DevFree {                     // device scratch freed on every return path
    void* p = nullptr;
    ~DevFree() { if (p) cudaFree(p); }
};

// The raw records on the device and k_zkey_coef_check over them; *nc = num_constraints (0 without records)
int coef_upload_check(b200zk_ctx* ctx, Slot& sl, const uint8_t* file, const sjf::Zkey& h, DevFree& raw, uint32_t* nc) {
    const uint32_t n = h.n_coef;
    cudaStream_t st = sl.stream;
    *nc = 0;
    if (!n) return B200ZK_OK;
    B2_CUDA_OK(ctx, cudaMalloc(&raw.p, (size_t)n * 44));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(raw.p, file + h.coef, (size_t)n * 44, cudaMemcpyHostToDevice, st));
    B2_CUDA_OK(ctx, sl.small.reserve(1024));
    unsigned long long* bad = reinterpret_cast<unsigned long long*>(sl.small.p);
    B2_CUDA_OK(ctx, cudaMemsetAsync(bad, 0, 24, st));
    B2_CUDA_OK(ctx, cudaMemsetAsync(bad + 1, 0xFF, 8, st));
    B2_TRY(launch(ctx, st, "zkey_coef_check", k_zkey_coef_check, (n + 255) / 256, 256, 0, (const uint32_t*)raw.p, n, h.n_vars,
                  h.domain_size, bad, reinterpret_cast<uint32_t*>(bad + 2)));
    unsigned long long hb[3];
    B2_CUDA_OK(ctx, cudaMemcpyAsync(hb, bad, 24, cudaMemcpyDeviceToHost, st));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(st));
    if (hb[0]) {
        char msg[256];
        snprintf(msg, sizeof(msg), "zkey coefficient section: %llu of %u records have matrix index > 1, signal index >= n_vars or "
                 "constraint index >= domain size, the first at index %llu", hb[0], n, hb[1]);
        return set_error(ctx, B200ZK_ERR_ARG, msg);
    }
    const uint32_t max_c = (uint32_t)hb[2];
    if (max_c < h.n_public) {
        char msg[160];
        snprintf(msg, sizeof(msg), "zkey coefficient section: the largest constraint index %u is below n_public = %u", max_c,
                 h.n_public);
        return set_error(ctx, B200ZK_ERR_ARG, msg);
    }
    *nc = max_c - h.n_public;
    return B200ZK_OK;
}

// The kept records of `raw` in CSR under `key` (L - 1 keys) in one new allocation *csr: row_ptr (L entries, padded to 16
// bytes), then val (n Fr), then col (n u32).  The caller frees *csr, also on failure.
template <class Key>
int coef_csr(b200zk_ctx* ctx, Slot& sl, const DevFree& raw, uint32_t n, uint32_t nc, Key key, size_t L, void** csr, uint32_t** row_ptr,
             uint32_t** col, Fr** val) {
    cudaStream_t st = sl.stream;
    const size_t ptr_bytes = (L * 4 + 15) & ~(size_t)15;
    B2_CUDA_OK(ctx, cudaMalloc(csr, ptr_bytes + (size_t)n * 36 + 16));
    *row_ptr = reinterpret_cast<uint32_t*>(*csr);
    *val = reinterpret_cast<Fr*>(reinterpret_cast<char*>(*csr) + ptr_bytes);
    *col = reinterpret_cast<uint32_t*>(*val + n);
    if (n == 0) {
        B2_CUDA_OK(ctx, cudaMemsetAsync(*row_ptr, 0, L * 4, st));
        B2_CUDA_OK(ctx, cudaStreamSynchronize(st));
        return B200ZK_OK;
    }
    const size_t nblk = (L + 2047) / 2048;            // the scan's tiles (msm.cu SCAN_TILE)
    DevFree scratch;
    B2_CUDA_OK(ctx, cudaMalloc(&scratch.p, (L + nblk) * 4));
    uint32_t* counts = reinterpret_cast<uint32_t*>(scratch.p);
    B2_CUDA_OK(ctx, cudaMemsetAsync(counts, 0, L * 4, st));
    const uint32_t* rec = (const uint32_t*)raw.p;
    B2_TRY(launch(ctx, st, "zkey_coef_hist", k_zkey_coef_hist<Key>, (n + 255) / 256, 256, 0, rec, n, nc, key, counts));
    B2_TRY(exclusive_scan(ctx, st, counts, *row_ptr, counts + L, (uint32_t)L));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(counts, *row_ptr, L * 4, cudaMemcpyDeviceToDevice, st));
    B2_TRY(launch(ctx, st, "zkey_coef_scatter", k_zkey_coef_scatter<Key>, (n + 255) / 256, 256, 0, rec, n, nc, key, counts, *col, *val));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(st));
    return B200ZK_OK;
}
}  // namespace

int zkey_header(const uint8_t* file, size_t len, sjf::Zkey* h, std::string* err) {
    if (!sjf::parse_zkey(file, len, h, err)) return B200ZK_ERR_ARG;
    if (h->domain_size > (1u << 27)) {
        *err = "zkey domain size " + std::to_string(h->domain_size) +
               " exceeds 2^27: the h step needs twice the domain within Fr's 2^28 subgroup";
        return B200ZK_ERR_DOMAIN;
    }
    return B200ZK_OK;
}

void zkey_vk_points(const uint8_t* file, const sjf::Zkey& h, uint64_t vk[56]) {
    // b200zk_pk_upload's order from the header's alpha_1 beta_1 beta_2 gamma_2 delta_1 delta_2
    const uint8_t* hp = file + h.hdr_points;
    memcpy(vk, hp, 128);                    // alpha_1, beta_1
    memcpy(vk + 16, hp + 384, 64);          // delta_1
    memcpy(vk + 24, hp + 128, 128);         // beta_2
    memcpy(vk + 40, hp + 448, 128);         // delta_2
}

int zkey_matrices_dev(b200zk_ctx* ctx, Slot& sl, const uint8_t* file, const sjf::Zkey& h, b200zk_zkey* zk) {
    DevFree raw;
    uint32_t nc;
    B2_TRY(coef_upload_check(ctx, sl, file, h, raw, &nc));
    zk->num_constraints = nc;
    return coef_csr(ctx, sl, raw, h.n_coef, nc, RowKey{nc}, 2 * (size_t)nc + 1, &zk->csr, &zk->row_ptr, &zk->col, &zk->val);
}

int zkey_group_matrices_dev(b200zk_ctx* ctx, Slot& sl, const uint8_t* file, const sjf::Zkey& h, const ColumnLayout& cl, ZkeyCsr* out) {
    DevFree raw;
    B2_TRY(coef_upload_check(ctx, sl, file, h, raw, &out->nc));
    const uint32_t loc = 1u << (cl.log_rows + cl.log_cg);
    return coef_csr(ctx, sl, raw, h.n_coef, out->nc, SlotKey{cl, loc}, 2 * (size_t)h.domain_size + 1, &out->csr, &out->row_ptr, &out->col,
                    &out->val);
}

__global__ void k_rebase(uint32_t* p, uint32_t n, uint32_t base) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] -= base;
}

int rebase_dev(b200zk_ctx* ctx, Slot& sl, uint32_t* p, size_t n, uint32_t base) {
    if (!base) return B200ZK_OK;
    return launch(ctx, sl.stream, "zkey_rebase", k_rebase, (unsigned)((n + 255) / 256), 256, 0, p, (uint32_t)n, base);
}

// A uniform scalar mod r from the OS (getrandom), as Montgomery limbs: x R^-1 is uniform when x is.
static bool draw_scalar(uint64_t out[4]) {
    for (;;) {
        uint8_t b[32];
        size_t got = 0;
        while (got < sizeof(b)) {
            const ssize_t k = getrandom(b + got, sizeof(b) - got, 0);
            if (k < 0) {
                if (errno == EINTR) continue;
                return false;
            }
            got += (size_t)k;
        }
        b[31] &= 0x3F;                                   // r < 2^254: rejection keeps about 3 draws in 4
        if (sjf::below_r(b)) {
            memcpy(out, b, 32);
            return true;
        }
    }
}

int wtns_prologue(const uint8_t* wtns, size_t wtns_len, size_t n_vars, size_t n_public, const uint64_t* r_in, const uint64_t* s_in,
                  const char* proof_json, size_t* proof_json_len, const char* public_json, size_t* public_json_len, WtnsJob* job,
                  std::string* err) {
    sjf::Wtns w;
    if (!sjf::parse_wtns(wtns, wtns_len, &w, err)) return B200ZK_ERR_ARG;
    if (w.n != n_vars) {
        char msg[128];
        snprintf(msg, sizeof(msg), "witness has %u entries, the key expects %zu", w.n, n_vars);
        *err = msg;
        return B200ZK_ERR_LENGTH;
    }
    job->z = wtns + w.data;
    job->pub = sjf::public_json(wtns + w.data + 32, n_public);
    const size_t need_proof = B200ZK_PROOF_JSON_MAX, need_public = job->pub.size() + 1;
    if ((proof_json && *proof_json_len < need_proof) || (public_json && *public_json_len < need_public)) {
        char msg[160];
        snprintf(msg, sizeof(msg), "output buffer too small: proof.json needs %zu bytes and public.json %zu (with the NUL)", need_proof,
                 need_public);
        if (proof_json_len) *proof_json_len = need_proof;
        if (public_json_len) *public_json_len = need_public;
        *err = msg;
        return B200ZK_ERR_SHORT_BUFFER;
    }
    if (r_in) memcpy(job->r, r_in, 32);
    else if (!draw_scalar(job->r)) { *err = "getrandom failed: no randomness for r"; return B200ZK_ERR_ARG; }
    if (s_in) memcpy(job->s, s_in, 32);
    else if (!draw_scalar(job->s)) { *err = "getrandom failed: no randomness for s"; return B200ZK_ERR_ARG; }
    return B200ZK_OK;
}

int witness_to_device(b200zk_ctx* ctx, Slot& sl, const uint8_t* z, size_t nv, Fr* d_z) {
    cudaStream_t st = sl.stream;
    B2_CUDA_OK(ctx, cudaMemcpyAsync(d_z, z, nv * sizeof(Fr), cudaMemcpyHostToDevice, st));
    B2_CUDA_OK(ctx, sl.small.reserve(1024));
    unsigned long long* bad = reinterpret_cast<unsigned long long*>(sl.small.p);
    B2_CUDA_OK(ctx, cudaMemsetAsync(bad, 0, 8, st));
    B2_CUDA_OK(ctx, cudaMemsetAsync(bad + 1, 0xFF, 8, st));
    B2_TRY(launch(ctx, st, "wtns_to_mont", k_wtns_to_mont, (unsigned)((nv + 255) / 256), 256, 0, d_z, nv, bad));
    unsigned long long hb[2];
    B2_CUDA_OK(ctx, cudaMemcpyAsync(hb, bad, 16, cudaMemcpyDeviceToHost, st));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(st));
    if (hb[0]) {
        char msg[160];
        snprintf(msg, sizeof(msg), "witness: %llu of %zu entries are not below r, the first is w[%llu]", hb[0], nv, hb[1]);
        return set_error(ctx, B200ZK_ERR_ARG, msg);
    }
    return B200ZK_OK;
}

int zkey_outputs_dev(b200zk_ctx* ctx, Slot& sl, const uint8_t proof[128], const WtnsJob& job, uint8_t* proof_out, char* proof_json,
                     size_t* proof_json_len, char* public_json, size_t* public_json_len) {
    if (proof_out) memcpy(proof_out, proof, 128);
    if (public_json) {
        memcpy(public_json, job.pub.c_str(), job.pub.size() + 1);
        *public_json_len = job.pub.size();
    }
    if (!proof_json) return B200ZK_OK;
    // A || C (G1) and B (G2) compressed -> affine -> ffjavascript encodings in io_a's first JSON_SCRATCH bytes: compressed at
    // [0, 128), affine at [256, 512), encodings at [512, 768); whatever io_a held is no longer needed (the prover returned
    // after synchronising the slot's stream)
    cudaStream_t st = sl.stream;
    B2_CUDA_OK(ctx, sl.io_a.reserve(JSON_SCRATCH));
    uint8_t cmp[128], enc[256];
    memcpy(cmp, proof, 32);
    memcpy(cmp + 32, proof + 96, 32);
    memcpy(cmp + 64, proof + 32, 64);
    uint8_t* d = reinterpret_cast<uint8_t*>(sl.io_a.p);
    B2_CUDA_OK(ctx, cudaMemcpyAsync(d, cmp, 128, cudaMemcpyHostToDevice, st));
    B2_TRY(points_decompress_dev(ctx, sl, 0, d, 2, 0, d + 256, nullptr));
    B2_TRY(points_decompress_dev(ctx, sl, 1, d + 64, 1, 0, d + 384, nullptr));
    B2_TRY(points_encode_dev(ctx, sl, 0, d + 256, 2, 0, d + 512));
    B2_TRY(points_encode_dev(ctx, sl, 1, d + 384, 1, 0, d + 640));
    B2_CUDA_OK(ctx, cudaMemcpyAsync(enc, d + 512, 256, cudaMemcpyDeviceToHost, st));
    B2_CUDA_OK(ctx, cudaStreamSynchronize(st));
    const std::string pj = sjf::proof_json(enc, enc + 128, enc + 64);
    memcpy(proof_json, pj.c_str(), pj.size() + 1);
    *proof_json_len = pj.size();
    return B200ZK_OK;
}

int zkey_prove_dev(b200zk_ctx* ctx, Slot& sl, const b200zk_zkey* zk, const uint8_t* wtns, size_t wtns_len, const uint64_t* r_in,
                   const uint64_t* s_in, uint8_t* proof_out, char* proof_json, size_t* proof_json_len, char* public_json,
                   size_t* public_json_len) {
    WtnsJob job;
    std::string err;
    const int prc = wtns_prologue(wtns, wtns_len, zk->n_vars, zk->n_public, r_in, s_in, proof_json, proof_json_len, public_json,
                                  public_json_len, &job, &err);
    if (prc) return set_error(ctx, prc, err);

    const size_t nv = zk->n_vars, m = zk->domain_size;
    // io_a: z and a, b, c for the proof, then (proof.json) the points and encodings of JSON_SCRATCH bytes, which is more than
    // z, a, b, c take for the smallest keys (domain 1 or 2 and a few variables)
    B2_CUDA_OK(ctx, sl.io_a.reserve(std::max((nv + 3 * m) * sizeof(Fr), JSON_SCRATCH)));
    Fr* d_z = reinterpret_cast<Fr*>(sl.io_a.p);
    Fr* d_abc = d_z + nv;
    B2_TRY(witness_to_device(ctx, sl, job.z, nv, d_z));
    const size_t nc = zk->num_constraints;
    B2_TRY(qap_dev(ctx, sl, zk->row_ptr, zk->col, zk->val, zk->row_ptr + nc, zk->col, zk->val, nc, zk->n_public + 1, d_z,
                   ceil_log2(m), d_abc, d_abc + m, d_abc + 2 * m));
    uint8_t proof[128];
    B2_TRY(prove_dev(ctx, zk->pk, d_z, d_abc, d_abc + m, d_abc + 2 * m, job.r, job.s, 0, proof));
    return zkey_outputs_dev(ctx, sl, proof, job, proof_out, proof_json, proof_json_len, public_json, public_json_len);
}

}  // namespace b200zk
