// msm.cu -- Pippenger bucket MSM over BN254 G1 / G2 for sm_90a.
//
// Replaces `G::msm(bases, scalars)` -- THE hot line of the reference
// (/root/reference/dist-primitives/src/dmsm/mod.rs:82, reached from groth16/src/prove.rs:41,80,119,121,123)
// which is arkworks' CPU `VariableBaseMSM::msm_bigint_wnaf`.  The result is the same group element
// sum_i scalars[i] * bases[i]; only its canonical affine form ever leaves the library.
//
// Pipeline (all on one stream, no host round trips):
//   1 digits     scalar Montgomery -> canonical, signed c-bit windows; per (window, |digit|) histogram
//                with atomics that also hand every entry its rank inside the bucket
//   2 scan       exclusive prefix sum of the W * 2^(c-1) bucket sizes
//   3 scatter    entries[offset[bucket] + rank] = point index | sign  (counting sort, no comparison sort)
//   4 accumulate one thread per bucket task: gather affine points (the 2^20 x 64 B base array is larger
//                than H100's 50 MB L2), mixed XYZZ additions
//   5 reduce     per window sum_b b * bucket_b as segment running sums + small scalar multiples,
//                tree-combined per window in shared memory
//   6 combine    Horner over windows (c doublings each)
#include "common.cuh"
#include "glv.cuh"

namespace b200zk {

static const uint32_t KEY_NONE = 0xFFFFFFFFu;

// ---------------------------------------------------------------------------------------------
// 1. digits + histogram
// ---------------------------------------------------------------------------------------------
// Fixed-base tables (section 7): every window shares ONE bucket set, the window is carried by the entry index
// (w * n + i selects 2^{cw} P_i in the table) instead of by the bucket index.
__global__ void k_msm_digits(const Fr* scalars, uint32_t n, uint32_t c, uint32_t W, uint32_t* keys, uint32_t* ranks,
                             uint32_t* counts) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr s = Fr::from_mont(ld16(scalars + i));
    uint32_t k[9];
#pragma unroll
    for (int j = 0; j < 8; ++j) k[j] = s.l[j];
    k[8] = 0;
    const uint32_t B = 1u << (c - 1);
    const uint32_t mask = (1u << c) - 1;
    uint32_t carry = 0;
    for (uint32_t w = 0; w < W; ++w) {
        uint32_t off = w * c, limb = off >> 5, sh = off & 31;
        uint64_t v = limb < 8 ? ((uint64_t)k[limb] | ((uint64_t)k[limb + 1] << 32)) : 0;
        uint32_t d = ((uint32_t)(v >> sh) & mask) + carry;
        uint32_t key = KEY_NONE, rank = 0;
        carry = 0;
        uint32_t neg = 0;
        if (d > B) { d = (1u << c) - d; neg = 1; carry = 1; }
        if (d != 0) {
            uint32_t g = d - 1;
            rank = atomicAdd(counts + g, 1u);
            key = g | (neg << 31);
        }
        const size_t slot = (size_t)w * n + i;
        keys[slot] = key;
        ranks[slot] = rank;
    }
}

// Every other MSM: k = k1 + k2 lambda (glv.cuh; G1 and, with beta^2, G2); window w of |k1| fills bucket set 2 (Wh - 1 - w),
// window w of |k2| set 2 (Wh - 1 - w) + 1 over the same points.  Sets are numbered in the order the Horner chain consumes
// them (top window first, the two halves interleaved), so that a *group* of consecutive sets can be reduced and folded
// into the chain while the bucket kernel of the next group is still running (host side, "window-group pipeline").  phi
// is applied once to the second chain's result in k_msm_horner_glv.
__global__ void k_msm_digits_glv(const Fr* scalars, uint32_t n, uint32_t c, uint32_t Wh, uint32_t* keys, uint32_t* ranks,
                                 uint32_t* counts) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Fr s = Fr::from_mont(ld16(scalars + i));
    GlvSplit sp = glv_decompose(s.l);
    const uint32_t B = 1u << (c - 1);
    const uint32_t mask = (1u << c) - 1;
    for (uint32_t h = 0; h < 2; ++h) {
        uint32_t k[5];
#pragma unroll
        for (int j = 0; j < 4; ++j) k[j] = h ? sp.k2[j] : sp.k1[j];
        k[4] = 0;
        const uint32_t sgn = h ? (sp.neg2 ? 1u : 0u) : (sp.neg1 ? 1u : 0u);
        uint32_t carry = 0;
        for (uint32_t w = 0; w < Wh; ++w) {
            uint32_t off = w * c, limb = off >> 5, sh = off & 31;
            uint64_t v = limb < 4 ? ((uint64_t)k[limb] | ((uint64_t)k[limb + 1] << 32)) : 0;
            uint32_t d = ((uint32_t)(v >> sh) & mask) + carry;
            uint32_t key = KEY_NONE, rank = 0;
            carry = 0;
            uint32_t neg = 0;
            if (d > B) { d = (1u << c) - d; neg = 1; carry = 1; }
            if (d != 0) {
                uint32_t g = (2 * (Wh - 1 - w) + h) * B + (d - 1);
                rank = atomicAdd(counts + g, 1u);
                key = g | ((neg ^ sgn) << 31);
            }
            size_t slot = (size_t)(2 * (Wh - 1 - w) + h) * n + i;
            keys[slot] = key;
            ranks[slot] = rank;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// 2. exclusive scan (uint32), three small kernels
// ---------------------------------------------------------------------------------------------
static const uint32_t SCAN_THREADS = 512, SCAN_ITEMS = 4, SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* total, uint32_t* warp_sums) {
    uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= (uint32_t)o) x += y;
    }
    if (lane == 31) warp_sums[wid] = x;
    __syncthreads();
    if (wid == 0) {
        uint32_t nw = blockDim.x >> 5;
        uint32_t s = lane < nw ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t y = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= (uint32_t)o) s += y;
        }
        if (lane < nw) warp_sums[lane] = s;
    }
    __syncthreads();
    uint32_t base = wid ? warp_sums[wid - 1] : 0;
    *total = warp_sums[(blockDim.x >> 5) - 1];
    return base + x - v;
}

__global__ void __launch_bounds__(SCAN_THREADS) k_scan_local(const uint32_t* in, uint32_t* out, uint32_t* sums, uint32_t n) {
    __shared__ uint32_t warp_sums[32];
    uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS], t = 0;
#pragma unroll
    for (uint32_t j = 0; j < SCAN_ITEMS; ++j) { v[j] = base + j < n ? in[base + j] : 0; t += v[j]; }
    uint32_t total;
    uint32_t ex = block_exclusive_scan(t, &total, warp_sums);
#pragma unroll
    for (uint32_t j = 0; j < SCAN_ITEMS; ++j) { if (base + j < n) out[base + j] = ex; ex += v[j]; }
    if (threadIdx.x == 0) sums[blockIdx.x] = total;
}
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_sums(uint32_t* sums, uint32_t n) {
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += SCAN_THREADS) {
        uint32_t i = base + threadIdx.x;
        uint32_t v = i < n ? sums[i] : 0, total;
        uint32_t ex = block_exclusive_scan(v, &total, warp_sums);
        uint32_t carry = carry_s;
        if (i < n) sums[i] = ex + carry;
        __syncthreads();
        if (threadIdx.x == 0) carry_s = carry + total;
        __syncthreads();
    }
}
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_add(uint32_t* out, const uint32_t* sums, uint32_t n) {
    uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
    uint32_t add = sums[blockIdx.x];
#pragma unroll
    for (uint32_t j = 0; j < SCAN_ITEMS; ++j) if (base + j < n) out[base + j] += add;
}

// ---------------------------------------------------------------------------------------------
// 3. scatter
// ---------------------------------------------------------------------------------------------
// slots [t0, t0 + total) of keys / ranks (one window group); offsets / entries are indexed globally
__global__ void k_msm_scatter(const uint32_t* keys, const uint32_t* ranks, const uint32_t* offsets, uint32_t n, size_t t0,
                              size_t total, uint32_t fold, uint32_t* entries) {
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    t += t0;
    uint32_t key = keys[t];
    if (key == KEY_NONE) return;
    uint32_t i = fold ? (uint32_t)t : (uint32_t)(t % n);
    uint32_t g = key & 0x7FFFFFFFu;
    entries[offsets[g] + ranks[t]] = i | (key & 0x80000000u);
}

// ---------------------------------------------------------------------------------------------
// 4. bucket accumulation over bounded-size tasks
//    A bucket of s entries is cut into ceil(s / TASK_LEN) tasks, so a "giant" bucket (the short top
//    window, or the digit-1 bucket of a 0/1-heavy witness) is spread over many threads instead of
//    serialising one.  Single-task buckets write their sum straight into buckets[g]; the rare
//    multi-task buckets go through task_sums[] and a block-level merge.
// ---------------------------------------------------------------------------------------------
static const uint32_t TASK_LEN = 128, MAX_TASK_LEN = 1024;    // default / largest task length (runtime: task_len)
static const uint32_t ACC_MINBLOCKS = 4, ACC_MINBLOCKS_G2 = 4;  // bucket kernel blocks per SM (k_msm_accumulate)

__global__ void k_msm_task_counts(const uint32_t* offsets, uint32_t nbuckets, uint32_t task_len, uint32_t* ntasks) {
    uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g > nbuckets) return;
    ntasks[g] = g < nbuckets ? (offsets[g + 1] - offsets[g] + task_len - 1) / task_len : 0;
}

// task_bucket[t] = owning bucket; buckets with > 1 task are appended to multi_list from the front when they have more
// than MERGE_SMALL tasks (block-level merge) and from the back otherwise (one thread each); counts[0] / counts[1]
static const uint32_t MERGE_SMALL = 8;
__global__ void k_msm_fill_tasks(const uint32_t* task_off, uint32_t nbuckets, uint32_t* task_bucket, uint32_t* multi_list,
                                 uint32_t list_cap, uint32_t* multi_count) {
    uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= nbuckets) return;
    uint32_t lo = task_off[g], hi = task_off[g + 1];
    for (uint32_t t = lo; t < hi; ++t) task_bucket[t] = g;
    if (hi - lo > MERGE_SMALL) multi_list[atomicAdd(multi_count, 1u)] = g;
    else if (hi - lo > 1) multi_list[list_cap - 1 - atomicAdd(multi_count + 1, 1u)] = g;
}

// Counting sort of the tasks by length (descending): the lanes of a warp then run loops of (almost)
// equal length.  Unsorted, bucket sizes ~Poisson(32) leave only 23 of 32 lanes active on average
// (ncu smsp__thread_inst_executed_per_inst_executed).
__device__ __forceinline__ uint32_t task_length(const uint32_t* offsets, const uint32_t* task_off, uint32_t g, uint32_t t,
                                                uint32_t task_len) {
    uint32_t lo = offsets[g] + (t - task_off[g]) * task_len, end = offsets[g + 1];
    return (lo + task_len < end ? lo + task_len : end) - lo;
}
__global__ void __launch_bounds__(256) k_msm_task_hist(const uint32_t* offsets, const uint32_t* task_off, const uint32_t* task_bucket,
                                uint32_t nbuckets, uint32_t task_len, uint32_t* hist, uint32_t* task_rank) {
    __shared__ uint32_t sh_cnt[MAX_TASK_LEN + 1], sh_base[MAX_TASK_LEN + 1];     // block-local histogram first:
    for (uint32_t i = threadIdx.x; i <= task_len; i += blockDim.x) sh_cnt[i] = 0;   // few hot bins -> keep contention in smem
    __syncthreads();
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    bool live = t < task_off[nbuckets];
    uint32_t len = 0, local = 0;
    if (live) {
        len = task_length(offsets, task_off, task_bucket[t], t, task_len);
        local = atomicAdd(sh_cnt + len, 1u);
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i <= task_len; i += blockDim.x)
        if (sh_cnt[i]) sh_base[i] = atomicAdd(hist + i, sh_cnt[i]);
    __syncthreads();
    if (live) task_rank[t] = sh_base[len] + local;
}
__global__ void k_msm_task_hist_scan(uint32_t* hist, uint32_t task_len) {      // base[len] = #tasks longer than len; 1 thread
    uint32_t run = 0;
    for (int len = (int)task_len; len >= 0; --len) { uint32_t c = hist[len]; hist[len] = run; run += c; }
}
__global__ void k_msm_task_order(const uint32_t* offsets, const uint32_t* task_off, const uint32_t* task_bucket,
                                 uint32_t nbuckets, uint32_t task_len, const uint32_t* hist, const uint32_t* task_rank,
                                 uint32_t* order) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= task_off[nbuckets]) return;
    uint32_t len = task_length(offsets, task_off, task_bucket[t], t, task_len);
    order[hist[len] + task_rank[t]] = t;
}

// G2 (Fq2 coordinates): 250 registers uncapped = 8 warps/SM with `wait` the top stall; capped at 128 (4 blocks/SM, some
// spills) it was faster at 2^20; 5+ blocks lose again
template <class F, bool RMW>
__global__ void __launch_bounds__(128, sizeof(F) > 32 ? ACC_MINBLOCKS_G2 : ACC_MINBLOCKS) k_msm_accumulate(const affine_t<F>* bases, const uint32_t* entries, const uint32_t* offsets,
                                 const uint32_t* task_off, const uint32_t* task_bucket, const uint32_t* order,
                                 uint32_t nbuckets, uint32_t task_len, uint32_t wave, xyzz_t<F>* buckets, xyzz_t<F>* task_sums) {
    // Block order over the length-sorted task list: the first `wave` blocks (one per resident slot) take an evenly
    // strided sample of the list, i.e. every length from the longest to the shortest, the others follow in descending
    // order.  In plain descending order each generation of resident blocks has equal lengths and ends at the same
    // moment: every SM stays held for a long stretch at a time, and the short kernels of concurrent streams (sort phases of the
    // next MSM, NTT passes of the h pipeline) wait that long for a slot whatever their priority.  Staggered once, the
    // slots free up continuously and the longest-first property is kept for all but the sampled blocks.
    const uint32_t ntask = task_off[nbuckets];
    const uint32_t nblk = (ntask + blockDim.x - 1) / blockDim.x;
    if (blockIdx.x >= nblk) return;
    uint32_t vb = blockIdx.x;
    const uint32_t stride = nblk / wave;
    if (stride > 1) {
        if (vb < wave) vb *= stride;
        else {
            uint32_t j = vb - wave;
            vb = j < wave * (stride - 1) ? (j / (stride - 1)) * stride + j % (stride - 1) + 1 : wave * stride + (j - wave * (stride - 1));
        }
    }
    uint32_t tid = vb * blockDim.x + threadIdx.x;
    if (tid >= ntask) return;
    uint32_t t = order[tid];
    uint32_t g = task_bucket[t];
    uint32_t t0 = task_off[g], nt = task_off[g + 1] - t0;
    uint32_t lo = offsets[g] + (t - t0) * task_len, end = offsets[g + 1];
    uint32_t hi = lo + task_len < end ? lo + task_len : end;
    // rmw (several input parts, msm_dev_impl): a single-task bucket continues from what the earlier parts left in it
    xyzz_t<F> acc = xyzz_t<F>::identity();
    if (RMW && nt == 1) acc = ld16(buckets + g);
    for (uint32_t k = lo; k < hi; ++k) {
        uint32_t e = entries[k];
        affine_t<F> p = ld16(bases + (e & 0x7FFFFFFFu));
        xyzz_t<F>::madd(acc, p, (e >> 31) != 0);
    }
    if (nt == 1) st16(buckets + g, acc);
    else st16(task_sums + t, acc);
}

template <class F>
__device__ __forceinline__ xyzz_t<F> add_sel(const xyzz_t<F>& a, const xyzz_t<F>& b) {
    if (sizeof(F) == 32) return xyzz_t<F>::add_inl(a, b);      // G1: inline (see k_msm_reduce_segments)
    return xyzz_t<F>::add(a, b);
}

// buckets[g] = sum of the task sums of g, for every multi-task bucket; one block per bucket, grid-strided
template <class F>
__global__ void __launch_bounds__(128) k_msm_merge_tasks(const uint32_t* multi_list, const uint32_t* multi_count,
                                  const uint32_t* task_off, const xyzz_t<F>* task_sums, uint32_t rmw, xyzz_t<F>* buckets) {
    __shared__ xyzz_t<F> sh[128];
    uint32_t cnt = *multi_count;
    for (uint32_t i = blockIdx.x; i < cnt; i += gridDim.x) {
        uint32_t g = multi_list[i];
        uint32_t lo = task_off[g], hi = task_off[g + 1];
        xyzz_t<F> acc = xyzz_t<F>::identity();
        for (uint32_t t = lo + threadIdx.x; t < hi; t += 128) acc = add_sel<F>(acc, ld16(task_sums + t));
        sh[threadIdx.x] = acc;
        __syncthreads();
        for (int s = 64; s > 0; s >>= 1) {
            if ((int)threadIdx.x < s) {
                xyzz_t<F> a = sh[threadIdx.x], b = sh[threadIdx.x + s];
                sh[threadIdx.x] = add_sel<F>(a, b);
            }
            __syncthreads();
        }
        if (threadIdx.x == 0) st16(buckets + g, rmw ? add_sel<F>(ld16(buckets + g), sh[0]) : sh[0]);
        __syncthreads();
    }
}

// the buckets with 2..MERGE_SMALL tasks (n >> 2^c: most of them): one thread per bucket
template <class F>
__global__ void __launch_bounds__(128) k_msm_merge_small(const uint32_t* multi_list, uint32_t list_cap, const uint32_t* small_count,
                                                         const uint32_t* task_off, const xyzz_t<F>* task_sums, uint32_t rmw, xyzz_t<F>* buckets) {
    uint32_t cnt = *small_count;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += gridDim.x * blockDim.x) {
        uint32_t g = multi_list[list_cap - 1 - i];
        uint32_t lo = task_off[g], hi = task_off[g + 1];
        xyzz_t<F> acc = ld16(task_sums + lo);
        for (uint32_t t = lo + 1; t < hi; ++t) acc = add_sel<F>(acc, ld16(task_sums + t));
        if (rmw) acc = add_sel<F>(ld16(buckets + g), acc);
        st16(buckets + g, acc);
    }
}

// ---------------------------------------------------------------------------------------------
// 5. window reduction: S_w = sum_{k<B} (k+1) * bucket[w][k]
// ---------------------------------------------------------------------------------------------
// one thread per (window, segment).  (A quad-cooperative version of this kernel was measured slower at 2^20:
// it is throughput- not latency-bound.)
template <class F>
__global__ void __launch_bounds__(128) k_msm_reduce_segments(const xyzz_t<F>* buckets, uint32_t W, uint32_t B, uint32_t seg_len,
                                      xyzz_t<F>* partials) {
    uint32_t nseg = B / seg_len;
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= W * nseg) return;
    uint32_t w = t / nseg, seg = t % nseg;
    uint32_t lo = seg * seg_len;
    const xyzz_t<F>* bw = buckets + (size_t)w * B;
    xyzz_t<F> run = xyzz_t<F>::identity(), acc = xyzz_t<F>::identity();
    // G1: the group law is inlined here (an out-of-line call moves 3 x 128 B through local memory per
    // operation, which dominated this latency-bound chain); G2 keeps the calls to bound code size.
    constexpr bool INL = sizeof(F) == 32;
    for (uint32_t k = lo + seg_len; k-- > lo;) {
        xyzz_t<F> bk = ld16(bw + k);
        if (INL) { run = xyzz_t<F>::add_inl(run, bk); acc = xyzz_t<F>::add_inl(acc, run); }
        else { run = xyzz_t<F>::add(run, bk); acc = xyzz_t<F>::add(acc, run); }
    }
    if (lo) {   // + lo * run
        xyzz_t<F> m = xyzz_t<F>::identity();
        for (int bit = 31 - __clz(lo); bit >= 0; --bit) {
            if (INL) m = xyzz_t<F>::dbl_inl(m); else m = xyzz_t<F>::dbl(m);
            if ((lo >> bit) & 1) { if (INL) m = xyzz_t<F>::add_inl(m, run); else m = xyzz_t<F>::add(m, run); }
        }
        if (INL) acc = xyzz_t<F>::add_inl(acc, m); else acc = xyzz_t<F>::add(acc, m);
    }
    st16(partials + t, acc);
}

// The same reduction with one QUAD per (window, segment): the (up to 4) independent field products of every level of a point
// operation run in the 4 lanes (quad_ops).  For small bucket sets -- a 30 k-point MSM has ~1000 segments, i.e. 1000 threads each
// running a chain of ~50 dependent point operations on an otherwise empty machine -- the chain is 3-4x shorter (the reference's
// sha256 circuit).  Large bucket sets are throughput-bound and keep the
// one-thread version (see above).
template <class F>
__global__ void __launch_bounds__(128) k_msm_reduce_segments_quad(const xyzz_t<F>* buckets, uint32_t W, uint32_t B, uint32_t seg_len,
                                                                  xyzz_t<F>* partials) {
    typedef quad_ops<F, false> Q;
    __shared__ typename Q::xch_t xch[32];
    typename Q::xch_t* x = &xch[threadIdx.x >> 2];
    const uint32_t nseg = B / seg_len;
    const uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) >> 2;
    if (t >= W * nseg) return;                                     // uniform per quad
    const uint32_t w = t / nseg, seg = t % nseg;
    const uint32_t lo = seg * seg_len;
    const xyzz_t<F>* bw = buckets + (size_t)w * B;
    xyzz_t<F> run = xyzz_t<F>::identity(), acc = xyzz_t<F>::identity();
    for (uint32_t k = lo + seg_len; k-- > lo;) {
        run = Q::add(x, run, ld16(bw + k));
        acc = Q::add(x, acc, run);
    }
    if (lo) {   // + lo * run
        xyzz_t<F> m = xyzz_t<F>::identity();
        for (int bit = 31 - __clz(lo); bit >= 0; --bit) {
            m = Q::dbl(x, m);
            if ((lo >> bit) & 1) m = Q::add(x, m, run);
        }
        acc = Q::add(x, acc, m);
    }
    if ((threadIdx.x & 3) == 0) st16(partials + t, acc);
}

// one block per window: sum nseg partials
template <class F, int THREADS>
__global__ void __launch_bounds__(THREADS) k_msm_window_sum(const xyzz_t<F>* partials, uint32_t nseg, xyzz_t<F>* wsum) {
    __shared__ xyzz_t<F> sh[THREADS];
    const xyzz_t<F>* p = partials + (size_t)blockIdx.x * nseg;
    xyzz_t<F> acc = xyzz_t<F>::identity();
    for (uint32_t i = threadIdx.x; i < nseg; i += THREADS) acc = add_sel<F>(acc, ld16(p + i));
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int s = THREADS / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) {
            xyzz_t<F> a = sh[threadIdx.x], b = sh[threadIdx.x + s];
            sh[threadIdx.x] = add_sel<F>(a, b);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) st16(wsum + blockIdx.x, sh[0]);
}

// 6. Combine.  Fixed-base tables (one bucket set): k_msm_horner with c = 0 adds up the `nset` partial sums of the
// window-sum blocks.  (Without the constant c and its doubling loop ptxas gives the kernel more registers and stack.)
// One quad: the (up to 4) independent field products of each level of a point operation are computed by the 4 lanes
// in the same instruction stream and exchanged through shared memory (quad_ops).
template <class F>
__global__ void __launch_bounds__(32) k_msm_horner(const xyzz_t<F>* wsum, uint32_t nset, uint32_t c, uint32_t first, uint32_t last,
                                                   xyzz_t<F>* state, xyzz_t<F>* out) {
    typedef quad_ops<F, false> Q;
    __shared__ typename Q::xch_t xch;
    if (blockIdx.x != 0 || threadIdx.x >= 4) return;
    xyzz_t<F> total;
    uint32_t k = 0;
    if (first) { total = ld16(wsum); k = 1; }
    else total = ld16(state);
    for (; k < nset; ++k) {
        for (uint32_t j = 0; j < c; ++j) total = Q::dbl(&xch, total);
        total = Q::add(&xch, total, ld16(wsum + k));
    }
    if (threadIdx.x == 0) st16(last ? out : state, total);
}

// Horner over the bucket sets of the GLV digits, in the order k_msm_digits_glv numbers them (top window first).  One
// launch folds the window sums of ONE window group into the running chains kept in `state` (first: the chains start
// here; last: the result goes to `out`), so the c doublings per window of group g run while the bucket kernel of group
// g + 1 occupies the SMs.  Quad 0 runs the chain of the |k1| windows (sets 2k), quad 1 that of the |k2| windows (sets
// 2k + 1) in the same warp (half as many sequential doublings); result = H0 + phi(H1), phi(X, Y, ZZ, ZZZ) =
// (beta X, Y, ZZ, ZZZ) on G1 and (beta^2 X, Y, ZZ, ZZZ) on the twist (glv_phi_x).
template <class F>
__global__ void __launch_bounds__(32) k_msm_horner_glv(const xyzz_t<F>* wsum, uint32_t nwin, uint32_t c, uint32_t first, uint32_t last,
                                                       xyzz_t<F>* state, xyzz_t<F>* out) {
    typedef quad_ops<F, false> Q;
    __shared__ typename Q::xch_t xch[2];
    __shared__ xyzz_t<F> h1;
    if (blockIdx.x != 0 || threadIdx.x >= 8) return;
    const uint32_t half = threadIdx.x >> 2;
    xyzz_t<F> total;
    uint32_t k = 0;
    if (first) { total = ld16(wsum + half); k = 1; }
    else total = ld16(state + half);
    for (; k < nwin; ++k) {
        for (uint32_t j = 0; j < c; ++j) total = Q::dbl(&xch[half], total);
        total = Q::add(&xch[half], total, ld16(wsum + 2 * k + half));
    }
    if (!last) {
        if ((threadIdx.x & 3) == 0) st16(state + half, total);
        return;
    }
    if (threadIdx.x == 4) h1 = total;
    __syncwarp(0xFFu);
    if (half == 0) {
        xyzz_t<F> p = h1;
        if (!p.is_inf()) glv_phi_x(p.x);
        total = Q::add(&xch[0], total, p);
        if (threadIdx.x == 0) st16(out, total);
    }
}

// sum `count` XYZZ points, normalise; out = affine followed by one u64 infinity flag
template <class F>
__global__ void k_sum_to_affine(const xyzz_t<F>* pts, uint32_t count, affine_t<F>* out, uint64_t* flag) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    xyzz_t<F> acc = xyzz_t<F>::identity();
    for (uint32_t i = 0; i < count; ++i) acc = xyzz_t<F>::add(acc, ld16(pts + i));
    affine_t<F> a = xyzz_t<F>::to_affine(acc);
    st16(out, a);
    *flag = acc.is_inf() ? 1 : 0;
}

template <class F>
__global__ void k_set_identity(xyzz_t<F>* out) {
    if (threadIdx.x == 0 && blockIdx.x == 0) st16(out, xyzz_t<F>::identity());
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static unsigned choose_window(size_t n) {
    unsigned lg = ceil_log2(n < 2 ? 2 : n);
    int c = (int)lg - 4;
    if (c < 5) c = 5;
    if (c > 20) c = 20;
    const char* env = getenv("B200ZK_MSM_WINDOW");
    if (env) { int v = atoi(env); if (v >= 2 && v <= 24) c = v; }
    return (unsigned)c;
}

static int exclusive_scan(b200zk_ctx* ctx, cudaStream_t st, const uint32_t* in, uint32_t* out, uint32_t* sums, uint32_t n) {
    uint32_t nblk = (n + SCAN_TILE - 1) / SCAN_TILE;
    {
        LaunchScope ls(ctx, st, "msm_scan");
        k_scan_local<<<nblk, SCAN_THREADS, 0, st>>>(in, out, sums, n);
    }
    {
        LaunchScope ls(ctx, st, "msm_scan");
        k_scan_sums<<<1, SCAN_THREADS, 0, st>>>(sums, nblk);
    }
    {
        LaunchScope ls(ctx, st, "msm_scan");
        k_scan_add<<<nblk, SCAN_THREADS, 0, st>>>(out, sums, n);
    }
    return check_launch(ctx, "scan");
}

// event `idx` of MSM channel `ch` (common.cuh), created on first use; only called under the owning slot's mutex
static cudaEvent_t msm_event(b200zk_ctx* ctx, int ch, size_t idx) {
    std::vector<cudaEvent_t>& v = ctx->msm_events[ch];
    while (v.size() <= idx) {
        cudaEvent_t e = nullptr;
        if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return nullptr;
        v.push_back(e);
    }
    return v[idx];
}

// Streams of one MSM.  `seq`: digit / sort phases and, per window group, merge + bucket reduction + Horner step;
// `acc`: the bucket kernels, on the caller's stream, which the result is ordered on.  `seq` is the channel's
// high-priority side stream.
struct MsmStreams {
    cudaStream_t seq, acc;
    int channel;
};

// One input part of an MSM: `n` pairs, and (host-staged callers) the events that signal the arrival of its scalars / bases.
struct MsmPart {
    const void* bases;
    const void* scalars;
    size_t n;
    cudaEvent_t bases_ready, scalars_ready;
};

// The window-group pipeline (one MSM, no host round trips):
//   seq : digits, scan | prep(0) | prep(1) .. prep(G-1) | wait A0: tail(0) | wait A1: tail(1) | ...
//   acc :                 wait P0: accumulate(0) -> A0 | wait P1: accumulate(1) -> A1 | ...
// prep(g) = task tables + scatter of group g's bucket sets, tail(g) = merge + bucket reduction + window sums + Horner
// step.  Groups hold consecutive bucket sets in Horner order (top windows first), so tail(g) -- a chain of dependent
// point operations that used to follow the bucket kernel (a quarter of a 2^20 MSM) -- overlaps accumulate(g + 1); only
// the last group's tail is exposed.  `seq` has the higher stream priority: its short kernels get the SM slots that
// the running bucket kernel frees, instead of queueing behind it.
//
// Several input PARTS (host-staged MSMs, api.cu): the pairs arrive over PCIe in `nparts` pieces.  Every part is sorted on
// its own (digits / scan / task tables / scatter on seq as soon as its scalars are there) and its bucket kernel ADDS into
// the one shared bucket set as soon as its bases are there (read-modify-write of the XYZZ buckets), so the transfer of
// part p + 1 hides behind the bucket kernel of part p and the reduction / Horner tail runs once.  (Two complete MSMs
// on two streams instead -- two bucket sets, two tails -- were slower.)
template <class F>
static int msm_dev_impl(b200zk_ctx* ctx, const MsmStreams& ms, DevBuf& ws_buf, const MsmPart* parts, unsigned nparts,
                        void* d_out, const char* acc_name, unsigned tab_c = 0) {
    const int ch = ms.channel;
    size_t nev = 0;
    auto next_event = [&]() { return msm_event(ctx, ch, nev++); };
    size_t n = 0, n_max = 0;                                 // all parts together / the largest part
    for (unsigned p = 0; p < nparts; ++p) { n += parts[p].n; n_max = parts[p].n > n_max ? parts[p].n : n_max; }
    xyzz_t<F>* out = reinterpret_cast<xyzz_t<F>*>(d_out);
    if (n == 0) {
        {
            LaunchScope ls(ctx, ms.acc, "msm_small");
            k_set_identity<F><<<1, 32, 0, ms.acc>>>(out);
        }
        return check_launch(ctx, "k_set_identity");
    }
    if (n >= (1ull << 31)) return set_error(ctx, B200ZK_ERR_ARG, "MSM length must be < 2^31");
    // tab_c != 0: the bases are a fixed-base table of msm_table_windows(tab_c) x n points (section 7); all digit windows
    // then share one bucket set and the Horner chain disappears
    const bool fold = tab_c != 0;
    if (fold && nparts != 1) return set_error(ctx, B200ZK_ERR_ARG, "fixed-base tables take one input part");
    const unsigned c = fold ? tab_c : choose_window(n);
    // every other MSM splits its scalars (glv.cuh; G2: the same split, phi = (beta^2 x, y))
    const unsigned Wh = (128 + c - 1) / c;                   // |k1|, |k2| < 2^127: Wh * c >= 128 leaves the carry room
    const unsigned W = fold ? msm_table_windows(c) : 2 * Wh; // digit windows
    const unsigned WB = fold ? 1 : W;                        // bucket sets
    if ((uint64_t)W * n >= (fold ? (1ull << 31) : (1ull << 32)))
        return set_error(ctx, B200ZK_ERR_ARG, "MSM too large for 32-bit bucket offsets / entry indices (W * n)");
    const uint32_t B = 1u << (c - 1);
    const uint32_t nb = WB * B;
    uint32_t seg_len = B < 16 ? B : 16;
    // Small bucket sets (<= 8192 16-bucket segments in all: a 30 k-point MSM, the small windows of a 2^16 one) are reduced by one
    // QUAD per segment (k_msm_reduce_segments_quad) and, being pure latency chains, in 8-bucket segments whatever the caller's
    // hint: 16 + ~16 dependent point operations per segment instead of 64 + ~15 with the 32-bucket segments a 2^20 proof prefers.
    const bool quad_reduce = (uint64_t)WB * (B / seg_len) <= 8192;
    if (quad_reduce) seg_len = B < 8 ? B : 8;
    else if (ctx->msm_seg_hint && ctx->msm_seg_hint <= B) seg_len = ctx->msm_seg_hint;
    const uint32_t nseg = B / seg_len;
    // fold (one bucket set): the segment partials are summed by `wsplit` blocks whose results the Horner kernel adds up
    const uint32_t wsplit = fold ? (nseg >= 16 * 256 ? 16 : (nseg >= 1024 ? 4 : 1)) : 1;

    // window groups: consecutive bucket sets (whole windows, i.e. both GLV halves).  Measured on an earlier GPU:
    // at 2^20 the extra launches, the drain bubble at the end of every bucket kernel and the slowdown of the latency-bound
    // tail kernels when they share SMs with a bucket kernel cost more than the hidden tail saves (1 group beats 2 and 4);
    // from 2^22 up four groups win; uneven groups lose.  Fixed-base tables have one bucket set;
    // several input parts already cut the bucket work into pieces.
    const unsigned unit_sets = fold ? 1 : 2;
    const unsigned units = fold ? 1 : Wh;                    // windows
    unsigned ngroups = 1;
    if (!fold && nparts == 1 && n >= (1u << 22)) ngroups = units < 4 ? units : 4;
    auto group_first_unit = [&](unsigned g) { return (unsigned)(((uint64_t)units * g) / ngroups); };   // balanced split
    const uint32_t rmw = nparts > 1 ? 1u : 0u;               // bucket kernels add into the shared buckets

    // Streams.  One group and one part (every MSM of a proof, the 2^20 benchmark point): nothing to overlap inside the MSM, so
    // everything runs in order on the caller's stream -- a high-priority side stream would only let this MSM's
    // reductions take SM time from the bucket kernels of the proof's other MSMs (measured: a slower 2^20 proof).
    // Otherwise `seq` (the side stream) runs sort + tail and `acc` the bucket kernels.
    const bool split_streams = ngroups > 1 || nparts > 1;
    const cudaStream_t st = split_streams ? ms.seq : ms.acc, ast = ms.acc;
    if (split_streams) {                  // inputs were produced in `acc`-stream order
        cudaEvent_t e = next_event();
        if (!e) return set_error(ctx, B200ZK_ERR_CUDA, "cudaEventCreate failed");
        B2_CUDA_OK(ctx, cudaEventRecord(e, ast));
        B2_CUDA_OK(ctx, cudaStreamWaitEvent(st, e, 0));
    }
    auto finish = [&]() -> int {          // the result (written on seq) becomes visible in `acc`-stream order
        if (split_streams) {
            cudaEvent_t e = next_event();
            if (!e) return set_error(ctx, B200ZK_ERR_CUDA, "cudaEventCreate failed");
            B2_CUDA_OK(ctx, cudaEventRecord(e, st));
            B2_CUDA_OK(ctx, cudaStreamWaitEvent(ast, e, 0));
        }
        return B200ZK_OK;
    };

    // workspace carve-up (256-byte aligned): the sort arrays once per part, the bucket set and the reduction buffers once
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    // task length: 128 unless the average bucket is already that long (n >> 2^c: every bucket would be cut in two);
    // then the next power of two above 3x the average -- only outliers are split -- as long as that leaves enough
    // tasks (>= 2^19) to fill the machine
    const size_t total_max = (size_t)W * n_max;
    uint32_t task_len = TASK_LEN;
    while (task_len < MAX_TASK_LEN && (uint64_t)task_len * nb < 3 * (uint64_t)total_max &&
           total_max / (2 * task_len) + nb >= (1u << 19))
        task_len *= 2;
    // Small inputs cannot fill the machine with 128-entry tasks, and a real witness (29 821 of the 29 823 entries of the
    // reference's sha256 witness are 0 or 1, groth16/examples/sha256.rs:182-185) puts thousands of entries into ONE bucket:
    // 118 serial chains of 128 additions for a 30 k-point MSM.  Shorter tasks turn that bucket into ~900 parallel
    // chains of 16 plus a block-level tree (k_msm_merge_tasks); buckets that stay below 16 entries are unaffected.
    if (n_max <= (1u << 16))
        while (task_len > 16 && total_max / task_len < (1u << 17)) task_len /= 2;
    const size_t max_tasks = total_max / task_len + nb + ngroups;             // per part, all groups together
    size_t o = 0;
    auto carve = [&](size_t bytes) { size_t r = o; o += al(bytes); return r; };
    struct PartWs { size_t keys, ranks, entries, counts, offsets, ntasks, taskoff, taskbucket, multi, hist, rank, order, tasksums; };
    std::vector<PartWs> pw(nparts);
    for (unsigned p = 0; p < nparts; ++p) {
        const size_t total = (size_t)W * parts[p].n;
        pw[p].keys = carve(total * 4); pw[p].ranks = carve(total * 4); pw[p].entries = carve(total * 4);
        pw[p].counts = carve(((size_t)nb + 1) * 4); pw[p].offsets = carve(((size_t)nb + 1) * 4);
        pw[p].ntasks = carve(((size_t)nb + ngroups) * 4); pw[p].taskoff = carve(((size_t)nb + ngroups) * 4);
        pw[p].taskbucket = carve(max_tasks * 4);
        pw[p].multi = carve((total_max / task_len + 4 * ngroups + 4) * 4);
        pw[p].hist = carve((size_t)ngroups * (MAX_TASK_LEN + 1) * 4);
        pw[p].rank = carve(max_tasks * 4); pw[p].order = carve(max_tasks * 4);
        pw[p].tasksums = carve(max_tasks * sizeof(xyzz_t<F>));
    }
    const size_t o_sums = carve(((size_t)nb / SCAN_TILE + 2) * 4);
    const size_t o_buckets = carve((size_t)nb * sizeof(xyzz_t<F>));
    const size_t o_partials = carve((size_t)WB * nseg * sizeof(xyzz_t<F>));
    const size_t o_wsum = carve((size_t)WB * wsplit * sizeof(xyzz_t<F>));
    const size_t o_state = carve(2 * sizeof(xyzz_t<F>));
    B2_CUDA_OK(ctx, ws_buf.reserve(o));
    char* ws = reinterpret_cast<char*>(ws_buf.p);
    uint32_t* sums = reinterpret_cast<uint32_t*>(ws + o_sums);
    xyzz_t<F>* buckets = reinterpret_cast<xyzz_t<F>*>(ws + o_buckets);
    xyzz_t<F>* partials = reinterpret_cast<xyzz_t<F>*>(ws + o_partials);
    xyzz_t<F>* wsum = reinterpret_cast<xyzz_t<F>*>(ws + o_wsum);
    xyzz_t<F>* hstate = reinterpret_cast<xyzz_t<F>*>(ws + o_state);
    B2_CUDA_OK(ctx, cudaMemsetAsync(buckets, 0, (size_t)nb * sizeof(xyzz_t<F>), st));   // all-zero XYZZ = identity
    cudaEvent_t buckets_clear = nullptr;
    if (rmw) {                                               // the first bucket kernel reads the buckets it adds into
        buckets_clear = next_event();
        if (!buckets_clear) return set_error(ctx, B200ZK_ERR_CUDA, "cudaEventCreate failed");
        B2_CUDA_OK(ctx, cudaEventRecord(buckets_clear, st));
        B2_CUDA_OK(ctx, cudaStreamWaitEvent(ast, buckets_clear, 0));
    }

    // per-group views of the task tables (same geometry for every part)
    struct Group {
        uint32_t set0, nsets, b0, nbk;          // bucket sets [set0, set0 + nsets), buckets [b0, b0 + nbk)
        size_t task_cap, task_base;             // task arrays: [task_base, task_base + task_cap)
        uint32_t list_cap; size_t list_base;    // multi-task bucket list
    };
    std::vector<Group> groups(ngroups);
    {
        size_t tb = 0, lb = 2 * (size_t)ngroups;
        for (unsigned g = 0; g < ngroups; ++g) {
            Group& G = groups[g];
            const unsigned u0 = group_first_unit(g), u1 = group_first_unit(g + 1);
            G.set0 = u0 * unit_sets; G.nsets = (u1 - u0) * unit_sets;
            G.b0 = G.set0 * B; G.nbk = G.nsets * B;
            const size_t gtotal = fold ? total_max : (size_t)G.nsets * n_max;
            G.task_cap = gtotal / task_len + G.nbk + 1;
            G.task_base = tb; tb += G.task_cap;
            G.list_cap = (uint32_t)(gtotal / task_len + 1);
            G.list_base = lb; lb += G.list_cap;
        }
    }
    std::vector<cudaEvent_t> prepped((size_t)nparts * ngroups), accumulated((size_t)nparts * ngroups);
    for (auto& e : prepped) if (!(e = next_event())) return set_error(ctx, B200ZK_ERR_CUDA, "cudaEventCreate failed");
    for (auto& e : accumulated) if (!(e = next_event())) return set_error(ctx, B200ZK_ERR_CUDA, "cudaEventCreate failed");

    for (unsigned p = 0; p < nparts; ++p) {
        const MsmPart& P = parts[p];
        const size_t np = P.n, total = (size_t)W * np;
        uint32_t* keys = reinterpret_cast<uint32_t*>(ws + pw[p].keys);
        uint32_t* ranks = reinterpret_cast<uint32_t*>(ws + pw[p].ranks);
        uint32_t* entries = reinterpret_cast<uint32_t*>(ws + pw[p].entries);
        uint32_t* counts = reinterpret_cast<uint32_t*>(ws + pw[p].counts);
        uint32_t* offsets = reinterpret_cast<uint32_t*>(ws + pw[p].offsets);
        uint32_t* ntasks_all = reinterpret_cast<uint32_t*>(ws + pw[p].ntasks);
        uint32_t* task_off_all = reinterpret_cast<uint32_t*>(ws + pw[p].taskoff);
        uint32_t* task_bucket_all = reinterpret_cast<uint32_t*>(ws + pw[p].taskbucket);
        uint32_t* multi_all = reinterpret_cast<uint32_t*>(ws + pw[p].multi);
        uint32_t* hist_all = reinterpret_cast<uint32_t*>(ws + pw[p].hist);
        uint32_t* task_rank_all = reinterpret_cast<uint32_t*>(ws + pw[p].rank);
        uint32_t* order_all = reinterpret_cast<uint32_t*>(ws + pw[p].order);
        xyzz_t<F>* task_sums_all = reinterpret_cast<xyzz_t<F>*>(ws + pw[p].tasksums);
        if (np == 0) {                                           // nothing to add: keep the event chain intact
            for (unsigned g = 0; g < ngroups; ++g) {
                B2_CUDA_OK(ctx, cudaEventRecord(prepped[(size_t)p * ngroups + g], st));
                B2_CUDA_OK(ctx, cudaEventRecord(accumulated[(size_t)p * ngroups + g], ast));
            }
            continue;
        }
        // ---- digits + scan of part p on seq (its scalars may still be arriving) ----------------------------------------------
        if (P.scalars_ready) B2_CUDA_OK(ctx, cudaStreamWaitEvent(st, P.scalars_ready, 0));
        B2_CUDA_OK(ctx, cudaMemsetAsync(counts, 0, ((size_t)nb + 1) * 4, st));
        {
            LaunchScope ls(ctx, st, "msm_digits");
            if (fold) k_msm_digits<<<(unsigned)((np + 255) / 256), 256, 0, st>>>(reinterpret_cast<const Fr*>(P.scalars), (uint32_t)np, c, W,
                                                                               keys, ranks, counts);
            else k_msm_digits_glv<<<(unsigned)((np + 255) / 256), 256, 0, st>>>(reinterpret_cast<const Fr*>(P.scalars), (uint32_t)np, c,
                                                                                Wh, keys, ranks, counts);
        }
        B2_TRY(check_launch(ctx, "k_msm_digits"));
        B2_TRY(exclusive_scan(ctx, st, counts, offsets, sums, nb + 1));
        B2_CUDA_OK(ctx, cudaMemsetAsync(multi_all, 0, (size_t)ngroups * 8, st));          // [2 g], [2 g + 1] = big / small counts
        B2_CUDA_OK(ctx, cudaMemsetAsync(hist_all, 0, (size_t)ngroups * (MAX_TASK_LEN + 1) * 4, st));

        // ---- prep(g): task tables (counting sort of the <= task_len-entry tasks by length) + scatter, on seq ----------------
        for (unsigned g = 0; g < ngroups; ++g) {
            const Group& G = groups[g];
            uint32_t* ntasks = ntasks_all + G.b0 + g;               // nbk + 1 entries per group
            uint32_t* task_off = task_off_all + G.b0 + g;
            uint32_t* task_bucket = task_bucket_all + G.task_base;
            uint32_t* task_rank = task_rank_all + G.task_base;
            uint32_t* order = order_all + G.task_base;
            uint32_t* hist = hist_all + (size_t)g * (MAX_TASK_LEN + 1);
            {
                LaunchScope ls(ctx, st, "msm_tasks");
                k_msm_task_counts<<<(G.nbk + 1 + 255) / 256, 256, 0, st>>>(offsets + G.b0, G.nbk, task_len, ntasks);
            }
            B2_TRY(check_launch(ctx, "k_msm_task_counts"));
            B2_TRY(exclusive_scan(ctx, st, ntasks, task_off, sums, G.nbk + 1));
            {
                LaunchScope ls(ctx, st, "msm_tasks");
                k_msm_fill_tasks<<<(G.nbk + 255) / 256, 256, 0, st>>>(task_off, G.nbk, task_bucket, multi_all + G.list_base, G.list_cap,
                                                                      multi_all + 2 * g);
            }
            B2_TRY(check_launch(ctx, "k_msm_fill_tasks"));
            {
                LaunchScope ls(ctx, st, "msm_tasks");
                k_msm_task_hist<<<(unsigned)((G.task_cap + 255) / 256), 256, 0, st>>>(offsets + G.b0, task_off, task_bucket, G.nbk, task_len, hist, task_rank);
            }
            {
                LaunchScope ls(ctx, st, "msm_tasks");
                k_msm_task_hist_scan<<<1, 1, 0, st>>>(hist, task_len);
            }
            {
                LaunchScope ls(ctx, st, "msm_tasks");
                k_msm_task_order<<<(unsigned)((G.task_cap + 255) / 256), 256, 0, st>>>(offsets + G.b0, task_off, task_bucket, G.nbk, task_len, hist, task_rank, order);
            }
            B2_TRY(check_launch(ctx, "k_msm_task_order"));
            {
                const size_t t0 = fold ? 0 : (size_t)G.set0 * np, cnt = fold ? total : (size_t)G.nsets * np;
                LaunchScope ls(ctx, st, "msm_scatter");
                k_msm_scatter<<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(keys, ranks, offsets, (uint32_t)np, t0, cnt, fold ? 1u : 0u, entries);
            }
            B2_TRY(check_launch(ctx, "k_msm_scatter"));
            B2_CUDA_OK(ctx, cudaEventRecord(prepped[(size_t)p * ngroups + g], st));
        }

        // ---- accumulate(g) of part p on acc: the sort phases above only read the scalars, the (2-4x larger) base array of a
        //      host-staged part may still be on its way and signals its arrival here ------------------------------------------------
        if (P.bases_ready) B2_CUDA_OK(ctx, cudaStreamWaitEvent(ast, P.bases_ready, 0));
        for (unsigned g = 0; g < ngroups; ++g) {
            const Group& G = groups[g];
            B2_CUDA_OK(ctx, cudaStreamWaitEvent(ast, prepped[(size_t)p * ngroups + g], 0));
            {
                LaunchScope ls(ctx, ast, acc_name);
                const unsigned grid = (unsigned)((G.task_cap + 127) / 128);
                const uint32_t wave = (uint32_t)ctx->sm_count * (sizeof(F) > 32 ? ACC_MINBLOCKS_G2 : ACC_MINBLOCKS);
                const affine_t<F>* bp = reinterpret_cast<const affine_t<F>*>(P.bases);
                if (rmw) k_msm_accumulate<F, true><<<grid, 128, 0, ast>>>(bp, entries, offsets + G.b0, task_off_all + G.b0 + g, task_bucket_all + G.task_base,
                                                                       order_all + G.task_base, G.nbk, task_len, wave, buckets + G.b0, task_sums_all + G.task_base);
                else k_msm_accumulate<F, false><<<grid, 128, 0, ast>>>(bp, entries, offsets + G.b0, task_off_all + G.b0 + g, task_bucket_all + G.task_base,
                                                                        order_all + G.task_base, G.nbk, task_len, wave, buckets + G.b0, task_sums_all + G.task_base);
            }
            B2_TRY(check_launch(ctx, "k_msm_accumulate"));
            if (rmw) {
                // several parts: the next part's bucket kernel reads what this part's merges write, so they stay on `acc`
                {
                    LaunchScope ls(ctx, ast, "msm_merge");
                    k_msm_merge_tasks<F><<<2 * ctx->sm_count, 128, 0, ast>>>(multi_all + G.list_base, multi_all + 2 * g, task_off_all + G.b0 + g,
                                                                            task_sums_all + G.task_base, rmw, buckets + G.b0);
                }
                {
                    LaunchScope ls(ctx, ast, "msm_merge");
                    k_msm_merge_small<F><<<4 * ctx->sm_count, 128, 0, ast>>>(multi_all + G.list_base, G.list_cap, multi_all + 2 * g + 1,
                                                                            task_off_all + G.b0 + g, task_sums_all + G.task_base, rmw, buckets + G.b0);
                }
                B2_TRY(check_launch(ctx, "k_msm_merge_tasks"));
            }
            B2_CUDA_OK(ctx, cudaEventRecord(accumulated[(size_t)p * ngroups + g], ast));
        }
    }
    // ---- tail(g) on seq: merge, bucket reduction, window sums, Horner step ----------------------------------------------
    for (unsigned g = 0; g < ngroups; ++g) {
        const Group& G = groups[g];
        for (unsigned p = 0; p < nparts; ++p) B2_CUDA_OK(ctx, cudaStreamWaitEvent(st, accumulated[(size_t)p * ngroups + g], 0));
        if (!rmw) {
            uint32_t* multi_all = reinterpret_cast<uint32_t*>(ws + pw[0].multi);
            uint32_t* task_off = reinterpret_cast<uint32_t*>(ws + pw[0].taskoff) + G.b0 + g;
            xyzz_t<F>* task_sums = reinterpret_cast<xyzz_t<F>*>(ws + pw[0].tasksums) + G.task_base;
            {
                LaunchScope ls(ctx, st, "msm_merge");
                k_msm_merge_tasks<F><<<2 * ctx->sm_count, 128, 0, st>>>(multi_all + G.list_base, multi_all + 2 * g, task_off, task_sums, 0u, buckets + G.b0);
            }
            {
                LaunchScope ls(ctx, st, "msm_merge");
                k_msm_merge_small<F><<<4 * ctx->sm_count, 128, 0, st>>>(multi_all + G.list_base, G.list_cap, multi_all + 2 * g + 1, task_off, task_sums,
                                                                       0u, buckets + G.b0);
            }
            B2_TRY(check_launch(ctx, "k_msm_merge_tasks"));
        }
        {
            LaunchScope ls(ctx, st, "msm_reduce");
            if (quad_reduce)                                       // latency-bound: fewer segments than the machine has warps
                k_msm_reduce_segments_quad<F><<<(G.nsets * nseg * 4 + 127) / 128, 128, 0, st>>>(buckets + G.b0, G.nsets, B, seg_len,
                                                                                               partials + (size_t)G.set0 * nseg);
            else
                k_msm_reduce_segments<F><<<(G.nsets * nseg + 127) / 128, 128, 0, st>>>(buckets + G.b0, G.nsets, B, seg_len,
                                                                                      partials + (size_t)G.set0 * nseg);
        }
        B2_TRY(check_launch(ctx, "k_msm_reduce_segments"));
        {
            LaunchScope ls(ctx, st, "msm_window_sum");
            constexpr int T = sizeof(F) > 32 ? 128 : 256;
            // fold: the single bucket set's partials are summed by `wsplit` blocks, then added up by the Horner kernel
            // with zero doublings per step
            k_msm_window_sum<F, T><<<G.nsets * wsplit, T, 0, st>>>(partials + (size_t)G.set0 * nseg, nseg / wsplit, wsum + (size_t)G.set0 * wsplit);
        }
        B2_TRY(check_launch(ctx, "k_msm_window_sum"));
        {
            LaunchScope ls(ctx, st, "msm_combine");
            const uint32_t first = g == 0, last = g + 1 == ngroups;
            if (fold) k_msm_horner<F><<<1, 32, 0, st>>>(wsum, wsplit, 0u, first, last, hstate, out);
            else k_msm_horner_glv<F><<<1, 32, 0, st>>>(wsum + G.set0, G.nsets / 2, c, first, last, hstate, out);
        }
        B2_TRY(check_launch(ctx, "k_msm_horner"));
    }
    return finish();
}

// single-part convenience wrapper
template <class F>
static int msm_dev_impl(b200zk_ctx* ctx, const MsmStreams& ms, DevBuf& ws_buf, const void* d_bases, const void* d_scalars, size_t n,
                        void* d_out, const char* acc_name, cudaEvent_t bases_ready, cudaEvent_t scalars_ready = nullptr,
                        unsigned tab_c = 0) {
    const MsmPart part{d_bases, d_scalars, n, bases_ready, scalars_ready};
    return msm_dev_impl<F>(ctx, ms, ws_buf, &part, 1, d_out, acc_name, tab_c);
}

static MsmStreams slot_streams(b200zk_ctx* ctx, Slot& sl, int aux) {
    const int ch = 2 * (int)(&sl - ctx->slots) + (aux ? 1 : 0);
    return MsmStreams{ctx->msm_side[ch], aux ? sl.aux_stream : sl.stream, ch};
}

int msm_g1_dev(b200zk_ctx* ctx, Slot& sl, const void* d_bases, const void* d_scalars, size_t n, void* d_out,
               cudaEvent_t bases_ready, int aux) {
    return msm_dev_impl<Fq>(ctx, slot_streams(ctx, sl, aux), aux ? sl.ws_msm_aux : sl.ws_msm, d_bases, d_scalars, n, d_out,
                            "msm_accumulate_g1", bases_ready);
}
int msm_g2_dev(b200zk_ctx* ctx, Slot& sl, const void* d_bases, const void* d_scalars, size_t n, void* d_out,
               cudaEvent_t bases_ready, int aux) {
    return msm_dev_impl<Fq2>(ctx, slot_streams(ctx, sl, aux), aux ? sl.ws_msm_aux : sl.ws_msm, d_bases, d_scalars, n, d_out,
                             "msm_accumulate_g2", bases_ready);
}

// ---------------------------------------------------------------------------------------------
// 7. fixed-base window tables.  A proving key's query vectors never change between proofs, and an H100 has the HBM
//    to keep table[w * n + i] = 2^{c w} * P_i for every digit window w: the digit (w, d) of scalar i then adds
//    table[w * n + i] into bucket d of ONE bucket set -- no per-window bucket sets, no Horner doublings -- which lets
//    c grow to ~log2(n) (13 bucket additions per scalar at c = 20 instead of 16) for the same reduction cost.
// ---------------------------------------------------------------------------------------------
unsigned msm_table_windows(unsigned c) { return (255 + c - 1) / c; }
// Window for n fixed bases: about log2(n) (the bucket reduction then costs what the 13-17 additions per scalar save),
// in [10, 20], preferring a c whose top digit window still has >= 6 bits: a 2-3 bit top window sends n / 4 entries
// to each of a handful of buckets, which serialises the histogram atomics of k_msm_digits (c = 18 against c = 20)
unsigned msm_table_auto_window(size_t n) {
    int L = (int)ceil_log2(n < 2 ? 2 : n);
    L = L < 10 ? 10 : (L > 20 ? 20 : L);
    const int cand[4] = {L, L - 1, L + 1, L - 2};
    for (int c : cand) {
        if (c < 10 || c > 20) continue;
        int top = 254 - ((int)msm_table_windows((unsigned)c) - 1) * c;
        if (top >= 6) return (unsigned)c;
    }
    return (unsigned)L;
}

template <class F>
__global__ void __launch_bounds__(128) k_msm_table_build(const affine_t<F>* bases, uint32_t n, uint32_t c, uint32_t W,
                                                         affine_t<F>* table) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    affine_t<F> p = ld16(bases + i);
    st16(table + i, p);
    for (uint32_t w = 1; w < W; ++w) {
        if (!p.is_inf()) {
            xyzz_t<F> acc = xyzz_t<F>::from_affine(p);
            for (uint32_t k = 0; k < c; ++k) acc = xyzz_t<F>::dbl(acc);
            p = xyzz_t<F>::to_affine(acc);
        }
        st16(table + (size_t)w * n + i, p);
    }
}

template <class F>
static int table_build_impl(b200zk_ctx* ctx, cudaStream_t st, const void* d_bases, size_t n, unsigned c, void* d_table) {
    if (c < 2 || c > 24) return set_error(ctx, B200ZK_ERR_ARG, "table window must be in [2, 24]");
    if (n == 0) return B200ZK_OK;
    const unsigned W = msm_table_windows(c);
    if ((uint64_t)W * n >= (1ull << 31)) return set_error(ctx, B200ZK_ERR_ARG, "table too large (W * n >= 2^31)");
    {
        LaunchScope ls(ctx, st, "msm_table_build");
        k_msm_table_build<F><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(reinterpret_cast<const affine_t<F>*>(d_bases), (uint32_t)n,
                                                                      c, W, reinterpret_cast<affine_t<F>*>(d_table));
    }
    return check_launch(ctx, "k_msm_table_build");
}
int msm_table_build_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_bases, size_t n, unsigned c, void* d_table) {
    return g2 ? table_build_impl<Fq2>(ctx, sl.stream, d_bases, n, c, d_table)
              : table_build_impl<Fq>(ctx, sl.stream, d_bases, n, c, d_table);
}
int msm_table_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_table, const void* d_scalars, size_t n, unsigned c,
                  void* d_out, int aux) {
    if (c < 2 || c > 24) return set_error(ctx, B200ZK_ERR_ARG, "table window must be in [2, 24]");
    const MsmStreams st = slot_streams(ctx, sl, aux);
    DevBuf& ws = aux ? sl.ws_msm_aux : sl.ws_msm;
    return g2 ? msm_dev_impl<Fq2>(ctx, st, ws, d_table, d_scalars, n, d_out, "msm_accumulate_g2", nullptr, nullptr, c)
              : msm_dev_impl<Fq>(ctx, st, ws, d_table, d_scalars, n, d_out, "msm_accumulate_g1", nullptr, nullptr, c);
}

// Host-staged MSM in `nparts` pieces (api.cu): d_bases / d_scalars are the device staging buffers the caller is filling on its copy
// stream; cnt[p] pairs per piece, ev_scalars[p] / ev_bases[p] recorded after the piece's scalars / bases have been queued.  One bucket
// set, one reduction tail: see msm_dev_impl.
int msm_parts_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_bases, const void* d_scalars, const size_t* cnt, unsigned nparts,
                  const cudaEvent_t* ev_scalars, const cudaEvent_t* ev_bases, void* d_out) {
    if (nparts == 0 || nparts > 16) return set_error(ctx, B200ZK_ERR_ARG, "1..16 input parts");
    MsmPart parts[16];
    const size_t PB = g2 ? 128 : 64;
    size_t lo = 0;
    for (unsigned p = 0; p < nparts; ++p) {
        parts[p] = MsmPart{reinterpret_cast<const char*>(d_bases) + lo * PB, reinterpret_cast<const char*>(d_scalars) + lo * 32, cnt[p],
                           ev_bases ? ev_bases[p] : nullptr, ev_scalars ? ev_scalars[p] : nullptr};
        lo += cnt[p];
    }
    return g2 ? msm_dev_impl<Fq2>(ctx, slot_streams(ctx, sl, 0), sl.ws_msm, parts, nparts, d_out, "msm_accumulate_g2")
              : msm_dev_impl<Fq>(ctx, slot_streams(ctx, sl, 0), sl.ws_msm, parts, nparts, d_out, "msm_accumulate_g1");
}

// out = sum of `count` XYZZ points at pts[i * stride] (no normalisation): combines gathered per-rank partials
template <class F>
__global__ void k_sum_xyzz(const xyzz_t<F>* pts, uint32_t count, uint32_t stride, xyzz_t<F>* out) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    xyzz_t<F> acc = xyzz_t<F>::identity();
    for (uint32_t i = 0; i < count; ++i) acc = xyzz_t<F>::add(acc, ld16(pts + (size_t)i * stride));
    st16(out, acc);
}
int xyzz_sum_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_in, size_t count, size_t stride, void* d_out) {
    {
        LaunchScope ls(ctx, sl.stream, "point_sum");
        if (g2) k_sum_xyzz<Fq2><<<1, 32, 0, sl.stream>>>((const xyzz_t<Fq2>*)d_in, (uint32_t)count, (uint32_t)stride, (xyzz_t<Fq2>*)d_out);
        else k_sum_xyzz<Fq><<<1, 32, 0, sl.stream>>>((const xyzz_t<Fq>*)d_in, (uint32_t)count, (uint32_t)stride, (xyzz_t<Fq>*)d_out);
    }
    return check_launch(ctx, "k_sum_xyzz");
}

template <class F>
static int sum_impl(b200zk_ctx* ctx, Slot& sl, const void* d_xyzz, size_t count, void* d_out_affine) {
    affine_t<F>* out = reinterpret_cast<affine_t<F>*>(d_out_affine);
    {
        LaunchScope ls(ctx, sl.stream, "point_normalise");
        k_sum_to_affine<F><<<1, 32, 0, sl.stream>>>(reinterpret_cast<const xyzz_t<F>*>(d_xyzz), (uint32_t)count, out,
                                                     reinterpret_cast<uint64_t*>(out + 1));
    }
    return check_launch(ctx, "k_sum_to_affine");
}
int g1_sum_dev(b200zk_ctx* ctx, Slot& sl, const void* d, size_t count, void* d_out) { return sum_impl<Fq>(ctx, sl, d, count, d_out); }
int g2_sum_dev(b200zk_ctx* ctx, Slot& sl, const void* d, size_t count, void* d_out) { return sum_impl<Fq2>(ctx, sl, d, count, d_out); }

// ---------------------------------------------------------------------------------------------
// 8. d_msm's exchange as ONE kernel over peer memory (the king's gather + `unpackexp` + sum + scatter of
//    dist-primitives/src/dmsm/mod.rs:87-97, and round 1's all-gather + host-synchronising sum): every rank stores its XYZZ
//    partial into slot [parity][rank] of every peer's mailbox (NVLink stores), raises the slot's sequence flag, waits until
//    all slots of its own mailbox carry this step's sequence number, adds the partials up and normalises.  No NCCL call, no
//    host round trip; the two parities alternate so a fast peer's next partial never overwrites one still being read (a rank
//    publishes step s + 1 only after its own sum of step s, and nobody can pass step s + 1 before everyone published it).
//    Mailbox layout (bytes): [2][MAX_PEERS] slots of 256 B, then [2][MAX_PEERS] u64 flags.
// ---------------------------------------------------------------------------------------------
static const uint32_t XCH_MAX_PEERS = 8, XCH_SLOT = 256;
struct PeerMailboxes { char* box[XCH_MAX_PEERS]; };

__device__ __forceinline__ void st_release_sys(uint64_t* p, uint64_t v) { asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ uint64_t ld_acquire_sys(const uint64_t* p) {
    uint64_t v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

template <class F>
__global__ void __launch_bounds__(32) k_msm_exchange_sum(const xyzz_t<F>* partial, PeerMailboxes peers, uint32_t n_peers, uint32_t rank,
                                                         uint64_t seq, affine_t<F>* out, uint64_t* out_flag) {
    const uint32_t par = (uint32_t)(seq & 1), lane = threadIdx.x;
    constexpr uint32_t WORDS = sizeof(xyzz_t<F>) / 16;               // uint4 per partial: 8 (G1) or 16 (G2)
    const uint4* src = reinterpret_cast<const uint4*>(partial);
    // publish: lanes spread over (peer, 16-byte word); then one release-store of the flag per peer
    for (uint32_t i = lane; i < n_peers * WORDS; i += 32) {
        const uint32_t p = i / WORDS, w = i % WORDS;
        reinterpret_cast<uint4*>(peers.box[p] + (size_t)(par * XCH_MAX_PEERS + rank) * XCH_SLOT)[w] = src[w];
    }
    __threadfence_system();
    __syncwarp();
    if (lane < n_peers) {
        uint64_t* flags = reinterpret_cast<uint64_t*>(peers.box[lane] + 2 * XCH_MAX_PEERS * XCH_SLOT);
        st_release_sys(flags + par * XCH_MAX_PEERS + rank, seq);
    }
    // wait for every rank's partial of this step in my own mailbox
    char* mine = peers.box[rank];
    const uint64_t* my_flags = reinterpret_cast<const uint64_t*>(mine + 2 * XCH_MAX_PEERS * XCH_SLOT);
    if (lane < n_peers) {
        while (ld_acquire_sys(my_flags + par * XCH_MAX_PEERS + lane) < seq) __nanosleep(200);
    }
    __syncwarp();
    if (lane != 0) return;
    xyzz_t<F> acc = xyzz_t<F>::identity();
    for (uint32_t g = 0; g < n_peers; ++g) {
        xyzz_t<F> v;
        const volatile uint4* s4 = reinterpret_cast<const volatile uint4*>(mine + (size_t)(par * XCH_MAX_PEERS + g) * XCH_SLOT);
        uint4* d4 = reinterpret_cast<uint4*>(&v);
        for (uint32_t w = 0; w < WORDS; ++w) { uint4 t; t.x = s4[w].x; t.y = s4[w].y; t.z = s4[w].z; t.w = s4[w].w; d4[w] = t; }
        acc = xyzz_t<F>::add(acc, v);
    }
    st16(out, xyzz_t<F>::to_affine(acc));
    *out_flag = acc.is_inf() ? 1 : 0;
}

int msm_exchange_sum_dev(b200zk_ctx* ctx, Slot& sl, int g2, const void* d_partial, void* const* peer_boxes, unsigned n_peers, unsigned rank,
                         uint64_t seq, void* d_out_affine) {
    if (n_peers == 0 || n_peers > XCH_MAX_PEERS || rank >= n_peers || seq == 0) return set_error(ctx, B200ZK_ERR_ARG, "bad peer exchange geometry");
    PeerMailboxes pm;
    for (unsigned g = 0; g < XCH_MAX_PEERS; ++g) pm.box[g] = g < n_peers ? reinterpret_cast<char*>(peer_boxes[g]) : nullptr;
    {
        LaunchScope ls(ctx, sl.stream, "msm_exchange_sum");
        if (g2) {
            affine_t<Fq2>* o = reinterpret_cast<affine_t<Fq2>*>(d_out_affine);
            k_msm_exchange_sum<Fq2><<<1, 32, 0, sl.stream>>>(reinterpret_cast<const xyzz_t<Fq2>*>(d_partial), pm, n_peers, rank, seq, o, reinterpret_cast<uint64_t*>(o + 1));
        } else {
            affine_t<Fq>* o = reinterpret_cast<affine_t<Fq>*>(d_out_affine);
            k_msm_exchange_sum<Fq><<<1, 32, 0, sl.stream>>>(reinterpret_cast<const xyzz_t<Fq>*>(d_partial), pm, n_peers, rank, seq, o, reinterpret_cast<uint64_t*>(o + 1));
        }
    }
    return check_launch(ctx, "k_msm_exchange_sum");
}

// ---------------------------------------------------------------------------------------------
// deterministic dummy inputs + element-wise self-test
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}

// P_i = k_i * G, k_i = splitmix64(seed + i) | 1
template <class F>
__global__ void __launch_bounds__(128) k_generate_points(uint64_t seed, size_t n, affine_t<F>* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t k = splitmix64(seed + i) | 1ULL;
    affine_t<F> g = curve_generator<F>();
    xyzz_t<F> acc = xyzz_t<F>::identity();
    for (int bit = 63; bit >= 0; --bit) {
        acc = xyzz_t<F>::dbl(acc);
        if ((k >> bit) & 1) xyzz_t<F>::madd(acc, g, false);
    }
    st16(out + i, xyzz_t<F>::to_affine(acc));
}

__global__ void k_generate_fr(uint64_t seed, size_t n, Fr* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t v[4];
    for (int k = 0; k < 4; ++k) v[k] = splitmix64(seed * 0x100000001B3ULL + 4 * (uint64_t)i + k);
    v[3] &= 0x3FFFFFFFFFFFFFFFULL;
    uint32_t t[8];
    for (int k = 0; k < 4; ++k) { t[2 * k] = (uint32_t)v[k]; t[2 * k + 1] = (uint32_t)(v[k] >> 32); }
    Fr r;
    Fr::final_sub(r, t);      // v < 2^254 < 2r
    st16(out + i, r);
}

template <class F>
__global__ void k_field_op(int op, const F* a, const F* b, F* out, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    F x = ld16(a + i), y = ld16(b + i), r;
    if (op == 0) r = F::mul(x, y);
    else if (op == 1) r = F::add(x, y);
    else r = F::sub(x, y);
    st16(out + i, r);
}

int generate_points_dev(b200zk_ctx* ctx, Slot& sl, int g2, uint64_t seed, size_t n, void* d_out) {
    if (n == 0) return B200ZK_OK;
    {
        LaunchScope ls(ctx, sl.stream, "generate_points");
        unsigned grid = (unsigned)((n + 127) / 128);
        if (g2) k_generate_points<Fq2><<<grid, 128, 0, sl.stream>>>(seed, n, reinterpret_cast<affine_t<Fq2>*>(d_out));
        else k_generate_points<Fq><<<grid, 128, 0, sl.stream>>>(seed, n, reinterpret_cast<affine_t<Fq>*>(d_out));
    }
    return check_launch(ctx, "k_generate_points");
}
int generate_fr_dev(b200zk_ctx* ctx, Slot& sl, uint64_t seed, size_t n, void* d_out) {
    if (n == 0) return B200ZK_OK;
    {
        LaunchScope ls(ctx, sl.stream, "generate_fr");
        k_generate_fr<<<(unsigned)((n + 255) / 256), 256, 0, sl.stream>>>(seed, n, reinterpret_cast<Fr*>(d_out));
    }
    return check_launch(ctx, "k_generate_fr");
}
int field_op_dev(b200zk_ctx* ctx, Slot& sl, int field, int op, const void* d_a, const void* d_b, void* d_out, size_t n) {
    if (n == 0) return B200ZK_OK;
    {
        LaunchScope ls(ctx, sl.stream, "field_op");
        unsigned grid = (unsigned)((n + 255) / 256);
        if (field == 0) k_field_op<Fq><<<grid, 256, 0, sl.stream>>>(op, (const Fq*)d_a, (const Fq*)d_b, (Fq*)d_out, n);
        else k_field_op<Fr><<<grid, 256, 0, sl.stream>>>(op, (const Fr*)d_a, (const Fr*)d_b, (Fr*)d_out, n);
    }
    return check_launch(ctx, "k_field_op");
}

}  // namespace b200zk
