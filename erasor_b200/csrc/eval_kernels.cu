// eval_kernels.cu -- PR / RR of a static map on the device: the four counts of erasor_b200/evaluate.py (the reference's
// scripts/analysis_runner.py) by an exact grid-indexed 1-NN from every ground-truth point into the estimate, and the C ABI
// around it (erasor_eval_*, include/erasor_b200.h).  DESIGN.md section 11 has the contract and the exactness argument;
// tests/test_eval_grid_model.py restates every kernel in numpy.
//
//   k_eval_bounds         one pass over the estimate (and its keep mask): min / max of the selected points, non-finite flag
//   (host)                eval_grid_setup: cell edge voxelsize, doubled until the 3x3x3 block provably holds every point within thr
//   k_eval_keys           cell key per estimate point, 0xFFFFFFFF for points the keep mask drops
//   k_eval_radix_*        device-wide stable LSD radix sort of (key, index), 8-bit digits, only the passes the key width needs
//   k_eval_heads_*        run heads of the sorted keys -> vox_key[nv], vox_start[nv + 1]
//   k_eval_query          per GT point: 9 contiguous key ranges, exact double distances, lowest-index ties, counters
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>

#include "../../include/erasor_b200.h"
#include "device_common.cuh"

namespace erasor {

constexpr int      kThreads   = 256;
constexpr int      kWarps     = kThreads / 32;
constexpr uint32_t kSeg       = 4096;          // points per warp segment of the radix sort
constexpr uint32_t kHeadChunk = 4096;          // points per CTA chunk of the run-head scan
constexpr uint32_t kNoKey     = 0xFFFFFFFFu;   // key of an estimate point the keep mask drops: sorts behind every cell key

// The kernels' parameter types stay outside the anonymous namespace, so the kernels' symbol names are stable.
// device-side scalars of one call
struct EvalStats {
    uint32_t mn[3], mx[3];        // float_to_ordered min / max of the selected estimate points
    uint32_t n_sel;               // selected estimate points
    uint32_t bad;                 // bit 0: non-finite coordinate in a selected estimate point, bit 1: in a GT point
    uint32_t nv;                  // occupied cells
    uint32_t pad_;
    unsigned long long cnt[6];    // gt_static, gt_dynamic, preserved_static, preserved_dynamic, inliers, ambiguous_ties
};

// the cell grid, set up on the host by eval_grid_setup
struct EvalGrid {
    float  leaf, inv;             // cell edge and fl(1 / leaf)
    int    min_b[3], div[3];      // first cell and cell count per axis (keys: i + j div[0] + k div[0] div[1], < 2^32 - 1)
    float  lo[3], hi[3];          // guard window on fl(x * inv): a GT point outside it has no occupied cell within reach
    float  thr2f;                 // (float)(thr * thr), for the conservative range skip
    double thr;                   // inlier radius voxelsize * sqrt(3) / 2
};

namespace {

// SemanticKITTI dynamic classes 252..259 carried in the intensity: numpy's astype(np.uint32) & 0xFFFF on x86-64 is
// (uint32_t)(int64_t)v; NaN, +-inf and |v| >= 2^63 convert to 0x8000000000000000 there, i.e. class 0.
__device__ __forceinline__ bool is_dynamic(float v) {
    if (!(fabsf(v) < 9223372036854775808.0f)) return false;
    const uint32_t s = (uint32_t)(long long)v & 0xFFFFu;
    return s >= 252u && s <= 259u;
}

__device__ __forceinline__ bool finite3(float4 p) { return isfinite(p.x) && isfinite(p.y) && isfinite(p.z); }

__device__ __forceinline__ uint32_t cell_key(const EvalGrid& g, int i, int j, int k) {
    return (uint32_t)i + (uint32_t)j * (uint32_t)g.div[0] + (uint32_t)k * ((uint32_t)g.div[0] * (uint32_t)g.div[1]);
}

// rank of this thread's flag among the CTA's set flags (thread order); `round` = how many are set
__device__ __forceinline__ uint32_t cta_rank(bool f, uint32_t* s_w /*[kWarps]*/, uint32_t& round) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned bal = __ballot_sync(FULL_MASK, f);
    __syncthreads();                                  // s_w may still be read from the previous round
    if (lane == 0) s_w[warp] = __popc(bal);
    __syncthreads();
    uint32_t before = 0u;
    round = 0u;
    for (int w = 0; w < kWarps; ++w) { const uint32_t c = s_w[w]; if (w < warp) before += c; round += c; }
    return before + __popc(bal & ((1u << lane) - 1u));
}

}  // namespace

// ---- 1. bounds of the selected estimate points -----------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) k_eval_bounds(const float4* __restrict__ est, const uint8_t* __restrict__ keep, uint32_t n,
                                                          EvalStats* __restrict__ st) {
    uint32_t mn[3] = {~0u, ~0u, ~0u}, mx[3] = {0u, 0u, 0u}, sel = 0u, bad = 0u;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        if (keep && !keep[i]) continue;
        const float4 p = est[i];
        ++sel;
        if (!finite3(p)) { bad = 1u; continue; }
        const uint32_t o[3] = {float_to_ordered(p.x + 0.0f), float_to_ordered(p.y + 0.0f), float_to_ordered(p.z + 0.0f)};   // -0 -> +0
#pragma unroll
        for (int k = 0; k < 3; ++k) { mn[k] = min(mn[k], o[k]); mx[k] = max(mx[k], o[k]); }
    }
    sel = __reduce_add_sync(FULL_MASK, sel);
    bad = __reduce_or_sync(FULL_MASK, bad);
#pragma unroll
    for (int k = 0; k < 3; ++k) { mn[k] = __reduce_min_sync(FULL_MASK, mn[k]); mx[k] = __reduce_max_sync(FULL_MASK, mx[k]); }
    if ((threadIdx.x & 31) == 0 && sel) {
        atomicAdd(&st->n_sel, sel);
        if (bad) atomicOr(&st->bad, 1u);
        for (int k = 0; k < 3; ++k) { atomicMin(&st->mn[k], mn[k]); atomicMax(&st->mx[k], mx[k]); }
    }
}

// ---- 3. cell keys ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) k_eval_keys(const float4* __restrict__ est, const uint8_t* __restrict__ keep, uint32_t n, EvalGrid g,
                                                        uint32_t* __restrict__ key, uint32_t* __restrict__ idx) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        uint32_t k = kNoKey;
        if (!keep || keep[i]) {
            const float4 p = est[i];      // inside [mn, mx]: fl(x * inv) is monotonic in x, so every cell lies in [0, div)
            k = cell_key(g, voxel_cell(p.x, g.inv, g.min_b[0]), voxel_cell(p.y, g.inv, g.min_b[1]), voxel_cell(p.z, g.inv, g.min_b[2]));
        }
        key[i] = k;
        idx[i] = (uint32_t)i;
    }
}

// ---- radix sort, per pass: digit counts per warp segment, then each digit's row scanned, then a stable scatter ------------
__global__ void __launch_bounds__(kThreads) k_eval_radix_hist(const uint32_t* __restrict__ key, uint32_t n, uint32_t nseg, int shift,
                                                              uint32_t* __restrict__ cnt /*[256][nseg]*/) {
    __shared__ uint32_t s_h[kWarps][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t seg = blockIdx.x * kWarps + warp;
    uint32_t* h = s_h[warp];
    for (int d = lane; d < 256; d += 32) h[d] = 0u;
    __syncwarp();
    if (seg >= nseg) return;
    const uint32_t b0 = seg * kSeg, b1 = (uint32_t)min((unsigned long long)n, (unsigned long long)b0 + kSeg);
    for (uint32_t o = lane; o < b1 - b0; o += 32u) atomicAdd(&h[(key[b0 + o] >> shift) & 255u], 1u);   // offsets: b0 + o cannot wrap
    __syncwarp();
    for (int d = lane; d < 256; d += 32) cnt[(size_t)d * nseg + seg] = h[d];
}

// one warp per digit: its row of per-segment counts becomes exclusive prefixes in place, tot[d] = the digit's total
__global__ void __launch_bounds__(kThreads) k_eval_radix_rows(uint32_t* __restrict__ cnt, uint32_t nseg, uint32_t* __restrict__ tot) {
    const int lane = threadIdx.x & 31;
    const uint32_t d = blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (d >= 256u) return;
    uint32_t* row = cnt + (size_t)d * nseg;
    uint32_t carry = 0u;
    for (uint32_t c0 = 0; c0 < nseg; c0 += 512u) {                  // 16 consecutive counters per lane and round
        const uint32_t a = c0 + (uint32_t)lane * 16u;
        uint32_t v[16], sum = 0u;
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] = (a + j < nseg) ? row[a + j] : 0u;
#pragma unroll
        for (int j = 0; j < 16; ++j) { const uint32_t t = v[j]; v[j] = sum; sum += t; }
        uint32_t incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(FULL_MASK, incl, o); if (lane >= o) incl += t; }
        const uint32_t base = carry + incl - sum;
#pragma unroll
        for (int j = 0; j < 16; ++j) if (a + j < nseg) row[a + j] = base + v[j];
        carry += __shfl_sync(FULL_MASK, incl, 31);
    }
    if (lane == 0) tot[d] = carry;
}

// one warp per segment: points of digit d go to (points of smaller digits) + (points of d in earlier segments) + (rank of
// the point among the segment's points of d, in order) -- stable
__global__ void __launch_bounds__(kThreads) k_eval_radix_scatter(const uint32_t* __restrict__ ki, const uint32_t* __restrict__ ii,
                                                                 uint32_t* __restrict__ ko, uint32_t* __restrict__ io, uint32_t n, uint32_t nseg,
                                                                 int shift, const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ tot) {
    __shared__ uint32_t s_c[kWarps][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t seg = blockIdx.x * kWarps + warp;
    if (seg >= nseg) return;
    uint32_t* my_c = s_c[warp];
    {
        constexpr int DL = 256 / 32;                       // digits per lane
        uint32_t t[DL], c[DL], sum = 0u;
#pragma unroll
        for (int j = 0; j < DL; ++j) { t[j] = tot[lane * DL + j]; c[j] = cnt[(size_t)(lane * DL + j) * nseg + seg]; }
#pragma unroll
        for (int j = 0; j < DL; ++j) { const uint32_t x = t[j]; t[j] = sum; sum += x; }
        uint32_t incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t x = __shfl_up_sync(FULL_MASK, incl, o); if (lane >= o) incl += x; }
#pragma unroll
        for (int j = 0; j < DL; ++j) my_c[lane * DL + j] = incl - sum + t[j] + c[j];
    }
    __syncwarp();
    const uint32_t b0 = seg * kSeg, b1 = (uint32_t)min((unsigned long long)n, (unsigned long long)b0 + kSeg);
    for (uint32_t o0 = 0; o0 < b1 - b0; o0 += 32u) {
        const uint32_t e = b0 + o0 + lane;
        const bool valid = o0 + lane < b1 - b0;
        const unsigned vm = __ballot_sync(FULL_MASK, valid);
        if (valid) {
            const uint32_t k = ki[e], v = ii[e];
            const uint32_t d = (k >> shift) & 255u;
            const unsigned peers = __match_any_sync(vm, d);
            const uint32_t base = my_c[d];
            __syncwarp(vm);
            if (lane == __ffs(peers) - 1) my_c[d] = base + __popc(peers);
            const uint32_t o = base + __popc(peers & ((1u << lane) - 1u));
            ko[o] = k;
            io[o] = v;
        }
        __syncwarp();
    }
}

// ---- 4. run heads of the sorted keys: count per chunk, one CTA scans the counts, ordered scatter -----------------------------
__global__ void __launch_bounds__(kThreads) k_eval_heads_count(const uint32_t* __restrict__ skey, uint32_t n, uint32_t* __restrict__ chunk) {
    __shared__ uint32_t s_w[kWarps];
    const uint32_t b0 = blockIdx.x * kHeadChunk, b1 = (uint32_t)min((unsigned long long)n, (unsigned long long)b0 + kHeadChunk);
    uint32_t c = 0u;
    for (uint32_t o = threadIdx.x; o < b1 - b0; o += kThreads) { const uint32_t i = b0 + o; c += (i == 0 || skey[i] != skey[i - 1]) ? 1u : 0u; }
    c = __reduce_add_sync(FULL_MASK, c);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0u;
        for (int w = 0; w < kWarps; ++w) t += s_w[w];
        chunk[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(1024) k_eval_heads_scan(uint32_t* __restrict__ chunk, uint32_t nch, EvalStats* __restrict__ st) {
    __shared__ uint32_t s_part[34];
    const uint32_t t = block_excl_scan(chunk, chunk, (int)nch, s_part);
    if (threadIdx.x == 0) st->nv = t;
}

__global__ void __launch_bounds__(kThreads) k_eval_heads_scatter(const uint32_t* __restrict__ skey, uint32_t n, const uint32_t* __restrict__ chunk,
                                                                 const EvalStats* __restrict__ st, uint32_t* __restrict__ vox_key,
                                                                 uint32_t* __restrict__ vox_start) {
    __shared__ uint32_t s_w[kWarps];
    const uint32_t b0 = blockIdx.x * kHeadChunk, b1 = (uint32_t)min((unsigned long long)n, (unsigned long long)b0 + kHeadChunk);
    uint32_t base = chunk[blockIdx.x];
    for (uint32_t o0 = 0; o0 < b1 - b0; o0 += kThreads) {
        const uint32_t i = b0 + o0 + threadIdx.x;
        const bool hd = o0 + threadIdx.x < b1 - b0 && (i == 0 || skey[i] != skey[i - 1]);
        uint32_t round;
        const uint32_t r = cta_rank(hd, s_w, round);
        if (hd) { vox_key[base + r] = skey[i]; vox_start[base + r] = i; }
        base += round;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) vox_start[st->nv] = n;
}

// ---- 5. the query: one GT point per thread ---------------------------------------------------------------------------------
// Every estimate point within thr of q lies in the 3x3x3 block of cells around q's cell (eval_grid_setup), and keys are
// contiguous in x, so the block is 9 key ranges (i-1..i+1, j+b, k+c), each found with one lower bound.  A range whose
// conservative gap in y and z is at least thr holds no inlier candidate and is skipped.  Distances are sklearn's, in double
// without contraction: sqrt((dx*dx + dy*dy) + dz*dz).  Ties go to the lowest estimate index.
__global__ void __launch_bounds__(kThreads) k_eval_query(const float4* __restrict__ gt, uint32_t n_gt, const float4* __restrict__ est,
                                                         const uint32_t* __restrict__ order, const uint32_t* __restrict__ vox_start,
                                                         const uint32_t* __restrict__ vox_key, EvalGrid g, uint32_t* __restrict__ match,
                                                         EvalStats* __restrict__ st) {
    __shared__ uint32_t s_c[kWarps][7];
    const uint32_t nv = st->nv;
    uint32_t c[7] = {0u, 0u, 0u, 0u, 0u, 0u, 0u};         // the six counts of EvalStats::cnt, then the non-finite flag
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_gt) {
        const float4 q = gt[i];
        uint32_t best_i = kNoPoint;
        if (!finite3(q)) {
            c[6] = 2u;
        } else {
            const bool q_dyn = is_dynamic(q.w);
            c[0] = q_dyn ? 0u : 1u;
            c[1] = q_dyn ? 1u : 0u;
            double best = __longlong_as_double(0x7FF0000000000000LL);
            bool best_dyn = false, tie_dyn = false, tie_sta = false;
            const float ax = FM(q.x, g.inv), ay = FM(q.y, g.inv), az = FM(q.z, g.inv);
            // guard before any float -> int conversion: outside the window every cell of q's 3x3x3 block is outside the grid
            if (nv && ax >= g.lo[0] && ax < g.hi[0] && ay >= g.lo[1] && ay < g.hi[1] && az >= g.lo[2] && az < g.hi[2]) {
                const int ci = voxel_cell(q.x, g.inv, g.min_b[0]), cj = voxel_cell(q.y, g.inv, g.min_b[1]), ck = voxel_cell(q.z, g.inv, g.min_b[2]);
                const int i0 = max(ci - 1, 0), i1 = min(ci + 1, g.div[0] - 1);
                const float slack = 1.0e-3f * g.leaf + 4.0e-6f * fmaxf(fabsf(q.y), fabsf(q.z));
                const double qx = q.x, qy = q.y, qz = q.z;
                for (int tb = 0; tb < 3 && i0 <= i1; ++tb) {                  // offsets 0, -1, +1: q's own row first
                    const int b = (tb == 0) ? 0 : (tb == 1 ? -1 : 1), jj = cj + b;
                    if (jj < 0 || jj >= g.div[1]) continue;
                    const float gy = cell_gap(q.y, jj + g.min_b[1], b, g.leaf, slack);
                    for (int tc = 0; tc < 3; ++tc) {
                        const int cc = (tc == 0) ? 0 : (tc == 1 ? -1 : 1), kk = ck + cc;
                        if (kk < 0 || kk >= g.div[2]) continue;
                        const float gz = cell_gap(q.z, kk + g.min_b[2], cc, g.leaf, slack);
                        // skip the range when even its nearest face is provably beyond thr, or strictly farther than the best
                        // so far (then it cannot even hold a tie); 0.999 covers the float rounding of the gaps and of (float)best
                        const float gap2 = 0.999f * (gy * gy + gz * gz);
                        if (gap2 >= g.thr2f || gap2 > (float)best) continue;
                        const uint32_t k_lo = cell_key(g, i0, jj, kk), k_hi = k_lo + (uint32_t)(i1 - i0);
                        uint32_t lo = 0, hi = nv;                     // first cell with vox_key >= k_lo
                        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (vox_key[mid] < k_lo) lo = mid + 1; else hi = mid; }
                        uint32_t v1 = lo;
                        while (v1 < nv && vox_key[v1] <= k_hi) ++v1;
                        if (v1 == lo) continue;
                        const uint32_t e = vox_start[v1];
                        for (uint32_t k = vox_start[lo]; k < e; ++k) {
                            const uint32_t j = order[k];
                            const float4 p = est[j];
                            const double dx = __dsub_rn(qx, (double)p.x), dy = __dsub_rn(qy, (double)p.y), dz = __dsub_rn(qz, (double)p.z);
                            const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
                            if (d2 > best) continue;
                            const bool p_dyn = is_dynamic(p.w);
                            if (d2 < best) {
                                best = d2; best_i = j; best_dyn = p_dyn; tie_dyn = p_dyn; tie_sta = !p_dyn;
                            } else {
                                tie_dyn |= p_dyn; tie_sta |= !p_dyn;
                                if (j < best_i) { best_i = j; best_dyn = p_dyn; }
                            }
                        }
                    }
                }
            }
            if (best_i != kNoPoint && __dsqrt_rn(best) < g.thr) {
                c[4] = 1u;
                if (!q_dyn && !best_dyn) c[2] = 1u;
                if (q_dyn && best_dyn) c[3] = 1u;
                if (tie_dyn && tie_sta) c[5] = 1u;
            } else {
                best_i = kNoPoint;
            }
        }
        if (match) match[i] = best_i;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 6; ++k) c[k] = __reduce_add_sync(FULL_MASK, c[k]);
    c[6] = __reduce_or_sync(FULL_MASK, c[6]);
    if (lane == 0) for (int k = 0; k < 7; ++k) s_c[warp][k] = c[k];
    __syncthreads();
    if (threadIdx.x < 7) {
        uint32_t t = 0u;
        for (int w = 0; w < kWarps; ++w) t = (threadIdx.x == 6) ? (t | s_c[w][6]) : (t + s_c[w][threadIdx.x]);
        if (threadIdx.x == 6) { if (t) atomicOr(&st->bad, t); }
        else if (t) atomicAdd(&st->cnt[threadIdx.x], (unsigned long long)t);
    }
}

}  // namespace erasor

// ============================================================================================================================
// C ABI
// ============================================================================================================================
using namespace erasor;

namespace {
struct DevBuf {
    void* p = nullptr; size_t cap = 0;
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) { cudaFree(p); p = nullptr; cap = 0; }
        const size_t want = bytes + bytes / 4 + 4096;
        const cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};
thread_local std::string g_eval_err;
}  // namespace

struct erasor_eval_ctx {
    int device = 0;
    cudaStream_t st = nullptr;
    std::string err;
    DevBuf gt, est, keep, match;              // staging of host inputs / the match output
    DevBuf key_a, key_b, idx_a, idx_b;        // 16 B per estimate point: the sort's ping-pong; the free half holds vox_key / vox_start
    DevBuf cnt, chunk, stats;                 // per-segment digit counts + digit totals, per-chunk head counts, EvalStats
    EvalStats* h_stats = nullptr;             // pinned
    int sm_count = 132;
};

namespace {
#define ECK(call) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) { e->err = std::string(#call) + ": " + cudaGetErrorString(e__); return ERASOR_E_CUDA; } } while (0)

int fail(erasor_eval_t e, int rc, const char* msg) { e->err = msg; return rc; }

// Cell edge: voxelsize, doubled until (a) the cell count fits a 32-bit key below 0xFFFFFFFF, (b) every coordinate the query
// converts scales below 2^22 cells, so floorf, the int conversion and voxel_cell's subtraction are exact, and (c) the float
// cell assignment puts every estimate point within thr of a GT point q into q's 3x3x3 block.
// (c), the rounding margin: a = fl(x * fl(1 / leaf)) = (x / leaf)(1 + e0)(1 + e1), |e0|, |e1| <= 2^-24, so |a - x / leaf| <=
// |x| / leaf * 2^-22.99.  For |p|, |q| <= R along an axis, |a_p - a_q| < (|p - q| + R * 2^-21) / leaf, and |a_p - a_q| < 1 gives
// |floor(a_p) - floor(a_q)| <= 1.  An inlier has sqrt(d2) < thr in double, so its true distance is below thr (1 + 2^-50).  Hence
// the rule  thr (1 + 1e-12) + R * 2^-21 < leaf,  with R bounding both the estimate points and every GT point inside the guard
// window (cells min_b - 2 .. min_b + div + 1): R = (max |cell| + 3) * leaf.
bool eval_grid_setup(const float mn[3], const float mx[3], double voxelsize, EvalGrid& g) {
    const double thr = voxelsize * 1.7320508075688772 / 2.0;
    float leaf = (float)voxelsize;
    for (int it = 0; it < 300 && std::isfinite(leaf) && leaf > 0.0f; ++it, leaf *= 2.0f) {
        const float inv = 1.0f / leaf;
        unsigned long long cells = 1ull;
        double cmax = 0.0;
        bool ok = true;
        for (int k = 0; k < 3 && ok; ++k) {
            const float a = std::floor(mn[k] * inv), b = std::floor(mx[k] * inv);
            if (!(std::fabs(a) < 4194304.0f && std::fabs(b) < 4194304.0f)) { ok = false; break; }   // 2^22
            g.min_b[k] = (int)a;
            g.div[k] = (int)b - (int)a + 1;
            cells *= (unsigned long long)g.div[k];
            ok = cells <= 0xFFFFFFFEull;
            cmax = std::max(cmax, std::max(std::fabs((double)a), std::fabs((double)b) + 1.0));
        }
        if (!ok) continue;
        const double R = (cmax + 3.0) * (double)leaf;
        if (!(thr * (1.0 + 1e-12) + R * (1.0 / 2097152.0) < (double)leaf)) continue;
        g.leaf = leaf;
        g.inv = inv;
        for (int k = 0; k < 3; ++k) { g.lo[k] = (float)(g.min_b[k] - 2); g.hi[k] = (float)(g.min_b[k] + g.div[k] + 2); }
        g.thr = thr;
        g.thr2f = (float)(thr * thr);
        return true;
    }
    return false;
}

int grid_for(int n, int per_cta) { return std::max(1, (n + per_cta - 1) / per_cta); }
// ceil(n / per) in 64 bits: n may be up to 2^32 - 2, where n + per - 1 wraps in uint32
uint32_t ceil_div(uint64_t n, uint64_t per) { return (uint32_t)((n + per - 1) / per); }
}  // namespace

extern "C" {

int erasor_eval_create(int device, erasor_eval_t* out) {
    if (!out) { g_eval_err = "null argument"; return ERASOR_E_INVALID; }
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); g_eval_err = "no CUDA device"; return ERASOR_E_CUDA; }
    if (device < 0 || device >= ndev) { g_eval_err = "device index out of range"; return ERASOR_E_INVALID; }
    erasor_eval_ctx* e = new erasor_eval_ctx();
    e->device = device;
    cudaError_t c = cudaSetDevice(device);
    if (c == cudaSuccess) c = cudaStreamCreateWithFlags(&e->st, cudaStreamNonBlocking);
    if (c == cudaSuccess) c = cudaMallocHost(&e->h_stats, sizeof(EvalStats));
    if (c == cudaSuccess) c = e->stats.ensure(sizeof(EvalStats));
    if (c == cudaSuccess) c = cudaDeviceGetAttribute(&e->sm_count, cudaDevAttrMultiProcessorCount, device);
    if (c != cudaSuccess) {
        g_eval_err = std::string("erasor_eval_create: ") + cudaGetErrorString(c);
        erasor_eval_destroy(e);
        return ERASOR_E_CUDA;
    }
    *out = e;
    return ERASOR_OK;
}

void erasor_eval_destroy(erasor_eval_t e) {
    if (!e) return;
    cudaSetDevice(e->device);
    if (e->st) cudaStreamSynchronize(e->st);
    for (DevBuf* b : {&e->gt, &e->est, &e->keep, &e->match, &e->key_a, &e->key_b, &e->idx_a, &e->idx_b, &e->cnt, &e->chunk, &e->stats}) b->release();
    if (e->h_stats) cudaFreeHost(e->h_stats);
    if (e->st) cudaStreamDestroy(e->st);
    delete e;
}

const char* erasor_eval_last_error(erasor_eval_t e) { return e ? e->err.c_str() : g_eval_err.c_str(); }

int erasor_evaluate(erasor_eval_t e, const float* gt_xyzi, size_t n_gt, const float* est_xyzi, size_t n_est, const uint8_t* est_keep,
                    double voxelsize, int ptr_kind, uint32_t* match, erasor_eval_counts_t* out) {
    if (!e) return ERASOR_E_INVALID;
    e->err.clear();
    if (!out) return fail(e, ERASOR_E_INVALID, "null counts pointer");
    if ((n_gt && !gt_xyzi) || (n_est && !est_xyzi)) return fail(e, ERASOR_E_INVALID, "null cloud pointer");
    if (ptr_kind != ERASOR_PTR_HOST && ptr_kind != ERASOR_PTR_DEVICE) return fail(e, ERASOR_E_INVALID, "ptr_kind must be ERASOR_PTR_HOST or ERASOR_PTR_DEVICE");
    if (!(voxelsize > 0.0) || !std::isfinite(voxelsize) || !std::isfinite((float)voxelsize)) return fail(e, ERASOR_E_INVALID, "voxelsize must be positive and finite");
    if (n_est >= 0xFFFFFFFFull || n_gt >= 0xFFFFFFFFull) return fail(e, ERASOR_E_INVALID, "n_gt and n_est must be below 2^32 - 1");
    ECK(cudaSetDevice(e->device));
    const bool dev = ptr_kind == ERASOR_PTR_DEVICE;
    const uint32_t ng = (uint32_t)n_gt, ne = (uint32_t)n_est;
    const float4* d_gt = reinterpret_cast<const float4*>(gt_xyzi);
    const float4* d_est = reinterpret_cast<const float4*>(est_xyzi);
    const uint8_t* d_keep = est_keep;
    if (dev) {
        if ((reinterpret_cast<uintptr_t>(gt_xyzi) | reinterpret_cast<uintptr_t>(est_xyzi)) & 15u)
            return fail(e, ERASOR_E_INVALID, "device clouds must be 16-byte aligned (one float4 per point)");
    } else {
        if (ng) { ECK(e->gt.ensure(sizeof(float4) * n_gt)); ECK(cudaMemcpyAsync(e->gt.p, gt_xyzi, sizeof(float4) * n_gt, cudaMemcpyHostToDevice, e->st)); d_gt = e->gt.as<float4>(); }
        if (ne) { ECK(e->est.ensure(sizeof(float4) * n_est)); ECK(cudaMemcpyAsync(e->est.p, est_xyzi, sizeof(float4) * n_est, cudaMemcpyHostToDevice, e->st)); d_est = e->est.as<float4>(); }
        if (ne && est_keep) { ECK(e->keep.ensure(n_est)); ECK(cudaMemcpyAsync(e->keep.p, est_keep, n_est, cudaMemcpyHostToDevice, e->st)); d_keep = e->keep.as<uint8_t>(); }
    }
    if (!ne) d_keep = nullptr;
    EvalStats* d_st = e->stats.as<EvalStats>();
    EvalStats* h = e->h_stats;
    std::memset(h, 0, sizeof(EvalStats));
    for (int k = 0; k < 3; ++k) h->mn[k] = ~0u;
    ECK(cudaMemcpyAsync(d_st, h, sizeof(EvalStats), cudaMemcpyHostToDevice, e->st));

    // 1. bounds, read back for the grid set-up
    const int g_stream = e->sm_count * 8;
    if (ne) k_eval_bounds<<<std::min(grid_for((int)std::min<uint32_t>(ne, 1u << 30), kThreads), g_stream), kThreads, 0, e->st>>>(d_est, d_keep, ne, d_st);
    ECK(cudaGetLastError());
    ECK(cudaMemcpyAsync(h, d_st, sizeof(EvalStats), cudaMemcpyDeviceToHost, e->st));
    ECK(cudaStreamSynchronize(e->st));
    if (h->bad & 1u) return fail(e, ERASOR_E_INVALID, "non-finite x, y or z in a selected estimate point");
    const uint32_t n_sel = h->n_sel;

    EvalGrid g{};
    const uint32_t *order = nullptr, *vox_start = nullptr, *vox_key = nullptr;
    if (n_sel) {
        // 2. grid
        float mn[3], mx[3];
        for (int k = 0; k < 3; ++k) { mn[k] = ordered_to_float(h->mn[k]); mx[k] = ordered_to_float(h->mx[k]); }
        if (!eval_grid_setup(mn, mx, voxelsize, g)) return fail(e, ERASOR_E_INVALID, "no cell grid covers the estimate's extent");
        unsigned long long cells = 1ull;
        for (int k = 0; k < 3; ++k) cells *= (unsigned long long)g.div[k];
        // 3. keys + radix sort: only the passes the key width needs (dropped points' 0xFFFFFFFF keeps its all-ones low bits,
        //    which exceed every cell key of that width, so they sort behind the selected points)
        const size_t words = (size_t)ne + 1;
        ECK(e->key_a.ensure(4 * words)); ECK(e->key_b.ensure(4 * words));
        ECK(e->idx_a.ensure(4 * words)); ECK(e->idx_b.ensure(4 * words));
        const uint32_t nseg = ceil_div(ne, kSeg);
        ECK(e->cnt.ensure(sizeof(uint32_t) * (256ull * nseg + 256ull)));
        uint32_t* cnt = e->cnt.as<uint32_t>();
        uint32_t* tot = cnt + 256ull * nseg;
        k_eval_keys<<<std::min(grid_for((int)std::min<uint32_t>(ne, 1u << 30), kThreads), g_stream), kThreads, 0, e->st>>>(d_est, d_keep, ne, g,
                                                                                                                          e->key_a.as<uint32_t>(), e->idx_a.as<uint32_t>());
        ECK(cudaGetLastError());
        int bits = 1;
        while (bits < 32 && (1ull << bits) <= cells) ++bits;          // cells < 2^bits: the largest cell key is below 2^bits - 1
        const int npass = (bits + 7) / 8;
        const int seg_ctas = (int)((nseg + kWarps - 1) / kWarps);
        for (int pass = 0; pass < npass; ++pass) {
            const uint32_t* ki = (pass & 1) ? e->key_b.as<uint32_t>() : e->key_a.as<uint32_t>();
            const uint32_t* ii = (pass & 1) ? e->idx_b.as<uint32_t>() : e->idx_a.as<uint32_t>();
            uint32_t* ko = (pass & 1) ? e->key_a.as<uint32_t>() : e->key_b.as<uint32_t>();
            uint32_t* io = (pass & 1) ? e->idx_a.as<uint32_t>() : e->idx_b.as<uint32_t>();
            k_eval_radix_hist<<<seg_ctas, kThreads, 0, e->st>>>(ki, ne, nseg, 8 * pass, cnt);
            k_eval_radix_rows<<<256 / kWarps, kThreads, 0, e->st>>>(cnt, nseg, tot);
            k_eval_radix_scatter<<<seg_ctas, kThreads, 0, e->st>>>(ki, ii, ko, io, ne, nseg, 8 * pass, cnt, tot);
            ECK(cudaGetLastError());
        }
        const uint32_t* skey = (npass & 1) ? e->key_b.as<uint32_t>() : e->key_a.as<uint32_t>();
        order = (npass & 1) ? e->idx_b.as<uint32_t>() : e->idx_a.as<uint32_t>();
        uint32_t* vk = (npass & 1) ? e->key_a.as<uint32_t>() : e->key_b.as<uint32_t>();
        uint32_t* vs = (npass & 1) ? e->idx_a.as<uint32_t>() : e->idx_b.as<uint32_t>();
        // 4. run heads over the selected prefix
        const uint32_t nch = ceil_div(n_sel, kHeadChunk);
        ECK(e->chunk.ensure(sizeof(uint32_t) * nch));
        k_eval_heads_count<<<nch, kThreads, 0, e->st>>>(skey, n_sel, e->chunk.as<uint32_t>());
        k_eval_heads_scan<<<1, 1024, 0, e->st>>>(e->chunk.as<uint32_t>(), nch, d_st);
        k_eval_heads_scatter<<<nch, kThreads, 0, e->st>>>(skey, n_sel, e->chunk.as<uint32_t>(), d_st, vk, vs);
        ECK(cudaGetLastError());
        vox_key = vk;
        vox_start = vs;
    }
    // 5. query
    uint32_t* d_match = match;
    if (match && !dev && ng) { ECK(e->match.ensure(sizeof(uint32_t) * n_gt)); d_match = e->match.as<uint32_t>(); }
    if (ng) {
        k_eval_query<<<ceil_div(ng, kThreads), kThreads, 0, e->st>>>(d_gt, ng, d_est, order, vox_start, vox_key, g, d_match, d_st);
        ECK(cudaGetLastError());
    }
    if (match && !dev && ng) ECK(cudaMemcpyAsync(match, d_match, sizeof(uint32_t) * n_gt, cudaMemcpyDeviceToHost, e->st));
    ECK(cudaMemcpyAsync(h, d_st, sizeof(EvalStats), cudaMemcpyDeviceToHost, e->st));
    ECK(cudaStreamSynchronize(e->st));
    if (h->bad & 2u) return fail(e, ERASOR_E_INVALID, "non-finite x, y or z in a ground-truth point");
    out->gt_static = h->cnt[0];
    out->gt_dynamic = h->cnt[1];
    out->preserved_static = h->cnt[2];
    out->preserved_dynamic = h->cnt[3];
    out->inliers = h->cnt[4];
    out->ambiguous_ties = h->cnt[5];
    return ERASOR_OK;
}

}  // extern "C"
