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
#include "buffers.h"
#include "device_common.cuh"
#include "radix_sort.h"

namespace erasor {

constexpr int      kThreads   = 256;
constexpr int      kWarps     = kThreads / 32;
constexpr uint32_t kSeg       = kRadixSeg;     // points per warp segment of the radix sort
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

cudaError_t radix_sort_passes(cudaStream_t st, uint32_t* scratch, uint32_t* const k[2], uint32_t* const v[2], uint32_t n, int first, int npass) {
    const uint32_t nseg = (uint32_t)(((uint64_t)n + kSeg - 1) / kSeg);
    uint32_t* cnt = scratch;
    uint32_t* tot = cnt + 256ull * nseg;
    const int seg_ctas = (int)((nseg + kWarps - 1) / kWarps);
    for (int pass = 0; pass < npass; ++pass) {
        const int a = pass & 1;
        k_eval_radix_hist<<<seg_ctas, kThreads, 0, st>>>(k[a], n, nseg, 8 * (first + pass), cnt);
        k_eval_radix_rows<<<256 / kWarps, kThreads, 0, st>>>(cnt, nseg, tot);
        k_eval_radix_scatter<<<seg_ctas, kThreads, 0, st>>>(k[a], v[a], k[a ^ 1], v[a ^ 1], n, nseg, 8 * (first + pass), cnt, tot);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
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

// ============================================================================================================================
// The overlap report (erasor_eval_overlap, DESIGN.md section 11.1): the exact, unbounded 1-NN distance from every selected
// estimate point into the GT.  The GT is indexed twice (no keep mask): on the fine grid of eval_grid_setup with the kernels
// above, and on a coarse grid whose cells are aligned blocks of 2^cshift fine cells per axis, at most kOvlCoarseDiv per axis
// (k_ovl_ckeys, then the same sort and run heads); each coarse cell carries the tight bounding box of its points (k_ovl_boxes).
//   k_ovl_ckeys           coarse key per GT point: its fine cell, shifted right by cshift per axis
//   k_ovl_boxes           one warp per coarse cell: min / max of its points
//   k_ovl_query           per estimate point: fine shells of Chebyshev radius 0..kOvlShellMax with a provable stopping bound,
//                         else the far path over the coarse boxes; sklearn's double distance; the report's counters
//   k_ovl_split           distance bit patterns -> (low, high) words for the radix sort (non-negative doubles order like uint64)
//   k_ovl_gather          the sorted patterns at the caller's ranks
constexpr int kOvlShellMax  = 4;        // fine shells searched before a point takes the far path
constexpr int kOvlCoarseDiv = 32;       // coarse cells per axis at most (<= 32768 coarse cells)
constexpr int kOvlCnt       = 9;        // n, est_static, est_dynamic, below_half, below_one, below_two, far_points, max bits, bad
constexpr double kShrink = 1.0 - 1.0 / 1099511627776.0;    // 1 - 2^-40: covers the rounding of a squared gap / bound in double
constexpr double kGrow   = 1.0 + 1.0 / 1099511627776.0;

struct OvlGrid {
    EvalGrid g;                   // the fine GT grid (eval_grid_setup over the GT's bounds)
    double   leaf;                // (double)g.leaf
    double   marg;                // a GT point assigned to cell c lies within [c leaf - marg, (c + 1) leaf + marg] (ovl_setup)
    double   half, one, two;      // 0.5 * voxelsize, voxelsize, 2 * voxelsize, as the report computes them
    int      cshift;              // coarse cell = fine cells (i >> cshift, j >> cshift, k >> cshift)
    int      cdiv[3];             // coarse cells per axis, ((div - 1) >> cshift) + 1 <= kOvlCoarseDiv
};

namespace {

// sklearn's squared distance: (dx*dx + dy*dy) + dz*dz in double from the float coordinates, no contraction
__device__ __forceinline__ double ovl_d2(double qx, double qy, double qz, float4 p) {
    const double dx = __dsub_rn(qx, (double)p.x), dy = __dsub_rn(qy, (double)p.y), dz = __dsub_rn(qz, (double)p.z);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// lower bound on |x - p| along one axis for every GT point p assigned to an absolute cell in [c0, c1]
__device__ __forceinline__ double ovl_axis_gap(double x, int c0, int c1, const OvlGrid& o) {
    const double lo = (double)c0 * o.leaf - o.marg, hi = (double)(c1 + 1) * o.leaf + o.marg;
    return fmax(0.0, fmax(lo - x, x - hi));
}

// lower bound on the distance along axis a from x to every GT point in a cell more than s cells from x's cell c (relative index)
// along that axis: the two faces of the searched block, widened by marg; a side with no grid cell behind it gives +inf
__device__ __forceinline__ double ovl_face_bound(double x, int c, int s, int a, const OvlGrid& o) {
    double lb = __longlong_as_double(0x7FF0000000000000LL);
    if (c + s + 1 <= o.g.div[a] - 1) lb = (double)(c + s + 1 + o.g.min_b[a]) * o.leaf - o.marg - x;
    if (c - s - 1 >= 0) lb = fmin(lb, x - ((double)(c - s + o.g.min_b[a]) * o.leaf + o.marg));
    return lb;
}

// the t-th entry of c, c - 1, c + 1, c - 2, c + 2, ... (t < 2 (hi - lo) + 2), or -1 when it falls outside [lo, hi]
__device__ __forceinline__ int centre_out(int c, int t, int lo, int hi) {
    const int v = c + ((t & 1) ? -((t + 1) >> 1) : (t >> 1));
    return (v < lo || v > hi) ? -1 : v;
}

// min over the GT points of fine cells x0..x1 of row (jj, kk) of the squared distance to q, folded into best
__device__ __forceinline__ void ovl_scan_row(const EvalGrid& g, const uint32_t* __restrict__ vox_key, const uint32_t* __restrict__ vox_start,
                                             const uint32_t* __restrict__ order, const float4* __restrict__ gt, uint32_t nv, int x0, int x1,
                                             int jj, int kk, double qx, double qy, double qz, double& best) {
    const uint32_t k_lo = cell_key(g, x0, jj, kk), k_hi = k_lo + (uint32_t)(x1 - x0);
    uint32_t lo = 0, hi = nv;             // first cell with vox_key >= k_lo
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (vox_key[mid] < k_lo) lo = mid + 1; else hi = mid; }
    uint32_t v1 = lo;
    while (v1 < nv && vox_key[v1] <= k_hi) ++v1;
    if (v1 == lo) return;
    const uint32_t e = vox_start[v1];
    for (uint32_t k = vox_start[lo]; k < e; ++k) best = fmin(best, ovl_d2(qx, qy, qz, gt[order[k]]));
}

// relative fine cell of coordinate x clamped to [lo, hi], in double (x may be far outside the grid: no out-of-range conversion)
__device__ __forceinline__ int ovl_clamped_cell(double x, int a, int lo, int hi, const OvlGrid& o) {
    return (int)fmin(fmax(floor(x / o.leaf) - (double)o.g.min_b[a], (double)lo), (double)hi);
}

// The far path's visit of one coarse cell: its block of fine rows, nearest to q first along y and z.  A row is skipped when its
// y / z gap, squared, is beyond `bound` (the upper bound or the best so far); otherwise only its cells whose x gap can still be
// within sqrt(bound - gyz) are searched -- the window is widened by marg and one cell on either side, so it is conservative.
__device__ __noinline__ void ovl_visit_block(const OvlGrid& o, uint32_t ckey, const uint32_t* __restrict__ vox_key,
                                                const uint32_t* __restrict__ vox_start, const uint32_t* __restrict__ order,
                                                const float4* __restrict__ gt, uint32_t nv, double qx, double qy, double qz, double ub,
                                                double& best) {
    const EvalGrid& g = o.g;
    const int bi = (int)(ckey % (uint32_t)o.cdiv[0]), bj = (int)((ckey / (uint32_t)o.cdiv[0]) % (uint32_t)o.cdiv[1]);
    const int bk = (int)(ckey / ((uint32_t)o.cdiv[0] * (uint32_t)o.cdiv[1]));
    const int w = 1 << o.cshift;
    const int X0 = bi << o.cshift, X1 = min(X0 + w - 1, g.div[0] - 1);
    const int Y0 = bj << o.cshift, Y1 = min(Y0 + w - 1, g.div[1] - 1);
    const int Z0 = bk << o.cshift, Z1 = min(Z0 + w - 1, g.div[2] - 1);
    const int jc = ovl_clamped_cell(qy, 1, Y0, Y1, o), kc = ovl_clamped_cell(qz, 2, Z0, Z1, o);
    for (int tk = 0; tk < 2 * (Z1 - Z0) + 2; ++tk) {
        const int kk = centre_out(kc, tk, Z0, Z1);
        if (kk < 0) continue;
        const double gz = ovl_axis_gap(qz, kk + g.min_b[2], kk + g.min_b[2], o);
        if (gz * gz * kShrink > fmin(ub, best)) continue;
        for (int tj = 0; tj < 2 * (Y1 - Y0) + 2; ++tj) {
            const int jj = centre_out(jc, tj, Y0, Y1);
            if (jj < 0) continue;
            const double gy = ovl_axis_gap(qy, jj + g.min_b[1], jj + g.min_b[1], o);
            const double gyz = gy * gy + gz * gz, bound = fmin(ub, best);
            if (gyz * kShrink > bound) continue;
            const double r = sqrt(fmax(bound * kGrow - gyz, 0.0)) * kGrow;
            const double xl = fmax(floor((qx - r - o.marg) / o.leaf) - (double)g.min_b[0] - 1.0, (double)X0);
            const double xh = fmin(floor((qx + r + o.marg) / o.leaf) - (double)g.min_b[0] + 1.0, (double)X1);
            if (!(xl <= xh)) continue;
            const int x0 = (int)xl, x1 = (int)xh;
            const double gx = ovl_axis_gap(qx, x0 + g.min_b[0], x1 + g.min_b[0], o);
            if ((gx * gx + gyz) * kShrink > bound) continue;
            ovl_scan_row(g, vox_key, vox_start, order, gt, nv, x0, x1, jj, kk, qx, qy, qz, best);
        }
    }
}

// lower bound on |x - p| for a point p in a box [lo, hi] (float bounds, exact in double)
__device__ __forceinline__ double box_gap(double x, float lo, float hi) { return fmax(0.0, fmax((double)lo - x, x - (double)hi)); }
__device__ __forceinline__ double box_far(double x, float lo, float hi) { return fmax(fabs(x - (double)lo), fabs(x - (double)hi)); }

}  // namespace

__global__ void __launch_bounds__(kThreads) k_ovl_ckeys(const float4* __restrict__ pts, uint32_t n, EvalGrid g, int cshift, int cdiv0, int cdiv1,
                                                        uint32_t* __restrict__ key, uint32_t* __restrict__ idx) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float4 p = pts[i];          // inside the GT's bounds: every fine cell lies in [0, div)
        const uint32_t ci = (uint32_t)voxel_cell(p.x, g.inv, g.min_b[0]) >> cshift, cj = (uint32_t)voxel_cell(p.y, g.inv, g.min_b[1]) >> cshift;
        const uint32_t ck = (uint32_t)voxel_cell(p.z, g.inv, g.min_b[2]) >> cshift;
        key[i] = ci + cj * (uint32_t)cdiv0 + ck * ((uint32_t)cdiv0 * (uint32_t)cdiv1);
        idx[i] = (uint32_t)i;
    }
}

__global__ void __launch_bounds__(kThreads) k_ovl_boxes(const float4* __restrict__ gt, const uint32_t* __restrict__ c_order,
                                                        const uint32_t* __restrict__ c_start, const EvalStats* __restrict__ cst,
                                                        float* __restrict__ box /*[nvc][6]: lo xyz, hi xyz*/) {
    const int lane = threadIdx.x & 31;
    const uint32_t v = blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (v >= cst->nv) return;
    uint32_t mn[3] = {~0u, ~0u, ~0u}, mx[3] = {0u, 0u, 0u};
    const uint32_t b = c_start[v], e = c_start[v + 1];
    for (uint32_t k = b + lane; k < e; k += 32u) {
        const float4 p = gt[c_order[k]];
        const uint32_t u[3] = {float_to_ordered(p.x + 0.0f), float_to_ordered(p.y + 0.0f), float_to_ordered(p.z + 0.0f)};
#pragma unroll
        for (int a = 0; a < 3; ++a) { mn[a] = min(mn[a], u[a]); mx[a] = max(mx[a], u[a]); }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) { mn[a] = __reduce_min_sync(FULL_MASK, mn[a]); mx[a] = __reduce_max_sync(FULL_MASK, mx[a]); }
    if (lane == 0)
        for (int a = 0; a < 3; ++a) { box[6 * (size_t)v + a] = ordered_to_float(mn[a]); box[6 * (size_t)v + 3 + a] = ordered_to_float(mx[a]); }
}

// One thread per estimate point.  Fine stage: the shells of Chebyshev radius s = 0, 1, .. around the point's cell; a shell row
// (j, k) is one x-contiguous key range on the shell's y / z faces and its two end cells inside them, each found with one lower
// bound and skipped when its conservative gap is strictly beyond the best distance so far.  After shell s every GT point not yet
// seen lies in a cell at least s + 1 cells away along some axis, hence beyond one of the block's six faces widened by marg (faces
// with no grid cell behind them drop out); when the best distance is at most that bound (shrunk by 2^-40 for the rounding of the
// bound and of the distances), nothing unseen can be nearer and the search stops.  A point outside the grid's guard window (no
// float -> int conversion happens for it), or not settled after kOvlShellMax shells, takes the far path: an upper bound from the
// farthest corners of the coarse boxes, then the coarse cell with the nearest box, then every other coarse cell whose box gap is
// within the upper bound and the best so far -- each through its fine rows, pruned by their gaps (ovl_visit_block).
// Only distances leave the kernel, so which of several equally near points is seen first does not matter.
__global__ void __launch_bounds__(kThreads) k_ovl_query(const float4* __restrict__ est, const uint8_t* __restrict__ keep, uint32_t n_est,
                                                        const float4* __restrict__ gt, const uint32_t* __restrict__ order,
                                                        const uint32_t* __restrict__ vox_start, const uint32_t* __restrict__ vox_key,
                                                        const EvalStats* __restrict__ st, const uint32_t* __restrict__ c_key,
                                                        const float* __restrict__ c_box,
                                                        const EvalStats* __restrict__ cst, OvlGrid o, double* __restrict__ dist,
                                                        unsigned long long* __restrict__ cnt /*[kOvlCnt]*/) {
    __shared__ uint32_t s_c[kWarps][9];
    const EvalGrid& g = o.g;
    const uint32_t nv = st->nv;
    uint32_t c[7] = {0u, 0u, 0u, 0u, 0u, 0u, 0u};       // n, est_static, est_dynamic, below_half, below_one, below_two, far
    uint32_t bad = 0u;
    unsigned long long dbits = 0ull;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_est) {
        double d = __longlong_as_double(0x7FF8000000000000LL);         // NaN: deselected or invalid
        if (!keep || keep[i]) {
            const float4 q = est[i];
            if (!finite3(q)) {
                bad = 1u;
            } else {
                const bool dyn = is_dynamic(q.w);
                c[0] = 1u; c[1] = dyn ? 0u : 1u; c[2] = dyn ? 1u : 0u;
                const double INF = __longlong_as_double(0x7FF0000000000000LL);
                const double qx = q.x, qy = q.y, qz = q.z;
                double best = INF;
                bool far = nv != 0u;
                const float ax = FM(q.x, g.inv), ay = FM(q.y, g.inv), az = FM(q.z, g.inv);
                if (nv && ax >= g.lo[0] && ax < g.hi[0] && ay >= g.lo[1] && ay < g.hi[1] && az >= g.lo[2] && az < g.hi[2]) {
                    const int ci = voxel_cell(q.x, g.inv, g.min_b[0]), cj = voxel_cell(q.y, g.inv, g.min_b[1]), ck = voxel_cell(q.z, g.inv, g.min_b[2]);
                    for (int s = 0; s <= kOvlShellMax; ++s) {
                        for (int b = -s; b <= s; ++b) {
                            const int jj = cj + b;
                            if (jj < 0 || jj >= g.div[1]) continue;
                            const double gy = ovl_axis_gap(qy, jj + g.min_b[1], jj + g.min_b[1], o);
                            for (int cc = -s; cc <= s; ++cc) {
                                const int kk = ck + cc;
                                if (kk < 0 || kk >= g.div[2]) continue;
                                const double gz = ovl_axis_gap(qz, kk + g.min_b[2], kk + g.min_b[2], o);
                                const double gyz = gy * gy + gz * gz;
                                if (gyz * kShrink > best) continue;
                                const bool face = b == -s || b == s || cc == -s || cc == s;
                                for (int t = 0; t < (face ? 1 : 2); ++t) {
                                    int x0 = (face || t == 0) ? ci - s : ci + s, x1 = face ? ci + s : x0;
                                    x0 = max(x0, 0);
                                    x1 = min(x1, g.div[0] - 1);
                                    if (x0 > x1) continue;
                                    const double gx = ovl_axis_gap(qx, x0 + g.min_b[0], x1 + g.min_b[0], o);
                                    if ((gx * gx + gyz) * kShrink > best) continue;
                                    ovl_scan_row(g, vox_key, vox_start, order, gt, nv, x0, x1, jj, kk, qx, qy, qz, best);
                                }
                            }
                        }
                        // the stopping bound: the nearest face of the searched block behind which the grid has cells
                        const double lb = fmin(ovl_face_bound(qx, ci, s, 0, o), fmin(ovl_face_bound(qy, cj, s, 1, o), ovl_face_bound(qz, ck, s, 2, o)));
                        if (lb == INF || (best < INF && __dsqrt_rn(best) <= lb * kShrink)) { far = false; break; }
                    }
                }
                if (far) {
                    const uint32_t nvc = cst->nv;
                    double ub = best, gmin = INF;
                    uint32_t vmin = 0u;
                    for (uint32_t v = 0; v < nvc; ++v) {   // every coarse box holds a point no farther than its farthest corner
                        const float* bx = c_box + 6 * (size_t)v;
                        const double fx = box_far(qx, bx[0], bx[3]), fy = box_far(qy, bx[1], bx[4]), fz = box_far(qz, bx[2], bx[5]);
                        ub = fmin(ub, (fx * fx + fy * fy + fz * fz) * kGrow);
                        const double gx = box_gap(qx, bx[0], bx[3]), gy = box_gap(qy, bx[1], bx[4]), gz = box_gap(qz, bx[2], bx[5]);
                        const double g2 = gx * gx + gy * gy + gz * gz;
                        if (g2 < gmin) { gmin = g2; vmin = v; }
                    }
                    ovl_visit_block(o, c_key[vmin], vox_key, vox_start, order, gt, nv, qx, qy, qz, ub, best);
                    for (uint32_t v = 0; v < nvc; ++v) {
                        if (v == vmin) continue;
                        const float* bx = c_box + 6 * (size_t)v;
                        const double gx = box_gap(qx, bx[0], bx[3]), gy = box_gap(qy, bx[1], bx[4]), gz = box_gap(qz, bx[2], bx[5]);
                        if ((gx * gx + gy * gy + gz * gz) * kShrink > fmin(ub, best)) continue;
                        ovl_visit_block(o, c_key[v], vox_key, vox_start, order, gt, nv, qx, qy, qz, ub, best);
                    }
                    c[6] = 1u;
                }
                d = __dsqrt_rn(best);                                         // +inf for an empty GT
                c[3] = d < o.half ? 1u : 0u;
                c[4] = d < o.one ? 1u : 0u;
                c[5] = d < o.two ? 1u : 0u;
                dbits = (unsigned long long)__double_as_longlong(d);
            }
        }
        if (dist) dist[i] = d;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 7; ++k) c[k] = __reduce_add_sync(FULL_MASK, c[k]);
    bad = __reduce_or_sync(FULL_MASK, bad);
    const uint32_t mhi = __reduce_max_sync(FULL_MASK, (uint32_t)(dbits >> 32));
    const uint32_t mlo = __reduce_max_sync(FULL_MASK, (uint32_t)(dbits >> 32) == mhi ? (uint32_t)dbits : 0u);
    if (lane == 0) {
        for (int k = 0; k < 7; ++k) s_c[warp][k] = c[k];
        s_c[warp][7] = mhi; s_c[warp][8] = mlo;
        if (bad) atomicOr(&cnt[8], 1ull);
    }
    __syncthreads();
    if (threadIdx.x < 7) {
        uint32_t t = 0u;
        for (int w = 0; w < kWarps; ++w) t += s_c[w][threadIdx.x];
        if (t) atomicAdd(&cnt[threadIdx.x], (unsigned long long)t);
    } else if (threadIdx.x == 7) {
        unsigned long long m = 0ull;
        for (int w = 0; w < kWarps; ++w) m = max(m, ((unsigned long long)s_c[w][7] << 32) | s_c[w][8]);
        if (m) atomicMax(&cnt[7], m);
    }
}

// how many of n keep bytes are nonzero
__global__ void __launch_bounds__(kThreads) k_ovl_count(const uint8_t* __restrict__ keep, size_t n, unsigned long long* __restrict__ out) {
    uint32_t c = 0u;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) c += keep[i] ? 1u : 0u;
    c = __reduce_add_sync(FULL_MASK, c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, (unsigned long long)c);
}

__global__ void __launch_bounds__(kThreads) k_ovl_split(const double* __restrict__ dist, uint32_t n, uint32_t* __restrict__ lo,
                                                        uint32_t* __restrict__ hi) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const double d = dist[i];
        const unsigned long long b = (d == d) ? (unsigned long long)__double_as_longlong(d) : ~0ull;   // deselected sort last
        lo[i] = (uint32_t)b;
        hi[i] = (uint32_t)(b >> 32);
    }
}

__global__ void k_ovl_gather(const uint32_t* __restrict__ hi, const uint32_t* __restrict__ lo, const unsigned long long* __restrict__ ranks,
                             uint32_t nr, double* __restrict__ out) {
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < nr; r += gridDim.x * blockDim.x) {
        const size_t k = (size_t)ranks[r];
        out[r] = __longlong_as_double((long long)(((unsigned long long)hi[k] << 32) | lo[k]));
    }
}

}  // namespace erasor

// ============================================================================================================================
// C ABI
// ============================================================================================================================
using namespace erasor;

namespace {
thread_local std::string g_eval_err;
}  // namespace

struct erasor_eval_ctx {
    int device = 0;
    cudaStream_t st = nullptr;
    std::string err;
    DeviceBuffer gt, est, keep, match;        // staging of host inputs / the match output
    DeviceBuffer key_a, key_b, idx_a, idx_b;  // 16 B per estimate point: the sort's ping-pong; the free half holds vox_key / vox_start
    DeviceBuffer cnt, chunk, stats;           // per-segment digit counts + digit totals, per-chunk head counts, EvalStats
    PinnedBuffer h_stats;                     // EvalStats
    // erasor_eval_overlap: the coarse index's ping-pong, its boxes and EvalStats, the distances, counters + ranks + rank values
    DeviceBuffer ckey_a, ckey_b, cidx_a, cidx_b, cbox, cstats, dist, ovl;
    int sm_count = 132;
};

namespace {
#define ECK(call) ERASOR_CUDA_TRY(e->err, call, #call)

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

// npass 8-bit passes of the stable LSD radix sort (radix_sort.h) in the context's scratch
int radix_passes(erasor_eval_t e, uint32_t* const k[2], uint32_t* const v[2], uint32_t n, int first, int npass) {
    ECK(e->cnt.ensure(sizeof(uint32_t) * radix_scratch_words(n)));
    ECK(radix_sort_passes(e->st, e->cnt.as<uint32_t>(), k, v, n, first, npass));
    return ERASOR_OK;
}

// the sorted cell table of one cloud: point order[vox_start[v] .. vox_start[v + 1]) in cell vox_key[v], ascending over v < nv
struct CellIndex { const uint32_t *order = nullptr, *vox_key = nullptr, *vox_start = nullptr; };

// keys + radix sort (only the passes the key width needs: a dropped point's 0xFFFFFFFF keeps its all-ones low bits, which exceed
// every cell key of that width, so it sorts behind the selected points), then the run heads over the selected prefix; nv goes to
// st->nv.  kb / ib: the key and index ping-pong, 4 (n + 1) bytes each; the half the sort does not end in holds vox_key / vox_start.
// With o (the overlap search's grids), the points are keyed by their coarse cell instead (k_ovl_ckeys; g is then o.g, no keep mask).
int build_cells(erasor_eval_t e, const float4* pts, const uint8_t* keep, uint32_t n, uint32_t n_sel, const EvalGrid& g, DeviceBuffer* const kb[2],
                DeviceBuffer* const ib[2], EvalStats* st, CellIndex& ix, const OvlGrid* o = nullptr) {
    unsigned long long cells = 1ull;
    for (int k = 0; k < 3; ++k) cells *= (unsigned long long)(o ? o->cdiv[k] : g.div[k]);
    const size_t words = (size_t)n + 1;
    for (int a = 0; a < 2; ++a) { ECK(kb[a]->ensure(4 * words)); ECK(ib[a]->ensure(4 * words)); }
    uint32_t* const K[2] = {kb[0]->as<uint32_t>(), kb[1]->as<uint32_t>()};
    uint32_t* const V[2] = {ib[0]->as<uint32_t>(), ib[1]->as<uint32_t>()};
    const int g_stream = e->sm_count * 8;
    if (o) k_ovl_ckeys<<<std::min(grid_for((int)std::min<uint32_t>(n, 1u << 30), kThreads), g_stream), kThreads, 0, e->st>>>(pts, n, g, o->cshift, o->cdiv[0],
                                                                                                                            o->cdiv[1], K[0], V[0]);
    else k_eval_keys<<<std::min(grid_for((int)std::min<uint32_t>(n, 1u << 30), kThreads), g_stream), kThreads, 0, e->st>>>(pts, keep, n, g, K[0], V[0]);
    ECK(cudaGetLastError());
    int bits = 1;
    while (bits < 32 && (1ull << bits) <= cells) ++bits;          // cells < 2^bits: the largest cell key is below 2^bits - 1
    const int npass = (bits + 7) / 8;
    const int rc = radix_passes(e, K, V, n, 0, npass);
    if (rc != ERASOR_OK) return rc;
    const uint32_t* skey = K[npass & 1];
    uint32_t* vk = K[(npass & 1) ^ 1];
    uint32_t* vs = V[(npass & 1) ^ 1];
    const uint32_t nch = ceil_div(n_sel, kHeadChunk);
    ECK(e->chunk.ensure(sizeof(uint32_t) * nch));
    k_eval_heads_count<<<nch, kThreads, 0, e->st>>>(skey, n_sel, e->chunk.as<uint32_t>());
    k_eval_heads_scan<<<1, 1024, 0, e->st>>>(e->chunk.as<uint32_t>(), nch, st);
    k_eval_heads_scatter<<<nch, kThreads, 0, e->st>>>(skey, n_sel, e->chunk.as<uint32_t>(), st, vk, vs);
    ECK(cudaGetLastError());
    ix.order = V[npass & 1];
    ix.vox_key = vk;
    ix.vox_start = vs;
    return ERASOR_OK;
}

// The overlap search's grids over the GT's bounds.  Fine: eval_grid_setup's cell edge (so keys fit, every converted coordinate
// stays below 2^22 cells, and R 2^-21 < leaf).  marg: a GT point p assigned to cell c along an axis has
// floor(fl(p * fl(1 / leaf))) = c, and fl(p * fl(1 / leaf)) is within |p| / leaf * 2^-22.99 of p / leaf, so p lies within
// |p| 2^-22.99 of [c leaf, (c + 1) leaf]; |p| <= R = (max |cell| + 3) leaf, and marg = R 2^-21 is four times that, which also
// covers the rounding of the face coordinates and gaps computed from it in double.  Coarse: blocks of 2^cshift fine cells per axis,
// cshift the smallest with at most kOvlCoarseDiv blocks per axis (the coarse boxes need no margin: they are the points' own bounds).
bool ovl_setup(const float mn[3], const float mx[3], double voxelsize, OvlGrid& o) {
    if (!eval_grid_setup(mn, mx, voxelsize, o.g)) return false;
    double cmax = 0.0;
    for (int k = 0; k < 3; ++k) cmax = std::max(cmax, std::max(std::fabs((double)o.g.min_b[k]), std::fabs((double)(o.g.min_b[k] + o.g.div[k] - 1)) + 1.0));
    o.leaf = (double)o.g.leaf;
    o.marg = (cmax + 3.0) * o.leaf * (1.0 / 2097152.0);
    o.half = 0.5 * voxelsize;
    o.one = voxelsize;
    o.two = 2 * voxelsize;
    o.cshift = 0;
    while (((o.g.div[0] - 1) >> o.cshift) + 1 > kOvlCoarseDiv || ((o.g.div[1] - 1) >> o.cshift) + 1 > kOvlCoarseDiv ||
           ((o.g.div[2] - 1) >> o.cshift) + 1 > kOvlCoarseDiv)
        ++o.cshift;
    for (int k = 0; k < 3; ++k) o.cdiv[k] = ((o.g.div[k] - 1) >> o.cshift) + 1;
    return true;
}
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
    if (c == cudaSuccess) c = e->h_stats.allocate(sizeof(EvalStats));
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
        if (ng) { ECK(e->gt.ensure(sizeof(float4) * n_gt)); ECK(cudaMemcpyAsync(e->gt.p(), gt_xyzi, sizeof(float4) * n_gt, cudaMemcpyHostToDevice, e->st)); d_gt = e->gt.as<float4>(); }
        if (ne) { ECK(e->est.ensure(sizeof(float4) * n_est)); ECK(cudaMemcpyAsync(e->est.p(), est_xyzi, sizeof(float4) * n_est, cudaMemcpyHostToDevice, e->st)); d_est = e->est.as<float4>(); }
        if (ne && est_keep) { ECK(e->keep.ensure(n_est)); ECK(cudaMemcpyAsync(e->keep.p(), est_keep, n_est, cudaMemcpyHostToDevice, e->st)); d_keep = e->keep.as<uint8_t>(); }
    }
    if (!ne) d_keep = nullptr;
    EvalStats* d_st = e->stats.as<EvalStats>();
    EvalStats* h = e->h_stats.as<EvalStats>();
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
    CellIndex ix;
    if (n_sel) {
        // 2. grid
        float mn[3], mx[3];
        for (int k = 0; k < 3; ++k) { mn[k] = ordered_to_float(h->mn[k]); mx[k] = ordered_to_float(h->mx[k]); }
        if (!eval_grid_setup(mn, mx, voxelsize, g)) return fail(e, ERASOR_E_INVALID, "no cell grid covers the estimate's extent");
        // 3. keys + radix sort, 4. run heads
        DeviceBuffer* kb[2] = {&e->key_a, &e->key_b};
        DeviceBuffer* ib[2] = {&e->idx_a, &e->idx_b};
        const int rc = build_cells(e, d_est, d_keep, ne, n_sel, g, kb, ib, d_st, ix);
        if (rc != ERASOR_OK) return rc;
    }
    const uint32_t *order = ix.order, *vox_start = ix.vox_start, *vox_key = ix.vox_key;
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

int erasor_eval_count_selected(erasor_eval_t e, const uint8_t* keep, size_t n, int ptr_kind, uint64_t* count) {
    if (!e) return ERASOR_E_INVALID;
    e->err.clear();
    if (!count || (n && !keep)) return fail(e, ERASOR_E_INVALID, "null argument");
    if (ptr_kind != ERASOR_PTR_HOST && ptr_kind != ERASOR_PTR_DEVICE) return fail(e, ERASOR_E_INVALID, "ptr_kind must be ERASOR_PTR_HOST or ERASOR_PTR_DEVICE");
    if (ptr_kind == ERASOR_PTR_HOST) {
        uint64_t c = 0;
        for (size_t i = 0; i < n; ++i) c += keep[i] ? 1u : 0u;
        *count = c;
        return ERASOR_OK;
    }
    ECK(cudaSetDevice(e->device));
    ECK(e->ovl.ensure(8 * kOvlCnt));
    unsigned long long* d = e->ovl.as<unsigned long long>();
    ECK(cudaMemsetAsync(d, 0, 8, e->st));
    if (n) k_ovl_count<<<std::min(grid_for((int)std::min<size_t>(n, 1u << 30), kThreads), e->sm_count * 8), kThreads, 0, e->st>>>(keep, n, d);
    ECK(cudaGetLastError());
    unsigned long long h = 0;
    ECK(cudaMemcpyAsync(&h, d, 8, cudaMemcpyDeviceToHost, e->st));
    ECK(cudaStreamSynchronize(e->st));
    *count = h;
    return ERASOR_OK;
}

int erasor_eval_overlap(erasor_eval_t e, const float* gt_xyzi, size_t n_gt, const float* est_xyzi, size_t n_est, const uint8_t* est_keep,
                        double voxelsize, int ptr_kind, const uint64_t* ranks, size_t n_ranks, double* rank_values, double* est_dist,
                        erasor_eval_overlap_t* out) {
    if (!e) return ERASOR_E_INVALID;
    e->err.clear();
    if (!out) return fail(e, ERASOR_E_INVALID, "null overlap pointer");
    if ((n_gt && !gt_xyzi) || (n_est && !est_xyzi)) return fail(e, ERASOR_E_INVALID, "null cloud pointer");
    if (n_ranks && (!ranks || !rank_values)) return fail(e, ERASOR_E_INVALID, "null rank array");
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
        if (reinterpret_cast<uintptr_t>(est_dist) & 7u) return fail(e, ERASOR_E_INVALID, "est_dist must be 8-byte aligned");
    } else {
        if (ng) { ECK(e->gt.ensure(sizeof(float4) * n_gt)); ECK(cudaMemcpyAsync(e->gt.p(), gt_xyzi, sizeof(float4) * n_gt, cudaMemcpyHostToDevice, e->st)); d_gt = e->gt.as<float4>(); }
        if (ne) { ECK(e->est.ensure(sizeof(float4) * n_est)); ECK(cudaMemcpyAsync(e->est.p(), est_xyzi, sizeof(float4) * n_est, cudaMemcpyHostToDevice, e->st)); d_est = e->est.as<float4>(); }
        if (ne && est_keep) { ECK(e->keep.ensure(n_est)); ECK(cudaMemcpyAsync(e->keep.p(), est_keep, n_est, cudaMemcpyHostToDevice, e->st)); d_keep = e->keep.as<uint8_t>(); }
    }
    if (!ne) d_keep = nullptr;
    EvalStats* d_st = e->stats.as<EvalStats>();
    EvalStats* h = e->h_stats.as<EvalStats>();
    std::memset(h, 0, sizeof(EvalStats));
    for (int k = 0; k < 3; ++k) h->mn[k] = ~0u;
    ECK(cudaMemcpyAsync(d_st, h, sizeof(EvalStats), cudaMemcpyHostToDevice, e->st));
    ECK(e->cstats.ensure(sizeof(EvalStats)));
    EvalStats* d_cst = e->cstats.as<EvalStats>();
    ECK(cudaMemsetAsync(d_cst, 0, sizeof(EvalStats), e->st));
    // counters, then the ranks and their values
    ECK(e->ovl.ensure(8 * (kOvlCnt + 2 * n_ranks)));
    unsigned long long* d_cnt = e->ovl.as<unsigned long long>();
    unsigned long long* d_ranks = d_cnt + kOvlCnt;
    double* d_vals = reinterpret_cast<double*>(d_ranks + n_ranks);
    ECK(cudaMemsetAsync(d_cnt, 0, 8 * kOvlCnt, e->st));

    // 1. the GT's bounds (no keep mask: bit 0 of bad flags a non-finite GT point here)
    const int g_stream = e->sm_count * 8;
    if (ng) k_eval_bounds<<<std::min(grid_for((int)std::min<uint32_t>(ng, 1u << 30), kThreads), g_stream), kThreads, 0, e->st>>>(d_gt, nullptr, ng, d_st);
    ECK(cudaGetLastError());
    ECK(cudaMemcpyAsync(h, d_st, sizeof(EvalStats), cudaMemcpyDeviceToHost, e->st));
    ECK(cudaStreamSynchronize(e->st));
    if (h->bad & 1u) return fail(e, ERASOR_E_INVALID, "non-finite x, y or z in a ground-truth point");

    // 2. the fine and the coarse index of the GT, and the coarse boxes
    OvlGrid o{};
    o.half = 0.5 * voxelsize;
    o.one = voxelsize;
    o.two = 2 * voxelsize;
    CellIndex fx, cx;
    const size_t words = (size_t)std::max(ng, ne) + 1;           // the distance sort reuses the fine index's buffers
    ECK(e->key_a.ensure(4 * words)); ECK(e->key_b.ensure(4 * words));
    ECK(e->idx_a.ensure(4 * words)); ECK(e->idx_b.ensure(4 * words));
    if (ng) {
        float mn[3], mx[3];
        for (int k = 0; k < 3; ++k) { mn[k] = ordered_to_float(h->mn[k]); mx[k] = ordered_to_float(h->mx[k]); }
        if (!ovl_setup(mn, mx, voxelsize, o)) return fail(e, ERASOR_E_INVALID, "no cell grid covers the ground truth's extent");
        DeviceBuffer* kb[2] = {&e->key_a, &e->key_b};
        DeviceBuffer* ib[2] = {&e->idx_a, &e->idx_b};
        int rc = build_cells(e, d_gt, nullptr, ng, ng, o.g, kb, ib, d_st, fx);
        if (rc != ERASOR_OK) return rc;
        DeviceBuffer* ckb[2] = {&e->ckey_a, &e->ckey_b};
        DeviceBuffer* cib[2] = {&e->cidx_a, &e->cidx_b};
        rc = build_cells(e, d_gt, nullptr, ng, ng, o.g, ckb, cib, d_cst, cx, &o);
        if (rc != ERASOR_OK) return rc;
        const uint32_t max_cells = (uint32_t)o.cdiv[0] * (uint32_t)o.cdiv[1] * (uint32_t)o.cdiv[2];
        ECK(e->cbox.ensure(sizeof(float) * 6 * max_cells));
        k_ovl_boxes<<<ceil_div(max_cells, kWarps), kThreads, 0, e->st>>>(d_gt, cx.order, cx.vox_start, d_cst, e->cbox.as<float>());
        ECK(cudaGetLastError());
    }
    // 3. the query
    double* d_dist = (dev && est_dist) ? est_dist : nullptr;
    if (!d_dist && ne && (est_dist || n_ranks)) { ECK(e->dist.ensure(sizeof(double) * n_est)); d_dist = e->dist.as<double>(); }
    if (ne) {
        k_ovl_query<<<ceil_div(ne, kThreads), kThreads, 0, e->st>>>(d_est, d_keep, ne, d_gt, fx.order, fx.vox_start, fx.vox_key, d_st, cx.vox_key,
                                                                    e->cbox.as<float>(), d_cst, o, d_dist, d_cnt);
        ECK(cudaGetLastError());
    }
    unsigned long long hc[kOvlCnt];
    ECK(cudaMemcpyAsync(hc, d_cnt, 8 * kOvlCnt, cudaMemcpyDeviceToHost, e->st));
    ECK(cudaStreamSynchronize(e->st));
    if (hc[8]) return fail(e, ERASOR_E_INVALID, "non-finite x, y or z in a selected estimate point");
    const uint64_t n_sel = hc[0];
    for (size_t r = 0; r < n_ranks; ++r)
        if (ranks[r] >= n_sel) return fail(e, ERASOR_E_INVALID, "a rank is not below the number of selected estimate points");
    // 4. order statistics: the stable LSD radix sort of the 64-bit patterns (low word first, carrying the high word, then the
    //    high word carrying the low one); deselected points' all-ones patterns sort last
    if (n_ranks) {
        uint32_t* lo0 = e->key_a.as<uint32_t>();
        uint32_t* hi0 = e->idx_a.as<uint32_t>();
        k_ovl_split<<<std::min(grid_for((int)std::min<uint32_t>(ne, 1u << 30), kThreads), g_stream), kThreads, 0, e->st>>>(d_dist, ne, lo0, hi0);
        ECK(cudaGetLastError());
        uint32_t* const K1[2] = {lo0, e->key_b.as<uint32_t>()};
        uint32_t* const V1[2] = {hi0, e->idx_b.as<uint32_t>()};
        int rc = radix_passes(e, K1, V1, ne, 0, 4);                   // -> (lo0, hi0) sorted by the low word
        if (rc != ERASOR_OK) return rc;
        uint32_t* const K2[2] = {hi0, e->idx_b.as<uint32_t>()};
        uint32_t* const V2[2] = {lo0, e->key_b.as<uint32_t>()};
        rc = radix_passes(e, K2, V2, ne, 0, 4);                       // -> (hi0, lo0) sorted by the whole pattern
        if (rc != ERASOR_OK) return rc;
        ECK(cudaMemcpyAsync(d_ranks, ranks, 8 * n_ranks, cudaMemcpyHostToDevice, e->st));
        k_ovl_gather<<<ceil_div(n_ranks, kThreads), kThreads, 0, e->st>>>(hi0, lo0, d_ranks, (uint32_t)n_ranks, d_vals);
        ECK(cudaGetLastError());
        ECK(cudaMemcpyAsync(rank_values, d_vals, 8 * n_ranks, cudaMemcpyDeviceToHost, e->st));
    }
    if (est_dist && !dev && ne) ECK(cudaMemcpyAsync(est_dist, d_dist, sizeof(double) * n_est, cudaMemcpyDeviceToHost, e->st));
    ECK(cudaStreamSynchronize(e->st));
    out->n = n_sel;
    out->est_static = hc[1];
    out->est_dynamic = hc[2];
    out->below_half = hc[3];
    out->below_one = hc[4];
    out->below_two = hc[5];
    out->far_points = hc[6];
    uint64_t mb = hc[7];
    std::memcpy(&out->max, &mb, 8);
    if (!n_sel) out->max = std::nan("");
    return ERASOR_OK;
}

}  // extern "C"
