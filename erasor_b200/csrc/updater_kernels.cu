// updater_kernels.cu -- device versions of the caller-side steps either side of the R-POD -> SRT -> R-GPF path
// (SURVEY.md section 8f, rows 1-3), so that the map never leaves HBM between frames:
//
//   U1  stable partition of the map by a per-point predicate, with the float affine of pcl::transformPointCloud
//       fused into the copy of the selected side:
//         * OfflineMapUpdater::fetch_VoI  ("naive" mode)          reference OfflineMapUpdater.cpp:381-438
//         * OfflineMapUpdater::set_submap (large-scale window)    reference OfflineMapUpdater.cpp:360-379
//   U2  affine copy (body2origin, lidar2body: pcl::transformPointCloud)             :240, :286-288, :441-449
//   U3  erasor_utils::voxelize_preserving_labels for clouds of any size             erasor_utils.cpp:80-114
//       (pcl::VoxelGrid keys -> stable global radix sort -> centroids -> exact 1-NN label restore);
//       used on the query scan (:238) and by save_static_map (:186)
//
// Arithmetic is spelled with round-to-nearest intrinsics (no FMA contraction), exactly as restated in oracle/.
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>
#include <cstdint>

#include "device_common.cuh"
#include "updater_kernels.h"

namespace erasor {

__device__ __forceinline__ bool part_pred(const PartPred& P, float4 p) {
    if (P.kind == PART_RADIUS) {
        // double dist_square = pow(pt.x - x_criterion, 2) + pow(pt.y - y_criterion, 2); dist_square < max_dist_square
        const double dx = __dsub_rn((double)p.x, P.x), dy = __dsub_rn((double)p.y, P.y);
        const double d2 = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
        return d2 < P.limit;
    }
    if (P.kind == PART_NOT_NEAR) {
        // mapgen's vehicle-body cut (src/mapgen/mapgen.hpp:218-229): dist_square = pow(pt.x, 2) + pow(pt.y, 2) in double;
        // points with dist_square < max_dist_square are dropped, everything else (NaN included) is kept
        const double xd = (double)p.x, yd = (double)p.y;
        const double d2 = __dadd_rn(__dmul_rn(xd, xd), __dmul_rn(yd, yd));
        return !(d2 < P.limit);
    }
    // set_submap: fabs(x - pt.x) < submap_size && fabs(y - pt.y) < submap_size
    const double dx = fabs(__dsub_rn(P.x, (double)p.x)), dy = fabs(__dsub_rn(P.y, (double)p.y));
    return (dx < P.limit) && (dy < P.limit);
}

constexpr int PART_CHUNK = 4096;          // points per partition / head-count chunk (one virtual block)

__global__ void k_affine_copy(Mat4 T, int do_transform, const float4* in, float4* out, uint32_t n) {   // in may alias out
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = do_transform ? pcl_affine(T.m, in[i]) : in[i];
}
__global__ void __launch_bounds__(256) k_copy_segments(Mat4 T, CopySeg s0, CopySeg s1, CopySeg s2, CopySeg s3) {
    const CopySeg segs[4] = {s0, s1, s2, s3};
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint32_t blocks = (segs[k].n + 255u) / 256u * 256u;     // segments start on block boundaries: no divergence inside a warp
        if (i < blocks) {
            if (i < segs[k].n) { const float4 p = segs[k].src[i]; segs[k].dst[i] = segs[k].xform ? pcl_affine(T.m, p) : p; }
            return;
        }
        i -= blocks;
    }
}
cudaError_t launch_copy_segments(cudaStream_t st, const Mat4& T, const CopySeg* segs, int n_segs) {
    CopySeg s[4] = {{nullptr, nullptr, 0u, 0}, {nullptr, nullptr, 0u, 0}, {nullptr, nullptr, 0u, 0}, {nullptr, nullptr, 0u, 0}};
    uint32_t blocks = 0;
    for (int k = 0; k < n_segs && k < 4; ++k) { s[k] = segs[k]; blocks += (segs[k].n + 255u) / 256u; }
    if (blocks == 0) return cudaSuccess;
    k_copy_segments<<<blocks, 256, 0, st>>>(T, s[0], s[1], s[2], s[3]);
    return cudaGetLastError();
}
cudaError_t launch_affine_copy(cudaStream_t st, const Mat4& T, bool do_transform, const float4* in, float4* out, uint32_t n) {
    if (n == 0) return cudaSuccess;
    k_affine_copy<<<(n + 255) / 256, 256, 0, st>>>(T, do_transform ? 1 : 0, in, out, n);
    return cudaGetLastError();
}

// ============================================================================================
// U3  voxelize_preserving_labels
// ============================================================================================
// Radix-sort segment = the run of points one warp ranks (stably, match.any) in a pass.  The walk is a serial chain of rows, so
// segments are as short as the counter matrices allow: 8 rows of 32 up to 2 M points, longer beyond (<= 8192 segments).
constexpr uint32_t RS_ROWS_MIN = 8, RS_MAX_SEGS = 8192;
constexpr int      RB = 9;                  // radix digit: 9 bits -- a LiDAR scan's 27-bit voxel keys sort in three passes
constexpr uint32_t RD = 1u << RB;
__host__ __device__ inline uint32_t rs_seg_len(uint32_t n) {
    uint32_t rows = (uint32_t)(((unsigned long long)n + 32ull * RS_MAX_SEGS - 1ull) / (32ull * RS_MAX_SEGS));
    rows = (rows + RS_ROWS_MIN - 1u) / RS_ROWS_MIN * RS_ROWS_MIN;
    return 32u * (rows < RS_ROWS_MIN ? RS_ROWS_MIN : rows);
}

// ============================================================================================
// Fused form: one cooperative launch per node (grid-wide barriers between the phases above)
// ============================================================================================
// The per-node prologue of OfflineMapUpdater::callback_node is 25 small dependent kernels in the stepwise form (U3: 22,
// U1: 3) and is bound by launch latency, not by work.  k_node_fused runs the same phases -- same arithmetic, same
// order, bit-identical results -- as ONE cooperative kernel: every phase is a loop over the virtual blocks of the stepwise
// kernel, phases are separated by grid.sync().  The fetch_VoI partition of the map (U1) is independent of the scan's
// voxelisation (U3), so its three phases ride in U3's first three.  The radix sort runs only the passes the key width
// needs (the stepwise form always runs four).
namespace cg = cooperative_groups;
constexpr int FT = 1024;                 // threads per CTA
constexpr int FW = FT / 32;

// rank of the flagged threads of one FT-wide row in thread order: `before` = flagged threads in front of this one, `round` = all
__device__ __forceinline__ void cta_rank(bool flag, uint32_t* s_w /*[FW]*/, uint32_t& before, uint32_t& round) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned bal = __ballot_sync(FULL_MASK, flag);
    if (lane == 0) s_w[warp] = __popc(bal);
    __syncthreads();
    uint32_t b = 0, r = 0;
#pragma unroll
    for (int w = 0; w < FW; ++w) { const uint32_t c = s_w[w]; b += (w < warp) ? c : 0u; r += c; }
    before = b + __popc(bal & ((1u << lane) - 1u));
    round = r;
    __syncthreads();
}
__device__ __forceinline__ uint32_t cta_sum(uint32_t c, uint32_t* s_w /*[FW]*/) {
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(FULL_MASK, c, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = c;
    __syncthreads();
    uint32_t t = 0;
#pragma unroll
    for (int w = 0; w < FW; ++w) t += s_w[w];
    __syncthreads();
    return t;
}

// U3's 1-NN, out of line: k_node_fused runs at __launch_bounds__(1024, 1), which allows at most 64 registers per thread
__device__ __noinline__ uint32_t u3_nearest(const float4* __restrict__ pts, const uint32_t* __restrict__ order, const uint32_t* __restrict__ vox_start,
                                            const uint32_t* __restrict__ vox_key, uint32_t nv, VoxelGridDims g, float4 c) {
    return voxel_grid_nn(pts, order, vox_start, vox_key, nv, g, c);
}

struct VoxPlan {                          // carve-up of the voxeliser's scratch (host and device agree through this one function)
    uint32_t *key_a, *idx_a, *key_b, *idx_b, *cnt_x, *cnt_y, *tot, *chunk, *vstart, *vkey, *partial;
    uint32_t seg, nseg;
};
__host__ __device__ inline VoxPlan vox_plan(void* tmp, uint32_t n) {
    VoxPlan p;
    uint32_t* w = reinterpret_cast<uint32_t*>(tmp);
    p.seg  = rs_seg_len(n);
    p.nseg = (n + p.seg - 1) / p.seg;
    p.key_a = w;            p.idx_a = p.key_a + n;
    p.key_b = p.idx_a + n;  p.idx_b = p.key_b + n;
    p.cnt_x = p.idx_b + n;                                            // [RD][nseg] digit histogram per segment (even passes)
    p.cnt_y = p.cnt_x + (size_t)RD * (p.nseg + 1);                    // ... (odd passes)
    p.tot   = p.cnt_y + (size_t)RD * (p.nseg + 1);                    // [RD] points per digit
    p.chunk = p.tot + RD;                                            // (n + PART_CHUNK - 1) / PART_CHUNK + 1
    p.vstart = p.chunk + ((size_t)(n + PART_CHUNK - 1) / PART_CHUNK + 1);   // n + 2
    p.vkey   = p.vstart + ((size_t)n + 2);                            // n + 2
    p.partial = p.vkey + ((size_t)n + 2);                             // 6 * kFusedMaxGrid
    return p;
}

// U1 of a fused launch, one function per phase (grid barriers between them are the caller's).
// (0) selected points per chunk
__device__ __forceinline__ void u1_count(const FusedJob& J, uint32_t pchunks, uint32_t* s_w) {
    const int tid = threadIdx.x;
    for (uint32_t vb = blockIdx.x; vb < pchunks; vb += gridDim.x) {
        const uint32_t b0 = vb * PART_CHUNK, b1 = min(J.pn, b0 + PART_CHUNK);
        uint32_t c = 0;
        for (uint32_t i = b0 + tid; i < b1; i += FT) c += part_pred(J.P, J.pin[i]) ? 1u : 0u;
        const uint32_t t = cta_sum(c, s_w);
        if (tid == 0) J.chunk_tmp[vb] = t;
    }
}
// (1) chunk offsets and the total (last CTA)
__device__ __forceinline__ void u1_offsets(const FusedJob& J, uint32_t pchunks, uint32_t* s_part) {
    if (blockIdx.x != gridDim.x - 1) return;
    const uint32_t t = block_excl_scan(J.chunk_tmp, J.chunk_tmp, (int)pchunks, s_part);
    if (threadIdx.x == 0) *J.d_total_sel = t;
}
// (2) stable scatter.  kChain: the selected points go through T_sel, then T_sel2 (two transformPointCloud calls in sequence, each
// rounded on its own); the rest is not written.
template <bool kChain>
__device__ __forceinline__ void u1_scatter(const FusedJob& J, uint32_t pchunks, uint32_t* s_w) {
    const int tid = threadIdx.x;
    for (uint32_t vb = blockIdx.x; vb < pchunks; vb += gridDim.x) {
        const uint32_t b0 = vb * PART_CHUNK, b1 = min(J.pn, b0 + PART_CHUNK);
        uint32_t sel_base = J.chunk_tmp[vb];
        uint32_t rest_base = b0 - sel_base;
        for (uint32_t r0 = b0; r0 < b1; r0 += FT) {
            const uint32_t i = r0 + tid;
            const bool ok = i < b1;
            const float4 p = ok ? J.pin[i] : make_float4(0.f, 0.f, 0.f, 0.f);
            const bool s = ok && part_pred(J.P, p);
            uint32_t rank_sel, round;
            cta_rank(s, s_w, rank_sel, round);
            if (ok) {
                if (kChain) {
                    if (s) J.out_sel[sel_base + rank_sel] = pcl_affine(J.T_sel2.m, pcl_affine(J.T_sel.m, p));
                } else {
                    if (s) J.out_sel[sel_base + rank_sel] = J.xform_sel ? pcl_affine(J.T_sel.m, p) : p;
                    else   J.out_rest[rest_base + (i - r0) - rank_sel] = p;
                }
            }
            const uint32_t valid = min((uint32_t)FT, b1 - r0);
            sel_base += round;
            rest_base += valid - round;
        }
    }
}

// kChain = false: U1 and U3 are independent jobs and U1's phases ride in U3's first three (the updater's prologue).
// kChain = true: the resident map generator's modes (FusedJob::map / d_map, DESIGN.md section 8).  With has_part, one mapgen
// node: U1 runs first, then U3 voxelises U1's output out_sel[0 .. *d_total_sel) -- a count only the device knows -- and the voxels
// go to vout and to the map at its tail d_map[0], which moves past them.  Without has_part, parking: U3 voxelises the map's current
// chunk map[d_map[1] .. d_map[0]) into vout and, after a grid barrier (the 1-NN reads the chunk until then), moves the voxels to
// the chunk's start, where the next chunk starts behind them.
template <bool kChain>
__global__ void __launch_bounds__(FT, 1) k_node_fused(FusedJob J) {
    cg::grid_group grid = cg::this_grid();
    extern __shared__ uint32_t s_c[];        // [FW][RD] next free destination per digit, one row per warp (also the min/max staging)
    __shared__ uint32_t s_w[FW];
    __shared__ uint32_t s_part[34];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t G = gridDim.x, bid = blockIdx.x;
    const uint32_t pchunks = (J.pn + PART_CHUNK - 1) / PART_CHUNK;
    VoxGrid* g = J.grid;
    // phase profile of CTA 0 (nanoseconds, %globaltimer): read back by erasor_updater_get_fused_profile
#define PH(slot) do { if (bid == 0 && tid == 0) { unsigned long long t__; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t__)); g->prof[slot] = t__; } } while (0)
    PH(0);
    // the map's tail and chunk start, read by every CTA before the first barrier (CTA 0 moves them after one)
    uint32_t map_tail = 0, map_chunk = 0;
    if (kChain) {
        const volatile uint32_t* dm = J.d_map;
        map_tail = dm[0]; map_chunk = dm[1];
        if (J.has_part) {
            u1_count(J, pchunks, s_w);
            grid.sync();
            u1_offsets(J, pchunks, s_part);
            grid.sync();
            u1_scatter<true>(J, pchunks, s_w);
            grid.sync();
        }
    }
    const bool part = !kChain && J.has_part;             // the independent U1 job
    const float4* const vin = !kChain ? J.vin : (J.has_part ? J.out_sel : J.map + map_chunk);
    const uint32_t n = !kChain ? J.vn : (J.has_part ? *J.d_total_sel : map_tail - map_chunk);
    const VoxPlan vp = vox_plan(J.vtmp, n);
    const uint32_t nseg = vp.nseg, SEG = vp.seg;

    // ---- phase 0: getMinMax3D partials per CTA | partition: selected points per chunk ----
    if (n) {
        for (uint32_t i = bid * FT + tid; i < 2u * RD * (nseg + 1u); i += G * FT) vp.cnt_x[i] = 0u;      // both histogram matrices (contiguous)
        uint32_t mn[3] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu}, mx[3] = {0u, 0u, 0u};
        for (uint32_t i = bid * FT + tid; i < n; i += G * FT) {
            const float4 p = vin[i];
            const uint32_t a = float_to_ordered(p.x + 0.0f), b = float_to_ordered(p.y + 0.0f), c = float_to_ordered(p.z + 0.0f);
            mn[0] = min(mn[0], a); mx[0] = max(mx[0], a);
            mn[1] = min(mn[1], b); mx[1] = max(mx[1], b);
            mn[2] = min(mn[2], c); mx[2] = max(mx[2], c);
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const uint32_t a = __reduce_min_sync(FULL_MASK, mn[k]), b = __reduce_max_sync(FULL_MASK, mx[k]);
            if (lane == 0) { s_c[warp * 6 + k] = a; s_c[warp * 6 + 3 + k] = b; }
        }
        __syncthreads();
        if (tid < 6) {
            uint32_t r = (tid < 3) ? 0xFFFFFFFFu : 0u;
            for (int w = 0; w < FW; ++w) r = (tid < 3) ? min(r, s_c[w * 6 + tid]) : max(r, s_c[w * 6 + tid]);
            vp.partial[bid * 6 + tid] = r;
        }
        __syncthreads();
    }
    if (part) u1_count(J, pchunks, s_w);
    grid.sync();
    PH(1);

    // ---- phase 1: VoxelGrid set-up (CTA 0) | partition: chunk offsets (last CTA) ----
    if (bid == 0) {
        if (n && warp < 6) {                    // reduce the per-CTA partials: warp k < 3 the minimum of axis k, warps 3..5 the maxima
            uint32_t r = (warp < 3) ? 0xFFFFFFFFu : 0u;
            for (uint32_t c = lane; c < G; c += 32) r = (warp < 3) ? min(r, vp.partial[c * 6 + warp]) : max(r, vp.partial[c * 6 + warp]);
            r = (warp < 3) ? __reduce_min_sync(FULL_MASK, r) : __reduce_max_sync(FULL_MASK, r);
            if (lane == 0) s_w[warp] = r;
        }
        __syncthreads();
        if (tid == 0) {
            g->n_vox = 0; g->overflow = 0; g->npass = 0;
            if (n == 0) {
                *J.d_n_out = 0u;
            } else {
                float mm[6];                    // min x, y, z, max x, y, z
                for (int k = 0; k < 6; ++k) mm[k] = ordered_to_float(s_w[k]);
                bool ovf;
                unsigned long long cells;
                g->dims = voxel_grid_setup(mm, mm + 3, J.leaf, ovf, cells);
                g->overflow = ovf;
                // radix passes the keys need: keys are < cells (int32 arithmetic as in PCL), or < n in the overflow case
                unsigned long long lim = ovf ? (unsigned long long)n : cells;
                int bits = 32;
                if (lim <= 0x80000000ull) { bits = 1; while ((1ull << bits) < lim) ++bits; }
                g->npass = (bits + RB - 1) / RB;
            }
        }
        __syncthreads();
    }
    if (part) u1_offsets(J, pchunks, s_part);
    grid.sync();
    PH(2);

    // ---- phase 2: voxel keys + digit-0 histogram, one warp per 1024-point segment | partition: stable scatter ----
    const int npass = n ? g->npass : 0;
    uint32_t* const my_c = s_c + warp * RD;
    if (n) {
        const int ovf = g->overflow;
        const VoxelGridDims vg = g->dims;
        for (uint32_t e = bid * FT + tid; e < n; e += G * FT) {
            const float4 p = vin[e];
            const uint32_t k = ovf ? e : voxel_key_of(vg, p.x, p.y, p.z);   // overflow ("Leaf size is too small"): one voxel per point
            vp.key_a[e] = k; vp.idx_a[e] = e;
            atomicAdd(&vp.cnt_x[(size_t)(k & (RD - 1u)) * nseg + e / SEG], 1u);      // pass 0's histogram (counts: order-free)
        }
    }
    if (part) u1_scatter<false>(J, pchunks, s_w);
    grid.sync();
    PH(3);

    // ---- stable LSD radix sort of (key, cloud index), 9-bit digits, only the passes the key width needs.  Per pass:
    //   (a) one warp per digit scans its row of per-segment counts in place (exclusive) and leaves the digit's total;
    //   (b) one warp per segment ranks its points stably (match.any) behind base[digit] + row prefix and scatters them;
    //       on the way it counts the NEXT pass's digits per destination segment with RED (counts are order-free),
    //       so there is no separate histogram phase.
    for (int pass = 0; pass < npass; ++pass) {
        const uint32_t* ki = (pass & 1) ? vp.key_b : vp.key_a;  const uint32_t* ii = (pass & 1) ? vp.idx_b : vp.idx_a;
        uint32_t* ko = (pass & 1) ? vp.key_a : vp.key_b;        uint32_t* io = (pass & 1) ? vp.idx_a : vp.idx_b;
        uint32_t* cnt  = (pass & 1) ? vp.cnt_y : vp.cnt_x;     // this pass's histogram
        uint32_t* cntn = (pass & 1) ? vp.cnt_x : vp.cnt_y;     // the next pass's (zero on entry to (b))
        const int shift = pass * RB;
        const bool more = pass + 1 < npass;
        // (a)
        if (pass > 0 && more) for (uint32_t i = bid * FT + tid; i < RD * nseg; i += G * FT) cntn[i] = 0u;      // consumed two phases ago
        for (uint32_t d = (uint32_t)warp * G + bid; d < RD; d += G * FW) {
            uint32_t* row = cnt + (size_t)d * nseg;
            uint32_t carry = 0u;
            for (uint32_t c0 = 0; c0 < nseg; c0 += 512u) {              // 16 consecutive counters per lane and round, loaded together
                const uint32_t a = c0 + (uint32_t)lane * 16u;
                uint32_t v[16], sum = 0u;
#pragma unroll
                for (int j = 0; j < 16; ++j) { v[j] = (a + j < nseg) ? row[a + j] : 0u; }
#pragma unroll
                for (int j = 0; j < 16; ++j) { const uint32_t t = v[j]; v[j] = sum; sum += t; }
                uint32_t incl = sum;
                for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(FULL_MASK, incl, o); if (lane >= o) incl += t; }
                const uint32_t base = carry + incl - sum;
#pragma unroll
                for (int j = 0; j < 16; ++j) { if (a + j < nseg) row[a + j] = base + v[j]; }
                carry += __shfl_sync(FULL_MASK, incl, 31);
            }
            if (lane == 0) vp.tot[d] = carry;
        }
        grid.sync();
        PH(4 + 2 * pass);
        // (b)
        for (uint32_t seg = (uint32_t)warp * G + bid; seg < nseg; seg += G * FW) {     // consecutive segments on different SMs (match.any is a per-SM unit)
            const uint32_t b0 = seg * SEG, b1 = min(n, b0 + SEG);
            {   // next free destination per digit: points of smaller digits + points of this digit in earlier segments
                constexpr int DL = RD / 32;            // digits per lane
                uint32_t t[DL], c[DL], sum = 0u;
#pragma unroll
                for (int j = 0; j < DL; ++j) { t[j] = vp.tot[lane * DL + j]; }
#pragma unroll
                for (int j = 0; j < DL; ++j) { c[j] = cnt[(size_t)(lane * DL + j) * nseg + seg]; }
#pragma unroll
                for (int j = 0; j < DL; ++j) { const uint32_t x = t[j]; t[j] = sum; sum += x; }
                uint32_t incl = sum;
                for (int o = 1; o < 32; o <<= 1) { const uint32_t x = __shfl_up_sync(FULL_MASK, incl, o); if (lane >= o) incl += x; }
#pragma unroll
                for (int j = 0; j < DL; ++j) my_c[lane * DL + j] = incl - sum + t[j] + c[j];
            }
            __syncwarp();
            for (uint32_t r0 = b0; r0 < b1; r0 += 32u * RS_ROWS_MIN) {       // blocks of 8 rows: keys and indices loaded together, then ranked row by row
                uint32_t kk[RS_ROWS_MIN], vv[RS_ROWS_MIN];
#pragma unroll
                for (int r = 0; r < (int)RS_ROWS_MIN; ++r) {
                    const uint32_t e = r0 + (uint32_t)r * 32u + lane;
                    kk[r] = (e < b1) ? ki[e] : 0u; vv[r] = (e < b1) ? ii[e] : 0u;
                }
#pragma unroll
                for (int r = 0; r < (int)RS_ROWS_MIN; ++r) {
                    const uint32_t e = r0 + (uint32_t)r * 32u + lane;
                    const bool valid = e < b1;
                    const unsigned vm = __ballot_sync(FULL_MASK, valid);
                    unsigned my_peers = 0u;
                    uint32_t dst_o = 0u;
                    if (valid) {
                        const uint32_t d = (kk[r] >> shift) & (RD - 1u);
                        const unsigned peers = __match_any_sync(vm, d);
                        const uint32_t base = my_c[d];
                        __syncwarp(vm);
                        if (lane == __ffs(peers) - 1) my_c[d] = base + __popc(peers);
                        const uint32_t o = base + __popc(peers & ((1u << lane) - 1u));
                        ko[o] = kk[r]; io[o] = vv[r];
                        my_peers = peers; dst_o = o;
                    }
                    if (more) {
                        // next pass's histogram: one RED per run of equal digits when the whole run lands in one counter (the usual
                        // case -- neighbouring voxels share their upper key bits), else one per point
                        const uint32_t slot = valid ? ((kk[r] >> (shift + RB)) & (RD - 1u)) * nseg + dst_o / SEG : 0xFFFFFFFFu;
                        const int      lead = valid ? __ffs(my_peers) - 1 : lane;
                        const uint32_t lslot = __shfl_sync(FULL_MASK, slot, lead);
                        const unsigned differ = __ballot_sync(FULL_MASK, valid && slot != lslot);
                        if (valid) {
                            if ((my_peers & differ) == 0u) { if (lane == lead) atomicAdd(&cntn[slot], (uint32_t)__popc(my_peers)); }
                            else atomicAdd(&cntn[slot], 1u);
                        }
                    }
                    __syncwarp();
                }
            }
            __syncwarp();
        }
        grid.sync();
        PH(4 + 2 * pass + 1);
    }
    PH(12);
    if (n == 0) return;                                   // (grid-uniform)
    const uint32_t* skey = (npass & 1) ? vp.key_b : vp.key_a;
    const uint32_t* sidx = (npass & 1) ? vp.idx_b : vp.idx_a;

    // ---- heads of equal-key runs: count per chunk, offsets, ordered scatter ----
    const uint32_t hchunks = (n + PART_CHUNK - 1) / PART_CHUNK;
    for (uint32_t vb = bid; vb < hchunks; vb += G) {
        const uint32_t b0 = vb * PART_CHUNK, b1 = min(n, b0 + PART_CHUNK);
        uint32_t c = 0;
        for (uint32_t i = b0 + tid; i < b1; i += FT) c += (i == 0 || skey[i] != skey[i - 1]) ? 1u : 0u;
        const uint32_t t = cta_sum(c, s_w);
        if (tid == 0) vp.chunk[vb] = t;
    }
    grid.sync();
    if (bid == 0) {
        const uint32_t t = block_excl_scan(vp.chunk, vp.chunk, (int)hchunks, s_part);
        if (tid == 0) *J.d_n_out = t;
    }
    grid.sync();
    PH(13);
    const uint32_t n_vox = *J.d_n_out;
    if (bid == 0 && tid == 0) {
        g->n_vox = n_vox; vp.vstart[n_vox] = n;
        if (kChain) {                                  // every CTA has read the old values before the first barrier
            if (J.has_part) { J.d_map[0] = map_tail + n_vox; }
            else            { J.d_map[0] = map_chunk + n_vox; J.d_map[1] = map_chunk + n_vox; }
        }
    }
    for (uint32_t vb = bid; vb < hchunks; vb += G) {
        const uint32_t b0 = vb * PART_CHUNK, b1 = min(n, b0 + PART_CHUNK);
        uint32_t base = vp.chunk[vb];
        for (uint32_t r0 = b0; r0 < b1; r0 += FT) {
            const uint32_t i = r0 + tid;
            const bool hd = (i < b1) && (i == 0 || skey[i] != skey[i - 1]);
            uint32_t before, round;
            cta_rank(hd, s_w, before, round);
            if (hd) { vp.vstart[base + before] = i; vp.vkey[base + before] = skey[i]; }
            base += round;
        }
    }
    grid.sync();

    // ---- centroids (pcl::CentroidPoint, members in cloud order), exact 1-NN label, optional affine on the way out ----
    PH(14);
    for (uint32_t v0 = ((uint32_t)warp * G + bid) * 32u; v0 < n_vox; v0 += G * FT) {     // 32 consecutive voxels per warp, warps dealt round-robin over the SMs
        const uint32_t v = v0 + lane;
        if (v >= n_vox) continue;
        float4 c = voxel_centroid(vin, sidx, vp.vstart[v], vp.vstart[v + 1]);
        if (!g->overflow) {        // else every point is its own voxel: the nearest point is itself (or an identical earlier one)
            const uint32_t i = u3_nearest(vin, sidx, vp.vstart, vp.vkey, n_vox, g->dims, c);
            if (i != kNoPoint) c.w = vin[i].w;
        }
        if (kChain) {
            J.vout[v] = c;
            if (J.has_part) J.map[map_tail + v] = c;          // cloud_map += cloud_curr
        } else {
            J.vout[v] = J.xform_out ? pcl_affine(J.T_out.m, c) : c;
        }
    }
    PH(15);
    if (kChain && !J.has_part) {                           // parking: the chunk is read; its voxels take its place
        grid.sync();
        for (uint32_t v = bid * FT + tid; v < n_vox; v += G * FT) J.map[map_chunk + v] = J.vout[v];
    }
#undef PH
}

size_t partition_tmp_words(uint32_t n) { return (size_t)(n + PART_CHUNK - 1) / PART_CHUNK + 1; }

size_t voxelize_tmp_bytes(uint32_t n) {
    const size_t nseg = ((size_t)n + rs_seg_len(n) - 1) / rs_seg_len(n) + 1;
    // key/idx ping-pong (4 arrays), two digit-histogram matrices + digit totals, head-chunk counters, voxel starts/keys, per-CTA min/max partials
    return sizeof(uint32_t) * ((size_t)4 * n + 2 * (size_t)RD * nseg + RD + partition_tmp_words(n) + 2 * ((size_t)n + 2) + 64 + 6 * (size_t)kFusedMaxGrid);
}
size_t voxelize_tmp_bytes_upto(uint32_t n) {
    // every term of voxelize_tmp_bytes grows with n except the segment count, which drops where the segment length steps up;
    // it never exceeds min(RS_MAX_SEGS, ceil(n / (32 RS_ROWS_MIN)))
    const size_t nseg_max = std::min<size_t>(RS_MAX_SEGS, ((size_t)n + 32 * RS_ROWS_MIN - 1) / (32 * RS_ROWS_MIN));
    const size_t nseg = ((size_t)n + rs_seg_len(n) - 1) / rs_seg_len(n);
    return voxelize_tmp_bytes(n) + sizeof(uint32_t) * 2 * (size_t)RD * (nseg_max > nseg ? nseg_max - nseg : 0);
}

template <bool kChain>
static cudaError_t launch_fused_kernel(cudaStream_t st, const FusedJob& J, uint32_t work, int sm_count, int max_ctas) {
    constexpr size_t SMEM = sizeof(uint32_t) * FW * RD;
    static int max_ctas_per_sm = -1;
    if (max_ctas_per_sm < 0) {
        cudaError_t e = cudaFuncSetAttribute(k_node_fused<kChain>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM);
        if (e != cudaSuccess) return e;
        int v = 0;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, k_node_fused<kChain>, FT, SMEM);
        if (e != cudaSuccess) return e;
        max_ctas_per_sm = v;
    }
    if (max_ctas_per_sm < 1) return cudaErrorLaunchOutOfResources;
    uint32_t G = (work + FT - 1) / FT;
    const uint32_t cap = (uint32_t)std::min<long long>((long long)sm_count * max_ctas_per_sm, (long long)kFusedMaxGrid);
    G = G < 1u ? 1u : (G > cap ? cap : G);
    if (max_ctas > 0 && G > (uint32_t)max_ctas) G = (uint32_t)max_ctas;      // look-ahead jobs leave most SMs to the current node's path
    FusedJob jj = J;
    void* args[] = {&jj};
    return cudaLaunchCooperativeKernel((const void*)k_node_fused<kChain>, dim3(G), dim3(FT), args, SMEM, st);
}

cudaError_t launch_node_fused(cudaStream_t st, const FusedJob& J, int sm_count, int max_ctas) {
    return launch_fused_kernel<false>(st, J, J.vn > J.pn ? J.vn : J.pn, sm_count, max_ctas);
}

cudaError_t launch_map_chained(cudaStream_t st, const FusedJob& J, int sm_count) {
    return launch_fused_kernel<true>(st, J, J.vn > J.pn ? J.vn : J.pn, sm_count, 0);
}

}  // namespace erasor
