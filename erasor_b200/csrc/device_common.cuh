// device_common.cuh -- device arithmetic shared by kernels.cu and updater_kernels.cu.  Everything here has to be bit-identical
// to oracle/, so each rule exists once: the no-FMA float spelling, PCL's affine, pcl::VoxelGrid's set-up, keys and centroids,
// and the grid-pruned exact 1-NN of voxelize_preserving_labels (erasor_utils.cpp:80-114), plus the CTA-wide exclusive scan.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "device_types.h"

namespace erasor {

#define FULL_MASK 0xFFFFFFFFu

// Float arithmetic that must match the reference is spelled with round-to-nearest intrinsics so that nvcc cannot contract
// a*b+c into an FMA: the reference's x86-64 build (no -march, CMakeLists.txt:3-4) has none.
#define FM(a, b) __fmul_rn((a), (b))
#define FA(a, b) __fadd_rn((a), (b))
#define FS(a, b) __fsub_rn((a), (b))
#define FD(a, b) __fdiv_rn((a), (b))

// pcl::transformPointCloud, PCL 1.8 scalar path: ((m0*x + m1*y) + m2*z) + m3 in float, no contraction -- oracle
// transform_point_cloud (OfflineMapUpdater.cpp:436).  T: the top three rows of a row-major 4x4 (12 floats).
__device__ __forceinline__ float4 pcl_affine(const float* __restrict__ T, float4 p) {
    float4 o;
    o.x = FA(FA(FA(FM(T[0], p.x), FM(T[1], p.y)), FM(T[2], p.z)), T[3]);
    o.y = FA(FA(FA(FM(T[4], p.x), FM(T[5], p.y)), FM(T[6], p.z)), T[7]);
    o.z = FA(FA(FA(FM(T[8], p.x), FM(T[9], p.y)), FM(T[10], p.z)), T[11]);
    o.w = p.w;
    return o;
}

// exclusive scan of in[0..n) into out[0..n) (may alias) by the whole CTA; every thread returns the total.
__device__ inline uint32_t block_excl_scan(const uint32_t* in, uint32_t* out, int n, uint32_t* s_part /*[34]*/) {
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
    const int seg = (n + nt - 1) / nt;
    const int b0 = min(n, tid * seg), b1 = min(n, b0 + seg);
    uint32_t sum = 0;
    for (int i = b0; i < b1; ++i) sum += in[i];
    uint32_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(FULL_MASK, incl, o);
        if (lane >= o) incl += v;
    }
    __syncthreads();                     // s_part may still be read from a previous call
    if (lane == 31) s_part[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        const uint32_t w = lane < nw ? s_part[lane] : 0u;
        uint32_t wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(FULL_MASK, wi, o);
            if (lane >= o) wi += v;
        }
        if (lane < nw) s_part[lane] = wi - w;
        if (lane == 31) s_part[33] = wi;
    }
    __syncthreads();
    uint32_t run = s_part[warp] + incl - sum;
    const uint32_t total = s_part[33];
    for (int i = b0; i < b1; ++i) {
        const uint32_t v = in[i];
        out[i] = run;
        run += v;
    }
    __syncthreads();
    return total;
}

// ============================================================================================
// pcl::VoxelGrid (VoxelGridDims: device_types.h)
// ============================================================================================
// applyFilter's set-up from the cloud's getMinMax3D.  `overflow`: dx * dy * dz does not fit in int32 ("Leaf size is too small
// for the input dataset"; the filter then returns its input).  `cells` = div[0] * div[1] * div[2], exact.
__device__ __forceinline__ VoxelGridDims voxel_grid_setup(const float* mn, const float* mx, float leaf, bool& overflow, unsigned long long& cells) {
    VoxelGridDims g;
    g.leaf = leaf;
    g.inv = FD(1.0f, leaf);
    long long d = 1;
    cells = 1ull;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        d *= (long long)FM(FS(mx[k], mn[k]), g.inv) + 1;
        g.min_b[k] = (int)floorf(FM(mn[k], g.inv));
        g.div[k] = (int)floorf(FM(mx[k], g.inv)) - g.min_b[k] + 1;
        cells *= (unsigned long long)(unsigned)g.div[k];
    }
    overflow = d > 2147483647LL;
    return g;
}

// cell of coordinate x along one axis, counted from the grid's first cell
__device__ __forceinline__ int voxel_cell(float x, float inv, int min_b) { return (int)FS(floorf(FM(x, inv)), (float)min_b); }
// key of cell (i, j, k): int32 arithmetic as in PCL
__device__ __forceinline__ uint32_t voxel_key(const VoxelGridDims& g, int i, int j, int k) {
    return (uint32_t)(i + j * g.div[0] + k * (g.div[0] * g.div[1]));
}
__device__ __forceinline__ uint32_t voxel_key_of(const VoxelGridDims& g, float x, float y, float z) {
    return voxel_key(g, voxel_cell(x, g.inv, g.min_b[0]), voxel_cell(y, g.inv, g.min_b[1]), voxel_cell(z, g.inv, g.min_b[2]));
}

// Both voxelisers hand their points over as an accessor: pts[i] is point i as a float4 (x, y, z, intensity).
// A voxel is a run order[a..e) of point indices in cloud order.

// pcl::CentroidPoint: float sums over the voxel's members in cloud order, divided by float(count)
template <class Pts>
__device__ __forceinline__ float4 voxel_centroid(Pts pts, const uint32_t* __restrict__ order, uint32_t a, uint32_t e) {
    float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f;
    for (uint32_t k = a; k < e; ++k) {
        const float4 p = pts[order[k]];
        sx = FA(sx, p.x); sy = FA(sy, p.y); sz = FA(sz, p.z); si = FA(si, p.w);
    }
    const float cn = (float)(e - a);
    return make_float4(FD(sx, cn), FD(sy, cn), FD(sz, cn), FD(si, cn));
}

// Conservative distance along one axis from coordinate x to the voxel cell with (absolute) index `cell`, which lies `off` cells
// away from x's own cell (off < 0: below, > 0: above, 0: the same slab).  A point is assigned to `cell` when
// floorf(x * (1 / leaf)) == cell in float arithmetic, so the cell's faces sit within a few ulp of cell * leaf and (cell + 1) * leaf;
// `slack` covers that and the rounding of this expression, so the returned gap never exceeds the true one.
__device__ __forceinline__ float cell_gap(float x, int cell, int off, float leaf, float slack) {
    if (off == 0) return 0.0f;
    const float g = (off > 0) ? ((float)cell * leaf - x) : (x - (float)(cell + 1) * leaf);
    return fmaxf(g - slack, 0.0f);
}

constexpr uint32_t kNoPoint = 0xFFFFFFFFu;

// Exact 1-NN of the centroid c into the un-voxelised points, through the voxel grid itself (cells = voxels): c's own cell first,
// then the shells of Chebyshev radius 1, 2, ... around it, each cell skipped when even its nearest corner is provably farther
// than the best so far, until nothing unseen can be closer.  Ties go to the lowest point index.  Same result as comparing c
// against every point (tests/test_grid_nn_model.py), at a few cells per centroid; the loop is oracle/'s, line by line.
// Voxel v (key vox_key[v], ascending over v < nv) holds order[vox_start[v] .. vox_start[v + 1]).  Returns the nearest point's
// index, or kNoPoint when 4096 shells held none.
// The oracle also stops after shell 64 once it has a candidate.  For a finite centroid that rule never decides: the centroid lies
// within rounding of its own non-empty voxel, so after shell 1 the best distance is <= ~3 leaf^2, and the reach test ends the
// search after shell 2, since (2 * leaf * 0.9999)^2 > 3 leaf^2.
template <class Pts>
__device__ __forceinline__ uint32_t voxel_grid_nn(Pts pts, const uint32_t* __restrict__ order, const uint32_t* __restrict__ vox_start,
                                                  const uint32_t* __restrict__ vox_key, uint32_t nv, VoxelGridDims g, float4 c) {
    const int ci = voxel_cell(c.x, g.inv, g.min_b[0]), cj = voxel_cell(c.y, g.inv, g.min_b[1]), ck = voxel_cell(c.z, g.inv, g.min_b[2]);
    float best_d = __int_as_float(0x7f800000);
    uint32_t best_i = kNoPoint;
    const float slack = 1.0e-3f * g.leaf + 4.0e-6f * fmaxf(fabsf(c.x), fmaxf(fabsf(c.y), fabsf(c.z)));
    int rad = 0;
    while (true) {
        // scan the shell of Chebyshev radius `rad`
        for (int a = -rad; a <= rad; ++a) {
            const int ii = ci + a;
            if (ii < 0 || ii >= g.div[0]) continue;
            for (int b = -rad; b <= rad; ++b) {
                const int jj = cj + b;
                if (jj < 0 || jj >= g.div[1]) continue;
                for (int cc = -rad; cc <= rad; ++cc) {
                    if (max(abs(a), max(abs(b), abs(cc))) != rad) continue;
                    const int kk = ck + cc;
                    if (kk < 0 || kk >= g.div[2]) continue;
                    // Skip the cell when even its nearest corner is provably farther than the best so far (strictly: no tie can hide
                    // there).  The gaps are shortened by more than the float error of the cell assignment, so this only drops work.
                    if (rad > 0) {
                        const float gx = cell_gap(c.x, ii + g.min_b[0], a, g.leaf, slack);
                        const float gy = cell_gap(c.y, jj + g.min_b[1], b, g.leaf, slack);
                        const float gz = cell_gap(c.z, kk + g.min_b[2], cc, g.leaf, slack);
                        if (0.999f * (gx * gx + gy * gy + gz * gz) > best_d) continue;
                    }
                    const uint32_t key = voxel_key(g, ii, jj, kk);
                    uint32_t lo = 0, hi = nv;                 // first voxel with vox_key >= key
                    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (vox_key[mid] < key) lo = mid + 1; else hi = mid; }
                    if (lo >= nv || vox_key[lo] != key) continue;
                    for (uint32_t k = vox_start[lo]; k < vox_start[lo + 1]; ++k) {
                        const uint32_t i = order[k];
                        const float4 p = pts[i];
                        const float dx = FS(c.x, p.x), dy = FS(c.y, p.y), dz = FS(c.z, p.z);
                        const float d = FA(FA(FM(dx, dx), FM(dy, dy)), FM(dz, dz));
                        if (d < best_d || (d == best_d && i < best_i)) { best_d = d; best_i = i; }
                    }
                }
            }
        }
        const float reach = FM(FM((float)rad, g.leaf), 0.9999f);
        if (best_i != kNoPoint && best_d < FM(reach, reach)) break;
        ++rad;
        if (rad > 64 && best_i != kNoPoint) break;
        if (rad > 4096) break;
    }
    return best_i;
}

}  // namespace erasor
