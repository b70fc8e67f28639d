// updater_kernels.h -- launch wrappers of the caller-side device steps (definitions in updater_kernels.cu)
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "device_types.h"

namespace erasor {

struct Mat4 { float m[16]; };            // row-major 4x4, like Eigen::Matrix4f(r, c) = m[4 r + c]

enum { PART_RADIUS = 0, PART_SUBMAP = 1, PART_NOT_NEAR = 2 };
struct PartPred {
    int    kind;
    int    pad_;
    double x, y;                         // criterion point
    double limit;                        // PART_RADIUS: max_dist_square; PART_SUBMAP: submap_size; PART_NOT_NEAR: squared vehicle-body radius
};

struct VoxGrid {                         // pcl::VoxelGrid state of one filter call, kept on the device
    VoxelGridDims dims;
    uint32_t n_vox;
    int      overflow;
    int      npass;                      // 8-bit radix passes the key width needs
    unsigned long long prof[16];         // phase boundaries of the fused kernel's CTA 0 (ns, %globaltimer)
};

constexpr int kFusedMaxGrid = 1024;      // CTAs of the fused kernel (one per SM in practice); sizes the per-CTA min/max partials

// One cooperative launch = erasor_utils::voxelize_preserving_labels of one cloud (U3) and, optionally and independently, one
// stable partition of another (U1: fetch_VoI / set_submap / mapgen's body cut).  Either job may be empty.
struct FusedJob {
    // U3: vout[0..*d_n_out) = voxelised vin[0..vn) in ascending voxel key, labels restored by exact 1-NN, then (xform_out) T_out
    const float4* vin; uint32_t vn; float leaf; VoxGrid* grid; void* vtmp /*voxelize_tmp_bytes(vn)*/; float4* vout; uint32_t* d_n_out;
    Mat4 T_out; int xform_out;
    // U1: pred-true points of pin[0..pn) (optionally through the affine T_sel) to out_sel, the rest to out_rest, both in source
    // order; *d_total_sel receives the number selected
    int has_part; PartPred P; Mat4 T_sel; int xform_sel; const float4* pin; uint32_t pn; uint32_t* chunk_tmp /*partition_tmp_words(pn)*/;
    uint32_t* d_total_sel; float4* out_sel; float4* out_rest;
    // chained mode only (launch_map_chained): the resident map of the map generator and its two device-held offsets,
    // d_map[0] = tail (points in the map), d_map[1] = start of the current chunk; T_sel2 follows T_sel on the selected points
    Mat4 T_sel2; float4* map; uint32_t* d_map;
};
size_t partition_tmp_words(uint32_t n);
size_t voxelize_tmp_bytes(uint32_t n);
size_t voxelize_tmp_bytes_upto(uint32_t n);   // enough for any cloud of at most n points (voxelize_tmp_bytes is not monotone in n)
cudaError_t launch_node_fused(cudaStream_t st, const FusedJob& job, int sm_count, int max_ctas = 0 /*0: as many as the job wants, up to one per SM*/);
// The chained mode of the same kernel (updater_kernels.cu), for the resident map generator (mapgen_capi.cu):
//   has_part = 1  one mapgen node: U1 (P, T_sel then T_sel2 on the selected points, out_rest unused), grid barrier, U3 over
//                 out_sel[0 .. *d_total_sel) into vout[0 .. *d_n_out) and map[d_map[0] ..); d_map[0] advances.
//                 vin is unused; vn bounds the voxeliser's count (pn) and vtmp holds voxelize_tmp_bytes_upto(vn).
//   has_part = 0  parking: U3 over map[d_map[1] .. d_map[0]) into vout, grid barrier, the voxels moved to map[d_map[1] ..);
//                 both offsets end behind them.  vn bounds the chunk's size.
cudaError_t launch_map_chained(cudaStream_t st, const FusedJob& job, int sm_count);

cudaError_t launch_affine_copy(cudaStream_t st, const Mat4& T, bool do_transform, const float4* in, float4* out, uint32_t n);

// epilogue of callback_node (OfflineMapUpdater.cpp:281-290) in one launch: up to four copy segments, each optionally through
// the float affine T (pcl::transformPointCloud)
struct CopySeg { const float4* src; float4* dst; uint32_t n; int xform; };
cudaError_t launch_copy_segments(cudaStream_t st, const Mat4& T, const CopySeg* segs, int n_segs);

}  // namespace erasor
