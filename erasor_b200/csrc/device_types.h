// device_types.h -- shared host/device structs of the path's HBM layout (see DESIGN.md section 3).
#pragma once
#include <cstdint>

#include "binning.h"

namespace erasor {

constexpr uint32_t kSkip      = 0xFFFFFFFFu;   // dst_start value of a bin that is not scattered
constexpr uint16_t kNoBin16   = 0xFFFFu;       // bin id of a point that failed the z window / range test
constexpr uint32_t kIdPad     = 1024;          // slack entries behind the bin-id arrays: K2 prefetches ids without bounds checks
constexpr uint32_t kMapPad    = 256;           // slack points behind the resident map: node-mode K1 streams it without bounds checks
constexpr int      kListWarps = 32;            // node mode: per-chunk stride of the per-warp VoI list counters (K1 runs 8 or 32 warps)
constexpr uint32_t kK2Stage   = 512;           // node mode: per K2 warp and window, taken VoI entries staged for the scatter (beyond: re-walk)
constexpr int      kMaxIter   = 8;             // gf_iter upper bound for the tap arrays

// K1's profiling build (erasor_profile_k1): per warp, SM cycles spent in each phase of the node-mode map path, the warp's
// total from the end of the table set-up to the end of the flush, and its dense-row count
enum : int { kK1ProfScan = 0, kK1ProfCompact, kK1ProfBin, kK1ProfTable, kK1ProfLists, kK1ProfFlush, kK1ProfTotal, kK1ProfRows, kK1ProfSlots };

// status codes held on the device (values published through erasor_get_status)
enum : uint8_t { ST_LITTLE = 0, ST_MERGE = 1, ST_MAP_HIGH = 2, ST_BLOCKED = 3, ST_CURR_HIGH = 4 };
// what the selected bin is made of (erasor.cpp:493-563 / 346-427)
enum : uint8_t { ACT_MAP = 0, ACT_FLAG = 1, ACT_MERGE = 2, ACT_CURR = 3, ACT_NONE = 4, ACT_CURR_REJECTED_BIT = 0x10 };

// One contiguous run of points of one cloud of one frame, processed by one CTA of K1 / one warp of K2.
struct ChunkDesc {
    uint32_t begin;        // first point (index into the source cloud array: the concatenated batch clouds, or the resident global map in node mode)
    uint32_t len;          // points in this chunk
    uint32_t frame;        // frame index
    uint32_t cloud;        // 0 map, 1 query
    uint32_t frame_begin;  // source index of the frame's first point (node mode, map cloud: 0 -- every frame scans a prefix of the map)
    uint32_t bin_begin;    // index of the chunk's first point in the bin-id array (batch mode: == begin; node mode: the frame's map offset
                           // + begin, the offsets being f * n_map, or a re-test map's cumulative extents)
    uint32_t out_base;     // base of the frame's region in the scattered arrays and the per-frame masks (batch: frame_begin; node: the
                           // frame's map offset)
    uint32_t pad_;
};

// Node mode (map resident in HBM, erasor_process_nodes): what OfflineMapUpdater::fetch_VoI needs per frame
// (reference OfflineMapUpdater.cpp:381-438): the radius cut around the body position, in double on float
// differences, and the origin -> body affine (float, pcl::transformPointCloud association, no contraction).
struct NodePose {
    double px, py;         // tf_body2origin(0,3), (1,3) as the reference reads them (:246-247)
    double limit;          // pow(max_range, 2)
    float  T[12];          // rows 0..2 of tf_body2origin.inverse()
    float  pxf, pyf;       // px, py as floats (they are floats widened to double, so this is exact)
    float  lim_lo, lim_hi; // float guard band around limit: d2f < lim_lo => inside for sure, d2f > lim_hi => outside for sure
};

// pcl::VoxelGrid's cell grid of one filter call (device_common.cuh: voxel_grid_setup)
struct VoxelGridDims {
    float leaf, inv;           // leaf size and 1 / leaf
    int   min_b[3], div[3];    // first cell and number of cells per axis
};

struct SrtParams {
    double scan_ratio_threshold;
    double th_bin_max_h;
    int    minimum_num_pts;
    int    version;
    int    R, S, B;
    int    scatter_mode;       // 0: every bin (cloud outputs), 1: flagged bins only (mask outputs)
};

// Sweeps (erasor_process_nodes_sweep[_ex], DESIGN.md sections 8.5 and 8.6): the Scan Ratio Test fields of one setting and the
// settings of one K2 launch, passed by value (32 x 24 = 768 bytes of kernel parameters)
constexpr int kMaxSweepVariants = 32;
struct SrtVariant {
    double scan_ratio_threshold;
    double th_bin_max_h;
    int    minimum_num_pts;
    int    reserved;
};
struct SrtSweep {
    SrtVariant v[kMaxSweepVariants];
    int        n;                  // variants in use, 1..32
    int        pad_;
    uint32_t*  n_flagged;          // [F][32] flagged bins per (frame, variant) of the submission
};

struct GpfParams {
    double th_dist;            // gf_dist_thr
    double th_seeds;           // gf_th_seeds_height
    int    num_lowest_pts;
    int    num_lpr;
    int    iters;
    int    cov_mode;
};

// The sweep's R-GPF and fold (DESIGN.md sections 8.5 and 8.6).  The settings are grouped by their ground-filter fields: group g
// fits with gp[g] and holds the settings in bits[g] (the groups partition the settings and are ordered by their lowest setting).
// A bin fits once per group that shares a setting with its record (FlagRec::cursor) and zeroes keep[v * n + src] for every
// point that fit rejects and every such setting v; rejected[frame * 32 + v] counts them.  Passed as a __grid_constant__
// kernel parameter (32 x 36 bytes of groups).
struct K4Sweep {
    uint8_t*  keep;                // [V][n] variant masks
    uint32_t* rejected;            // [F][32]
    uint32_t  n;                   // map points (writes beyond it are dropped)
    int       n_groups;            // 1..32
    uint32_t  bits[kMaxSweepVariants];
    GpfParams gp[kMaxSweepVariants];
};

// Geometry sweeps (erasor_process_nodes_tune, DESIGN.md section 8.7): K1's geometry form bins every VoI point of the node batch
// under n geometries in one scan of the resident map.  Geometry g's polar tables are T, its outputs the arrays of one plain
// node-mode K1 launch with B bins, and its shared count / min / max tables the k1_smem_bytes(T.R, B) bytes at smem_off in the
// launch's dynamic shared memory.  Passed as a __grid_constant__ kernel parameter.
struct K1GeoTables {
    BinTablesView T;
    uint16_t*     bin_map;         // per dense VoI-list entry, as the plain launch writes them
    uint16_t*     bin_qry;
    uint32_t*     ch_cnt;          // [n_chunks][B + 1]
    uint32_t*     zmin;            // [2][F][B]
    uint32_t*     zmax;
    uint32_t*     cnt;             // [2][F][B + 1]
    int           B;
    uint32_t      smem_off;        // 16-byte aligned
};
struct K1Geo {
    K1GeoTables g[kMaxSweepVariants];
    int         n;                 // geometries of the launch, 1..32
    int         pad_;
};

// The multi-GPU fold, done in K4's epilogue: global_keep[index ? index[frame_base + src] : src] = 0 for every rejected point.
struct K4Fold {
    uint8_t*        keep;      // global keep mask of the map (null: no fold)
    const uint32_t* index;     // per-VoI-point global index (batch mode); null: the source index is the global index (node mode)
    uint32_t        n;         // size of the global mask (writes beyond it are dropped)
    uint32_t        pad_;
};

// R-GPF work queue.  K3 appends every flagged-bin record to the bucket of its size; K4's three size classes
// (A: one warp per bin, B: one 256-thread CTA per bin, C: one 1024-thread CTA per bin) walk their buckets from the
// largest bins to the smallest through an atomic cursor, so the long bins start first and no group idles while
// records of its class remain.
constexpr uint32_t kClassAMax   = 512;     // class A: n <= 512          (register bitonic sort, 16 keys per lane)
constexpr uint32_t kClassBMax   = 2560;    // class B: 512 < n <= 2560   (8 warps x 512 keys)
constexpr int      kNumBuckets  = 9;       // 0: C | 1-4: B | 5-8: A
constexpr int      kBucketC0 = 0, kBucketB0 = 1, kBucketA0 = 5;
constexpr int      kQueueCursor = 16;      // queue[kQueueCursor + class] : next virtual index of the class (0 A, 1 B, 2 C)
constexpr int      kQueueWords  = 32;      // queue[0 .. kNumBuckets) : records per bucket
ERASOR_HD int rgpf_bucket_of(uint32_t n) {
    if (n > kClassBMax) return 0;
    if (n > 2048u) return 1;
    if (n > 1536u) return 2;
    if (n > 1024u) return 3;
    if (n > kClassAMax) return 4;
    if (n > 384u) return 5;
    if (n > 256u) return 6;
    if (n > 128u) return 7;
    return 8;
}

// K4b's global scratch (bins beyond its shared-memory cap, cloud mode): the region of bin b starts at this byte offset, where
// dsq_b / dsm_b are the bin's scatter offsets in the query / map cloud.  The region holds 36 n + 4 bytes (n = qc + n_ground_final
// <= qc + cm: X Y Z I KEY, VST with n + 1 entries, ORD ORD2 VK); the 16 bytes per bin beyond 36 (qc + cm) keep it clear of the
// next bin's region when every map point of the bin is ground.  d_vox_scratch holds k4b_scratch_offset(NQ, NM, B) + 36 + 64 bytes.
ERASOR_HD uint64_t k4b_scratch_offset(uint32_t dsq_b, uint32_t dsm_b, uint32_t b) {
    return 36ull * ((uint64_t)dsq_b + dsm_b) + 16ull * b;
}

// Per flagged bin record written by K3 and completed by K4
struct FlagRec {
    uint32_t frame;
    uint32_t bin;
    uint32_t slot;             // index among the frame's flagged bins (bin order)
    uint32_t n_points;
    uint32_t src_begin;        // offset of the bin's points in the scattered map array (absolute)
    uint32_t n_seeds;
    uint32_t n_empty_fits;
    uint32_t n_ground_final;
    uint32_t cursor;           // a sweep's variants that flag the bin (bit v); 0 outside a sweep
    uint32_t n_rejected;       // points handed to map_rejected (0 when gf_iter == 0: the reference fills no outliers then)
    double   lpr_height;
    double   normal_d[kMaxIter][4];
    uint32_t n_ground[kMaxIter];
    uint32_t prof[8];          // SM cycles per phase (thread 0): load+idx sort, z sort, seeds, accumulate, svd, classify+compact, outputs, sweeps
};

}  // namespace erasor
