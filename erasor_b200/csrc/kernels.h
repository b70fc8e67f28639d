// kernels.h -- launch wrappers of the path's kernels (definitions in kernels.cu; K1's geometry form in k1_geo.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "device_types.h"

namespace erasor {

struct CopyJob {
    const float4* src;
    float4*       dst;
    uint32_t      n;
    uint32_t      pad_;
};

size_t k1_smem_bytes(int R, int B);
size_t k3_smem_bytes(int B);

// K1's warps per CTA over shared tables of this many bytes: beyond 56 KB (40 x 360 bins: 173 KB) one CTA fits per SM and needs 32
// warps to cover K1's latencies, else four 8-warp CTAs do.  K2 walks the VoI lists with the count of the K1 launch that wrote them.
constexpr size_t kK1SmallTables = 56 * 1024;
inline int k1_warps(size_t table_smem_bytes) { return table_smem_bytes > kK1SmallTables ? 32 : 8; }

// The most table bytes the K1 launch over tables of table_bytes can take on a device whose blocks opt in to smem_optin bytes of
// shared memory: the opt-in less the static shared memory of the kernel the launch runs.  launch_k1 (node: node mode, prof: its
// profiling build; else the mask and cloud modes) and launch_k1_geo (table_bytes: the sum of its geometries' k1_geo_smem_bytes).
// Node mode's 32-warp kernels keep a 32 KB VoI ring in static shared memory, so they reach fewer bins than the other modes
// (H100, 227 KB opt-in: about 16 560 bins against 19 300).
cudaError_t k1_table_limit(size_t table_bytes, bool node, bool prof, size_t smem_optin, size_t* limit);
cudaError_t k1_geo_table_limit(size_t table_bytes, size_t smem_optin, size_t* limit);

cudaError_t launch_init_tables(cudaStream_t st, uint32_t* zmin, uint32_t* zmax, size_t n, uint32_t* cnt, size_t n_cnt, uint32_t* n_recs,
                               uint32_t* frame_rejected, uint32_t* n_flagged, int F, uint32_t* queue);

// poses != null: node mode (the map cloud is the resident global map; fetch_VoI's cut + transform fused into the binning)
cudaError_t launch_k1(cudaStream_t st, const K1GeoTables& t, const float4* map_pts, const float4* qry_pts, const ChunkDesc* chunks, int n_chunks, int F,
                      unsigned long long* fence, const NodePose* poses,
                      uint32_t* list_idx /*node mode: map index of every VoI point, per chunk*/, uint32_t* list_cnt /*node mode: VoI points per chunk*/,
                      bool qry_xyz = false /*the query cloud is packed x y z, 12 bytes per point (mask modes)*/,
                      uint32_t* prof = nullptr /*node mode only: run the profiling build, kK1ProfSlots cycle counters per warp*/);

// K1's geometry form (node mode): G's geometries binned in one scan of the map; smem = the sum of their k1_geo_smem_bytes.
size_t k1_geo_smem_bytes(int R, int B);
cudaError_t launch_k1_geo(cudaStream_t st, const K1Geo& G, size_t smem, const float4* map_pts, const float4* qry_pts, const ChunkDesc* chunks,
                          int n_chunks, int F, unsigned long long* fence, const NodePose* poses, uint32_t* list_idx, uint32_t* list_cnt, bool qry_xyz);

cudaError_t launch_k3(cudaStream_t st, const SrtParams& P, int F, const K1GeoTables& t, const uint32_t* chunk_range, const uint32_t* frame_off,
                      uint32_t* dst_start, uint8_t* status, uint8_t* action, uint32_t* flag_slot, uint32_t* n_flagged, uint32_t* frame_rec_base,
                      FlagRec* recs, uint32_t* n_recs, uint32_t rec_capacity, uint32_t* queue, uint32_t* bucket_list);

// mask modes: Scan Ratio Test + stable scatter of the flagged bins + R-GPF records / queue in one kernel (no k3_srt launch);
// t.ch_cnt holds K1's raw per-chunk counts
cudaError_t launch_k2_srt(cudaStream_t st, const SrtParams& P, int F, const K1GeoTables& t, const ChunkDesc* chunks, const uint32_t* chunk_range,
                          uint32_t n_chunks_map, const float4* pts, const NodePose* poses, const uint32_t* frame_off, uint32_t* n_flagged, FlagRec* recs,
                          uint32_t* n_recs, uint32_t rec_capacity, uint32_t* queue, uint32_t* bucket_list, float4* out_pts, uint32_t* out_src,
                          const uint32_t* list_idx, const uint32_t* list_cnt, int k1_warps /*warps of the K1 launch that wrote the lists*/,
                          const SrtSweep* sweep /*node mode: a Scan Ratio Test sweep, or null*/);

// the stable scatter of one cloud (0 map, 1 query: whose bin ids it reads); flag_slot == null: every bin of dst_start's cloud that
// has an offset is scattered (cloud mode); otherwise the flagged bins only
cudaError_t launch_k2(cudaStream_t st, const K1GeoTables& t, int cloud, const ChunkDesc* chunks, uint32_t chunk_base, uint32_t n_chunks,
                      const float4* pts, const NodePose* poses, const uint32_t* dst_start, const uint32_t* flag_slot, const uint32_t* n_flagged,
                      float4* out_pts, uint32_t* out_src, const uint32_t* list_idx, const uint32_t* list_cnt, int k1_warps);

// cloud mode: both clouds' stable scatters in one launch (chunk rows: map first, then query)
cudaError_t launch_k2_both(cudaStream_t st, const K1GeoTables& t, const ChunkDesc* chunks, uint32_t n_chunks_map, uint32_t n_chunks_qry,
                           const float4* map_pts, const uint32_t* dst_start_map, float4* out_map, uint32_t* src_map,
                           const float4* qry_pts, const uint32_t* dst_start_qry, float4* out_qry, uint32_t* src_qry);

int k4_num_launches(bool with_class_c);
// sorted_pts / sorted_src: K2's output (bins contiguous in source order + source index of every slot).
// queue / bucket_list: the size-bucketed work queue K3 filled (device_types.h).
cudaError_t launch_k4(cudaStream_t st, cudaStream_t st_b, cudaStream_t st_c, const GpfParams& P, FlagRec* recs, uint32_t* queue,
                      const uint32_t* bucket_list, uint32_t rec_capacity, const float4* sorted_pts, uint32_t* sorted_src, const uint32_t* frame_off,
                      float4* part_pts, uint8_t* keep_mask, uint8_t* ground_mask, uint32_t* frame_rejected, unsigned char* gscratch,
                      int sm_count, unsigned long long* fence, const K4Fold& fold, int classes /*bit 0|1: A and B, bit 2: C*/,
                      const K4Sweep* sweep = nullptr /*a sweep's ground-filter groups and per-setting fold (node mode, records from k2_srt_sweep_scatter)*/);

// every record of the batch (F frames; cnt / dst_start [2][F][...], qry_off: the query half of frame_off); vox_cnt / vox_start
// per record
cudaError_t launch_k4b(cudaStream_t st, float leaf, int B, int F, const FlagRec* recs, const uint32_t* n_recs, uint32_t rec_capacity,
                       const uint32_t* cnt, const uint32_t* dst_start, const uint32_t* qry_off, const float4* qry_sorted, const float4* part_pts,
                       float4* vox_pts, uint32_t* vox_cnt, uint32_t* vox_start, unsigned char* gscratch, int grid);

// node-mode inserts: after K1, the action / flag slot of every (frame, bin) and the query scatter plan of the inserting bins
cudaError_t launch_ins_plan(cudaStream_t st, const SrtParams& P, int F, const K1GeoTables& t, const uint32_t* chunk_range, uint8_t* action,
                            uint32_t* flag_slot, uint32_t* ins_slot, uint32_t* n_ins, uint32_t* dst_start);
// after R-GPF (and K4b): per-frame sizes and offsets ins_off [F+1], then every frame's inserts into out, body -> origin by fwd [F][12]
cudaError_t launch_ins_assemble(cudaStream_t st, int B, int F, int vox, const uint8_t* action, const uint32_t* flag_slot, uint32_t* frame_rec_base,
                                const FlagRec* recs, const uint32_t* n_recs, uint32_t rec_capacity, const uint32_t* cnt, const uint32_t* dst_start,
                                const uint32_t* qry_off, const uint32_t* vox_cnt, const uint32_t* vox_start, const float4* qry_sorted,
                                const float4* part_pts, const float4* vox_pts, const float* fwd, uint32_t* bin_off, uint32_t* frame_cnt,
                                uint32_t* ins_off, float4* out, int sm_count);
constexpr int kInsAssembleLaunches = 4;

cudaError_t launch_k5(cudaStream_t st, int B, int version, int skip_voxelize, const uint32_t* cnt, const uint32_t* dst_start,
                      const uint8_t* action, const uint32_t* flag_slot, const FlagRec* recs, const uint32_t* n_recs,
                      const uint32_t* vox_cnt, const uint32_t* vox_start, const float4* map_sorted, const float4* qry_sorted,
                      const float4* part_pts, const float4* vox_pts, float4* arranged, float4* map_rej, float4* curr_rej,
                      CopyJob* jobs, uint32_t* out_sizes, uint32_t* tmp, int copy_grid);

cudaError_t launch_fold_keep(cudaStream_t st, const uint8_t* keep, const uint32_t* voi_index, size_t n, uint8_t* global_keep, size_t n_global);
cudaError_t launch_fill_u8(cudaStream_t st, uint8_t* p, size_t n, uint8_t v);
// the re-test map (erasor_map_create_retest): order-preserving compaction of pts[keep != 0], n < 2^32, in tiles of kCompactTile
// points.  launch_compact_count: the tiles' kept counts (tile_cnt), their exclusive prefix (tile_off) and the kept total (*total),
// compact_tiles(n) entries each; launch_compact_scatter then writes the kept points to out[0, *total) in point order.
constexpr uint32_t kCompactTile = 4096;
inline size_t compact_tiles(size_t n) { return (n + kCompactTile - 1) / kCompactTile; }
cudaError_t launch_compact_count(cudaStream_t st, const uint8_t* keep, size_t n, uint32_t* tile_cnt, uint32_t* tile_off, uint32_t* total);
cudaError_t launch_compact_scatter(cudaStream_t st, const float4* pts, const uint8_t* keep, size_t n, const uint32_t* tile_off, float4* out);
// exchange step of the frame-sharded job: pack the keep bytes into bits, AND the all-gathered words of every rank, unpack
cudaError_t launch_pack_keep_bits(cudaStream_t st, const uint8_t* keep, size_t n, uint32_t* words);
cudaError_t launch_and_unpack_keep(cudaStream_t st, const uint32_t* gathered, int n_ranks, size_t n, uint8_t* keep);

}  // namespace erasor
