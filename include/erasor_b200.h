/* ============================================================================
 * erasor_b200.h -- C ABI of the H100-native R-POD -> Scan Ratio Test -> R-GPF path
 *
 * This is the drop-in boundary for the reference's `class ERASOR`
 * (reference include/erasor/erasor.h:43-147, src/offline_map_updater/src/erasor.cpp)
 * as used by its single caller OfflineMapUpdater::callback_node
 * (src/offline_map_updater/src/OfflineMapUpdater.cpp:266-284).  The reference has no
 * FFI layer of its own; each entry point below names the C++ member it replaces.
 *
 * Conventions
 *   - plain C types only; clouds are float[n][4] = x, y, z, intensity (pcl::PointXYZI's
 *     four used floats; on the device this is one float4 per point, 16-byte aligned);
 *   - every function returns 0 (ERASOR_OK) or a negative error code and never throws;
 *     erasor_last_error() gives the text;
 *   - one handle <-> one CUDA device + one stream; a handle is not thread-safe, but distinct handles may be driven from
 *     distinct host threads, and several handles on one device overlap on the GPU (the *_async entry points);
 *   - device buffers are owned by the handle, caller buffers by the caller;
 *     `ptr_kind` says whether caller buffers are host (pageable or pinned) or device memory;
 *   - bins are indexed  bin = sector * num_rings + ring  (theta outer, r inner: the order
 *     in which the reference walks and flattens its R-POD, erasor.cpp:309-320);
 *   - there is no CPU fallback: without a CUDA device erasor_create fails with ERASOR_E_CUDA.
 * ========================================================================== */
#ifndef ERASOR_B200_H
#define ERASOR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ERASOR_B200_ABI_VERSION 2

typedef struct erasor_ctx* erasor_handle_t;

/* The 15 keys ERASOR's constructor reads from /erasor/ (erasor.h:47-61), /erasor/version
 * (OfflineMapUpdater.cpp:81) and three mode switches that pin choices the reference leaves
 * to its third-party libraries. */
typedef struct {
    double max_range;              /* /erasor/max_range             erasor.h:47 */
    double min_h;                  /* /erasor/min_h                 erasor.h:51 */
    double max_h;                  /* /erasor/max_h                 erasor.h:50 */
    double th_bin_max_h;           /* /erasor/th_bin_max_h          erasor.h:52 (v2 only) */
    double scan_ratio_threshold;   /* /erasor/scan_ratio_threshold  erasor.h:53 */
    double rejection_ratio;        /* /erasor/rejection_ratio       erasor.h:56 (unused by the path) */
    double gf_dist_thr;            /* /erasor/gf_dist_thr           erasor.h:57 */
    double gf_th_seeds_height;     /* /erasor/gf_th_seeds_height    erasor.h:60 */
    double map_voxel_size;         /* /erasor/map_voxel_size        erasor.h:61 */
    int    num_rings;              /* /erasor/num_rings             erasor.h:48 */
    int    num_sectors;            /* /erasor/num_sectors           erasor.h:49 */
    int    num_lowest_pts;         /* /erasor/num_lowest_pts        erasor.h:54 */
    int    minimum_num_pts;        /* /erasor/minimum_num_pts       erasor.h:55 */
    int    gf_iter;                /* /erasor/gf_iter               erasor.h:58 */
    int    gf_num_lpr;             /* /erasor/gf_num_lpr            erasor.h:59 */
    int    version;                /* /erasor/version               OfflineMapUpdater.cpp:81 */
    int    cov_mode;               /* 0: pcl::computeMeanAndCovarianceMatrix of PCL<=1.10 (default), 1: PCL>=1.11 (shifted) */
    int    sort_mode;              /* must be 1: R-GPF z-sort ties in source order (std::sort's tie order is unspecified) */
    int    skip_voxelize;          /* 1: leave out v3's in-bin voxelize_preserving_labels (erasor.cpp:526-528) */
} erasor_params_t;

enum { ERASOR_PTR_HOST = 0, ERASOR_PTR_DEVICE = 1,
       /* OR-able onto either, mask modes only (erasor_process_frames* / erasor_process_nodes*): the QUERY cloud is packed
        * x y z, three floats per point.  The masks never read the query's intensity (it only travels into the cloud outputs,
        * erasor.cpp:526-563), and a caller that repacks pcl::PointXYZI (32 bytes) anyway ships a quarter less over PCIe. */
       ERASOR_PTR_QUERY_XYZ = 16 };
enum { ERASOR_CLOUD_MAP = 0, ERASOR_CLOUD_QUERY = 1 };

enum {
    ERASOR_OK            = 0,
    ERASOR_E_INVALID     = -1,   /* bad argument / parameter */
    ERASOR_E_CUDA        = -2,   /* CUDA runtime error, or no device */
    ERASOR_E_STATE       = -3,   /* call order violated (set_inputs -> compare -> get_*) */
    ERASOR_E_CAPACITY    = -4,   /* caller buffer too small */
    ERASOR_E_UNSUPPORTED = -5    /* e.g. num_rings*num_sectors beyond the shared-memory table limit */
};

/* status values, as the reference publishes them (erasor.h:12-18) */
#define ERASOR_STATUS_LITTLE_NUM     0.0f
#define ERASOR_STATUS_MERGE_BINS     0.25f
#define ERASOR_STATUS_MAP_IS_HIGHER  0.5f
#define ERASOR_STATUS_BLOCKED        0.8f
#define ERASOR_STATUS_CURR_IS_HIGHER 1.0f

/* ---- lifetime --------------------------------------------------------------------------- */
/* replaces ERASOR::ERASOR(ros::NodeHandle*) (erasor.h:46-103): parameters are fixed here. */
int  erasor_create(const erasor_params_t* params, int device, erasor_handle_t* out);
void erasor_destroy(erasor_handle_t h);
const char* erasor_last_error(erasor_handle_t h);   /* h may be NULL: error of the last failed erasor_create */
int  erasor_abi_version(void);
/* the handle's CUDA stream (cudaStream_t as void*), so callers can order their own work after it */
void* erasor_stream(erasor_handle_t h);
int  erasor_synchronize(erasor_handle_t h);

/* ---- the per-frame path, in the reference's call order ------------------------------------ */
/* replaces ERASOR::set_inputs(map_voi, query_voi) (erasor.cpp:57-85): both clouds already in the
 * egocentric body frame.  Builds both R-PODs (bin of every point, per-bin min/max z and count). */
int erasor_set_inputs(erasor_handle_t h, const float* map_voi_xyzi, size_t n_map,
                      const float* query_voi_xyzi, size_t n_query, int ptr_kind);
/* replaces compare_vois_and_revert_ground(frame) [version 2, erasor.cpp:332-434] and
 * compare_vois_and_revert_ground_w_block(frame) [version 3, erasor.cpp:438-571]:
 * Scan Ratio Test, status per bin, R-GPF on the flagged bins, selection. */
int erasor_compare(erasor_handle_t h, int version, int frame);
/* sizes of the four output clouds of the last compare (so the caller can allocate) */
int erasor_get_output_sizes(erasor_handle_t h, size_t* n_arranged, size_t* n_complement,
                            size_t* n_map_rejected, size_t* n_curr_rejected);
/* replaces ERASOR::get_static_estimate(arranged, complement) (erasor.cpp:612-626); output in the
 * reference's order: selected bins theta-major / r-minor, then ground_viz; complement in source order. */
int erasor_get_static_estimate(erasor_handle_t h, float* arranged_xyzi, size_t cap_arranged, size_t* n_arranged,
                               float* complement_xyzi, size_t cap_complement, size_t* n_complement, int ptr_kind);
/* replaces ERASOR::get_outliers(map_rejected, curr_rejected) (erasor.cpp:322-327) */
int erasor_get_outliers(erasor_handle_t h, float* map_rejected_xyzi, size_t cap_map, size_t* n_map_rejected,
                        float* curr_rejected_xyzi, size_t cap_curr, size_t* n_curr_rejected, int ptr_kind);
/* ERASOR::ground_viz (public member, erasor.h:127): ground points of the flagged bins, the tail of `arranged`.
 * ground_xyzi may be NULL to query *n_ground. */
int erasor_get_ground_viz(erasor_handle_t h, float* ground_xyzi, size_t cap, size_t* n_ground, int ptr_kind);
/* Device-resident callers (the OfflineMapUpdater mirror, erasor_updater_*): device pointers to the four output clouds of the
 * last compare, in place -- no copy, no synchronisation.  Sizes: erasor_get_output_sizes.  They live in the handle's own
 * buffers on erasor_stream(h) and are valid until the next erasor_set_inputs / batch call on this handle; work that reads
 * them must be ordered on that stream.  Any pointer may be NULL. */
int erasor_device_outputs(erasor_handle_t h, const float** arranged, const float** complement, const float** map_rejected,
                          const float** curr_rejected);
/* replaces ERASOR::get_max_range() (erasor.cpp:628) */
double erasor_get_max_range(erasor_handle_t h);

/* ---- parity taps (the reference exposes these only as public members / rviz topics) --------- */
/* r_pod_map / r_pod_curr (erasor.h:143-144): bin of every input point (-1: complement / dropped),
 * per-bin min z, max z (NaN where the bin is empty) and count.  Any pointer may be NULL. Host buffers.
 * After a one-node erasor_process_nodes: the tables of that node's VoI and query (bin_of_point must be NULL there). */
int erasor_get_bins(erasor_handle_t h, int which_cloud, int32_t* bin_of_point, float* min_h, float* max_h, uint32_t* count);
/* per-bin status of the last compare as published on /SCDR/debug/polygons_marker (erasor.cpp:439-441,570) */
int erasor_get_status(erasor_handle_t h, float* status);
/* R-GPF taps: for each bin that ran extract_ground (processing order), its bin id, point count, seed count,
 * LPR height, and per iteration the plane (nx,ny,nz,d) and the ground count.  *n_planes in: capacity, out: count. */
int erasor_get_planes(erasor_handle_t h, int32_t* bin_ids, int32_t* n_points, int32_t* n_seeds, double* lpr_height,
                      double* normal_d /* [n][gf_iter][4] */, int32_t* n_ground /* [n][gf_iter] */, size_t* n_planes);
/* per map_voi point (source order): keep_map = 0 where the point is rejected as dynamic (non-ground point of a
 * flagged bin), is_ground = 1 where R-GPF retained it as ground.  Host buffers, either may be NULL. */
int erasor_get_static_mask(erasor_handle_t h, uint8_t* keep_map, uint8_t* is_ground);
/* events the reference would have thrown / invoked UB on (SURVEY App. B-1, B-3): points with y == -0.0f and
 * x <= -0 (fenced to y = +0), plane fits on an empty set (fenced to normal (0,0,1), d = 0), and sector decisions
 * that stayed ambiguous after double-double arithmetic (never observed). */
int erasor_get_fence_counts(erasor_handle_t h, uint64_t* negzero_points, uint64_t* empty_plane_fits, uint64_t* ambiguous_sector);

/* ---- frame-independent batch mode (north_star: frames shard across GPUs, masks all-gathered) --- */
/* Runs the whole path on n_frames independent (map_voi, query_voi) pairs and writes, for every map point of
 * every frame, keep = 0 where the frame rejects it.  Frame f's map points are
 * map_xyzi[map_offsets[f] .. map_offsets[f+1]) (offsets in points, n_frames+1 entries, host memory);
 * likewise the queries.  keep_mask has map_offsets[n_frames] bytes.  Clouds / mask: host or device (ptr_kind).
 * A batch too large for one submission (more than 2^32 points, or more flagged-bin records than the work queue holds)
 * is split into consecutive sub-batches internally. */
int erasor_process_frames(erasor_handle_t h, const float* map_xyzi, const uint64_t* map_offsets,
                          const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                          uint8_t* keep_mask, int ptr_kind);
/* Same, returning as soon as the work is enqueued on the handle's stream; erasor_wait(h) completes it (and reports its
 * error, if any).  Host buffers must stay valid and -- to actually be asynchronous -- be pinned.  Two or three handles
 * fed round-robin overlap consecutive batches on the GPU (one batch's R-GPF runs under the next one's binning). */
int erasor_process_frames_async(erasor_handle_t h, const float* map_xyzi, const uint64_t* map_offsets,
                                const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                                uint8_t* keep_mask, int ptr_kind);
int erasor_wait(erasor_handle_t h);
/* Multi-GPU exchange helper: fold per-frame keep masks onto the global map (a point survives unless some frame
 * rejected it): global_keep[voi_index[i]] = 0 where keep_mask[i] == 0.  The mask ACCUMULATES over calls -- start a job
 * with erasor_reset_keep_mask.  Indices >= n_global are ignored.  DEVICE pointers; asynchronous on the handle's stream. */
int erasor_fold_keep_masks(erasor_handle_t h, const uint8_t* keep_mask, const uint32_t* voi_index, size_t n, uint8_t* global_keep, size_t n_global);
int erasor_reset_keep_mask(erasor_handle_t h, uint8_t* global_keep, size_t n_global);   /* global_keep[] = 1; DEVICE pointer, asynchronous */
/* erasor_process_frames with the fold done in R-GPF's epilogue (no extra pass over the masks): what a rank of the
 * frame-sharded job runs per batch.  voi_index (global index of every VoI point, map_offsets[n_frames] entries) and
 * global_keep: DEVICE.  global_keep accumulates (see erasor_reset_keep_mask). */
int erasor_process_frames_fold(erasor_handle_t h, const float* map_xyzi, const uint64_t* map_offsets,
                               const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                               uint8_t* keep_mask, int ptr_kind,
                               const uint32_t* voi_index, uint8_t* global_keep, size_t n_global);
int erasor_process_frames_fold_async(erasor_handle_t h, const float* map_xyzi, const uint64_t* map_offsets,
                                     const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                                     uint8_t* keep_mask, int ptr_kind,
                                     const uint32_t* voi_index, uint8_t* global_keep, size_t n_global);
/* per-frame counters of the last erasor_process_frames / erasor_process_nodes: flagged bins and rejected points (host arrays of n_frames) */
int erasor_get_frame_stats(erasor_handle_t h, uint32_t* n_flagged_bins, uint32_t* n_rejected_points);

/* ---- map-resident frame-independent mode: the global map is uploaded once, per node only pose + query cross PCIe ---- */
/* The initial map of OfflineMapUpdater::load_global_map (OfflineMapUpdater.cpp:107-167), origin frame, resident in HBM,
 * together with its global keep mask (one byte per map point, 1 = static so far).  One map may be attached to any
 * number of handles on the same device. */
typedef struct erasor_map_ctx* erasor_map_t;
int    erasor_map_create(const float* map_xyzi, size_t n_map, int ptr_kind, int device, erasor_map_t* out);
void   erasor_map_destroy(erasor_map_t m);
size_t erasor_map_size(erasor_map_t m);
int    erasor_map_reset_keep(erasor_map_t m);                              /* keep[] = 1 (synchronous) */
int    erasor_map_get_keep(erasor_map_t m, uint8_t* keep, int ptr_kind);   /* synchronous copy; wait for the handles first */
uint8_t*     erasor_map_keep_device(erasor_map_t m);                       /* the mask in HBM (n_map bytes) */
const float* erasor_map_points_device(erasor_map_t m);
int    erasor_attach_map(erasor_handle_t h, erasor_map_t m);
/* n_frames nodes against the attached map, every one tested against the same (initial) map.  For node f:
 *   poses7[7 f .. 7 f + 7) = msg->odom, body -> origin, x y z qx qy qz qw (HOST memory; OfflineMapUpdater.cpp:219);
 *   query cloud = query_xyzi[query_offsets[f] .. query_offsets[f+1]): the scan as callback_node hands it to
 *   ERASOR::set_inputs, i.e. voxelised and in the body frame (OfflineMapUpdater.cpp:237-241).
 * On the device, per node: fetch_VoI (OfflineMapUpdater.cpp:381-438: radius cut at voi_max_range around the body position
 * in double, origin -> body transform; <= 0 selects /erasor/max_range) fused into the polar binning, then SRT and R-GPF
 * as in erasor_process_frames.  Results:
 *   - the map's keep mask &= this batch's verdicts (always; written by R-GPF's epilogue);
 *   - frame_keep (nullable): n_frames x n_map bytes, frame f's keep mask over the GLOBAL map indices
 *     (1 also for points outside the node's VoI);
 *   - keep_out (nullable): copy of the map's keep mask after this batch (n_map bytes).
 * query_xyzi / frame_keep / keep_out: host or device (ptr_kind); host buffers should be pinned.  With ERASOR_PTR_QUERY_XYZ
 * in ptr_kind, query_xyzi holds 3 floats per point.  Node mode's K1 keeps a 32 KB VoI ring in shared memory next to its bin
 * tables, so it reaches fewer bins than erasor_create admits (H100: about 16 560 against 19 300 at 100 rings): a larger geometry
 * runs in the other modes, and node mode, its sweeps and tune refuse it with ERASOR_E_UNSUPPORTED before enqueuing anything. */
int erasor_process_nodes(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                         double voi_max_range, uint8_t* frame_keep, uint8_t* keep_out, int ptr_kind);
int erasor_process_nodes_async(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                               double voi_max_range, uint8_t* frame_keep, uint8_t* keep_out, int ptr_kind);
/* per-node counters of the last erasor_process_nodes: points inside the VoI (|map_voi_|), flagged bins, rejected points */
int erasor_get_node_stats(erasor_handle_t h, uint32_t* n_voi_points, uint32_t* n_flagged_bins, uint32_t* n_rejected_points);

/* ---- Scan Ratio Test sweep: one node-mode pass, one keep mask per setting (DESIGN.md section 8.5) ---- */
/* The three per-sensor knobs of the Scan Ratio Test, one setting of a sweep (reserved: 0). */
typedef struct {
    double scan_ratio_threshold;
    double th_bin_max_h;
    int    minimum_num_pts;
    int    reserved;
} erasor_srt_variant_t;
/* erasor_process_nodes (same map, voi_max_range, queries, ptr_kind, sub-batches, geometry, version, gf_* and cov_mode) run under
 * n_variants settings of the Scan Ratio Test at once: K1's binning and R-GPF run once, over the union of the bins the settings
 * flag, and each setting's verdicts go to its own mask.  The handle's own scan_ratio_threshold, th_bin_max_h and minimum_num_pts
 * are not read.  variant_keep: DEVICE, n_variants x n_map bytes, mask v at [v * n_map, (v + 1) * n_map); it ACCUMULATES like
 * erasor_process_frames_fold's global_keep (start with erasor_reset_keep_mask(h, variant_keep, n_variants * n_map)); handles
 * may share one.  Mask v equals the map's keep mask after erasor_process_nodes with setting v on a fresh map.  The map's own
 * keep mask is not written.  ERASOR_E_INVALID: n_variants outside [1, 32], a null variants or variant_keep, no attached map,
 * node inserts on; ERASOR_E_STATE: a submission pending. */
int erasor_process_nodes_sweep(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                               double voi_max_range, const erasor_srt_variant_t* variants, int n_variants, uint8_t* variant_keep, int ptr_kind);
int erasor_process_nodes_sweep_async(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                                     double voi_max_range, const erasor_srt_variant_t* variants, int n_variants, uint8_t* variant_keep, int ptr_kind);
/* per (setting, node) counters of the last sweep (erasor_process_nodes_sweep or erasor_process_nodes_sweep_ex), HOST arrays
 * [n_variants][n_frames] (nullable): flagged bins and rejected points, as erasor_get_node_stats reports them for that setting.
 * After a sweep, erasor_get_node_stats gives n_voi_points as usual and the counts of the union of the settings' flagged bins
 * (rejected points: each union bin's fit under the ground-filter fields of the lowest setting that flags it).  ERASOR_E_STATE
 * when the last node call was not a sweep. */
int erasor_get_sweep_stats(erasor_handle_t h, uint32_t* n_flagged_bins, uint32_t* n_rejected_points);

/* ---- Scan Ratio Test and ground-filter sweep (DESIGN.md section 8.6) ---- */
/* The eight per-sensor knobs of one setting: the Scan Ratio Test's three and R-GPF's five. */
typedef struct {
    double scan_ratio_threshold;
    double th_bin_max_h;
    double gf_dist_thr;
    double gf_th_seeds_height;
    int    minimum_num_pts;
    int    num_lowest_pts;
    int    gf_num_lpr;
    int    gf_iter;
} erasor_sweep_setting_t;
/* erasor_process_nodes_sweep with settings that also carry the ground-filter fields (geometry, version, cov_mode, skip_voxelize
 * and max_range still come from the handle, whose eight fields above are not read).  The settings are grouped by their five
 * ground-filter fields: each bin of the union of the settings' flagged bins is loaded and sorted by z once, then fitted once per
 * group among the settings that flag it.  Mask v equals the map's keep mask after erasor_process_nodes with setting v on a fresh
 * map; erasor_get_sweep_stats gives that run's flagged and rejected counts.  With every setting's ground-filter fields equal to
 * the handle's, it returns what erasor_process_nodes_sweep returns.  Arguments and refusals as erasor_process_nodes_sweep, and
 * ERASOR_E_UNSUPPORTED for a gf_iter above 8 (as erasor_create). */
int erasor_process_nodes_sweep_ex(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                                  double voi_max_range, const erasor_sweep_setting_t* settings, int n_settings, uint8_t* variant_keep, int ptr_kind);
int erasor_process_nodes_sweep_ex_async(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                                        double voi_max_range, const erasor_sweep_setting_t* settings, int n_settings, uint8_t* variant_keep, int ptr_kind);

/* ---- geometry and height-window sweep (DESIGN.md section 8.7) ---- */
/* ERASOR's polar geometry and z window (/erasor/max_range, min_h, max_h, num_rings, num_sectors), as erasor_params_t carries them */
typedef struct {
    double max_range;
    double min_h;
    double max_h;
    int    num_rings;
    int    num_sectors;
} erasor_geometry_t;
/* one setting of a tune call: a geometry and the eight fields of erasor_sweep_setting_t */
typedef struct {
    erasor_geometry_t      geometry;
    erasor_sweep_setting_t s;
} erasor_tune_setting_t;
/* erasor_process_nodes_sweep_ex over settings that may also differ in geometry (version, cov_mode and skip_voxelize still come
 * from the handle).  The VoI cut and the origin -> body transform run once per point; K1 bins each VoI point under every
 * distinct geometry in as few scans of the map as shared memory allows, and each geometry then runs the sweep_ex path on its own
 * bins.  Mask v equals the map's keep mask after erasor_process_nodes on a fresh map with a handle created with the handle's
 * parameters and setting v's thirteen fields, the same voi_max_range, queries and ptr_kind; erasor_get_sweep_stats gives that
 * run's counts.  voi_max_range <= 0 takes the settings' common max_range.  erasor_get_node_stats gives n_voi_points as usual;
 * its flagged-bin and rejected-point counts are the union counts of the geometry of setting 0.  With every setting carrying the
 * handle's own geometry the call is erasor_process_nodes_sweep_ex.  Refusals as erasor_process_nodes_sweep_ex, and with
 * erasor_create's codes a geometry it would refuse (num_rings * num_sectors outside [1, 65534], a table it cannot build, tables
 * beyond the device's shared memory), ERASOR_E_UNSUPPORTED for one beyond node mode's K1 (erasor_process_nodes); ERASOR_E_INVALID for voi_max_range <= 0 when the settings' max_range differ. */
int erasor_process_nodes_tune(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                              double voi_max_range, const erasor_tune_setting_t* settings, int n_settings, uint8_t* variant_keep, int ptr_kind);
int erasor_process_nodes_tune_async(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                                    double voi_max_range, const erasor_tune_setting_t* settings, int n_settings, uint8_t* variant_keep, int ptr_kind);

/* ---- node-mode inserts: the query points each node's static estimate puts back into the map (DESIGN.md section 8.4) ---- */
/* Opt-in per handle (default off; off changes nothing).  With it on, erasor_process_nodes also builds, per node f, inserted_f:
 * bin by bin in r_pod2pc order, the bins whose selected points hold query points -- R-GPF bins: bin_curr then the R-GPF ground
 * (version 3 without skip_voxelize: voxelize_preserving_labels of that, at map_voxel_size); version 2 also MERGE_BINS bins and
 * bins with query points only: bin_curr -- moved body -> origin with the node's pose (OfflineMapUpdater.cpp:281-290, 441-449),
 * intensity carried through.  The masks and counters are those of inserts off.
 * erasor_set_node_inserts: ERASOR_E_STATE while a submission is pending.  With inserts on, ERASOR_PTR_QUERY_XYZ queries are
 * refused (ERASOR_E_INVALID: the inserts need the intensity). */
int erasor_set_node_inserts(erasor_handle_t h, int enable);
/* after erasor_process_nodes (erasor_wait for the asynchronous form): the last call's inserts, node after node -- *d_xyzi: float4
 * device memory valid until the handle's next submission; offsets (HOST, n_frames + 1): node f is [offsets[f], offsets[f+1]) */
int erasor_get_node_inserts(erasor_handle_t h, const float** d_xyzi, uint64_t* offsets);
/* The map's insert store: erasor_map_append_inserts appends h's last call (synchronous); callers append in node order -- lanes
 * sharing a map append after their own erasor_wait.  The store also records where each appended node's inserts start (the
 * re-test map's extents below).  erasor_map_inserts: device pointer and point count; clear empties it. */
int erasor_map_append_inserts(erasor_map_t m, erasor_handle_t h);
int erasor_map_inserts(erasor_map_t m, const float** d_xyzi, size_t* n);
int erasor_map_clear_inserts(erasor_map_t m);
/* node mode's save_static_map: voxelize_preserving_labels(map[keep] ++ the map's inserts, leaf) through erasor_voxelize_batch
 * (its output rules and errors); with an empty store, the kept map alone.  Waits for h; *d_out valid until h's next voxelize. */
int erasor_save_node_map(erasor_handle_t h, erasor_map_t m, float leaf, const float** d_out, size_t* n_out);

/* ---- node-mode re-test: the inserts of every node tested again by the nodes after it (DESIGN.md section 8.4.1) ---- */
/* The re-test map of a node-mode job (DESIGN.md section 8.4.1): m's kept points in map order, then m's insert store in node
 * order, on m's device; keep all ones, empty store.  Node k of the store (k = 0 .. n_nodes-1) sees the prefix
 * [0, extent[k]), extent[k] = n_kept + store offset of node k.  m is not changed.  Synchronous (wait for the handles that write
 * m first).  Errors as erasor_map_create (erasor_last_error(NULL)); ERASOR_E_INVALID for a result of 2^32 points or more. */
int erasor_map_create_retest(erasor_map_t m, erasor_map_t* out);
/* n_nodes of a re-test map, and (nullable, n_nodes entries) the extents; ERASOR_E_INVALID for a map not made by the call above */
int erasor_map_retest_extents(erasor_map_t m, size_t* n_nodes, uint64_t* extents);
/* erasor_process_nodes against an attached re-test map: node f of the call is store node first_node + f and sees only its
 * extent.  Same poses / queries / ptr_kind / voi_max_range / keep_out / sub-batch rules as erasor_process_nodes; no frame_keep.
 * The map's keep mask &= the verdicts on the points each node sees.  Packed x y z queries (ERASOR_PTR_QUERY_XYZ) are allowed:
 * the pass has no inserts.  ERASOR_E_INVALID: the attached map is not a re-test map, first_node < 0 or first_node + n_frames >
 * n_nodes, node inserts on for h; ERASOR_E_STATE: no map attached, a submission pending.  A re-test map attached to
 * erasor_process_nodes or to the sweeps is a plain map (every point visible to every node). */
int erasor_process_nodes_retest(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets,
                                int n_frames, int first_node, double voi_max_range, uint8_t* keep_out, int ptr_kind);
int erasor_process_nodes_retest_async(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets,
                                      int n_frames, int first_node, double voi_max_range, uint8_t* keep_out, int ptr_kind);

/* erasor_utils::voxelize_preserving_labels (erasor_utils.cpp:80-114) of n_clouds clouds in one submission, each on its own
 * pcl::VoxelGrid, optionally followed by one pcl::transformPointCloud.  Cloud c is xyzi[offsets[c] .. offsets[c+1]) (offsets: HOST,
 * n_clouds + 1 entries, offsets[0] = 0); keep (nullable, offsets[n_clouds] bytes) selects the points with keep != 0; xyzi and keep
 * are host or device memory (ptr_kind; a device cloud 16-byte aligned).  pose7 (nullable, HOST, x y z qx qy qz qw) is applied to the
 * output as the updater applies /tf/lidar2body (geoPose2eigen(pose) * Identity, OfflineMapUpdater.cpp:89-104,240).
 * Cloud c's voxels are (*d_out)[out_offsets[c] .. out_offsets[c+1]) (float4 each; out_offsets: HOST, n_clouds + 1 entries), in
 * ascending voxel key, centroids summed in cloud order, labels from the exact 1-NN among the cloud's selected points with ties to
 * the lowest index; a cloud whose grid overflows int32 passes through with its labels restored.  *d_out is the handle's device
 * memory on erasor_stream(h), valid until the next erasor_voxelize_batch on h: it can go straight into erasor_process_nodes with
 * ERASOR_PTR_DEVICE, or erasor_map_points_device(m) with erasor_map_keep_device(m) can go in to save a node-mode map.
 * Synchronous: one device -> host read of the offsets.  ERASOR_E_INVALID: n_clouds < 1, offsets[0] != 0 or not monotone, leaf not
 * positive and finite, a non-finite x, y or z in a selected point (the message names the cloud and the point; the handle stays usable).
 * ERASOR_E_CAPACITY: a cloud of 2^31 points or more, or 2^32 - 1 points or more in all. */
int erasor_voxelize_batch(erasor_handle_t h, const float* xyzi, const uint64_t* offsets, int n_clouds, const uint8_t* keep, float leaf,
                          const double* pose7, int ptr_kind, const float** d_out, uint64_t* out_offsets);

/* ---- the path's single collective, behind the C ABI (north_star: one NCCL all-gather of the static masks) ------------ */
/* A communicator owned by the handle (NCCL is loaded with dlopen("libnccl.so.2") on first use).  Rank 0 calls
 * erasor_comm_unique_id and ships the 128 bytes to the other ranks by whatever means the host program has
 * (MPI, torch.distributed, a file); every rank then calls erasor_comm_init (collective). */
#define ERASOR_COMM_ID_BYTES 128
int erasor_comm_unique_id(uint8_t* id128);
int erasor_comm_init(erasor_handle_t h, const uint8_t* id128, int n_ranks, int rank);
int erasor_comm_destroy(erasor_handle_t h);
/* global_keep (DEVICE, n_global bytes, this rank's folded mask) <- AND over all ranks: the bytes are packed to bits
 * (8x less traffic), all-gathered with ONE ncclAllGather over NVLink and AND-ed + unpacked by a library kernel.
 * Asynchronous on the handle's stream.  Without a communicator (single GPU) it is a no-op. */
int erasor_allgather_and_keep(erasor_handle_t h, uint8_t* global_keep, size_t n_global);
/* The local half of that exchange on its own: out[i] = AND over r of masks[r][i] (DEVICE, contiguous [n_masks][n] bytes),
 * through the same bit-pack / AND / unpack kernels.  For callers with their own transport, and for single-GPU tests. */
int erasor_and_keep_masks(erasor_handle_t h, const uint8_t* masks, int n_masks, size_t n, uint8_t* out);

/* ---- instrumentation ---------------------------------------------------------------------- */
/* per flagged bin of the last run: point count and SM cycles per R-GPF phase (load + index sort, z sort, seeds,
 * accumulate, SVD + plane, classify + compact, outputs) plus the Jacobi sweep count in slot 7.  *n in: capacity, out: count. */
int erasor_get_rgpf_profile(erasor_handle_t h, uint32_t* n_points, uint32_t* prof8, size_t* n);
/* SM cycles per phase of the SRT kernel (K3), frame 0 of the last run: status passes, chunk-row prefixes, flagged-bin scan +
 * record base, map scatter offsets, records + R-GPF queue, query scatter offsets; slots 6-7 reserved (host array of 8). */
int erasor_get_srt_profile(erasor_handle_t h, uint32_t* cycles8);
/* K1 of the last node-mode batch again, as a profiling build: per warp of every chunk ([chunk][warp][8] words), the SM cycles
 * of the map path's phases -- scan (loads + radius test), ring compaction, transform + bin, list stores, table update,
 * barrier + flush -- then the warp's total and its dense-row count (all ones for a query chunk).  Rebuilds that batch's K1
 * tables with the same values.  *n in: capacity in words, out: words; out == null only queries the size. */
int erasor_profile_k1(erasor_handle_t h, uint32_t* out, size_t* n, int* warps_per_cta);
/* number of kernels this library launched on the handle since creation */
uint64_t erasor_kernel_launch_count(erasor_handle_t h);
/* CUDA-event time (ms) spent in the binning kernel (K1) since the last reset, and its launch count */
int erasor_get_kernel_time_ms(erasor_handle_t h, int kernel_id, double* total_ms, uint64_t* launches);
int erasor_reset_kernel_times(erasor_handle_t h, int enable_timing);
/* forget what earlier runs taught the handle (whether R-GPF's class C, bins beyond 2560 points, has been seen): the next run
 * launches what a new handle's first run would.  Results never depend on it, only which kernels are launched. */
int erasor_forget_run_history(erasor_handle_t h);

/* ============================================================================================
 * The caller, device-resident: erasor::OfflineMapUpdater (reference include/erasor/OfflineMapUpdater.h,
 * src/offline_map_updater/src/OfflineMapUpdater.cpp) with ROS stripped -- SURVEY.md section 8f rows 1-3.
 * The global map lives in HBM; per node only the raw scan and the pose cross PCIe.
 * ========================================================================================== */
typedef struct erasor_updater_ctx* erasor_updater_t;

typedef struct {
    double query_voxel_size;   /* /MapUpdater/query_voxel_size   OfflineMapUpdater.cpp:66 */
    double map_voxel_size;     /* /MapUpdater/map_voxel_size     :67 (unused by the path) */
    int    removal_interval;   /* /MapUpdater/removal_interval   :69 */
    int    is_large_scale;     /* /large_scale/is_large_scale    :75 */
    double submap_size;        /* /large_scale/submap_size       :76 */
    double max_range;          /* /erasor/max_range as read by the updater, default 60.0  :78 */
    int    version;            /* /erasor/version                :81 */
    int    pad_;
    double lidar2body[7];      /* /tf/lidar2body  x y z qx qy qz qw   :89-104 */
} erasor_updater_params_t;

/* replaces OfflineMapUpdater::OfflineMapUpdater() = set_params + load_global_map + new ERASOR (:5-32, 63-167);
 * the initial map is handed over as a host cloud instead of a PCD path. */
int  erasor_updater_create(const erasor_updater_params_t* up, const erasor_params_t* ep, const float* initial_map_xyzi, size_t n_map,
                           int device, erasor_updater_t* out);
void erasor_updater_destroy(erasor_updater_t u);
/* load_global_map again (:107-167) on a live updater: new initial map, counters and the handle's run history
 * (erasor_forget_run_history) reset, device buffers kept */
int  erasor_updater_reset(erasor_updater_t u, const float* initial_map_xyzi, size_t n_map);
const char* erasor_updater_last_error(erasor_updater_t u);
/* replaces OfflineMapUpdater::callback_node(msg) (:203-330): seq = msg->header.seq, odom7 = msg->odom as x y z qx qy qz qw
 * (body -> origin), lidar = msg->lidar in the LIDAR frame.  *processed = 1 when the node was processed (every
 * removal_interval-th call), 0 for the reference's "PASS!". */
int  erasor_updater_process_node(erasor_updater_t u, int seq, const double* odom7, const float* lidar_xyzi, size_t n_lidar, int ptr_kind,
                                 int* processed);
/* Optional look-ahead for callers that know the coming nodes' scans (file-based / offline runs: the reference replays a rosbag,
 * OfflineMapUpdater.cpp:203): starts a scan's upload, voxelize_preserving_labels and lidar -> body (:237-241) on a second stream,
 * so that it runs under the path of the node being processed.  Two look-aheads can be pending: hand in node k + 1's scan, then
 * call erasor_updater_process_node for node k.  A process_node call given the same (pointer, n, ptr_kind) consumes the
 * look-ahead -- results are identical with and without; one that matches nothing runs the usual way.  The scan buffer must
 * stay valid and unchanged until it has been consumed; a DEVICE scan must be complete (its producer synchronised) before the
 * call, because the look-ahead reads it on the updater's own second stream. */
int  erasor_updater_prefetch_scan(erasor_updater_t u, const float* lidar_xyzi, size_t n_lidar, int ptr_kind);
int  erasor_updater_map_size(erasor_updater_t u, size_t* n);
/* clouds of the last processed node (parity taps): 0 map_arranged_, 1 map_voi_ (body), 2 query_voi_ (body),
 * 5 map_rejected_ (origin), 7 map_outskirts_, 8 map_arranged_complement_ (large-scale).  xyzi may be NULL to query *n. */
int  erasor_updater_get_cloud(erasor_updater_t u, int which, float* xyzi, size_t cap, size_t* n, int ptr_kind);
/* replaces OfflineMapUpdater::save_static_map(voxel_size) minus the PCD write (:174-196) */
int  erasor_updater_save_static_map(erasor_updater_t u, float voxel_size, float* out_xyzi, size_t cap, size_t* n);
/* erasor_utils::voxelize_preserving_labels on a free-standing host cloud (erasor_utils.cpp:80-114) */
int  erasor_updater_voxelize(erasor_updater_t u, const float* xyzi, size_t n_in, float leaf, float* out_xyzi, size_t cap, size_t* n);
/* mapgen's per-node producer on the device (reference src/mapgen/mapgen.hpp:198-239): 2.7 m vehicle-body cut, 1.73 m lift,
 * pose transform, voxelize_preserving_labels at 0.2 m -> cloud_curr.  out_xyzi needs room for n_lidar points (cap). */
int  erasor_updater_mapgen_node(erasor_updater_t u, const double* odom7, const float* lidar_xyzi, size_t n_lidar, int ptr_kind,
                                float* out_xyzi, size_t cap, size_t* n);
/* the ERASOR handle inside the updater (for the parity taps above) */
erasor_handle_t erasor_updater_erasor(erasor_updater_t u);
uint64_t erasor_updater_kernel_launch_count(erasor_updater_t u);
/* phase boundaries (ns, %globaltimer of CTA 0) of the last fused prologue launch -- the per-node cooperative kernel that
 * voxelises the scan and cuts the VoI: [0] start, [1] min/max + partition count, [2] set-up + chunk offsets, [3] keys + partition
 * scatter, [4+2p] histogram + offsets of radix pass p, [5+2p] its scatter, [12] sort done, [13] run heads counted, [14] heads
 * scattered, [15] centroids + labels written. */
int erasor_updater_get_fused_profile(erasor_updater_t u, uint64_t* ns16);

/* ============================================================================================
 * PR / RR on the device: the reference's scripts/analysis_runner.py metric (erasor_b200/evaluate.py) by an exact
 * grid-indexed 1-NN from every ground-truth point into the estimate.  A handle of its own: one CUDA device + one stream,
 * scratch (16 B per estimate point plus the cell table) kept and grown on demand; not thread-safe.
 * ========================================================================================== */
typedef struct erasor_eval_ctx* erasor_eval_t;

typedef struct {
    uint64_t gt_static;          /* GT points whose class is not dynamic (252..259) */
    uint64_t gt_dynamic;
    uint64_t preserved_static;   /* static GT inliers whose nearest estimate point is static */
    uint64_t preserved_dynamic;  /* dynamic GT inliers whose nearest estimate point is dynamic */
    uint64_t inliers;            /* GT points with an estimate point at distance < voxelsize * sqrt(3) / 2 */
    uint64_t ambiguous_ties;     /* inliers whose equally-nearest estimate points hold both classes: only these may differ from sklearn */
} erasor_eval_counts_t;

int  erasor_eval_create(int device, erasor_eval_t* out);
void erasor_eval_destroy(erasor_eval_t e);
const char* erasor_eval_last_error(erasor_eval_t e);   /* e may be NULL: error of the last failed erasor_eval_create */
/* gt_xyzi: n_gt points; est_xyzi: n_est points, of which est_keep (nullable, n_est bytes) selects those with keep != 0.
 * The nearest estimate point is the one with the smallest double distance sqrt((dx*dx + dy*dy) + dz*dz); ties go to the lowest
 * estimate index (original index, also under a keep mask).  match (nullable, n_gt entries): that index for inliers, 0xFFFFFFFF
 * otherwise.  All buffers host or device (ptr_kind); device clouds 16-byte aligned.  With ERASOR_PTR_DEVICE a resident map is
 * scored in place: gt = est = erasor_map_points_device(m), est_keep = erasor_map_keep_device(m) (wait for its handles first).
 * Synchronous.  ERASOR_E_INVALID: a non-finite x, y or z in gt or in a selected estimate point, n_gt or n_est >= 2^32 - 1,
 * voxelsize <= 0.  An empty (or fully deselected) estimate gives no inliers, where sklearn would raise; an empty gt all-zero counts. */
int  erasor_evaluate(erasor_eval_t e, const float* gt_xyzi, size_t n_gt, const float* est_xyzi, size_t n_est,
                     const uint8_t* est_keep, double voxelsize, int ptr_kind, uint32_t* match, erasor_eval_counts_t* out);

/* The overlap report of analysis_runner.py (its overlap_report and est_S / est_D): the exact distance d from every selected
 * estimate point to its nearest GT point, at any range, as sklearn computes it (sqrt((dx*dx + dy*dy) + dz*dz) in double from the
 * float coordinates), with no bound on d.  Counts are over the selected estimate points. */
typedef struct {
    uint64_t n;                  /* selected estimate points */
    uint64_t est_static;         /* of them, not dynamic (252..259) */
    uint64_t est_dynamic;
    uint64_t below_half;         /* d < 0.5 * voxelsize (double comparisons, as numpy makes them) */
    uint64_t below_one;          /* d < voxelsize */
    uint64_t below_two;          /* d < 2 * voxelsize */
    uint64_t far_points;         /* points the far path settled (more than a few cells from every GT point) */
    double   max;                /* the largest d; NaN when n = 0 */
} erasor_eval_overlap_t;
/* Same inputs, pointer kinds and errors as erasor_evaluate (a resident map is scored in place the same way).  ranks / rank_values:
 * HOST arrays of n_ranks entries; rank_values[r] is the value at 0-based position ranks[r] of the selected points' distances
 * sorted ascending (ERASOR_E_INVALID when a rank is >= n).  est_dist (nullable, n_est doubles, host or device per ptr_kind): d per
 * estimate point, NaN where the keep mask drops it.  An empty selection gives n = 0 and no ranks; an empty GT gives d = +inf for
 * every selected point (sklearn raises on both).  Synchronous. */
int  erasor_eval_overlap(erasor_eval_t e, const float* gt_xyzi, size_t n_gt, const float* est_xyzi, size_t n_est,
                         const uint8_t* est_keep, double voxelsize, int ptr_kind, const uint64_t* ranks, size_t n_ranks,
                         double* rank_values, double* est_dist, erasor_eval_overlap_t* out);
/* *count = how many of the n keep bytes are nonzero (host or device per ptr_kind; synchronous): the n of erasor_eval_overlap for a
 * keep mask, so that a caller can compute its ranks before the call. */
int  erasor_eval_count_selected(erasor_eval_t e, const uint8_t* keep, size_t n, int ptr_kind, uint64_t* count);

/* ============================================================================================
 * ASCII PCD files on the device: the text of a whole file -> float[n][4] x y z intensity, and a cloud -> the text that
 * erasor_b200/evaluate.py's write_pcd_ascii and include/erasor/offline_map_updater.hpp's save_pcd_ascii write (the layout of
 * pcl::io::savePCDFileASCII).  Bit-identical to the host readers (np.loadtxt + astype(float32); istream >> double + (float)) and
 * byte-identical to the host writers ("%.8g"), except that NaN is written "nan" whatever its sign.  A handle of its own: one CUDA
 * device + one stream, scratch kept and grown on demand; not thread-safe.  Every call is synchronous.
 * ========================================================================================== */
typedef struct erasor_pcd_ctx* erasor_pcd_t;

typedef struct {
    uint64_t points;             /* POINTS of the header */
    uint64_t rows;               /* rows parsed: POINTS, or fewer when the file holds fewer data rows */
    uint64_t slow_tokens;        /* kept values the fast path could not decide, settled by exact big-integer arithmetic */
    uint64_t error_line;         /* 1-based line of the file that made the call fail with ERASOR_E_INVALID, else 0 */
    uint64_t header_lines;       /* lines up to and including DATA; 0 when the text holds no DATA line (the rest is then 0 too) */
    uint32_t fields;             /* bit 0 x, 1 y, 2 z, 3 intensity: which of them FIELDS names */
    uint32_t has_intensity;      /* 1 when FIELDS names intensity (otherwise the intensity column is 0) */
} erasor_pcd_info_t;

int  erasor_pcd_create(int device, erasor_pcd_t* out);
void erasor_pcd_destroy(erasor_pcd_t p);
const char* erasor_pcd_last_error(erasor_pcd_t p);    /* p may be NULL: error of the last failed erasor_pcd_create */
/* text: the whole file, len bytes, host or device (text_kind).  The header is read on the host: FIELDS (any order, extras allowed;
 * x, y, z required), COUNT (all 1), POINTS and DATA (ascii); otherwise ERASOR_E_UNSUPPORTED (binary files, COUNT > 1) or
 * ERASOR_E_INVALID.  Lines end at '\n', "\r\n" or a lone '\r' (Python's universal newlines, as read_pcd_ascii opens the file).
 * Rows follow np.loadtxt: '#' starts a comment, blank lines are skipped, blanks are ' ' \t \r \v \f, every row
 * holds one value per field (each one checked, kept or not), and reading stops after POINTS rows.  A bad row gives ERASOR_E_INVALID,
 * with its line in info->error_line and erasor_pcd_last_error.  out_xyzi (host or device per out_kind; a device cloud 16-byte
 * aligned) needs room for POINTS points; NULL only asks for *n = POINTS.  *n = rows parsed.  info (nullable) is written on every
 * return, as far as the header was read. */
int  erasor_pcd_parse_ascii(erasor_pcd_t p, const char* text, size_t len, int text_kind, float* out_xyzi, size_t cap, int out_kind,
                            size_t* n, erasor_pcd_info_t* info);
/* The whole file for n points (host or device per in_kind): the header, then "x y z intensity\n" per point, each value as
 * printf("%.8g", (double)v).  out == NULL (or cap too small: ERASOR_E_CAPACITY) returns the exact size in *len and keeps the text
 * for the following call with the same (xyzi, n, in_kind), which then only copies it out.  out: host or device per out_kind. */
int  erasor_pcd_format_ascii(erasor_pcd_t p, const float* xyzi, size_t n, int in_kind, char* out, size_t cap, int out_kind, size_t* len);

/* A PCD file in any DATA mode for n points (DESIGN.md section 12.3), with the same header as erasor_pcd_format_ascii (only the DATA
 * word differs).  ERASOR_PCD_ASCII is erasor_pcd_format_ascii, unchanged.  ERASOR_PCD_BINARY: the header, then the cloud's 16-byte
 * points in order, bit for bit.  ERASOR_PCD_BINARY_COMPRESSED: the header, uint32 compressed_size and uint32 uncompressed_size
 * (little-endian), then one LZF stream over x[n] | y[n] | z[n] | intensity[n] (PCL 1.8's writeBinaryCompressed layout for these
 * fields), encoded in independent segments by the rule of DESIGN.md section 12.3; erasor_pcd_load and PCL's reader rules read it
 * back bit for bit.  Byte identity with PCL's writers is not claimed.  Arguments and caching as erasor_pcd_format_ascii, keyed on
 * (xyzi, n, in_kind, data_mode); one cache serves both functions.  Errors: an unknown data_mode, a misaligned device cloud
 * (ERASOR_E_INVALID); binary_compressed with n x 16 > 0xFFFFFFFF (checked before anything is read) or a stream longer than
 * 0xFFFFFFFF bytes (ERASOR_E_UNSUPPORTED: the format's sizes are uint32).  n == 0 is a header-only file (binary_compressed: and
 * two zero sizes).  info (nullable) is written whenever *len is.  Synchronous. */
#define ERASOR_PCD_ASCII              0   /* the same numbering as erasor_pcd_load_info_t.data_mode */
#define ERASOR_PCD_BINARY             1
#define ERASOR_PCD_BINARY_COMPRESSED  2

typedef struct {
    uint32_t data_mode;
    uint32_t segments;            /* binary_compressed: independently encoded LZF segments */
    uint64_t header_bytes;
    uint64_t uncompressed_size;   /* binary_compressed: POINTS x 16 */
    uint64_t compressed_size;     /* binary_compressed: bytes of the LZF stream */
    uint64_t lzf_tokens;          /* binary_compressed: literal runs + back-references */
} erasor_pcd_format_info_t;

int  erasor_pcd_format(erasor_pcd_t p, const float* xyzi, size_t n, int in_kind, int data_mode, char* out, size_t cap, int out_kind,
                       size_t* len, erasor_pcd_format_info_t* info);

/* Any PCD DATA mode on the device (DESIGN.md section 12.1), with the field rules of PCL 1.8's PCDReader and
 * fromPCLPointCloud2<PointXYZI> (restated; PCL is not built here).  ascii goes to erasor_pcd_parse_ascii unchanged (results, errors
 * and info->ascii).  binary and binary_compressed: SIZE and TYPE are required (F 4/8, I/U 1/2/4, else ERASOR_E_UNSUPPORTED); COUNT is
 * optional (default 1); FIELDS/SIZE/TYPE/COUNT of different lengths, WIDTH x HEIGHT != POINTS, a file shorter than its header
 * promises, uncompressed_size != POINTS x point_step and a malformed LZF stream are ERASOR_E_INVALID.  x, y and z must be F 4 COUNT
 * 1 (else ERASOR_E_UNSUPPORTED); intensity is taken when it is F 4 COUNT 1 and is 0 otherwise, as is a missing one.  Values are
 * copied bit for bit.  Arguments as erasor_pcd_parse_ascii: file in host or device memory, out_xyzi == NULL only asks for
 * *n = POINTS, a device out_xyzi is 16-byte aligned, the call is synchronous and info (nullable) is written on every return. */
typedef struct {
    uint32_t data_mode;              /* 0 ascii, 1 binary, 2 binary_compressed */
    uint32_t fields;                 /* bit 0 x, 1 y, 2 z, 3 intensity: which of them the cloud takes from the file */
    uint32_t intensity_zero_filled;  /* binary modes: FIELDS names intensity, but not as TYPE F SIZE 4 COUNT 1 -> 0, as PCL does */
    uint32_t point_step;             /* binary: bytes per point in the file; binary_compressed: sum of the non-"_" fields' bytes */
    uint64_t width, height, points;
    uint64_t data_offset;            /* first byte after the DATA line */
    uint64_t compressed_size, uncompressed_size, lzf_tokens;   /* binary_compressed only */
    erasor_pcd_info_t ascii;         /* the ascii branch's info, exactly as erasor_pcd_parse_ascii writes it */
} erasor_pcd_load_info_t;

int  erasor_pcd_load(erasor_pcd_t p, const char* file, size_t len, int file_kind, float* out_xyzi, size_t cap, int out_kind,
                     size_t* n, erasor_pcd_load_info_t* info);

/* ROS bag 2.0 files of erasor/node messages (DESIGN.md section 12.2; the format restated from its public description, rosbag is
 * not built here).  erasor_bag_index walks the file on the host -- every record, uncompressed chunks included -- and keeps the
 * messages on `topic` (NULL: "/node/combined/optimized") in delivery order, a stable sort by record time.  Unless keep_first, the
 * first of them is dropped, as the reference's subscribers drop it.  file: host memory, len bytes, which must stay valid and
 * unchanged until the next erasor_bag_index on p; pinned memory is read by the device directly, pageable memory through a pinned
 * staging buffer.  Errors: ERASOR_E_UNSUPPORTED for another bag version, a chunk compressed with anything but lz4 or bz2, a topic whose type
 * is not erasor/node, a cloud without FLOAT32 x, y or z; ERASOR_E_INVALID (with the byte offset) for a record or field running past
 * its container, a chunk whose data length differs from its size, a message on an undefined connection, a missing header field, a
 * message longer or shorter than an erasor/node, a point read past its cloud's data; ERASOR_E_CAPACITY for a cloud of 2^31 points.
 * A failed erasor_bag_index leaves no index: erasor_bag_nodes and erasor_bag_load then fail with ERASOR_E_STATE.
 *
 * lz4 chunks (DESIGN.md section 12.2.1): the messages of such a chunk are the entries of the index data records that follow it;
 * the chunks holding a kept node are copied to the device, decoded there (LZ4 frames of independent blocks; block and content
 * checksums verified) and their nodes parsed there.  The call then uses the device and is synchronous; the decoded chunks stay in
 * device memory held by p until the next erasor_bag_index or erasor_pcd_destroy (erasor_bag_lz4_stats: decoded_bytes); the
 * compressed copy is released before the call returns.  Further
 * errors: ERASOR_E_UNSUPPORTED for chunk data that is not an LZ4 frame, frame version other than 1, a dictionary, linked blocks, an
 * lz4 chunk no index data record follows; ERASOR_E_INVALID for a reserved bit, a block max id below 4, a header checksum, content
 * size or decoded length other than the chunk's size, a block above the block max, a malformed block (naming the chunk, the block
 * and the byte of the frame), a block or content checksum mismatch, an index entry that does not point to its message record.  A
 * bag without lz4 or bz2 chunks does no device work here.
 *
 * bz2 chunks (DESIGN.md section 12.2.2) are indexed as lz4 chunks are; each holds one bzip2 stream, decoded on the device in the
 * same submission as the lz4 chunks, into the same decoded buffer (erasor_bag_bz2_stats).  The error reported is the first in file
 * order across both kinds.  Further errors, naming the chunk and, where they apply, the block and the bit of the chunk data:
 * ERASOR_E_UNSUPPORTED for data that does not start with "BZh", a randomised block, a second stream after the first, a bz2 chunk
 * no index data record follows; ERASOR_E_INVALID for a level digit outside 1..9, a stream running past the chunk or followed by
 * other bytes, a missing block or end-of-stream magic, an empty symbol map, nGroups outside 2..6, nSelectors of 0, a selector
 * index at or above nGroups, a code length outside 1..20, an over-subscribed or incomplete code, a run or block longer than
 * level x 100 000 bytes, no end-of-block symbol, origPtr at or past the block length, four equal
 * bytes ending a block without their count, a block or stream CRC mismatch, a decoded length other than the chunk's size. */
typedef struct {
    uint32_t version;                /* 200 for V2.0 */
    uint32_t pad_;
    uint64_t chunks, connections;    /* chunk records; distinct connection ids */
    uint64_t messages, selected;     /* message records in the file (the index entries of lz4 chunks, the records walked in the
                                        others); those on the topic (before the first is dropped) */
    uint64_t unknown_records;        /* records of an op this reader does not know, skipped: only records the walk sees, so none
                                        inside lz4 chunks */
    uint64_t nodes;                  /* the nodes erasor_bag_nodes / erasor_bag_load index */
    uint64_t total_points;           /* width x height summed over the nodes */
    uint64_t intensity_zero_filled;  /* nodes whose cloud has no FLOAT32 intensity: read as 0 */
    uint64_t big_endian;             /* nodes whose cloud sets is_bigendian (ignored, as PCL ignores it) */
    char md5sum[40];                 /* the topic's connection md5sum, reported and not checked */
} erasor_bag_info_t;

/* one node's cloud as the gather reads it: point (r, c) at data_offset + r row_step + c point_step of the file -- of the chunk's
 * decoded data for a node in an lz4 chunk; bit s of fields (x y z intensity) set when that value is read from offset[s], clear
 * when it is 0 */
typedef struct {
    uint64_t data_offset, data_len;
    uint32_t width, height, point_step, row_step;
    uint32_t fields, big_endian;
    uint32_t offset[4];
} erasor_bag_cloud_t;

int  erasor_bag_index(erasor_pcd_t p, const char* file, size_t len, const char* topic, int keep_first, size_t* n_nodes,
                      erasor_bag_info_t* info);
/* nodes [first, first + count): header.seq, the record time in ns, odom (x y z qx qy qz qw, doubles as stored) and the cloud
 * layouts; every output host memory and nullable */
int  erasor_bag_nodes(erasor_pcd_t p, size_t first, size_t count, uint32_t* seq, uint64_t* stamp_ns, double* odom7,
                      erasor_bag_cloud_t* clouds);
/* The clouds of nodes [first, first + count), one gather launch: float[n][4] x y z intensity back to back into out_xyzi (host or
 * device per out_kind; a device cloud 16-byte aligned), offsets (host, count + 1) the first point of each node and the total.
 * out_xyzi == NULL only writes the offsets.  Only the selected clouds' data crosses to the device.  Exactly the input of
 * erasor_voxelize_batch and erasor_process_nodes, and node by node of erasor_updater_process_node and erasor_mapgen_accum.
 * ERASOR_E_CAPACITY: cap below the total, or 2^32 - 1 points or more.  Synchronous. */
int  erasor_bag_load(erasor_pcd_t p, size_t first, size_t count, float* out_xyzi, size_t cap, int out_kind, uint64_t* offsets);
/* the same for the listed nodes, in list order (e.g. every removal_interval-th node); ERASOR_E_INVALID for an index past the bag */
int  erasor_bag_load_list(erasor_pcd_t p, const uint64_t* nodes, size_t count, float* out_xyzi, size_t cap, int out_kind, uint64_t* offsets);

/* The lz4 chunks of the last erasor_bag_index (all 0 after a failed one, or for a bag without lz4 chunks).  Only the chunks
 * holding a kept node are uploaded and decoded; the nodes of a load in them are read from the decoded chunks (no upload). */
typedef struct {
    uint64_t chunks;                 /* lz4 chunks in the file */
    uint64_t decoded_chunks;         /* of them, those holding a kept node: copied to the device and decoded */
    uint64_t compressed_bytes;       /* their frames, copied host to device */
    uint64_t decoded_bytes;          /* their decoded data, held on the device until the next erasor_bag_index */
    uint64_t blocks, stored_blocks;  /* the blocks of the decoded chunks; of them stored (not compressed) */
    uint64_t block_checksums;        /* block checksums verified */
    uint64_t content_checksums;      /* content checksums verified */
    double decode_ms;                /* device time of the size pass, placement and block decode (CUDA events) */
    double checksum_ms;              /* device time of the checksum kernel (CUDA events) */
} erasor_bag_lz4_stats_t;

int  erasor_bag_lz4_stats(erasor_pcd_t p, erasor_bag_lz4_stats_t* stats);

/* The bz2 chunks of the last erasor_bag_index (all 0 after a failed one, or for a bag without bz2 chunks).  As for lz4, only the
 * chunks holding a kept node are uploaded and decoded, and a load reads their nodes from the decoded chunks. */
typedef struct {
    uint64_t chunks;                 /* bz2 chunks in the file */
    uint64_t decoded_chunks;         /* of them, those holding a kept node: copied to the device and decoded */
    uint64_t compressed_bytes;       /* their streams, copied host to device */
    uint64_t decoded_bytes;          /* their decoded data, held on the device until the next erasor_bag_index */
    uint64_t blocks;                 /* the true blocks of the decoded streams */
    uint64_t candidates;             /* bit offsets holding the block magic: blocks, and false positives inside blocks */
    uint64_t streams_by_level[9];    /* the bz2 chunks of the file by their stream's level 1..9 */
    uint64_t scratch_bytes;          /* the peak device scratch of the decode, released before erasor_bag_index returns */
    double scan_ms;                  /* device time of the candidate scan, the speculative walks and the chain (CUDA events) */
    double decode_ms;                /* ... of the Huffman, RUNA/RUNB and MTF decode and the LF vectors */
    double bwt_ms;                   /* ... of the inverse BWT */
    double rle_ms;                   /* ... of RLE1, the block CRCs and the placement */
} erasor_bag_bz2_stats_t;

int  erasor_bag_bz2_stats(erasor_pcd_t p, erasor_bag_bz2_stats_t* stats);

/* ============================================================================================
 * The naive map generator with its map resident on the device: the reference's mapgen (src/mapgen/mapgen.hpp:198-305,
 * accumPointCloud / getPointClouds / saveNaiveMap without the files), DESIGN.md section 8.2.  A handle of its own: one CUDA
 * device + one stream, not thread-safe; every function returns 0 or a negative error code and never throws.
 * Per node: the 2.7 m vehicle-body cut, the 1.73 m lift, the pose, voxelize_preserving_labels at 0.2 m, appended to the map --
 * one H2D copy (none for a device scan) and one kernel launch, with no host synchronisation unless a buffer has to grow.  In
 * large-scale mode the map's current chunk is voxelised at leafsize and parked at the 2nd node, then every 500 nodes (one more
 * launch).  Every call that returns data synchronises.
 * ========================================================================================== */
typedef struct erasor_mapgen_ctx* erasor_mapgen_t;

typedef struct {
    float leafsize;              /* /map/voxelsize (reference main.cpp:87, default 0.05) */
    int   is_large_scale;        /* /large_scale/is_large_scale (main.cpp:95, default false) */
} erasor_mapgen_params_t;

/* cloud ids of erasor_mapgen_get_cloud / erasor_mapgen_device_cloud */
enum { ERASOR_MAPGEN_CLOUD_MAP = 0,          /* cloud_map: the current chunk (the whole map unless large-scale) */
       ERASOR_MAPGEN_CLOUD_CURR = 1,         /* cloud_curr: the last node's voxelised scan, map frame */
       ERASOR_MAPGEN_SAVED_ORIGINAL = 2,     /* saveNaiveMap's <..>_original.pcd: the parked submaps, then cloud_map */
       ERASOR_MAPGEN_SAVED_VOXELIZED = 3 };  /* saveNaiveMap's map: SAVED_ORIGINAL voxelised at leafsize (kept until the next accum) */

/* ERASOR_E_INVALID: leafsize not positive and finite */
int  erasor_mapgen_create(const erasor_mapgen_params_t* params, int device, erasor_mapgen_t* out);
void erasor_mapgen_destroy(erasor_mapgen_t g);
const char* erasor_mapgen_last_error(erasor_mapgen_t g);   /* g may be NULL: error of the last failed erasor_mapgen_create */
/* accumPointCloud: odom7 = x y z qx qy qz qw (body -> map, double), lidar = n points x y z intensity in the lidar frame, host or
 * device (ptr_kind; ERASOR_PTR_QUERY_XYZ is ERASOR_E_INVALID: the labels ride in intensity).  A DEVICE scan is read
 * asynchronously: it must stay valid and unchanged until the next call that returns data, or until erasor_mapgen_synchronize.
 * ERASOR_E_CAPACITY: n or the map would reach 2^31 points. */
int  erasor_mapgen_accum(erasor_mapgen_t g, const double* odom7, const float* lidar_xyzi, size_t n, int ptr_kind);
/* A cloud (ids above) into out_xyzi (host or device per out_kind); out_xyzi == NULL only returns *n; cap < *n is
 * ERASOR_E_CAPACITY.  Synchronous. */
int  erasor_mapgen_get_cloud(erasor_mapgen_t g, int which, float* out_xyzi, size_t cap, int out_kind, size_t* n);
/* The same cloud in place, in the handle's device memory: no copy; valid until the next accum on this handle. */
int  erasor_mapgen_device_cloud(erasor_mapgen_t g, int which, const float** d_xyzi, size_t* n);
int  erasor_mapgen_synchronize(erasor_mapgen_t g);
/* instrumentation: kernel launches, host synchronisations and buffer regrowths (each one synchronisation) since creation */
int  erasor_mapgen_get_counters(erasor_mapgen_t g, uint64_t* launches, uint64_t* host_syncs, uint64_t* regrowths);

#ifdef __cplusplus
}
#endif
#endif /* ERASOR_B200_H */
