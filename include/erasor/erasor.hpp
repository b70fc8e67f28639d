// include/erasor/erasor.hpp -- ROS-free C++ host mirror of the reference's `class ERASOR`
// (reference include/erasor/erasor.h:43-147) on top of the C ABI in include/erasor_b200.h.
//
// Same public method names, argument meaning, call order and error behaviour (exceptions) as the
// reference, so that OfflineMapUpdater::callback_node (OfflineMapUpdater.cpp:266-284) compiles against it
// with two substitutions only:
//     pcl::PointCloud<pcl::PointXYZI>   ->  erasor_b200::PointCloud   (x, y, z, intensity; 16 bytes)
//     ERASOR(ros::NodeHandle*)          ->  ERASOR(const erasor_params_t&)   (the same /erasor/* keys)
// Everything the methods compute runs in the sm_90a kernels behind the C ABI; this header holds no
// arithmetic.  The rviz / debug publishers of the reference (erasor.h:67-77) are not mirrored.
#pragma once
#include <algorithm>
#include <array>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "../erasor_b200.h"

namespace erasor_b200 {

struct PointXYZI {          // the four floats of pcl::PointXYZI that the path uses
    float x, y, z, intensity;
};
static_assert(sizeof(PointXYZI) == 16, "PointXYZI must be one float4");
using PointCloud = std::vector<PointXYZI>;

// defaults of erasor.h:47-61 and OfflineMapUpdater.cpp:81
inline erasor_params_t default_params() {
    erasor_params_t p{};
    p.max_range = 10.0; p.num_rings = 20; p.num_sectors = 60; p.max_h = 3.0; p.min_h = 0.0; p.th_bin_max_h = 0.39;
    p.scan_ratio_threshold = 0.22; p.num_lowest_pts = 5; p.minimum_num_pts = 4; p.rejection_ratio = 0.33;
    p.gf_dist_thr = 0.05; p.gf_iter = 3; p.gf_num_lpr = 10; p.gf_th_seeds_height = 0.5; p.map_voxel_size = 0.2;
    p.version = 3; p.cov_mode = 0; p.sort_mode = 1; p.skip_voxelize = 0;
    return p;
}

class ERASOR {
public:
    // replaces ERASOR(ros::NodeHandle*): parameters are read once, R-PODs are allocated once (erasor.h:46-103)
    explicit ERASOR(const erasor_params_t& params, int device = 0) : params_(params), device_(device) {
        const int rc = erasor_create(&params_, device, &h_);
        if (rc != ERASOR_OK) throw std::runtime_error(std::string("ERASOR: ") + erasor_last_error(nullptr));
    }
    ~ERASOR() { erasor_destroy(h_); if (map_) erasor_map_destroy(map_); }
    ERASOR(const ERASOR&) = delete;
    ERASOR& operator=(const ERASOR&) = delete;

    // Inputs: transformed & cut pcs, both in the egocentric body frame (erasor.cpp:54-59)
    void set_inputs(const PointCloud& map_voi, const PointCloud& query_voi) {
        check(erasor_set_inputs(h_, reinterpret_cast<const float*>(map_voi.data()), map_voi.size(),
                                reinterpret_cast<const float*>(query_voi.data()), query_voi.size(), ERASOR_PTR_HOST));
    }
    // Version 2 algorithm (erasor.cpp:332-434)
    void compare_vois_and_revert_ground(int frame) { check(erasor_compare(h_, 2, frame)); }
    // Version 3 algorithm (erasor.cpp:438-571)
    void compare_vois_and_revert_ground_w_block(int frame) { check(erasor_compare(h_, 3, frame)); }

    void get_static_estimate(PointCloud& arranged, PointCloud& complement) {   // erasor.cpp:612-626
        size_t na = 0, nc = 0;
        check(erasor_get_output_sizes(h_, &na, &nc, nullptr, nullptr));
        arranged.resize(na); complement.resize(nc);
        check(erasor_get_static_estimate(h_, reinterpret_cast<float*>(arranged.data()), na, &na,
                                         reinterpret_cast<float*>(complement.data()), nc, &nc, ERASOR_PTR_HOST));
    }
    void get_outliers(PointCloud& map_rejected, PointCloud& curr_rejected) {   // erasor.cpp:322-327
        size_t nm = 0, nq = 0;
        check(erasor_get_output_sizes(h_, nullptr, nullptr, &nm, &nq));
        map_rejected.resize(nm); curr_rejected.resize(nq);
        check(erasor_get_outliers(h_, reinterpret_cast<float*>(map_rejected.data()), nm, &nm,
                                  reinterpret_cast<float*>(curr_rejected.data()), nq, &nq, ERASOR_PTR_HOST));
    }
    double get_max_range() { return erasor_get_max_range(h_); }               // erasor.cpp:628

    // ---- the reference's public data members (erasor.h:127, 139-145), refreshed by refresh_debug_members() ----------
    // The reference fills them as a side effect of compare_*; here they cost device -> host copies, so they are filled on
    // request: call refresh_debug_members() after compare_* (OfflineMapUpdater.cpp never reads them; rviz publishers do).
    PointCloud ground_viz;             // erasor.h:127  ground points of the flagged bins (also the tail of `arranged`)
    PointCloud debug_curr_rejected;    // erasor.h:139
    PointCloud debug_map_rejected;     // erasor.h:140
    PointCloud map_complement;         // erasor.h:141
    void refresh_debug_members() {
        size_t ng = 0;
        check(erasor_get_ground_viz(h_, nullptr, 0, &ng, ERASOR_PTR_HOST));
        ground_viz.resize(ng);
        if (ng) check(erasor_get_ground_viz(h_, reinterpret_cast<float*>(ground_viz.data()), ng, &ng, ERASOR_PTR_HOST));
        get_outliers(debug_map_rejected, debug_curr_rejected);
        PointCloud arranged_unused;
        get_static_estimate(arranged_unused, map_complement);
    }
    // r_pod_map / r_pod_curr (erasor.h:143-144) as flat tables: bin = sector * num_rings + ring.  which: ERASOR_CLOUD_MAP / _QUERY
    struct RPodTables { std::vector<int32_t> bin_of_point; std::vector<float> min_h, max_h; std::vector<uint32_t> count; };
    RPodTables r_pod(int which, size_t n_points) {
        RPodTables t;
        const size_t B = static_cast<size_t>(params_.num_rings) * params_.num_sectors;
        t.bin_of_point.resize(n_points); t.min_h.resize(B); t.max_h.resize(B); t.count.resize(B);
        check(erasor_get_bins(h_, which, t.bin_of_point.data(), t.min_h.data(), t.max_h.data(), t.count.data()));
        return t;
    }
    // ERASOR::is_dynamic_obj_close (public, erasor.h:132 / erasor.cpp:573-595) on the status of the last compare: is any of
    // the 8 neighbours of bin (r_target, theta_target) CURR_IS_HIGHER?  The theta wrap uses num_rings like the reference
    // (sic, SURVEY App. B-2); candidates that wrap out of range are skipped (the reference would index out of bounds).
    bool is_dynamic_obj_close(int r_target, int theta_target, int r_size = 1, int theta_size = 1) {
        const std::vector<float> st = get_status();
        const int R = params_.num_rings, S = params_.num_sectors;
        for (int j = theta_target - theta_size; j <= theta_target + theta_size; ++j) {
            int tj = j;
            if (j < 0) tj = j + R; else if (j >= S) tj = j - R;
            if (tj < 0 || tj >= S) continue;
            for (int r = std::max(0, r_target - r_size); r <= std::min(r_target + r_size, R - 1); ++r) {
                if (r == r_target && tj == theta_target) continue;
                if (st[static_cast<size_t>(tj) * R + r] == ERASOR_STATUS_CURR_IS_HIGHER) return true;
            }
        }
        return false;
    }

    // Frame-independent batch mode (no counterpart in the reference; BASELINE.json north_star): F independent
    // (map VoI, query VoI) pairs in one submission.  keep[f][i] == 0 where frame f rejects the i-th point of its map VoI.
    std::vector<std::vector<uint8_t>> process_frames(const std::vector<PointCloud>& map_vois, const std::vector<PointCloud>& query_vois) {
        if (map_vois.size() != query_vois.size() || map_vois.empty()) throw std::invalid_argument("ERASOR: one query VoI per map VoI");
        const size_t F = map_vois.size();
        std::vector<uint64_t> mo(F + 1, 0), qo(F + 1, 0);
        for (size_t f = 0; f < F; ++f) { mo[f + 1] = mo[f] + map_vois[f].size(); qo[f + 1] = qo[f] + query_vois[f].size(); }
        PointCloud m(mo[F]), q(qo[F]);
        for (size_t f = 0; f < F; ++f) {
            std::copy(map_vois[f].begin(), map_vois[f].end(), m.begin() + static_cast<std::ptrdiff_t>(mo[f]));
            std::copy(query_vois[f].begin(), query_vois[f].end(), q.begin() + static_cast<std::ptrdiff_t>(qo[f]));
        }
        std::vector<uint8_t> keep(mo[F] ? mo[F] : 1);
        check(erasor_process_frames(h_, reinterpret_cast<const float*>(m.data()), mo.data(), reinterpret_cast<const float*>(q.data()), qo.data(),
                                    static_cast<int>(F), keep.data(), ERASOR_PTR_HOST));
        std::vector<std::vector<uint8_t>> out(F);
        for (size_t f = 0; f < F; ++f) out[f].assign(keep.begin() + static_cast<std::ptrdiff_t>(mo[f]), keep.begin() + static_cast<std::ptrdiff_t>(mo[f + 1]));
        return out;
    }

    // ---- map-resident frame-independent mode + the single collective (north_star's multi-GPU form), C++ face ---------
    // Upload the global map once (load_global_map), then per batch only poses + body-frame queries cross PCIe.
    void load_global_map(const PointCloud& map_origin_frame) {
        if (map_) { erasor_attach_map(h_, nullptr); erasor_map_destroy(map_); map_ = nullptr; }
        int dev = 0;
        if (erasor_map_create(reinterpret_cast<const float*>(map_origin_frame.data()), map_origin_frame.size(), ERASOR_PTR_HOST, device_, &map_) != ERASOR_OK)
            throw std::runtime_error(std::string("ERASOR: ") + erasor_last_error(nullptr));
        (void)dev;
        check(erasor_attach_map(h_, map_));
    }
    // poses: x y z qx qy qz qw (body -> origin) per node; queries voxelised and in the body frame.  Returns the map's keep
    // mask after this batch (1 = static so far); it accumulates over calls (reset_static_mask() starts a job).
    std::vector<uint8_t> process_nodes(const std::vector<std::array<double, 7>>& poses, const std::vector<PointCloud>& query_vois, double voi_max_range = 0.0) {
        if (!map_) throw std::logic_error("ERASOR: load_global_map first");
        if (poses.size() != query_vois.size() || poses.empty()) throw std::invalid_argument("ERASOR: one pose per query VoI");
        const size_t F = poses.size();
        std::vector<uint64_t> qo(F + 1, 0);
        for (size_t f = 0; f < F; ++f) qo[f + 1] = qo[f] + query_vois[f].size();
        PointCloud q(qo[F]);
        for (size_t f = 0; f < F; ++f) std::copy(query_vois[f].begin(), query_vois[f].end(), q.begin() + static_cast<std::ptrdiff_t>(qo[f]));
        std::vector<uint8_t> keep(std::max<size_t>(erasor_map_size(map_), 1));
        check(erasor_process_nodes(h_, poses[0].data(), reinterpret_cast<const float*>(q.data()), qo.data(), static_cast<int>(F), voi_max_range,
                                   nullptr, keep.data(), ERASOR_PTR_HOST));
        if (inserts_) check(erasor_map_append_inserts(map_, h_));
        keep.resize(erasor_map_size(map_));
        return keep;
    }
    // Scan Ratio Test sweep (DESIGN.md section 8.5): the batch of process_nodes under every setting of `variants` (1..32) in one pass.
    // d_variant_keep: DEVICE, variants.size() x n_map bytes; mask v accumulates setting v's verdicts (reset it with
    // erasor_reset_keep_mask).  The map's own keep mask is left as it is.  Queries: host or device per ptr_kind, as erasor_process_nodes.
    void process_nodes_sweep(const std::vector<std::array<double, 7>>& poses, const float* query_xyzi, const std::vector<uint64_t>& query_offsets,
                             const std::vector<erasor_srt_variant_t>& variants, uint8_t* d_variant_keep, double voi_max_range = 0.0,
                             int ptr_kind = ERASOR_PTR_HOST) {
        if (!map_) throw std::logic_error("ERASOR: load_global_map first");
        if (poses.empty() || poses.size() + 1 != query_offsets.size()) throw std::invalid_argument("ERASOR: one pose per query VoI");
        check(erasor_process_nodes_sweep(h_, poses[0].data(), query_xyzi, query_offsets.data(), static_cast<int>(poses.size()), voi_max_range,
                                         variants.data(), static_cast<int>(variants.size()), d_variant_keep, ptr_kind));
    }
    // The same sweep over settings that also carry R-GPF's five fields (DESIGN.md section 8.6): each flagged bin is sorted by z
    // once and fitted once per distinct ground-filter tuple among the settings that flag it.
    void process_nodes_sweep(const std::vector<std::array<double, 7>>& poses, const float* query_xyzi, const std::vector<uint64_t>& query_offsets,
                             const std::vector<erasor_sweep_setting_t>& settings, uint8_t* d_variant_keep, double voi_max_range = 0.0,
                             int ptr_kind = ERASOR_PTR_HOST) {
        if (!map_) throw std::logic_error("ERASOR: load_global_map first");
        if (poses.empty() || poses.size() + 1 != query_offsets.size()) throw std::invalid_argument("ERASOR: one pose per query VoI");
        check(erasor_process_nodes_sweep_ex(h_, poses[0].data(), query_xyzi, query_offsets.data(), static_cast<int>(poses.size()), voi_max_range,
                                            settings.data(), static_cast<int>(settings.size()), d_variant_keep, ptr_kind));
    }
    // The same sweep over settings that may also differ in the polar geometry and z window (DESIGN.md section 8.7): the map is cut to
    // each node's VoI once and binned under every geometry; voi_max_range <= 0 takes the settings' common max_range.
    void process_nodes_tune(const std::vector<std::array<double, 7>>& poses, const float* query_xyzi, const std::vector<uint64_t>& query_offsets,
                            const std::vector<erasor_tune_setting_t>& settings, uint8_t* d_variant_keep, double voi_max_range = 0.0,
                            int ptr_kind = ERASOR_PTR_HOST) {
        if (!map_) throw std::logic_error("ERASOR: load_global_map first");
        if (poses.empty() || poses.size() + 1 != query_offsets.size()) throw std::invalid_argument("ERASOR: one pose per query VoI");
        check(erasor_process_nodes_tune(h_, poses[0].data(), query_xyzi, query_offsets.data(), static_cast<int>(poses.size()), voi_max_range,
                                        settings.data(), static_cast<int>(settings.size()), d_variant_keep, ptr_kind));
    }
    // Node-mode inserts (DESIGN.md section 8.4): with enable, process_nodes / process_scans also append the query points each node's
    // static estimate puts back into the map to the map's store, and save_static_map voxelises them with the kept map.
    void set_node_inserts(bool enable) { check(erasor_set_node_inserts(h_, enable ? 1 : 0)); inserts_ = enable; }
    void clear_node_inserts() { if (map_ && erasor_map_clear_inserts(map_) != ERASOR_OK) throw std::runtime_error("ERASOR: erasor_map_clear_inserts"); }
    // Node-mode re-test (DESIGN.md section 8.4.1), after a first pass with inserts on: the held map becomes its re-test map -- the
    // kept points, then every node's inserts in node order, keep all ones -- and inserts go off.  process_nodes_retest /
    // process_scans_retest then run the same nodes again, node k seeing the kept points and the inserts of the nodes before it;
    // save_static_map saves the re-test map under its keep mask.  Returns the store's node count.
    size_t begin_retest() {
        if (!map_) throw std::logic_error("ERASOR: load_global_map first");
        check(erasor_synchronize(h_));
        erasor_map_t r = nullptr;
        if (erasor_map_create_retest(map_, &r) != ERASOR_OK) throw std::runtime_error(std::string("ERASOR: ") + erasor_last_error(nullptr));
        set_node_inserts(false);
        erasor_attach_map(h_, nullptr);
        erasor_map_destroy(map_);
        map_ = r;
        check(erasor_attach_map(h_, map_));
        size_t n = 0;
        erasor_map_retest_extents(map_, &n, nullptr);
        return n;
    }
    // process_nodes for the re-test pass: node f of the batch is store node first_node + f
    std::vector<uint8_t> process_nodes_retest(const std::vector<std::array<double, 7>>& poses, const std::vector<PointCloud>& query_vois,
                                              int first_node, double voi_max_range = 0.0) {
        if (!map_) throw std::logic_error("ERASOR: load_global_map first");
        if (poses.size() != query_vois.size() || poses.empty()) throw std::invalid_argument("ERASOR: one pose per query VoI");
        const size_t F = poses.size();
        std::vector<uint64_t> qo(F + 1, 0);
        for (size_t f = 0; f < F; ++f) qo[f + 1] = qo[f] + query_vois[f].size();
        PointCloud q(qo[F]);
        for (size_t f = 0; f < F; ++f) std::copy(query_vois[f].begin(), query_vois[f].end(), q.begin() + static_cast<std::ptrdiff_t>(qo[f]));
        std::vector<uint8_t> keep(std::max<size_t>(erasor_map_size(map_), 1));
        check(erasor_process_nodes_retest(h_, poses[0].data(), reinterpret_cast<const float*>(q.data()), qo.data(), static_cast<int>(F), first_node,
                                          voi_max_range, keep.data(), ERASOR_PTR_HOST));
        keep.resize(erasor_map_size(map_));
        return keep;
    }
    // the same, from a map already in device memory (16-byte aligned float4 per point), e.g. read by PcdCodec::load_device
    void load_global_map_device(const float* d_map_xyzi, size_t n) {
        if (map_) { erasor_attach_map(h_, nullptr); erasor_map_destroy(map_); map_ = nullptr; }
        if (erasor_map_create(d_map_xyzi, n, ERASOR_PTR_DEVICE, device_, &map_) != ERASOR_OK)
            throw std::runtime_error(std::string("ERASOR: ") + erasor_last_error(nullptr));
        check(erasor_attach_map(h_, map_));
    }
    void reset_static_mask() { if (map_ && erasor_map_reset_keep(map_) != ERASOR_OK) throw std::runtime_error("ERASOR: erasor_map_reset_keep"); }
    // the map's keep mask (1 = static so far), after the work queued on this handle
    std::vector<uint8_t> static_mask() {
        if (!map_) throw std::logic_error("ERASOR: load_global_map first");
        check(erasor_synchronize(h_));
        std::vector<uint8_t> keep(std::max<size_t>(erasor_map_size(map_), 1));
        if (erasor_map_get_keep(map_, keep.data(), ERASOR_PTR_HOST) != ERASOR_OK) throw std::runtime_error("ERASOR: erasor_map_get_keep");
        keep.resize(erasor_map_size(map_));
        return keep;
    }

    // ---- voxelize_preserving_labels of many clouds in one submission (erasor_voxelize_batch) ---------------------------------
    // Voxels in the handle's device memory: cloud c is float4 points offsets[c] .. offsets[c+1] of d_xyzi, valid until the next
    // voxelize_batch / process_scans / save_static_map on this handle.
    struct DeviceClouds { const float* d_xyzi = nullptr; std::vector<uint64_t> offsets; };
    // cloud c = xyzi points raw_offsets[c] .. raw_offsets[c+1] (host or device per ptr_kind); keep (nullable, same memory kind)
    // selects points; pose7 (nullable) moves the voxels as the updater's tf_lidar2body_ does
    DeviceClouds voxelize_batch(const float* xyzi, const std::vector<uint64_t>& offsets, float leaf, const uint8_t* keep = nullptr,
                                const double* pose7 = nullptr, int ptr_kind = ERASOR_PTR_HOST) {
        if (offsets.size() < 2) throw std::invalid_argument("ERASOR: voxelize_batch needs at least one cloud");
        DeviceClouds out;
        out.offsets.assign(offsets.size(), 0);
        check(erasor_voxelize_batch(h_, xyzi, offsets.data(), static_cast<int>(offsets.size() - 1), keep, leaf, pose7, ptr_kind, &out.d_xyzi,
                                    out.offsets.data()));
        return out;
    }
    // Node mode from raw lidar scans: callback_node's query preparation (voxelize_preserving_labels at query_voxel_size, then
    // lidar -> body, OfflineMapUpdater.cpp:237-241) for every scan in one submission, then process_nodes on the device-held queries.
    // raw scans: host or device (ptr_kind).  The map's keep mask accumulates as in process_nodes (static_mask() reads it).
    void process_scans(const std::vector<std::array<double, 7>>& poses, const float* raw_xyzi, const std::vector<uint64_t>& raw_offsets,
                       double query_voxel_size, const std::array<double, 7>& lidar2body, double voi_max_range = 0.0,
                       int ptr_kind = ERASOR_PTR_HOST) {
        if (!map_) throw std::logic_error("ERASOR: load_global_map first");
        if (poses.empty() || poses.size() + 1 != raw_offsets.size()) throw std::invalid_argument("ERASOR: one pose per raw scan");
        const DeviceClouds q = voxelize_batch(raw_xyzi, raw_offsets, static_cast<float>(query_voxel_size), nullptr, lidar2body.data(), ptr_kind);
        check(erasor_process_nodes(h_, poses[0].data(), q.d_xyzi, q.offsets.data(), static_cast<int>(poses.size()), voi_max_range, nullptr, nullptr,
                                   ERASOR_PTR_DEVICE));
        if (inserts_) check(erasor_map_append_inserts(map_, h_));
    }
    std::vector<uint8_t> process_scans(const std::vector<std::array<double, 7>>& poses, const std::vector<PointCloud>& raw_scans,
                                       double query_voxel_size, const std::array<double, 7>& lidar2body, double voi_max_range = 0.0) {
        std::vector<uint64_t> off(raw_scans.size() + 1, 0);
        for (size_t f = 0; f < raw_scans.size(); ++f) off[f + 1] = off[f] + raw_scans[f].size();
        PointCloud raw(off.back());
        for (size_t f = 0; f < raw_scans.size(); ++f) std::copy(raw_scans[f].begin(), raw_scans[f].end(), raw.begin() + static_cast<std::ptrdiff_t>(off[f]));
        process_scans(poses, reinterpret_cast<const float*>(raw.data()), off, query_voxel_size, lidar2body, voi_max_range, ERASOR_PTR_HOST);
        return static_mask();
    }
    // process_scans for the re-test pass (after begin_retest): the scans are voxelised again -- the same queries as the first pass --
    // and node f of the batch is store node first_node + f
    void process_scans_retest(const std::vector<std::array<double, 7>>& poses, const float* raw_xyzi, const std::vector<uint64_t>& raw_offsets,
                              int first_node, double query_voxel_size, const std::array<double, 7>& lidar2body, double voi_max_range = 0.0,
                              int ptr_kind = ERASOR_PTR_HOST) {
        if (!map_) throw std::logic_error("ERASOR: load_global_map first");
        if (poses.empty() || poses.size() + 1 != raw_offsets.size()) throw std::invalid_argument("ERASOR: one pose per raw scan");
        const DeviceClouds q = voxelize_batch(raw_xyzi, raw_offsets, static_cast<float>(query_voxel_size), nullptr, lidar2body.data(), ptr_kind);
        check(erasor_process_nodes_retest(h_, poses[0].data(), q.d_xyzi, q.offsets.data(), static_cast<int>(poses.size()), first_node, voi_max_range,
                                          nullptr, ERASOR_PTR_DEVICE));
    }
    // save_static_map of node mode (OfflineMapUpdater.cpp:174-196 without the file): the map load_global_map holds, under its
    // current keep mask, followed by the map's insert store (empty unless inserts are on), voxelised at voxel_size -- one cloud,
    // in the handle's device memory (offsets {0, n})
    DeviceClouds save_static_map(float voxel_size) {
        if (!map_) throw std::logic_error("ERASOR: load_global_map first");
        DeviceClouds out;
        size_t n = 0;
        check(erasor_save_node_map(h_, map_, voxel_size, &out.d_xyzi, &n));
        out.offsets = {0, static_cast<uint64_t>(n)};
        return out;
    }
    // frame-sharded job: every rank processes its own nodes, then ONE all-gather (bit-packed masks over NVLink) + AND gives
    // every rank the job's static mask.  id128 from erasor_comm_unique_id() on rank 0, shipped by the host program.
    void init_communicator(const uint8_t* id128, int n_ranks, int rank) { check(erasor_comm_init(h_, id128, n_ranks, rank)); }
    std::vector<uint8_t> allgather_static_mask() {
        if (!map_) throw std::logic_error("ERASOR: load_global_map first");
        const size_t n = erasor_map_size(map_);
        check(erasor_allgather_and_keep(h_, erasor_map_keep_device(map_), n));
        check(erasor_synchronize(h_));
        std::vector<uint8_t> keep(std::max<size_t>(n, 1));
        if (erasor_map_get_keep(map_, keep.data(), ERASOR_PTR_HOST) != ERASOR_OK) throw std::runtime_error("ERASOR: erasor_map_get_keep");
        keep.resize(n);
        return keep;
    }

    // what the reference exposes as /SCDR/debug/polygons_marker likelihoods (erasor.cpp:439-441,570);
    // index = sector * num_rings + ring
    std::vector<float> get_status() {
        std::vector<float> st(static_cast<size_t>(params_.num_rings) * params_.num_sectors);
        check(erasor_get_status(h_, st.data()));
        return st;
    }
    erasor_handle_t handle() const { return h_; }
    const erasor_params_t& params() const { return params_; }

private:
    void check(int rc) const {
        if (rc == ERASOR_OK) return;
        const std::string msg = std::string("ERASOR: ") + erasor_last_error(h_);
        if (rc == ERASOR_E_INVALID) throw std::invalid_argument(msg);   // e.g. "Other version is not implemented!" (OfflineMapUpdater.cpp:274)
        throw std::runtime_error(msg);
    }
    erasor_params_t params_;
    int             device_ = 0;
    erasor_handle_t h_ = nullptr;
    erasor_map_t    map_ = nullptr;
    bool            inserts_ = false;
};

}  // namespace erasor_b200

// The reference's class lives in the global namespace (`class ERASOR`, erasor.h:43).  Define ERASOR_B200_GLOBAL_NAMES before
// including this header to get that spelling, so that OfflineMapUpdater.cpp's `unique_ptr<ERASOR> erasor_` compiles unchanged.
#ifdef ERASOR_B200_GLOBAL_NAMES
using ERASOR = erasor_b200::ERASOR;
#endif
