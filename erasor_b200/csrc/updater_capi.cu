// updater_capi.cu -- device-resident mirror of erasor::OfflineMapUpdater (reference
// src/offline_map_updater/src/OfflineMapUpdater.cpp:203-449, 174-196), ROS stripped: SURVEY.md section 8f rows 1-3.
// The global map stays in HBM between nodes; per node only the raw scan and a pose cross PCIe.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/erasor_b200.h"
#include "buffers.h"
#include "pose_math.h"
#include "updater_kernels.h"

using namespace erasor;

struct erasor_updater_ctx {
    erasor_updater_params_t up{};
    erasor_params_t ep{};
    erasor_handle_t er = nullptr;
    int device = 0;
    cudaStream_t st = nullptr;
    std::string err;
    Mat4 tf_lidar2body{}, tf_body2origin{};
    // maps (origin frame), double-buffered
    DeviceBuffer map_a, map_b;        size_t n_map = 0;
    DeviceBuffer global_a;            size_t n_global = 0;      // large-scale: map_arranged_global_
    DeviceBuffer complement;          size_t n_complement = 0;  // large-scale: map_arranged_complement_
    DeviceBuffer scan, qvox, voi, outskirts, tmp_rej, part_tmp, vox_tmp, grid, counters, save_out;
    size_t n_query = 0, n_voi = 0, n_out = 0, n_rej = 0;
    bool submap_uninit = true;
    double submap_cx = 0, submap_cy = 0;
    size_t num_pcs_init = 0;
    int stack_count = 0;
    uint64_t launches = 0;
    // look-ahead (erasor_updater_prefetch_scan): scans of coming nodes are uploaded and voxelised on a second stream while the current
    // node's path runs.  Two slots, so that the caller can hand in node k + 1's scan before it calls process_node for node k.
    struct Lookahead {
        DeviceBuffer scan, qvox, vox_tmp, grid, counters;
        PinnedBuffer h_words;
        cudaEvent_t ev = nullptr;
        const float* ptr = nullptr; size_t n = 0; int kind = 0; bool valid = false; uint64_t ticket = 0;
    };
    cudaStream_t st2 = nullptr;
    Lookahead la[2];
    uint64_t la_ticket = 0;
    PinnedBuffer h_words;                            // pinned read-back of the two device counters (a copy into pageable memory would
                                                     // block until the stream has drained and then some)
    int sm_count = 132;
    uint64_t map_version = 0;                       // bumped whenever the map changes (processed node, reset)
    uint64_t save_version = ~0ull; float save_leaf = 0.0f; size_t save_n = 0;   // what save_out currently holds
};

namespace {
thread_local std::string g_uerr;
#define UCK(call) ERASOR_CUDA_TRY(u->err, call, #call)
#define ECK(call) do { int rc__ = (call); if (rc__ != ERASOR_OK) { u->err = std::string(#call) + ": " + erasor_last_error(u->er); return rc__; } } while (0)

// counters[0] = points selected by the partition, counters[1] = voxels: both read back with one synchronisation
int read_counters(erasor_updater_ctx* u, size_t* n_sel, size_t* n_vox) {
    UCK(cudaMemcpyAsync(u->h_words.p(), u->counters.p(), 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, u->st));
    UCK(cudaStreamSynchronize(u->st));
    if (n_sel) *n_sel = u->h_words.as<uint32_t>()[0];
    if (n_vox) *n_vox = u->h_words.as<uint32_t>()[1];
    return ERASOR_OK;
}

void no_partition(FusedJob& J) {
    J.has_part = 0; J.P = PartPred{PART_RADIUS, 0, 0.0, 0.0, 0.0}; J.T_sel = Mat4{}; J.xform_sel = 0; J.pin = nullptr; J.pn = 0;
    J.chunk_tmp = nullptr; J.d_total_sel = nullptr; J.out_sel = nullptr; J.out_rest = nullptr;
}
void no_voxelize(erasor_updater_ctx* u, FusedJob& J) {
    J.vin = nullptr; J.vn = 0; J.leaf = 1.0f; J.grid = u->grid.as<VoxGrid>(); J.vtmp = u->vox_tmp.p(); J.vout = nullptr;
    J.d_n_out = u->counters.as<uint32_t>() + 1; J.T_out = Mat4{}; J.xform_out = 0;
}
// U1 job: stable partition of src[0..n) into sel / rest (both in order)
int add_partition(erasor_updater_ctx* u, FusedJob& J, const PartPred& P, const Mat4& T, bool xform, const float4* src, size_t n, DeviceBuffer& sel, DeviceBuffer& rest) {
    UCK(sel.ensure(sizeof(float4) * std::max<size_t>(n, 1)));
    UCK(rest.ensure(sizeof(float4) * std::max<size_t>(n, 1)));
    UCK(u->part_tmp.ensure(sizeof(uint32_t) * partition_tmp_words((uint32_t)n)));
    J.has_part = 1; J.P = P; J.T_sel = T; J.xform_sel = xform ? 1 : 0; J.pin = src; J.pn = (uint32_t)n;
    J.chunk_tmp = u->part_tmp.as<uint32_t>(); J.d_total_sel = u->counters.as<uint32_t>(); J.out_sel = sel.as<float4>(); J.out_rest = rest.as<float4>();
    return ERASOR_OK;
}
// U3 job: voxelize_preserving_labels of src[0..n) at `leaf` into out, optionally followed by the affine T_out
int add_voxelize(erasor_updater_ctx* u, FusedJob& J, const float4* src, size_t n, float leaf, DeviceBuffer& out, const Mat4* T_out) {
    UCK(out.ensure(sizeof(float4) * std::max<size_t>(n, 1)));
    UCK(u->vox_tmp.ensure(voxelize_tmp_bytes((uint32_t)n)));
    J.vin = src; J.vn = (uint32_t)n; J.leaf = leaf; J.grid = u->grid.as<VoxGrid>(); J.vtmp = u->vox_tmp.p(); J.vout = out.as<float4>();
    J.d_n_out = u->counters.as<uint32_t>() + 1; J.T_out = T_out ? *T_out : Mat4{}; J.xform_out = T_out ? 1 : 0;
    return ERASOR_OK;
}
int launch_fused(erasor_updater_ctx* u, const FusedJob& J, int max_ctas = 0) {
    u->launches += 1;
    UCK(launch_node_fused(u->st, J, u->sm_count, max_ctas));
    return ERASOR_OK;
}

// stable partition of src[0..n) into sel / rest (both in order); returns the number selected
int partition(erasor_updater_ctx* u, const PartPred& P, const Mat4& T, bool xform, const float4* src, size_t n, DeviceBuffer& sel, DeviceBuffer& rest, size_t* n_sel) {
    FusedJob J;
    no_voxelize(u, J);
    int rc = add_partition(u, J, P, T, xform, src, n, sel, rest);
    if (rc || (rc = launch_fused(u, J))) return rc;
    return read_counters(u, n_sel, nullptr);
}

int voxelize(erasor_updater_ctx* u, const float4* src, size_t n, float leaf, DeviceBuffer& out, size_t* n_out) {
    FusedJob J;
    no_partition(J);
    int rc = add_voxelize(u, J, src, n, leaf, out, nullptr);
    if (rc || (rc = launch_fused(u, J))) return rc;
    return read_counters(u, nullptr, n_out);
}

// set_submap + bookkeeping of reassign_submap (OfflineMapUpdater.cpp:332-379)
int reassign_submap(erasor_updater_ctx* u, double px, double py) {
    auto split = [&]() -> int {
        PartPred P{PART_SUBMAP, 0, px, py, u->up.submap_size};
        Mat4 I{};
        size_t nsel = 0;
        int rc = partition(u, P, I, false, u->global_a.as<float4>(), u->n_global, u->map_a, u->complement, &nsel);
        if (rc) return rc;
        u->n_map = nsel; u->n_complement = u->n_global - nsel;
        u->submap_cx = px; u->submap_cy = py;
        return ERASOR_OK;
    };
    if (u->submap_uninit) {
        int rc = split();
        if (rc) return rc;
        u->submap_uninit = false;
        return ERASOR_OK;
    }
    const double dx = std::abs(u->submap_cx - px), dy = std::abs(u->submap_cy - py), half = u->up.submap_size / 2.0;
    if (dx > half || dy > half) {
        // map_arranged_global_ = map_arranged_ + map_arranged_complement_
        const size_t n = u->n_map + u->n_complement;
        UCK(u->global_a.ensure(sizeof(float4) * std::max<size_t>(n, 1)));
        if (u->n_map) UCK(cudaMemcpyAsync(u->global_a.p(), u->map_a.p(), sizeof(float4) * u->n_map, cudaMemcpyDeviceToDevice, u->st));
        if (u->n_complement) UCK(cudaMemcpyAsync(u->global_a.as<float4>() + u->n_map, u->complement.p(), sizeof(float4) * u->n_complement, cudaMemcpyDeviceToDevice, u->st));
        u->n_global = n;
        return split();
    }
    return ERASOR_OK;
}

// map_arranged_: in large-scale mode, until the first processed node splits the window off, the whole initial map
// (load_global_map copies it to both map_arranged_ and map_arranged_global_; the complement is still empty)
const DeviceBuffer& arranged(const erasor_updater_ctx* u, size_t* n) {
    const bool whole = u->up.is_large_scale && u->submap_uninit;
    *n = whole ? u->n_global : u->n_map;
    return whole ? u->global_a : u->map_a;
}
}  // namespace

extern "C" {

const char* erasor_updater_last_error(erasor_updater_t u) { return u ? u->err.c_str() : g_uerr.c_str(); }

int erasor_updater_create(const erasor_updater_params_t* up, const erasor_params_t* ep, const float* initial_map_xyzi, size_t n_map,
                          int device, erasor_updater_t* out) {
    if (!up || !ep || !out || (n_map && !initial_map_xyzi)) { g_uerr = "null argument"; return ERASOR_E_INVALID; }
    *out = nullptr;
    if (up->removal_interval < 1) { g_uerr = "removal_interval must be >= 1"; return ERASOR_E_INVALID; }
    erasor_updater_ctx* u = new erasor_updater_ctx();
    u->up = *up; u->ep = *ep; u->device = device;
    erasor_params_t e2 = *ep;
    e2.version = up->version;                              // /erasor/version is read by the updater (OfflineMapUpdater.cpp:81)
    int rc = erasor_create(&e2, device, &u->er);
    if (rc != ERASOR_OK) { g_uerr = erasor_last_error(nullptr); delete u; return rc; }
    u->st = (cudaStream_t)erasor_stream(u->er);
    auto fail = [&](const char* what, cudaError_t ce) { g_uerr = std::string(what) + ": " + cudaGetErrorString(ce); erasor_updater_destroy(u); return ERASOR_E_CUDA; };
    cudaError_t e;
    if ((e = u->counters.allocate(64)) != cudaSuccess) return fail("cudaMalloc", e);
    if ((e = u->h_words.allocate(64)) != cudaSuccess) return fail("cudaMallocHost", e);
    if ((e = cudaStreamCreateWithFlags(&u->st2, cudaStreamNonBlocking)) != cudaSuccess) return fail("cudaStreamCreate", e);
    for (auto& la : u->la) {
        if ((e = la.h_words.allocate(64)) != cudaSuccess) return fail("cudaMallocHost", e);
        if ((e = cudaEventCreateWithFlags(&la.ev, cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", e);
        if ((e = la.counters.allocate(64)) != cudaSuccess) return fail("cudaMalloc", e);
        if ((e = la.grid.ensure(sizeof(VoxGrid))) != cudaSuccess) return fail("cudaMalloc", e);
    }
    if ((e = cudaDeviceGetAttribute(&u->sm_count, cudaDevAttrMultiProcessorCount, device)) != cudaSuccess) return fail("cudaDeviceGetAttribute", e);
    if ((e = u->grid.ensure(sizeof(VoxGrid))) != cudaSuccess) return fail("cudaMalloc", e);
    // set_params (OfflineMapUpdater.cpp:89-104): tf_lidar2body_ = geoPose2eigen(pose) * Identity
    Mat4 G, I{};
    for (int i = 0; i < 4; ++i) I.m[i * 5] = 1.0f;
    pose_to_mat(up->lidar2body, G);
    mat_mul(G, I, u->tf_lidar2body);
    u->tf_body2origin = I;
    // load_global_map (OfflineMapUpdater.cpp:107-167), outdoor
    u->num_pcs_init = n_map;
    DeviceBuffer& dst = up->is_large_scale ? u->global_a : u->map_a;
    if ((e = dst.ensure(sizeof(float4) * std::max<size_t>(n_map, 1))) != cudaSuccess) return fail("cudaMalloc", e);
    if (n_map && (e = cudaMemcpy(dst.p(), initial_map_xyzi, sizeof(float4) * n_map, cudaMemcpyHostToDevice)) != cudaSuccess) return fail("cudaMemcpy", e);
    if (up->is_large_scale) { u->n_global = n_map; u->n_map = 0; } else { u->n_map = n_map; }
    *out = u;
    return ERASOR_OK;
}

void erasor_updater_destroy(erasor_updater_t u) {
    if (!u) return;
    cudaSetDevice(u->device);
    if (u->st) cudaStreamSynchronize(u->st);
    if (u->st2) { cudaStreamSynchronize(u->st2); cudaStreamDestroy(u->st2); }
    for (auto& la : u->la)
        if (la.ev) cudaEventDestroy(la.ev);
    if (u->er) erasor_destroy(u->er);
    delete u;
}

// re-arm the updater with a (new) initial map, keeping every device buffer: load_global_map again (OfflineMapUpdater.cpp:107-167)
int erasor_updater_reset(erasor_updater_t u, const float* initial_map_xyzi, size_t n_map) {
    if (!u || (n_map && !initial_map_xyzi)) { if (u) u->err = "null argument"; return ERASOR_E_INVALID; }
    UCK(cudaSetDevice(u->device));
    UCK(cudaStreamSynchronize(u->st));
    UCK(cudaStreamSynchronize(u->st2));
    for (auto& la : u->la) la.valid = false;
    DeviceBuffer& dst = u->up.is_large_scale ? u->global_a : u->map_a;
    UCK(dst.ensure(sizeof(float4) * std::max<size_t>(n_map, 1)));
    if (n_map) UCK(cudaMemcpyAsync(dst.p(), initial_map_xyzi, sizeof(float4) * n_map, cudaMemcpyHostToDevice, u->st));
    UCK(cudaStreamSynchronize(u->st));
    u->num_pcs_init = n_map;
    u->n_map = u->up.is_large_scale ? 0 : n_map;
    u->n_global = u->up.is_large_scale ? n_map : 0;
    u->n_complement = 0; u->n_query = u->n_voi = u->n_out = u->n_rej = 0;
    u->submap_uninit = true; u->stack_count = 0;
    u->map_version++;
    ECK(erasor_forget_run_history(u->er));            // a re-armed pass launches what the first pass did
    return ERASOR_OK;
}

erasor_handle_t erasor_updater_erasor(erasor_updater_t u) { return u ? u->er : nullptr; }

// OfflineMapUpdater::callback_node (OfflineMapUpdater.cpp:203-330)
int erasor_updater_process_node(erasor_updater_t u, int seq, const double* odom7, const float* lidar_xyzi, size_t n_lidar, int ptr_kind, int* processed) {
    if (!u || !odom7 || (n_lidar && !lidar_xyzi)) { if (u) u->err = "null argument"; return ERASOR_E_INVALID; }
    if (processed) *processed = 0;
    u->stack_count++;
    if (u->stack_count % u->up.removal_interval != 0) return ERASOR_OK;                      // "PASS!" (:328)
    UCK(cudaSetDevice(u->device));
    pose_to_mat(odom7, u->tf_body2origin);                                                    // :219
    // 1. query: voxelize_preserving_labels, lidar -> body (:237-241)
    erasor_updater_ctx::Lookahead* la = nullptr;
    for (auto& c : u->la) if (c.valid && c.ptr == lidar_xyzi && c.n == n_lidar && c.kind == ptr_kind && (!la || c.ticket < la->ticket)) la = &c;
    const bool prefetched = la != nullptr;
    const float4* d_scan = reinterpret_cast<const float4*>(lidar_xyzi);
    if (!prefetched && ptr_kind != ERASOR_PTR_DEVICE) {
        UCK(u->scan.ensure(sizeof(float4) * std::max<size_t>(n_lidar, 1)));
        if (n_lidar) UCK(cudaMemcpyAsync(u->scan.p(), lidar_xyzi, sizeof(float4) * n_lidar, cudaMemcpyHostToDevice, u->st));
        d_scan = u->scan.as<float4>();
    }
    // 1 + 2 in ONE cooperative launch: the scan's voxelisation + lidar -> body (:237-241) and, independent of it, the map's
    //        VoI cut + origin -> body (fetch_VoI, :246-254, :381-438)
    int rc;
    const double x_curr = u->tf_body2origin.m[3], y_curr = u->tf_body2origin.m[7];
    if (u->up.is_large_scale && (rc = reassign_submap(u, x_curr, y_curr))) return rc;
    Mat4 Tinv;
    mat_inv(u->tf_body2origin, Tinv);
    PartPred P{PART_RADIUS, 0, x_curr, y_curr, std::pow(u->up.max_range + 0.0, 2)};
    if (prefetched) {
        // the scan was voxelised ahead of time on the second stream (erasor_updater_prefetch_scan): only the map's VoI cut is left
        FusedJob J;
        no_voxelize(u, J);
        if ((rc = add_partition(u, J, P, Tinv, true, u->map_a.as<float4>(), u->n_map, u->voi, u->outskirts))) return rc;
        // (a cooperative grid must be resident as a whole: leave the quarter of the SMs a look-ahead for the next node may be holding)
        if ((rc = launch_fused(u, J, u->sm_count - std::max(1, u->sm_count / 4)))) return rc;
        UCK(cudaEventSynchronize(la->ev));                      // the look-ahead's counters are in its pinned words
        if ((rc = read_counters(u, &u->n_voi, nullptr))) return rc;
        u->n_query = la->h_words.as<uint32_t>()[1];
        std::swap(u->qvox, la->qvox);
        la->valid = false;
    } else {
        FusedJob J;
        if ((rc = add_voxelize(u, J, d_scan, n_lidar, (float)u->up.query_voxel_size, u->qvox, &u->tf_lidar2body))) return rc;
        if ((rc = add_partition(u, J, P, Tinv, true, u->map_a.as<float4>(), u->n_map, u->voi, u->outskirts))) return rc;
        if ((rc = launch_fused(u, J))) return rc;
        if ((rc = read_counters(u, &u->n_voi, &u->n_query))) return rc;
    }
    u->n_out = u->n_map - u->n_voi;
    // 3. the path (:266-275)
    if (u->up.version != 2 && u->up.version != 3) { u->err = "Other version is not implemented!"; return ERASOR_E_INVALID; }
    ECK(erasor_set_inputs(u->er, u->voi.as<float>(), u->n_voi, u->qvox.as<float>(), u->n_query, ERASOR_PTR_DEVICE));
    ECK(erasor_compare(u->er, u->up.version, seq));
    size_t n_arr = 0, n_cmp = 0, n_rej = 0, n_crej = 0;
    ECK(erasor_get_output_sizes(u->er, &n_arr, &n_cmp, &n_rej, &n_crej));
    const float* d_arr = nullptr; const float* d_cmp = nullptr; const float* d_rej = nullptr;
    ECK(erasor_device_outputs(u->er, &d_arr, &d_cmp, &d_rej, nullptr));
    // 4. map_filtered = static + complement, body -> origin, + outskirts; map_rejected body -> origin (:281-290): one launch,
    //    straight from the handle's output buffers (stream-ordered: the next node's set_inputs runs behind it)
    const size_t n_new = n_arr + n_cmp + u->n_out;
    UCK(u->map_b.ensure(sizeof(float4) * std::max<size_t>(n_new, 1)));
    UCK(u->tmp_rej.ensure(sizeof(float4) * std::max<size_t>(n_rej, 1)));
    const CopySeg segs[4] = {
        {reinterpret_cast<const float4*>(d_arr), u->map_b.as<float4>(), (uint32_t)n_arr, 1},
        {reinterpret_cast<const float4*>(d_cmp), u->map_b.as<float4>() + n_arr, (uint32_t)n_cmp, 1},
        {u->outskirts.as<float4>(), u->map_b.as<float4>() + n_arr + n_cmp, (uint32_t)u->n_out, 0},
        {reinterpret_cast<const float4*>(d_rej), u->tmp_rej.as<float4>(), (uint32_t)n_rej, 1}};
    u->launches += 1;
    UCK(launch_copy_segments(u->st, u->tf_body2origin, segs, 4));
    u->n_rej = n_rej;
    std::swap(u->map_a, u->map_b);
    u->n_map = n_new;
    u->map_version++;
    if (processed) *processed = 1;
    return ERASOR_OK;
}

// Look-ahead for callers that know the coming nodes' scans (file-based / offline runs): upload + voxelize_preserving_labels
// + lidar -> body of a scan on a second stream, on a quarter of the SMs, while the current node's path runs.  Two slots.
int erasor_updater_prefetch_scan(erasor_updater_t u, const float* lidar_xyzi, size_t n_lidar, int ptr_kind) {
    if (!u || (n_lidar && !lidar_xyzi)) { if (u) u->err = "null argument"; return ERASOR_E_INVALID; }
    UCK(cudaSetDevice(u->device));
    // a free slot, else the older of the two (its look-ahead is dropped)
    erasor_updater_ctx::Lookahead* la = !u->la[0].valid ? &u->la[0] : (!u->la[1].valid ? &u->la[1] : (u->la[0].ticket < u->la[1].ticket ? &u->la[0] : &u->la[1]));
    if (la->valid) { UCK(cudaEventSynchronize(la->ev)); la->valid = false; }
    const float4* d_scan = reinterpret_cast<const float4*>(lidar_xyzi);
    if (ptr_kind != ERASOR_PTR_DEVICE) {
        UCK(la->scan.ensure(sizeof(float4) * std::max<size_t>(n_lidar, 1)));
        if (n_lidar) UCK(cudaMemcpyAsync(la->scan.p(), lidar_xyzi, sizeof(float4) * n_lidar, cudaMemcpyHostToDevice, u->st2));
        d_scan = la->scan.as<float4>();
    }
    UCK(la->qvox.ensure(sizeof(float4) * std::max<size_t>(n_lidar, 1)));
    UCK(la->vox_tmp.ensure(voxelize_tmp_bytes((uint32_t)n_lidar)));
    FusedJob J;
    no_partition(J);
    J.vin = d_scan; J.vn = (uint32_t)n_lidar; J.leaf = (float)u->up.query_voxel_size; J.grid = la->grid.as<VoxGrid>(); J.vtmp = la->vox_tmp.p();
    J.vout = la->qvox.as<float4>(); J.d_n_out = la->counters.as<uint32_t>() + 1; J.T_out = u->tf_lidar2body; J.xform_out = 1;
    u->launches += 1;
    UCK(launch_node_fused(u->st2, J, u->sm_count, std::max(1, u->sm_count / 4)));
    UCK(cudaMemcpyAsync(la->h_words.p(), la->counters.p(), 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, u->st2));
    UCK(cudaEventRecord(la->ev, u->st2));
    la->ptr = lidar_xyzi; la->n = n_lidar; la->kind = ptr_kind; la->valid = true; la->ticket = ++u->la_ticket;
    return ERASOR_OK;
}

int erasor_updater_map_size(erasor_updater_t u, size_t* n) {
    if (!u || !n) return ERASOR_E_INVALID;
    arranged(u, n);
    return ERASOR_OK;
}

// which: 0 map_arranged_, 1 map_voi_ (body frame), 2 query_voi_ (body frame), 5 map_rejected_ (origin frame), 7 map_outskirts_,
//        8 map_arranged_complement_ (large-scale)
int erasor_updater_get_cloud(erasor_updater_t u, int which, float* xyzi, size_t cap, size_t* n, int ptr_kind) {
    if (!u || !n) return ERASOR_E_INVALID;
    const void* src = nullptr; size_t k = 0;
    switch (which) {
        case 0: src = arranged(u, &k).p(); break;
        case 1: src = u->voi.p(); k = u->n_voi; break;
        case 2: src = u->qvox.p(); k = u->n_query; break;
        case 5: src = u->tmp_rej.p(); k = u->n_rej; break;
        case 7: src = u->outskirts.p(); k = u->n_out; break;
        case 8: src = u->complement.p(); k = u->n_complement; break;
        default: u->err = "unknown cloud id"; return ERASOR_E_INVALID;
    }
    *n = k;
    if (!xyzi) return ERASOR_OK;
    if (cap < k) { u->err = "output buffer too small"; return ERASOR_E_CAPACITY; }
    UCK(cudaSetDevice(u->device));
    if (k) UCK(cudaMemcpyAsync(xyzi, src, sizeof(float4) * k, ptr_kind == ERASOR_PTR_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, u->st));
    UCK(cudaStreamSynchronize(u->st));
    return ERASOR_OK;
}

// OfflineMapUpdater::save_static_map minus the file write (OfflineMapUpdater.cpp:174-196)
int erasor_updater_save_static_map(erasor_updater_t u, float voxel_size, float* out_xyzi, size_t cap, size_t* n) {
    if (!u || !n) return ERASOR_E_INVALID;
    UCK(cudaSetDevice(u->device));
    size_t ns = 0;
    const float4* src = arranged(u, &ns).as<float4>();
    if (u->up.is_large_scale && !u->submap_uninit) {
        // *ptr_src = *map_arranged_ + *map_arranged_complement_
        UCK(u->map_b.ensure(sizeof(float4) * std::max<size_t>(u->n_map + u->n_complement, 1)));
        if (u->n_map) UCK(cudaMemcpyAsync(u->map_b.p(), u->map_a.p(), sizeof(float4) * u->n_map, cudaMemcpyDeviceToDevice, u->st));
        if (u->n_complement) UCK(cudaMemcpyAsync(u->map_b.as<float4>() + u->n_map, u->complement.p(), sizeof(float4) * u->n_complement, cudaMemcpyDeviceToDevice, u->st));
        src = u->map_b.as<float4>(); ns = u->n_map + u->n_complement;
    }
    // the usual call pattern is size query (out == NULL) followed by the fetch: the second call reuses the first one's result
    // instead of voxelising the whole map again
    size_t k = u->save_n;
    if (!(u->save_version == u->map_version && u->save_leaf == voxel_size)) {
        int rc = voxelize(u, src, ns, voxel_size, u->save_out, &k);
        if (rc) return rc;
        u->save_version = u->map_version; u->save_leaf = voxel_size; u->save_n = k;
    }
    *n = k;
    if (!out_xyzi) return ERASOR_OK;
    if (cap < k) { u->err = "output buffer too small"; return ERASOR_E_CAPACITY; }
    if (k) UCK(cudaMemcpyAsync(out_xyzi, u->save_out.p(), sizeof(float4) * k, cudaMemcpyDeviceToHost, u->st));
    UCK(cudaStreamSynchronize(u->st));
    return ERASOR_OK;
}

// voxelize_preserving_labels on a free-standing host cloud (unit-test entry for U3)
int erasor_updater_voxelize(erasor_updater_t u, const float* xyzi, size_t n_in, float leaf, float* out_xyzi, size_t cap, size_t* n) {
    if (!u || !n || (n_in && !xyzi)) return ERASOR_E_INVALID;
    UCK(cudaSetDevice(u->device));
    UCK(u->scan.ensure(sizeof(float4) * std::max<size_t>(n_in, 1)));
    if (n_in) UCK(cudaMemcpyAsync(u->scan.p(), xyzi, sizeof(float4) * n_in, cudaMemcpyHostToDevice, u->st));
    size_t k = 0;
    u->save_version = ~0ull;                         // save_out is about to hold something else
    int rc = voxelize(u, u->scan.as<float4>(), n_in, leaf, u->save_out, &k);
    if (rc) return rc;
    *n = k;
    if (!out_xyzi) return ERASOR_OK;
    if (cap < k) { u->err = "output buffer too small"; return ERASOR_E_CAPACITY; }
    if (k) UCK(cudaMemcpyAsync(out_xyzi, u->save_out.p(), sizeof(float4) * k, cudaMemcpyDeviceToHost, u->st));
    UCK(cudaStreamSynchronize(u->st));
    return ERASOR_OK;
}

// mapgen's per-node producer on the device (reference src/mapgen/mapgen.hpp:198-239, accumPointCloud up to cloud_curr):
// drop the points within CAR_BODY_SIZE = 2.7 m of the sensor, lift by 1.73 m, move to the map frame with the node's pose,
// voxelize_preserving_labels at 0.2 m.  The map bookkeeping around it (concatenation, large-scale parking) stays with the caller.
int erasor_updater_mapgen_node(erasor_updater_t u, const double* odom7, const float* lidar_xyzi, size_t n_lidar, int ptr_kind,
                               float* out_xyzi, size_t cap, size_t* n) {
    if (!u || !odom7 || !n || (n_lidar && !lidar_xyzi)) { if (u) u->err = "null argument"; return ERASOR_E_INVALID; }
    UCK(cudaSetDevice(u->device));
    const float4* d_scan = reinterpret_cast<const float4*>(lidar_xyzi);
    if (ptr_kind != ERASOR_PTR_DEVICE) {
        UCK(u->scan.ensure(sizeof(float4) * std::max<size_t>(n_lidar, 1)));
        if (n_lidar) UCK(cudaMemcpyAsync(u->scan.p(), lidar_xyzi, sizeof(float4) * n_lidar, cudaMemcpyHostToDevice, u->st));
        d_scan = u->scan.as<float4>();
    }
    const float max_dist_square = (float)std::pow(2.7, 2);                    // `float max_dist_square = pow(CAR_BODY_SIZE, 2)` (:219)
    PartPred P{PART_NOT_NEAR, 0, 0.0, 0.0, (double)max_dist_square};
    Mat4 I{};
    for (int i = 0; i < 4; ++i) I.m[i * 5] = 1.0f;
    size_t n_keep = 0;
    int rc = partition(u, P, I, false, d_scan, n_lidar, u->voi, u->outskirts, &n_keep);
    if (rc) return rc;
    Mat4 lift = I, pose;
    lift.m[11] = 1.73f;                                                        // tf_lidar2origin (:209-214)
    pose_to_mat(odom7, pose);                                                  // :234
    u->launches += 2;
    UCK(launch_affine_copy(u->st, lift, true, u->voi.as<float4>(), u->voi.as<float4>(), (uint32_t)n_keep));   // :231-232
    UCK(launch_affine_copy(u->st, pose, true, u->voi.as<float4>(), u->voi.as<float4>(), (uint32_t)n_keep));   // :236-237
    size_t k = 0;
    u->save_version = ~0ull;
    if ((rc = voxelize(u, u->voi.as<float4>(), n_keep, 0.2f, u->save_out, &k))) return rc;                    // :239 (fixed 0.2)
    *n = k;
    if (!out_xyzi) return ERASOR_OK;
    if (cap < k) { u->err = "output buffer too small"; return ERASOR_E_CAPACITY; }
    if (k) UCK(cudaMemcpyAsync(out_xyzi, u->save_out.p(), sizeof(float4) * k, ptr_kind == ERASOR_PTR_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, u->st));
    UCK(cudaStreamSynchronize(u->st));
    return ERASOR_OK;
}

int erasor_updater_get_fused_profile(erasor_updater_t u, uint64_t* ns16) {
    if (!u || !ns16) return ERASOR_E_INVALID;
    UCK(cudaSetDevice(u->device));
    UCK(cudaStreamSynchronize(u->st));
    VoxGrid g;
    UCK(cudaMemcpy(&g, u->grid.p(), sizeof(VoxGrid), cudaMemcpyDeviceToHost));
    for (int i = 0; i < 16; ++i) ns16[i] = g.prof[i];
    return ERASOR_OK;
}

uint64_t erasor_updater_kernel_launch_count(erasor_updater_t u) { return u ? u->launches + erasor_kernel_launch_count(u->er) : 0; }

}  // extern "C"
