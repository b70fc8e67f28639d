// mapgen_capi.cu -- the naive map generator with its map resident on the device: reference src/mapgen/mapgen.hpp:198-305
// (accumPointCloud, getPointClouds, saveNaiveMap without the files), ROS stripped.  DESIGN.md section 8.2.
//
// The map is one device buffer  [parked, voxelised submaps | current chunk, raw]  whose two offsets (tail, chunk start) live in
// device memory.  A node is one cooperative launch of the chained fused kernel (updater_kernels.cu): body cut, lift, pose,
// 0.2 m voxelisation, append at the tail.  Large-scale parking is one more launch of the same kernel.  The host never needs the
// node's voxel count: it keeps an upper bound on the map's size (the last size it read back plus the points handed in since) and
// synchronises only when that bound would overflow a buffer.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <utility>

#include "../../include/erasor_b200.h"
#include "buffers.h"
#include "pose_math.h"
#include "updater_kernels.h"

using namespace erasor;

namespace {
constexpr size_t kMaxPoints = size_t(1) << 31;   // the kernels count points in 32 bits and stride over them without wrapping
constexpr int    kParkEvery = 500;               // mapgen.hpp:248
enum { W_TAIL = 0, W_CHUNK = 1, W_SEL = 2, W_CURR = 3, W_PARK = 4, W_SAVE = 5, W_COUNT = 8 };
}  // namespace

struct erasor_mapgen_ctx {
    erasor_mapgen_params_t prm{};
    int device = 0, sm_count = 132;
    cudaStream_t st = nullptr;
    std::string err;
    DeviceBuffer map;                             // float4 [cap]: parked submaps, then the current chunk
    DeviceBuffer scan, sel, part_tmp, vox_tmp, curr, vox_out, grid, words;
    PinnedBuffer h_words;                         // pinned read-back of the device words
    size_t ub_tail = 0, ub_chunk = 0;             // upper bounds on the map's size and on its current chunk's size
    size_t tail = 0, chunk = 0, n_curr = 0;       // exact values as of the last read-back
    bool fresh = false;                           // tail / chunk / n_curr describe the map as it is now
    bool idle = true;                             // nothing enqueued since the last synchronisation
    bool initial = true;                          // mapgen.hpp is_initial
    long long cnt_voxel = 0;                      // mapgen.hpp cnt_voxel (large-scale)
    uint64_t launches = 0, host_syncs = 0, regrowths = 0;
    uint64_t version = 0, saved_version = ~0ull;  // SAVED_VOXELIZED is vox_out[0 .. saved_n) while saved_version == version
    size_t saved_n = 0;
};

namespace {
thread_local std::string g_merr;
#define MCK(call) ERASOR_CUDA_TRY(g->err, call, #call)

int host_sync(erasor_mapgen_ctx* g) {
    g->host_syncs += 1;
    MCK(cudaStreamSynchronize(g->st));
    g->idle = true;
    return ERASOR_OK;
}

// the device words -> tail, chunk, n_curr (one synchronisation); the bounds become exact
int read_state(erasor_mapgen_ctx* g) {
    if (g->fresh) return ERASOR_OK;
    MCK(cudaMemcpyAsync(g->h_words.p(), g->words.p(), sizeof(uint32_t) * W_COUNT, cudaMemcpyDeviceToHost, g->st));
    int rc = host_sync(g);
    if (rc) return rc;
    const uint32_t* w = g->h_words.as<uint32_t>();
    g->tail = w[W_TAIL]; g->chunk = w[W_CHUNK]; g->n_curr = w[W_CURR];
    g->ub_tail = g->tail; g->ub_chunk = g->tail - g->chunk;
    g->fresh = true;
    return ERASOR_OK;
}

// b holds at least `bytes`: otherwise wait for the stream (work in flight may use b) unless it is idle, reallocate with headroom
// and keep the first keep_bytes.
int grow(erasor_mapgen_ctx* g, DeviceBuffer& b, size_t bytes, size_t keep_bytes = 0) {
    if (bytes <= b.cap() && b.p()) return ERASOR_OK;
    int rc = g->idle ? ERASOR_OK : host_sync(g);
    if (rc) return rc;
    const size_t want = std::max<size_t>(std::max(bytes, 2 * b.cap()), 4096);
    DeviceBuffer q;
    MCK(q.allocate(want));
    if (b.p() && keep_bytes) {
        cudaError_t e = cudaMemcpyAsync(q.p(), b.p(), keep_bytes, cudaMemcpyDeviceToDevice, g->st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(g->st);
        if (e != cudaSuccess) { g->err = std::string("regrowth copy: ") + cudaGetErrorString(e); return ERASOR_E_CUDA; }
    }
    b = std::move(q);
    g->regrowths += 1;
    return ERASOR_OK;
}

void base_job(erasor_mapgen_ctx* g, FusedJob& J) {
    Mat4 I{};
    for (int i = 0; i < 4; ++i) I.m[i * 5] = 1.0f;
    J.vin = nullptr; J.vn = 0; J.leaf = 1.0f; J.grid = g->grid.as<VoxGrid>(); J.vtmp = g->vox_tmp.p(); J.vout = nullptr; J.d_n_out = nullptr;
    J.T_out = I; J.xform_out = 0;
    J.has_part = 0; J.P = PartPred{PART_NOT_NEAR, 0, 0.0, 0.0, 0.0}; J.T_sel = I; J.xform_sel = 0; J.pin = nullptr; J.pn = 0;
    J.chunk_tmp = nullptr; J.d_total_sel = nullptr; J.out_sel = nullptr; J.out_rest = nullptr;
    J.T_sel2 = I; J.map = g->map.as<float4>(); J.d_map = g->words.as<uint32_t>();
}

// the current chunk -> voxelize_preserving_labels at leafsize -> parked in place (mapgen.hpp:249-256)
int park(erasor_mapgen_ctx* g) {
    int rc;
    if (g->ub_chunk > g->vox_out.cap() / sizeof(float4) || voxelize_tmp_bytes_upto((uint32_t)g->ub_chunk) > g->vox_tmp.cap()) {
        if ((rc = read_state(g))) return rc;             // tighten the bound before sizing scratch by it
    }
    if ((rc = grow(g, g->vox_out, sizeof(float4) * std::max<size_t>(g->ub_chunk, 1)))) return rc;
    if ((rc = grow(g, g->vox_tmp, voxelize_tmp_bytes_upto((uint32_t)g->ub_chunk)))) return rc;
    FusedJob J;
    base_job(g, J);
    J.vn = (uint32_t)g->ub_chunk; J.leaf = g->prm.leafsize; J.vout = g->vox_out.as<float4>(); J.d_n_out = g->words.as<uint32_t>() + W_PARK;
    g->launches += 1;
    MCK(launch_map_chained(g->st, J, g->sm_count));
    g->idle = false;
    g->fresh = false;                                    // a read-back above saw the map before parking
    g->ub_chunk = 0;                                    // ub_tail stays a bound: the map only shrinks
    return ERASOR_OK;
}

// SAVED_VOXELIZED: the whole map voxelised at leafsize (mapgen.hpp:296), kept until the next accum
int ensure_saved(erasor_mapgen_ctx* g) {
    int rc = read_state(g);
    if (rc) return rc;
    if (g->saved_version == g->version) return ERASOR_OK;
    if ((rc = grow(g, g->vox_out, sizeof(float4) * std::max<size_t>(g->tail, 1)))) return rc;
    if ((rc = grow(g, g->vox_tmp, voxelize_tmp_bytes((uint32_t)g->tail)))) return rc;
    FusedJob J;
    base_job(g, J);
    J.vin = g->map.as<float4>(); J.vn = (uint32_t)g->tail; J.leaf = g->prm.leafsize; J.vtmp = g->vox_tmp.p();
    J.vout = g->vox_out.as<float4>(); J.d_n_out = g->words.as<uint32_t>() + W_SAVE;
    g->launches += 1;
    MCK(launch_node_fused(g->st, J, g->sm_count));
    g->idle = false;
    MCK(cudaMemcpyAsync(g->h_words.p(), g->words.p(), sizeof(uint32_t) * W_COUNT, cudaMemcpyDeviceToHost, g->st));
    if ((rc = host_sync(g))) return rc;
    g->saved_n = g->h_words.as<uint32_t>()[W_SAVE];
    g->saved_version = g->version;
    return ERASOR_OK;
}

int locate(erasor_mapgen_ctx* g, int which, const float4** src, size_t* k) {
    if (which < 0 || which > 3) { g->err = "unknown cloud id"; return ERASOR_E_INVALID; }
    int rc = (which == 3) ? ensure_saved(g) : read_state(g);
    if (rc) return rc;
    switch (which) {
        case 0: *src = g->map.as<float4>() + g->chunk; *k = g->tail - g->chunk; break;      // CLOUD_MAP: the current chunk
        case 1: *src = g->curr.as<float4>(); *k = g->n_curr; break;                          // CLOUD_CURR
        case 2: *src = g->map.as<float4>(); *k = g->tail; break;                             // SAVED_ORIGINAL: the whole buffer
        default: *src = g->vox_out.as<float4>(); *k = g->saved_n; break;                     // SAVED_VOXELIZED
    }
    return ERASOR_OK;
}
}  // namespace

extern "C" {

const char* erasor_mapgen_last_error(erasor_mapgen_t g) { return g ? g->err.c_str() : g_merr.c_str(); }

int erasor_mapgen_create(const erasor_mapgen_params_t* prm, int device, erasor_mapgen_t* out) {
    if (!prm || !out) { g_merr = "null argument"; return ERASOR_E_INVALID; }
    *out = nullptr;
    if (!(prm->leafsize > 0.0f) || !std::isfinite(prm->leafsize)) { g_merr = "leafsize must be a positive finite number"; return ERASOR_E_INVALID; }
    erasor_mapgen_ctx* g = new erasor_mapgen_ctx();
    g->prm = *prm; g->device = device;
    auto fail = [&](const char* what, cudaError_t ce) { g_merr = std::string(what) + ": " + cudaGetErrorString(ce); erasor_mapgen_destroy(g); return ERASOR_E_CUDA; };
    cudaError_t e;
    if ((e = cudaSetDevice(device)) != cudaSuccess) return fail("cudaSetDevice", e);
    if ((e = cudaDeviceGetAttribute(&g->sm_count, cudaDevAttrMultiProcessorCount, device)) != cudaSuccess) return fail("cudaDeviceGetAttribute", e);
    if ((e = cudaStreamCreateWithFlags(&g->st, cudaStreamNonBlocking)) != cudaSuccess) return fail("cudaStreamCreate", e);
    if ((e = g->h_words.allocate(sizeof(uint32_t) * W_COUNT)) != cudaSuccess) return fail("cudaMallocHost", e);
    if ((e = g->words.allocate(sizeof(uint32_t) * W_COUNT)) != cudaSuccess) return fail("cudaMalloc", e);
    if ((e = g->grid.allocate(sizeof(VoxGrid))) != cudaSuccess) return fail("cudaMalloc", e);
    if ((e = cudaMemsetAsync(g->words.p(), 0, sizeof(uint32_t) * W_COUNT, g->st)) != cudaSuccess) return fail("cudaMemsetAsync", e);
    if ((e = cudaStreamSynchronize(g->st)) != cudaSuccess) return fail("cudaStreamSynchronize", e);
    g->fresh = true;
    *out = g;
    return ERASOR_OK;
}

void erasor_mapgen_destroy(erasor_mapgen_t g) {
    if (!g) return;
    cudaSetDevice(g->device);
    if (g->st) { cudaStreamSynchronize(g->st); cudaStreamDestroy(g->st); }
    delete g;
}

// accumPointCloud (mapgen.hpp:198-263)
int erasor_mapgen_accum(erasor_mapgen_t g, const double* odom7, const float* lidar_xyzi, size_t n, int ptr_kind) {
    if (!g) return ERASOR_E_INVALID;
    if (!odom7 || (n && !lidar_xyzi)) { g->err = "null argument"; return ERASOR_E_INVALID; }
    if (ptr_kind & ERASOR_PTR_QUERY_XYZ) { g->err = "ERASOR_PTR_QUERY_XYZ: mapgen needs the labels in intensity"; return ERASOR_E_INVALID; }
    if (ptr_kind != ERASOR_PTR_HOST && ptr_kind != ERASOR_PTR_DEVICE) { g->err = "unknown ptr_kind"; return ERASOR_E_INVALID; }
    if (n >= kMaxPoints) { g->err = "scan of 2^31 points or more"; return ERASOR_E_CAPACITY; }
    MCK(cudaSetDevice(g->device));
    int rc;
    // room for the worst case: every point survives the cut and is its own voxel.  When the bound would overflow the map buffer,
    // one synchronisation reads the true size back and the buffer doubles (at least), so the next one is as far away again.
    const size_t map_cap = g->map.cap() / sizeof(float4);
    if (g->ub_tail + n > map_cap) {
        if ((rc = read_state(g))) return rc;
        if (g->tail + n >= kMaxPoints) { g->err = "the map would reach 2^31 points"; return ERASOR_E_CAPACITY; }
        const size_t want = std::max(std::max(g->tail + n, 2 * map_cap), size_t(1) << 16);
        if ((rc = grow(g, g->map, sizeof(float4) * want, sizeof(float4) * g->tail))) return rc;
    }
    const size_t n1 = std::max<size_t>(n, 1);
    if ((rc = grow(g, g->sel, sizeof(float4) * n1)) || (rc = grow(g, g->curr, sizeof(float4) * n1)) ||
        (rc = grow(g, g->part_tmp, sizeof(uint32_t) * partition_tmp_words((uint32_t)n))) ||
        (rc = grow(g, g->vox_tmp, voxelize_tmp_bytes_upto((uint32_t)n))))
        return rc;
    const float4* d_scan = reinterpret_cast<const float4*>(lidar_xyzi);
    if (ptr_kind == ERASOR_PTR_HOST) {
        if ((rc = grow(g, g->scan, sizeof(float4) * n1))) return rc;
        if (n) MCK(cudaMemcpyAsync(g->scan.p(), lidar_xyzi, sizeof(float4) * n, cudaMemcpyHostToDevice, g->st));
        g->idle = false;
        d_scan = g->scan.as<float4>();
    }
    FusedJob J;
    base_job(g, J);
    const float max_dist_square = (float)std::pow(2.7, 2);                    // `float max_dist_square = pow(CAR_BODY_SIZE, 2)` (:219)
    J.has_part = 1; J.P = PartPred{PART_NOT_NEAR, 0, 0.0, 0.0, (double)max_dist_square};
    J.T_sel.m[11] = 1.73f; J.xform_sel = 1;                                    // tf_lidar2origin (:209-214, :231-232)
    pose_to_mat(odom7, J.T_sel2);                                              // geoPose2eigen (:234, :236-237)
    J.pin = d_scan; J.pn = (uint32_t)n; J.chunk_tmp = g->part_tmp.as<uint32_t>();
    J.d_total_sel = g->words.as<uint32_t>() + W_SEL; J.out_sel = g->sel.as<float4>();
    J.vn = (uint32_t)n; J.leaf = 0.2f;                                         // :239 (fixed 0.2)
    J.vtmp = g->vox_tmp.p(); J.vout = g->curr.as<float4>(); J.d_n_out = g->words.as<uint32_t>() + W_CURR;
    g->launches += 1;
    MCK(launch_map_chained(g->st, J, g->sm_count));
    g->idle = false;
    g->ub_tail += n; g->ub_chunk += n;
    g->fresh = false;
    g->version += 1;
    if (g->initial) { g->initial = false; return ERASOR_OK; }                  // cloud_map = cloud_curr (:241-243)
    if (g->prm.is_large_scale && (g->cnt_voxel++ % kParkEvery) == 0) return park(g);
    return ERASOR_OK;
}

int erasor_mapgen_get_cloud(erasor_mapgen_t g, int which, float* out_xyzi, size_t cap, int out_kind, size_t* n) {
    if (!g) return ERASOR_E_INVALID;
    if (!n) { g->err = "null argument"; return ERASOR_E_INVALID; }
    if (out_kind != ERASOR_PTR_HOST && out_kind != ERASOR_PTR_DEVICE) { g->err = "unknown ptr_kind"; return ERASOR_E_INVALID; }
    MCK(cudaSetDevice(g->device));
    const float4* src = nullptr;
    size_t k = 0;
    int rc = locate(g, which, &src, &k);
    if (rc) return rc;
    *n = k;
    if (!out_xyzi) return ERASOR_OK;
    if (cap < k) { g->err = "output buffer too small"; return ERASOR_E_CAPACITY; }
    if (k) MCK(cudaMemcpyAsync(out_xyzi, src, sizeof(float4) * k, out_kind == ERASOR_PTR_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, g->st));
    g->idle = false;
    return host_sync(g);
}

int erasor_mapgen_device_cloud(erasor_mapgen_t g, int which, const float** d_xyzi, size_t* n) {
    if (!g) return ERASOR_E_INVALID;
    if (!d_xyzi || !n) { g->err = "null argument"; return ERASOR_E_INVALID; }
    MCK(cudaSetDevice(g->device));
    const float4* src = nullptr;
    size_t k = 0;
    int rc = locate(g, which, &src, &k);
    if (rc) return rc;
    *d_xyzi = reinterpret_cast<const float*>(src); *n = k;
    return ERASOR_OK;
}

int erasor_mapgen_synchronize(erasor_mapgen_t g) {
    if (!g) return ERASOR_E_INVALID;
    MCK(cudaSetDevice(g->device));
    return host_sync(g);
}

int erasor_mapgen_get_counters(erasor_mapgen_t g, uint64_t* launches, uint64_t* host_syncs, uint64_t* regrowths) {
    if (!g) return ERASOR_E_INVALID;
    if (launches) *launches = g->launches;
    if (host_syncs) *host_syncs = g->host_syncs;
    if (regrowths) *regrowths = g->regrowths;
    return ERASOR_OK;
}

}  // extern "C"
