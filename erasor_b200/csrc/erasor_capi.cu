// erasor_capi.cu -- the extern "C" boundary (include/erasor_b200.h): context, HBM buffers, launch order.
// There is no host compute path in this file: every entry point either launches the sm_90a kernels of
// kernels.cu or fails with an error code.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>      // types only: the library is loaded with dlopen on first use (erasor_comm_*)

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <memory>
#include <string>
#include <vector>

#include "../../include/erasor_b200.h"
#include "binning_tables.h"
#include "buffers.h"
#include "device_types.h"
#include "kernels.h"
#include "pose_math.h"
#include "voxelize_batch.h"

using namespace erasor;

namespace {

thread_local std::string g_create_error;

constexpr int kNumTimers = 6;   // 0 whole pipeline, 1..5 = K1..K5
constexpr size_t kMaxRecords = (size_t)1 << 21;   // flagged-bin records of one submission (larger batches are split)

struct Timer {
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending;
    double   total_ms = 0;
    uint64_t launches = 0;
};

}  // namespace

struct erasor_map_ctx {
    int          device = 0;
    DeviceBuffer d_pts, d_keep;                // float4 [n + kMapPad], uint8 [max(n, 1)]
    size_t       n = 0;
    DeviceBuffer d_ins;                        // node-mode inserts appended by the callers (erasor_map_append_inserts), float4 [n_ins]
    size_t       n_ins = 0;
    std::vector<uint64_t> ins_node_off{0};     // the store offset of every appended node, in append order, then n_ins
    bool         retest = false;               // made by erasor_map_create_retest ...
    std::vector<uint64_t> extents;             // ... and then node k of its source's store sees the prefix [0, extents[k])
    cudaStream_t st = nullptr;
    std::string  err;
};

namespace {

// One submission of a mask mode, as enqueue() runs it: everything its copies and launches read besides the handle's buffers and
// chunk descriptors (whose changes alloc_epoch and desc_epoch track).  The caller fills in the first part, submit() the rest.  A
// captured graph replays the step it was captured from, so the graph cache is keyed on it; erasor_wait's class-C fix-up and
// erasor_profile_k1 read the last one.
struct SweepPlan;

struct Step {
    int           mode = 1;                   // 1: batch of (map_voi, query_voi) pairs, 2: nodes against the resident map
    int           ptr_kind = ERASOR_PTR_HOST; // of the caller's buffers: HOST or DEVICE
    bool          qry_xyz = false;            // the query cloud is packed x y z (ERASOR_PTR_QUERY_XYZ)
    int           f0 = 0;                     // first frame of the sub-batch within the caller's batch (per-frame counters)
    const float*  map_xyzi = nullptr;         // mode 1
    const float*  qry_xyzi = nullptr;
    uint8_t*      user_keep = nullptr;        // mode 1: one byte per VoI point; mode 2: frame_keep [F][n_map] (nullable)
    uint8_t*      keep_out = nullptr;         // mode 2: receives the map's mask (nullable)
    K4Fold        fold{nullptr, nullptr, 0u, 0u};   // mode 1: onto the caller's global mask (mode 2: submit() sets the map's)
    std::shared_ptr<const SweepPlan> sweep;   // mode 2: the sweep of erasor_process_nodes_sweep / _sweep_ex / _tune (null: none)
    // set by submit()
    bool          inserts = false;            // node-mode inserts
    bool          with_c = true;              // R-GPF class C launched up front
    const float4* cur_map = nullptr;          // what K1 reads: the caller's device clouds, their staging buffers or the resident map
    const float4* cur_qry = nullptr;
    uint8_t*      d_keep = nullptr;           // where R-GPF writes user_keep (itself, or staging for a host mask) ...
    size_t        n_keep = 0;                 // ... and its bytes (0: none)
    const erasor_map_ctx* map = nullptr;      // mode 2
    size_t        n_map_global = 0;           // mode 2: map points
};

// A geometry's polar tables, built by build_bin_tables and kept by the handle: its own geometry's by erasor_create, a sweep
// geometry's on first use
struct GeoTables {
    erasor_geometry_t key{};
    HostBinTables     host;
    DeviceBuffer      d_ring, d_pos, d_neg, d_guard;   // written once
    BinTablesView     view{};
    int               B = 0;
};

// A sweep's submission (erasor_process_nodes_sweep / _sweep_ex / _tune, DESIGN.md sections 8.5-8.7): its distinct geometries in
// order of first appearance (geo[0] carries setting 0), each with the Scan Ratio Test fields of every setting -- those of the
// other geometries switched off (minimum_num_pts -1) -- and the ground-filter groups of its own settings.  An own plan's one
// geometry is the handle's: K1 bins into the handle's per-batch tables, as in a plain call.  Any other plan bins geometry g into
// the handle's k1_sweep[g], in the K1 launches of launch_begin (geometries [launch_begin[l], launch_begin[l + 1])).
struct SweepGeo {
    const GeoTables* t;
    int              launch;                   // the K1 launch that bins it (not own)
    SrtSweep         ssw;
    K4Sweep          ksw;
};
struct SweepPlan {
    bool                  own = false;
    int                   B_max = 0;
    std::vector<SweepGeo> geo;
    std::vector<int>      launch_begin;        // not own: K1 launches + 1 entries
    std::vector<size_t>   launch_smem;         // ... and each launch's shared memory
};

bool same_plan(const SweepPlan* a, const SweepPlan* b) {
    if (!a || !b) return a == b;
    if (a->geo.size() != b->geo.size() || a->launch_begin != b->launch_begin) return false;
    for (size_t g = 0; g < a->geo.size(); ++g) {
        const SrtSweep &as = a->geo[g].ssw, &bs = b->geo[g].ssw;
        const K4Sweep &ak = a->geo[g].ksw, &bk = b->geo[g].ksw;
        if (a->geo[g].t != b->geo[g].t || a->geo[g].launch != b->geo[g].launch || as.n != bs.n || as.n_flagged != bs.n_flagged ||
            std::memcmp(as.v, bs.v, sizeof(SrtVariant) * (size_t)as.n) != 0 || ak.keep != bk.keep || ak.rejected != bk.rejected ||
            ak.n != bk.n || ak.n_groups != bk.n_groups || std::memcmp(ak.bits, bk.bits, sizeof(uint32_t) * (size_t)ak.n_groups) != 0 ||
            std::memcmp(ak.gp, bk.gp, sizeof(GpfParams) * (size_t)ak.n_groups) != 0)
            return false;
    }
    return true;
}

bool same_step(const Step& a, const Step& b) {
    return a.mode == b.mode && a.ptr_kind == b.ptr_kind && a.qry_xyz == b.qry_xyz && a.inserts == b.inserts && a.with_c == b.with_c &&
           a.f0 == b.f0 && a.map_xyzi == b.map_xyzi && a.qry_xyzi == b.qry_xyzi && a.cur_map == b.cur_map && a.cur_qry == b.cur_qry &&
           a.user_keep == b.user_keep && a.d_keep == b.d_keep && a.n_keep == b.n_keep && a.keep_out == b.keep_out &&
           a.n_map_global == b.n_map_global && a.map == b.map &&
           a.fold.keep == b.fold.keep && a.fold.index == b.fold.index && a.fold.n == b.fold.n && same_plan(a.sweep.get(), b.sweep.get());
}

}  // namespace

struct NcclApi {
    void* lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    const char*  (*GetErrorString)(ncclResult_t) = nullptr;
};

struct erasor_ctx {
    erasor_params_t p{};
    int             device = 0;
    cudaStream_t    stream = nullptr, stream_a = nullptr, stream_b = nullptr, stream_c = nullptr;   // a/b/c: concurrent R-GPF size classes (high priority)
    cudaEvent_t     ev_fork = nullptr, ev_join_a = nullptr, ev_join_b = nullptr, ev_join_c = nullptr;
    int             sm_count = 132;
    std::string     err;
    // Captured graphs hold raw device pointers: every (re)allocation of a device buffer of this handle bumps alloc_epoch, which
    // retires them.  HBuf cannot be built without the epoch, so a buffer added here cannot forget it.
    uint64_t        alloc_epoch = 0;
    struct HBuf : DeviceBuffer { explicit HBuf(uint64_t& e) : DeviceBuffer(&e) {} };
    int             B = 0;                     // bins of the handle's geometry (its polar tables: geo_tables[0])
    // one geometry's K1 outputs, the arrays of its K1GeoTables (sized by ensure_k1_bufs, read through k1_tables)
    struct K1Bufs { HBuf bin_map, bin_qry, ch_cnt, zmin, zmax, cnt; explicit K1Bufs(uint64_t& e) : bin_map(e), bin_qry(e), ch_cnt(e), zmin(e), zmax(e), cnt(e) {} };

    // per-batch buffers
    HBuf d_map_in{alloc_epoch}, d_qry_in{alloc_epoch};       // staging when the caller's clouds are host memory
    K1Bufs k1_own{alloc_epoch};                              // the handle's geometry
    HBuf d_chunks{alloc_epoch}, d_chunk_range{alloc_epoch}, d_frame_off{alloc_epoch};
    HBuf d_dst_start{alloc_epoch}, d_status{alloc_epoch}, d_action{alloc_epoch}, d_flag_slot{alloc_epoch}, d_nflag{alloc_epoch};
    HBuf d_recs{alloc_epoch}, d_nrecs{alloc_epoch}, d_frame_rej{alloc_epoch}, d_frame_rec_base{alloc_epoch}, d_queue{alloc_epoch}, d_bucket{alloc_epoch};
    HBuf d_map_sorted{alloc_epoch}, d_map_src{alloc_epoch}, d_qry_sorted{alloc_epoch}, d_qry_src{alloc_epoch}, d_part{alloc_epoch}, d_scratch{alloc_epoch};
    HBuf d_keep{alloc_epoch}, d_ground{alloc_epoch};
    HBuf d_arranged{alloc_epoch}, d_map_rej{alloc_epoch}, d_curr_rej{alloc_epoch}, d_jobs{alloc_epoch}, d_out_sizes{alloc_epoch}, d_k5tmp{alloc_epoch};
    HBuf d_vox{alloc_epoch}, d_vox_cnt{alloc_epoch}, d_vox_start{alloc_epoch}, d_vox_scratch{alloc_epoch};
    HBuf d_fence{alloc_epoch};                 // 4 x u64: negzero, empty fits, ambiguous, slow-path points
    HBuf d_poses{alloc_epoch};                 // node mode: NodePose per frame
    HBuf d_list_idx{alloc_epoch}, d_list_cnt{alloc_epoch};   // node mode: per chunk, the map index of every VoI point (dense, map order) and their number
    HBuf d_k1prof{alloc_epoch};                // erasor_profile_k1: per-warp cycle counters of K1's profiling build
    HBuf d_pack{alloc_epoch}, d_gather{alloc_epoch};         // exchange step: packed keep bits of this rank / of every rank
    HBuf d_sweep_flag{alloc_epoch}, d_sweep_rej{alloc_epoch};  // sweeps: flagged bins per (plan geometry, frame, variant) [G][stat_F][32] /
                                                               // rejected points per (frame, variant) [stat_F][32]
    PinnedBuffer h_stage, h_pose, h_words;     // h_words: small device -> host read-backs of a submission (pinned: an asynchronous copy into
                                               // pageable memory blocks the launching thread until the whole stream has drained, which
                                               // serialised overlapped handles)

    // batch geometry of the last run
    int      F = 0;
    size_t   NM = 0, NQ = 0;                   // points of the map-side arrays (node mode: F * n_map) / of the queries
    uint32_t n_chunks_map = 0, n_chunks_qry = 0;
    uint32_t rec_capacity = 0;
    const float4* cur_map = nullptr;           // K1's inputs: erasor_set_inputs's, or the last step's
    const float4* cur_qry = nullptr;
    uint32_t* k1_prof = nullptr;               // set only inside erasor_profile_k1: run_k1 launches K1's profiling build
    std::vector<uint64_t> map_off, qry_off;
    int      desc_mode = -1;                   // mode the uploaded chunk descriptors were built for (-1: none; 0 cloud, 1 batch masks, 2 node masks)
    uint64_t desc_epoch = 0;                   // bumped whenever the descriptors are rebuilt (invalidates cached graphs)
    int      stat_F = 0;                       // frames of the last batch call (all its sub-batches): extent of the per-frame counters
    int      f0 = 0;                           // first frame of the sub-batch being submitted
    std::vector<uint32_t> node_nvoi;           // node mode: |map_voi_| of the frames before f0 (the count tables hold the last sub-batch only)
    struct StepGraph { Step step; uint64_t desc_epoch, alloc_epoch; cudaGraphExec_t exec; uint64_t kernel_nodes; };
    std::vector<StepGraph> graphs;             // captured mask-mode steps (same_step, and the epochs they were captured at)
    bool     use_graphs = true;
    int      ctas_per_sm = 4;                  // K1 / K2 grid target: one wave of sm_count * ctas_per_sm CTAs (ERASOR_B200_CTAS_PER_SM)
    bool     fused_srt = true;                 // mask modes: Scan Ratio Test inside the scatter kernel (ERASOR_B200_UNFUSED_SRT=1: separate k3_srt)
    bool     pending = false;                  // an asynchronous submission has not been waited for yet
    // R-GPF class C (bins beyond 2560 points) is launched only while such bins are being seen (its CTAs need whole SMs even to
    // find their queue empty, which serialises overlapped submissions); if one turns up unannounced, erasor_wait runs the class.
    int      class_c_state = -1;               // -1 unknown (launch it), 0 none in the last run, > 0 seen
    uint32_t class_c_count_host = 0;           // queue[kBucketC0] of the submission in flight
    Step     last;                             // the last mask-mode submission
    int      sweep_V = 0;                      // variants of the last node call when it was a sweep (erasor_get_sweep_stats), else 0

    // the polar tables of every geometry seen, the handle's own first; per geometry of a sweep plan that is not own its K1 outputs
    std::vector<std::unique_ptr<GeoTables>> geo_tables;
    std::vector<std::unique_ptr<K1Bufs>> k1_sweep;
    HBuf     d_list_idx32{alloc_epoch}, d_list_cnt32{alloc_epoch};   // the VoI lists of a plan's 32-warp K1 launches (k1_lists)
    size_t   smem_optin = 0;                   // sharedMemPerBlockOptin of the device
    bool     tune_unpacked = false;            // ERASOR_B200_TUNE_UNPACKED=1: one geometry per K1 launch (measurement of the packing)

    // node mode
    erasor_map_ctx* map = nullptr;
    // node-mode inserts (erasor_set_node_inserts, DESIGN.md section 8.4): per submission the query scatter plan, the assembled
    // inserts of its frames and their offsets; per call (all its sub-batches) the inserts in frame order
    bool node_inserts = false;
    HBuf d_ins{alloc_epoch}, d_ins_fwd{alloc_epoch}, d_ins_slot{alloc_epoch}, d_ins_n{alloc_epoch}, d_ins_bin_off{alloc_epoch},
         d_ins_frame_cnt{alloc_epoch}, d_ins_off{alloc_epoch};
    PinnedBuffer h_ins_fwd, h_ins_off;         // body -> origin rows [F][12] / offsets [F+1] of the submission
    DeviceBuffer d_ins_call;                   // the last call's inserts (never in a captured graph)
    std::vector<uint64_t> ins_call_off;        // its offsets: F + 1 entries once the call has completed
    DeviceBuffer d_save, d_save_keep;          // erasor_save_node_map: map ++ inserts and its keep bytes

    // erasor_voxelize_batch: its scratch and output cloud (created on first use)
    erasor::VoxBatch* vb = nullptr;

    // exchange
    ncclComm_t comm = nullptr;
    int        comm_ranks = 1, comm_rank = 0;

    // single-frame state machine
    int      stage = 0;                        // 0: nothing, 1: inputs set, 2: compared
    uint32_t out_sizes[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // arranged, complement, map_rejected, curr_rejected, ground_viz
    uint32_t complement_start = 0;
    uint32_t n_recs_host = 0;                  // (cloud mode; the mask modes read back into h_words)
    volatile uint32_t* words() { return h_words.as<volatile uint32_t>(); }   // [0] flagged-bin records, [1] class-C bins of the submission in flight

    uint64_t launches = 0;
    bool     timing = false;
    Timer    timers[kNumTimers];
};

namespace {

#define CK(call) ERASOR_CUDA_TRY(h->err, call, #call)

// NCCL is bound at run time: single-GPU users need no libnccl, and inside a torch process dlopen returns the copy torch
// already loaded (same soname), so the process keeps exactly one NCCL.
NcclApi* nccl_api(std::string& err) {
    static NcclApi api;
    static bool tried = false;
    if (api.lib) return &api;
    if (tried) { err = "libnccl.so.2 could not be loaded"; return nullptr; }
    tried = true;
    void* lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) { err = std::string("dlopen(libnccl.so.2): ") + dlerror(); return nullptr; }
    api.GetUniqueId    = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(lib, "ncclGetUniqueId"));
    api.CommInitRank   = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(lib, "ncclCommInitRank"));
    api.CommDestroy    = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(lib, "ncclCommDestroy"));
    api.AllGather      = reinterpret_cast<decltype(api.AllGather)>(dlsym(lib, "ncclAllGather"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(lib, "ncclGetErrorString"));
    if (!api.GetUniqueId || !api.CommInitRank || !api.CommDestroy || !api.AllGather || !api.GetErrorString) { err = "libnccl.so.2 lacks a required symbol"; return nullptr; }
    api.lib = lib;
    return &api;
}

struct Scope {   // optional CUDA-event bracket around a kernel (timing == true only)
    erasor_ctx* h; int id; cudaEvent_t a = nullptr, b = nullptr;
    Scope(erasor_ctx* h_, int id_) : h(h_), id(id_) {
        if (h->timing) { cudaEventCreate(&a); cudaEventCreate(&b); cudaEventRecord(a, h->stream); }
    }
    ~Scope() {
        if (h->timing) { cudaEventRecord(b, h->stream); h->timers[id].pending.emplace_back(a, b); }
    }
};

void drain_timers(erasor_ctx* h) {
    for (int i = 0; i < kNumTimers; ++i) {
        for (auto& pr : h->timers[i].pending) {
            cudaEventSynchronize(pr.second);
            float ms = 0;
            cudaEventElapsedTime(&ms, pr.first, pr.second);
            h->timers[i].total_ms += ms;
            h->timers[i].launches += 1;
            cudaEventDestroy(pr.first); cudaEventDestroy(pr.second);
        }
        h->timers[i].pending.clear();
    }
}

uint32_t choose_chunk(const erasor_ctx* h, const uint64_t* map_off, const uint64_t* qry_off, int F) {
    // Chunk = one CTA of K1 and of K2.  Aim at ONE wave of CTAs (4 resident per SM for both kernels): a second, nearly empty
    // wave costs a whole CTA latency.  Frames are chunked separately, so the count is taken over the real frame sizes.
    // The dense per-chunk count rows cost 4*(B+1) bytes each: keep the chunk at >= 5*B points (<= 5 % extra traffic).
    const size_t total = (size_t)(map_off[F] + qry_off[F]);
    const size_t slots = (size_t)h->sm_count * (k1_warps(k1_smem_bytes(h->p.num_rings, h->B)) == 32 ? 1 : h->ctas_per_sm);
    auto count = [&](size_t ch) {
        size_t n = 0;
        for (int f = 0; f < F; ++f) n += (size_t)((map_off[f + 1] - map_off[f] + ch - 1) / ch) + (size_t)((qry_off[f + 1] - qry_off[f] + ch - 1) / ch);
        return n;
    };
    const size_t cap = 65536;
    size_t ch = std::max<size_t>(total / slots + 1, std::max<size_t>(2048, (size_t)5 * h->B));
    ch = std::min<size_t>((ch + 127) & ~(size_t)127, cap);
    if (count(cap) <= slots) {
        while (ch < cap && count(ch) > slots) ch = std::min<size_t>(cap, (ch + std::max<size_t>(128, ch / 64) + 127) & ~(size_t)127);
    } else {
        ch = cap;      // several waves anyway
    }
    return (uint32_t)ch;
}

// k's room for K1's outputs over NM map and NQ query points, n_chunks chunks and F frames of B bins (the bin ids with kIdPad of
// slack: K2 prefetches ids past a chunk's end unchecked)
int ensure_k1_bufs(erasor_ctx* h, erasor_ctx::K1Bufs& k, size_t NM, size_t NQ, size_t n_chunks, size_t F, size_t B) {
    CK(k.bin_map.ensure(sizeof(uint16_t) * (NM + kIdPad)));
    CK(k.bin_qry.ensure(sizeof(uint16_t) * (NQ + kIdPad)));
    CK(k.ch_cnt.ensure(sizeof(uint32_t) * std::max<size_t>(n_chunks, 1) * (B + 1)));
    CK(k.zmin.ensure(sizeof(uint32_t) * 2 * F * B));
    CK(k.zmax.ensure(sizeof(uint32_t) * 2 * F * B));
    CK(k.cnt.ensure(sizeof(uint32_t) * 2 * F * (B + 1)));
    return ERASOR_OK;
}

// Build chunk descriptors + per-frame chunk ranges + frame offsets, upload them, size every buffer.
// mode 0: single frame, cloud outputs; 1: batch of (map_voi, query_voi) pairs, masks; 2: node mode -- frame f scans the prefix
// [0, map_off[f+1] - map_off[f]) of the resident map (fetch_VoI fused into K1): the whole map ({0, n_map, 2 n_map, ...}) or a
// re-test node's extent; masks on global indices.
int prepare_batch(erasor_ctx* h, const uint64_t* map_off, const uint64_t* qry_off, int F, int mode) {
    if (F <= 0) { h->err = "n_frames must be positive"; return ERASOR_E_INVALID; }
    const size_t NM = map_off[F], NQ = qry_off[F];
    if (NM >= 0xFFFFFFF0ull || NQ >= 0xFFFFFFF0ull) { h->err = "batch exceeds 2^32 points; split it"; return ERASOR_E_INVALID; }
    for (int f = 0; f < F; ++f)
        if (map_off[f + 1] < map_off[f] || qry_off[f + 1] < qry_off[f]) { h->err = "offsets must be non-decreasing"; return ERASOR_E_INVALID; }
    const int B = h->B;
    // per-frame counters span the caller's whole batch (all its sub-batches), so they are sized before the shortcut below
    CK(h->d_nflag.ensure(sizeof(uint32_t) * (size_t)std::max(h->stat_F, h->f0 + F)));
    CK(h->d_frame_rej.ensure(sizeof(uint32_t) * (size_t)std::max(h->stat_F, h->f0 + F)));
    // same batch geometry as the previous call (the usual case when a caller streams equally-shaped batches):
    // the chunk descriptors already on the device are still valid -- skip rebuild, upload and the staging sync
    if (h->desc_mode == mode && h->F == F && h->map_off.size() == (size_t)F + 1 && h->qry_off.size() == (size_t)F + 1 &&
        std::equal(map_off, map_off + F + 1, h->map_off.begin()) && std::equal(qry_off, qry_off + F + 1, h->qry_off.begin()))
        return ERASOR_OK;
    h->desc_mode = -1;
    h->F = F; h->NM = NM; h->NQ = NQ;
    h->map_off.assign(map_off, map_off + F + 1);
    h->qry_off.assign(qry_off, qry_off + F + 1);
    const uint32_t CH = choose_chunk(h, map_off, qry_off, F);
    const bool node = mode == 2;

    std::vector<ChunkDesc> chunks;
    std::vector<uint32_t>  range(2 * (size_t)(F + 1)), foff(2 * (size_t)(F + 1));
    chunks.reserve((NM + NQ) / CH + 2 * (size_t)F + 2);
    for (int c = 0; c < 2; ++c) {
        const uint64_t* off = c == 0 ? map_off : qry_off;
        for (int f = 0; f < F; ++f) {
            range[(size_t)c * (F + 1) + f] = (uint32_t)chunks.size();
            foff[(size_t)c * (F + 1) + f]  = (uint32_t)off[f];
            for (uint64_t b = off[f]; b < off[f + 1]; b += CH) {
                ChunkDesc d{};
                d.len = (uint32_t)std::min<uint64_t>(CH, off[f + 1] - b);
                d.frame = (uint32_t)f; d.cloud = (uint32_t)c;
                d.bin_begin = (uint32_t)b; d.out_base = (uint32_t)off[f];
                if (node && c == 0) { d.begin = (uint32_t)(b - off[f]); d.frame_begin = 0u; }      // source = the resident map itself
                else                { d.begin = (uint32_t)b; d.frame_begin = (uint32_t)off[f]; }
                chunks.push_back(d);
            }
        }
        range[(size_t)c * (F + 1) + F] = (uint32_t)chunks.size();
        foff[(size_t)c * (F + 1) + F]  = (uint32_t)off[F];
        if (c == 0) h->n_chunks_map = (uint32_t)chunks.size();
    }
    h->n_chunks_qry = (uint32_t)chunks.size() - h->n_chunks_map;
    const size_t n_chunks = chunks.size();

    // device buffers
    CK(h->d_chunks.ensure(sizeof(ChunkDesc) * std::max<size_t>(n_chunks, 1)));
    CK(h->d_chunk_range.ensure(sizeof(uint32_t) * range.size()));
    CK(h->d_frame_off.ensure(sizeof(uint32_t) * foff.size()));
    if (const int rc = ensure_k1_bufs(h, h->k1_own, NM, NQ, n_chunks, (size_t)F, (size_t)B)) return rc;
    CK(h->d_map_sorted.ensure(sizeof(float4) * std::max<size_t>(NM, 1)));
    CK(h->d_dst_start.ensure(sizeof(uint32_t) * 2 * (size_t)F * (B + 2)));
    CK(h->d_status.ensure((size_t)F * B));
    CK(h->d_action.ensure((size_t)F * B));
    CK(h->d_flag_slot.ensure(sizeof(uint32_t) * (size_t)F * B));
    CK(h->d_frame_rec_base.ensure(sizeof(uint32_t) * (size_t)F));
    h->rec_capacity = (uint32_t)std::min<size_t>((size_t)F * B, kMaxRecords);
    CK(h->d_recs.ensure(sizeof(FlagRec) * (size_t)h->rec_capacity));
    CK(h->d_nrecs.ensure(sizeof(uint32_t) * 4));
    CK(h->d_queue.ensure(sizeof(uint32_t) * kQueueWords));
    CK(h->d_bucket.ensure(sizeof(uint32_t) * (size_t)kNumBuckets * h->rec_capacity));
    CK(h->d_map_src.ensure(sizeof(uint32_t) * std::max<size_t>(NM, 1)));
    CK(h->d_scratch.ensure((size_t)24 * std::max<size_t>(NM, 1) + 64));
    if (node) {
        CK(h->d_poses.ensure(sizeof(NodePose) * (size_t)F));
        CK(h->d_list_idx.ensure(sizeof(uint32_t) * (NM + kIdPad)));
        CK(h->d_list_cnt.ensure(sizeof(uint32_t) * kListWarps * std::max<size_t>(n_chunks, 1)));
    }
    if (mode == 0) {
        CK(h->d_qry_sorted.ensure(sizeof(float4) * std::max<size_t>(NQ, 1)));
        CK(h->d_qry_src.ensure(sizeof(uint32_t) * std::max<size_t>(NQ, 1)));
        CK(h->d_part.ensure(sizeof(float4) * std::max<size_t>(NM, 1)));
    }

    // upload descriptors through pinned staging
    const size_t b0 = sizeof(ChunkDesc) * n_chunks, b1 = sizeof(uint32_t) * range.size(), b2 = sizeof(uint32_t) * foff.size();
    CK(cudaStreamSynchronize(h->stream));   // staging may still be in flight from the previous call
    CK(h->h_stage.ensure(b0 + b1 + b2 + 64));
    unsigned char* st = h->h_stage.as<unsigned char>();
    if (b0) std::memcpy(st, chunks.data(), b0);
    std::memcpy(st + b0, range.data(), b1);
    std::memcpy(st + b0 + b1, foff.data(), b2);
    if (b0) CK(cudaMemcpyAsync(h->d_chunks.p(), st, b0, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_chunk_range.p(), st + b0, b1, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->d_frame_off.p(), st + b0 + b1, b2, cudaMemcpyHostToDevice, h->stream));
    h->desc_mode = mode;
    h->desc_epoch++;
    return ERASOR_OK;
}

// one caller cloud -> the device pointer the kernels read: the cloud itself (device memory) or its staging buffer (host memory,
// copied in by stage_host_clouds)
int device_cloud(erasor_ctx* h, DeviceBuffer& stage, const float* xyzi, size_t n, int ptr_kind, const float4** out, size_t bytes_per_point = sizeof(float4)) {
    if (ptr_kind == ERASOR_PTR_DEVICE) {
        const uintptr_t align = bytes_per_point == sizeof(float4) ? 15 : 3;
        if (n && (reinterpret_cast<uintptr_t>(xyzi) & align)) { h->err = "device clouds must be 16-byte aligned (float4; packed xyz: 4-byte)"; return ERASOR_E_INVALID; }
        *out = reinterpret_cast<const float4*>(xyzi);
        return ERASOR_OK;
    }
    CK(stage.ensure(sizeof(float4) * std::max<size_t>(n, 1)));
    *out = stage.as<float4>();
    return ERASOR_OK;
}

// host clouds into their staging buffers (map_xyzi null: node mode, whose map is resident)
int stage_host_clouds(erasor_ctx* h, int ptr_kind, const float* map_xyzi, const float* qry_xyzi, size_t qry_bytes_per_point) {
    if (ptr_kind == ERASOR_PTR_DEVICE) return ERASOR_OK;
    if (map_xyzi && h->NM) CK(cudaMemcpyAsync(h->d_map_in.p(), map_xyzi, sizeof(float4) * h->NM, cudaMemcpyHostToDevice, h->stream));
    if (h->NQ) CK(cudaMemcpyAsync(h->d_qry_in.p(), qry_xyzi, qry_bytes_per_point * h->NQ, cudaMemcpyHostToDevice, h->stream));
    return ERASOR_OK;
}

erasor_geometry_t own_geometry(const erasor_params_t& p) { return erasor_geometry_t{p.max_range, p.min_h, p.max_h, p.num_rings, p.num_sectors}; }

bool same_geometry(const erasor_geometry_t& a, const erasor_geometry_t& b) {
    return a.max_range == b.max_range && a.min_h == b.min_h && a.max_h == b.max_h && a.num_rings == b.num_rings && a.num_sectors == b.num_sectors;
}

// The tables of geometry x: the handle's cached ones, or built and uploaded now with erasor_create's checks and codes (erasor_create
// itself builds the handle's own this way, as the first entry)
int geometry_tables(erasor_ctx* h, const erasor_geometry_t& x, const GeoTables** out) {
    for (const auto& t : h->geo_tables)
        if (same_geometry(t->key, x)) { *out = t.get(); return ERASOR_OK; }
    const long long Bll = (long long)x.num_rings * (long long)x.num_sectors;
    if (x.num_rings < 1 || x.num_sectors < 1 || Bll > 65534) { h->err = "num_rings*num_sectors must be in [1, 65534]"; return ERASOR_E_INVALID; }
    erasor_params_t p = h->p;
    p.max_range = x.max_range; p.min_h = x.min_h; p.max_h = x.max_h; p.num_rings = x.num_rings; p.num_sectors = x.num_sectors;
    std::unique_ptr<GeoTables> t(new GeoTables());
    t->key = x; t->B = (int)Bll;
    std::string terr;
    if (build_bin_tables(p, t->host, terr) != 0) { h->err = terr; return ERASOR_E_INVALID; }
    const size_t k1_bytes = k1_smem_bytes(x.num_rings, t->B);
    size_t k1_max = 0;
    cudaError_t e;
    auto fail = [&](const char* what) { h->err = std::string(what) + ": " + cudaGetErrorString(e); return ERASOR_E_CUDA; };
    if ((e = k1_table_limit(k1_bytes, false, false, h->smem_optin, &k1_max)) != cudaSuccess) return fail("cudaFuncGetAttributes");
    if (k1_bytes > k1_max || k3_smem_bytes(t->B) > h->smem_optin) {
        h->err = "num_rings*num_sectors too large for the per-CTA shared-memory bin table";
        return ERASOR_E_UNSUPPORTED;
    }
    const HostBinTables& ht = t->host;
    const size_t rb = sizeof(double) * ht.ring_thr.size(), sb = sizeof(SectorBoundary) * ht.sec_pos.size(), gb = sizeof(float) * ht.ring_guard.size();
    if ((e = t->d_ring.allocate(rb)) != cudaSuccess || (e = t->d_pos.allocate(sb)) != cudaSuccess || (e = t->d_neg.allocate(sb)) != cudaSuccess ||
        (e = t->d_guard.allocate(gb)) != cudaSuccess)
        return fail("cudaMalloc");
    if ((e = cudaMemcpy(t->d_ring.p(), ht.ring_thr.data(), rb, cudaMemcpyHostToDevice)) != cudaSuccess ||
        (e = cudaMemcpy(t->d_pos.p(), ht.sec_pos.data(), sb, cudaMemcpyHostToDevice)) != cudaSuccess ||
        (e = cudaMemcpy(t->d_neg.p(), ht.sec_neg.data(), sb, cudaMemcpyHostToDevice)) != cudaSuccess ||
        (e = cudaMemcpy(t->d_guard.p(), ht.ring_guard.data(), gb, cudaMemcpyHostToDevice)) != cudaSuccess)
        return fail("cudaMemcpy");
    t->view = ht.view(t->d_ring.as<double>(), t->d_pos.as<SectorBoundary>(), t->d_neg.as<SectorBoundary>(), t->d_guard.as<float>());
    h->geo_tables.push_back(std::move(t));
    *out = h->geo_tables.back().get();
    return ERASOR_OK;
}

// Node mode's K1 over tables of table_bytes for the grid of geometry x (geo_form: K1's geometry form, a tune's launch; prof: the
// profiling build): ERASOR_E_UNSUPPORTED, before anything is enqueued, when the launch cannot take them.  geometry_tables admits a
// geometry by the K1 of the mask and cloud modes, whose static shared memory is 32 KB smaller, so a geometry may run there and
// not here.
int node_k1_fits(erasor_ctx* h, const char* fn, const erasor_geometry_t& x, size_t table_bytes, bool geo_form, bool prof) {
    size_t lim = 0;
    const cudaError_t e = geo_form ? k1_geo_table_limit(table_bytes, h->smem_optin, &lim) : k1_table_limit(table_bytes, true, prof, h->smem_optin, &lim);
    if (e != cudaSuccess) { h->err = std::string("cudaFuncGetAttributes: ") + cudaGetErrorString(e); return ERASOR_E_CUDA; }
    if (table_bytes <= lim) return ERASOR_OK;
    h->err = std::string(fn) + ": a " + std::to_string(x.num_rings) + " x " + std::to_string(x.num_sectors) + " polar grid needs " +
             std::to_string(table_bytes) + " bytes of K1 tables, node mode's K1 takes at most " + std::to_string(lim) +
             " on this device (the cloud and batch modes run it)";
    return ERASOR_E_UNSUPPORTED;
}

// The tables K1 writes for geometry g of a sweep plan: the handle's geometry into k1_own (no plan, or an own plan), any other into
// k1_sweep[g]
K1GeoTables k1_tables(const erasor_ctx* h, const SweepPlan* plan, int g) {
    const bool own = !plan || plan->own;
    const GeoTables& geo = own ? *h->geo_tables[0] : *plan->geo[g].t;
    const erasor_ctx::K1Bufs& k = own ? h->k1_own : *h->k1_sweep[g];
    K1GeoTables o{};
    o.T = geo.view; o.B = geo.B;
    o.bin_map = k.bin_map.as<uint16_t>(); o.bin_qry = k.bin_qry.as<uint16_t>(); o.ch_cnt = k.ch_cnt.as<uint32_t>();
    o.zmin = k.zmin.as<uint32_t>(); o.zmax = k.zmax.as<uint32_t>(); o.cnt = k.cnt.as<uint32_t>();
    return o;
}

// The node-mode K1 launch that bins geometry g of a sweep plan (null: a plain call): its warps per CTA and the VoI lists it writes.
// A plain call and an own plan run the plain K1 into d_list_*; a plan that is not own gives its 32-warp launches d_list_*32, since
// their split of a chunk differs from its 8-warp launches'.
struct K1Lists { int warps; erasor_ctx::HBuf& idx; erasor_ctx::HBuf& cnt; };
K1Lists k1_lists(erasor_ctx* h, const SweepPlan* plan, int g) {
    if (!plan || plan->own) return {k1_warps(k1_smem_bytes(h->p.num_rings, h->B)), h->d_list_idx, h->d_list_cnt};
    const int warps = k1_warps(plan->launch_smem[plan->geo[g].launch]);
    return warps == 32 ? K1Lists{warps, h->d_list_idx32, h->d_list_cnt32} : K1Lists{warps, h->d_list_idx, h->d_list_cnt};
}

// the reset of the submission's records, queue and frame counters, and with t the reset of K1's z / count tables t
int run_init(erasor_ctx* h, const K1GeoTables* t) {
    const size_t F = (size_t)h->F, B = t ? (size_t)t->B : 0;
    h->launches++;
    CK(launch_init_tables(h->stream, t ? t->zmin : nullptr, t ? t->zmax : nullptr, 2 * F * B, t ? t->cnt : nullptr, t ? 2 * F * (B + 1) : 0,
                          h->d_nrecs.as<uint32_t>(), h->d_frame_rej.as<uint32_t>() + h->f0, h->d_nflag.as<uint32_t>() + h->f0, h->F,
                          h->d_queue.as<uint32_t>()));
    return ERASOR_OK;
}

int run_k1(erasor_ctx* h, int mode) {
    const K1GeoTables t = k1_tables(h, nullptr, 0);
    int rc = run_init(h, &t);
    if (rc) return rc;
    Scope s(h, 1);
    if (h->n_chunks_map + h->n_chunks_qry) h->launches++;
    CK(launch_k1(h->stream, t, h->cur_map, h->cur_qry, h->d_chunks.as<ChunkDesc>(), (int)(h->n_chunks_map + h->n_chunks_qry), h->F,
                 h->d_fence.as<unsigned long long>(), mode == 2 ? h->d_poses.as<NodePose>() : nullptr, mode == 2 ? h->d_list_idx.as<uint32_t>() : nullptr,
                 mode == 2 ? h->d_list_cnt.as<uint32_t>() : nullptr, mode != 0 && h->last.qry_xyz, mode == 2 ? h->k1_prof : nullptr));
    return ERASOR_OK;
}

// the handle's Scan Ratio Test settings over the geometry of K1's tables t
SrtParams srt_params(const erasor_ctx* h, const K1GeoTables& t, int version, int mode) {
    SrtParams sp{};
    sp.scan_ratio_threshold = h->p.scan_ratio_threshold;
    sp.th_bin_max_h = h->p.th_bin_max_h;
    sp.minimum_num_pts = h->p.minimum_num_pts;
    sp.version = version; sp.R = t.T.R; sp.S = t.T.S; sp.B = t.B; sp.scatter_mode = mode == 0 ? 0 : 1;
    return sp;
}

// node mode with inserts: R-GPF also writes its partitioned copy (ground first), which the inserts read
bool inserts_on(const erasor_ctx* h, int mode) { return mode == 2 && h->node_inserts; }

int run_insert_plan(erasor_ctx* h);

// R-GPF's size classes on their streams (classes: bits 0|1 A and B, bit 2 C), under classes A and B the node inserts' plan when on
// (a late class-C run has no plan to redo); k4sweep: a sweep's ground-filter groups and masks
int run_k4(erasor_ctx* h, int mode, uint8_t* keep_mask, uint8_t* ground_mask, const K4Fold& fold, int classes, const K4Sweep* k4sweep) {
    Scope s(h, 4);
    GpfParams gp{};
    gp.th_dist = h->p.gf_dist_thr; gp.th_seeds = h->p.gf_th_seeds_height; gp.num_lowest_pts = h->p.num_lowest_pts;
    gp.num_lpr = h->p.gf_num_lpr; gp.iters = std::min(h->p.gf_iter, kMaxIter); gp.cov_mode = h->p.cov_mode;
    const bool with_c = (classes & 4) != 0;
    h->launches += k4_num_launches(with_c);
    CK(cudaEventRecord(h->ev_fork, h->stream));
    CK(cudaStreamWaitEvent(h->stream_a, h->ev_fork, 0));
    CK(cudaStreamWaitEvent(h->stream_b, h->ev_fork, 0));
    if (with_c) CK(cudaStreamWaitEvent(h->stream_c, h->ev_fork, 0));
    CK(launch_k4(h->stream_a, h->stream_b, h->stream_c, gp, h->d_recs.as<FlagRec>(), h->d_queue.as<uint32_t>(), h->d_bucket.as<uint32_t>(), h->rec_capacity,
                 h->d_map_sorted.as<float4>(), h->d_map_src.as<uint32_t>(), h->d_frame_off.as<uint32_t>(),
                 (mode == 0 || inserts_on(h, mode)) ? h->d_part.as<float4>() : nullptr, keep_mask, ground_mask,
                 h->d_frame_rej.as<uint32_t>() + h->f0, h->d_scratch.as<unsigned char>(), h->sm_count, h->d_fence.as<unsigned long long>(), fold, classes, k4sweep));
    CK(cudaEventRecord(h->ev_join_a, h->stream_a));
    CK(cudaEventRecord(h->ev_join_b, h->stream_b));
    if (with_c) CK(cudaEventRecord(h->ev_join_c, h->stream_c));
    // node-mode inserts: the plan and the query scatter need only K1's tables, so they run on the main stream under R-GPF
    if (inserts_on(h, mode) && (classes & 3)) { int rc = run_insert_plan(h); if (rc) return rc; }
    CK(cudaStreamWaitEvent(h->stream, h->ev_join_a, 0));
    CK(cudaStreamWaitEvent(h->stream, h->ev_join_b, 0));
    if (with_c) CK(cudaStreamWaitEvent(h->stream, h->ev_join_c, 0));
    return ERASOR_OK;
}

// The mask modes' K2: the Scan Ratio Test fused into the scatter of the flagged bins, over the tables t that K1 wrote.  Node mode
// (list_idx non-null) walks the VoI lists of the K1 launch that wrote t, with its k1_warps warps per CTA; sweep: a sweep's settings.
int run_k2_srt(erasor_ctx* h, const SrtParams& sp, const K1GeoTables& t, const uint32_t* list_idx, const uint32_t* list_cnt, int k1_warps,
               const SrtSweep* sweep) {
    Scope s(h, 2);
    if (h->n_chunks_map) h->launches++;
    CK(launch_k2_srt(h->stream, sp, h->F, t, h->d_chunks.as<ChunkDesc>(), h->d_chunk_range.as<uint32_t>(), h->n_chunks_map, h->cur_map,
                     list_idx ? h->d_poses.as<NodePose>() : nullptr, h->d_frame_off.as<uint32_t>(), h->d_nflag.as<uint32_t>() + h->f0,
                     h->d_recs.as<FlagRec>(), h->d_nrecs.as<uint32_t>(), h->rec_capacity, h->d_queue.as<uint32_t>(), h->d_bucket.as<uint32_t>(),
                     h->d_map_sorted.as<float4>(), h->d_map_src.as<uint32_t>(), list_idx, list_cnt, k1_warps, sweep));
    return ERASOR_OK;
}

// K3 -> K2 -> K4 ; mode 0: every bin scattered + partitioned copies (cloud outputs), mode 1 / 2: flagged only + masks
// classes: which R-GPF size classes to launch (bits 0|1: A and B, bit 2: C)
int run_compare(erasor_ctx* h, int version, int mode, uint8_t* keep_mask, uint8_t* ground_mask, const K4Fold& fold, int classes = 7) {
    const int F = h->F;
    const NodePose* poses = mode == 2 ? h->d_poses.as<NodePose>() : nullptr;
    uint32_t* nflag = h->d_nflag.as<uint32_t>() + h->f0;
    const K1GeoTables t = k1_tables(h, nullptr, 0);
    const SrtParams sp = srt_params(h, t, version, mode);
    const K1Lists l = k1_lists(h, nullptr, 0);
    uint32_t* list_idx = poses ? l.idx.as<uint32_t>() : nullptr;
    uint32_t* list_cnt = poses ? l.cnt.as<uint32_t>() : nullptr;
    if (mode != 0 && h->fused_srt) {      // mask modes: SRT inside the scatter kernel
        const int rc = run_k2_srt(h, sp, t, list_idx, list_cnt, l.warps, nullptr);
        if (rc) return rc;
    } else {
        {
            Scope s(h, 3);
            h->launches++;
            CK(launch_k3(h->stream, sp, F, t, h->d_chunk_range.as<uint32_t>(), h->d_frame_off.as<uint32_t>(), h->d_dst_start.as<uint32_t>(),
                         h->d_status.as<uint8_t>(), h->d_action.as<uint8_t>(), h->d_flag_slot.as<uint32_t>(), nflag,
                         h->d_frame_rec_base.as<uint32_t>(), h->d_recs.as<FlagRec>(), h->d_nrecs.as<uint32_t>(), h->rec_capacity,
                         h->d_queue.as<uint32_t>(), h->d_bucket.as<uint32_t>()));
        }
        Scope s(h, 2);
        if (mode == 0) {
            if (h->n_chunks_map + h->n_chunks_qry) h->launches++;
            CK(launch_k2_both(h->stream, t, h->d_chunks.as<ChunkDesc>(), h->n_chunks_map, h->n_chunks_qry,
                              h->cur_map, h->d_dst_start.as<uint32_t>(), h->d_map_sorted.as<float4>(), h->d_map_src.as<uint32_t>(),
                              h->cur_qry, h->d_dst_start.as<uint32_t>() + (size_t)F * (t.B + 2), h->d_qry_sorted.as<float4>(), h->d_qry_src.as<uint32_t>()));
        } else {
            // mask modes, unfused (ERASOR_B200_UNFUSED_SRT=1): the same stable scatter, restricted to the flagged bins (K3's dense slots)
            if (h->n_chunks_map) h->launches++;
            CK(launch_k2(h->stream, t, 0, h->d_chunks.as<ChunkDesc>(), 0u, h->n_chunks_map, h->cur_map, poses, h->d_dst_start.as<uint32_t>(),
                         h->d_flag_slot.as<uint32_t>(), nflag, h->d_map_sorted.as<float4>(), h->d_map_src.as<uint32_t>(), list_idx, list_cnt, l.warps));
        }
    }
    return run_k4(h, mode, keep_mask, ground_mask, fold, classes, nullptr);
}

// A sweep's launches after the query staging: K1, then per geometry the fused Scan Ratio Test + scatter and R-GPF with the
// geometry's settings, over the handle's one set of records and scattered points.  An own plan runs K1 as a plain call does.  Any
// other plan resets every geometry's tables and bins them with K1's geometry form (one scan of the map per launch of the plan),
// then runs the geometries in reverse order, resetting the records between them, so that the union counts of the frame tables are
// those of setting 0's geometry.  classes: R-GPF's size classes (submit() asks for class C up front unless the plan is own).
int run_sweep(erasor_ctx* h, const SweepPlan& plan, bool qry_xyz, int classes) {
    const int n_geo = (int)plan.geo.size();
    int rc;
    if (plan.own) {
        if ((rc = run_k1(h, 2))) return rc;
    } else {
        for (int g = 0; g < n_geo; ++g) {
            const K1GeoTables t = k1_tables(h, &plan, g);
            if ((rc = run_init(h, &t))) return rc;
        }
        const int n_chunks = (int)(h->n_chunks_map + h->n_chunks_qry);
        for (size_t l = 0; l + 1 < plan.launch_begin.size(); ++l) {
            Scope s(h, 1);
            K1Geo G{};
            for (int g = plan.launch_begin[l]; g < plan.launch_begin[l + 1]; ++g, ++G.n) {
                G.g[G.n] = k1_tables(h, &plan, g);
                G.g[G.n].smem_off = G.n ? G.g[G.n - 1].smem_off + (uint32_t)k1_geo_smem_bytes(G.g[G.n - 1].T.R, G.g[G.n - 1].B) : 0u;
            }
            const K1Lists lists = k1_lists(h, &plan, plan.launch_begin[l]);
            if (n_chunks) h->launches++;
            CK(launch_k1_geo(h->stream, G, plan.launch_smem[l], h->cur_map, h->cur_qry, h->d_chunks.as<ChunkDesc>(), n_chunks, h->F,
                             h->d_fence.as<unsigned long long>(), h->d_poses.as<NodePose>(), lists.idx.as<uint32_t>(), lists.cnt.as<uint32_t>(), qry_xyz));
        }
    }
    for (int g = n_geo - 1; g >= 0; --g) {
        const SweepGeo& sg = plan.geo[g];
        if (g != n_geo - 1 && (rc = run_init(h, nullptr))) return rc;      // records, queue and frame counters of the geometry before
        const K1GeoTables t = k1_tables(h, &plan, g);
        const K1Lists lists = k1_lists(h, &plan, g);
        if ((rc = run_k2_srt(h, srt_params(h, t, h->p.version, 2), t, lists.idx.as<uint32_t>(), lists.cnt.as<uint32_t>(), lists.warps, &sg.ssw)))
            return rc;
        if ((rc = run_k4(h, 2, nullptr, nullptr, K4Fold{nullptr, nullptr, 0u, 0u}, classes, &sg.ksw))) return rc;
    }
    return ERASOR_OK;
}

// Node-mode inserts of one submission: buffers (before any capture -- a reallocation retires the cached graphs) ...
int ensure_insert_buffers(erasor_ctx* h) {
    const size_t B = (size_t)h->B, F = (size_t)h->F, NM = h->NM, NQ = h->NQ;
    CK(h->d_part.ensure(sizeof(float4) * std::max<size_t>(NM, 1)));
    CK(h->d_qry_sorted.ensure(sizeof(float4) * std::max<size_t>(NQ, 1)));
    CK(h->d_qry_src.ensure(sizeof(uint32_t) * std::max<size_t>(NQ, 1)));
    CK(h->d_ins_slot.ensure(sizeof(uint32_t) * F * B));
    CK(h->d_ins_n.ensure(sizeof(uint32_t) * F));
    CK(h->d_ins_bin_off.ensure(sizeof(uint32_t) * F * B));
    CK(h->d_ins_frame_cnt.ensure(sizeof(uint32_t) * F));
    CK(h->d_ins_off.ensure(sizeof(uint32_t) * (F + 1)));
    CK(h->d_ins_fwd.ensure(sizeof(float) * 12 * F));
    CK(h->d_ins.ensure(sizeof(float4) * (NQ + NM + 1)));      // a frame inserts at most its binned queries + its flagged map points
    if (h->p.version == 3 && !h->p.skip_voxelize) {
        CK(h->d_vox.ensure(sizeof(float4) * (NM + NQ + 1)));
        CK(h->d_vox_cnt.ensure(sizeof(uint32_t) * std::max<size_t>(h->rec_capacity, 1)));
        CK(h->d_vox_start.ensure(sizeof(uint32_t) * std::max<size_t>(h->rec_capacity, 1)));
        CK(h->d_vox_scratch.ensure((size_t)k4b_scratch_offset((uint32_t)NQ, (uint32_t)NM, (uint32_t)(F * B)) + 36 + 64));
    }
    if (sizeof(float) * 12 * F > h->h_ins_fwd.cap() || sizeof(uint32_t) * (F + 1) > h->h_ins_off.cap()) h->alloc_epoch++;   // captured copies
    CK(h->h_ins_fwd.ensure(sizeof(float) * 12 * F));
    CK(h->h_ins_off.ensure(sizeof(uint32_t) * (F + 1)));
    return ERASOR_OK;
}

// ... after K1: the action of every bin and the stable scatter of the inserting bins' query points ...
int run_insert_plan(erasor_ctx* h) {
    const int F = h->F;
    const K1GeoTables t = k1_tables(h, nullptr, 0);
    CK(cudaMemcpyAsync(h->d_ins_fwd.p(), h->h_ins_fwd.p(), sizeof(float) * 12 * (size_t)F, cudaMemcpyHostToDevice, h->stream));
    h->launches += 1 + (h->n_chunks_qry ? 1 : 0);
    CK(launch_ins_plan(h->stream, srt_params(h, t, h->p.version, 2), F, t, h->d_chunk_range.as<uint32_t>(), h->d_action.as<uint8_t>(),
                       h->d_flag_slot.as<uint32_t>(), h->d_ins_slot.as<uint32_t>(), h->d_ins_n.as<uint32_t>(), h->d_dst_start.as<uint32_t>()));
    CK(launch_k2(h->stream, t, 1, h->d_chunks.as<ChunkDesc>(), h->n_chunks_map, h->n_chunks_qry, h->cur_qry, nullptr,
                 h->d_dst_start.as<uint32_t>() + (size_t)F * (t.B + 2), h->d_ins_slot.as<uint32_t>(), h->d_ins_n.as<uint32_t>(),
                 h->d_qry_sorted.as<float4>(), h->d_qry_src.as<uint32_t>(), nullptr, nullptr, 8));
    return ERASOR_OK;
}

// ... after R-GPF: K4b over every frame's flagged bins (v3), then sizes, offsets and the copy; the offsets are read back through
// pinned memory (again after a late class-C run, which changes the ground of its bins)
int run_insert_assemble(erasor_ctx* h) {
    const int F = h->F;
    const K1GeoTables t = k1_tables(h, nullptr, 0);
    const bool vox = h->p.version == 3 && !h->p.skip_voxelize;
    const uint32_t* qoff = h->d_frame_off.as<uint32_t>() + (F + 1);
    if (vox) {
        h->launches++;
        CK(launch_k4b(h->stream, (float)h->p.map_voxel_size, t.B, F, h->d_recs.as<FlagRec>(), h->d_nrecs.as<uint32_t>(), h->rec_capacity,
                      t.cnt, h->d_dst_start.as<uint32_t>(), qoff, h->d_qry_sorted.as<float4>(), h->d_part.as<float4>(),
                      h->d_vox.as<float4>(), h->d_vox_cnt.as<uint32_t>(), h->d_vox_start.as<uint32_t>(), h->d_vox_scratch.as<unsigned char>(), h->sm_count));
    }
    h->launches += kInsAssembleLaunches;
    CK(launch_ins_assemble(h->stream, t.B, F, vox ? 1 : 0, h->d_action.as<uint8_t>(), h->d_flag_slot.as<uint32_t>(), h->d_frame_rec_base.as<uint32_t>(),
                           h->d_recs.as<FlagRec>(), h->d_nrecs.as<uint32_t>(), h->rec_capacity, t.cnt, h->d_dst_start.as<uint32_t>(),
                           qoff, vox ? h->d_vox_cnt.as<uint32_t>() : nullptr, vox ? h->d_vox_start.as<uint32_t>() : nullptr,
                           h->d_qry_sorted.as<float4>(), h->d_part.as<float4>(), vox ? h->d_vox.as<float4>() : nullptr, h->d_ins_fwd.as<float>(),
                           h->d_ins_bin_off.as<uint32_t>(), h->d_ins_frame_cnt.as<uint32_t>(), h->d_ins_off.as<uint32_t>(), h->d_ins.as<float4>(),
                           h->sm_count));
    CK(cudaMemcpyAsync(h->h_ins_off.p(), h->d_ins_off.p(), sizeof(uint32_t) * ((size_t)F + 1), cudaMemcpyDeviceToHost, h->stream));
    return ERASOR_OK;
}

// room for n_new float4 in buf, its first n_old kept (the copy is ordered on st and finished before the old allocation goes)
cudaError_t grow_points(DeviceBuffer& buf, size_t n_old, size_t n_new, cudaStream_t st) {
    const size_t bytes = sizeof(float4) * n_new;
    if (bytes <= buf.cap()) return cudaSuccess;
    DeviceBuffer nb;
    cudaError_t e = nb.allocate(bytes + bytes / 4 + 4096);
    if (e == cudaSuccess && n_old) e = cudaMemcpyAsync(nb.p(), buf.p(), sizeof(float4) * n_old, cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e == cudaSuccess) buf = std::move(nb);
    return e;
}

// a completed submission's inserts, appended to the call's (sub-batches in frame order)
int collect_inserts(erasor_ctx* h) {
    const uint32_t* off = h->h_ins_off.as<uint32_t>();
    const size_t base = h->ins_call_off.back(), n = off[h->F];
    CK(grow_points(h->d_ins_call, base, base + n, h->stream));
    if (n) CK(cudaMemcpyAsync(h->d_ins_call.as<float4>() + base, h->d_ins.p(), sizeof(float4) * n, cudaMemcpyDeviceToDevice, h->stream));
    for (int f = 1; f <= h->F; ++f) h->ins_call_off.push_back(base + off[f]);
    CK(cudaStreamSynchronize(h->stream));
    return ERASOR_OK;
}

int copy_out(erasor_ctx* h, const void* dev_src, void* user_dst, size_t bytes, int ptr_kind) {
    if (!bytes) return ERASOR_OK;
    CK(cudaMemcpyAsync(user_dst, dev_src, bytes, ptr_kind == ERASOR_PTR_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, h->stream));
    return ERASOR_OK;
}

float status_value(uint8_t code) {
    switch (code) {
        case ST_MERGE: return ERASOR_STATUS_MERGE_BINS;
        case ST_MAP_HIGH: return ERASOR_STATUS_MAP_IS_HIGHER;
        case ST_BLOCKED: return ERASOR_STATUS_BLOCKED;
        case ST_CURR_HIGH: return ERASOR_STATUS_CURR_IS_HIGHER;
        default: return ERASOR_STATUS_LITTLE_NUM;
    }
}

}  // namespace

extern "C" {

int erasor_abi_version(void) { return ERASOR_B200_ABI_VERSION; }

const char* erasor_last_error(erasor_handle_t h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int erasor_create(const erasor_params_t* params, int device, erasor_handle_t* out) {
    if (!params || !out) { g_create_error = "null argument"; return ERASOR_E_INVALID; }
    *out = nullptr;
    const erasor_params_t& p = *params;
    const long long Bll = (long long)p.num_rings * (long long)p.num_sectors;
    if (p.num_rings < 1 || p.num_sectors < 1 || Bll > 65534) { g_create_error = "num_rings*num_sectors must be in [1, 65534]"; return ERASOR_E_INVALID; }
    if (p.version != 2 && p.version != 3) { g_create_error = "Other version is not implemented!"; return ERASOR_E_INVALID; }   // OfflineMapUpdater.cpp:274
    if (p.sort_mode != 1) { g_create_error = "sort_mode must be 1 (stable z order)"; return ERASOR_E_UNSUPPORTED; }
    if (p.gf_iter > kMaxIter) { g_create_error = "gf_iter above the tap capacity (8)"; return ERASOR_E_UNSUPPORTED; }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        g_create_error = std::string("no CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0") +
                         " (this library has no CPU path)";
        return ERASOR_E_CUDA;
    }
    if (device < 0 || device >= ndev) { g_create_error = "bad device index"; return ERASOR_E_INVALID; }
    erasor_ctx* h = new erasor_ctx();
    h->p = p; h->device = device; h->B = (int)Bll;
    if (const char* ng = std::getenv("ERASOR_B200_NO_GRAPH")) h->use_graphs = !(ng[0] == '1');
    if (const char* uf = std::getenv("ERASOR_B200_UNFUSED_SRT")) h->fused_srt = !(uf[0] == '1');
    if (const char* cs = std::getenv("ERASOR_B200_CTAS_PER_SM")) h->ctas_per_sm = std::max(1, std::min(8, std::atoi(cs)));
    auto fail = [&](const char* what, cudaError_t ce) {
        g_create_error = std::string(what) + ": " + cudaGetErrorString(ce);
        erasor_destroy(h);
        return ERASOR_E_CUDA;
    };
    if ((e = cudaSetDevice(device)) != cudaSuccess) return fail("cudaSetDevice", e);
    cudaDeviceProp prop;
    if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) return fail("cudaGetDeviceProperties", e);
    h->sm_count = prop.multiProcessorCount;
    h->smem_optin = (size_t)prop.sharedMemPerBlockOptin;
    if (const char* tu = std::getenv("ERASOR_B200_TUNE_UNPACKED")) h->tune_unpacked = tu[0] == '1';
    // the handle's polar tables: the first entry of its geometry cache (tables build_bin_tables rejects: ERASOR_E_INVALID; beyond
    // the device's shared memory: ERASOR_E_UNSUPPORTED)
    const GeoTables* own = nullptr;
    if (const int rc = geometry_tables(h, own_geometry(p), &own)) {
        g_create_error = h->err;
        erasor_destroy(h);
        return rc;
    }
    // R-GPF's bins are long serial chains: its CTAs go first whenever SM resources free up (highest stream priority), the
    // bandwidth / issue-bound kernels of this and of overlapped handles fill in around them
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    if (const char* np = std::getenv("ERASOR_B200_NO_PRIORITY")) { if (np[0] == '1') prio_hi = prio_lo; }
    if ((e = cudaStreamCreateWithPriority(&h->stream, cudaStreamNonBlocking, prio_lo)) != cudaSuccess) return fail("cudaStreamCreate", e);
    if ((e = cudaStreamCreateWithPriority(&h->stream_a, cudaStreamNonBlocking, prio_hi)) != cudaSuccess) return fail("cudaStreamCreate", e);
    if ((e = cudaStreamCreateWithPriority(&h->stream_b, cudaStreamNonBlocking, prio_hi)) != cudaSuccess) return fail("cudaStreamCreate", e);
    if ((e = cudaStreamCreateWithPriority(&h->stream_c, cudaStreamNonBlocking, prio_hi)) != cudaSuccess) return fail("cudaStreamCreate", e);
    if ((e = cudaEventCreateWithFlags(&h->ev_join_a, cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", e);
    if ((e = cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", e);
    if ((e = cudaEventCreateWithFlags(&h->ev_join_b, cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", e);
    if ((e = cudaEventCreateWithFlags(&h->ev_join_c, cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", e);
    if ((e = h->h_words.allocate(128)) != cudaSuccess) return fail("cudaMallocHost", e);
    std::memset(h->h_words.p(), 0, 128);
    if ((e = h->d_fence.ensure(sizeof(unsigned long long) * 4)) != cudaSuccess) return fail("cudaMalloc", e);
    if ((e = cudaMemset(h->d_fence.p(), 0, sizeof(unsigned long long) * 4)) != cudaSuccess) return fail("cudaMemset", e);
    *out = h;
    return ERASOR_OK;
}

void erasor_destroy(erasor_handle_t h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    drain_timers(h);
    for (auto& g : h->graphs) cudaGraphExecDestroy(g.exec);
    h->graphs.clear();
    if (h->comm) { NcclApi* api = nccl_api(h->err); if (api) api->CommDestroy(h->comm); h->comm = nullptr; }
    vox_batch_destroy(h->vb);
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    if (h->ev_join_a) cudaEventDestroy(h->ev_join_a);
    if (h->ev_join_b) cudaEventDestroy(h->ev_join_b);
    if (h->ev_join_c) cudaEventDestroy(h->ev_join_c);
    if (h->stream_a) cudaStreamDestroy(h->stream_a);
    if (h->stream_b) cudaStreamDestroy(h->stream_b);
    if (h->stream_c) cudaStreamDestroy(h->stream_c);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

void* erasor_stream(erasor_handle_t h) { return h ? (void*)h->stream : nullptr; }

int erasor_synchronize(erasor_handle_t h) {
    if (!h) return ERASOR_E_INVALID;
    CK(cudaStreamSynchronize(h->stream));
    return ERASOR_OK;
}

double erasor_get_max_range(erasor_handle_t h) { return h ? h->p.max_range : 0.0; }

int erasor_set_inputs(erasor_handle_t h, const float* map_voi_xyzi, size_t n_map, const float* query_voi_xyzi, size_t n_query, int ptr_kind) {
    if (!h) return ERASOR_E_INVALID;
    if ((n_map && !map_voi_xyzi) || (n_query && !query_voi_xyzi)) { h->err = "null cloud"; return ERASOR_E_INVALID; }
    CK(cudaSetDevice(h->device));
    int rc;
    if (h->pending && (rc = erasor_wait(h))) return rc;
    h->stage = 0;
    h->f0 = 0; h->stat_F = 1;
    h->ins_call_off.clear();                   // the inserts of an earlier node call end with this submission
    if (ptr_kind != ERASOR_PTR_HOST && ptr_kind != ERASOR_PTR_DEVICE) { h->err = "erasor_set_inputs: ptr_kind must be HOST or DEVICE (the cloud outputs carry the query's intensity)"; return ERASOR_E_INVALID; }
    const uint64_t mo[2] = {0, n_map}, qo[2] = {0, n_query};
    rc = prepare_batch(h, mo, qo, 1, 0);
    if (rc) return rc;
    if ((rc = device_cloud(h, h->d_map_in, map_voi_xyzi, h->NM, ptr_kind, &h->cur_map)) ||
        (rc = device_cloud(h, h->d_qry_in, query_voi_xyzi, h->NQ, ptr_kind, &h->cur_qry)) ||
        (rc = stage_host_clouds(h, ptr_kind, map_voi_xyzi, query_voi_xyzi, sizeof(float4)))) return rc;
    if ((rc = run_k1(h, 0))) return rc;
    h->stage = 1;
    return ERASOR_OK;
}

int erasor_compare(erasor_handle_t h, int version, int frame) {
    (void)frame;   // the reference uses it only for a commented-out csv dump (erasor.cpp:341-343)
    if (!h) return ERASOR_E_INVALID;
    if (h->stage < 1) { h->err = "erasor_compare before erasor_set_inputs"; return ERASOR_E_STATE; }
    if (h->stage > 1) { h->err = "erasor_compare called twice: set_inputs -> exactly one compare (OfflineMapUpdater.cpp:266-272)"; return ERASOR_E_STATE; }
    if (version != 2 && version != 3) { h->err = "Other version is not implemented!"; return ERASOR_E_INVALID; }
    CK(cudaSetDevice(h->device));
    const K1GeoTables t = k1_tables(h, nullptr, 0);
    const int B = t.B;
    const size_t NM = h->NM, NQ = h->NQ;
    CK(h->d_keep.ensure(std::max<size_t>(NM, 1)));
    CK(h->d_ground.ensure(std::max<size_t>(NM, 1)));
    CK(cudaMemsetAsync(h->d_keep.p(), 1, std::max<size_t>(NM, 1), h->stream));
    CK(cudaMemsetAsync(h->d_ground.p(), 0, std::max<size_t>(NM, 1), h->stream));
    // R-GPF class C (bins beyond 2560 points, 1024-thread CTAs) is launched only while such bins are being seen; if one turns up
    // unannounced the class runs after the fact and the output assembly is repeated (same policy as the mask modes, erasor_wait)
    const bool with_c = h->class_c_state != 0;
    int rc = run_compare(h, version, 0, h->d_keep.as<uint8_t>(), h->d_ground.as<uint8_t>(), K4Fold{nullptr, nullptr, 0u, 0u}, with_c ? 7 : 3);
    if (rc) return rc;
    const bool vox = (version == 3) && !h->p.skip_voxelize;
    if (vox) {
        CK(h->d_vox.ensure(sizeof(float4) * (NM + NQ + 1)));
        CK(h->d_vox_cnt.ensure(sizeof(uint32_t) * (size_t)B));
        CK(h->d_vox_start.ensure(sizeof(uint32_t) * (size_t)B));
        CK(h->d_vox_scratch.ensure((size_t)k4b_scratch_offset((uint32_t)NQ, (uint32_t)NM, (uint32_t)B) + 36 + 64));
    }
    CK(h->d_arranged.ensure(sizeof(float4) * (2 * NM + NQ + 1)));
    CK(h->d_map_rej.ensure(sizeof(float4) * std::max<size_t>(NM, 1)));
    CK(h->d_curr_rej.ensure(sizeof(float4) * std::max<size_t>(NQ, 1)));
    CK(h->d_jobs.ensure(sizeof(CopyJob) * 5 * (size_t)B));
    CK(h->d_out_sizes.ensure(sizeof(uint32_t) * 8));
    CK(h->d_k5tmp.ensure(sizeof(uint32_t) * 3 * (size_t)(B + 1)));
    // in-bin voxelisation (v3) + output assembly + the sizes the caller needs, read back through pinned memory
    auto assemble = [&]() -> int {
        if (vox) {
            Scope s(h, 4);
            h->launches++;
            CK(launch_k4b(h->stream, (float)h->p.map_voxel_size, B, 1, h->d_recs.as<FlagRec>(), h->d_nrecs.as<uint32_t>(), h->rec_capacity,
                          t.cnt, h->d_dst_start.as<uint32_t>(), h->d_frame_off.as<uint32_t>() + 2, h->d_qry_sorted.as<float4>(), h->d_part.as<float4>(),
                          h->d_vox.as<float4>(), h->d_vox_cnt.as<uint32_t>(), h->d_vox_start.as<uint32_t>(),
                          h->d_vox_scratch.as<unsigned char>(), h->sm_count));
        }
        {
            Scope s(h, 5);
            h->launches += 2;
            CK(launch_k5(h->stream, B, version, h->p.skip_voxelize, t.cnt, h->d_dst_start.as<uint32_t>(), h->d_action.as<uint8_t>(),
                         h->d_flag_slot.as<uint32_t>(), h->d_recs.as<FlagRec>(), h->d_nrecs.as<uint32_t>(),
                         vox ? h->d_vox_cnt.as<uint32_t>() : nullptr, vox ? h->d_vox_start.as<uint32_t>() : nullptr,
                         h->d_map_sorted.as<float4>(), h->d_qry_sorted.as<float4>(), h->d_part.as<float4>(),
                         vox ? h->d_vox.as<float4>() : nullptr, h->d_arranged.as<float4>(),
                         h->d_map_rej.as<float4>(), h->d_curr_rej.as<float4>(), h->d_jobs.as<CopyJob>(), h->d_out_sizes.as<uint32_t>(),
                         h->d_k5tmp.as<uint32_t>(), h->sm_count * 4));
        }
        uint32_t* w = h->h_words.as<uint32_t>();
        CK(cudaMemcpyAsync(w + 4, h->d_out_sizes.p(), sizeof(uint32_t) * 5, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaMemcpyAsync(w + 9, h->d_dst_start.as<uint32_t>() + B, sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
        CK(cudaMemcpyAsync(w + 10, h->d_nrecs.p(), sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
        CK(cudaMemcpyAsync(w + 11, h->d_queue.as<uint32_t>() + kBucketC0, sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        return ERASOR_OK;
    };
    if ((rc = assemble())) return rc;
    const uint32_t n_class_c = h->words()[11];
    if (!with_c && n_class_c > 0) {
        if ((rc = run_k4(h, 0, h->d_keep.as<uint8_t>(), h->d_ground.as<uint8_t>(), K4Fold{nullptr, nullptr, 0u, 0u}, 4, nullptr))) return rc;
        if ((rc = assemble())) return rc;
    }
    h->class_c_state = (int)std::min<uint32_t>(n_class_c, 0x7FFFFFFFu);
    for (int i = 0; i < 5; ++i) h->out_sizes[i] = h->words()[4 + i];
    h->complement_start = h->words()[9];
    h->n_recs_host = h->words()[10];
    h->stage = 2;
    return ERASOR_OK;
}

int erasor_get_output_sizes(erasor_handle_t h, size_t* n_arranged, size_t* n_complement, size_t* n_map_rejected, size_t* n_curr_rejected) {
    if (!h) return ERASOR_E_INVALID;
    if (h->stage < 2) { h->err = "no compare result"; return ERASOR_E_STATE; }
    if (n_arranged) *n_arranged = h->out_sizes[0];
    if (n_complement) *n_complement = h->out_sizes[1];
    if (n_map_rejected) *n_map_rejected = h->out_sizes[2];
    if (n_curr_rejected) *n_curr_rejected = h->out_sizes[3];
    return ERASOR_OK;
}

int erasor_get_static_estimate(erasor_handle_t h, float* arranged_xyzi, size_t cap_arranged, size_t* n_arranged,
                               float* complement_xyzi, size_t cap_complement, size_t* n_complement, int ptr_kind) {
    if (!h) return ERASOR_E_INVALID;
    if (h->stage < 2) { h->err = "erasor_get_static_estimate before erasor_compare"; return ERASOR_E_STATE; }
    if (n_arranged) *n_arranged = h->out_sizes[0];
    if (n_complement) *n_complement = h->out_sizes[1];
    if ((arranged_xyzi && cap_arranged < h->out_sizes[0]) || (complement_xyzi && cap_complement < h->out_sizes[1])) {
        h->err = "output buffer too small"; return ERASOR_E_CAPACITY;
    }
    CK(cudaSetDevice(h->device));
    int rc;
    if (arranged_xyzi && (rc = copy_out(h, h->d_arranged.p(), arranged_xyzi, sizeof(float4) * h->out_sizes[0], ptr_kind))) return rc;
    if (complement_xyzi && (rc = copy_out(h, h->d_map_sorted.as<float4>() + h->complement_start, complement_xyzi,
                                          sizeof(float4) * h->out_sizes[1], ptr_kind))) return rc;
    CK(cudaStreamSynchronize(h->stream));
    return ERASOR_OK;
}

int erasor_get_outliers(erasor_handle_t h, float* map_rejected_xyzi, size_t cap_map, size_t* n_map_rejected,
                        float* curr_rejected_xyzi, size_t cap_curr, size_t* n_curr_rejected, int ptr_kind) {
    if (!h) return ERASOR_E_INVALID;
    if (h->stage < 2) { h->err = "erasor_get_outliers before erasor_compare"; return ERASOR_E_STATE; }
    if (n_map_rejected) *n_map_rejected = h->out_sizes[2];
    if (n_curr_rejected) *n_curr_rejected = h->out_sizes[3];
    if ((map_rejected_xyzi && cap_map < h->out_sizes[2]) || (curr_rejected_xyzi && cap_curr < h->out_sizes[3])) {
        h->err = "output buffer too small"; return ERASOR_E_CAPACITY;
    }
    CK(cudaSetDevice(h->device));
    int rc;
    if (map_rejected_xyzi && (rc = copy_out(h, h->d_map_rej.p(), map_rejected_xyzi, sizeof(float4) * h->out_sizes[2], ptr_kind))) return rc;
    if (curr_rejected_xyzi && (rc = copy_out(h, h->d_curr_rej.p(), curr_rejected_xyzi, sizeof(float4) * h->out_sizes[3], ptr_kind))) return rc;
    CK(cudaStreamSynchronize(h->stream));
    return ERASOR_OK;
}

int erasor_device_outputs(erasor_handle_t h, const float** arranged, const float** complement, const float** map_rejected, const float** curr_rejected) {
    if (!h) return ERASOR_E_INVALID;
    if (h->stage < 2) { h->err = "erasor_device_outputs before erasor_compare"; return ERASOR_E_STATE; }
    if (arranged) *arranged = h->d_arranged.as<float>();
    if (complement) *complement = reinterpret_cast<const float*>(h->d_map_sorted.as<float4>() + h->complement_start);
    if (map_rejected) *map_rejected = h->d_map_rej.as<float>();
    if (curr_rejected) *curr_rejected = h->d_curr_rej.as<float>();
    return ERASOR_OK;
}

// ERASOR::ground_viz (public member, erasor.h:127): the R-GPF ground points of the flagged bins of the last compare, in
// processing order -- the tail get_static_estimate appends to `arranged` (erasor.cpp:616)
int erasor_get_ground_viz(erasor_handle_t h, float* ground_xyzi, size_t cap, size_t* n_ground, int ptr_kind) {
    if (!h) return ERASOR_E_INVALID;
    if (h->stage < 2) { h->err = "erasor_get_ground_viz before erasor_compare"; return ERASOR_E_STATE; }
    const size_t n = h->out_sizes[4];
    if (n_ground) *n_ground = n;
    if (!ground_xyzi) return ERASOR_OK;
    if (cap < n) { h->err = "output buffer too small"; return ERASOR_E_CAPACITY; }
    CK(cudaSetDevice(h->device));
    int rc;
    if ((rc = copy_out(h, h->d_arranged.as<float4>() + (h->out_sizes[0] - n), ground_xyzi, sizeof(float4) * n, ptr_kind))) return rc;
    CK(cudaStreamSynchronize(h->stream));
    return ERASOR_OK;
}

int erasor_get_bins(erasor_handle_t h, int which_cloud, int32_t* bin_of_point, float* min_h, float* max_h, uint32_t* count) {
    if (!h) return ERASOR_E_INVALID;
    const bool node = h->desc_mode == 2 && h->F == 1 && h->stage < 1;      // one node of erasor_process_nodes: tables only
    if ((h->stage < 1 && !node) || h->F != 1) { h->err = "erasor_get_bins needs a single-frame erasor_set_inputs or a one-node erasor_process_nodes"; return ERASOR_E_STATE; }
    if (node && bin_of_point) { h->err = "node mode keeps no per-point bins of the map"; return ERASOR_E_STATE; }
    if (which_cloud != 0 && which_cloud != 1) { h->err = "which_cloud"; return ERASOR_E_INVALID; }
    CK(cudaSetDevice(h->device));
    const K1GeoTables t = k1_tables(h, nullptr, 0);
    const int B = t.B;
    const size_t n = which_cloud == 0 ? h->NM : h->NQ;
    CK(cudaStreamSynchronize(h->stream));
    if (bin_of_point && n) {
        std::vector<uint16_t> tmp(n);
        CK(cudaMemcpy(tmp.data(), which_cloud == 0 ? t.bin_map : t.bin_qry, sizeof(uint16_t) * n, cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < n; ++i) bin_of_point[i] = tmp[i] == kNoBin16 ? -1 : (int32_t)tmp[i];
    }
    if (min_h || max_h || count) {
        std::vector<uint32_t> mn(B), mx(B);
        CK(cudaMemcpy(mn.data(), t.zmin + (size_t)which_cloud * B, sizeof(uint32_t) * B, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(mx.data(), t.zmax + (size_t)which_cloud * B, sizeof(uint32_t) * B, cudaMemcpyDeviceToHost));
        std::vector<uint32_t> c(B, 0);
        CK(cudaMemcpy(c.data(), t.cnt + (size_t)which_cloud * (B + 1), sizeof(uint32_t) * B, cudaMemcpyDeviceToHost));
        const float nan = std::numeric_limits<float>::quiet_NaN();
        for (int b = 0; b < B; ++b) {
            const bool empty = mn[b] == 0xFFFFFFFFu && mx[b] == 0u;
            if (min_h) min_h[b] = empty ? nan : ordered_to_float(mn[b]);
            if (max_h) max_h[b] = empty ? nan : ordered_to_float(mx[b]);
            if (count) count[b] = c[b];
        }
    }
    return ERASOR_OK;
}

int erasor_get_status(erasor_handle_t h, float* status) {
    if (!h || !status) return ERASOR_E_INVALID;
    if (h->stage < 2) { h->err = "erasor_get_status before erasor_compare"; return ERASOR_E_STATE; }
    CK(cudaSetDevice(h->device));
    std::vector<uint8_t> st(h->B);
    CK(cudaMemcpy(st.data(), h->d_status.p(), h->B, cudaMemcpyDeviceToHost));
    for (int b = 0; b < h->B; ++b) status[b] = status_value(st[b]);
    return ERASOR_OK;
}

int erasor_get_planes(erasor_handle_t h, int32_t* bin_ids, int32_t* n_points, int32_t* n_seeds, double* lpr_height,
                      double* normal_d, int32_t* n_ground, size_t* n_planes) {
    if (!h || !n_planes) return ERASOR_E_INVALID;
    if (h->stage < 2) { h->err = "erasor_get_planes before erasor_compare"; return ERASOR_E_STATE; }
    CK(cudaSetDevice(h->device));
    const size_t n = h->n_recs_host, cap = *n_planes;
    *n_planes = n;
    if (!bin_ids && !n_points && !n_seeds && !lpr_height && !normal_d && !n_ground) return ERASOR_OK;
    if (cap < n) { h->err = "plane buffer too small"; return ERASOR_E_CAPACITY; }
    std::vector<FlagRec> recs(n);
    if (n) CK(cudaMemcpy(recs.data(), h->d_recs.p(), sizeof(FlagRec) * n, cudaMemcpyDeviceToHost));
    const int it = std::min(h->p.gf_iter, kMaxIter);
    for (size_t i = 0; i < n; ++i) {
        const FlagRec& r = recs[i];   // single frame: record index == slot == processing order (bin order)
        if (bin_ids) bin_ids[i] = (int32_t)r.bin;
        if (n_points) n_points[i] = (int32_t)r.n_points;
        if (n_seeds) n_seeds[i] = (int32_t)r.n_seeds;
        if (lpr_height) lpr_height[i] = r.lpr_height;
        for (int k = 0; k < it; ++k) {
            if (normal_d) for (int c = 0; c < 4; ++c) normal_d[(i * it + k) * 4 + c] = r.normal_d[k][c];
            if (n_ground) n_ground[i * it + k] = (int32_t)r.n_ground[k];
        }
    }
    return ERASOR_OK;
}

int erasor_get_static_mask(erasor_handle_t h, uint8_t* keep_map, uint8_t* is_ground) {
    if (!h) return ERASOR_E_INVALID;
    if (h->stage < 2) { h->err = "erasor_get_static_mask before erasor_compare"; return ERASOR_E_STATE; }
    CK(cudaSetDevice(h->device));
    if (keep_map && h->NM) CK(cudaMemcpy(keep_map, h->d_keep.p(), h->NM, cudaMemcpyDeviceToHost));
    if (is_ground && h->NM) CK(cudaMemcpy(is_ground, h->d_ground.p(), h->NM, cudaMemcpyDeviceToHost));
    return ERASOR_OK;
}

int erasor_get_fence_counts(erasor_handle_t h, uint64_t* negzero_points, uint64_t* empty_plane_fits, uint64_t* ambiguous_sector) {
    if (!h) return ERASOR_E_INVALID;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    unsigned long long v[4];
    CK(cudaMemcpy(v, h->d_fence.p(), sizeof(v), cudaMemcpyDeviceToHost));
    if (negzero_points) *negzero_points = v[0];
    if (empty_plane_fits) *empty_plane_fits = v[1];
    if (ambiguous_sector) *ambiguous_sector = v[2];
    return ERASOR_OK;
}

namespace {

bool is_pinned_host(const void* p) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

// the step's masks back to the caller: a host caller's per-frame masks from their staging, and the map's mask into keep_out
int copy_masks_out(erasor_ctx* h, const Step& s) {
    const bool host = s.ptr_kind != ERASOR_PTR_DEVICE;
    if (host && s.n_keep) CK(cudaMemcpyAsync(s.user_keep, s.d_keep, s.n_keep, cudaMemcpyDeviceToHost, h->stream));
    if (s.keep_out && s.n_map_global)
        CK(cudaMemcpyAsync(s.keep_out, s.map->d_keep.as<uint8_t>(), s.n_map_global, host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, h->stream));
    return ERASOR_OK;
}

// Enqueue one step on the handle's stream without waiting: copies, memsets, K1, K3, K2, the three concurrent K4 classes with the
// fold in their epilogue, the node inserts, the mask / counter read-back.  Once the batch geometry and the buffers are known this
// is a fixed launch sequence, so submit() captures it into a CUDA graph the first time and replays it afterwards (one launch
// instead of ~15 API calls).
int enqueue(erasor_ctx* h, const Step& s) {
    int rc;
    if ((rc = stage_host_clouds(h, s.ptr_kind, s.mode == 1 ? s.map_xyzi : nullptr, s.qry_xyzi, s.qry_xyz ? 3 * sizeof(float) : sizeof(float4)))) return rc;
    if (s.mode == 2) CK(cudaMemcpyAsync(h->d_poses.p(), h->h_pose.p(), sizeof(NodePose) * (size_t)h->F, cudaMemcpyHostToDevice, h->stream));
    if (s.n_keep) CK(cudaMemsetAsync(s.d_keep, 1, s.n_keep, h->stream));
    if (s.sweep) {
        for (const SweepGeo& sg : s.sweep->geo)
            CK(cudaMemsetAsync(sg.ssw.n_flagged, 0, sizeof(uint32_t) * kMaxSweepVariants * (size_t)h->F, h->stream));
        CK(cudaMemsetAsync(s.sweep->geo[0].ksw.rejected, 0, sizeof(uint32_t) * kMaxSweepVariants * (size_t)h->F, h->stream));
        if ((rc = run_sweep(h, *s.sweep, s.qry_xyz, s.with_c ? 7 : 3))) return rc;
    } else {
        if ((rc = run_k1(h, s.mode))) return rc;
        if ((rc = run_compare(h, h->p.version, s.mode, s.d_keep, nullptr, s.fold, s.with_c ? 7 : 3))) return rc;
    }
    if (s.inserts && (rc = run_insert_assemble(h))) return rc;      // (run_compare ran the plan and the query scatter under R-GPF)
    CK(cudaMemcpyAsync(h->h_words.as<uint32_t>() + 1, h->d_queue.as<uint32_t>() + kBucketC0, sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
    if ((rc = copy_masks_out(h, s))) return rc;
    CK(cudaMemcpyAsync(h->h_words.as<uint32_t>(), h->d_nrecs.p(), sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
    return ERASOR_OK;
}

// The graph of step s at the handle's current epochs: the cached one, or one captured now.  *out stays null when capture is not
// possible here, which turns graphs off for the handle.
int step_graph(erasor_ctx* h, const Step& s, const erasor_ctx::StepGraph** out) {
    *out = nullptr;
    for (const auto& g : h->graphs)
        if (g.desc_epoch == h->desc_epoch && g.alloc_epoch == h->alloc_epoch && same_step(g.step, s)) { *out = &g; return ERASOR_OK; }
    // drop graphs of older geometries, bound the cache
    for (size_t i = 0; i < h->graphs.size();) {
        if (h->graphs[i].desc_epoch != h->desc_epoch || h->graphs[i].alloc_epoch != h->alloc_epoch || h->graphs.size() > 64) { cudaGraphExecDestroy(h->graphs[i].exec); h->graphs.erase(h->graphs.begin() + i); }
        else ++i;
    }
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    const uint64_t launches_before = h->launches, alloc_epoch = h->alloc_epoch;
    CK(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeRelaxed));
    const int rc = enqueue(h, s);
    const uint64_t kernel_nodes = h->launches - launches_before;   // init, K1, K3, K2, K4 classes, inserts
    h->launches = launches_before;                                  // captured, not launched
    const cudaError_t ce = cudaStreamEndCapture(h->stream, &graph);
    if (rc == ERASOR_OK && ce == cudaSuccess && graph && h->alloc_epoch == alloc_epoch && cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess) {
        h->graphs.push_back({s, h->desc_epoch, alloc_epoch, exec, kernel_nodes});
        *out = &h->graphs.back();
    } else {
        cudaGetLastError();
        h->use_graphs = false;                                      // capture not possible here: plain launches for good
    }
    if (graph) cudaGraphDestroy(graph);
    return ERASOR_OK;
}

// Complete the caller's step (map_off / qry_off / F: the batch geometry; mode 2: poses [F] and the caller's poses7 of these
// frames) and enqueue it: as a replay of the graph captured from an equal step, a new capture, or plain launches.
int submit(erasor_ctx* h, Step st, const uint64_t* map_off, const uint64_t* qry_off, int F, const NodePose* poses = nullptr, const double* poses7 = nullptr) {
    int rc;
    CK(cudaSetDevice(h->device));
    if (h->pending && (rc = erasor_wait(h))) return rc;      // one submission in flight per handle (buffers and staging are reused)
    h->stage = 0;
    h->f0 = st.f0;
    if ((rc = prepare_batch(h, map_off, qry_off, F, st.mode))) return rc;
    if (st.mode == 1 && ((h->NM && !st.map_xyzi) || (h->NQ && !st.qry_xyzi))) { h->err = "null cloud"; return ERASOR_E_INVALID; }
    if (st.mode == 2 && h->NQ && !st.qry_xyzi) { h->err = "null cloud"; return ERASOR_E_INVALID; }
    st.inserts = inserts_on(h, st.mode);
    st.with_c = h->class_c_state != 0;
    const bool host = st.ptr_kind != ERASOR_PTR_DEVICE;
    if (st.mode == 2) {
        st.map = h->map; st.n_map_global = h->map->n; st.cur_map = h->map->d_pts.as<const float4>();
    } else if ((rc = device_cloud(h, h->d_map_in, st.map_xyzi, h->NM, st.ptr_kind, &st.cur_map))) {
        return rc;
    }
    if ((rc = device_cloud(h, h->d_qry_in, st.qry_xyzi, h->NQ, st.ptr_kind, &st.cur_qry, st.qry_xyz ? 3 * sizeof(float) : sizeof(float4)))) return rc;
    st.n_keep = st.user_keep ? h->NM : 0;
    if (st.n_keep) {
        if (host) CK(h->d_keep.ensure(st.n_keep));
        st.d_keep = host ? h->d_keep.as<uint8_t>() : st.user_keep;
    }
    if (st.mode == 2) {
        if (sizeof(NodePose) * (size_t)F > h->h_pose.cap()) h->alloc_epoch++;      // captured graphs copy from this staging buffer
        CK(h->h_pose.ensure(sizeof(NodePose) * (size_t)F));
        std::memcpy(h->h_pose.p(), poses, sizeof(NodePose) * (size_t)F);
    }
    if (st.inserts) {
        if ((rc = ensure_insert_buffers(h))) return rc;
        for (int f = 0; f < F; ++f) {
            Mat4 T;
            pose_to_mat(poses7 + 7 * (size_t)f, T);         // tf_body2origin_ = geoPose2eigen(odom), as body2origin applies it
            std::memcpy(h->h_ins_fwd.as<float>() + 12 * (size_t)f, T.m, sizeof(float) * 12);
        }
    }
    if (st.sweep) {
        // a sweep: one block of per-setting flag counters per geometry, records for the largest geometry; a plan that is not own
        // also bins every geometry into its batch tables (and a 32-warp launch into its own VoI lists) and runs class C up front
        // (the records of one geometry are gone once the next one has run)
        auto plan = std::make_shared<SweepPlan>(*st.sweep);
        const size_t n_geo = plan->geo.size(), n_chunks = (size_t)h->n_chunks_map + h->n_chunks_qry;
        if (!plan->own) {
            while (h->k1_sweep.size() < n_geo) h->k1_sweep.emplace_back(new erasor_ctx::K1Bufs(h->alloc_epoch));
            for (size_t g = 0; g < n_geo; ++g) {
                if ((rc = ensure_k1_bufs(h, *h->k1_sweep[g], h->NM, h->NQ, n_chunks, (size_t)F, (size_t)plan->geo[g].t->B))) return rc;
                const K1Lists lists = k1_lists(h, plan.get(), (int)g);     // (an 8-warp launch's are prepare_batch's, sized already)
                CK(lists.idx.ensure(sizeof(uint32_t) * (h->NM + kIdPad)));
                CK(lists.cnt.ensure(sizeof(uint32_t) * kListWarps * std::max<size_t>(n_chunks, 1)));
            }
            st.with_c = true;
        }
        const uint32_t recs = (uint32_t)std::min<size_t>((size_t)F * plan->B_max, kMaxRecords);
        if (recs > h->rec_capacity) {
            CK(h->d_recs.ensure(sizeof(FlagRec) * (size_t)recs));
            CK(h->d_bucket.ensure(sizeof(uint32_t) * (size_t)kNumBuckets * recs));
            h->rec_capacity = recs;
        }
        const size_t rows = (size_t)kMaxSweepVariants * (size_t)std::max(h->stat_F, h->f0 + F);
        CK(h->d_sweep_flag.ensure(sizeof(uint32_t) * rows * n_geo));
        CK(h->d_sweep_rej.ensure(sizeof(uint32_t) * rows));
        for (size_t g = 0; g < n_geo; ++g) {
            plan->geo[g].ssw.n_flagged = h->d_sweep_flag.as<uint32_t>() + rows * g + (size_t)kMaxSweepVariants * st.f0;
            plan->geo[g].ksw.rejected = h->d_sweep_rej.as<uint32_t>() + (size_t)kMaxSweepVariants * st.f0;
            plan->geo[g].ksw.n = (uint32_t)st.n_map_global;
        }
        st.sweep = plan;
    } else if (st.mode == 2) {
        st.fold = K4Fold{h->map->d_keep.as<uint8_t>(), nullptr, (uint32_t)st.n_map_global, 0u};   // a sweep leaves the map's mask alone
    }
    h->last = st;                                            // erasor_wait and erasor_profile_k1 read the step that ran, replayed or not
    h->cur_map = st.cur_map; h->cur_qry = st.cur_qry;
    bool graphable = h->use_graphs && !h->timing;
    if (graphable && host) {
        // host buffers must be pinned for copies to be capturable
        if (st.mode == 1 && h->NM && !is_pinned_host(st.map_xyzi)) graphable = false;
        if (h->NQ && !is_pinned_host(st.qry_xyzi)) graphable = false;
        if (st.n_keep && !is_pinned_host(st.user_keep)) graphable = false;
        if (st.keep_out && st.n_map_global && !is_pinned_host(st.keep_out)) graphable = false;
    }
    const erasor_ctx::StepGraph* g = nullptr;
    if (graphable && (rc = step_graph(h, st, &g))) return rc;
    if (g) {
        CK(cudaGraphLaunch(g->exec, h->stream));
        h->launches += g->kernel_nodes;
    } else {
        Scope whole(h, 0);
        if ((rc = enqueue(h, st))) return rc;
    }
    h->pending = true;
    return ERASOR_OK;
}

// frames [f0, f1) that fit one submission: < 2^32 points per side and at most kMaxRecords flagged-bin records
int sub_batch_end(const erasor_ctx* h, const uint64_t* map_off, const uint64_t* qry_off, int f0, int F) {
    const uint64_t lim = 0xFFFFFFF0ull;
    const int max_frames = (int)std::max<size_t>(1, kMaxRecords / (size_t)h->B);
    int f1 = f0;
    while (f1 < F && f1 - f0 < max_frames && map_off[f1 + 1] - map_off[f0] < lim && qry_off[f1 + 1] - qry_off[f0] < lim) ++f1;
    return f1;
}

int process_frames_impl(erasor_handle_t h, const float* map_xyzi, const uint64_t* map_offsets, const float* query_xyzi,
                        const uint64_t* query_offsets, int n_frames, uint8_t* keep_mask, int ptr_kind,
                        const uint32_t* fold_index, uint8_t* fold_global, size_t fold_n_global, bool async) {
    if (!h || !map_offsets || !query_offsets || !keep_mask) { if (h) h->err = "null argument"; return ERASOR_E_INVALID; }
    if (n_frames <= 0) { h->err = "n_frames must be positive"; return ERASOR_E_INVALID; }
    const bool qxyz = (ptr_kind & ERASOR_PTR_QUERY_XYZ) != 0;
    ptr_kind &= ~ERASOR_PTR_QUERY_XYZ;
    if (ptr_kind != ERASOR_PTR_HOST && ptr_kind != ERASOR_PTR_DEVICE) { h->err = "bad ptr_kind"; return ERASOR_E_INVALID; }
    int rc;
    if (h->pending && (rc = erasor_wait(h))) return rc;
    h->stat_F = n_frames;
    h->sweep_V = 0;
    h->ins_call_off.clear();                   // the inserts of an earlier node call end with this submission
    std::vector<uint64_t> mo, qo;
    for (int f0 = 0; f0 < n_frames;) {
        const int f1 = sub_batch_end(h, map_offsets, query_offsets, f0, n_frames);
        if (f1 == f0) { h->err = "a single frame exceeds 2^32 points"; return ERASOR_E_INVALID; }
        const uint64_t m0 = map_offsets[f0], q0 = query_offsets[f0];
        const uint64_t *mof = map_offsets, *qof = query_offsets;
        if (f0 != 0 || f1 != n_frames) {
            mo.assign(map_offsets + f0, map_offsets + f1 + 1); qo.assign(query_offsets + f0, query_offsets + f1 + 1);
            for (auto& v : mo) v -= m0;
            for (auto& v : qo) v -= q0;
            mof = mo.data(); qof = qo.data();
        }
        Step st;
        st.mode = 1; st.ptr_kind = ptr_kind; st.qry_xyz = qxyz; st.f0 = f0;
        st.map_xyzi = map_xyzi ? map_xyzi + 4 * m0 : nullptr;
        st.qry_xyzi = query_xyzi ? query_xyzi + (qxyz ? 3 : 4) * q0 : nullptr;
        st.user_keep = keep_mask + m0;
        if (fold_global) st.fold = K4Fold{fold_global, fold_index ? fold_index + m0 : nullptr, (uint32_t)std::min<size_t>(fold_n_global, 0xFFFFFFFFu), 0u};
        if ((rc = submit(h, st, mof, qof, f1 - f0))) return rc;
        f0 = f1;
        if (f0 < n_frames && (rc = erasor_wait(h))) return rc;      // the next sub-batch reuses the handle's buffers
    }
    return async ? ERASOR_OK : erasor_wait(h);
}

// |map_voi_| of every node of the last submission = binned + complement counts of the map cloud (K1's tables), into out[0, F)
// (after a sweep: the tables of any of its geometries hold them; those of geometry 0 are read)
int read_node_voi_counts(erasor_handle_t h, uint32_t* out) {
    const K1GeoTables t = k1_tables(h, h->last.mode == 2 ? h->last.sweep.get() : nullptr, 0);
    const size_t row = (size_t)t.B + 1;
    std::vector<uint32_t> c((size_t)h->F * row);
    CK(cudaMemcpy(c.data(), t.cnt, sizeof(uint32_t) * c.size(), cudaMemcpyDeviceToHost));
    for (int f = 0; f < h->F; ++f) {
        uint64_t t = 0;
        for (size_t b = 0; b < row; ++b) t += c[(size_t)f * row + b];
        out[f] = (uint32_t)t;
    }
    return ERASOR_OK;
}

// extents (nullable, n_frames entries): frame f scans only the prefix [0, extents[f]) of the attached map (a re-test map's nodes,
// erasor_process_nodes_retest); without them every frame scans the whole map
int process_nodes_impl(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                       double voi_max_range, uint8_t* frame_keep, uint8_t* keep_out, int ptr_kind, bool async,
                       std::shared_ptr<const SweepPlan> sweep = nullptr, const uint64_t* extents = nullptr) {
    if (!h || !poses7 || !query_offsets) { if (h) h->err = "null argument"; return ERASOR_E_INVALID; }
    if (!h->map) { h->err = "erasor_process_nodes: no map attached (erasor_attach_map)"; return ERASOR_E_STATE; }
    if (n_frames <= 0) { h->err = "n_frames must be positive"; return ERASOR_E_INVALID; }
    const bool qxyz = (ptr_kind & ERASOR_PTR_QUERY_XYZ) != 0;
    ptr_kind &= ~ERASOR_PTR_QUERY_XYZ;
    if (ptr_kind != ERASOR_PTR_HOST && ptr_kind != ERASOR_PTR_DEVICE) { h->err = "bad ptr_kind"; return ERASOR_E_INVALID; }
    if (qxyz && h->node_inserts) {
        h->err = "node inserts carry the query's intensity: packed x y z queries (ERASOR_PTR_QUERY_XYZ) need erasor_set_node_inserts(h, 0)";
        return ERASOR_E_INVALID;
    }
    int rc;
    if (!sweep || sweep->own) {                                    // (any other sweep plan: process_nodes_sweep checks its launches)
        const erasor_geometry_t x = own_geometry(h->p);
        if ((rc = node_k1_fits(h, "node mode", x, k1_smem_bytes(x.num_rings, h->B), false, false))) return rc;
    }
    if (h->pending && (rc = erasor_wait(h))) return rc;
    const size_t N = h->map->n;
    const double range = voi_max_range > 0.0 ? voi_max_range : h->p.max_range;
    h->stat_F = n_frames;
    h->sweep_V = sweep ? sweep->geo[0].ssw.n : 0;
    h->ins_call_off.assign(h->node_inserts ? 1 : 0, 0);
    // scratch per (frame, map point): bin id 2 + scattered point 16 + source index 4 + class-C scratch 24 bytes; with inserts also
    // R-GPF's partitioned copy 16 + the inserts 16 + K4b's voxels 16 and scratch 36 bytes
    size_t budget = (size_t)16 << 30;
    if (const char* e = std::getenv("ERASOR_B200_NODE_SCRATCH_GB")) budget = (size_t)std::max(1.0, std::atof(e)) << 30;
    // (a sweep plan that is not own: also per geometry its bin id 2 bytes and its chunk count rows, at most 4 (B + 1) / (5 B) bytes,
    // and the VoI lists of its 32-warp K1 launches 4 bytes)
    const size_t per_point = (h->node_inserts ? 130 : 46) + (sweep && !sweep->own ? 3 * sweep->geo.size() + 4 : 0);
    const size_t by_mem = std::max<size_t>(1, budget / (per_point * std::max<size_t>(N, 1)));
    const size_t by_idx = std::max<size_t>(1, (size_t)0xFFFFFFF0ull / std::max<size_t>(N, 1) - 1);
    const size_t B_max = sweep ? (size_t)std::max(h->B, sweep->B_max) : (size_t)h->B;
    const int max_frames = (int)std::min<size_t>({by_mem, by_idx, std::max<size_t>(1, kMaxRecords / B_max), (size_t)n_frames});
    std::vector<uint64_t> mo, qo;
    std::vector<NodePose> poses;
    for (int f0 = 0; f0 < n_frames;) {
        int f1 = f0;
        // with inserts, the scattered query and map points of a sub-batch index one array (K4b's voxels, the inserts)
        auto fits = [&](int f) { return query_offsets[f + 1] - query_offsets[f0] < 0xFFFFFFF0ull &&
                                        (!h->node_inserts || (uint64_t)(f + 1 - f0) * N + (query_offsets[f + 1] - query_offsets[f0]) < 0xFFFFFFF0ull); };
        while (f1 < n_frames && f1 - f0 < max_frames && fits(f1)) ++f1;
        if (f1 == f0) { h->err = "a single query exceeds 2^32 points"; return ERASOR_E_INVALID; }
        const int F = f1 - f0;
        // each frame's map side is its own range of the bin-id / scatter arrays, the map read from index 0 (prepare_batch, mode 2)
        mo.assign((size_t)F + 1, 0);
        for (int f = 0; f < F; ++f) mo[f + 1] = mo[f] + (extents ? extents[f0 + f] : N);
        const uint64_t q0 = query_offsets[f0];
        qo.assign(query_offsets + f0, query_offsets + f1 + 1);
        for (auto& v : qo) v -= q0;
        poses.resize(F);
        for (int f = 0; f < F; ++f) node_pose_of(poses7 + 7 * (size_t)(f0 + f), range, poses[f]);
        Step st;
        st.mode = 2; st.ptr_kind = ptr_kind; st.qry_xyz = qxyz; st.f0 = f0;
        st.qry_xyzi = query_xyzi ? query_xyzi + (qxyz ? 3 : 4) * q0 : nullptr;
        st.user_keep = frame_keep ? frame_keep + (size_t)f0 * N : nullptr;
        st.keep_out = (f1 == n_frames) ? keep_out : nullptr;
        st.sweep = sweep;
        if ((rc = submit(h, st, mo.data(), qo.data(), F, poses.data(), poses7 + 7 * (size_t)f0))) return rc;
        if (f1 < n_frames) {                                         // the next sub-batch reuses the handle's buffers
            if ((rc = erasor_wait(h))) return rc;
            h->node_nvoi.resize((size_t)f1);
            if ((rc = read_node_voi_counts(h, h->node_nvoi.data() + f0))) return rc;
        }
        f0 = f1;
    }
    return async ? ERASOR_OK : erasor_wait(h);
}
}  // namespace

int erasor_wait(erasor_handle_t h) {
    if (!h) return ERASOR_E_INVALID;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    if (h->pending) {
        h->pending = false;
        h->n_recs_host = h->words()[0];
        h->class_c_count_host = h->words()[1];
        if (h->n_recs_host > h->rec_capacity) { h->err = "internal: flagged-bin records overflowed the work queue"; return ERASOR_E_CAPACITY; }
        h->class_c_state = (int)std::min<uint32_t>(h->class_c_count_host, 0x7FFFFFFFu);
        const Step& s = h->last;
        if (!s.with_c && h->class_c_count_host > 0) {
            // bins beyond class B's capacity turned up in a submission that ran without class C: run that class now (R-GPF only; the
            // bins are independent, the masks only gain zeros), then repeat the output copies.  The next submissions launch it up front.
            // (A sweep that gets here has an own plan, whose geometry 0 is the handle's: the others launch class C up front.)
            int rc = run_k4(h, s.mode, s.d_keep, nullptr, s.fold, 4, s.sweep ? &s.sweep->geo[0].ksw : nullptr);
            if (rc) return rc;
            if (s.inserts && (rc = run_insert_assemble(h))) return rc;
            if ((rc = copy_masks_out(h, s))) return rc;
            CK(cudaStreamSynchronize(h->stream));
        }
        if (s.inserts) return collect_inserts(h);
    }
    return ERASOR_OK;
}

int erasor_process_frames(erasor_handle_t h, const float* map_xyzi, const uint64_t* map_offsets, const float* query_xyzi,
                          const uint64_t* query_offsets, int n_frames, uint8_t* keep_mask, int ptr_kind) {
    return process_frames_impl(h, map_xyzi, map_offsets, query_xyzi, query_offsets, n_frames, keep_mask, ptr_kind, nullptr, nullptr, 0, false);
}
int erasor_process_frames_async(erasor_handle_t h, const float* map_xyzi, const uint64_t* map_offsets, const float* query_xyzi,
                                const uint64_t* query_offsets, int n_frames, uint8_t* keep_mask, int ptr_kind) {
    return process_frames_impl(h, map_xyzi, map_offsets, query_xyzi, query_offsets, n_frames, keep_mask, ptr_kind, nullptr, nullptr, 0, true);
}

int erasor_process_frames_fold(erasor_handle_t h, const float* map_xyzi, const uint64_t* map_offsets, const float* query_xyzi,
                               const uint64_t* query_offsets, int n_frames, uint8_t* keep_mask, int ptr_kind,
                               const uint32_t* voi_index, uint8_t* global_keep, size_t n_global) {
    if (!h) return ERASOR_E_INVALID;
    if (!voi_index || !global_keep) { h->err = "null fold argument"; return ERASOR_E_INVALID; }
    return process_frames_impl(h, map_xyzi, map_offsets, query_xyzi, query_offsets, n_frames, keep_mask, ptr_kind, voi_index, global_keep, n_global, false);
}
int erasor_process_frames_fold_async(erasor_handle_t h, const float* map_xyzi, const uint64_t* map_offsets, const float* query_xyzi,
                                     const uint64_t* query_offsets, int n_frames, uint8_t* keep_mask, int ptr_kind,
                                     const uint32_t* voi_index, uint8_t* global_keep, size_t n_global) {
    if (!h) return ERASOR_E_INVALID;
    if (!voi_index || !global_keep) { h->err = "null fold argument"; return ERASOR_E_INVALID; }
    return process_frames_impl(h, map_xyzi, map_offsets, query_xyzi, query_offsets, n_frames, keep_mask, ptr_kind, voi_index, global_keep, n_global, true);
}

// Multi-GPU exchange helper (DESIGN.md section 7): fold per-frame keep masks onto the global map
// (global_keep[voi_index[i]] = 0 where keep[i] == 0).  Accumulates; all pointers are DEVICE pointers; asynchronous on the
// handle's stream.  (erasor_process_frames_fold / erasor_process_nodes do this inside R-GPF's epilogue instead.)
int erasor_fold_keep_masks(erasor_handle_t h, const uint8_t* keep_mask, const uint32_t* voi_index, size_t n, uint8_t* global_keep, size_t n_global) {
    if (!h || !global_keep || (n && (!keep_mask || !voi_index))) { if (h) h->err = "null argument"; return ERASOR_E_INVALID; }
    if (n_global > 0xFFFFFFFFull) { h->err = "global map beyond 2^32 points"; return ERASOR_E_INVALID; }
    CK(cudaSetDevice(h->device));
    if (n) h->launches++;
    CK(launch_fold_keep(h->stream, keep_mask, voi_index, n, global_keep, n_global));
    return ERASOR_OK;
}

int erasor_reset_keep_mask(erasor_handle_t h, uint8_t* global_keep, size_t n_global) {
    if (!h || (n_global && !global_keep)) { if (h) h->err = "null argument"; return ERASOR_E_INVALID; }
    CK(cudaSetDevice(h->device));
    if (n_global) h->launches++;
    CK(launch_fill_u8(h->stream, global_keep, n_global, 1));
    return ERASOR_OK;
}

// ---- map-resident mode -------------------------------------------------------------------------------------------
int erasor_map_create(const float* map_xyzi, size_t n_map, int ptr_kind, int device, erasor_map_t* out) {
    if (!out || (n_map && !map_xyzi)) { g_create_error = "null argument"; return ERASOR_E_INVALID; }
    *out = nullptr;
    if (n_map >= 0xFFFFFFF0ull) { g_create_error = "map beyond 2^32 points"; return ERASOR_E_INVALID; }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) { g_create_error = "no CUDA device (this library has no CPU path)"; return ERASOR_E_CUDA; }
    if (device < 0 || device >= ndev) { g_create_error = "bad device index"; return ERASOR_E_INVALID; }
    erasor_map_ctx* m = new erasor_map_ctx();
    m->device = device; m->n = n_map;
    auto fail = [&](const char* what, cudaError_t ce) { g_create_error = std::string(what) + ": " + cudaGetErrorString(ce); erasor_map_destroy(m); return ERASOR_E_CUDA; };
    if ((e = cudaSetDevice(device)) != cudaSuccess) return fail("cudaSetDevice", e);
    if ((e = cudaStreamCreateWithFlags(&m->st, cudaStreamNonBlocking)) != cudaSuccess) return fail("cudaStreamCreate", e);
    if ((e = m->d_pts.allocate(sizeof(float4) * (n_map + kMapPad))) != cudaSuccess) return fail("cudaMalloc", e);
    if ((e = cudaMemsetAsync(m->d_pts.as<float4>() + n_map, 0, sizeof(float4) * kMapPad, m->st)) != cudaSuccess) return fail("cudaMemset", e);
    if ((e = m->d_keep.allocate(std::max<size_t>(n_map, 1))) != cudaSuccess) return fail("cudaMalloc", e);
    if (n_map) {
        const cudaMemcpyKind k = ptr_kind == ERASOR_PTR_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
        if ((e = cudaMemcpyAsync(m->d_pts.p(), map_xyzi, sizeof(float4) * n_map, k, m->st)) != cudaSuccess) return fail("cudaMemcpy", e);
        if ((e = cudaMemsetAsync(m->d_keep.as<uint8_t>(), 1, n_map, m->st)) != cudaSuccess) return fail("cudaMemset", e);
    }
    if ((e = cudaStreamSynchronize(m->st)) != cudaSuccess) return fail("cudaStreamSynchronize", e);
    *out = m;
    return ERASOR_OK;
}

void erasor_map_destroy(erasor_map_t m) {
    if (!m) return;
    cudaSetDevice(m->device);
    if (m->st) { cudaStreamSynchronize(m->st); cudaStreamDestroy(m->st); }
    delete m;
}

size_t erasor_map_size(erasor_map_t m) { return m ? m->n : 0; }
uint8_t* erasor_map_keep_device(erasor_map_t m) { return m ? m->d_keep.as<uint8_t>() : nullptr; }
const float* erasor_map_points_device(erasor_map_t m) { return m ? m->d_pts.as<const float>() : nullptr; }

int erasor_map_reset_keep(erasor_map_t m) {
    if (!m) return ERASOR_E_INVALID;
    if (cudaSetDevice(m->device) != cudaSuccess) return ERASOR_E_CUDA;
    if (m->n && cudaMemsetAsync(m->d_keep.as<uint8_t>(), 1, m->n, m->st) != cudaSuccess) return ERASOR_E_CUDA;
    return cudaStreamSynchronize(m->st) == cudaSuccess ? ERASOR_OK : ERASOR_E_CUDA;
}

int erasor_map_get_keep(erasor_map_t m, uint8_t* keep, int ptr_kind) {
    if (!m || (m->n && !keep)) return ERASOR_E_INVALID;
    if (cudaSetDevice(m->device) != cudaSuccess) return ERASOR_E_CUDA;
    const cudaMemcpyKind k = ptr_kind == ERASOR_PTR_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    if (m->n && cudaMemcpyAsync(keep, m->d_keep.as<uint8_t>(), m->n, k, m->st) != cudaSuccess) return ERASOR_E_CUDA;
    return cudaStreamSynchronize(m->st) == cudaSuccess ? ERASOR_OK : ERASOR_E_CUDA;
}

int erasor_attach_map(erasor_handle_t h, erasor_map_t m) {
    if (!h) return ERASOR_E_INVALID;
    if (m && m->device != h->device) { h->err = "map and handle live on different devices"; return ERASOR_E_INVALID; }
    int rc;
    if (h->pending && (rc = erasor_wait(h))) return rc;
    h->map = m;
    h->desc_mode = -1;
    return ERASOR_OK;
}

int erasor_process_nodes(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                         double voi_max_range, uint8_t* frame_keep, uint8_t* keep_out, int ptr_kind) {
    return process_nodes_impl(h, poses7, query_xyzi, query_offsets, n_frames, voi_max_range, frame_keep, keep_out, ptr_kind, false);
}
int erasor_process_nodes_async(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                               double voi_max_range, uint8_t* frame_keep, uint8_t* keep_out, int ptr_kind) {
    return process_nodes_impl(h, poses7, query_xyzi, query_offsets, n_frames, voi_max_range, frame_keep, keep_out, ptr_kind, true);
}

extern "C++" {
namespace {
// pass 2 of the node-mode re-test (DESIGN.md section 8.4.1): the plain node path with each frame's map side cut to its node's extent
int process_nodes_retest(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                         int first_node, double voi_max_range, uint8_t* keep_out, int ptr_kind, bool async) {
    if (!h) return ERASOR_E_INVALID;
    if (!poses7 || !query_offsets) { h->err = "null argument"; return ERASOR_E_INVALID; }
    if (!h->map) { h->err = "erasor_process_nodes_retest: no map attached (erasor_attach_map)"; return ERASOR_E_STATE; }
    if (h->pending) { h->err = "erasor_process_nodes_retest while a submission is pending (erasor_wait first)"; return ERASOR_E_STATE; }
    if (!h->map->retest) { h->err = "erasor_process_nodes_retest: the attached map was not made by erasor_map_create_retest"; return ERASOR_E_INVALID; }
    if (h->node_inserts) { h->err = "the re-test pass has no node inserts: erasor_set_node_inserts(h, 0) first"; return ERASOR_E_INVALID; }
    const size_t n_nodes = h->map->extents.size();
    if (n_frames <= 0 || first_node < 0 || (size_t)first_node + (size_t)n_frames > n_nodes) {
        h->err = "erasor_process_nodes_retest: nodes [first_node, first_node + n_frames) must lie in [0, " + std::to_string(n_nodes) + ")";
        return ERASOR_E_INVALID;
    }
    return process_nodes_impl(h, poses7, query_xyzi, query_offsets, n_frames, voi_max_range, nullptr, keep_out, ptr_kind, async, nullptr,
                              h->map->extents.data() + first_node);
}
}  // namespace
}  // extern "C++"

int erasor_process_nodes_retest(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                                int first_node, double voi_max_range, uint8_t* keep_out, int ptr_kind) {
    return process_nodes_retest(h, poses7, query_xyzi, query_offsets, n_frames, first_node, voi_max_range, keep_out, ptr_kind, false);
}
int erasor_process_nodes_retest_async(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                                      int first_node, double voi_max_range, uint8_t* keep_out, int ptr_kind) {
    return process_nodes_retest(h, poses7, query_xyzi, query_offsets, n_frames, first_node, voi_max_range, keep_out, ptr_kind, true);
}

extern "C++" {   // (a template and overloads: C++ linkage)
namespace {
// Every sweep entry point's settings as erasor_process_nodes_tune takes them: erasor_process_nodes_sweep's with the handle's
// geometry and ground-filter fields, erasor_process_nodes_sweep_ex's with the handle's geometry
erasor_tune_setting_t widen(const erasor_ctx*, const erasor_tune_setting_t& x) { return x; }
erasor_tune_setting_t widen(const erasor_ctx* h, const erasor_sweep_setting_t& x) { return erasor_tune_setting_t{own_geometry(h->p), x}; }
erasor_tune_setting_t widen(const erasor_ctx* h, const erasor_srt_variant_t& x) {
    return widen(h, erasor_sweep_setting_t{x.scan_ratio_threshold, x.th_bin_max_h, h->p.gf_dist_thr, h->p.gf_th_seeds_height, x.minimum_num_pts,
                                           h->p.num_lowest_pts, h->p.gf_num_lpr, h->p.gf_iter});
}

// The sweeps' one path (fn: the entry point, for the messages): the settings' checks, then their plan.  The settings are split by
// geometry (first appearance order); per geometry their Scan Ratio Test fields go to K2 and their ground-filter fields are grouped
// for K4 (one GpfParams per distinct tuple, in order of first appearance, with the settings that carry it).  The plan is own when
// every setting carries the handle's geometry.  Otherwise its geometries are packed into K1 launches of at most 56 KB of tables, so
// that every launch keeps the four 8-warp CTAs per SM of the plain kernel (a geometry beyond that runs alone in the 32-warp form,
// as it would in a plain call).
template <class Setting>
int process_nodes_sweep(erasor_handle_t h, const char* fn, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets,
                        int n_frames, double voi_max_range, const Setting* settings, int n_settings, uint8_t* variant_keep, int ptr_kind, bool async) {
    if (!h) return ERASOR_E_INVALID;
    if (n_settings < 1 || n_settings > kMaxSweepVariants) { h->err = "n_variants must be in [1, 32]"; return ERASOR_E_INVALID; }
    if (!settings || !variant_keep) { h->err = "null variants or variant_keep"; return ERASOR_E_INVALID; }
    erasor_tune_setting_t x[kMaxSweepVariants];
    for (int v = 0; v < n_settings; ++v) x[v] = widen(h, settings[v]);
    for (int v = 0; v < n_settings; ++v)
        if (x[v].s.gf_iter > kMaxIter) { h->err = "gf_iter above the tap capacity (8)"; return ERASOR_E_UNSUPPORTED; }
    if (!h->map) { h->err = std::string(fn) + ": no map attached (erasor_attach_map)"; return ERASOR_E_INVALID; }
    if (h->node_inserts) { h->err = "a sweep has no node inserts: erasor_set_node_inserts(h, 0) first"; return ERASOR_E_INVALID; }
    if (h->pending) { h->err = std::string(fn) + " while a submission is pending (erasor_wait first)"; return ERASOR_E_STATE; }
    double range = voi_max_range;
    if (!(range > 0.0)) {
        for (int v = 1; v < n_settings; ++v)
            if (x[v].geometry.max_range != x[0].geometry.max_range) {
                h->err = "voi_max_range <= 0 takes the settings' max_range, and they differ: pass the VoI radius";
                return ERASOR_E_INVALID;
            }
        range = x[0].geometry.max_range;
    }
    CK(cudaSetDevice(h->device));
    auto plan = std::make_shared<SweepPlan>();
    int geo_of[kMaxSweepVariants];
    for (int v = 0; v < n_settings; ++v) {
        size_t g = 0;
        while (g < plan->geo.size() && !same_geometry(plan->geo[g].t->key, x[v].geometry)) ++g;
        if (g == plan->geo.size()) {
            const GeoTables* t = nullptr;
            int rc = geometry_tables(h, x[v].geometry, &t);
            if (rc) return rc;
            plan->geo.push_back(SweepGeo{t, 0, {}, {}});
            plan->B_max = std::max(plan->B_max, t->B);
        }
        geo_of[v] = (int)g;
    }
    plan->own = plan->geo.size() == 1 && plan->geo[0].t == h->geo_tables[0].get();
    for (int g = 0; g < (int)plan->geo.size(); ++g) {
        // the settings of geometry g; the others take part with no bin flagged
        SweepGeo& sg = plan->geo[g];
        sg.ssw.n = n_settings;
        sg.ksw.keep = variant_keep;
        for (int v = 0; v < n_settings; ++v) {
            const erasor_sweep_setting_t& s = x[v].s;
            sg.ssw.v[v] = SrtVariant{s.scan_ratio_threshold, s.th_bin_max_h, geo_of[v] == g ? s.minimum_num_pts : -1, 0};
            if (geo_of[v] != g) continue;
            GpfParams gp{};
            gp.th_dist = s.gf_dist_thr; gp.th_seeds = s.gf_th_seeds_height; gp.num_lowest_pts = s.num_lowest_pts;
            gp.num_lpr = s.gf_num_lpr; gp.iters = s.gf_iter; gp.cov_mode = h->p.cov_mode;
            int k = 0;
            while (k < sg.ksw.n_groups && std::memcmp(&sg.ksw.gp[k], &gp, sizeof(GpfParams)) != 0) ++k;
            if (k == sg.ksw.n_groups) sg.ksw.gp[sg.ksw.n_groups++] = gp;
            sg.ksw.bits[k] |= 1u << v;
        }
        if (plan->own) continue;
        // K1 packing
        const size_t bytes = k1_geo_smem_bytes(sg.t->view.R, sg.t->B);
        if (g == 0 || h->tune_unpacked || k1_warps(plan->launch_smem.back() + bytes) == 32) {
            plan->launch_begin.push_back(g);
            plan->launch_smem.push_back(0);
        }
        sg.launch = (int)plan->launch_smem.size() - 1;
        plan->launch_smem.back() += bytes;
    }
    if (!plan->own) plan->launch_begin.push_back((int)plan->geo.size());
    for (size_t l = 0; l < plan->launch_smem.size(); ++l) {      // (a launch beyond 56 KB holds one geometry)
        const int rc = node_k1_fits(h, fn, plan->geo[plan->launch_begin[l]].t->key, plan->launch_smem[l], true, false);
        if (rc) return rc;
    }
    return process_nodes_impl(h, poses7, query_xyzi, query_offsets, n_frames, range, nullptr, nullptr, ptr_kind, async, plan);
}
}  // namespace
}  // extern "C++"

int erasor_process_nodes_sweep(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                               double voi_max_range, const erasor_srt_variant_t* variants, int n_variants, uint8_t* variant_keep, int ptr_kind) {
    return process_nodes_sweep(h, "erasor_process_nodes_sweep", poses7, query_xyzi, query_offsets, n_frames, voi_max_range, variants, n_variants,
                               variant_keep, ptr_kind, false);
}
int erasor_process_nodes_sweep_async(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                                     double voi_max_range, const erasor_srt_variant_t* variants, int n_variants, uint8_t* variant_keep, int ptr_kind) {
    return process_nodes_sweep(h, "erasor_process_nodes_sweep", poses7, query_xyzi, query_offsets, n_frames, voi_max_range, variants, n_variants,
                               variant_keep, ptr_kind, true);
}
int erasor_process_nodes_sweep_ex(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                                  double voi_max_range, const erasor_sweep_setting_t* settings, int n_settings, uint8_t* variant_keep, int ptr_kind) {
    return process_nodes_sweep(h, "erasor_process_nodes_sweep_ex", poses7, query_xyzi, query_offsets, n_frames, voi_max_range, settings, n_settings,
                               variant_keep, ptr_kind, false);
}
int erasor_process_nodes_sweep_ex_async(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                                        double voi_max_range, const erasor_sweep_setting_t* settings, int n_settings, uint8_t* variant_keep, int ptr_kind) {
    return process_nodes_sweep(h, "erasor_process_nodes_sweep_ex", poses7, query_xyzi, query_offsets, n_frames, voi_max_range, settings, n_settings,
                               variant_keep, ptr_kind, true);
}

int erasor_process_nodes_tune(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                              double voi_max_range, const erasor_tune_setting_t* settings, int n_settings, uint8_t* variant_keep, int ptr_kind) {
    return process_nodes_sweep(h, "erasor_process_nodes_tune", poses7, query_xyzi, query_offsets, n_frames, voi_max_range, settings, n_settings,
                               variant_keep, ptr_kind, false);
}
int erasor_process_nodes_tune_async(erasor_handle_t h, const double* poses7, const float* query_xyzi, const uint64_t* query_offsets, int n_frames,
                                    double voi_max_range, const erasor_tune_setting_t* settings, int n_settings, uint8_t* variant_keep, int ptr_kind) {
    return process_nodes_sweep(h, "erasor_process_nodes_tune", poses7, query_xyzi, query_offsets, n_frames, voi_max_range, settings, n_settings,
                               variant_keep, ptr_kind, true);
}

int erasor_get_sweep_stats(erasor_handle_t h, uint32_t* n_flagged_bins, uint32_t* n_rejected_points) {
    if (!h) return ERASOR_E_INVALID;
    if (h->sweep_V <= 0 || h->desc_mode != 2) { h->err = "no erasor_process_nodes_sweep call has run"; return ERASOR_E_STATE; }
    int rc;
    if ((rc = erasor_wait(h))) return rc;
    const size_t F = (size_t)h->stat_F, V = (size_t)h->sweep_V;
    // the flag counters: one block per geometry of the plan, each setting counted in its own geometry's block only
    const size_t rows = (size_t)kMaxSweepVariants * F, G = h->last.sweep ? h->last.sweep->geo.size() : 1;
    std::vector<uint32_t> t(rows * G);
    for (int k = 0; k < 2; ++k) {
        uint32_t* out = k == 0 ? n_flagged_bins : n_rejected_points;
        if (!out) continue;
        const size_t blocks = k == 0 ? G : 1;
        CK(cudaMemcpy(t.data(), (k == 0 ? h->d_sweep_flag : h->d_sweep_rej).p(), sizeof(uint32_t) * rows * blocks, cudaMemcpyDeviceToHost));
        for (size_t v = 0; v < V; ++v)
            for (size_t f = 0; f < F; ++f) {
                uint32_t c = 0;
                for (size_t g = 0; g < blocks; ++g) c += t[g * rows + f * kMaxSweepVariants + v];
                out[v * F + f] = c;
            }
    }
    return ERASOR_OK;
}

// voxelize_preserving_labels of n_clouds clouds in one submission (voxelize_batch.cu): the checks that need only the host arrays
int erasor_voxelize_batch(erasor_handle_t h, const float* xyzi, const uint64_t* offsets, int n_clouds, const uint8_t* keep, float leaf,
                          const double* pose7, int ptr_kind, const float** d_out, uint64_t* out_offsets) {
    if (!h) return ERASOR_E_INVALID;
    h->err.clear();
    if (!offsets || !d_out || !out_offsets) { h->err = "null argument"; return ERASOR_E_INVALID; }
    if (n_clouds < 1) { h->err = "n_clouds must be at least 1"; return ERASOR_E_INVALID; }
    if (ptr_kind != ERASOR_PTR_HOST && ptr_kind != ERASOR_PTR_DEVICE) { h->err = "ptr_kind must be ERASOR_PTR_HOST or ERASOR_PTR_DEVICE"; return ERASOR_E_INVALID; }
    if (!(leaf > 0.0f) || !std::isfinite(leaf)) { h->err = "leaf must be positive and finite"; return ERASOR_E_INVALID; }
    if (offsets[0] != 0) { h->err = "offsets[0] must be 0 (offsets[n_clouds] is the point count)"; return ERASOR_E_INVALID; }
    for (int c = 0; c < n_clouds; ++c)
        if (offsets[c + 1] < offsets[c]) { h->err = "offsets are not monotone at cloud " + std::to_string(c); return ERASOR_E_INVALID; }
    for (int c = 0; c < n_clouds; ++c)
        if (offsets[c + 1] - offsets[c] >= (1ull << 31)) { h->err = "cloud " + std::to_string(c) + " has 2^31 points or more"; return ERASOR_E_CAPACITY; }
    const uint64_t n = offsets[n_clouds];
    if (n >= 0xFFFFFFFFull) { h->err = "a call takes fewer than 2^32 - 1 points"; return ERASOR_E_CAPACITY; }
    if (n && !xyzi) { h->err = "null cloud pointer"; return ERASOR_E_INVALID; }
    if (ptr_kind == ERASOR_PTR_DEVICE && (reinterpret_cast<uintptr_t>(xyzi) & 15u)) { h->err = "a device cloud must be 16-byte aligned (one float4 per point)"; return ERASOR_E_INVALID; }
    CK(cudaSetDevice(h->device));
    Mat4 T{};
    if (pose7) {
        // as the updater's tf_lidar2body_ (set_params, OfflineMapUpdater.cpp:89-104): geoPose2eigen(pose) * Identity
        Mat4 G, I{};
        for (int i = 0; i < 4; ++i) I.m[i * 5] = 1.0f;
        pose_to_mat(pose7, G);
        mat_mul(G, I, T);
    }
    if (!h->vb) h->vb = vox_batch_create();
    return vox_batch_run(h->vb, h->stream, xyzi, offsets, n_clouds, keep, leaf, pose7 ? T.m : nullptr, ptr_kind == ERASOR_PTR_DEVICE, d_out,
                         out_offsets, h->launches, h->err);
}

int erasor_get_node_stats(erasor_handle_t h, uint32_t* n_voi_points, uint32_t* n_flagged_bins, uint32_t* n_rejected_points) {
    if (!h) return ERASOR_E_INVALID;
    if (h->F <= 0 || h->desc_mode != 2) { h->err = "no node batch has run"; return ERASOR_E_STATE; }
    int rc;
    if ((rc = erasor_wait(h))) return rc;
    if (n_voi_points) {
        // earlier sub-batches of the call were counted before the next one overwrote the tables; the last one is read here
        std::copy(h->node_nvoi.begin(), h->node_nvoi.begin() + std::min<size_t>(h->node_nvoi.size(), (size_t)h->f0), n_voi_points);
        if ((rc = read_node_voi_counts(h, n_voi_points + h->f0))) return rc;
    }
    if (n_flagged_bins) CK(cudaMemcpy(n_flagged_bins, h->d_nflag.p(), sizeof(uint32_t) * h->stat_F, cudaMemcpyDeviceToHost));
    if (n_rejected_points) CK(cudaMemcpy(n_rejected_points, h->d_frame_rej.p(), sizeof(uint32_t) * h->stat_F, cudaMemcpyDeviceToHost));
    return ERASOR_OK;
}

int erasor_set_node_inserts(erasor_handle_t h, int enable) {
    if (!h) return ERASOR_E_INVALID;
    if (h->pending) { h->err = "erasor_set_node_inserts while a submission is pending (erasor_wait first)"; return ERASOR_E_STATE; }
    h->node_inserts = enable != 0;
    h->ins_call_off.clear();
    return ERASOR_OK;
}

int erasor_get_node_inserts(erasor_handle_t h, const float** d_xyzi, uint64_t* offsets) {
    if (!h) return ERASOR_E_INVALID;
    if (!d_xyzi || !offsets) { h->err = "null argument"; return ERASOR_E_INVALID; }
    int rc;
    if ((rc = erasor_wait(h))) return rc;
    if (!h->node_inserts || h->ins_call_off.size() != (size_t)h->stat_F + 1) {
        h->err = "no erasor_process_nodes call with inserts on has completed"; return ERASOR_E_STATE;
    }
    *d_xyzi = h->d_ins_call.as<const float>();
    std::copy(h->ins_call_off.begin(), h->ins_call_off.end(), offsets);
    return ERASOR_OK;
}

int erasor_map_append_inserts(erasor_map_t m, erasor_handle_t h) {
    if (!h) return ERASOR_E_INVALID;
    if (!m) { h->err = "null map"; return ERASOR_E_INVALID; }
    if (m->device != h->device) { h->err = "map and handle live on different devices"; return ERASOR_E_INVALID; }
    CK(cudaSetDevice(h->device));
    int rc;
    if ((rc = erasor_wait(h))) return rc;
    if (!h->node_inserts || h->ins_call_off.size() != (size_t)h->stat_F + 1) {
        h->err = "no erasor_process_nodes call with inserts on has completed"; return ERASOR_E_STATE;
    }
    const size_t n = h->ins_call_off.back();
    CK(grow_points(m->d_ins, m->n_ins, m->n_ins + n, h->stream));
    if (n) CK(cudaMemcpyAsync(m->d_ins.as<float4>() + m->n_ins, h->d_ins_call.p(), sizeof(float4) * n, cudaMemcpyDeviceToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    m->ins_node_off.pop_back();                // (the old end: the first appended node's start)
    for (size_t f = 0; f < h->ins_call_off.size(); ++f) m->ins_node_off.push_back(m->n_ins + h->ins_call_off[f]);
    m->n_ins += n;
    return ERASOR_OK;
}

int erasor_map_inserts(erasor_map_t m, const float** d_xyzi, size_t* n) {
    if (!m || !d_xyzi || !n) return ERASOR_E_INVALID;
    *d_xyzi = m->d_ins.as<const float>();
    *n = m->n_ins;
    return ERASOR_OK;
}

int erasor_map_clear_inserts(erasor_map_t m) {
    if (!m) return ERASOR_E_INVALID;
    m->n_ins = 0;
    m->ins_node_off.assign(1, 0);
    return ERASOR_OK;
}

// The re-test map (DESIGN.md section 8.4.1): m's kept points compacted in map order on the device, then m's insert store, with
// kMapPad zeroed points of slack as erasor_map_create leaves them; one read of the kept count sizes it.  Node k of the store sees the
// prefix of the map that holds m's kept points and the inserts of the nodes before k.
int erasor_map_create_retest(erasor_map_t m, erasor_map_t* out) {
    if (!m || !out) { g_create_error = "null argument"; return ERASOR_E_INVALID; }
    *out = nullptr;
    erasor_map_ctx* r = new erasor_map_ctx();
    r->device = m->device;
    cudaError_t e;
    auto fail = [&](const char* what, cudaError_t ce) { g_create_error = std::string(what) + ": " + cudaGetErrorString(ce); erasor_map_destroy(r); return ERASOR_E_CUDA; };
    if ((e = cudaSetDevice(m->device)) != cudaSuccess) return fail("cudaSetDevice", e);
    if ((e = cudaStreamCreateWithFlags(&r->st, cudaStreamNonBlocking)) != cudaSuccess) return fail("cudaStreamCreate", e);
    if ((e = cudaStreamSynchronize(m->st)) != cudaSuccess) return fail("cudaStreamSynchronize", e);
    const size_t tiles = compact_tiles(m->n);
    DeviceBuffer d_tiles;                      // per tile its kept count and its offset, then the kept total
    if ((e = d_tiles.allocate(sizeof(uint32_t) * (2 * tiles + 1))) != cudaSuccess) return fail("cudaMalloc", e);
    uint32_t* tile_cnt = d_tiles.as<uint32_t>();
    uint32_t* tile_off = tile_cnt + tiles;
    uint32_t* d_total = tile_off + tiles;
    if ((e = launch_compact_count(r->st, m->d_keep.as<const uint8_t>(), m->n, tile_cnt, tile_off, d_total)) != cudaSuccess) return fail("k_compact_count", e);
    uint32_t n_kept = 0;
    if ((e = cudaMemcpyAsync(&n_kept, d_total, sizeof(uint32_t), cudaMemcpyDeviceToHost, r->st)) != cudaSuccess) return fail("cudaMemcpy", e);
    if ((e = cudaStreamSynchronize(r->st)) != cudaSuccess) return fail("cudaStreamSynchronize", e);
    const size_t n = (size_t)n_kept + m->n_ins;
    if (n >= 0xFFFFFFF0ull) { g_create_error = "re-test map beyond 2^32 points"; erasor_map_destroy(r); return ERASOR_E_INVALID; }
    r->n = n;
    if ((e = r->d_pts.allocate(sizeof(float4) * (n + kMapPad))) != cudaSuccess) return fail("cudaMalloc", e);
    if ((e = r->d_keep.allocate(std::max<size_t>(n, 1))) != cudaSuccess) return fail("cudaMalloc", e);
    if ((e = launch_compact_scatter(r->st, m->d_pts.as<const float4>(), m->d_keep.as<const uint8_t>(), m->n, tile_off, r->d_pts.as<float4>())) != cudaSuccess)
        return fail("k_compact_scatter", e);
    if (m->n_ins && (e = cudaMemcpyAsync(r->d_pts.as<float4>() + n_kept, m->d_ins.p(), sizeof(float4) * m->n_ins, cudaMemcpyDeviceToDevice, r->st)) != cudaSuccess)
        return fail("cudaMemcpy", e);
    if ((e = cudaMemsetAsync(r->d_pts.as<float4>() + n, 0, sizeof(float4) * kMapPad, r->st)) != cudaSuccess) return fail("cudaMemset", e);
    if (n && (e = cudaMemsetAsync(r->d_keep.p(), 1, n, r->st)) != cudaSuccess) return fail("cudaMemset", e);
    if ((e = cudaStreamSynchronize(r->st)) != cudaSuccess) return fail("cudaStreamSynchronize", e);
    r->retest = true;
    r->extents.resize(m->ins_node_off.size() - 1);
    for (size_t k = 0; k < r->extents.size(); ++k) r->extents[k] = n_kept + m->ins_node_off[k];
    *out = r;
    return ERASOR_OK;
}

int erasor_map_retest_extents(erasor_map_t m, size_t* n_nodes, uint64_t* extents) {
    if (!m || !n_nodes || !m->retest) return ERASOR_E_INVALID;
    *n_nodes = m->extents.size();
    if (extents) std::copy(m->extents.begin(), m->extents.end(), extents);
    return ERASOR_OK;
}

// node mode's save_static_map: voxelize_preserving_labels(map[keep] ++ the map's inserts, leaf), one erasor_voxelize_batch cloud
int erasor_save_node_map(erasor_handle_t h, erasor_map_t m, float leaf, const float** d_out, size_t* n_out) {
    if (!h) return ERASOR_E_INVALID;
    if (!m || !d_out || !n_out) { h->err = "null argument"; return ERASOR_E_INVALID; }
    if (m->device != h->device) { h->err = "map and handle live on different devices"; return ERASOR_E_INVALID; }
    CK(cudaSetDevice(h->device));
    int rc;
    if ((rc = erasor_wait(h))) return rc;
    const size_t n = m->n + m->n_ins;
    const float* pts = m->d_pts.as<const float>();
    const uint8_t* keep = m->d_keep.as<const uint8_t>();
    if (m->n_ins) {
        CK(h->d_save.ensure(sizeof(float4) * n));
        CK(h->d_save_keep.ensure(n));
        CK(cudaMemcpyAsync(h->d_save.p(), m->d_pts.p(), sizeof(float4) * m->n, cudaMemcpyDeviceToDevice, h->stream));
        CK(cudaMemcpyAsync(h->d_save.as<float4>() + m->n, m->d_ins.p(), sizeof(float4) * m->n_ins, cudaMemcpyDeviceToDevice, h->stream));
        if (m->n) CK(cudaMemcpyAsync(h->d_save_keep.p(), m->d_keep.p(), m->n, cudaMemcpyDeviceToDevice, h->stream));
        CK(cudaMemsetAsync(h->d_save_keep.as<uint8_t>() + m->n, 1, m->n_ins, h->stream));
        pts = h->d_save.as<const float>();
        keep = h->d_save_keep.as<const uint8_t>();
    }
    const uint64_t off[2] = {0, n};
    uint64_t out_off[2] = {0, 0};
    if ((rc = erasor_voxelize_batch(h, pts, off, 1, keep, leaf, nullptr, ERASOR_PTR_DEVICE, d_out, out_off))) return rc;
    *n_out = out_off[1];
    return ERASOR_OK;
}

// ---- the path's single collective ---------------------------------------------------------------------------------
int erasor_comm_unique_id(uint8_t* id128) {
    if (!id128) return ERASOR_E_INVALID;
    NcclApi* api = nccl_api(g_create_error);
    if (!api) return ERASOR_E_UNSUPPORTED;
    static_assert(sizeof(ncclUniqueId) == ERASOR_COMM_ID_BYTES, "NCCL unique id size");
    ncclUniqueId id;
    const ncclResult_t r = api->GetUniqueId(&id);
    if (r != ncclSuccess) { g_create_error = std::string("ncclGetUniqueId: ") + api->GetErrorString(r); return ERASOR_E_CUDA; }
    std::memcpy(id128, &id, sizeof(id));
    return ERASOR_OK;
}

int erasor_comm_init(erasor_handle_t h, const uint8_t* id128, int n_ranks, int rank) {
    if (!h || !id128 || n_ranks < 1 || rank < 0 || rank >= n_ranks) { if (h) h->err = "bad communicator arguments"; return ERASOR_E_INVALID; }
    NcclApi* api = nccl_api(h->err);
    if (!api) return ERASOR_E_UNSUPPORTED;
    CK(cudaSetDevice(h->device));
    if (h->comm) { api->CommDestroy(h->comm); h->comm = nullptr; }
    ncclUniqueId id;
    std::memcpy(&id, id128, sizeof(id));
    const ncclResult_t r = api->CommInitRank(&h->comm, n_ranks, id, rank);
    if (r != ncclSuccess) { h->comm = nullptr; h->err = std::string("ncclCommInitRank: ") + api->GetErrorString(r); return ERASOR_E_CUDA; }
    h->comm_ranks = n_ranks; h->comm_rank = rank;
    return ERASOR_OK;
}

int erasor_comm_destroy(erasor_handle_t h) {
    if (!h) return ERASOR_E_INVALID;
    if (h->comm) {
        NcclApi* api = nccl_api(h->err);
        if (!api) return ERASOR_E_UNSUPPORTED;
        CK(cudaSetDevice(h->device));
        CK(cudaStreamSynchronize(h->stream));
        api->CommDestroy(h->comm);
        h->comm = nullptr; h->comm_ranks = 1; h->comm_rank = 0;
    }
    return ERASOR_OK;
}

// The local half of the exchange on its own (what runs after the all-gather): AND n_masks byte masks of n points each
// (DEVICE, contiguous [n_masks][n]) through the bit-packed form into out (DEVICE, n bytes).  Lets a single-GPU test and
// a caller with its own transport use the library's pack / AND kernels.
int erasor_and_keep_masks(erasor_handle_t h, const uint8_t* masks, int n_masks, size_t n, uint8_t* out) {
    if (!h || n_masks < 1 || (n && (!masks || !out))) { if (h) h->err = "bad argument"; return ERASOR_E_INVALID; }
    if (n == 0) return ERASOR_OK;
    CK(cudaSetDevice(h->device));
    const size_t words = (n + 31) / 32;
    CK(h->d_gather.ensure(sizeof(uint32_t) * words * (size_t)n_masks));
    for (int r = 0; r < n_masks; ++r) {
        h->launches++;
        CK(launch_pack_keep_bits(h->stream, masks + (size_t)r * n, n, h->d_gather.as<uint32_t>() + (size_t)r * words));
    }
    h->launches++;
    CK(launch_and_unpack_keep(h->stream, h->d_gather.as<uint32_t>(), n_masks, n, out));
    return ERASOR_OK;
}

int erasor_allgather_and_keep(erasor_handle_t h, uint8_t* global_keep, size_t n_global) {
    if (!h || (n_global && !global_keep)) { if (h) h->err = "null argument"; return ERASOR_E_INVALID; }
    if (!h->comm || h->comm_ranks <= 1 || n_global == 0) return ERASOR_OK;      // one rank: the folded mask is already the answer
    NcclApi* api = nccl_api(h->err);
    if (!api) return ERASOR_E_UNSUPPORTED;
    CK(cudaSetDevice(h->device));
    const size_t words = (n_global + 31) / 32;
    CK(h->d_pack.ensure(sizeof(uint32_t) * words));
    CK(h->d_gather.ensure(sizeof(uint32_t) * words * (size_t)h->comm_ranks));
    h->launches += 2;
    CK(launch_pack_keep_bits(h->stream, global_keep, n_global, h->d_pack.as<uint32_t>()));
    const ncclResult_t r = api->AllGather(h->d_pack.p(), h->d_gather.p(), words, ncclUint32, h->comm, h->stream);
    if (r != ncclSuccess) { h->err = std::string("ncclAllGather: ") + api->GetErrorString(r); return ERASOR_E_CUDA; }
    CK(launch_and_unpack_keep(h->stream, h->d_gather.as<uint32_t>(), h->comm_ranks, n_global, global_keep));
    return ERASOR_OK;
}

int erasor_get_frame_stats(erasor_handle_t h, uint32_t* n_flagged_bins, uint32_t* n_rejected_points) {
    if (!h) return ERASOR_E_INVALID;
    if (h->F <= 0) { h->err = "no batch has run"; return ERASOR_E_STATE; }
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    const int nf = std::max(h->stat_F, h->F);
    if (n_flagged_bins) CK(cudaMemcpy(n_flagged_bins, h->d_nflag.p(), sizeof(uint32_t) * nf, cudaMemcpyDeviceToHost));
    if (n_rejected_points) CK(cudaMemcpy(n_rejected_points, h->d_frame_rej.p(), sizeof(uint32_t) * nf, cudaMemcpyDeviceToHost));
    return ERASOR_OK;
}

// instrumentation: per flagged bin of the last run, n_points and the SM cycles thread 0 spent per phase
// (load + index sort, z sort, seeds, accumulate, SVD + plane, classify + compact, outputs) and the Jacobi sweep count
int erasor_get_rgpf_profile(erasor_handle_t h, uint32_t* n_points, uint32_t* prof8, size_t* n) {
    if (!h || !n) return ERASOR_E_INVALID;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    uint32_t nr = 0;
    CK(cudaMemcpy(&nr, h->d_nrecs.p(), sizeof(uint32_t), cudaMemcpyDeviceToHost));
    nr = std::min(nr, h->rec_capacity);
    const size_t cap = *n;
    *n = nr;
    if (!n_points && !prof8) return ERASOR_OK;
    if (cap < nr) { h->err = "profile buffer too small"; return ERASOR_E_CAPACITY; }
    std::vector<FlagRec> recs(nr);
    if (nr) CK(cudaMemcpy(recs.data(), h->d_recs.p(), sizeof(FlagRec) * nr, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < nr; ++i) {
        if (n_points) n_points[i] = recs[i].n_points;
        if (prof8) for (int k = 0; k < 8; ++k) prof8[i * 8 + k] = recs[i].prof[k];
    }
    return ERASOR_OK;
}

// instrumentation: K1 of the last node-mode batch again, as its profiling build.  It rebuilds the per-frame tables and lists that
// batch's K1 built (with the same values); the outputs of the later kernels are left as they are.
int erasor_profile_k1(erasor_handle_t h, uint32_t* out, size_t* n, int* warps_per_cta) {
    if (!h || !n) return ERASOR_E_INVALID;
    if (h->desc_mode != 2 || !h->cur_map) { h->err = "no node-mode batch has run"; return ERASOR_E_STATE; }
    CK(cudaSetDevice(h->device));
    int rc;
    if (h->pending && (rc = erasor_wait(h))) return rc;
    const int nw = k1_lists(h, nullptr, 0).warps;
    const size_t words = (size_t)(h->n_chunks_map + h->n_chunks_qry) * nw * kK1ProfSlots;
    const size_t cap = *n;
    *n = words;
    if (warps_per_cta) *warps_per_cta = nw;
    if (!out) return ERASOR_OK;
    if (cap < words) { h->err = "profile buffer too small"; return ERASOR_E_CAPACITY; }
    if ((rc = node_k1_fits(h, "erasor_profile_k1", own_geometry(h->p), k1_smem_bytes(h->p.num_rings, h->B), false, true))) return rc;
    CK(h->d_k1prof.ensure(sizeof(uint32_t) * std::max<size_t>(words, 1)));
    h->k1_prof = h->d_k1prof.as<uint32_t>();
    rc = run_k1(h, 2);
    h->k1_prof = nullptr;
    if (rc) return rc;
    CK(cudaStreamSynchronize(h->stream));
    CK(cudaMemcpy(out, h->d_k1prof.p(), sizeof(uint32_t) * words, cudaMemcpyDeviceToHost));
    return ERASOR_OK;
}

int erasor_get_srt_profile(erasor_handle_t h, uint32_t* cycles8) {
    if (!h || !cycles8) return ERASOR_E_INVALID;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    if (!h->d_queue.p()) { h->err = "no run yet"; return ERASOR_E_STATE; }
    CK(cudaMemcpy(cycles8, h->d_queue.as<uint32_t>() + 20, sizeof(uint32_t) * 8, cudaMemcpyDeviceToHost));
    return ERASOR_OK;
}

uint64_t erasor_kernel_launch_count(erasor_handle_t h) { return h ? h->launches : 0; }

int erasor_forget_run_history(erasor_handle_t h) {
    if (!h) return ERASOR_E_INVALID;
    h->class_c_state = -1;
    return ERASOR_OK;
}

int erasor_reset_kernel_times(erasor_handle_t h, int enable_timing) {
    if (!h) return ERASOR_E_INVALID;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    drain_timers(h);
    for (auto& t : h->timers) { t.total_ms = 0; t.launches = 0; }
    h->timing = enable_timing != 0;
    return ERASOR_OK;
}

int erasor_get_kernel_time_ms(erasor_handle_t h, int kernel_id, double* total_ms, uint64_t* launches) {
    if (!h || kernel_id < 0 || kernel_id >= kNumTimers) return ERASOR_E_INVALID;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    drain_timers(h);
    if (total_ms) *total_ms = h->timers[kernel_id].total_ms;
    if (launches) *launches = h->timers[kernel_id].launches;
    return ERASOR_OK;
}

}  // extern "C"
