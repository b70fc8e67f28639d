// voxelize_batch.cu -- erasor_voxelize_batch: erasor_utils::voxelize_preserving_labels (erasor_utils.cpp:80-114) of F clouds in
// one submission, each cloud on its own pcl::VoxelGrid, then optionally one pcl::transformPointCloud (DESIGN.md section 8.3).
// Within a cloud the result is bit-identical to oracle voxelize(cloud[keep], leaf) (followed by oracle transform).  The arithmetic
// is device_common.cuh's single copy (voxel_grid_setup, voxel_key_of, voxel_centroid, voxel_grid_nn, pcl_affine).
//
//   k_vb_init         per-cloud statistics and voxel counters reset
//   k_vb_bounds       segmented getMinMax3D of the selected points of all clouds in one pass (order-preserving encodings), the
//                     selected count per cloud and the lowest index of a selected point with a non-finite x, y or z
//   k_vb_setup        per cloud: voxel_grid_setup from the cloud's own bounds, overflow decision
//   k_vb_keys         voxel key per point (0xFFFFFFFF for a deselected point; an overflowing cloud: the point's index in its cloud)
//   radix             stable LSD passes (radix_sort.h): 4 over the voxel key, then over the cloud index (at least one pass)
//   k_vb_cloud_keys   between the two: sorted position -> its cloud (F for a deselected point, which keeps them last)
//   k_vb_rekey        sorted position -> its voxel key again
//   k_vb_heads_*      run heads of (cloud, key) -> voxel key, first position and cloud per voxel; voxels per cloud
//   k_vb_offsets      exclusive scan of the voxels per cloud: the output offsets
//   k_vb_voxels       per voxel: centroid in cloud order, exact 1-NN label among the cloud's selected points, optional affine
//
// The launch count depends only on the cloud-index digits (ceil(bits(F) / 8), at least 1): nothing waits for the host until the
// one read-back of the output offsets at the end.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <string>

#include "../../include/erasor_b200.h"
#include "buffers.h"
#include "device_common.cuh"
#include "radix_sort.h"
#include "voxelize_batch.h"

namespace erasor {

constexpr int      kVbThreads = 256;
constexpr int      kVbWarps   = kVbThreads / 32;
constexpr uint32_t kVbRows    = 64;            // rows of 32 points per warp of the bounds pass
constexpr uint32_t kVbChunk   = 4096;          // sorted positions per CTA of the run-head count and scatter
constexpr uint32_t kVbNoKey   = 0xFFFFFFFFu;   // voxel key of a deselected point: sorts behind every cell key
constexpr uint32_t kVbNone    = 0xFFFFFFFFu;
constexpr int      kVbKeyPasses = 4;           // 8-bit passes over the 32-bit voxel key

// The kernels' parameter types stay outside the anonymous namespace, so the kernels' symbol names are stable.
struct VbCloud {
    uint32_t mn[3], mx[3];        // float_to_ordered min / max of the cloud's selected finite points
    uint32_t n_sel;               // selected points
    uint32_t overflow;            // the grid overflows int32 ("Leaf size is too small"): every selected point is its own voxel
    VoxelGridDims g;
};

// the call's scalars; the F + 1 voxel counts / output offsets follow them in the same buffer, so one copy reads back both
struct VbHead {
    uint32_t bad;                 // lowest index of a selected point with a non-finite x, y or z (kVbNone: none)
    uint32_t n_sel;               // selected points of all clouds
    uint32_t nv;                  // voxels of all clouds
    uint32_t pad_;
};

struct VbAffine { float m[12]; };

namespace {

// the cloud of point i: the last c with off[c] <= i (empty clouds before it are passed over); off[F] > i
__device__ __forceinline__ uint32_t vb_cloud_of(const uint32_t* __restrict__ off, int F, uint32_t i) {
    int lo = 0, hi = F;
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (off[mid] <= i) lo = mid; else hi = mid; }
    return (uint32_t)lo;
}

__device__ __forceinline__ bool vb_finite3(float4 p) { return isfinite(p.x) && isfinite(p.y) && isfinite(p.z); }

// a warp's running bounds of cloud `cur` into the cloud's statistics (whole warp, warp-uniform arguments)
__device__ __forceinline__ void vb_flush(VbCloud* __restrict__ cl, int cur, uint32_t (&mn)[3], uint32_t (&mx)[3], uint32_t& sel) {
    const uint32_t s = __reduce_add_sync(FULL_MASK, sel);
    uint32_t a[3], b[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { a[k] = __reduce_min_sync(FULL_MASK, mn[k]); b[k] = __reduce_max_sync(FULL_MASK, mx[k]); }
    if ((threadIdx.x & 31) == 0 && cur >= 0 && s) {
        atomicAdd(&cl[cur].n_sel, s);
        for (int k = 0; k < 3; ++k) { atomicMin(&cl[cur].mn[k], a[k]); atomicMax(&cl[cur].mx[k], b[k]); }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) { mn[k] = 0xFFFFFFFFu; mx[k] = 0u; }
    sel = 0u;
}

}  // namespace

__global__ void __launch_bounds__(kVbThreads) k_vb_init(VbCloud* __restrict__ cl, int F, VbHead* __restrict__ hd, uint32_t* __restrict__ vcnt) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < F) {
        VbCloud z{};
        for (int k = 0; k < 3; ++k) { z.mn[k] = 0xFFFFFFFFu; z.mx[k] = 0u; }
        cl[c] = z;
    }
    if (c <= F) vcnt[c] = 0u;
    if (c == 0) { hd->bad = kVbNone; hd->n_sel = 0u; hd->nv = 0u; hd->pad_ = 0u; }
}

// One warp per run of kVbRows x 32 consecutive points.  A row whose points all belong to one cloud is folded into the warp's
// running bounds (flushed when the cloud changes); a row that straddles clouds (at most one per cloud boundary) goes point by point.
__global__ void __launch_bounds__(kVbThreads) k_vb_bounds(const float4* __restrict__ pts, const uint8_t* __restrict__ keep, uint32_t n,
                                                          const uint32_t* __restrict__ off, int F, VbCloud* __restrict__ cl,
                                                          VbHead* __restrict__ hd) {
    const int lane = threadIdx.x & 31;
    const uint64_t b0 = ((uint64_t)blockIdx.x * kVbWarps + (threadIdx.x >> 5)) * 32ull * kVbRows;
    int cur = -1;
    uint32_t mn[3] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu}, mx[3] = {0u, 0u, 0u}, sel = 0u, bad = kVbNone;
    for (uint32_t r = 0; r < kVbRows; ++r) {
        const uint64_t r0 = b0 + 32ull * r;
        if (r0 >= n) break;                                           // warp-uniform
        const bool in = r0 + lane < n;
        const uint32_t i = (uint32_t)(r0 + lane);
        const int c = in ? (int)vb_cloud_of(off, F, i) : -1;
        const int c0 = __shfl_sync(FULL_MASK, c, 0);
        const bool uni = __all_sync(FULL_MASK, !in || c == c0);
        if (!uni || c0 != cur) { vb_flush(cl, cur, mn, mx, sel); cur = uni ? c0 : -1; }
        if (!in || (keep && !keep[i])) continue;
        const float4 p = pts[i];
        const bool fin = vb_finite3(p);
        if (!fin) bad = min(bad, i);
        const uint32_t o[3] = {float_to_ordered(p.x + 0.0f), float_to_ordered(p.y + 0.0f), float_to_ordered(p.z + 0.0f)};   // -0 -> +0
        if (uni) {
            ++sel;
            if (fin) for (int k = 0; k < 3; ++k) { mn[k] = min(mn[k], o[k]); mx[k] = max(mx[k], o[k]); }
        } else {
            atomicAdd(&cl[c].n_sel, 1u);
            if (fin) for (int k = 0; k < 3; ++k) { atomicMin(&cl[c].mn[k], o[k]); atomicMax(&cl[c].mx[k], o[k]); }
        }
    }
    vb_flush(cl, cur, mn, mx, sel);
    bad = __reduce_min_sync(FULL_MASK, bad);
    if (lane == 0 && bad != kVbNone) atomicMin(&hd->bad, bad);
}

__global__ void __launch_bounds__(kVbThreads) k_vb_setup(VbCloud* __restrict__ cl, int F, float leaf, VbHead* __restrict__ hd) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t s = 0u;
    if (c < F) {
        s = cl[c].n_sel;
        if (s) {
            float mn[3], mx[3];
            for (int k = 0; k < 3; ++k) { mn[k] = ordered_to_float(cl[c].mn[k]); mx[k] = ordered_to_float(cl[c].mx[k]); }
            bool ovf;
            unsigned long long cells;
            cl[c].g = voxel_grid_setup(mn, mx, leaf, ovf, cells);
            cl[c].overflow = ovf ? 1u : 0u;
        }
    }
    s = __reduce_add_sync(FULL_MASK, s);
    if ((threadIdx.x & 31) == 0 && s) atomicAdd(&hd->n_sel, s);
}

__global__ void __launch_bounds__(kVbThreads) k_vb_keys(const float4* __restrict__ pts, const uint8_t* __restrict__ keep, uint32_t n,
                                                        const uint32_t* __restrict__ off, int F, const VbCloud* __restrict__ cl,
                                                        uint32_t* __restrict__ key, uint32_t* __restrict__ idx) {
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
        const uint32_t i = (uint32_t)e;
        uint32_t k = kVbNoKey;
        if (!keep || keep[i]) {
            const uint32_t c = vb_cloud_of(off, F, i);
            if (cl[c].overflow) {
                k = i - off[c];
            } else {
                const float4 p = pts[i];      // inside the cloud's [mn, mx]: every cell lies in [0, div)
                k = voxel_key_of(cl[c].g, p.x, p.y, p.z);
            }
        }
        key[i] = k;
        idx[i] = i;
    }
}

__global__ void __launch_bounds__(kVbThreads) k_vb_cloud_keys(const uint8_t* __restrict__ keep, uint32_t n, const uint32_t* __restrict__ off,
                                                              int F, const uint32_t* __restrict__ idx, uint32_t* __restrict__ key) {
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
        const uint32_t i = idx[e];
        key[e] = (keep && !keep[i]) ? (uint32_t)F : vb_cloud_of(off, F, i);
    }
}

__global__ void __launch_bounds__(kVbThreads) k_vb_rekey(const float4* __restrict__ pts, uint32_t n, const uint32_t* __restrict__ off,
                                                         const VbCloud* __restrict__ cl, const VbHead* __restrict__ hd,
                                                         const uint32_t* __restrict__ scl, const uint32_t* __restrict__ idx,
                                                         uint32_t* __restrict__ skey) {
    const uint32_t ns = hd->n_sel;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < ns; e += (size_t)gridDim.x * blockDim.x) {
        const uint32_t c = scl[e], i = idx[e];
        if (cl[c].overflow) { skey[e] = i - off[c]; continue; }
        const float4 p = pts[i];
        skey[e] = voxel_key_of(cl[c].g, p.x, p.y, p.z);
    }
}

namespace {
__device__ __forceinline__ bool vb_head(const uint32_t* __restrict__ skey, const uint32_t* __restrict__ scl, uint32_t i) {
    return i == 0 || skey[i] != skey[i - 1] || scl[i] != scl[i - 1];
}
}  // namespace

__global__ void __launch_bounds__(kVbThreads) k_vb_heads_count(const uint32_t* __restrict__ skey, const uint32_t* __restrict__ scl,
                                                               const VbHead* __restrict__ hd, uint32_t* __restrict__ chunk) {
    __shared__ uint32_t s_w[kVbWarps];
    const uint32_t ns = hd->n_sel;
    const uint32_t b0 = blockIdx.x * kVbChunk, b1 = (uint32_t)min((unsigned long long)ns, (unsigned long long)b0 + kVbChunk);
    uint32_t c = 0u;
    for (uint32_t i = b0 + threadIdx.x; i < b1; i += kVbThreads) c += vb_head(skey, scl, i) ? 1u : 0u;
    c = __reduce_add_sync(FULL_MASK, c);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0u;
        for (int w = 0; w < kVbWarps; ++w) t += s_w[w];
        chunk[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(1024) k_vb_heads_scan(uint32_t* __restrict__ chunk, uint32_t nch, VbHead* __restrict__ hd) {
    __shared__ uint32_t s_part[34];
    const uint32_t t = block_excl_scan(chunk, chunk, (int)nch, s_part);
    if (threadIdx.x == 0) hd->nv = t;
}

__global__ void __launch_bounds__(kVbThreads) k_vb_heads_scatter(const uint32_t* __restrict__ skey, const uint32_t* __restrict__ scl,
                                                                 const uint32_t* __restrict__ chunk, const VbHead* __restrict__ hd,
                                                                 uint32_t* __restrict__ vkey, uint32_t* __restrict__ vstart,
                                                                 uint32_t* __restrict__ vcloud, uint32_t* __restrict__ vcnt) {
    __shared__ uint32_t s_w[kVbWarps];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t ns = hd->n_sel;
    const uint32_t b0 = blockIdx.x * kVbChunk, b1 = (uint32_t)min((unsigned long long)ns, (unsigned long long)b0 + kVbChunk);
    uint32_t base = chunk[blockIdx.x];
    for (uint32_t o0 = b0; o0 < b1; o0 += kVbThreads) {          // block-uniform bounds
        const uint32_t i = o0 + threadIdx.x;
        const bool h = i < b1 && vb_head(skey, scl, i);
        const unsigned bal = __ballot_sync(FULL_MASK, h);
        __syncthreads();                                          // s_w may still be read from the previous round
        if (lane == 0) s_w[warp] = __popc(bal);
        __syncthreads();
        uint32_t before = 0u, round = 0u;
        for (int w = 0; w < kVbWarps; ++w) { const uint32_t c = s_w[w]; if (w < warp) before += c; round += c; }
        if (h) {
            const uint32_t r = base + before + __popc(bal & ((1u << lane) - 1u)), c = scl[i];
            vkey[r] = skey[i]; vstart[r] = i; vcloud[r] = c;
            const unsigned peers = __match_any_sync(bal, c);
            if (lane == __ffs(peers) - 1) atomicAdd(&vcnt[c], (uint32_t)__popc(peers));
        }
        base += round;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) vstart[hd->nv] = ns;
}

// voxels per cloud -> output offsets, in place (F + 1 entries: the last count is 0, so the last offset is the total)
__global__ void __launch_bounds__(1024) k_vb_offsets(uint32_t* __restrict__ vcnt, int F) {
    __shared__ uint32_t s_part[34];
    block_excl_scan(vcnt, vcnt, F + 1, s_part);
}

// One thread per voxel.  The 1-NN of a cloud whose grid overflows (every selected point its own voxel, in cloud order) is the
// lowest index at distance 0 from the point, found by a scan of the cloud's points from its first: slow, exact, and only the
// threads of such clouds take it.
__global__ void __launch_bounds__(kVbThreads) k_vb_voxels(const float4* __restrict__ pts, const uint32_t* __restrict__ order,
                                                          const uint32_t* __restrict__ vstart, const uint32_t* __restrict__ vkey,
                                                          const uint32_t* __restrict__ vcloud, const VbCloud* __restrict__ cl,
                                                          const VbHead* __restrict__ hd, const uint32_t* __restrict__ out_off, VbAffine T,
                                                          int xform, float4* __restrict__ out) {
    if (hd->bad != kVbNone) return;                   // a non-finite centroid would send the 1-NN through 4096 shells
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= hd->nv) return;
    const uint32_t c = vcloud[v], base = out_off[c], nvc = out_off[c + 1] - base;
    float4 cen = voxel_centroid(pts, order, vstart[v], vstart[v + 1]);
    uint32_t best = kNoPoint;
    if (!cl[c].overflow) {
        best = voxel_grid_nn(pts, order, vstart + base, vkey + base, nvc, cl[c].g, cen);
    } else {
        for (uint32_t u = base; u < base + nvc; ++u) {
            const uint32_t j = order[vstart[u]];
            const float4 p = pts[j];
            const float dx = FS(cen.x, p.x), dy = FS(cen.y, p.y), dz = FS(cen.z, p.z);
            if (FA(FA(FM(dx, dx), FM(dy, dy)), FM(dz, dz)) == 0.0f) { best = j; break; }
        }
    }
    if (best != kNoPoint) cen.w = pts[best].w;
    out[v] = xform ? pcl_affine(T.m, cen) : cen;
}

// ============================================================================================================================
// host side
// ============================================================================================================================
namespace {
int grid_of(uint64_t n, uint64_t per) { return (int)std::max<uint64_t>(1, (n + per - 1) / per); }
}  // namespace

struct VoxBatch {
    DeviceBuffer in, keep, off, clouds, head, key_a, key_b, idx_a, idx_b, vkey, vcloud, chunk, radix, out;
    PinnedBuffer h_off, h_back;        // offsets on their way up, head + output offsets on their way back (pinned: DESIGN.md 6(i))
    bool in_flight = false;            // a failed call may have left copies from h_off queued
    int  sm_count = 0;
};

VoxBatch* vox_batch_create() { return new VoxBatch(); }

void vox_batch_destroy(VoxBatch* b) { delete b; }

#define VCK(call) ERASOR_CUDA_TRY(err, call, #call)

int vox_batch_run(VoxBatch* b, cudaStream_t st, const float* xyzi, const uint64_t* offsets, int F, const uint8_t* keep, float leaf,
                  const float* T12, bool dev, const float** d_out, uint64_t* out_offsets, uint64_t& launches, std::string& err) {
    const uint64_t N64 = offsets[F];
    const uint32_t N = (uint32_t)N64;
    if (N == 0) {
        for (int c = 0; c <= F; ++c) out_offsets[c] = 0;
        *d_out = b->out.as<const float>();
        return ERASOR_OK;
    }
    if (b->in_flight) { VCK(cudaStreamSynchronize(st)); b->in_flight = false; }
    if (!b->sm_count) {
        int dev_id = 0;
        VCK(cudaGetDevice(&dev_id));
        VCK(cudaDeviceGetAttribute(&b->sm_count, cudaDevAttrMultiProcessorCount, dev_id));
    }
    const float4* pts = reinterpret_cast<const float4*>(xyzi);
    const uint8_t* d_keep = keep;
    if (!dev) {
        VCK(b->in.ensure(sizeof(float4) * N64));
        VCK(cudaMemcpyAsync(b->in.p(), xyzi, sizeof(float4) * N64, cudaMemcpyHostToDevice, st));
        pts = b->in.as<const float4>();
        if (keep) {
            VCK(b->keep.ensure(N64));
            VCK(cudaMemcpyAsync(b->keep.p(), keep, N64, cudaMemcpyHostToDevice, st));
            d_keep = b->keep.as<const uint8_t>();
        }
    }
    VCK(b->h_off.ensure(sizeof(uint32_t) * (F + 1)));
    uint32_t* ho = b->h_off.as<uint32_t>();
    for (int c = 0; c <= F; ++c) ho[c] = (uint32_t)offsets[c];
    VCK(b->off.ensure(sizeof(uint32_t) * (F + 1)));
    VCK(cudaMemcpyAsync(b->off.p(), ho, sizeof(uint32_t) * (F + 1), cudaMemcpyHostToDevice, st));
    b->in_flight = true;

    const size_t words = (size_t)N + 1;
    VCK(b->clouds.ensure(sizeof(VbCloud) * F));
    VCK(b->head.ensure(sizeof(VbHead) + sizeof(uint32_t) * (F + 1)));
    for (DeviceBuffer* x : {&b->key_a, &b->key_b, &b->idx_a, &b->idx_b, &b->vkey, &b->vcloud}) VCK(x->ensure(sizeof(uint32_t) * words));
    const uint32_t nch = (uint32_t)((N64 + kVbChunk - 1) / kVbChunk);
    VCK(b->chunk.ensure(sizeof(uint32_t) * nch));
    VCK(b->radix.ensure(sizeof(uint32_t) * radix_scratch_words(N)));
    VCK(b->out.ensure(sizeof(float4) * N64));
    const uint32_t* off = b->off.as<const uint32_t>();
    VbCloud* cl = b->clouds.as<VbCloud>();
    VbHead* hd = b->head.as<VbHead>();
    uint32_t* vcnt = reinterpret_cast<uint32_t*>(hd + 1);
    uint32_t* const K[2] = {b->key_a.as<uint32_t>(), b->key_b.as<uint32_t>()};
    uint32_t* const V[2] = {b->idx_a.as<uint32_t>(), b->idx_b.as<uint32_t>()};
    const int g_stream = b->sm_count * 8;

    // bounds, grids, keys
    k_vb_init<<<grid_of((uint64_t)F + 1, kVbThreads), kVbThreads, 0, st>>>(cl, F, hd, vcnt);
    k_vb_bounds<<<grid_of(N64, 32ull * kVbRows * kVbWarps), kVbThreads, 0, st>>>(pts, d_keep, N, off, F, cl, hd);
    k_vb_setup<<<grid_of((uint64_t)F, kVbThreads), kVbThreads, 0, st>>>(cl, F, leaf, hd);
    k_vb_keys<<<std::min(grid_of(N64, kVbThreads), g_stream), kVbThreads, 0, st>>>(pts, d_keep, N, off, F, cl, K[0], V[0]);
    VCK(cudaGetLastError());
    launches += 4;
    // (voxel key, index) stably by key, then stably by cloud: the points in ascending key within each cloud, members in cloud order
    VCK(radix_sort_passes(st, b->radix.as<uint32_t>(), K, V, N, 0, kVbKeyPasses));                 // -> K[0], V[0]
    k_vb_cloud_keys<<<std::min(grid_of(N64, kVbThreads), g_stream), kVbThreads, 0, st>>>(d_keep, N, off, F, V[0], K[0]);
    VCK(cudaGetLastError());
    int cbits = 1;
    while (cbits < 32 && (1ull << cbits) <= (unsigned long long)F) ++cbits;                         // cloud keys are <= F
    const int cpass = (cbits + 7) / 8;
    VCK(radix_sort_passes(st, b->radix.as<uint32_t>(), K, V, N, 0, cpass));
    launches += 3ull * (kVbKeyPasses + cpass) + 1;
    const uint32_t* scl = K[cpass & 1];
    const uint32_t* order = V[cpass & 1];
    uint32_t* skey = K[(cpass & 1) ^ 1];
    uint32_t* vstart = V[(cpass & 1) ^ 1];
    k_vb_rekey<<<std::min(grid_of(N64, kVbThreads), g_stream), kVbThreads, 0, st>>>(pts, N, off, cl, hd, scl, order, skey);
    // voxels: run heads, per-cloud counts, output offsets, then centroids + labels
    k_vb_heads_count<<<nch, kVbThreads, 0, st>>>(skey, scl, hd, b->chunk.as<uint32_t>());
    k_vb_heads_scan<<<1, 1024, 0, st>>>(b->chunk.as<uint32_t>(), nch, hd);
    k_vb_heads_scatter<<<nch, kVbThreads, 0, st>>>(skey, scl, b->chunk.as<uint32_t>(), hd, b->vkey.as<uint32_t>(), vstart, b->vcloud.as<uint32_t>(), vcnt);
    k_vb_offsets<<<1, 1024, 0, st>>>(vcnt, F);
    VbAffine T{};
    if (T12) std::memcpy(T.m, T12, sizeof(T.m));
    k_vb_voxels<<<grid_of(N64, kVbThreads), kVbThreads, 0, st>>>(pts, order, vstart, b->vkey.as<uint32_t>(), b->vcloud.as<uint32_t>(), cl, hd, vcnt, T,
                                                                  T12 ? 1 : 0, b->out.as<float4>());
    VCK(cudaGetLastError());
    launches += 6;
    // the one read-back: scalars + output offsets
    const size_t back = sizeof(VbHead) + sizeof(uint32_t) * (F + 1);
    VCK(b->h_back.ensure(back));
    VCK(cudaMemcpyAsync(b->h_back.p(), hd, back, cudaMemcpyDeviceToHost, st));
    VCK(cudaStreamSynchronize(st));
    b->in_flight = false;
    const VbHead* h = b->h_back.as<const VbHead>();
    if (h->bad != kVbNone) {
        const int c = (int)(std::upper_bound(offsets, offsets + F + 1, (uint64_t)h->bad) - offsets) - 1;
        err = "non-finite x, y or z in point " + std::to_string((uint64_t)h->bad - offsets[c]) + " of cloud " + std::to_string(c);
        return ERASOR_E_INVALID;
    }
    const uint32_t* ro = reinterpret_cast<const uint32_t*>(h + 1);
    for (int c = 0; c <= F; ++c) out_offsets[c] = ro[c];
    *d_out = b->out.as<const float>();
    return ERASOR_OK;
}

}  // namespace erasor
