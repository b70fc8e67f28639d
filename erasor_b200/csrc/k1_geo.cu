// k1_geo.cu -- K1's geometry form (erasor_process_nodes_tune, DESIGN.md section 8.7).  A translation unit of its own: the exact
// binning path's out-of-line functions are shared by every caller in a module, so a new caller in kernels.cu would change the
// register allocation of the plain K1 kernels.
#include <cuda_runtime.h>

#include <cstdint>

#include "device_common.cuh"
#include "device_types.h"
#include "k1_common.cuh"
#include "kernels.h"

namespace erasor {

// the exact path of binning.h, kept out of line: it is taken by ~1e-4 of the points
__device__ __noinline__ int bin_exact_geo(const BinTablesView& T, float x, float y, float z, BinFenceCounters* fc) {
    return bin_of_point(T, T.ring_thr, x, y, z, fc);
}

// K1's geometry form (node mode, erasor_process_nodes_tune): the node-mode path of k1_rpod_bin -- the map scan, the VoI cut, the
// warp-local compaction, the origin -> body transform and the VoI lists -- once per point, then per geometry of G its polar bin,
// its bin id and its shared-table update; each geometry's flush goes to its own tables.  Per geometry the arithmetic is
// k1_rpod_bin's, so every geometry's ids, counts and z extremes equal those of a plain launch with its tables.
template <int THREADS, int UNROLL>
__global__ void __launch_bounds__(THREADS, THREADS == 256 ? 4 : 1)
k1_geo_bin(const __grid_constant__ K1Geo G, const float4* __restrict__ map_pts, const float4* __restrict__ qry_pts,
           const ChunkDesc* __restrict__ chunks, int F, unsigned long long* __restrict__ fence, const NodePose* __restrict__ poses,
           uint32_t* __restrict__ list_idx, uint32_t* __restrict__ list_cnt, int qry_xyz) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int NW = THREADS / 32;
    const ChunkDesc cd = chunks[blockIdx.x];
    __shared__ NodePose s_pose;
    const int NG = G.n;
    auto tabs = [&](int g, float2*& s_ring, uint32_t*& s_cnt, uint32_t*& s_mn, uint32_t*& s_mx) {
        s_ring = reinterpret_cast<float2*>(smem_raw + G.g[g].smem_off);
        s_cnt  = reinterpret_cast<uint32_t*>(s_ring + ((G.g[g].T.R + 2) & ~1));
        s_mn   = s_cnt + (G.g[g].B + 1);
        s_mx   = s_mn + G.g[g].B;
    };
    for (int g = 0; g < NG; ++g) {
        float2* s_ring; uint32_t *s_cnt, *s_mn, *s_mx;
        tabs(g, s_ring, s_cnt, s_mn, s_mx);
        const int R = G.g[g].T.R, B = G.g[g].B;
        for (int i = tid; i <= R; i += THREADS) s_ring[i] = make_float2(G.g[g].T.ring_guard[2 * i], G.g[g].T.ring_guard[2 * i + 1]);
        for (int i = tid; i <= B; i += THREADS) s_cnt[i] = 0u;
        for (int i = tid; i < B; i += THREADS) { s_mn[i] = 0xFFFFFFFFu; s_mx[i] = 0u; }
    }
    if (tid == 0) s_pose = poses[cd.frame];
    __syncthreads();

    BinFenceCounters fc{0u, 0u, 0u};
    // one point (valid when ok) of the cloud under every geometry: its bin id at position pos of the geometry's id array
    auto bin_all = [&](const float4& pp, bool ok, bool map, size_t pos) {
        const uint32_t zenc = float_to_ordered(pp.z);
        for (int g = 0; g < NG; ++g) {
            const BinTablesView& T = G.g[g].T;
            float2* s_ring; uint32_t *s_cnt, *s_mn, *s_mx;
            tabs(g, s_ring, s_cnt, s_mn, s_mx);
            const int B = G.g[g].B;
            int b = bin_fast(pp.x, pp.y, pp.z, T.z_lo, T.z_hi, T.smax_lo, T.smax_hi, T.inv_ring, T.inv_ss, T.eps_q, T.R, T.S, s_ring);
            if (__any_sync(FULL_MASK, ok && b == -3)) {
                if (ok && b == -3) b = bin_exact_geo(T, pp.x, pp.y, pp.z, &fc);   // exact path (rare)
            }
            int key = -2;
            if (ok) {
                (map ? G.g[g].bin_map : G.g[g].bin_qry)[pos] = (b < 0) ? kNoBin16 : (uint16_t)b;
                key = (b < 0) ? B : b;
            }
            k1_aggregate(key, zenc, lane, s_cnt, s_mn, s_mx, B);
        }
    };

    if (cd.cloud == 0) {
        // the map path of k1_rpod_bin<..., NODE = true>: every warp streams its sub-range, compacts the points inside the VoI
        // into its 64-entry ring and bins full rows with all 32 lanes busy
        __shared__ float4 s_ring_q[NW * 64];
        float4* __restrict__ q = s_ring_q + warp * 64;
        const float4* __restrict__ src = map_pts + cd.begin;
        const uint32_t sub = (((cd.len + NW - 1) / NW) + 31u) & ~31u;
        const uint32_t w0 = min(cd.len, (uint32_t)warp * sub), w1 = min(cd.len, w0 + sub);
        const size_t lpos = (size_t)cd.bin_begin + w0;
        uint32_t* __restrict__ lidx = list_idx + lpos;
        uint32_t qh = 0, qt = 0;
        auto dense_row = [&](uint32_t n) {
            const bool ok = (uint32_t)lane < n;
            const float4 e = q[(qh + lane) & 63u];
            const float4 pp = pcl_affine(s_pose.T, e);
            if (ok) lidx[qh + lane] = cd.begin + __float_as_uint(e.w);
            bin_all(pp, ok, true, lpos + qh + lane);
            qh += n;
            __syncwarp();
        };
        const float pxf = s_pose.pxf, pyf = s_pose.pyf, lim_lo = s_pose.lim_lo, lim_hi = s_pose.lim_hi;
        for (uint32_t base = w0; base < w1; base += 32u * UNROLL) {
            float4 p[UNROLL];
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) p[u] = __ldg(src + (base + u * 32u + lane));
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) {
                const uint32_t i = base + u * 32u + lane;
                const float dxf = p[u].x - pxf, dyf = p[u].y - pyf;
                const float d2f = fmaf(dyf, dyf, dxf * dxf);
                const bool in = (i < w1) && (d2f < lim_lo || (!(d2f > lim_hi) && in_voi_radius(s_pose, p[u].x, p[u].y)));
                const unsigned bal = __ballot_sync(FULL_MASK, in);
                if (bal == 0u) continue;
                if (in) q[(qt + __popc(bal & ((1u << lane) - 1u))) & 63u] = make_float4(p[u].x, p[u].y, p[u].z, __uint_as_float(i));
                qt += __popc(bal);
                __syncwarp();
                if (qt - qh >= 32u) dense_row(32u);
            }
        }
        if (qt != qh) dense_row(qt - qh);
        if (lane == 0) list_cnt[(size_t)blockIdx.x * kListWarps + warp] = qt;
    } else {
        const float4* __restrict__ src = qry_pts + cd.begin;
        const float* __restrict__ q3 = reinterpret_cast<const float*>(qry_pts) + (size_t)cd.begin * 3u;
        for (uint32_t base = warp * (32u * UNROLL); base < cd.len; base += NW * (32u * UNROLL)) {
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) {
                const uint32_t i = base + u * 32u + lane;
                const bool ok = i < cd.len;
                const float4 pp = !ok ? make_float4(0.f, 0.f, 0.f, 0.f)
                                : qry_xyz ? make_float4(__ldg(q3 + 3u * (size_t)i), __ldg(q3 + 3u * (size_t)i + 1u), __ldg(q3 + 3u * (size_t)i + 2u), 0.f)
                                          : ld_stream_f4(src + i);
                bin_all(pp, ok, false, (size_t)cd.bin_begin + i);
            }
        }
    }
    __syncthreads();

    for (int g = 0; g < NG; ++g) {
        float2* s_ring; uint32_t *s_cnt, *s_mn, *s_mx;
        tabs(g, s_ring, s_cnt, s_mn, s_mx);
        const int B = G.g[g].B;
        uint32_t* __restrict__ row = G.g[g].ch_cnt + (size_t)blockIdx.x * (B + 1);
        const size_t ft = ((size_t)cd.cloud * F + cd.frame) * B;
        const size_t ct = ((size_t)cd.cloud * F + cd.frame) * (B + 1);
        for (int i = tid; i <= B; i += THREADS) {
            const uint32_t c = s_cnt[i];
            row[i] = c;
            if (c != 0u) {
                atomicAdd(&G.g[g].cnt[ct + i], c);
                if (i < B) {
                    atomicMin(&G.g[g].zmin[ft + i], s_mn[i]);
                    atomicMax(&G.g[g].zmax[ft + i], s_mx[i]);
                }
            }
        }
    }
    if (fc.negzero) atomicAdd(&fence[0], (unsigned long long)fc.negzero);
    if (fc.ambiguous) atomicAdd(&fence[2], (unsigned long long)fc.ambiguous);
    if (fc.slow) atomicAdd(&fence[3], (unsigned long long)fc.slow);
}

size_t k1_geo_smem_bytes(int R, int B) { return (k1_smem_bytes(R, B) + 15) & ~(size_t)15; }

// the kernel launch_k1_geo runs over tables of smem bytes
static auto k1_geo_kernel(size_t smem) { return k1_warps(smem) == 32 ? k1_geo_bin<1024, 4> : k1_geo_bin<256, 4>; }

cudaError_t k1_geo_table_limit(size_t table_bytes, size_t smem_optin, size_t* limit) {
    return max_dyn_smem(k1_geo_kernel(table_bytes), smem_optin, limit);
}

cudaError_t launch_k1_geo(cudaStream_t st, const K1Geo& G, size_t smem, const float4* map_pts, const float4* qry_pts, const ChunkDesc* chunks,
                          int n_chunks, int F, unsigned long long* fence, const NodePose* poses, uint32_t* list_idx, uint32_t* list_cnt, bool qry_xyz) {
    if (n_chunks == 0) return cudaSuccess;
    const bool big = k1_warps(smem) == 32;
    auto kern = k1_geo_kernel(smem);
    cudaError_t e = ensure_dyn_smem(kern, smem);
    if (e != cudaSuccess) return e;
    kern<<<n_chunks, big ? 1024 : 256, smem, st>>>(G, map_pts, qry_pts, chunks, F, fence, poses, list_idx, list_cnt, qry_xyz ? 1 : 0);
    return cudaGetLastError();
}

}  // namespace erasor
