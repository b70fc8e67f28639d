// k1_common.cuh -- the per-point pieces of K1 that its plain form (kernels.cu) and its geometry form (k1_geo.cu) share, and the
// dynamic shared-memory helper of their launches.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <mutex>
#include <unordered_map>

#include "device_common.cuh"
#include "device_types.h"

namespace erasor {

// cudaFuncSetAttribute costs a few microseconds per call; the dynamic shared-memory ceiling of a kernel only ever has
// to grow, so remember the largest value set per kernel and skip the call otherwise.  A refused ceiling is returned and
// cleared: left as the thread's last error, the launch check of the next good launch (cudaGetLastError) would report it,
// on whichever handle made that launch.
template <class K>
static cudaError_t ensure_dyn_smem(K kern, size_t bytes) {
    static std::mutex mu;
    static std::unordered_map<const void*, size_t> seen;
    std::lock_guard<std::mutex> lock(mu);
    const void* key = reinterpret_cast<const void*>(kern);
    auto it = seen.find(key);
    if (it != seen.end() && it->second >= bytes) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) seen[key] = bytes;
    else cudaGetLastError();
    return e;
}

// The most dynamic shared memory kern can launch with on a device whose blocks opt in to smem_optin bytes: the opt-in less
// the kernel's static shared memory
template <class K>
static cudaError_t max_dyn_smem(K kern, size_t smem_optin, size_t* out) {
    cudaFuncAttributes a;
    const cudaError_t e = cudaFuncGetAttributes(&a, kern);
    if (e != cudaSuccess) { cudaGetLastError(); return e; }
    *out = smem_optin > a.sharedSizeBytes ? smem_optin - a.sharedSizeBytes : 0;
    return cudaSuccess;
}

__device__ __forceinline__ float4 ld_stream_f4(const float4* p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}

// Warp-level pre-aggregation of (bin, z) into the CTA's shared tables.  Input clouds are spatially
// coherent (voxel-key order, or bin order after the first frame), so most warps hold 1-3 runs of equal bins:
// one REDUX pair + three shared atomics per run instead of three atomics per point.
__device__ __forceinline__ void k1_aggregate(int key, uint32_t zenc, int lane, uint32_t* s_cnt, uint32_t* s_mn, uint32_t* s_mx, int B) {
    // key: bin id in [0,B), B for "not binned", -2 for an out-of-range lane
    const int key0 = __shfl_sync(FULL_MASK, key, 0);
    if (__all_sync(FULL_MASK, key == key0)) {
        if (key0 >= 0) {
            if (key0 < B) {
                const uint32_t mn = __reduce_min_sync(FULL_MASK, zenc);
                const uint32_t mx = __reduce_max_sync(FULL_MASK, zenc);
                if (lane == 0) {
                    atomicMin(&s_mn[key0], mn);
                    atomicMax(&s_mx[key0], mx);
                    atomicAdd(&s_cnt[key0], 32u);
                }
            } else if (lane == 0) {
                atomicAdd(&s_cnt[B], 32u);
            }
        }
        return;
    }
    // Mixed warp (in node mode every lane of a dense row lies inside the VoI, but the bins change along the row: 96 % of the
    // rows are mixed, ~5 keys each, scripts/k1_row_stats.py): per-lane shared-memory atomics, but only where they can
    // change something -- a bin's min / max settle after its first few points, and a plain (possibly stale) read is a safe
    // filter because the values only move one way.  One update per distinct key measured slower on an H100 (DESIGN section 5):
    // match.any + REDUX over each key's lanes (the REDUX runs once per key group) and a segmented shuffle reduction over runs.
    if (key >= 0) {
        if (key < B) {
            if (zenc < s_mn[key]) atomicMin(&s_mn[key], zenc);
            if (zenc > s_mx[key]) atomicMax(&s_mx[key], zenc);
        }
        atomicAdd(&s_cnt[key], 1u);          // key == B: the complement's count
    }
}

__device__ __forceinline__ float rsqrt_ftz(float v) { float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v)); return r; }
__device__ __forceinline__ float div_ftz(float a, float b) { float r; asm("div.approx.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }

// Branch-free fast path of binning.h's bin_of_point for the device, float arithmetic only: returns the bin, -1 (not
// binned) or -3 when the point needs the exact path (r^2 inside the guard band of s_max or of a ring threshold, ring guess
// off, sector coordinate inside its guard band, y == 0).  Every decision taken here is one the exact path would take too:
// the float r^2 is compared against thresholds widened by its own worst-case error (binning_tables.cpp).
__device__ __forceinline__ int bin_fast(float x, float y, float z, float z_lo, float z_hi, float smax_lo, float smax_hi, float inv_ring, float inv_ss,
                                        float eps_q, int R, int S, const float2* __restrict__ s_ringf) {
    const float sf   = fmaf(y, y, x * x);
    const bool  zin  = (z < z_hi) && (z > z_lo);
    const bool  in_sure  = sf <= smax_lo;
    const bool  out_sure = !(sf <= smax_hi);                  // also NaN
    const float sfc = fmaxf(sf, 1e-30f);
    int g = (int)(sfc * rsqrt_ftz(sfc) * inv_ring);
    g = min(g, R - 1);
    const float2 t0 = s_ringf[g], t1 = s_ringf[g + 1];         // {up, dn} of thresholds g and g + 1
    const bool ring_ok = (sf >= t0.x) && (sf < t1.y);
    const float ax = fabsf(x), ay = fabsf(y);
    const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
    float a = atan_unit(div_ftz(mn, mx));
    if (ay > ax)  a = 1.57079637f - a;
    if (x < 0.0f) a = 3.14159274f - a;
    if (y < 0.0f) a = 6.28318548f - a;
    const float q  = a * inv_ss;
    const int   k  = (int)q;
    const float fr = q - (float)k;
    const bool sec_ok = (fr >= eps_q) && (fr <= 1.0f - eps_q) && (ay != 0.0f);
    if (!zin || out_sure) return -1;
    if (!(in_sure && ring_ok && sec_ok)) return -3;
    return min(k, S - 1) * R + g;
}

// OfflineMapUpdater::fetch_VoI's cut (OfflineMapUpdater.cpp:394-396): pow(pt.x - x, 2) + pow(pt.y - y, 2) < max_dist_square in
// double on float differences.  A float evaluation decides every point outside a 1e-6 band around the limit (its error is
// below 2.4e-7 relative); points inside the band get the reference's double expression.
__device__ __forceinline__ bool in_voi_radius(const NodePose& P, float x, float y) {
    const float dxf = x - P.pxf, dyf = y - P.pyf;
    const float d2f = fmaf(dyf, dyf, dxf * dxf);
    if (d2f < P.lim_lo) return true;
    if (d2f > P.lim_hi) return false;
    const double dx = __dsub_rn((double)x, P.px), dy = __dsub_rn((double)y, P.py);
    return __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)) < P.limit;
}

}  // namespace erasor
