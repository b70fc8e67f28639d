// micro-benchmark: latency of match.any / ballot / shuffle-min on one warp (cycles per op), used to size K2 / K1 aggregation
#include <cstdio>
#include <cstdint>
__global__ void k(int mode, long long* out) {
    const int lane = threadIdx.x;
    int key = (mode == 0) ? lane : (mode == 1) ? (lane & 3) : (mode == 2) ? 7 : lane;
    unsigned mask = (mode == 3) ? 0x11110000u : 0xFFFFFFFFu;
    unsigned acc = 0;
    long long t0 = clock64();
    if (mask >> lane & 1) {
        for (int i = 0; i < 1000; ++i) {
            unsigned p = __match_any_sync(mask, key);
            acc += p; key ^= (p & 1) << 9;          // dependent chain
        }
    }
    long long t1 = clock64();
    if (lane == 16) { out[mode * 2] = t1 - t0; out[mode * 2 + 1] = acc; }
}
__global__ void k_thr(int warps_active, long long* out) {   // throughput with many warps per SM: distinct keys
    const int lane = threadIdx.x & 31;
    int key = lane; unsigned acc = 0;
    long long t0 = clock64();
    for (int i = 0; i < 1000; ++i) { unsigned p = __match_any_sync(0xFFFFFFFFu, key); acc += p; key ^= (p & 1) << 9; }
    long long t1 = clock64();
    if (threadIdx.x == 0 && blockIdx.x == 0) { out[0] = t1 - t0; out[1] = acc; }
}
int main() {
    long long* d; cudaMalloc(&d, 64 * 8); long long h[64];
    for (int m = 0; m < 4; ++m) k<<<1, 32>>>(m, d);
    cudaMemcpy(h, d, 64, cudaMemcpyDeviceToHost);
    const char* names[] = {"32 distinct keys", "4 distinct keys", "1 key", "4 lanes, 4 keys"};
    for (int m = 0; m < 4; ++m) printf("match_any %-18s : %.1f cycles/op\n", names[m], h[m * 2] / 1000.0);
    for (int w : {1, 4, 8, 16, 32}) {
        k_thr<<<132, w * 32>>>(w, d); cudaMemcpy(h, d, 16, cudaMemcpyDeviceToHost);
        printf("match_any 32 distinct, %2d warps/SM: %.1f cycles/op per warp\n", w, h[0] / 1000.0);
    }
    return 0;
}
