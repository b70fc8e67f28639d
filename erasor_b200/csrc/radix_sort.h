// radix_sort.h -- the device-wide stable LSD radix sort of (key, value) word pairs, 8-bit digits (kernels k_eval_radix_* in
// eval_kernels.cu).  Shared by the evaluator's cell index (eval_kernels.cu) and the batched voxeliser (voxelize_batch.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

namespace erasor {

constexpr uint32_t kRadixSeg = 4096;   // entries per warp segment of a pass

// scratch of radix_sort_passes for n entries: per-segment digit counts and the digit totals
inline size_t radix_scratch_words(uint32_t n) { return 256ull * (((uint64_t)n + kRadixSeg - 1) / kRadixSeg) + 256ull; }

// npass stable passes over (k[0], v[0]) of n entries, digits first, first + 1, ... (digit d = bits 8d .. 8d + 7 of the key);
// k[1] and v[1] are the ping-pong halves, and the result is in k[npass & 1], v[npass & 1].  Three launches per pass, on st.
cudaError_t radix_sort_passes(cudaStream_t st, uint32_t* scratch /*radix_scratch_words(n)*/, uint32_t* const k[2], uint32_t* const v[2],
                              uint32_t n, int first, int npass);

}  // namespace erasor
