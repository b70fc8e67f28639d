// voxelize_batch.h -- erasor_voxelize_batch's device work (voxelize_batch.cu), owned by an erasor handle (erasor_capi.cu)
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

namespace erasor {

struct VoxBatch;                           // scratch, output cloud and pinned read-back of one handle
VoxBatch* vox_batch_create();
void      vox_batch_destroy(VoxBatch* b);

// erasor_voxelize_batch after the handle's own checks: xyzi / keep host or device (dev), offsets validated by the caller
// (offsets[0] = 0, monotone, offsets[F] < 2^32 - 1, every cloud below 2^31 points).  T12 (nullable): rows 0..2 of the output
// affine.  Returns an ERASOR_* code; *d_out / out_offsets as documented in include/erasor_b200.h.
int vox_batch_run(VoxBatch* b, cudaStream_t st, const float* xyzi, const uint64_t* offsets, int F, const uint8_t* keep, float leaf,
                  const float* T12, bool dev, const float** d_out, uint64_t* out_offsets, uint64_t& launches, std::string& err);

}  // namespace erasor
