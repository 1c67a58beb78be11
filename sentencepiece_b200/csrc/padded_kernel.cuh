// padded_kernel.cuh -- the padded writer of spm_encode_ids_device_padded: a batch's ids as rows of one width.
//
// The encode kernels leave sentence i's raw ids in completion order at src + src_start[i] (count[i] of them), the
// input of the packed writer (scan_write_gather_kernel) as well.  Here row i of the [n, w] output gets the framed list
//   prefix ++ body[:B] ++ suffix,  body = the raw ids, reversed when the frame says so,
// with B = count[i], or min(count[i], w - np - ns) when truncating, at the start of the row or (left) at its end, and
// pad_id in every other cell.  The host has checked that every untruncated row fits.
#ifndef SPM_B200_PADDED_KERNEL_CUH_
#define SPM_B200_PADDED_KERNEL_CUH_

#include <cstdint>

#include "device_model.h"

namespace spm_b200 {

// The longest framed row: max(count[i]) + added into *out (zeroed by the caller).  n > 0.
__global__ void __launch_bounds__(256) row_max_kernel(const uint32_t *counts, uint32_t n, uint32_t added,
                                                      unsigned long long *out) {
  uint32_t m = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) m = max(m, counts[i]);
  m = __reduce_max_sync(0xFFFFFFFFu, m);
  if ((threadIdx.x & 31) == 0) atomicMax(out, static_cast<unsigned long long>(m) + added);
}

// One warp per row; every cell of the row is written, lane t of the warp taking cells t, t + 32, ... (coalesced).
// lengths[i] = the real cells of row i.
__global__ void __launch_bounds__(256) write_padded_kernel(const uint32_t *counts, const unsigned long long *src_start,
                                                           const int32_t *src, uint32_t n, KFrame F, uint32_t w,
                                                           int32_t pad_id, uint32_t truncate, uint32_t left,
                                                           int32_t *out, int32_t *lengths) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t frame = F.np + F.ns;
  for (uint32_t row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < n; row += warps) {
    const uint32_t c = counts[row];
    const uint32_t body = truncate ? min(c, w - frame) : c;
    const uint32_t real = body + frame;
    const uint32_t lead = left ? w - real : 0u;
    // F.at reads the kept body in raw order: its first `body` raw ids, or with a reversed frame its last ones
    const int32_t *s = src + src_start[row] + (F.reverse ? c - body : 0u);
    int32_t *o = out + static_cast<unsigned long long>(row) * w;
    for (uint32_t t = lane; t < w; t += 32) {
      const uint32_t k = t - lead;  // wraps past `real` for the leading pad cells
      __stcs(o + t, k < real ? F.at(body, k, [&](uint32_t q) { return __ldcs(s + q); }) : pad_id);
    }
    if (lane == 0) lengths[row] = static_cast<int32_t>(real);
  }
}

}  // namespace spm_b200
#endif
