// padded_kernel.cuh -- the padded writer of spm_encode_ids_device_padded: a batch's ids as rows of one width.
//
// The encode kernels leave sentence i's raw ids in completion order at src + src_start[i] (count[i] of them), the
// input of the packed writer (scan_write_gather_kernel) as well.  Here row i of the [n, w] output gets the framed list
//   prefix ++ body[:B] ++ suffix,  body = the raw ids, reversed when the frame says so,
// with B = count[i], or min(count[i], w - np - ns) when truncating, at the start of the row or (left) at its end, and
// pad_id in every other cell.  The host has checked that every untruncated row fits.
// Windows (spm_encode_windows_device) are rows of the same kind: each holds a stretch of its sentence's body.
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
// lengths[row] = the real cells of the row.  WINDOWS (spm_encode_windows_device): row r is window row_first[r] of
// sentence row_sentence[r], the body ids [f, f + min(count - f, w - np - ns)) in body order (reversed when the frame
// says so) between the prefix and the suffix; the padded rows are the case row = sentence, f = 0.
template <bool WINDOWS>
__device__ __forceinline__ void write_rows(const uint32_t *counts, const unsigned long long *src_start,
                                           const int32_t *src, uint32_t rows, const KFrame &F, uint32_t w,
                                           int32_t pad_id, uint32_t truncate, uint32_t left, int32_t *out,
                                           int32_t *lengths, const int32_t *row_sentence, const int32_t *row_first) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t frame = F.np + F.ns;
  for (uint32_t row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
    uint32_t i = row, f = 0;
    if constexpr (WINDOWS) {
      i = static_cast<uint32_t>(row_sentence[row]);
      f = static_cast<uint32_t>(row_first[row]);
    }
    const uint32_t c = counts[i] - f;  // the body ids from the window's first on
    const uint32_t body = truncate ? min(c, w - frame) : c;
    const uint32_t real = body + frame;
    const uint32_t lead = left ? w - real : 0u;
    // F.at reads the kept body in raw order: raw ids [f, f + body), or with a reversed frame [c - body, c) of the
    // raw list (body index k is raw index count - 1 - k)
    const int32_t *s = src + src_start[i] + (F.reverse ? c - body : f);
    int32_t *o = out + static_cast<unsigned long long>(row) * w;
    for (uint32_t t = lane; t < w; t += 32) {
      const uint32_t k = t - lead;  // wraps past `real` for the leading pad cells
      __stcs(o + t, k < real ? F.at(body, k, [&](uint32_t q) { return __ldcs(s + q); }) : pad_id);
    }
    if (lane == 0) lengths[row] = static_cast<int32_t>(real);
  }
}

__global__ void __launch_bounds__(256) write_padded_kernel(const uint32_t *counts, const unsigned long long *src_start,
                                                           const int32_t *src, uint32_t n, KFrame F, uint32_t w,
                                                           int32_t pad_id, uint32_t truncate, uint32_t left,
                                                           int32_t *out, int32_t *lengths) {
  write_rows<false>(counts, src_start, src, n, F, w, pad_id, truncate, left, out, lengths, nullptr, nullptr);
}

__global__ void __launch_bounds__(256) write_windows_kernel(const uint32_t *counts, const unsigned long long *src_start,
                                                            const int32_t *src, uint32_t rows, KFrame F, uint32_t w,
                                                            int32_t pad_id, uint32_t left, int32_t *out,
                                                            int32_t *lengths, const int32_t *row_sentence,
                                                            const int32_t *row_first) {
  write_rows<true>(counts, src_start, src, rows, F, w, pad_id, 1u, left, out, lengths, row_sentence, row_first);
}

// The window plan of spm_encode_windows_device: sentence i of counts[i] body ids gets m[i] = 1 window when
// counts[i] <= B, else 1 + ceil((counts[i] - B) / step).
__global__ void __launch_bounds__(256) window_count_kernel(const uint32_t *counts, uint32_t n, uint32_t B,
                                                           uint32_t step, uint32_t *m) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint64_t L = counts[i];
    m[i] = L <= B ? 1u : static_cast<uint32_t>(1u + (L - B + step - 1u) / step);
  }
}

// The rows' sentence and first body index: one warp per sentence, whose rows are row_start[i] .. row_start[i + 1]
// (the exclusive scan of window_count_kernel's m).  A long document has thousands of rows.
__global__ void __launch_bounds__(256) window_rows_kernel(const unsigned long long *row_start, uint32_t n,
                                                          uint32_t step, int32_t *row_sentence, int32_t *row_first) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
    const unsigned long long r0 = row_start[i];
    const uint32_t m = static_cast<uint32_t>(row_start[i + 1] - r0);
    for (uint32_t j = lane; j < m; j += 32) {
      __stcs(row_sentence + r0 + j, static_cast<int32_t>(i));
      __stcs(row_first + r0 + j, static_cast<int32_t>(j * step));
    }
  }
}

}  // namespace spm_b200
#endif
