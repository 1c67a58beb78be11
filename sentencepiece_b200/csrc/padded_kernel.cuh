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
// (the exclusive scan of window_count_kernel's m).  A long document has thousands of rows.  Window j starts j * step
// ids in, step being steps[i] when steps is given (sentence pairs, whose room differs per pair), else `step`.
__global__ void __launch_bounds__(256) window_rows_kernel(const unsigned long long *row_start, uint32_t n,
                                                          uint32_t step, const uint32_t *steps, int32_t *row_sentence,
                                                          int32_t *row_first) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
    const unsigned long long r0 = row_start[i];
    const uint32_t m = static_cast<uint32_t>(row_start[i + 1] - r0);
    const uint32_t s = steps ? steps[i] : step;
    for (uint32_t j = lane; j < m; j += 32) {
      __stcs(row_sentence + r0 + j, static_cast<int32_t>(i));
      __stcs(row_first + r0 + j, static_cast<int32_t>(j * s));
    }
  }
}

// ---- sentence pairs (spm_encode_pairs_device) ----
// The batch holds 2n sentences; pair i is (A, B) = (sentence i, sentence n + i).  A row of pair i holds
//   prefix ++ A[fa, fa + ca) ++ middle ++ B[fb, fb + cb) ++ suffix
// with the template's ids at tmpl[0, np), [np, np + nm) and [np + nm, np + nm + ns).  Type ids are 0 up to the end of
// the middle and 1 from B's first cell on; pad cells get 0.
enum : uint32_t { kPairTruncNone = 0, kPairLongestFirst = 1, kPairOnlyFirst = 2, kPairOnlySecond = 3 };

struct KPairs {
  const int32_t *tmpl;
  uint32_t np, nm, ns;
  uint32_t windowed;  // the member cut into windows: 0 none, 1 A, 2 B
};

// The plan of pair i, a = counts[i], b = counts[n + i] raw ids, T = np + nm + ns, Bt = w - T (w > T unless
// truncation is kPairTruncNone):
//   keep[i] = the most ids of A / B one row holds; m[i] = its rows; step[i] = the step between its windows (0 when
//   it has one row); into *need (zeroed by the caller) the max of each pair's least workable width, clamped to
//   2^32 - 1: T + a + b without truncation (the longest row), T + min(a + b, other + 1 + stride) when one member is
//   cut (the room Bt - other must exceed the stride), nothing under longest-first (every w > T works).
// Longest-first drops the last id of the longer body, B's on ties, while a + b > Bt; its closed form is
// a' = min(a, max(Bt - b, ceil(Bt / 2))), b' = min(b, Bt - a').
__global__ void __launch_bounds__(256) pair_plan_kernel(const uint32_t *counts, uint32_t n, KPairs T, uint32_t w,
                                                        uint32_t trunc, uint32_t overflow, uint32_t stride,
                                                        uint2 *keep, uint32_t *m, uint32_t *step,
                                                        unsigned long long *need) {
  const unsigned long long tsz = T.np + T.nm + T.ns;
  uint32_t most = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned long long a = counts[i], b = counts[n + i];
    unsigned long long ka = a, kb = b, lp = 0;
    uint32_t rows = 1, s = 0;
    if (trunc == kPairTruncNone) {
      lp = tsz + a + b;
    } else {
      const unsigned long long bt = w - tsz;
      if (trunc == kPairLongestFirst) {
        if (a + b > bt) {
          ka = min(a, max(bt > b ? bt - b : 0ull, (bt + 1) / 2));
          kb = min(b, bt - ka);
        }
      } else {
        const bool first = trunc == kPairOnlyFirst;
        const unsigned long long len = first ? a : b, other = first ? b : a;
        const unsigned long long room = bt > other ? bt - other : 0ull;
        lp = tsz + min(a + b, other + 1 + stride);
        if (len > room && room > stride) {
          if (overflow) {
            s = static_cast<uint32_t>(room - stride);
            rows = static_cast<uint32_t>(1 + (len - room + s - 1) / s);
          }
          (first ? ka : kb) = room;
        }
      }
    }
    keep[i] = make_uint2(static_cast<uint32_t>(ka), static_cast<uint32_t>(kb));
    m[i] = rows;
    step[i] = s;
    most = max(most, static_cast<uint32_t>(min(lp, 0xFFFFFFFFull)));
  }
  most = __reduce_max_sync(0xFFFFFFFFu, most);
  if ((threadIdx.x & 31) == 0) atomicMax(need, static_cast<unsigned long long>(most));
}

// One pair row: the first id and the count of A and of B it holds, and its real cells.  f = the row's first id in the
// windowed member; a, b = the members' sizes.
struct PairRow {
  uint32_t fa, ca, fb, cb, real;
};

__device__ __forceinline__ PairRow pair_row(const KPairs &T, uint32_t f, uint2 keep, uint32_t a, uint32_t b) {
  PairRow p;
  p.fa = T.windowed == 1 ? f : 0u;
  p.fb = T.windowed == 2 ? f : 0u;
  p.ca = min(a - p.fa, keep.x);
  p.cb = min(b - p.fb, keep.y);
  p.real = T.np + T.nm + T.ns + p.ca + p.cb;
  return p;
}

// Where real cell k of a pair row comes from: 0 the template (q its index in tmpl), 1 A, 2 B (q the index in the
// member's ids).
__device__ __forceinline__ uint32_t pair_cell(const KPairs &T, const PairRow &p, uint32_t k, uint32_t &q) {
  if (k < T.np) { q = k; return 0; }
  k -= T.np;
  if (k < p.ca) { q = p.fa + k; return 1; }
  k -= p.ca;
  if (k < T.nm) { q = T.np + k; return 0; }
  k -= T.nm;
  if (k < p.cb) { q = p.fb + k; return 2; }
  q = T.np + T.nm + k - p.cb;
  return 0;
}

// The id rows of spm_encode_pairs_device without offsets: one warp per row, as write_rows, from the raw ids the encode
// stage leaves at src + src_start[i] (A) and src + src_start[n + i] (B).
__global__ void __launch_bounds__(256) write_pair_rows_kernel(const uint32_t *counts,
                                                              const unsigned long long *src_start, const int32_t *src,
                                                              uint32_t n, uint32_t rows, KPairs T, const uint2 *keep,
                                                              const int32_t *row_pair, const int32_t *row_first,
                                                              uint32_t w, int32_t pad_id, uint32_t left, int32_t *out,
                                                              int32_t *type_ids, int32_t *lengths) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
    const uint32_t i = static_cast<uint32_t>(row_pair[row]);
    const PairRow p = pair_row(T, static_cast<uint32_t>(row_first[row]), keep[i], counts[i], counts[n + i]);
    const int32_t *sa = src + src_start[i], *sb = src + src_start[n + i];
    const uint32_t lead = left ? w - p.real : 0u;
    const uint32_t second = T.np + p.ca + T.nm;  // the first cell of type 1
    int32_t *o = out + static_cast<unsigned long long>(row) * w;
    int32_t *ty = type_ids + static_cast<unsigned long long>(row) * w;
    for (uint32_t t = lane; t < w; t += 32) {
      const uint32_t k = t - lead;  // wraps past `real` for the leading pad cells
      int32_t id = pad_id, type = 0;
      if (k < p.real) {
        uint32_t q;
        const uint32_t c = pair_cell(T, p, k, q);
        id = c == 0 ? T.tmpl[q] : c == 1 ? sa[q] : sb[q];
        type = k >= second ? 1 : 0;
      }
      __stcs(o + t, id);
      __stcs(ty + t, type);
    }
    if (lane == 0) lengths[row] = static_cast<int32_t>(p.real);
  }
}

}  // namespace spm_b200
#endif
