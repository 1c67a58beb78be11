// normalize_kernel.cuh -- K10, spm_normalize: SentencePieceProcessor::Normalize (normalizer.cc:71-186) for a packed
// batch, without the encode.
//
// One warp per sentence runs normalize_tile (kernels.cuh), the normalizer of the general encode kernels, with its
// text and norm_to_orig in global memory: it walks the input in 32-byte windows and needs no shared-memory tile, so
// one kernel takes sentences of any length.  Sentence i writes into its own slab, sized from the model's worst-case
// expansion rounded up to whole bytes (ceil(spm_engine::max_expand_num / max_expand_den), at least 3); the engine then
// packs the slabs with the scan kernels (scan_total / scan_gather).  Slab i starts at norm_slab_start(bytes before
// sentence i, i): text at text + start, norm_to_orig at n2o + start, capacity start(i + 1) - start(i) - 1 normalized
// bytes (one more n2o entry).
#ifndef SPM_B200_NORMALIZE_KERNEL_CUH_
#define SPM_B200_NORMALIZE_KERNEL_CUH_

#include <cstdint>

#include "device_model.h"
#include "kernels.cuh"

namespace spm_b200 {

// The n2o entry of a sentence whose reference norm_to_orig is empty (SPM_NORM_TO_ORIG_EMPTY in spm_b200.h): the
// input is empty (normalizer.cc:77-79) or all of it is heading whitespace (:97-100).
constexpr uint32_t kNormToOrigEmpty = 0xFFFFFFFFu;

// rel * expand + 8 i: slab i holds len * expand + 7 normalized bytes, room for the dummy prefix and suffix (3 bytes
// each) behind the worst-case expansion of the input, and one more n2o entry.
__host__ __device__ __forceinline__ unsigned long long norm_slab_start(unsigned long long rel, uint32_t i, uint32_t expand) {
  return rel * expand + 8ull * i;
}

struct KNormalize {
  const uint8_t *bytes;       // sentence i: bytes[offsets[i] - offsets[0], offsets[i + 1] - offsets[0])
  const uint64_t *offsets;    // [n + 1]
  uint32_t n;
  uint32_t expand;            // normalized bytes per input byte, at most
  uint8_t *text;              // slabs
  uint32_t *n2o;              // slabs (WITH_OFFSETS)
  unsigned long long *slab;   // [n] out: start of slab i, the gather's source offsets
  uint32_t *len;              // [n] out: normalized length
  uint32_t *status;           // bit 0: a sentence outgrew its slab (the bound says it cannot)
};

// (min blocks 1: with the plain bound of 256 threads ptxas holds the kernel to 32 registers and spills)
template <bool WITH_OFFSETS>
__global__ void __launch_bounds__(256, 1) normalize_kernel(const KModel M, const KNormalize A) {
  const Tile T;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  const uint64_t base = A.offsets[0];
  for (uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; s < A.n; s += warps) {
    const uint64_t lo = A.offsets[s] - base, hi = A.offsets[s + 1] - base;
    const unsigned long long start = norm_slab_start(lo, s, A.expand);
    const unsigned long long end = norm_slab_start(hi, s + 1, A.expand);
    TileMem tm{};
    tm.text = A.text + start;
    tm.ncap = static_cast<uint32_t>(end - start - 1);
    if (WITH_OFFSETS) {
      tm.n2o = A.n2o + start;
      // normalize_tile leaves n2o[0] alone exactly when the reference's norm_to_orig is empty
      if (T.lane == 0) tm.n2o[0] = kNormToOrigEmpty;
      T.sync();
    }
    const NormResult r = normalize_tile<WITH_OFFSETS>(M, T, A.bytes + lo, static_cast<uint32_t>(hi - lo), tm);
    if (T.lane == 0) {
      A.slab[s] = start;
      A.len[s] = r.n > tm.ncap ? 0u : r.n;
      if (r.n > tm.ncap) atomicOr(A.status, 1u);
    }
  }
}

}  // namespace spm_b200
#endif
