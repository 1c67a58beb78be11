// chars_kernel.cuh -- the character offsets of spm_encode_offsets_device_padded (SPM_OFFSETS_CHARS): every byte offset
// p of a padded row becomes utf8_to_unicode[min(p, len)], the table of ConvertToUnicodeSpans
// (src/sentencepiece_processor.cc:63-91) over the sentence's input, as processor.char_index restates it:
//   - characters are the chain 0, c + OneCharLen(input[c]), ... cut at len (the reference does not guard a last lead
//     byte that claims more bytes than remain; the chain stops at len);
//   - a byte p < len gets the index of the character that holds it, len the number of characters;
//   - an empty input keeps its offsets (all 0), which is what the table gives too.
//
// One warp per row sweeps its sentence 32 bytes per block, keeping the chain's next start (`carry`) and the characters
// that start before the block.  In valid UTF-8 the chain's starts are exactly the bytes that are not continuation
// bytes (10xxxxxx), so a block's starts are one ballot; a block where the chain does not land on those bytes (a
// malformed sentence) is walked step by step from `carry` instead, through shuffles of the block's byte lengths.
// The row's offsets rise in the raw order of its tokens (the body; the frame is set apart), so the sweep visits every
// block once: each group of 32 tokens converts its begin / end while the sweep passes their blocks.  A group whose
// smallest offset lies behind the sweep restarts it from the sentence's start, which keeps any order correct.
// Frame cells: an entry equal to eos_id holds (len, len), which becomes the number of characters; the others hold
// (0, 0), which stays.
#ifndef SPM_B200_CHARS_KERNEL_CUH_
#define SPM_B200_CHARS_KERNEL_CUH_

#include <cstdint>

#include "device_model.h"
#include "kernels.cuh"

namespace spm_b200 {

// The sweep over one sentence of `len` bytes at s: `base` is the current block's first byte, `mask` its chain starts
// (bit j: byte base + j), `cnt` the characters that start before it.
struct CharSweep {
  const uint8_t *s;
  uint32_t len;
  uint32_t base, carry, cnt, mask, next;  // next: the chain's first start at or after base + 32 (or len)
  bool have;                              // mask / next belong to base

  __device__ __forceinline__ void reset() { base = carry = cnt = 0u; have = false; }

  __device__ __forceinline__ void block(uint32_t lane) {
    const uint32_t j = base + lane;
    const bool in = j < len;
    const uint32_t c = in ? s[j] : 0u;
    const bool st = in && (j == 0u || !is_trail(c));
    const uint32_t S = __ballot_sync(0xFFFFFFFFu, st);
    const uint32_t step = one_char_len(c);
    const uint32_t tgt = min(j + step, len);
    const uint32_t stop = min(base + 32u, len);
    bool ok = true;
    if (st) {
      const uint32_t above = lane == 31u ? 0u : S & (~0u << (lane + 1u));
      ok = above ? tgt == base + __ffs(above) - 1u : tgt >= stop;
    }
    ok = __all_sync(0xFFFFFFFFu, ok) && (S ? carry == base + __ffs(S) - 1u : carry >= stop);
    if (ok) {  // the chain is the non-continuation bytes here
      mask = S;
      next = S ? __shfl_sync(0xFFFFFFFFu, tgt, 31 - __clz(S)) : carry;
    } else {   // malformed: follow the chain
      uint32_t C = 0u, pos = carry;
      while (pos < stop) {
        const uint32_t l = pos - base;
        C |= 1u << l;
        pos = min(pos + __shfl_sync(0xFFFFFFFFu, step, l), len);
      }
      mask = C;
      next = pos;
    }
    have = true;
  }

  __device__ __forceinline__ void advance() {
    cnt += __popc(mask);
    carry = next;
    base += 32u;
    have = false;
  }

  // the character index of p (<= len) when p lies in the current block (base <= p < base + 32)
  __device__ __forceinline__ uint32_t index(uint32_t p) const {
    return cnt + __popc(mask & (0xFFFFFFFFu >> (31u - (p - base)))) - (p < len ? 1u : 0u);
  }
};

// One list's offsets in place: its body of B tokens at cells np + (B - 1 - q reversed, else q) for raw position q, its
// frame at cells [0, np) and [np + B, np + B + ns).  Cells: get(c) / set(c, v) of the (begin, end) at cell c.
template <typename Cells>
__device__ __forceinline__ void list_to_chars(CharSweep &sw, Cells cells, uint32_t B, const KFrame &F, int32_t eos_id,
                                              uint32_t lane) {
  const uint32_t fr = F.np + F.ns;
  for (uint32_t r0 = 0; r0 < B; r0 += 32) {
    const uint32_t q = r0 + lane;  // raw order
    const bool act = q < B;
    const uint32_t cell = F.np + (F.reverse ? B - 1u - q : q);
    int2 v = act ? cells.get(cell) : make_int2(0, 0);
    const uint32_t b = min(static_cast<uint32_t>(v.x), sw.len), e = min(static_cast<uint32_t>(v.y), sw.len);
    const uint32_t lo = __reduce_min_sync(0xFFFFFFFFu, act ? min(b, e) : 0xFFFFFFFFu);
    const uint32_t hi = __reduce_max_sync(0xFFFFFFFFu, act ? max(b, e) : 0u);
    if (lo < sw.base) sw.reset();
    uint32_t cb = 0, ce = 0;
    for (;;) {
      if (!sw.have) sw.block(lane);
      if (b - sw.base < 32u) cb = sw.index(b);
      if (e - sw.base < 32u) ce = sw.index(e);
      if (hi < sw.base + 32u) break;
      sw.advance();
    }
    if (act) cells.set(cell, make_int2(static_cast<int32_t>(cb), static_cast<int32_t>(ce)));
  }
  bool eos = false;
  for (uint32_t t = 0; t < fr; ++t) eos |= F.ids[t] == eos_id;
  if (!eos) return;
  // the number of characters: the sweep to the block that holds len
  if (sw.len < sw.base) sw.reset();
  for (;;) {
    if (!sw.have) sw.block(lane);
    if (sw.len < sw.base + 32u) break;
    sw.advance();
  }
  const int32_t chars = static_cast<int32_t>(sw.index(sw.len));
  for (uint32_t t = lane; t < fr; t += 32)
    if (F.ids[t] == eos_id) cells.set(t < F.np ? t : B + t, make_int2(chars, chars));
}

// One warp per row of the [n, w] spans tensor that the padded K11 wrote (byte offsets), rewritten in place.
__global__ void __launch_bounds__(256) spans_to_chars_kernel(const uint8_t *bytes, const uint64_t *offsets, uint32_t n,
                                                             int2 *spans, const int32_t *lengths, uint32_t w, KFrame F,
                                                             int32_t eos_id, uint32_t left) {
  struct Row {
    int2 *r;
    __device__ __forceinline__ int2 get(uint32_t c) const { return r[c]; }
    __device__ __forceinline__ void set(uint32_t c, int2 v) const { r[c] = v; }
  };
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t fr = F.np + F.ns;
  for (uint32_t row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < n; row += warps) {
    CharSweep sw;
    sw.s = bytes + offsets[row];
    sw.len = static_cast<uint32_t>(offsets[row + 1] - offsets[row]);
    sw.reset();
    sw.mask = sw.next = 0u;
    const uint32_t real = static_cast<uint32_t>(lengths[row]);
    list_to_chars(sw, Row{spans + static_cast<unsigned long long>(row) * w + (left ? w - real : 0u)}, real - fr, F,
                  eos_id, lane);
  }
}

// One warp per sentence of K11's framed, packed output (begin / end at id_offsets[i], byte offsets), rewritten in
// place: the character offsets of spm_encode_windows_device, converted once per sentence before the window rows
// copy them.
__global__ void __launch_bounds__(256) lists_to_chars_kernel(const uint8_t *bytes, const uint64_t *offsets, uint32_t n,
                                                             uint32_t *begin, uint32_t *end,
                                                             const unsigned long long *id_offsets, KFrame F,
                                                             int32_t eos_id) {
  struct List {
    uint32_t *b, *e;
    __device__ __forceinline__ int2 get(uint32_t c) const {
      return make_int2(static_cast<int32_t>(b[c]), static_cast<int32_t>(e[c]));
    }
    __device__ __forceinline__ void set(uint32_t c, int2 v) const {
      b[c] = static_cast<uint32_t>(v.x);
      e[c] = static_cast<uint32_t>(v.y);
    }
  };
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t fr = F.np + F.ns;
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
    CharSweep sw;
    sw.s = bytes + offsets[i];
    sw.len = static_cast<uint32_t>(offsets[i + 1] - offsets[i]);
    sw.reset();
    sw.mask = sw.next = 0u;
    const unsigned long long o = id_offsets[i];
    list_to_chars(sw, List{begin + o, end + o}, static_cast<uint32_t>(id_offsets[i + 1] - o) - fr, F, eos_id, lane);
  }
}

}  // namespace spm_b200
#endif
