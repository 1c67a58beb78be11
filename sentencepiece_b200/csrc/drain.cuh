// drain.cuh -- K6: in-kernel compaction of finished segments into the caller's result buffers.
//
// Fused host path (engine.cu, encode_host_fused): ONE launch of a lane kernel encodes the whole
// batch.  The ids of a sentence land in a temporary buffer in completion order (K4); the result
// the reference-facing API returns is ids in INPUT order plus id_offsets[n + 1]
// (SentencePieceProcessor::Encode over a list, sentencepiece_processor.cc:392-403).  The batch is
// cut into segments of 2^seg_shift consecutive sentences; the processing order is sorted over whole
// input pieces (2^piece_shift sentences, order_kernel.cuh), so a group of 32 lanes may hold
// sentences of many segments: finished sentences are counted per segment, and the warp that brings
// a segment's count to its size compacts that segment:
//   1. exclusive scan of the segment's id counts, segment total published;
//   2. decoupled look-back over the earlier segments' {total, inclusive prefix} words gives the
//      segment's first output position.  An earlier segment that is not finished yet is waited for:
//      one warp per finished-but-blocked segment (at most the segments of a piece or two) spins
//      while the other resident warps keep taking groups, so the wait always ends;
//   3. id_offsets (to pinned host memory) and the ids (to the device result buffer) are written; with an encode frame
//      (KFrame) every sentence counts |P| + |S| more and its ids are written between P and S, reversed if asked;
//   4. the run of finished segments is extended and its id count stored to a pinned host word: the
//      host polls it and fetches the finished prefix with the copy engine while later segments are
//      still being encoded (SM stores over PCIe reach only ~25 GB/s, the copy engine ~55 GB/s).
#ifndef SPM_B200_DRAIN_CUH_
#define SPM_B200_DRAIN_CUH_

#include "device_model.h"

namespace spm_b200 {

constexpr unsigned long long kSegFlag = 1ull << 63;

__device__ __forceinline__ unsigned long long ld_volatile_u64(const unsigned long long *p) {
  return *reinterpret_cast<const volatile unsigned long long *>(p);
}
__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, d);
  return v;
}

// Compaction of a finished segment (warp-collective), in two steps: drain_publish scans the segment's counts and
// publishes its total; drain_finish finds the segment's output position (look-back over the earlier segments, which
// may have to be waited for) and copies.  A warp that finishes several segments at once publishes ALL their totals
// before it waits for anything: a wait only ever depends on totals, and those are out before any waiting starts.
__device__ __forceinline__ void drain_publish(const KBatch &B, uint32_t seg, uint32_t lane);
__device__ __forceinline__ void drain_finish(const KBatch &B, uint32_t seg, uint32_t lane);

// Called by every warp after it has stored a group's results (sent_start / sent_count / tmp_ids): `sent` is the lane's
// sentence (valid when `have`).  The processing order may mix the sentences of many segments in one group (the order
// is sorted over a whole input piece, drain segments are much smaller), so completion is counted per SENTENCE: the
// lanes of a group that share a segment add their count with one atomic, and the warp that brings a segment's count
// to its size compacts it.
__device__ __forceinline__ void lane_drain(const KBatch &B, uint32_t sent, bool have, uint32_t lane) {
  if (!B.seg_done) return;
  // release: this group's results (stored by all 32 lanes) before the counters.  The warp barrier orders the lanes'
  // stores before the leaders' RELEASE atomics below; a __threadfence() here would also invalidate the SM's L1
  // (MEMBAR.SC + CCTL.IVALL) once per group -- see lane_wait_input.
  __syncwarp();
  const uint32_t seg = have ? sent >> B.seg_shift : 0xFFFFFFFFu;
  const uint32_t peers = __match_any_sync(0xFFFFFFFFu, seg);
  const uint32_t leader = static_cast<uint32_t>(__ffs(peers)) - 1u;
  bool completes = false;
  if (have && lane == leader) {
    const uint32_t cnt = static_cast<uint32_t>(__popc(peers));
    const uint32_t seg_lo = seg << B.seg_shift;
    const uint32_t seg_n = min(B.n - seg_lo, 1u << B.seg_shift);
    uint32_t before;
    asm volatile("atom.add.release.gpu.global.u32 %0, [%1], %2;" : "=r"(before) : "l"(B.seg_done + seg), "r"(cnt) : "memory");
    completes = before + cnt == seg_n;
  }
  const uint32_t done = __ballot_sync(0xFFFFFFFFu, completes);
  if (!done) return;  // the usual case
  __threadfence();  // acquire: the other groups' results
  for (uint32_t todo = done; todo; todo &= todo - 1u)   // one segment at a time, the whole warp works on it
    drain_publish(B, __shfl_sync(0xFFFFFFFFu, seg, static_cast<uint32_t>(__ffs(todo)) - 1u), lane);
  for (uint32_t todo = done; todo; todo &= todo - 1u)
    drain_finish(B, __shfl_sync(0xFFFFFFFFu, seg, static_cast<uint32_t>(__ffs(todo)) - 1u), lane);
}

__device__ __forceinline__ void drain_publish(const KBatch &B, uint32_t seg, uint32_t lane) {
  const uint32_t seg_lo = seg << B.seg_shift;
  const uint32_t seg_n = min(B.n - seg_lo, 1u << B.seg_shift);
  // ---- 1. scan of the counts; relative offsets parked in sent_rel ----
  uint32_t run = 0;
  const uint32_t framed = B.frame.np + B.frame.ns;  // ids the encode frame adds to every sentence
  for (uint32_t j = 0; j < seg_n; j += 32) {
    const uint32_t i = seg_lo + j + lane;
    const uint32_t cnt = j + lane < seg_n ? __ldcg(B.sent_count + i) + framed : 0u;
    uint32_t incl = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d);
      if (lane >= static_cast<uint32_t>(d)) incl += t;
    }
    if (j + lane < seg_n) B.sent_rel[i] = run + incl - cnt;
    run += __shfl_sync(0xFFFFFFFFu, incl, 31);
  }
  if (lane == 0) {
    *reinterpret_cast<volatile unsigned long long *>(B.seg_total + seg) = static_cast<unsigned long long>(run) | kSegFlag;
    __threadfence();
  }
  __syncwarp();
}

__device__ __forceinline__ void drain_finish(const KBatch &B, uint32_t seg, uint32_t lane) {
  const uint32_t seg_lo = seg << B.seg_shift;
  const uint32_t seg_n = min(B.n - seg_lo, 1u << B.seg_shift);
  const long long t_start = clock64();
  long long t_lb = 0;
  const unsigned long long total = ld_volatile_u64(B.seg_total + seg) & ~kSegFlag;
  // ---- 2. decoupled look-back, 32 predecessors per step ----
  const long long t_lb0 = clock64();
  unsigned long long prefix = 0;
  for (int t = static_cast<int>(seg) - 1; t >= 0;) {
    const int idx = t - static_cast<int>(lane);
    unsigned long long pv = kSegFlag, tv = 0;  // a virtual predecessor before segment 0 has prefix 0
    if (idx >= 0) {
      pv = ld_volatile_u64(B.seg_prefix + idx);
      if (!(pv & kSegFlag)) tv = ld_volatile_u64(B.seg_total + idx);
    }
    const uint32_t has_p = __ballot_sync(0xFFFFFFFFu, (pv & kSegFlag) != 0);
    const uint32_t has_any = __ballot_sync(0xFFFFFFFFu, ((pv | tv) & kSegFlag) != 0);
    const uint32_t first_p = has_p ? static_cast<uint32_t>(__ffs(has_p)) - 1u : 32u;
    const uint32_t need = first_p >= 32u ? 0xFFFFFFFFu : ((1u << first_p) - 1u);
    if ((has_any & need) != need) {  // a nearer segment has published nothing yet
      __nanosleep(100);
      // bounded like the input wait: ~3 s without progress fails the call (status bit 2) instead of hanging the GPU
      if (clock64() - t_lb0 > 6000000000ll || (*reinterpret_cast<const volatile uint32_t *>(B.status + 1) & 4u)) {
        if (lane == 0) atomicOr(B.status + 1, 4u);
        break;
      }
      continue;
    }
    unsigned long long mine = 0;
    if (lane < first_p) mine = tv & ~kSegFlag;
    else if (lane == first_p) mine = pv & ~kSegFlag;
    prefix += warp_sum_u64(mine);
    if (first_p < 32u) break;
    t -= 32;
  }
  t_lb = clock64() - t_lb0;
  if (lane == 0) {
    *reinterpret_cast<volatile unsigned long long *>(B.seg_prefix + seg) = (prefix + total) | kSegFlag;
    __threadfence();
  }
  // ---- 3. results ----
  const bool room = prefix + total <= B.out_cap;
  if (!room) {
    if (lane == 0) atomicOr(B.status + 2, 2u);
  }
  __syncwarp();
  for (uint32_t j = 0; j < seg_n; j += 32) {
    const uint32_t i = seg_lo + j + lane;
    const bool have = j + lane < seg_n;
    unsigned long long src = 0, dst = 0;
    uint32_t cnt = 0;
    if (have) {
      cnt = __ldcg(B.sent_count + i);
      src = __ldcg(B.sent_start + i);
      dst = prefix + __ldcg(B.sent_rel + i);
      B.out_offsets[i] = B.out_off_base + dst;
    }
    if (!room) continue;
    if (B.frame.active()) {
      // framed: P, the sentence's ids (backwards under reverse), S -- one sentence per step
      const uint32_t tot = have ? cnt + B.frame.np + B.frame.ns : 0u;
#pragma unroll 1
      for (uint32_t k = 0; k < 32; ++k) {
        const unsigned long long s = __shfl_sync(0xFFFFFFFFu, src, k), d = __shfl_sync(0xFFFFFFFFu, dst, k);
        const uint32_t c = __shfl_sync(0xFFFFFFFFu, cnt, k), m = __shfl_sync(0xFFFFFFFFu, tot, k);
        for (uint32_t r = lane; r < m; r += 32)
          B.out_ids[d + r] = B.frame.at(c, r, [&](uint32_t q) { return __ldcg(B.tmp_ids + s + q); });
      }
      continue;
    }
    // one sentence per step: its ids are contiguous on both sides -> coalesced 128-byte loads and stores; four
    // sentences are in flight at a time so that the loads overlap
#pragma unroll 1
    for (uint32_t k = 0; k < 32; k += 4) {
      unsigned long long s[4], d[4];
      uint32_t c[4];
      int32_t v[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        s[q] = __shfl_sync(0xFFFFFFFFu, src, k + q);
        d[q] = __shfl_sync(0xFFFFFFFFu, dst, k + q);
        c[q] = __shfl_sync(0xFFFFFFFFu, cnt, k + q);
        v[q] = lane < c[q] ? __ldcg(B.tmp_ids + s[q] + lane) : 0;
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (lane < c[q]) B.out_ids[d[q] + lane] = v[q];
        for (uint32_t r = 32 + lane; r < c[q]; r += 32) B.out_ids[d[q] + r] = __ldcg(B.tmp_ids + s[q] + r);
      }
    }
  }
  if (seg_lo + seg_n == B.n && lane == 0) B.out_offsets[B.n] = B.out_off_base + prefix + total;
  if (B.kstats && lane == 0) {
    atomicAdd(B.kstats + 1, static_cast<unsigned long long>(clock64() - t_start));
    atomicAdd(B.kstats + 2, static_cast<unsigned long long>(t_lb));
  }
  // ---- 4. progress: extend the run of finished segments and tell the host how many ids it may fetch ----
  if (B.seg_copied) {
    __threadfence();  // the segment's ids before its flag
    if (lane == 0) {
      atomicExch(B.seg_copied + seg, 1u);
      asm volatile("fence.sc.gpu;" ::: "memory");  // flag store before the counter load (two drainers may meet here)
      const uint32_t nseg = (B.n + (1u << B.seg_shift) - 1u) >> B.seg_shift;
      for (;;) {
        const uint32_t w = atomicAdd(B.drained_upto, 0u);
        if (w >= nseg || atomicAdd(B.seg_copied + w, 0u) == 0u) break;
        if (atomicCAS(B.drained_upto, w, w + 1u) == w) {
          const unsigned long long upto = ld_volatile_u64(B.seg_prefix + w) & ~kSegFlag;
          __threadfence_system();
          *reinterpret_cast<volatile unsigned long long *>(B.host_progress) = upto;  // the host keeps the maximum it sees
        }
      }
    }
  }
}

}  // namespace spm_b200
#endif
