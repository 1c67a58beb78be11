// nbest_kernel.cuh -- K5: exact n-best segmentation (config 5: SampleEncode nbest_size > 1,
// NBestEncode) on the GPU, one sentence per lane.
//
// Reference: unigram::Model::NBestEncode (src/unigram_model.cc:695-721) =
//   Lattice::SetSentence (:113-146)  character positions, BOS / EOS nodes
//   Model::PopulateNodes (:547-596)  one node per (start char, piece), UNK node last
//   Lattice::Viterbi     (:161-198)  float backtrace scores (the A* heuristic)
//   Lattice::NBest       (:345-509)  backward A* over a std::priority_queue<Hypothesis*>
// The ORDER of equal-priority results is whatever libstdc++'s binary heap yields
// (SURVEY.md 8a Q9: 37 % of sentences have tied candidates), so the heap discipline of
// std::push_heap / std::pop_heap (bits/stl_heap.h: sift-up stops at equal keys;
// __adjust_heap walks the hole to a leaf preferring the right child unless it is smaller,
// then pushes the saved last element back up) and the agenda shrink at 10,000 entries are
// reproduced step for step.  The search is sequential per sentence, so each lane runs it
// for its own sentence with its lattice, hypothesis pool and heap in a per-lane slab in HBM.
// Sentences a lane cannot hold go on a deferred list for nbest_long_kernel (below).
#ifndef SPM_B200_NBEST_KERNEL_CUH_
#define SPM_B200_NBEST_KERNEL_CUH_

#include "lane_kernel.cuh"

namespace spm_b200 {

struct NbestGeom {
  uint32_t cap;        // normalized bytes per sentence
  uint32_t node_cap;   // lattice nodes per sentence (<= 65535: hypotheses hold 16-bit node indices)
  uint32_t hyp_cap;    // hypotheses per sentence
  uint32_t heap_cap;   // agenda entries (>= 10000 + fan-out + 512 for the shrink list)
};
// per-lane scratch in HBM, 16-byte records so that one load / store moves a whole hypothesis or node:
//   hyp  [hyp_cap]     uint4 {next, gx bits, node | ids_so_far << 16, begin char | unk << 16}
//   heap [heap_cap+2]  uint2 {fx bits, hypothesis}; entry i lives in slot i + 1, which puts the children
//                      (2k+1, 2k+2) of any entry in one aligned 16-byte pair (one load per level of a pop)
//   node [node_cap]    uint4 {id, score bits, backtrace bits, begin char | end char << 16}   creation order
//   elist[node_cap]    uint4 {node | begin char << 16, backtrace bits, score bits, ids | unk << 31}   sorted by end char
//   end_off[cap+4] u32, maxbt[cap+4] f32 (reused as the sort cursors), surf[cap+4] u16
__host__ __device__ inline unsigned long long nbest_lane_bytes(const NbestGeom &g) {
  unsigned long long b = 0;
  b += 16ull * g.hyp_cap;
  b += 8ull * (g.heap_cap + 2);
  b += 32ull * g.node_cap;
  b += 4ull * (g.cap + 4) * 2;
  b += 2ull * (g.cap + 4);
  return (b + 15ull) & ~15ull;
}
// agenda entries kept in shared memory per lane (the top levels of the binary heap); odd, so that a pair of
// children never straddles the shared / global boundary
constexpr int kNbestTop = 15;
template <int TOP>
__host__ __device__ constexpr uint32_t nbest_smem_bytes(uint32_t warps) {
  return kLaneTableBytes + warps * 32u * 8u * TOP;
}

struct NbestOut {
  int32_t *tmp_ids;
  unsigned long long tmp_cap;
  unsigned long long *cursor;
  unsigned long long *cand_start;  // [n * nbest]
  uint32_t *cand_count;            // [n * nbest]
  float *cand_score;               // [n * nbest]
  uint32_t *n_cands;               // [n]
  uint32_t *status;                // [0] deferred sentences (shared with KBatch::status), [1] error, [2] overflow
};

// The agenda: std::push_heap / std::pop_heap on {fx bits, hypothesis} entries keyed by fx (comp: a.fx < b.fx).  Entry
// i lives in s_top[i * 32] (shared memory, lane-strided) for i < TOP, else in heap slot i + 1.
template <int TOP>
struct NbestAgenda {
  uint2 *s_top;
  uint2 *heap;
  __device__ __forceinline__ uint2 get(uint32_t i) const { return (TOP > 0 && i < TOP) ? s_top[i * 32] : heap[i + 1]; }
  __device__ __forceinline__ void set(uint32_t i, uint2 e) const {
    if (TOP > 0 && i < TOP) s_top[i * 32] = e;
    else heap[i + 1] = e;
  }
  __device__ __forceinline__ void push(uint32_t &hn, uint2 e) const {
    uint32_t hole = hn++;
    const float fv = __uint_as_float(e.x);
    while (hole > 0) {
      const uint32_t parent = (hole - 1) >> 1;
      const uint2 pe = get(parent);
      if (!(__uint_as_float(pe.x) < fv)) break;  // equal keys do not move up
      set(hole, pe);
      hole = parent;
    }
    set(hole, e);
  }
  __device__ __forceinline__ uint2 pop(uint32_t &hn) const {
    const uint2 top = get(0);
    const uint32_t len = --hn;
    if (len == 0) return top;
    const uint2 value = get(len);
    const float fv = __uint_as_float(value.x);
    uint32_t hole = 0, child = 0;
    while (child < (len - 1) / 2) {  // __adjust_heap: move the larger child up (the right one on ties)
      child = 2 * (child + 1);
      uint2 le, re;
      if (TOP > 0 && child < TOP) {
        re = s_top[child * 32];
        le = s_top[(child - 1) * 32];
      } else {
        const uint4 pr = *reinterpret_cast<const uint4 *>(heap + child);  // slots child, child + 1
        le = make_uint2(pr.x, pr.y);
        re = make_uint2(pr.z, pr.w);
      }
      if (__uint_as_float(re.x) < __uint_as_float(le.x)) { child--; re = le; }
      set(hole, re);
      hole = child;
    }
    if ((len & 1u) == 0 && child == (len - 2) / 2) {
      child = 2 * (child + 1);
      set(hole, get(child - 1));
      hole = child - 1;
    }
    while (hole > 0) {  // __push_heap of the saved last element
      const uint32_t parent = (hole - 1) >> 1;
      const uint2 pe = get(parent);
      if (!(__uint_as_float(pe.x) < fv)) break;
      set(hole, pe);
      hole = parent;
    }
    set(hole, value);
    return top;
  }
  // agenda shrink (:481-505): pop the best `shrink_to` into keep[], clear; the caller pushes them back in that order
  __device__ __forceinline__ void shrink_pop(uint32_t &hn, uint2 *keep, uint32_t shrink_to) const {
    for (uint32_t i = 0; i < shrink_to; ++i) keep[i] = pop(hn);
    hn = 0;
  }
};

// One result of Lattice::NBest as candidate `ck`: `cnt` ids of PopulateSentencePieceText's id path (UNK runs merged,
// byte-fallback UNK nodes spelled as byte pieces) over the nodes that path(emit) visits left to right as
// emit(id, begin char, end char); text_byte(k) is byte k of the normalized text, surf[c] the byte offset of char c.
template <typename SurfT, typename TextByte, typename Path>
__device__ __forceinline__ void nbest_write_result(const KModel &M, const NbestOut &O, size_t ck, uint32_t cnt, float score,
                                                   const SurfT *surf, TextByte &&text_byte, Path &&path) {
  const unsigned long long pos = atomicAdd(O.cursor, static_cast<unsigned long long>(cnt));
  O.cand_start[ck] = pos;
  O.cand_count[ck] = cnt;
  O.cand_score[ck] = score;
  if (pos + cnt > O.tmp_cap) {
    atomicOr(O.status + 2, 1u);
    O.cand_count[ck] = 0;
    return;
  }
  const bool bf = M.flags & kFlagByteFallback;
  uint32_t w = 0;
  bool prev_unk = false;
  path([&](int32_t id, uint32_t b, uint32_t e) {
    const bool isunk = id == M.unk_id;
    if (isunk) {
      if (bf) {
        for (uint32_t k = surf[b]; k < surf[e]; ++k) O.tmp_ids[pos + (w++)] = __ldg(M.byte_to_id + text_byte(k));
      } else if (!prev_unk) {
        O.tmp_ids[pos + (w++)] = M.unk_id;
      }
    } else {
      O.tmp_ids[pos + (w++)] = id;
    }
    prev_unk = isunk;
  });
  if (w != cnt) atomicOr(O.status + 1, 1u);
}

template <int TOP, int THREADS>
__global__ void __launch_bounds__(THREADS, 1) nbest_lane_kernel(const KModel M, const KBatch B, const NbestOut O,
                                                                 uint8_t *text_slabs, uint8_t *scratch, const NbestGeom G,
                                                                 uint32_t nbest) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint32_t *s_tab = reinterpret_cast<uint32_t *>(smem);
  fill_lane_tables(M, s_tab);
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp_global = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const LaneCtx c = lane_ctx(s_tab, text_slabs, G.cap, warp_global, lane);
  // per-lane scratch
  uint8_t *sp = scratch + (static_cast<size_t>(warp_global) * 32 + lane) * nbest_lane_bytes(G);
  uint4 *hyp = reinterpret_cast<uint4 *>(sp); sp += 16ull * G.hyp_cap;
  uint2 *heap = reinterpret_cast<uint2 *>(sp); sp += 8ull * (G.heap_cap + 2);   // slot = entry + 1
  uint4 *node = reinterpret_cast<uint4 *>(sp); sp += 16ull * G.node_cap;
  uint4 *elist = reinterpret_cast<uint4 *>(sp); sp += 16ull * G.node_cap;
  uint32_t *end_off = reinterpret_cast<uint32_t *>(sp); sp += 4ull * (G.cap + 4);
  float *maxbt = reinterpret_cast<float *>(sp); sp += 4ull * (G.cap + 4);
  uint16_t *surf = reinterpret_cast<uint16_t *>(sp);
  uint32_t *sort_cur = reinterpret_cast<uint32_t *>(maxbt);  // maxbt is dead once the nodes exist
  // agenda top: [warp][entry][lane]
  const NbestAgenda<TOP> ag{reinterpret_cast<uint2 *>(smem + kLaneTableBytes) + static_cast<size_t>(threadIdx.x >> 5) * (32 * TOP) + lane,
                            heap};

  const uint32_t root = __ldg(&M.trie_node2[0]).x;
  const bool bf = M.flags & kFlagByteFallback;

  uint32_t first = 0;
  while (lane_claim_group(B, lane, &first)) {
    if (first + lane < B.n) {
      const uint32_t sent = B.order ? B.order[first + lane] : first + lane;
      uint32_t n;
      const bool too_big = !lane_k1(M, B, c, sent, G.cap, &n);
      const size_t cbase = static_cast<size_t>(sent) * nbest;
      uint32_t K = 0;
      if (too_big) {
        lane_defer_long(B, sent, 0u);
      } else if (n == 0) {
        // NBestEncode of an empty normalized string: one empty candidate, score 0 (:697-699)
        O.cand_start[cbase] = 0; O.cand_count[cbase] = 0; O.cand_score[cbase] = 0.f;
        K = 1;
      } else {
        // ---- Lattice::SetSentence ----
        uint32_t L = 0;
        for (uint32_t p = 0; p < n;) {
          uint32_t mb = one_char_len(lane_text_byte_plain(c, p));
          if (mb > n - p) mb = n - p;
          surf[L] = static_cast<uint16_t>(p);
          maxbt[L] = -INFINITY;
          ++L;
          p += mb;
        }
        surf[L] = static_cast<uint16_t>(n);
        maxbt[L] = -INFINITY;
        maxbt[0] = 0.f;  // BOS
        // nodes 0 = BOS, 1 = EOS (EOS's backtrace score is filled in below)
        uint32_t nn = 2;
        node[0] = make_uint4(0xFFFFFFFFu, 0u, 0u, 0u);
        bool overflow = false;
        // ---- Model::PopulateNodes, with Lattice::Viterbi's backtrace scores folded in ----
        // backtrace(r) = max over nodes q ending where r begins of fl(backtrace(q) + score(r)); fl(x + s) is
        // monotone in x, so it equals fl(max_q backtrace(q) + score(r)), and every q is complete before r is made.
        for (uint32_t bp = 0; bp < L && !overflow; ++bp) {
          const float in_bt = maxbt[bp];
          const bool has_single = lane_populate_from(M, c, root, surf, bp, n, [&](uint32_t length, uint32_t v, float sc) {
            if (nn >= G.node_cap) { overflow = true; return false; }
            const float bt = __fadd_rn(in_bt, sc);
            node[nn] = make_uint4(static_cast<uint32_t>(__ldg(M.trie_id + v)), __float_as_uint(sc), __float_as_uint(bt),
                                  bp | ((bp + length) << 16));
            maxbt[bp + length] = fmaxf(maxbt[bp + length], bt);
            ++nn;
            return true;
          });
          if (!has_single && !overflow) {
            if (nn >= G.node_cap) { overflow = true; break; }
            const float bt = __fadd_rn(in_bt, M.unk_score);
            node[nn] = make_uint4(static_cast<uint32_t>(M.unk_id), __float_as_uint(M.unk_score), __float_as_uint(bt),
                                  bp | ((bp + 1) << 16));
            maxbt[bp + 1] = fmaxf(maxbt[bp + 1], bt);
            ++nn;
          }
        }
        if (!overflow) {
          const float eos_bt = __fadd_rn(maxbt[L], 0.f);
          // end_nodes lists in insertion order (stable counting sort by end character); BOS is the list of 0
          for (uint32_t p = 0; p <= L + 1; ++p) end_off[p] = 0;
          end_off[0 + 1] += 1;
          for (uint32_t i = 2; i < nn; ++i) end_off[(node[i].w >> 16) + 1] += 1;
          for (uint32_t p = 0; p <= L; ++p) end_off[p + 1] += end_off[p];
          for (uint32_t p = 0; p <= L; ++p) sort_cur[p] = end_off[p];
          elist[sort_cur[0]++] = make_uint4(0u, 0u, 0u, 0u);
          for (uint32_t i = 2; i < nn; ++i) {
            const uint4 nd = node[i];
            const uint32_t b = nd.w & 0xFFFFu, e = nd.w >> 16;
            const bool isunk = static_cast<int32_t>(nd.x) == M.unk_id;
            const uint32_t contrib = (isunk && bf) ? static_cast<uint32_t>(surf[e] - surf[b]) : 1u;
            elist[sort_cur[e]++] = make_uint4(i | (b << 16), nd.z, nd.y, contrib | (isunk ? 0x80000000u : 0u));
          }
          // ---- Lattice::NBest: backward A* ----
          uint32_t pn = 1, hn = 0;
          hyp[0] = make_uint4(0xFFFFFFFFu, 0u, 1u, L);  // EOS: next = null, gx = 0, no ids yet
          ag.push(hn, make_uint2(__float_as_uint(eos_bt), 0u));
          const uint32_t shrink_to = nbest * 10 < 512 ? nbest * 10 : 512;
          while (hn && !overflow) {
            const uint2 te = ag.pop(hn);
            const uint4 th = hyp[te.y];
            if ((th.z & 0xFFFFu) == 0) {  // reached BOS: one result
              nbest_write_result(M, O, cbase + K, th.z >> 16, __uint_as_float(te.x), surf,
                                 [&](uint32_t k) { return lane_text_byte_plain(c, k); }, [&](auto &&emit) {
                                   for (uint4 h = hyp[th.x]; h.x != 0xFFFFFFFFu; h = hyp[h.x]) {
                                     const uint4 nd = node[h.z & 0xFFFFu];
                                     emit(static_cast<int32_t>(nd.x), nd.w & 0xFFFFu, nd.w >> 16);
                                   }
                                 });
              if (++K == nbest) break;
              continue;
            }
            // expand: one hypothesis per node ending where this one begins, in end_nodes order
            const uint32_t p0 = th.w & 0xFFFFu;
            const bool top_unk = (th.w >> 16) & 1u;
            const float top_gx = __uint_as_float(th.y);
            const uint32_t top_cnt = th.z >> 16;
            uint32_t q = end_off[p0];
            const uint32_t qe = end_off[p0 + 1];
            if (pn + (qe - q) > G.hyp_cap || hn + (qe - q) + 1 >= G.heap_cap - 512u) { overflow = true; break; }
            uint4 rec = elist[q];
            for (; q < qe; ++q) {
              const uint4 nxt = elist[q + 1 < qe ? q + 1 : q];  // issued ahead of the agenda update below
              const bool isunk = rec.w >> 31;
              uint32_t cn = top_cnt + (rec.w & 0x7FFFFFFFu);
              if (!bf && isunk && top_unk) --cn;
              hyp[pn] = make_uint4(te.y, __float_as_uint(__fadd_rn(__uint_as_float(rec.z), top_gx)),
                                   (rec.x & 0xFFFFu) | (cn << 16), (rec.x >> 16) | (isunk ? 0x10000u : 0u));
              ag.push(hn, make_uint2(__float_as_uint(__fadd_rn(__uint_as_float(rec.y), top_gx)), pn));
              ++pn;
              rec = nxt;
            }
            if (hn >= 10000u) {  // agenda shrink (:481-505): pop the best `shrink_to`, clear, push them back in that order
              uint2 *keep = heap + (G.heap_cap + 1 - shrink_to);
              ag.shrink_pop(hn, keep, shrink_to);
              for (uint32_t i = 0; i < shrink_to; ++i) ag.push(hn, keep[i]);
            }
          }
        }
        if (overflow) lane_defer_long(B, sent, n);  // the long-sentence path redoes the sentence with 32-bit indices
      }
      O.n_cands[sent] = K;
      for (uint32_t k = K; k < nbest; ++k) { O.cand_count[cbase + k] = 0; O.cand_start[cbase + k] = 0; O.cand_score[cbase + k] = 0.f; }
    }
    __syncwarp();
  }
}

// ---- long-sentence path: one warp per sentence the lane kernel deferred (B.long_list: {sentence, normalized-byte
//      capacity}; B.long_scratch_off: its scratch slab).  The warp normalizes the sentence (normalize_tile), finds the
//      character starts and the nodes of every start in parallel; lane 0 folds the backtrace scores in node order and
//      runs the A* -- the agenda in the slab, node and hypothesis indices, id counts and positions 32 bits wide.  At
//      an agenda shrink that finds the hypothesis pool more than half full, the pool is compacted to what the kept
//      entries reach through `next` (CloneHypAndDependents, :313-341, which the reference runs at every shrink):
//      results do not depend on it, only the pool size does, and walking the kept chains at every shrink would cost a
//      long sentence more than its search.  A pool too small for the search leaves the sentence unfinished with
//      long_need[w] = a larger pool; the host relaunches it. ----
//   node  [node_cap]     uint4 {id, score bits, backtrace bits, begin char}   creation order: BOS, EOS, then by begin
//   nend  [node_cap]     u32   end char
//   elist [node_cap]     uint4 {node, backtrace bits, score bits, ids | unk << 31}   sorted by end char
//   hyp   [hyp_cap]      uint4 {next, gx bits, node, ids so far}
//   fwd   [hyp_cap]      u32   compaction map (0: unreached, else new index + 1)
//   heap  [heap_cap + 2] uint2 {fx bits, hypothesis}
//   end_off, maxbt (sort cursors, then per-start node offsets), surf: u32 [cap + 4]; text [cap + 16]
__host__ __device__ inline unsigned long long nbest_long_nodes(uint32_t cap, uint32_t mm1) {
  return static_cast<unsigned long long>(cap) * mm1 + 64ull;
}
__host__ __device__ inline unsigned long long nbest_long_bytes(uint32_t cap, uint32_t mm1, uint32_t hyp_cap, uint32_t heap_cap) {
  const unsigned long long b = 36ull * nbest_long_nodes(cap, mm1) + 20ull * hyp_cap + 8ull * (heap_cap + 2) +
                               12ull * (cap + 4) + cap + 16;
  return (b + 255ull) & ~255ull;
}

__global__ void __launch_bounds__(256) nbest_long_kernel(const KModel M, const KBatch B, const NbestOut O,
                                                          const uint32_t *hyp_caps, uint32_t *long_need, uint32_t mm1,
                                                          uint32_t heap_cap, uint32_t nbest) {
  const Tile T;
  const uint32_t lane = T.lane;
  const uint32_t root = __ldg(&M.trie_node2[0]).x;
  const bool bf = M.flags & kFlagByteFallback;
  const uint32_t kNull = 0xFFFFFFFFu;
  const uint32_t warps = blockDim.x >> 5;
  for (uint32_t w = blockIdx.x * warps + (threadIdx.x >> 5); w < B.long_n; w += gridDim.x * warps) {
    const uint32_t sent = B.long_list[2 * w], cap = B.long_list[2 * w + 1], hyp_cap = hyp_caps[w];
    const unsigned long long node_cap = nbest_long_nodes(cap, mm1);
    uint8_t *sp = B.long_scratch + B.long_scratch_off[w];
    uint4 *node = reinterpret_cast<uint4 *>(sp); sp += 16ull * node_cap;
    uint4 *elist = reinterpret_cast<uint4 *>(sp); sp += 16ull * node_cap;
    uint4 *hyp = reinterpret_cast<uint4 *>(sp); sp += 16ull * hyp_cap;
    uint2 *heap = reinterpret_cast<uint2 *>(sp); sp += 8ull * (heap_cap + 2);
    uint32_t *nend = reinterpret_cast<uint32_t *>(sp); sp += 4ull * node_cap;
    uint32_t *fwd = reinterpret_cast<uint32_t *>(sp); sp += 4ull * hyp_cap;
    uint32_t *end_off = reinterpret_cast<uint32_t *>(sp); sp += 4ull * (cap + 4);
    float *maxbt = reinterpret_cast<float *>(sp); sp += 4ull * (cap + 4);
    uint32_t *surf = reinterpret_cast<uint32_t *>(sp); sp += 4ull * (cap + 4);
    uint8_t *text = sp;
    uint32_t *nstart = reinterpret_cast<uint32_t *>(maxbt);  // per-start node offsets (before the backtrace fold)
    const NbestAgenda<0> ag{nullptr, heap};
    const size_t cbase = static_cast<size_t>(sent) * nbest;

    TileMem tm{};
    tm.text = text;
    tm.ncap = cap;
    const unsigned long long off = B.offsets[sent];
    const uint32_t n = normalize_tile<false>(M, T, B.bytes + off, static_cast<uint32_t>(B.offsets[sent + 1] - off), tm).n;
    if (n > cap) {  // the slab was sized from an upper bound of the normalized length
      if (lane == 0) atomicOr(O.status + 1, 8u);
      continue;
    }
    uint32_t K = 0;
    if (n == 0) {
      if (lane == 0) { O.cand_start[cbase] = 0; O.cand_count[cbase] = 0; O.cand_score[cbase] = 0.f; }
      K = 1;
    } else {
      const uint32_t L = long_char_starts(text, n, surf, lane);
      auto text_byte = [&](uint32_t k) -> uint32_t { return text[k]; };
      // ---- Model::PopulateNodes: count the nodes of every start, then write them at their offsets ----
      uint32_t nn = 2;  // BOS, EOS
      for (uint32_t b0 = 0; b0 < L; b0 += 32) {
        const uint32_t bp = b0 + lane;
        uint32_t cnt = 0;
        if (bp < L) {
          const bool single = populate_from(M, text_byte, root, surf, bp, n, [&](uint32_t, uint32_t, float) { ++cnt; return true; });
          cnt += single ? 0u : 1u;
        }
        const uint32_t incl = T.incl_scan(cnt);
        if (bp < L) nstart[bp] = nn + incl - cnt;
        nn += T.shfl(incl, 31);
      }
      if (nn > node_cap) {  // more matches per start than the model's trie reports
        if (lane == 0) atomicOr(O.status + 1, 16u);
        continue;
      }
      __syncwarp();
      for (uint32_t bp = lane; bp < L; bp += 32) {
        uint32_t k = nstart[bp];
        const bool single = populate_from(M, text_byte, root, surf, bp, n, [&](uint32_t length, uint32_t v, float sc) {
          node[k] = make_uint4(static_cast<uint32_t>(__ldg(M.trie_id + v)), __float_as_uint(sc), 0u, bp);
          nend[k++] = bp + length;
          return true;
        });
        if (!single) {
          node[k] = make_uint4(static_cast<uint32_t>(M.unk_id), __float_as_uint(M.unk_score), 0u, bp);
          nend[k] = bp + 1;
        }
      }
      for (uint32_t p = lane; p <= L + 1; p += 32) { maxbt[p] = -INFINITY; end_off[p] = 0; }
      for (uint32_t i = lane; i < hyp_cap; i += 32) fwd[i] = 0;
      __syncwarp();
      if (lane == 0) {
        node[0] = make_uint4(kNull, 0u, 0u, 0u);
        node[1] = make_uint4(kNull, 0u, 0u, L);
        nend[0] = 0;
        nend[1] = L + 1;
        // ---- Lattice::Viterbi's backtrace scores, in node (begin) order as in nbest_lane_kernel ----
        maxbt[0] = 0.f;
        for (uint32_t i = 2; i < nn; ++i) {
          const uint4 nd = node[i];
          const uint32_t e = nend[i];
          const float bt = __fadd_rn(maxbt[nd.w], __uint_as_float(nd.y));
          node[i].z = __float_as_uint(bt);
          maxbt[e] = fmaxf(maxbt[e], bt);
          end_off[e + 1] += 1;
        }
        const float eos_bt = __fadd_rn(maxbt[L], 0.f);
        // end_nodes lists in insertion order (stable counting sort by end character); BOS is the list of 0
        end_off[0 + 1] += 1;
        for (uint32_t p = 0; p <= L; ++p) end_off[p + 1] += end_off[p];
        uint32_t *sort_cur = reinterpret_cast<uint32_t *>(maxbt);  // maxbt is dead once eos_bt is known
        for (uint32_t p = 0; p <= L; ++p) sort_cur[p] = end_off[p];
        elist[sort_cur[0]++] = make_uint4(0u, 0u, 0u, 0u);
        for (uint32_t i = 2; i < nn; ++i) {
          const uint4 nd = node[i];
          const uint32_t e = nend[i];
          const bool isunk = static_cast<int32_t>(nd.x) == M.unk_id;
          const uint32_t contrib = (isunk && bf) ? surf[e] - surf[nd.w] : 1u;
          elist[sort_cur[e]++] = make_uint4(i, nd.z, nd.y, contrib | (isunk ? 0x80000000u : 0u));
        }
        // ---- Lattice::NBest: backward A* ----
        uint32_t pn = 1, hn = 0, need = 0;
        hyp[0] = make_uint4(kNull, 0u, 1u, 0u);  // EOS: next = null, gx = 0, no ids yet
        ag.push(hn, make_uint2(__float_as_uint(eos_bt), 0u));
        const uint32_t shrink_to = nbest * 10 < 512 ? nbest * 10 : 512;
        while (hn) {
          const uint2 te = ag.pop(hn);
          const uint4 th = hyp[te.y];
          if (th.z == 0) {  // reached BOS: one result
            nbest_write_result(M, O, cbase + K, th.w, __uint_as_float(te.x), surf, text_byte, [&](auto &&emit) {
              for (uint4 h = hyp[th.x]; h.x != kNull; h = hyp[h.x]) emit(static_cast<int32_t>(node[h.z].x), node[h.z].w, nend[h.z]);
            });
            if (++K == nbest) break;
            continue;
          }
          // expand: one hypothesis per node ending where this one begins, in end_nodes order
          const uint4 tn = node[th.z];
          const uint32_t p0 = tn.w;
          const bool top_unk = static_cast<int32_t>(tn.x) == M.unk_id;
          const float top_gx = __uint_as_float(th.y);
          uint32_t q = end_off[p0];
          const uint32_t qe = end_off[p0 + 1];
          if (hn + (qe - q) + 1 >= heap_cap - 512u) {  // more nodes end at one character than the agenda's slack
            atomicOr(O.status + 1, 16u);
            break;
          }
          if (pn + (qe - q) > hyp_cap) { need = 2u * hyp_cap > hyp_cap ? 2u * hyp_cap : 0xFFFFFFFFu; break; }
          for (; q < qe; ++q) {
            const uint4 rec = elist[q];
            uint32_t cn = th.w + (rec.w & 0x7FFFFFFFu);
            if (!bf && (rec.w >> 31) && top_unk) --cn;
            hyp[pn] = make_uint4(te.y, __float_as_uint(__fadd_rn(__uint_as_float(rec.z), top_gx)), rec.x, cn);
            ag.push(hn, make_uint2(__float_as_uint(__fadd_rn(__uint_as_float(rec.y), top_gx)), pn));
            ++pn;
          }
          if (hn >= 10000u) {  // agenda shrink (:481-505)
            uint2 *keep = heap + (heap_cap + 1 - shrink_to);
            ag.shrink_pop(hn, keep, shrink_to);
            if (pn <= hyp_cap / 2) {
              for (uint32_t i = 0; i < shrink_to; ++i) ag.push(hn, keep[i]);
              continue;
            }
            // compaction: mark what the kept entries reach, then move the marked hypotheses down in index order
            // (`next` always points to a lower index, so it is remapped before it is needed)
            for (uint32_t i = 0; i < shrink_to; ++i)
              for (uint32_t h = keep[i].y; h != kNull && fwd[h] == 0; h = hyp[h].x) fwd[h] = 1;
            uint32_t np = 0;
            for (uint32_t i = 0; i < pn; ++i) {
              if (!fwd[i]) continue;
              uint4 r = hyp[i];
              if (r.x != kNull) r.x = fwd[r.x] - 1;
              hyp[np] = r;
              fwd[i] = ++np;
            }
            for (uint32_t i = 0; i < shrink_to; ++i) ag.push(hn, make_uint2(keep[i].x, fwd[keep[i].y] - 1));
            for (uint32_t i = 0; i < pn; ++i) fwd[i] = 0;
            pn = np;
          }
        }
        long_need[w] = need;
      }
      K = T.shfl(K, 0);
    }
    if (lane == 0) O.n_cands[sent] = K;
    for (uint32_t k = K + lane; k < nbest; k += 32) { O.cand_count[cbase + k] = 0; O.cand_start[cbase + k] = 0; O.cand_score[cbase + k] = 0.f; }
    __syncwarp();
  }
}

// picked candidate per sentence -> (start, count) for the shared scan + gather
__global__ void __launch_bounds__(256) pick_candidates_kernel(const uint32_t *picks, uint32_t n, uint32_t nbest,
                                                              const unsigned long long *cand_start,
                                                              const uint32_t *cand_count, unsigned long long *sent_start,
                                                              uint32_t *sent_count) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t c = static_cast<size_t>(i) * nbest + picks[i];
  sent_start[i] = cand_start[c];
  sent_count[i] = cand_count[c];
}

}  // namespace spm_b200
#endif
