// bpe_lane2_kernel.cuh -- K3 fast path: BPE merge, one sentence per LANE, with WORDS as the unit of merge work.
//
// Reference: bpe::Model::SampleEncode with alpha = 0 (src/bpe_model.cc:38-203): repeat "merge the live
// adjacent pair with the greatest score, leftmost on ties" (the agenda's order, :51-57) until no adjacent pair is
// a piece.
//
// Exact decomposition used here (SURVEY.md 7, verified there on 20,000 sentences and by the parity tests): when no
// piece contains U+2581 anywhere but at byte 0 (the default split_by_whitespace=true vocabulary; checked at load,
// kFlagBpeWordSplit), a merge can never join a symbol with a following "▁..." symbol, so a sentence falls apart into
// independent words (▁ + following characters).  The greedy loop only ever compares raw piece scores, so running it
// per word gives exactly the reference's ids, and the ids of a word are a pure function of its bytes.
//
// Merging each lane's own words one at a time would leave most lanes idle: every lane would wait for the longest word
// of the warp, at every word.  Instead the warp works in two converged phases:
//   A  every lane scans ITS sentence byte by byte, walking the piece trie from the start of each word.  A word
//      that is itself a piece whose merge sequence reproduces it (M.word_fast[unit] = its id, computed at load
//      by running the reference's merge loop on the piece, engine.cu) is finished with that one id: 73 % of the
//      words of the English corpus.  Any other word is appended to a per-warp list in shared memory and gets a
//      run of slots (one per character, the most symbols it can end with) in its sentence's symbol log.
//   B  whenever the list fills up (and at the end), the 32 lanes each take one listed WORD -- of any sentence of
//      the warp -- and run the merge loop on it (bpe_merge_word) with tiny symbol arrays in shared memory
//      ([slot][lane], bank == lane) that cache the trie node of every symbol, so that "is left+right a piece?"
//      walks only the right symbol's bytes; the symbols go to the reserved log slots, unused slots are marked empty.
//   K4 each lane turns its sentence's log into ids (unk-run merging / byte fallback).
//
// Engine-side preconditions (else the general warp kernel of bpe_kernel.cuh runs): kFlagBpeWordSplit,
// escape_whitespaces, no user-defined symbols, no UNUSED pieces.  A word of more than kBpeWordSyms characters runs
// the same merge loop with its symbol arrays in HBM scratch (rare; no sentence is deferred for it: the fused host
// path has no second pass).
#ifndef SPM_B200_BPE_LANE2_KERNEL_CUH_
#define SPM_B200_BPE_LANE2_KERNEL_CUH_

#include "lane_kernel.cuh"

namespace spm_b200 {

constexpr uint32_t kBpeWordSyms = 24;       // symbols of one word held in shared memory
constexpr uint32_t kBpeDead = 0x3FFFFFu;    // 22-bit node field: not a trie path / not a piece
constexpr uint32_t kBpeListCap = 128;       // slow words listed per warp before a phase-B drain
constexpr uint32_t kBpeLogEmpty = 0xFFFFFFFFu;
constexpr uint32_t kBpeSymArrayBytes = kBpeWordSyms * 32 * 4 * 3;               // sym, pn, ps of 32 lanes
constexpr uint32_t kBpeLane2WarpBytes = kBpeSymArrayBytes + kBpeListCap * 8;   // + the word list

// ---- word cache ----
// Under the word-split condition the ids of a word are a pure function of its bytes, and natural text repeats its
// words: a word that is not a piece itself (word_fast) is looked up in a hash table in HBM (L2-resident: 2^18 entries
// of 64 bytes) before the merge loop is run on it, and entered after.  Entry (16 words):
//   [0] tag: 0 empty, 1 being written, else hash | 2     [1] byte length | symbols << 8
//   [2..8] the word's bytes, zero padded (<= kBpeKeyBytes)  [9..14] its symbols as log entries (<= kBpeCacheSyms)
// One slot per hash, first come first served, never evicted; the table is emptied when the model's tables change
// (engine.cu).  A writer claims the tag with a CAS, writes the entry, and releases the tag; a reader acquires the tag
// and then reads the entry through L2 (__ldcg: the L1 of another SM may hold a stale copy of the line).
constexpr uint32_t kBpeKeyBytes = 28;
constexpr uint32_t kBpeCacheSyms = 6;

struct BpeKey {
  uint32_t w[7];
  uint32_t hash;
};

// the word's bytes [p, p + blen) of text column `tw` as 7 zero-padded little-endian words + their hash (blen <= 28)
__device__ __forceinline__ void bpe_word_key(const uint32_t *tw, uint32_t p, uint32_t blen, BpeKey &k) {
  const uint32_t pw = p >> 2, sh = (p & 3u) * 8u;
  const uint32_t need = (p & 3u) + blen;  // bytes from the start of word pw
  uint32_t r[8];
#pragma unroll
  for (uint32_t i = 0; i < 8; ++i) r[i] = 4u * i < need ? tw[static_cast<size_t>(pw + i) * 32] : 0u;
  uint32_t h = 0x9E3779B9u ^ blen;
#pragma unroll
  for (uint32_t i = 0; i < 7; ++i) {
    uint32_t v = __funnelshift_r(r[i], r[i + 1], sh);
    if (blen < 4u * i + 4u) v = blen <= 4u * i ? 0u : (v & ((1u << (8u * (blen - 4u * i))) - 1u));
    k.w[i] = v;
    h = (h ^ v) * 0x85EBCA6Bu;
    h ^= h >> 13;
  }
  h *= 0xC2B2AE35u;
  h ^= h >> 16;
  k.hash = h;
}

// a hit writes the word's m0 log slots at `lg` (symbols, then empty markers) and returns true
__device__ __forceinline__ bool bpe_cache_lookup(const KModel &M, const uint32_t *tw, uint32_t p, uint32_t blen,
                                                 uint32_t m0, uint32_t *lg) {
  BpeKey k;
  bpe_word_key(tw, p, blen, k);
  const uint4 *e = M.bpe_cache + static_cast<size_t>((k.hash >> 7) & M.bpe_cache_mask) * 4;
  uint32_t t;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(t) : "l"(e) : "memory");
  if (t != (k.hash | 2u)) return false;
  const uint4 q0 = __ldcg(e), q1 = __ldcg(e + 1), q2 = __ldcg(e + 2), q3 = __ldcg(e + 3);
  if ((q0.y & 0xFFu) != blen || q0.z != k.w[0] || q0.w != k.w[1] || q1.x != k.w[2] || q1.y != k.w[3] || q1.z != k.w[4] ||
      q1.w != k.w[5] || q2.x != k.w[6])
    return false;
  const uint32_t cnt = q0.y >> 8;
  const uint32_t pay[kBpeCacheSyms] = {q2.y, q2.z, q2.w, q3.x, q3.y, q3.z};
#pragma unroll
  for (uint32_t i = 0; i < kBpeCacheSyms; ++i)
    if (i < m0) lg[static_cast<size_t>(i) * 32] = i < cnt ? pay[i] : 0xFFFFFFFFu;
  for (uint32_t i = kBpeCacheSyms; i < m0; ++i) lg[static_cast<size_t>(i) * 32] = 0xFFFFFFFFu;
  return true;
}

// enters a merged word (its `cnt` <= kBpeCacheSyms symbols are the first log entries at `lg`) if its slot is free
__device__ __forceinline__ void bpe_cache_insert(const KModel &M, const uint32_t *tw, uint32_t p, uint32_t blen,
                                                 uint32_t cnt, const uint32_t *lg) {
  BpeKey k;
  bpe_word_key(tw, p, blen, k);
  uint4 *e = M.bpe_cache + static_cast<size_t>((k.hash >> 7) & M.bpe_cache_mask) * 4;
  uint32_t *tp = reinterpret_cast<uint32_t *>(e);
  if (*reinterpret_cast<volatile uint32_t *>(tp) != 0u) return;  // taken (by this word or another)
  if (atomicCAS(tp, 0u, 1u) != 0u) return;
  uint32_t pay[kBpeCacheSyms];
#pragma unroll
  for (uint32_t i = 0; i < kBpeCacheSyms; ++i) pay[i] = i < cnt ? __ldcg(lg + static_cast<size_t>(i) * 32) : 0xFFFFFFFFu;
  tp[1] = blen | (cnt << 8);
  tp[2] = k.w[0];
  tp[3] = k.w[1];
  __stcg(e + 1, make_uint4(k.w[2], k.w[3], k.w[4], k.w[5]));
  __stcg(e + 2, make_uint4(k.w[6], pay[0], pay[1], pay[2]));
  __stcg(e + 3, make_uint4(pay[3], pay[4], pay[5], 0u));
  const uint32_t tag = k.hash | 2u;
  asm volatile("st.release.gpu.global.u32 [%0], %1;" :: "l"(tp), "r"(tag) : "memory");
}

// The reference's merge loop on ONE word (bpe_model.cc:110-173 restricted to the word, see the header): the word is
// `m0` characters starting at byte `p` of the text column `tw`; its symbols end up in the m0 log slots at `lg`
// (unused slots marked empty); returns the number of symbols.  sym / pn / ps are the symbol arrays, element i at [i * st]: shared memory with
// st = 32 for words of <= kBpeWordSyms characters, the warp's scratch in HBM with st = 1 for longer ones.
__device__ __forceinline__ uint32_t bpe_merge_word(const KModel &M, const uint32_t *tlink, uint32_t root, const uint32_t *tw,
                                               uint32_t p, uint32_t m0, uint32_t *lg, uint32_t *sym, uint32_t *pn,
                                               float *ps, const uint32_t st) {
  // the first 16 bytes of the word's text in registers (every byte is read several times: character split,
  // every pair evaluation); longer words read their tail from the slab
  const uint32_t pw = p >> 2;
  const uint32_t r0 = tw[static_cast<size_t>(pw) * 32], r1 = tw[static_cast<size_t>(pw + 1) * 32],
                 r2 = tw[static_cast<size_t>(pw + 2) * 32], r3 = tw[static_cast<size_t>(pw + 3) * 32];
  auto text_byte = [&](uint32_t k) -> uint32_t {
    const uint32_t wi = (k >> 2) - pw;
    uint32_t w;
    if (wi < 4u) w = (wi & 2u) ? ((wi & 1u) ? r3 : r2) : ((wi & 1u) ? r1 : r0);
    else w = tw[static_cast<size_t>(k >> 2) * 32];
    return (w >> ((k & 3u) * 8u)) & 0xFFu;
  };
  // walks `len` bytes at text offset `off` from link word `l`; returns the node reached or kBpeDead
  auto walk = [&](uint32_t l, uint32_t off, uint32_t len, uint32_t *link_out) -> uint32_t {
    uint32_t v = kBpeDead;
    for (uint32_t i = 0; i < len; ++i) {
      const uint32_t ch = text_byte(off + i);
      v = (l >> kLinkBaseShift) ^ ch;
      l = __ldg(&tlink[v]);
      if ((l & kLinkLabelMask) != ch) return kBpeDead;
    }
    *link_out = l;
    return v;
  };
  // -- split the word into characters (bpe_model.cc:110-120) and cache their trie nodes --
  uint32_t m = 0, q = p;
  for (; m < m0; ++m) {
    uint32_t l = one_char_len(text_byte(q));
    uint32_t lk = 0;
    const uint32_t node = walk(root, q, l, &lk);
    sym[m * st] = node | (l << 22);
    pn[m * st] = kBpeDead | ((q - p) << 22);
    q += l;
  }
  // MaybeAddNewSymbolPair (bpe_model.cc:83-107) for the pair (i, i+1)
  auto eval_pair = [&](uint32_t i) {
    const uint32_t si = sym[i * st], sj = sym[(i + 1) * st];
    const uint32_t offj = pn[(i + 1) * st] >> 22;
    uint32_t res = kBpeDead;
    float score = 0.f;
    if ((si & 0x3FFFFFu) != kBpeDead) {
      uint32_t lk = 0;
      const uint32_t v = walk(__ldg(&tlink[si & 0x3FFFFFu]), p + offj, sj >> 22, &lk);
      if (v != kBpeDead && ((lk >> kLinkKindShift) & 3u) != kKindNone) {
        res = v;
        score = __uint_as_float(__ldg(M.trie_val + v));
      }
    }
    pn[i * st] = res | (pn[i * st] & 0xFFC00000u);
    ps[i * st] = score;
  };
  for (uint32_t i = 0; i + 1 < m; ++i) eval_pair(i);
  // -- greedy merges: best score, leftmost on ties (bpe_model.cc:51-57,141-173) --
  for (;;) {
    int bi = -1;
    float best = 0.f;
    for (uint32_t i = 0; i + 1 < m; ++i) {
      if ((pn[i * st] & 0x3FFFFFu) != kBpeDead) {
        const float sc = ps[i * st];
        if (bi < 0 || sc > best) { best = sc; bi = static_cast<int>(i); }
      }
    }
    if (bi < 0) break;
    const uint32_t i = static_cast<uint32_t>(bi);
    const uint32_t nl = (sym[i * st] >> 22) + (sym[(i + 1) * st] >> 22);
    sym[i * st] = (pn[i * st] & 0x3FFFFFu) | (nl << 22);
    for (uint32_t jj = i + 1; jj + 1 < m; ++jj) {  // close the gap
      sym[jj * st] = sym[(jj + 1) * st];
      pn[jj * st] = pn[(jj + 1) * st];
      ps[jj * st] = ps[(jj + 1) * st];
    }
    --m;
    if (i > 0) eval_pair(i - 1);
    if (i + 1 < m) eval_pair(i);
    else pn[i * st] = kBpeDead | (pn[i * st] & 0xFFC00000u);
  }
  // -- the word's symbols go to its slots of the owner's log: PieceToId (model_interface.cc:51-61) --
  for (uint32_t i = 0; i < m0; ++i) {
    uint32_t entry = kBpeLogEmpty;
    if (i < m) {
      const uint32_t s = sym[i * st];
      int32_t id = M.unk_id;
      if ((s & 0x3FFFFFu) != kBpeDead) {
        const int32_t t = __ldg(M.trie_id + (s & 0x3FFFFFu));
        if (t >= 0) id = t;
      }
      entry = static_cast<uint32_t>(id) | ((s >> 22) << 24);
    }
    lg[static_cast<size_t>(i) * 32] = entry;
  }
  return m;  // symbols the word ended with
}

// scratch in HBM for the symbol arrays of a long word (one word at a time per warp): sym, pn, ps of cap + 4 entries
__host__ __device__ inline unsigned long long bpe_long_bytes(uint32_t cap) { return 3ull * (cap + 4u) * 4ull; }

__global__ void __launch_bounds__(704, 1) encode_bpe_lane2_kernel(const KModel M, const KBatch B, uint8_t *slabs,
                                                                   uint32_t cap, uint8_t *long_scratch) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint32_t *s_tab = reinterpret_cast<uint32_t *>(smem);
  uint8_t *arrays = smem + kLaneTableBytes;
  fill_lane_tables(M, s_tab);
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp_in_cta = threadIdx.x >> 5;
  const uint32_t warp_global = blockIdx.x * (blockDim.x >> 5) + warp_in_cta;
  const LaneCtx c = lane_ctx(s_tab, slabs, cap, warp_global, lane);
  uint32_t *const text_all = c.text_w - lane;  // the warp's slab without the lane offset (phase B reads other lanes' columns)
  uint32_t *const log_all = c.log - lane;
  uint32_t *sym, *pn, *list;
  float *ps;
  {
    uint8_t *a = arrays + static_cast<size_t>(warp_in_cta) * kBpeLane2WarpBytes;
    sym = reinterpret_cast<uint32_t *>(a) + lane;                             // node(22) | byte_len << 22
    pn = reinterpret_cast<uint32_t *>(a + kBpeWordSyms * 32 * 4) + lane;      // pair node(22) | offset_in_word << 22
    ps = reinterpret_cast<float *>(a + kBpeWordSyms * 32 * 8) + lane;         // pair score
    list = reinterpret_cast<uint32_t *>(a + kBpeSymArrayBytes);               // [kBpeListCap][2]
    long_scratch += static_cast<size_t>(warp_global) * bpe_long_bytes(cap);
  }
  const uint32_t *tlink = M.trie_link;
  const uint32_t root = __ldg(&tlink[0]);
  const bool bf = M.flags & kFlagByteFallback;

  uint32_t first = 0;
  while (lane_claim_group(B, lane, &first)) {
    LanePhaseClock clk(B);
    lane_wait_input(B, first, lane);
    const bool have = first + lane < B.n;
    const uint32_t sent = have && B.order ? B.order[first + lane] : first + lane;
    // ---------------- K1 ----------------
    uint32_t n = 0;
    bool defer = false;
    if (have) defer = !lane_k1(M, B, c, sent, cap, &n);  // recorded after phase B
    __syncwarp();  // the text of every lane is visible to the whole warp (phase B)
    clk.mark();

    // ---------------- phase B: one listed word per lane ----------------
    uint32_t count = 0;  // words in the list (warp-uniform)
    auto drain = [&]() {
      // Pass 1: every listed word is looked up in the word cache (all lanes together); the misses are compacted to
      // the front of the list for the merge rounds.
      if (M.bpe_cache_mask) {
        uint32_t kept = 0;
        for (uint32_t j0 = 0; j0 < count; j0 += 32) {
          const uint32_t j = j0 + lane;
          uint32_t e0 = 0, e1 = 0;
          bool miss = false;
          if (j < count) {
            e0 = list[2 * j]; e1 = list[2 * j + 1];
            const uint32_t blen = (e0 >> 15) & 0x3FFu, m0 = e1 & 0xFFFu;
            miss = !(blen <= kBpeKeyBytes && m0 <= kBpeWordSyms &&
                     bpe_cache_lookup(M, text_all + (e0 & 31u), (e0 >> 5) & 0x3FFu, blen, m0,
                                      log_all + (e0 & 31u) + static_cast<size_t>(e1 >> 12) * 32));
          }
          const uint32_t keep = __ballot_sync(0xFFFFFFFFu, miss);  // (also: this round's entries are in registers)
          if (miss) {
            const uint32_t d = kept + __popc(keep & ((1u << lane) - 1u));  // <= j: never ahead of the reads
            list[2 * d] = e0; list[2 * d + 1] = e1;
          }
          kept += __popc(keep);
          __syncwarp();
        }
        count = kept;
      }
      // The 32 words of a round cost what the longest of them costs (the merge loop is ~quadratic in the symbols), so
      // the list is first ordered by symbol count, longest first: a counting sort through the (now idle) `ps` array,
      // entries permuted in place by way of registers.  Which lane merges which word does not matter for the result:
      // every word writes to its own reserved log slots.
      if (count > 32u) {
        uint32_t *hist = reinterpret_cast<uint32_t *>(ps - lane);  // [kBpeWordSyms + 2] counters, lane-less view
        if (lane < kBpeWordSyms + 2u) hist[lane] = 0u;
        __syncwarp();
        uint32_t e0r[kBpeListCap / 32], e1r[kBpeListCap / 32], rk[kBpeListCap / 32], bk[kBpeListCap / 32];
#pragma unroll
        for (uint32_t t = 0; t < kBpeListCap / 32; ++t) {
          const uint32_t j = t * 32u + lane;
          bk[t] = 0xFFFFFFFFu;
          if (j < count) {
            e0r[t] = list[2 * j]; e1r[t] = list[2 * j + 1];
            bk[t] = kBpeWordSyms + 1u - min(e1r[t] & 0xFFFu, kBpeWordSyms + 1u);  // 0 = the long words, then 24, 23, ...
            rk[t] = atomicAdd(&hist[bk[t]], 1u);
          }
        }
        __syncwarp();
        {  // exclusive scan of the kBpeWordSyms + 2 (< 32) counters
          const uint32_t v = lane < kBpeWordSyms + 2u ? hist[lane] : 0u;
          uint32_t incl = v;
#pragma unroll
          for (int d = 1; d < 32; d <<= 1) {
            const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, d);
            if (lane >= static_cast<uint32_t>(d)) incl += u;
          }
          __syncwarp();
          if (lane < kBpeWordSyms + 2u) hist[lane] = incl - v;
        }
        __syncwarp();
#pragma unroll
        for (uint32_t t = 0; t < kBpeListCap / 32; ++t) {
          if (bk[t] != 0xFFFFFFFFu) {
            const uint32_t d = hist[bk[t]] + rk[t];
            list[2 * d] = e0r[t]; list[2 * d + 1] = e1r[t];
          }
        }
        __syncwarp();
      }
      for (uint32_t j0 = 0; j0 < count; j0 += 32) {
        const uint32_t j = j0 + lane;
        uint32_t owner = 0, p = 0, m0 = 0, slot = 0;
        if (j < count) {
          const uint32_t e0 = list[2 * j], e1 = list[2 * j + 1];
          owner = e0 & 31u; p = (e0 >> 5) & 0x3FFu;  // sentence (lane) and text position of the word
          m0 = e1 & 0xFFFu; slot = e1 >> 12;         // characters, first log slot
          if (m0 <= kBpeWordSyms) {
            uint32_t *lg = log_all + owner + static_cast<size_t>(slot) * 32;
            const uint32_t mm = bpe_merge_word(M, tlink, root, text_all + owner, p, m0, lg, sym, pn, ps, 32u);
            const uint32_t blen = (e0 >> 15) & 0x3FFu;
            if (M.bpe_cache_mask && blen <= kBpeKeyBytes && mm <= kBpeCacheSyms)
              bpe_cache_insert(M, text_all + owner, p, blen, mm, lg);
          }
        }
        // words of more symbols than the shared arrays hold (URLs, long numbers: ~0.4 per 1000 sentences of the bench
        // corpus): one at a time, on the lane that drew the word, with the symbol arrays in the warp's HBM scratch
        for (uint32_t todo = __ballot_sync(0xFFFFFFFFu, m0 > kBpeWordSyms); todo; todo &= todo - 1u) {
          if (lane == static_cast<uint32_t>(__ffs(todo)) - 1u) {
            uint32_t *g = reinterpret_cast<uint32_t *>(long_scratch);
            bpe_merge_word(M, tlink, root, text_all + owner, p, m0, log_all + owner + static_cast<size_t>(slot) * 32, g,
                           g + (cap + 4u), reinterpret_cast<float *>(g + 2u * (cap + 4u)), 1u);
          }
          __syncwarp();
        }
      }
      count = 0;
      __syncwarp();
    };

    // ---------------- phase A: byte scan, one byte per trip for every lane ----------------
    uint32_t k = 0, wp = 0, m = 0, l = root, v = kBpeDead, nlog = 0;
    bool alive = true, active = n != 0 && !defer;
    uint32_t wa = 0, wb = 0;  // text words k >> 2 and (k >> 2) + 1
    if (active) { wa = c.text_w[0]; wb = c.text_w[32]; }
    while (__any_sync(0xFFFFFFFFu, active)) {
      bool slow = false;
      uint32_t slow_p = 0, slow_m = 0, slow_slot = 0, slow_b = 0;
      if (active) {
        const uint32_t b3 = __funnelshift_r(wa, wb, (k & 3u) * 8u);
        const uint32_t ch = b3 & 0xFFu;
        const bool at_end = k >= n;
        const bool end_here = at_end || ((b3 & 0xFFFFFFu) == kWsWord && k > wp && k + 3u <= n);
        // the step of byte k is issued first: after a word end it starts from the root, so its load does not
        // depend on the loads of the finalize block
        const uint32_t l_step = end_here ? root : l;
        const bool alive_step = end_here || alive;
        const uint32_t v_step = (l_step >> kLinkBaseShift) ^ ch;
        uint32_t nl = 0;
        if (alive_step && !at_end) nl = __ldg(&tlink[v_step]);
        if (end_here) {
          // ---- the word [wp, k) is complete ----
          uint32_t fast_id = 0xFFFFFFFFu;
          if (alive && ((l >> kLinkKindShift) & 3u) != kKindNone) fast_id = __ldg(M.word_fast + v);
          if (fast_id != 0xFFFFFFFFu) {
            c.log[static_cast<size_t>(nlog) * 32] = fast_id | ((k - wp) << 24);
            ++nlog;
          } else {
            slow = true;
            slow_p = wp; slow_m = m; slow_slot = nlog; slow_b = k - wp;
            nlog += m;
          }
          wp = k;
          m = 0;
        }
        if (at_end || defer) {
          active = false;
        } else {
          m += (ch & 0xC0u) != 0x80u;  // characters of the word so far
          alive = alive_step && (nl & kLinkLabelMask) == ch;
          l = nl;
          v = v_step;
          ++k;
          if ((k & 3u) == 0u) {
            wa = wb;
            wb = c.text_w[static_cast<size_t>((k >> 2) + 1) * 32];
          }
        }
      }
      // list the slow words of this trip (warp-aggregated allocation), drain when the list may overflow next trip
      const uint32_t m_slow = __ballot_sync(0xFFFFFFFFu, slow);
      if (m_slow) {
        if (slow) {
          const uint32_t idx = count + __popc(m_slow & ((1u << lane) - 1u));
          list[2 * idx] = lane | (slow_p << 5) | (slow_b << 15);  // (cap <= 1020: 10 bits each)
          list[2 * idx + 1] = slow_m | (slow_slot << 12);
        }
        count += __popc(m_slow);
        __syncwarp();
        if (count + 32u > kBpeListCap) drain();
      }
    }
    if (count) drain();
    if (have && defer) {
      lane_defer(B, sent);
      nlog = 0;
    }
    clk.mark();
    // ---------------- K4: id path of PopulateSentencePieceText over the symbol log ----------------
    const uint32_t unk = static_cast<uint32_t>(M.unk_id);
    const uint32_t max_log = __reduce_max_sync(0xFFFFFFFFu, nlog);
    uint32_t cnt = 0;
    {
      bool prev_unk = false;
      for (uint32_t t = 0; t < max_log; ++t) {
        if (t < nlog) {
          const uint32_t e = c.log[static_cast<size_t>(t) * 32];
          if (e != kBpeLogEmpty) {
            const bool isunk = (e & 0xFFFFFFu) == unk;
            if (bf) cnt += isunk ? (e >> 24) : 1u;
            else cnt += !(isunk && prev_unk);
            prev_unk = isunk;
          }
        }
      }
    }
    bool room;
    const unsigned long long pos = lane_claim_output(B, lane, cnt, have, defer, sent, &room);
    if (room) {
      bool prev_unk = false;
      uint32_t w = 0, off = 0;
      for (uint32_t t = 0; t < max_log; ++t) {
        if (t < nlog) {
          const uint32_t e = c.log[static_cast<size_t>(t) * 32];
          if (e != kBpeLogEmpty) {
            const uint32_t plen = e >> 24;
            const bool isunk = (e & 0xFFFFFFu) == unk;
            if (isunk) {
              if (bf) {
                for (uint32_t i = 0; i < plen; ++i)
                  __stcs(B.tmp_ids + pos + (w++), __ldg(M.byte_to_id + lane_text_byte_plain(c, off + i)));
              } else if (!prev_unk) {
                __stcs(B.tmp_ids + pos + (w++), M.unk_id);
              }
            } else {
              __stcs(B.tmp_ids + pos + (w++), static_cast<int32_t>(e & 0xFFFFFFu));
            }
            prev_unk = isunk;
            off += plen;
          }
        }
      }
    }
    slab_discard(c, lane, (__reduce_max_sync(0xFFFFFFFFu, n) >> 2) + 4u, max_log);
    clk.mark();
    lane_drain(B, sent, have, lane);  // K6 (fused host path only)
    __syncwarp();
    clk.flush(lane);
  }
}

}  // namespace spm_b200
#endif
