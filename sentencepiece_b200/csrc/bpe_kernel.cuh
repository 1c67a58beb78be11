// bpe_kernel.cuh -- K3: the BPE merge loop on the GPU.
//
// Reference: bpe::Model::SampleEncode with alpha = 0 (src/bpe_model.cc:38-203).
// The reference keeps a std::priority_queue of adjacent symbol pairs ordered by
// (score desc, left index asc) with lazy invalidation; since every live pair is in
// the queue exactly once (stale entries are skipped, :147-151) that is the same as
// "repeat: merge the live adjacent pair with the greatest score, leftmost on ties"
// (SURVEY.md 8a Q6).  The candidate test is membership of the CONCATENATION in
// pieces_ (:88-94), which here is an exact-match walk of the piece trie starting
// from the left symbol's cached trie node over the right symbol's bytes.
//
// One warp owns one sentence.  All state lives in shared memory arrays indexed by
// the byte position at which a symbol starts; each merge step is
//   (1) every lane scans its strided share of positions for the best live pair,
//   (2) a 64-bit warp max (ordered score bits, then leftmost) picks the winner,
//   (3) two lanes re-evaluate the two new neighbour pairs.
// UNUSED pieces (SetVocabulary) are re-split with the reference's rev_merge rule
// (:102-106,175-193): last recorded split of that string wins, in the reference's
// own insertion order, which this sentence-global merge order preserves.
#ifndef SPM_B200_BPE_KERNEL_CUH_
#define SPM_B200_BPE_KERNEL_CUH_

#include "kernels.cuh"

namespace spm_b200 {

constexpr uint32_t kDead = 0xFFFFFFFFu;

struct BpeMem {
  uint8_t *text;     // [ncap + 16]
  uint8_t *slen;     // [ncap + 4] symbol byte length at its start position, 0 elsewhere (pieces are <= 255 bytes)
  uint8_t *frozen;   // [ncap + 4] user-defined symbol: never merged (bpe_model.cc:85-87)
  uint32_t *snode;   // [ncap + 4] trie unit reached by the symbol's bytes, kDead if not a trie path
  uint32_t *pval;    // [ncap + 4] score bits of (symbol here + next symbol) when pnode != kDead
  uint32_t *pnode;   // [ncap + 4] trie unit of that concatenation, kDead if it is not a piece
  uint32_t *sprev;   // [ncap + 4] start of the previous live symbol, kDead for the first
  uint32_t *rm_node; // [ncap + 4] rev_merge keys (trie unit == string identity)
  uint16_t *rm_llen; // [ncap + 4] rev_merge: byte length of the left part
  uint32_t *aux;     // [ncap + 4] output ids of the resegmentation pass
  uint32_t *n2o;     // (spans)
  uint8_t *stage;
  uint32_t ncap, stage_cap;
};

__host__ __device__ inline uint32_t bpe_tile_bytes(uint32_t ncap, bool spans) {
  uint32_t b = (ncap + 16) + 2 * (ncap + 4);      // text, slen, frozen
  b += 4 * (ncap + 4) * 6;                        // snode, pval, pnode, rm_node, aux, sprev
  b += 2 * (ncap + 4);                            // rm_llen
  if (spans) b += 4 * (ncap + 4);
  return (b + 15u) & ~15u;
}

__device__ __forceinline__ BpeMem carve_bpe(uint8_t *base, uint32_t ncap, bool spans) {
  BpeMem m;
  uint8_t *p = base;
  m.pval = reinterpret_cast<uint32_t *>(p); p += 4 * (ncap + 4);
  m.pnode = reinterpret_cast<uint32_t *>(p); p += 4 * (ncap + 4);
  m.stage = reinterpret_cast<uint8_t *>(m.pval);
  m.stage_cap = 8 * (ncap + 4);
  m.snode = reinterpret_cast<uint32_t *>(p); p += 4 * (ncap + 4);
  m.rm_node = reinterpret_cast<uint32_t *>(p); p += 4 * (ncap + 4);
  m.aux = reinterpret_cast<uint32_t *>(p); p += 4 * (ncap + 4);
  m.sprev = reinterpret_cast<uint32_t *>(p); p += 4 * (ncap + 4);
  m.n2o = reinterpret_cast<uint32_t *>(p); if (spans) p += 4 * (ncap + 4);
  m.rm_llen = reinterpret_cast<uint16_t *>(p); p += 2 * (ncap + 4);
  m.slen = p; p += ncap + 4;
  m.frozen = p; p += ncap + 4;
  m.text = p;
  m.ncap = ncap;
  return m;
}

// Walks `len` bytes from trie unit `from` (link word `l`); returns the unit reached or kDead.
__device__ __forceinline__ uint32_t trie_walk(const HotTrie &H, uint32_t from, const uint8_t *p, uint32_t len,
                                              uint32_t *link_out) {
  uint32_t l = H.link(from);
  uint32_t v = from;
  for (uint32_t i = 0; i < len; ++i) {
    const uint32_t c = p[i];
    v = (l >> kLinkBaseShift) ^ c;
    l = H.link(v);
    if ((l & kLinkLabelMask) != c) return kDead;
  }
  *link_out = l;
  return v;
}

// MaybeAddNewSymbolPair (bpe_model.cc:83-107) for the pair (left symbol at a, right at b).
// Sets pnode[a]/pval[a]; returns true if the concatenation is an UNUSED piece.
__device__ __forceinline__ bool bpe_eval_pair(const HotTrie &H, const BpeMem &bm, uint32_t a, uint32_t b) {
  uint32_t res = kDead, val = 0;
  bool unused = false;
  if (!bm.frozen[a] && !bm.frozen[b] && bm.snode[a] != kDead) {
    uint32_t l = 0;
    const uint32_t v = trie_walk(H, bm.snode[a], bm.text + b, bm.slen[b], &l);
    if (v != kDead) {
      const uint32_t kind = (l >> kLinkKindShift) & 3u;
      if (kind != kKindNone) {  // pieces_ holds NORMAL, USER_DEFINED and UNUSED pieces
        res = v;
        val = H.val(v);
        unused = kind == kKindUnused;
      }
    }
  }
  bm.pnode[a] = res;
  bm.pval[a] = val;
  return unused;
}

// rev_merge[piece] = (left, right): keyed by string content (== trie unit), last write wins.
__device__ __forceinline__ void bpe_record_rev(const BpeMem &bm, uint32_t *n_rev, uint32_t node, uint32_t llen) {
  for (uint32_t i = 0; i < *n_rev; ++i)
    if (bm.rm_node[i] == node) { bm.rm_llen[i] = static_cast<uint16_t>(llen); return; }
  if (*n_rev < bm.ncap) {
    bm.rm_node[*n_rev] = node;
    bm.rm_llen[*n_rev] = static_cast<uint16_t>(llen);
  }
  ++*n_rev;
}

// monotone map float bits -> unsigned (so integer max == float max); -0.0 == +0.0
__device__ __forceinline__ uint32_t ordered_bits(uint32_t f) {
  if (f == 0x80000000u) f = 0;
  return (f & 0x80000000u) ? ~f : (f | 0x80000000u);
}

template <bool SPANS>
__device__ __forceinline__ bool encode_bpe_sentence(const KModel &M, const KBatch &B, const Tile &T, const HotTrie &H,
                                                    const BpeMem &bm, const uint8_t *in, uint32_t len, uint32_t sent,
                                                    uint32_t *need) {
  TileMem tm{};
  tm.text = bm.text;
  tm.n2o = bm.n2o;
  tm.ncap = bm.ncap;
  const NormResult nr = normalize_tile<SPANS>(M, T, in, len, tm);
  const uint32_t n = nr.n;
  if (n > bm.ncap) { *need = n; return false; }
  if (SPANS) publish_norm_tile(B, T, tm, sent, n, n > 0);
  if (n == 0) {
    if (T.lane == 0) { B.sent_start[sent] = 0; B.sent_count[sent] = 0; }
    return true;
  }
  const uint8_t *text = bm.text;
  const bool has_unused = M.flags & kFlagHasUnused;
  // ---- split into characters; user-defined symbols are frozen (bpe_model.cc:110-120) ----
  for (uint32_t k = T.lane; k <= n; k += 32) { bm.slen[k] = 0; bm.frozen[k] = 0; }
  T.sync();
  if (M.flags & kFlagHasUserSymbols) {
    if (T.lane == 0) {
      uint32_t p = 0;
      while (p < n) {
        const uint32_t ul = user_longest(M, text + p, n - p);
        uint32_t l = ul;
        if (!ul) { l = one_char_len(text[p]); if (l > n - p) l = n - p; }
        if (l > 255) l = 255;  // cannot happen: pieces are <= 255 bytes
        bm.slen[p] = static_cast<uint8_t>(l);
        bm.frozen[p] = ul != 0;
        p += l;
      }
    }
  } else {
    for (uint32_t k = T.lane; k < n; k += 32) {
      const uint32_t c = text[k];
      if (!is_trail(c)) {
        uint32_t l = one_char_len(c);
        if (l > n - k) l = n - k;
        bm.slen[k] = static_cast<uint8_t>(l);
      }
    }
  }
  T.sync();
  // prev links + per-symbol trie nodes
  {
    uint32_t carry = kDead;
    for (uint32_t w = 0; w < n; w += 32) {
      const uint32_t k = w + T.lane;
      const bool st = k < n && bm.slen[k] != 0;
      const uint32_t m = T.ballot(st);
      if (st) {
        const uint32_t below = m & T.below();
        bm.sprev[k] = below ? w + (31 - __clz(below)) : carry;
        uint32_t l = 0;
        bm.snode[k] = trie_walk(H, 0, text + k, bm.slen[k], &l);
      }
      if (m) carry = w + (31 - __clz(m));
    }
  }
  T.sync();
  // ---- all bigrams (bpe_model.cc:126-129), left to right ----
  uint32_t n_rev = 0;
  for (uint32_t w = 0; w < n; w += 32) {
    const uint32_t k = w + T.lane;
    bool unused = false;
    if (k < n && bm.slen[k]) {
      const uint32_t j = k + bm.slen[k];
      if (j < n) unused = bpe_eval_pair(H, bm, k, j);
      else { bm.pnode[k] = kDead; bm.pval[k] = 0; }
    }
    if (has_unused) {
      uint32_t um = T.ballot(unused);
      T.sync();
      if (T.lane == 0)
        while (um) {
          const uint32_t kk = w + (__ffs(um) - 1);
          um &= um - 1;
          bpe_record_rev(bm, &n_rev, bm.pnode[kk], bm.slen[kk]);
        }
    }
  }
  T.sync();
  // ---- main loop (bpe_model.cc:141-173) ----
  for (;;) {
    unsigned long long best = 0;
    for (uint32_t k = T.lane; k < n; k += 32) {
      if (bm.slen[k] && bm.pnode[k] != kDead) {
        const unsigned long long key =
            (static_cast<unsigned long long>(ordered_bits(bm.pval[k])) << 32) | (0xFFFFFFFFu - k);
        best = key > best ? key : best;
      }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      const unsigned long long o = __shfl_xor_sync(0xFFFFFFFFu, best, d);
      best = o > best ? o : best;
    }
    if (best == 0) break;
    const uint32_t a = 0xFFFFFFFFu - static_cast<uint32_t>(best & 0xFFFFFFFFull);
    const uint32_t b = a + bm.slen[a];
    const uint32_t nl = bm.slen[a] + bm.slen[b];
    const uint32_t nx = a + nl;  // symbol after the merged one
    const uint32_t pv = bm.sprev[a];
    T.sync();
    if (T.lane == 0) {
      bm.slen[a] = static_cast<uint8_t>(nl);
      bm.slen[b] = 0;
      bm.snode[a] = bm.pnode[a];
      if (nx < n) bm.sprev[nx] = a;
    }
    T.sync();
    bool unused = false;
    if (T.lane == 0 && pv != kDead) unused = bpe_eval_pair(H, bm, pv, a);
    if (T.lane == 1) {
      if (nx < n) unused = bpe_eval_pair(H, bm, a, nx);
      else { bm.pnode[a] = kDead; bm.pval[a] = 0; }
    }
    T.sync();
    if (has_unused) {
      const uint32_t um = T.ballot(unused);
      if (T.lane == 0) {
        if (um & 1u) bpe_record_rev(bm, &n_rev, bm.pnode[pv], bm.slen[pv]);
        if (um & 2u) bpe_record_rev(bm, &n_rev, bm.pnode[a], bm.slen[a]);
      }
      T.sync();
    }
  }
  n_rev = T.shfl(n_rev, 0);
  if (n_rev > bm.ncap) { *need = 3 * n + 8; return false; }  // rev_merge table overflow: retry on the long path
  // ---- final symbols -> (end, id) tokens in order; PieceToId (model_interface.cc:51-61) ----
  uint32_t *tend = bm.pval;   // safe to reuse: the merge loop is over
  int32_t *tid = reinterpret_cast<int32_t *>(bm.pnode);
  uint32_t n_tok = 0;
  for (uint32_t w = 0; w < n; w += 32) {
    const uint32_t k = w + T.lane;
    const bool st = k < n && bm.slen[k] != 0;
    uint32_t end = 0;
    int32_t id = M.unk_id;
    if (st) {
      end = k + bm.slen[k];
      const uint32_t v = bm.snode[k];
      if (v != kDead) {
        const int32_t t = __ldg(M.trie_id + v);
        if (t >= 0) id = t;
      }
    }
    const uint32_t m = T.ballot(st);
    T.sync();  // every lane has read pval/pnode-aliased data of this window before it is overwritten
    if (st) {
      const uint32_t r = n_tok + __popc(m & T.below());
      tend[r] = end;
      tid[r] = id;
    }
    n_tok += __popc(m);
  }
  T.sync();
  // ---- resegmentation of UNUSED pieces (bpe_model.cc:175-200): sequential and rare ----
  if (has_unused) {
    bool any = false;
    for (uint32_t k = T.lane; k < n_tok; k += 32) {
      const int32_t id = tid[k];
      any |= id >= 0 && __ldg(M.types + id) == 5 /* UNUSED */;
    }
    if (T.ballot(any)) {
      // Depth-first, left to right.  Pieces are contiguous, so the stack only holds byte
      // lengths (depth <= piece length <= ncap); output goes to snode (ends) / aux (ids),
      // both free once the merge loop is over.
      uint32_t total = 0;
      if (T.lane == 0) {
        uint32_t *stk = bm.sprev;
        uint32_t off = 0;
        for (uint32_t k = 0; k < n_tok; ++k) {
          uint32_t sp = 0;
          stk[sp++] = tend[k] - off;
          while (sp) {
            const uint32_t l = stk[--sp];
            uint32_t lk = 0;
            const uint32_t v = trie_walk(H, 0, text + off, l, &lk);
            int32_t id = M.unk_id;  // PieceToId: pieces_ else unk
            if (v != kDead) { const int32_t t = __ldg(M.trie_id + v); if (t >= 0) id = t; }
            uint32_t ll = 0;
            if (v != kDead && id >= 0 && __ldg(M.types + id) == 5)
              for (uint32_t i = 0; i < n_rev; ++i)
                if (bm.rm_node[i] == v) { ll = bm.rm_llen[i]; break; }
            if (ll && ll < l) {
              stk[sp++] = l - ll;  // right part is resegmented second
              stk[sp++] = ll;
            } else {
              off += l;
              bm.snode[total] = off;
              bm.aux[total] = static_cast<uint32_t>(id);
              ++total;
            }
          }
        }
      }
      n_tok = T.shfl(total, 0);
      tend = bm.snode;
      tid = reinterpret_cast<int32_t *>(bm.aux);
      T.sync();
    }
  }
  finish_tokens<SPANS>(M, B, T, text, tend, tid, sent, n_tok);
  return true;
}


template <bool SPANS>
__global__ void __launch_bounds__(512, 1) encode_bpe_kernel(const KModel M, const KBatch B) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t *mbar = reinterpret_cast<uint64_t *>(smem);
  uint32_t *s_link = reinterpret_cast<uint32_t *>(smem + 16);
  uint32_t *s_val = s_link + M.hot_link;
  uint8_t *tiles = reinterpret_cast<uint8_t *>(s_val + M.hot_val);
  stage_hot_trie(M, mbar, s_link, s_val);
  HotTrie H{s_link, s_val, M.trie_link, M.trie_val, M.hot_link, M.hot_val};
  const Tile T;
  const BpeMem bm = carve_bpe(tiles + static_cast<size_t>(threadIdx.x >> 5) * B.tile_bytes, B.ncap, SPANS);
  for (;;) {
    uint32_t sent = 0;
    if (T.lane == 0) sent = atomicAdd(B.work_counter, 1u);
    sent = __shfl_sync(0xFFFFFFFFu, sent, 0);
    if (sent >= (B.sub_list ? B.sub_n : B.n)) break;
    if (B.sub_list) sent = B.sub_list[2 * sent];
    const unsigned long long off = B.offsets[sent];
    const unsigned long long len64 = B.offsets[sent + 1] - off;
    bool fits = len64 + 32ull <= bm.stage_cap;
    uint32_t need = 0;
    if (fits) {
      const uint32_t len = static_cast<uint32_t>(len64);
      const uint8_t *g = B.bytes + off;
      const uint32_t mis = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(g) & 15u);
      const uint4 *ga = reinterpret_cast<const uint4 *>(g - mis);
      const uint32_t nvec = (mis + len + 15u) >> 4;
      uint4 *sa = reinterpret_cast<uint4 *>(bm.stage);
      for (uint32_t v = T.lane; v < nvec; v += 32) sa[v] = __ldg(ga + v);
      T.sync();
      fits = encode_bpe_sentence<SPANS>(M, B, T, H, bm, bm.stage + mis, len, sent, &need);
    }
    if (!fits && T.lane == 0) {
      const uint32_t slot = atomicAdd(B.status, 1u);
      B.deferred[2 * slot] = sent;
      B.deferred[2 * slot + 1] = need;
    }
    __syncwarp();
  }
}

template <bool SPANS>
__global__ void __launch_bounds__(256) encode_bpe_long_kernel(const KModel M, const KBatch B) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t *mbar = reinterpret_cast<uint64_t *>(smem);
  uint32_t *s_link = reinterpret_cast<uint32_t *>(smem + 16);
  uint32_t *s_val = s_link + M.hot_link;
  stage_hot_trie(M, mbar, s_link, s_val);
  HotTrie H{s_link, s_val, M.trie_link, M.trie_val, M.hot_link, M.hot_val};
  const Tile T;
  const uint32_t warps_per_cta = blockDim.x >> 5;
  for (uint32_t w = blockIdx.x * warps_per_cta + (threadIdx.x >> 5); w < B.long_n; w += gridDim.x * warps_per_cta) {
    const uint32_t sent = B.long_list[2 * w];
    const uint32_t ncap = B.long_list[2 * w + 1];
    const BpeMem bm = carve_bpe(B.long_scratch + B.long_scratch_off[w], ncap, SPANS);
    const unsigned long long off = B.offsets[sent];
    const uint32_t len = static_cast<uint32_t>(B.offsets[sent + 1] - off);
    uint32_t need = 0;
    const bool ok = encode_bpe_sentence<SPANS>(M, B, T, H, bm, B.bytes + off, len, sent, &need);
    if (!ok && T.lane == 0) atomicOr(B.status + 1, 8u);  // the slab was too small: its own bit and message
    __syncwarp();
  }
}

}  // namespace spm_b200
#endif
