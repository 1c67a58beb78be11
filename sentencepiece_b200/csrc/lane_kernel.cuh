// lane_kernel.cuh -- unigram fast path: one sentence per LANE (32 sentences per warp).
//
// Motivation: with one sentence per warp the kernel is instruction-issue bound and most
// of the issued instructions are the ORDERED fold of Viterbi edges, where 31 of 32 lanes
// repeat the same scalar work.  The reference algorithm (src/unigram_model.cc:889-1020)
// is a short sequential state machine per sentence; running it one sentence per lane
// makes every instruction do 32 sentences' worth of work.
//
// Per lane, per sentence:
//   K1  Normalizer::Normalize / NormalizePrefix, sequentially (src/normalizer.cc:71-253).
//       Input bytes stream through a 32-byte register window (aligned 16-byte loads, next
//       chunk prefetched); the ASCII fast-path tables of the charsmap sit in shared
//       memory; normalized text goes to a per-lane slab in HBM/L2 with words interleaved
//       by lane.
//   K2  EncodeOptimized as a flat state machine: each loop trip is ONE trie transition
//       for every lane (hot trie prefix in shared memory, rest L2).  The text is read
//       through a 16-byte register window anchored at the current start (next word
//       prefetched at each start transition).  best_path_ends_at[] only ever needs the
//       positions [s, s + max_piece_len], so it lives in a per-lane RING in shared memory
//       laid out [slot][lane] (bank == lane: conflict free).  When a position becomes a
//       start its final back-pointer is appended to a per-lane LOG (entry t of every lane
//       shares a cache line), so the back-trace is a coalesced backward scan.
//   K4  back-trace + id path of PopulateSentencePieceText: two backward scans of the log
//       (count, then write) around one warp-aggregated claim of output space.
// Exactly the reference's relaxation order and mixed float/double comparison.
#ifndef SPM_B200_LANE_KERNEL_CUH_
#define SPM_B200_LANE_KERNEL_CUH_

#include "kernels.cuh"
#include "drain.cuh"

namespace spm_b200 {

constexpr uint32_t kLaneUnk = 0x3FFFFFu;  // 22-bit trie-unit field: UNK piece
// encode_unigram_lane_kernel spells U+2581 as this one byte, in its normalized text and in its trie (KModel::trie_node4):
// a walk from a word start takes one transition on it instead of three, and the text is two bytes shorter per word.
// 0xFF never occurs in the normalized text otherwise (it is valid UTF-8: malformed bytes become U+FFFD, pieces and
// charsmap targets are checked at load), and both sides of every comparison change alike, so the lattice -- characters,
// candidate pieces, scores, relaxation order -- is the same.
constexpr uint32_t kWsByte = 0xFFu;

// slab geometry: per warp [text words: cap/4 + 12][32] u32, then [log: cap + 4][32] u32
constexpr uint32_t kLaneTextSlack = 12;  // window loads may run a few words past the text
__host__ __device__ inline unsigned long long lane_slab_bytes(uint32_t cap) {
  return (static_cast<unsigned long long>(cap / 4 + kLaneTextSlack) + (cap + 4)) * 32ull * 4ull;
}
// shared memory for the normalizer's fast-path tables
constexpr uint32_t kLaneTableBytes = 32 + 4096 + 512 + 16 + 16;  // cm_lead[8] + cm_pair[1024] + cm_solo[128] + plain[4] + plain_or_space[4]

// Fills the normalizer's fast-path tables in shared memory (all threads of the CTA; caller synchronizes).
__device__ __forceinline__ void fill_lane_tables(const KModel &M, uint32_t *s_tab) {
  const bool has_cm = M.flags & kFlagHasCharsmap;
  for (uint32_t i = threadIdx.x; i < 8 + 1024 + 128 + 4; i += blockDim.x) {
    uint32_t v;
    if (i < 8) v = M.cm_lead[i];
    else if (i < 8 + 1024) v = M.cm_pair[i - 8];
    else if (i < 8 + 1024 + 128) v = static_cast<uint32_t>(M.cm_solo[i - 8 - 1024]);
    else {  // plain ASCII bytes: no charsmap rule starts with them and they are not the space
      const uint32_t wq = i - (8 + 1024 + 128);
      v = ~(has_cm ? M.cm_lead[wq] : 0u);
      if (wq == 1) v &= ~1u;  // ' ' = 0x20
    }
    s_tab[i] = v;
  }
  // "simple" ASCII bytes (space included): followed by another ASCII byte they are always their own chunk -- no
  // rule is the byte alone or the byte + an ASCII byte.  (nmt_nfkc has letter + combining-mark compositions, so
  // most letters DO start rules; those need a non-ASCII second byte, which the caller excludes.)
  for (uint32_t wq = threadIdx.x >> 5; wq < 4; wq += blockDim.x >> 5) {
    const uint32_t ch = wq * 32 + (threadIdx.x & 31);
    bool simple = true;
    if (has_cm && ((M.cm_lead[wq] >> (ch & 31u)) & 1u)) {
      simple = M.cm_solo[ch] < 0;
      for (uint32_t q = 0; q < 4; ++q) simple = simple && M.cm_pair[((ch * 256u) >> 5) + q] == 0u;
    }
    // The 4-byte step emits at most 8 bytes.  An escaped space is 3 bytes, so four bytes hold at most two of them: true
    // only when remove_extra_whitespaces drops the second of two adjacent spaces.  Otherwise the space is not simple.
    if (ch == ' ' && (M.flags & kFlagEscapeWs) && !(M.flags & kFlagRemoveExtraWs)) simple = false;
    const uint32_t word = __ballot_sync(0xFFFFFFFFu, simple);
    if ((threadIdx.x & 31) == 0) s_tab[8 + 1024 + 128 + 4 + wq] = word;
  }
}

// Streamed host batches (engine.cu, encode_host_streamed): the batch arrives in pieces of 2^piece_shift
// sentences and *B.ready counts the sentences whose bytes are in HBM.  Lane 0 of a warp waits for the piece
// that holds its group; the wait is bounded so that a stalled copy can never hang the GPU.
__device__ __forceinline__ void lane_wait_input(const KBatch &B, uint32_t first, uint32_t lane) {
  if (!B.ready) return;
  if (lane == 0) {
    uint32_t need = ((first >> B.piece_shift) + 1u) << B.piece_shift;
    if (need > B.n) need = B.n;
    need += B.ready_base;
    const volatile uint32_t *r = B.ready;
    if (B.kstats) atomicAdd(B.kstats + 3, 1ull);
    if (*r < need) {
      const long long t0 = clock64();
      while (*r < need) {
        __nanosleep(200);
        if (clock64() - t0 > 6000000000ll || (*reinterpret_cast<const volatile uint32_t *>(B.status + 1) & 2u)) {
          atomicOr(B.status + 1, 2u);  // ~3 s without progress: give up (the host reports the error)
          break;
        }
      }
      if (B.kstats) atomicAdd(B.kstats, static_cast<unsigned long long>(clock64() - t0));
    }
    // No fence here: __threadfence() is MEMBAR.SC + CCTL.IVALL on sm_90a, and wiping the SM's L1 twice per group makes
    // the whole kernel markedly slower on the mixed-script corpus.  The input loads below are issued
    // after this load has returned (the loop's exit depends on it), and they cannot hit a stale L1 line: a line of
    // the input is first touched by a sentence of the piece it arrived with (copies are cut at 128-byte lines).
  }
  __syncwarp();
}

struct LaneCtx {
  uint32_t *text_w;  // + word*32 (already offset by lane)
  uint32_t *log;     // + t*32    (already offset by lane)
  const uint32_t *s_lead, *s_pair;
  const int32_t *s_solo;
  const uint32_t *s_plain;  // bit b: ASCII byte b is copied verbatim (no rule starts with it, not a space)
  const uint32_t *s_plainsp;  // bit b: ASCII byte b followed by an ASCII byte is always its own chunk (space included)
  unsigned long long pol;     // L2 cache policy of the slab accesses (slab_policy())
};

// The per-lane slabs (normalized text, back-pointer log) are written and read back within one group: ~12 KB per
// resident warp, tens of MB per GPU, within H100's 50 MB L2 -- but only stays there if the batch's streamed input and ids do not
// push it out.  Every slab access carries an L2 cache policy (evict_normal); the once-read input and the once-written
// ids use the streaming forms (__ldcs / __stcs), and the dead rows are discarded at the end of a group (slab_discard).
// The hinted accesses read the policy from a uniform register.  The redux makes the value warp-uniform for the
// compiler, so it stays in uniform registers instead of being copied into one (R2UR) at every access.
__device__ __forceinline__ unsigned long long slab_policy() {
  unsigned long long pol;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
  const uint32_t lo = __reduce_or_sync(0xFFFFFFFFu, static_cast<uint32_t>(pol));
  const uint32_t hi = __reduce_or_sync(0xFFFFFFFFu, static_cast<uint32_t>(pol >> 32));
  return (static_cast<unsigned long long>(hi) << 32) | lo;
}
__device__ __forceinline__ uint32_t slab_ld(const uint32_t *p, unsigned long long pol) {
  uint32_t v;
  asm volatile("ld.global.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol) : "memory");
  return v;
}
__device__ __forceinline__ void slab_st(uint32_t *p, uint32_t v, unsigned long long pol) {
  asm volatile("st.global.L2::cache_hint.u32 [%0], %1, %2;" :: "l"(p), "r"(v), "l"(pol) : "memory");
}
// End of a group: the rows of the warp's slab that the group used are dead.  Without a hint L2 keeps them as dirty
// lines: they are written back to HBM when they are finally evicted (traffic for nothing) and, until then, they take
// the place of the rows that are still live in other warps.  discard.L2 drops a line without write-back.  Warp-
// collective; row r of a slab is one 128-byte line (32 lanes x 4 bytes).  The barriers order the group's last reads
// before the discards and the discards before the next group's first writes (other lanes' words of the same line).
__device__ __forceinline__ void slab_discard(const LaneCtx &c, uint32_t lane, uint32_t text_rows, uint32_t log_rows) {
  __syncwarp();
  const uint8_t *tb = reinterpret_cast<const uint8_t *>(c.text_w - lane);
  for (uint32_t r = lane; r < text_rows; r += 32)
    asm volatile("discard.global.L2 [%0], 128;" :: "l"(tb + static_cast<size_t>(r) * 128) : "memory");
  const uint8_t *lb = reinterpret_cast<const uint8_t *>(c.log - lane);
  for (uint32_t r = lane; r < log_rows; r += 32)
    asm volatile("discard.global.L2 [%0], 128;" :: "l"(lb + static_cast<size_t>(r) * 128) : "memory");
  __syncwarp();
}

// The lane's view of its warp's slab and of the normalizer's tables (s_tab, filled by fill_lane_tables).
__device__ __forceinline__ LaneCtx lane_ctx(const uint32_t *s_tab, uint8_t *slabs, uint32_t cap, uint32_t warp_global,
                                            uint32_t lane) {
  LaneCtx c;
  c.pol = slab_policy();
  uint8_t *slab = slabs + static_cast<size_t>(warp_global) * lane_slab_bytes(cap);
  c.text_w = reinterpret_cast<uint32_t *>(slab) + lane;
  c.log = reinterpret_cast<uint32_t *>(slab) + static_cast<size_t>(cap / 4 + kLaneTextSlack) * 32 + lane;
  c.s_lead = s_tab;
  c.s_pair = s_tab + 8;
  c.s_solo = reinterpret_cast<const int32_t *>(s_tab + 8 + 1024);
  c.s_plain = s_tab + 8 + 1024 + 128;
  c.s_plainsp = c.s_plain + 4;
  return c;
}

// Claims the warp's next group of 32 sentences, [*first, *first + 32) of the processing order; false once the batch
// is done.
__device__ __forceinline__ bool lane_claim_group(const KBatch &B, uint32_t lane, uint32_t *first) {
  uint32_t f = 0;
  if (lane == 0) f = atomicAdd(B.work_counter, 32u);
  *first = __shfl_sync(0xFFFFFFFFu, f, 0);
  return *first < B.n;
}

// Byte k of the lane's normalized text: L2-hinted slab load (the encode kernels) or plain load (n-best, lattice, and
// the BPE kernel's byte fallback).
__device__ __forceinline__ uint32_t lane_text_byte(const LaneCtx &c, uint32_t k) {
  return (slab_ld(c.text_w + static_cast<size_t>(k >> 2) * 32, c.pol) >> ((k & 3u) * 8u)) & 0xFFu;
}
__device__ __forceinline__ uint32_t lane_text_byte_plain(const LaneCtx &c, uint32_t k) {
  return (c.text_w[static_cast<size_t>(k >> 2) * 32] >> ((k & 3u) * 8u)) & 0xFFu;
}

// A sentence the lane kernel leaves to a later pass (the general warp-per-sentence kernels).
__device__ __forceinline__ void lane_defer(const KBatch &B, uint32_t sent) {
  const uint32_t slot = atomicAdd(B.status, 1u);
  B.deferred[2 * slot] = sent;
  B.deferred[2 * slot + 1] = 0;
  B.sent_count[sent] = 0;  // until a later pass encodes it
}

// Phase clocks of the encode lane kernels when B.kstats is set, summed by lane 0 of each warp: kstats[4] the whole
// group, [5] K1, [6] K2 (BPE: phases A and B), [7] K4.  Construct at the top of a group, mark() after K1, K2 and K4,
// flush() at the end of the group.
struct LanePhaseClock {
  unsigned long long *ks;
  uint32_t t[4];
  uint32_t i;
  __device__ __forceinline__ explicit LanePhaseClock(const KBatch &B) : ks(B.kstats), i(0) { mark(); }
  __device__ __forceinline__ void mark() { t[i++] = ks ? static_cast<uint32_t>(clock64()) : 0u; }
  __device__ __forceinline__ void flush(uint32_t lane) const {
    if (ks && lane == 0) {
      typedef unsigned long long ull;
      atomicAdd(ks + 4, ull(static_cast<uint32_t>(clock64()) - t[0])); atomicAdd(ks + 5, ull(t[1] - t[0]));
      atomicAdd(ks + 6, ull(t[2] - t[1])); atomicAdd(ks + 7, ull(t[3] - t[2]));
    }
  }
};

// Sequential byte stream over a lane's input: 16-byte aligned chunks (next chunk prefetched)
// feed a 64-bit shift register that always exposes the next >= 4 bytes.  The aligned chunks
// over-read into the neighbouring sentences by up to 15 bytes; a streamed host batch (engine.cu)
// therefore cuts its copies at 128-byte lines, so that every line a sentence touches has landed
// completely before the sentence's piece is announced.
struct ByteStream {
  const uint4 *cp;      // chunk that `nxt` was loaded from, + 1
  const uint4 *cend;    // first chunk past the sentence
  uint4 cur, nxt;
  uint32_t wi;          // next word of `cur` to feed (0..3)
  unsigned long long win;
  uint32_t have;        // valid bytes in win
  __device__ __forceinline__ uint32_t next_word() {
    const uint32_t w = wi == 0 ? cur.x : (wi == 1 ? cur.y : (wi == 2 ? cur.z : cur.w));
    if (++wi == 4) {
      wi = 0;
      cur = nxt;
      nxt = cp < cend ? __ldcs(cp) : make_uint4(0, 0, 0, 0);
      ++cp;
    }
    return w;
  }
  __device__ __forceinline__ void init(const uint8_t *p, const uint8_t *hi) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint4 *c0 = reinterpret_cast<const uint4 *>(a & ~static_cast<uintptr_t>(15));
    cend = reinterpret_cast<const uint4 *>((reinterpret_cast<uintptr_t>(hi) + 15) & ~static_cast<uintptr_t>(15));
    cur = __ldcs(c0);  // streaming (evict-first) loads: the input is read once and must not push the slabs out of L2
    nxt = c0 + 1 < cend ? __ldcs(c0 + 1) : make_uint4(0, 0, 0, 0);
    cp = c0 + 2;
    wi = static_cast<uint32_t>((a & 15) >> 2);
    const uint32_t mis = static_cast<uint32_t>(a & 3);
    const uint32_t w = next_word();
    win = static_cast<unsigned long long>(w >> (8 * mis));
    have = 4 - mis;
    win |= static_cast<unsigned long long>(next_word()) << (8 * have);
    have += 4;
  }
  __device__ __forceinline__ uint32_t peek(uint32_t i) const { return static_cast<uint32_t>(win >> (8 * i)) & 0xFFu; }
  __device__ __forceinline__ void consume(uint32_t c) {  // c <= 4
    win >>= 8 * c;
    have -= c;
    if (have <= 4) {
      win |= static_cast<unsigned long long>(next_word()) << (8 * have);
      have += 4;
    }
  }
};

// Sequential normalizer for one lane.  Returns the normalized length, or 0xFFFFFFFF if
// it exceeds `cap` (the caller defers the sentence).
// kWs1: every U+2581 -- escaped spaces, literal ones from the input or a charsmap target -- is written as kWsByte and
// the returned length counts it as one byte.  The cap still applies to the length with U+2581 as three bytes (out +
// saved), tested where the three-byte spelling tests it -- before the trailing strip, and again before the suffix --
// so the same sentences are deferred in either spelling.  (Before the strip out and saved only grow, so the test on
// their final sum sees the largest length, as the three-byte spelling's overflow flag does.)
template <bool kWs1 = false>
__device__ __forceinline__ uint32_t lane_normalize(const KModel &M, const uint8_t *in, uint32_t len, const LaneCtx &c,
                                                   uint32_t cap) {
  const bool rm = M.flags & kFlagRemoveExtraWs;
  const bool esc = M.flags & kFlagEscapeWs;
  const bool suffix = M.flags & kFlagWsSuffix;
  const bool addp = M.flags & kFlagAddDummyPrefix;
  const bool has_user = M.flags & kFlagHasUserSymbols;
  const bool has_cm = M.flags & kFlagHasCharsmap;
  if (len == 0) return 0;
  ByteStream S;
  S.init(in, in + len);
  uint32_t out = 0;  // normalized bytes produced
  uint32_t acc = 0;  // partial word
  uint32_t saved = 0;  // kWs1: 2 per U+2581 written (out + saved = the length with U+2581 as three bytes)
  bool overflow = false;
  auto put = [&](uint32_t ch) {
    acc |= ch << ((out & 3u) * 8u);
    if ((out & 3u) == 3u) {
      if (out < cap) slab_st(c.text_w + static_cast<size_t>(out >> 2) * 32, acc, c.pol); else overflow = true;
      acc = 0;
    }
    ++out;
  };
  auto put_u2581 = [&]() {
    if (kWs1) { put(kWsByte); saved += 2; } else { put(0xE2); put(0x96); put(0x81); }
  };
  auto put_ws = [&]() {
    if (esc) put_u2581(); else put(' ');
  };
  uint32_t pos = 0;
  bool is_prev_space = rm;  // normalizer.cc:130
  bool started = !rm;       // the heading-space loop (:86-95) is over
  if (started && addp && !suffix) put_ws();  // dummy prefix (:128); with the heading loop it is emitted when that ends
  // One chunk of NormalizePrefix (normalizer.cc:195-253) + the emit logic of Normalize (:131-163)
  while (pos < len) {
    const uint32_t rem = len - pos;
    // ---- fast path: four ASCII bytes at once, each "simple" (its own chunk when an ASCII byte follows) and with
    //      an ASCII byte (or the end of the sentence) after the window.  Branch-free restatement of :131-163 for
    //      such chunks: a space after a space is dropped (remove_extra_whitespaces), otherwise it becomes U+2581 or
    //      stays ' '; the <= 8 output bytes are appended with at most two word stores. ----
    if (started && !has_user && rem >= 4) {
      const uint32_t w4 = static_cast<uint32_t>(S.win);
      const uint32_t c0 = w4 & 0xFFu, c1 = (w4 >> 8) & 0xFFu, c2 = (w4 >> 16) & 0xFFu, c3 = w4 >> 24;
      if (!(w4 & 0x80808080u) && ((c.s_plainsp[c0 >> 5] >> (c0 & 31u)) & (c.s_plainsp[c1 >> 5] >> (c1 & 31u)) &
                                  (c.s_plainsp[c2 >> 5] >> (c2 & 31u)) & (c.s_plainsp[c3 >> 5] >> (c3 & 31u)) & 1u) &&
          (rem == 4 || S.peek(4) < 0x80u)) {
        unsigned long long chunk = 0;
        uint32_t clen = 0;
        bool prev = is_prev_space;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const uint32_t ch = (w4 >> (8 * i)) & 0xFFu;
          const bool sp = ch == ' ';
          const bool emit = !(sp && prev);
          const uint32_t bytes = (sp && esc) ? (kWs1 ? kWsByte : 0x8196E2u) : ch;  // U+2581 = E2 96 81
          const uint32_t blen = emit ? ((sp && esc && !kWs1) ? 3u : 1u) : 0u;
          chunk |= static_cast<unsigned long long>(emit ? bytes : 0u) << (8u * clen);
          clen += blen;
          if (kWs1) saved += (emit && sp && esc) ? 2u : 0u;
          prev = sp && rm;
        }
        is_prev_space = prev;
        const uint32_t r8 = (out & 3u) * 8u;
        const unsigned long long lo = static_cast<unsigned long long>(acc) | (chunk << r8);
        const uint32_t hi = r8 ? static_cast<uint32_t>(chunk >> (64u - r8)) : 0u;
        const uint32_t nw = ((out & 3u) + clen) >> 2;  // full words completed: 0..2
        if (out <= cap) {
          uint32_t *wp = c.text_w + static_cast<size_t>(out >> 2) * 32;
          if (nw >= 1) slab_st(wp + 0, static_cast<uint32_t>(lo), c.pol);
          if (nw >= 2) slab_st(wp + 32, static_cast<uint32_t>(lo >> 32), c.pol);
        }
        acc = nw == 0 ? static_cast<uint32_t>(lo) : (nw == 1 ? static_cast<uint32_t>(lo >> 32) : hi);
        out += clen;
        if (out > cap) overflow = true;
        pos += 4;
        S.consume(4);
        continue;
      }
    }
    const uint32_t b = S.peek(0);
    uint32_t consumed = 1;
    // replacement string: kind + (pointer | inline bytes)
    uint32_t kind = kChunkChar, spl = 1;
    const uint8_t *sp = nullptr;
    bool generic = false;
    if (has_user) {
      const uint32_t ul = user_longest(M, in + pos, rem);
      if (ul) { consumed = ul; spl = ul; kind = kChunkVerbatim; sp = in + pos; generic = true; }
    }
    if (!generic) {
      uint32_t longest = 0, value = 0;
      if (has_cm && ((c.s_lead[b >> 5] >> (b & 31u)) & 1u)) {
        if (b < 0x80u) {
          bool cont = false;
          if (rem > 1) {
            const uint32_t c2 = S.peek(1);
            cont = (c.s_pair[(b * 256u + c2) >> 5] >> (c2 & 31u)) & 1u;
          }
          if (cont) longest = charsmap_longest_win(M, S.win, S.have, in + pos, rem, &value);
          else {
            const int32_t so = c.s_solo[b];
            if (so >= 0) { longest = 1; value = static_cast<uint32_t>(so); }
          }
        } else {
          longest = charsmap_longest_win(M, S.win, S.have, in + pos, rem, &value);
        }
      }
      if (longest) {
        consumed = longest; kind = kChunkTarget; sp = M.cm_targets + value; generic = true;
        spl = 0;
        while (__ldg(sp + spl) != 0) ++spl;
      } else if (b < 0x80u) {
        // ---- fast path: one ASCII byte that is not a rule ----
        if (!started) {
          if (b == ' ') { ++pos; S.consume(1); continue; }  // heading space
          started = true;
          if (addp && !suffix) put_ws();
        }
        if (b == ' ') {
          if (!is_prev_space) { put_ws(); is_prev_space = rm; }
        } else {
          put(b);
          is_prev_space = false;
        }
        ++pos;
        S.consume(1);
        continue;
      } else {
        // DecodeUTF8 / IsValidDecodeUTF8 (util.cc:51-84) on the stream's look-ahead bytes
        uint32_t l = 0;
        const uint32_t b1 = S.peek(1), b2 = S.peek(2), b3 = S.peek(3);
        if (rem >= 2 && (b & 0xE0u) == 0xC0u) {
          if (is_trail(b1) && (((b & 0x1Fu) << 6) | (b1 & 0x3Fu)) >= 0x80u) l = 2;
        } else if (rem >= 3 && (b & 0xF0u) == 0xE0u) {
          const uint32_t cp = ((b & 0x0Fu) << 12) | ((b1 & 0x3Fu) << 6) | (b2 & 0x3Fu);
          if (is_trail(b1) && is_trail(b2) && cp >= 0x800u && (cp < 0xD800u || cp >= 0xE000u)) l = 3;
        } else if (rem >= 4 && (b & 0xF8u) == 0xF0u) {
          const uint32_t cp = ((b & 0x07u) << 18) | ((b1 & 0x3Fu) << 12) | ((b2 & 0x3Fu) << 6) | (b3 & 0x3Fu);
          if (is_trail(b1) && is_trail(b2) && is_trail(b3) && cp >= 0x10000u && cp <= 0x10FFFFu) l = 4;
        }
        if (!started) { started = true; if (addp && !suffix) put_ws(); }
        if (l) {  // a valid multi-byte character: never a space
          if (kWs1 && l == 3 && b == 0xE2u && b1 == 0x96u && b2 == 0x81u) {
            put_u2581();  // a literal U+2581 (still not a space for remove_extra_whitespaces)
          } else {
            put(b); put(b1);
            if (l > 2) put(b2);
            if (l > 3) put(b3);
          }
          consumed = l;
        } else {  // malformed: one byte -> U+FFFD (normalizer.cc:231-244)
          put(0xEF); put(0xBF); put(0xBD);
          consumed = 1;
        }
        is_prev_space = false;
        pos += consumed;
        S.consume(consumed);
        continue;
      }
    }
    // ---- generic path: rule targets and verbatim user symbols ----
    auto sp_byte = [&](uint32_t i) -> uint32_t { return __ldg(sp + i); };
    if (!started) {
      if (spl == 1 && sp_byte(0) == ' ') {  // a chunk that is exactly " " during the heading loop
        pos += consumed;
        if (consumed <= 4) S.consume(consumed); else S.init(in + pos, in + len);
        continue;
      }
      started = true;
      if (addp && !suffix) put_ws();
    }
    {
      uint32_t i0 = 0;
      while (is_prev_space && i0 < spl && sp_byte(i0) == ' ') ++i0;  // :137-138
      if (i0 < spl) {
        uint32_t last = 0;
        for (uint32_t i = i0; i < spl; ++i) {
          last = sp_byte(i);
          if (last == ' ' && esc) {
            put_u2581();
          } else if (kWs1 && last == 0xE2u && i + 2 < spl && sp_byte(i + 1) == 0x96u && sp_byte(i + 2) == 0x81u) {
            put_u2581();  // a literal U+2581 in a rule target or user symbol
            i += 2;
            last = 0x81u;
          } else {
            put(last);
          }
        }
        is_prev_space = last == ' ';
      }
      if (!rm) is_prev_space = false;
    }
    pos += consumed;
    if (consumed <= 4) S.consume(consumed); else S.init(in + pos, in + len);
  }
  if (!started) return 0;  // all chars are whitespace (:97-100)
  if (overflow || out + saved > cap) return 0xFFFFFFFFu;
  // flush the partial word, then strip trailing spaces on the escaped output (:166-176)
  slab_st(c.text_w + static_cast<size_t>(out >> 2) * 32, acc, c.pol);
  if (rm) {
    if (esc && kWs1) {
      while (out >= 1 && lane_text_byte(c, out - 1) == kWsByte) { out -= 1; saved -= 2; }
    } else if (esc) {
      while (out >= 3 && lane_text_byte(c, out - 3) == 0xE2 && lane_text_byte(c, out - 2) == 0x96 &&
             lane_text_byte(c, out - 1) == 0x81)
        out -= 3;
    } else {
      while (out >= 1 && lane_text_byte(c, out - 1) == ' ') out -= 1;
    }
  }
  if (suffix && addp) {  // :179
    if (out + saved + 3 > cap) return 0xFFFFFFFFu;
    acc = (out & 3u) ? (slab_ld(c.text_w + static_cast<size_t>(out >> 2) * 32, c.pol) & ((1u << ((out & 3u) * 8u)) - 1u)) : 0u;
    put_ws();
    slab_st(c.text_w + static_cast<size_t>(out >> 2) * 32, acc, c.pol);
  }
  return out;
}

// K1 of a lane kernel: normalizes sentence `sent` into the lane's slab, *n = the normalized length.  Returns false
// (*n = 0) when the kernel does not take the sentence: more than 4 * cap input bytes or cap normalized bytes, input
// outside the batch's valid range [B.off_lo, B.off_hi], or beyond `lim` (input lengths above it, normalized lengths
// from it up; for a kernel whose positions have fewer than 32 bits).
template <bool kWs1 = false>
__device__ __forceinline__ bool lane_k1(const KModel &M, const KBatch &B, const LaneCtx &c, uint32_t sent, uint32_t cap,
                                        uint32_t *n, unsigned long long lim = ~0ull) {
  const unsigned long long off = B.offsets[sent];
  const unsigned long long len64 = B.offsets[sent + 1] - off;
  *n = 0;
  if (len64 > 4ull * cap || len64 > lim || off < B.off_lo || off + len64 > B.off_hi) return false;
  *n = lane_normalize<kWs1>(M, B.bytes + off, static_cast<uint32_t>(len64), c, cap);
  if (*n == 0xFFFFFFFFu || *n >= lim) { *n = 0; return false; }
  return true;
}

// One claim of output space per warp (a scan of the lanes' id counts, one atomicAdd on B.cursor).  Returns the lane's
// first slot in B.tmp_ids and records the sentence's start and count.  *room is false on every lane when the warp's
// ids do not fit in B.tmp_cap: status[2] then tells the host to rerun the batch with a larger buffer.
__device__ __forceinline__ unsigned long long lane_claim_output(const KBatch &B, uint32_t lane, uint32_t count, bool have,
                                                                bool defer, uint32_t sent, bool *room) {
  uint32_t incl = count;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d);
    if (lane >= static_cast<uint32_t>(d)) incl += t;
  }
  const uint32_t total = __shfl_sync(0xFFFFFFFFu, incl, 31);
  unsigned long long pos = 0;
  if (lane == 0 && total) {
    pos = atomicAdd(B.cursor, static_cast<unsigned long long>(total));
    if (pos + total > B.tmp_cap) atomicOr(B.status + 2, 1u);
  }
  pos = __shfl_sync(0xFFFFFFFFu, pos, 0);
  *room = pos + total <= B.tmp_cap;
  pos += incl - count;
  if (have && !defer) {
    B.sent_start[sent] = pos;
    B.sent_count[sent] = *room ? count : 0u;
  }
  return pos;
}

// Model::PopulateNodes (unigram_model.cc:547-596) from begin character bp, whose byte offset is surf[bp] (surf[L] = n):
// walks the trie (trie_node2, root link word `root`) along the text and calls piece(length, v, score) for every
// NORMAL or USER_DEFINED piece that begins there, shortest first -- length in characters (get_chars_length, :548-552),
// trie unit, score (USER_DEFINED: float(double(length * max_score) - 0.1)).  piece returns false when the lattice is
// full, which ends the walk.  Returns whether a one-character piece was found (if not, the caller adds the UNK node).
// populate_from reads byte k of the normalized text as text_byte(k) and character offsets from surf (16-bit in the
// lane kernels' slabs, 32-bit on the long-sentence path).
template <typename TextByte, typename SurfT, typename F>
__device__ __forceinline__ bool populate_from(const KModel &M, TextByte &&text_byte, uint32_t root, const SurfT *surf,
                                              uint32_t bp, uint32_t n, F &&piece) {
  bool has_single = false;
  uint32_t l = root;
  uint32_t clen = 0;  // characters completed so far
  for (uint32_t kpos = surf[bp]; kpos < n; ++kpos) {
    const uint32_t ch = text_byte(kpos);
    const uint32_t v = (l >> kLinkBaseShift) ^ ch;
    l = __ldg(&M.trie_node2[v]).x;
    if ((l & kLinkLabelMask) != ch) break;
    if (kpos + 1 == surf[bp + clen + 1]) ++clen;
    const uint32_t kind = (l >> kLinkKindShift) & 3u;
    if (kind == kKindNone || kind == kKindUnused) continue;
    const uint32_t length = (kpos + 1 == surf[bp + clen]) ? clen : clen + 1;
    const float sc = kind == kKindUserDefined
                         ? static_cast<float>(static_cast<double>(__fmul_rn(static_cast<float>(length), M.max_score)) - 0.1)
                         : __uint_as_float(__ldg(M.trie_val + v));
    if (!piece(length, v, sc)) break;
    has_single |= length == 1;
  }
  return has_single;
}
template <typename F>
__device__ __forceinline__ bool lane_populate_from(const KModel &M, const LaneCtx &c, uint32_t root, const uint16_t *surf,
                                                   uint32_t bp, uint32_t n, F &&piece) {
  return populate_from(M, [&](uint32_t k) { return lane_text_byte_plain(c, k); }, root, surf, bp, n, piece);
}

// A sentence a lattice / n-best lane kernel leaves to the long-sentence path: (sentence, exact normalized length or 0
// when unknown) in B.deferred, counted in B.status[0].
__device__ __forceinline__ void lane_defer_long(const KBatch &B, uint32_t sent, uint32_t need) {
  const uint32_t slot = atomicAdd(B.status, 1u);
  B.deferred[2 * slot] = sent;
  B.deferred[2 * slot + 1] = need;
}

// Character starts of a normalized text on the long-sentence path: surf[c] = byte offset of character c (the
// sequential walk of Lattice::SetSentence, p += one_char_len(text[p]) clipped at n), surf[L] = n.  Warp-collective, 32
// bytes per step: the lanes' character lengths go into two ballots and every lane follows the same jumps.  Returns L.
__device__ __forceinline__ uint32_t long_char_starts(const uint8_t *text, uint32_t n, uint32_t *surf, uint32_t lane) {
  uint32_t L = 0, carry = 0;  // carry: first character start of the window, relative to it
  for (uint32_t w0 = 0; w0 < n; w0 += 32) {
    const uint32_t q = w0 + lane;
    const uint32_t len1 = q < n ? one_char_len(text[q]) - 1u : 0u;
    const uint32_t b0 = __ballot_sync(0xFFFFFFFFu, len1 & 1u), b1 = __ballot_sync(0xFFFFFFFFu, len1 & 2u);
    uint32_t starts = 0, p = carry;
    while (p < 32u && w0 + p < n) {
      starts |= 1u << p;
      p += 1u + ((b0 >> p) & 1u) + (((b1 >> p) & 1u) << 1);
    }
    carry = p - 32u;  // the sentence ends inside the window when w0 + p >= n: no later window
    if ((starts >> lane) & 1u) surf[L + __popc(starts & ((1u << lane) - 1u))] = q;
    L += __popc(starts);
  }
  if (lane == 0) surf[L] = n;
  __syncwarp();
  return L;
}

// K4: back-trace + id path of PopulateSentencePieceText (sentencepiece_processor.cc:547-636) over a lane's
// back-pointer log: two coalesced backward scans (count, then write) around one warp-aggregated claim of output space.
// entry t (t = 0..nlog-1) = plen (6 bits) << 24 | (previous char length - 1) << 22 | trie unit (kLaneUnk: UNK piece);
// bit 31 (lane2 whole-word entries): the previous logged position is plen bytes back.
// kWs1: the text and the units are those of lane_normalize<true> and trie_node4 (ids from trie_id_ws); an UNK character
// that is kWsByte falls back to the three byte pieces of E2 96 81.
template <bool kWs1 = false>
__device__ __forceinline__ void lane_finish(const KModel &M, const KBatch &B, const LaneCtx &c, uint32_t n, uint32_t nlog,
                                            uint32_t lane, bool have, bool defer, uint32_t sent, bool bf) {
  // ---------------- K4: coalesced backward scans of the log ----------------
  // entry t (t = 0..nlog-1) belongs to the (t+1)-th character boundary p_t; the character
  // before p_t has (entry>>22 & 3) + 1 bytes, so positions are recovered going backwards.
  const uint32_t max_log = __reduce_max_sync(0xFFFFFFFFu, nlog);
  uint32_t count = 0;
  {
    uint32_t pos_b = n, want = n;
    bool prev_unk = false;
    for (uint32_t tb = (max_log + 3u) & ~3u; tb > 0; tb -= 4) {
      uint32_t ev[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {  // four independent, coalesced loads per trip
        const uint32_t t = tb - 1 - j;
        ev[j] = t < nlog ? slab_ld(c.log + static_cast<size_t>(t) * 32, c.pol) : 0u;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t t = tb - 1 - j;
        if (t < nlog) {
          const uint32_t e = ev[j];
          if (pos_b == want) {
            const uint32_t plen = (e >> 24) & 63u;
            const bool isunk = (e & 0x3FFFFFu) == kLaneUnk;
            if (bf) count += !isunk ? 1u : (kWs1 && plen == 1u && lane_text_byte(c, want - 1u) == kWsByte) ? 3u : plen;
            else count += !(isunk && prev_unk);
            prev_unk = isunk;
            want -= plen;
          }
          pos_b -= (e >> 31) ? ((e >> 24) & 63u) : ((e >> 22) & 3u) + 1u;  // whole-word entries (lane2) step back plen bytes
        }
      }
    }
    if (n && want != 0) { atomicOr(B.status + 1, 1u); count = 0; }
  }
  bool room;
  const unsigned long long pos = lane_claim_output(B, lane, count, have, defer, sent, &room);
  // second backward scan: write ids from the end
  if (room) {
    uint32_t pos_b = n, want = n, w = count;
    bool prev_unk = false;
    for (uint32_t tb = (max_log + 3u) & ~3u; tb > 0; tb -= 4) {
      uint32_t ev[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t t = tb - 1 - j;
        ev[j] = t < nlog ? slab_ld(c.log + static_cast<size_t>(t) * 32, c.pol) : 0u;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
      const uint32_t t = tb - 1 - j;
      if (t < nlog && w > 0) {
        const uint32_t e = ev[j];
        if (pos_b == want) {
          const uint32_t plen = (e >> 24) & 63u;
          const uint32_t idx = e & 0x3FFFFFu;
          const bool isunk = idx == kLaneUnk;
          if (isunk) {
            if (bf) {
              for (uint32_t i = 0; i < plen; ++i) {
                const uint32_t ch = lane_text_byte(c, want - 1 - i);
                if (kWs1 && ch == kWsByte) {  // U+2581 = E2 96 81, written from the end
                  __stcs(B.tmp_ids + pos + (--w), __ldg(M.byte_to_id + 0x81));
                  __stcs(B.tmp_ids + pos + (--w), __ldg(M.byte_to_id + 0x96));
                  __stcs(B.tmp_ids + pos + (--w), __ldg(M.byte_to_id + 0xE2));
                } else {
                  __stcs(B.tmp_ids + pos + (--w), __ldg(M.byte_to_id + ch));
                }
              }
            } else if (!prev_unk) {
              __stcs(B.tmp_ids + pos + (--w), M.unk_id);
            }
          } else {
            __stcs(B.tmp_ids + pos + (--w), __ldg((kWs1 ? M.trie_id_ws : M.trie_id) + idx));  // streaming store
          }
          prev_unk = isunk;
          want -= plen;
        }
        pos_b -= (e >> 31) ? ((e >> 24) & 63u) : ((e >> 22) & 3u) + 1u;  // whole-word entries (lane2) step back plen bytes
      }
      }
    }
  }
  slab_discard(c, lane, (__reduce_max_sync(0xFFFFFFFFu, n) >> 2) + 4u, max_log);
}

// Ring of the unigram lane kernels, R slots per warp.  A slot is a row of 32 scores (f32), then a row of 32 back-pointers
// (u32) and, in encode_unigram_lane_kernel, a row of 32 position tags (u16).  K2 holds the 32-bit shared-memory offset
// of the lane's score in a slot: the back-pointer is kRingBp bytes further, the tag tag_delta = kRingTag - 2 * lane
// bytes further, and the next slot kRingSlot bytes further.  Stepping to a slot is one add and a wrap, and no pointer
// has to be rebuilt inside the loop.
constexpr uint32_t kRingBp = 32u * 4u, kRingTag = 32u * 8u;
constexpr uint32_t kRingSlot = 32u * (4u + 4u + 2u), kPlainRingSlot = 32u * (4u + 4u);
__host__ __device__ inline uint32_t lane_ring_bytes(uint32_t R) { return R * kRingSlot; }
// the same for encode_unigram_lane_plain_kernel, whose slots have no position tag
__host__ __device__ inline uint32_t lane_plain_ring_bytes(uint32_t R) { return R * kPlainRingSlot; }
// Ring accesses by shared-memory address (the kernels fold the CTA's shared-memory base into their ring offsets once).
static_assert(kRingBp == 128, "ring_ld_bp / ring_st_bp spell the back-pointer displacement as +128");
__device__ __forceinline__ float ring_ld_score(uint32_t a) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ring_ld_bp(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1+128];" : "=r"(v) : "r"(a) : "memory");  // + kRingBp
  return v;
}
__device__ __forceinline__ uint32_t ring_ld_tag(uint32_t a) {
  uint16_t v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void ring_st_score(uint32_t a, float v) {
  asm volatile("st.shared.f32 [%0], %1;" :: "r"(a), "f"(v) : "memory");
}
__device__ __forceinline__ void ring_st_bp(uint32_t a, uint32_t v) {
  asm volatile("st.shared.u32 [%0+128], %1;" :: "r"(a), "r"(v) : "memory");  // + kRingBp
}
__device__ __forceinline__ void ring_st_tag(uint32_t a, uint32_t v) {
  asm volatile("st.shared.u16 [%0], %1;" :: "r"(a), "h"(static_cast<uint16_t>(v)) : "memory");
}

// base_regular of the K2 loops: |x| in {0} U [2^-10, 2^18), the range in which the float two-sum decides the reference's
// double comparison exactly (Q1), tested on the bits.  NaN, infinities and denormals fail; -0.0 passes.
__device__ __forceinline__ bool score_regular(float x) {
  const uint32_t a = __float_as_uint(x) << 1;  // the bits of |x|, shifted left by one
  return a == 0u || a - (0x3A800000u << 1) < ((0x48800000u - 0x3A800000u) << 1);  // 2^-10 = 0x3A800000, 2^18 = 0x48800000
}

// Start steps of the unigram lane kernels' K2: the parked lanes (walk over, end-of-walk block pending) run that block
// together once at least kParkNum / kParkDen of the warp's live lanes are parked.  park_need(live) is that count,
// rounded up: 1 <= park_need(live) <= live for live >= 1, and 0 when no lane is live.
constexpr uint32_t kParkNum = 1, kParkDen = 2;
static_assert(0 < kParkNum && kParkNum <= kParkDen, "the start step must run at the latest when every live lane is parked");
__device__ __forceinline__ uint32_t park_need(uint32_t live) { return (live * kParkNum + kParkDen - 1u) / kParkDen; }

constexpr uint32_t kLogWordStep = 1u << 31;  // log entry: the previous logged position is plen bytes back (whole word)
constexpr uint32_t kWsWord = 0x8196E2u;      // U+2581 as the low three bytes of a little-endian word
// OneCharLen in the kWsByte spelling: U+2581 is one byte
__device__ __forceinline__ uint32_t one_char_len_ws1(uint32_t lead) { return lead == kWsByte ? 1u : one_char_len(lead); }

// Whole-word shortcut (kFlagFastWords; engine.cu upload_word_safe has the proof): when no piece contains U+2581
// past its first byte, every segmentation has a token boundary in front of every U+2581, so the Viterbi problem of
// a word [b, e) (U+2581 + the characters up to the next U+2581) only sees the rest of the sentence through the
// float best_path_score at b.  If the word IS a piece P whose score beats the best split of the word by more than
// the rounding noise the float recurrence can accumulate up to position e (M.word_safe[unit] = the largest such e),
// the reference necessarily ends the word with P alone.  The walk from b reaches e on P's node, P has just been
// relaxed into e exactly as the reference relaxes it (first candidate of e), and the starts inside the word are
// skipped: 73 % of the words of the English corpus, half of all character starts.
// The kernel works in the kWsByte spelling throughout (lane_normalize<true>, trie_node4, lane_finish<true>): a word
// starts with one transition on U+2581 instead of three.
__global__ void __launch_bounds__(1024, 1) encode_unigram_lane_kernel(const KModel M, const KBatch B, uint8_t *slabs,
                                                                       uint32_t cap, uint32_t R) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint32_t *s_tab = reinterpret_cast<uint32_t *>(smem);
  fill_lane_tables(M, s_tab);
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp_in_cta = threadIdx.x >> 5;
  const uint32_t warp_global = blockIdx.x * (blockDim.x >> 5) + warp_in_cta;
  const LaneCtx c = lane_ctx(s_tab, slabs, cap, warp_global, lane);
  // ring offsets (see kRingSlot): the lane's score in slot 0, one past the last slot.  Position tags: a slot belongs to
  // position p iff its tag == p (no clearing: skipped positions of whole words leave stale slots behind that simply
  // fail the test).
  const uint32_t ring_lo = static_cast<uint32_t>(__cvta_generic_to_shared(smem)) + kLaneTableBytes +
                           warp_in_cta * lane_ring_bytes(R) + lane * 4u;
  const uint32_t ring_span = lane_ring_bytes(R);
  const uint32_t ring_hi = ring_lo + ring_span;
  const uint32_t tag_delta = kRingTag - 2u * lane;
  const uint4 *node4 = M.trie_node4;
  const uint32_t root = __ldg(&node4[0]).x;
  const bool bf = M.flags & kFlagByteFallback;
  const bool regular = M.flags & kFlagRegularScores;
  const bool fastwords = M.flags & kFlagFastWords;

  uint32_t first = 0;
  while (lane_claim_group(B, lane, &first)) {
    LanePhaseClock clk(B);
    lane_wait_input(B, first, lane);
    const bool have = first + lane < B.n;
    const uint32_t sent = have && B.order ? B.order[first + lane] : first + lane;
    // ---------------- K1 ----------------
    uint32_t n = 0;
    bool defer = false;
    if (have) {
      defer = !lane_k1<true>(M, B, c, sent, cap, &n, 0xFFF0u);  // (positions are 16-bit ring tags)
      if (defer) lane_defer(B, sent);
    }
    __syncwarp();
    clk.mark();
    // ---------------- K2: flat state machine, one trie transition per trip (parked-lane schedule, see below) ----------------
    // text window: words w0..w3 = bytes [4*aw, 4*aw+16), aw = s >> 2; ch = the byte at the walk position k and `cur`
    // streams the bytes after it (low byte first).  ss = ring offset of s's slot.  When the walk ends, ch is the byte
    // that failed the label test or the child mask, for the word-end test of the start step.
    uint32_t s = 0, ss = ring_lo, k = 0, l = root, lsafe = 0, mblen = 1, nlog = 0, ch = 0;
    bool has_single = false, parked = false;  // the lane is done once s reaches n
    bool wstart = fastwords;  // the shortcut is on and s is the first character of a word (text start or kWsByte)
    float base = 0.f;
    bool base_regular = regular;  // base == 0
    uint32_t w0 = 0, w1 = 0, w2 = 0, w3 = 0;
    unsigned long long cur = 0;
    auto window_low = [&]() -> unsigned long long {  // bytes s .. s+7
      const uint32_t sh = (s & 3u) * 8u;
      return static_cast<unsigned long long>(__funnelshift_r(w0, w1, sh)) |
             (static_cast<unsigned long long>(__funnelshift_r(w1, w2, sh)) << 32);
    };
    auto window_high = [&]() -> unsigned long long {  // bytes s+8 .. (at least s+12)
      const uint32_t sh = (s & 3u) * 8u;
      return static_cast<unsigned long long>(__funnelshift_r(w2, w3, sh)) |
             (static_cast<unsigned long long>(w3 >> sh) << 32);
    };
    if (n != 0) {
      for (uint32_t r = 0; r < R; ++r) ring_st_tag(ring_lo + r * kRingSlot + tag_delta, 0xFFFFu);  // no slot belongs to a position of this sentence
      ring_st_score(ring_lo, 0.f);
      w0 = slab_ld(c.text_w + 0, c.pol); w1 = slab_ld(c.text_w + 32, c.pol); w2 = slab_ld(c.text_w + 64, c.pol); w3 = slab_ld(c.text_w + 96, c.pol);
      mblen = one_char_len_ws1(w0 & 0xFFu);
      if (mblen > n) mblen = n;
      cur = window_low();
      ch = static_cast<uint32_t>(cur) & 0xFFu;
      cur >>= 8;
    }
    // optional counters (engine: SPM_B200_KSTATS; device-resident path only): [8] warp trips, [9] lane trips,
    // [10] starts retired, [11] whole words, [12] groups, [13] normalized bytes, [14] start steps.  The loop counts the
    // lane's trips and the warp's trips and start steps (always: a test would cost more than the add); the starts are the
    // log entries and the whole words the entries with kLogWordStep.
    const bool kst = B.kstats != nullptr && B.seg_done == nullptr;
    uint32_t st_lane = 0, st_trips = 0, st_steps = 0;
    // Schedule: a lane whose walk ends parks (the end-of-walk block is pending), and the parked lanes run that block
    // together in a warp-uniform start step once there are park_need(live lanes) of them; every live, unparked lane
    // then takes one trie transition.  Each lane's own sequence of relaxations and log entries is the same as with an
    // end-of-walk block on every trip, only the trip on which it is issued moves.  need == 0: every lane is done.
    uint32_t need = park_need(__popc(__ballot_sync(0xFFFFFFFFu, s < n)));
    while (need != 0) {
      ++st_trips;
      if (__popc(__ballot_sync(0xFFFFFFFFu, parked)) >= need) {
        ++st_steps;
        if (parked) {
          // the walk from s is over (traverse() == -2, or end of text).  Whole word: the walk covered [s, k) from a
          // word start and ended on a NORMAL piece at the end of the word, early enough to be safe.
          const bool fast = wstart && k > s && ((l >> kLinkKindShift) & 3u) == kKindNormal && (k >= n || ch == kWsByte) &&
                            k <= lsafe;
          const uint32_t s_old = s;
          uint32_t steplog;
          if (fast) {
            // the piece was relaxed into k when the walk stepped onto its node; nothing else can win there
            ss += (k - s) * kRingSlot;
            if (ss >= ring_hi) ss -= ring_span;
            s = k;
            steplog = kLogWordStep;
          } else {
            uint32_t sl = ss + mblen * kRingSlot;
            if (sl >= ring_hi) sl -= ring_span;
            if (!has_single) {  // UNK edge, unigram_model.cc:995-1005
              const float cand = __fadd_rn(M.unk_score, base);
              if (ring_ld_tag(sl + tag_delta) != s + mblen || cand > ring_ld_score(sl)) {
                ring_st_score(sl, cand);
                ring_st_bp(sl, (mblen << 24) | kLaneUnk);
                ring_st_tag(sl + tag_delta, s + mblen);
              }
            }
            ss = sl;
            s += mblen;
            steplog = (mblen - 1u) << 22;
          }
          // position s is final: append (plen | previous char length or whole-word step | unit) to the log
          slab_st(c.log + static_cast<size_t>(nlog) * 32, ring_ld_bp(ss) | steplog, c.pol);
          ++nlog;
          if (s < n) {
            base = ring_ld_score(ss);
            base_regular = regular && score_regular(base);
            // slide the text window so that it is anchored at s; prefetch the new tail word
            const uint32_t jw = (s >> 2) - (s_old >> 2);
            if (jw == 1u) {
              w0 = w1; w1 = w2; w2 = w3;
              w3 = slab_ld(c.text_w + static_cast<size_t>((s >> 2) + 3) * 32, c.pol);
            } else if (jw == 2u) {
              w0 = w2; w1 = w3;
              w2 = slab_ld(c.text_w + static_cast<size_t>((s >> 2) + 2) * 32, c.pol);
              w3 = slab_ld(c.text_w + static_cast<size_t>((s >> 2) + 3) * 32, c.pol);
            } else if (jw != 0u) {
              const uint32_t *tw = c.text_w + static_cast<size_t>(s >> 2) * 32;
              w0 = slab_ld(tw + 0, c.pol); w1 = slab_ld(tw + 32, c.pol); w2 = slab_ld(tw + 64, c.pol); w3 = slab_ld(tw + 96, c.pol);
            }
            cur = window_low();
            ch = static_cast<uint32_t>(cur) & 0xFFu;  // the first byte of the new walk
            cur >>= 8;
            wstart = fastwords && ch == kWsByte;
            mblen = one_char_len_ws1(ch);
            if (mblen > n - s) mblen = n - s;
            k = s;
            l = root;
            has_single = false;
          }
          parked = false;
        }
        need = park_need(__popc(__ballot_sync(0xFFFFFFFFu, s < n)));
      }
      // walk step: one transition on ch (k < n holds for every live lane here: a walk that reaches n parks)
      if (s < n && !parked) {
        ++st_lane;
        const uint32_t v = (l >> kLinkBaseShift) ^ ch;
        const uint4 nd = __ldg(&node4[v]);  // {link, child mask, score, word_safe}: one 16-byte load (L1/L2)
        parked = true;
        if ((nd.x & kLinkLabelMask) == ch) {
          ++k;
          l = nd.x;
          lsafe = nd.w;
          const uint32_t kind = (nd.x >> kLinkKindShift) & 3u;
          if (kind == kKindNormal || kind == kKindUserDefined) {
            const uint32_t plen = k - s;
            uint32_t sl = ss + plen * kRingSlot;
            if (sl >= ring_hi) sl -= ring_span;
            const float curs = ring_ld_score(sl);
            const bool unset = ring_ld_tag(sl + tag_delta) != k;
            float ns;
            bool better;
            if (kind == kKindNormal && base_regular) {
              // Exact float formulation of the reference's double comparison (Q1).  With
              // |score|, |base| in {0} U [2^-10, 2^18) the double sum a + b is exact, so
              // (float)cand == fl(a + b) and cand > cur <=> ns > cur || (ns == cur && err > 0),
              // err being the exact rounding error of the float add (Knuth two-sum).
              const float a = __uint_as_float(nd.z);
              ns = __fadd_rn(a, base);
              const float bb = __fsub_rn(ns, a);
              const float err = __fadd_rn(__fsub_rn(a, __fsub_rn(ns, bb)), __fsub_rn(base, bb));
              better = unset || ns > curs || (ns == curs && err > 0.f);
            } else {
              const double sc = kind == kKindNormal
                                    ? static_cast<double>(__uint_as_float(nd.z))
                                    : static_cast<double>(__fmul_rn(static_cast<float>(plen), M.max_score)) - 0.1;
              const double cand = sc + static_cast<double>(base);
              better = unset || cand > static_cast<double>(curs);
              ns = static_cast<float>(cand);
            }
            if (better) {
              ring_st_score(sl, ns);
              ring_st_bp(sl, (plen << 24) | v);
              ring_st_tag(sl + tag_delta, k);
            }
            has_single |= plen == mblen;
          }
          // read the next byte; early termination: if the node has no child on it, the failing
          // probe (and its cold miss) is skipped and the lane parks now
          if (k < n) {
            const uint32_t d = k - s;
            if (d >= 13u) {  // beyond the register window: long piece, rare
              ch = lane_text_byte(c, k);
            } else {
              if (d == 8u) cur = window_high();
              ch = static_cast<uint32_t>(cur) & 0xFFu;
              cur >>= 8;
            }
            parked = !((nd.y >> (ch & 31u)) & 1u);
          }
        }
      }
    }
    if (kst) {
      typedef unsigned long long ull;
      uint32_t st_fast = 0;
      for (uint32_t t = 0; t < nlog; ++t) st_fast += slab_ld(c.log + static_cast<size_t>(t) * 32, c.pol) >> 31;
      st_lane = __reduce_add_sync(0xFFFFFFFFu, st_lane);
      const uint32_t st_starts = __reduce_add_sync(0xFFFFFFFFu, nlog);
      st_fast = __reduce_add_sync(0xFFFFFFFFu, st_fast);
      const uint32_t nb = __reduce_add_sync(0xFFFFFFFFu, n);
      if (lane == 0) {
        atomicAdd(B.kstats + 8, ull(st_trips)); atomicAdd(B.kstats + 9, ull(st_lane)); atomicAdd(B.kstats + 10, ull(st_starts));
        atomicAdd(B.kstats + 11, ull(st_fast)); atomicAdd(B.kstats + 12, ull(1)); atomicAdd(B.kstats + 13, ull(nb));
        atomicAdd(B.kstats + 14, ull(st_steps));
      }
    }
    clk.mark();
    lane_finish<true>(M, B, c, n, nlog, lane, have, defer, sent, bf);  // K4
    clk.mark();
    lane_drain(B, sent, have, lane);  // K6 (fused host path only)
    __syncwarp();
    clk.flush(lane);
  }
}

// The same kernel without the whole-word shortcut: the round-1 state machine (8-byte {link, child mask} nodes, score
// lookup on a match, cleared ring slots instead of position tags).  Text with few space-separated words -- CJK, the
// byte-fallback / mixed-script configuration -- gains nothing from the shortcut and would only pay for its bookkeeping,
// so the engine picks this instantiation for such batches (engine.cu,
// `pick_fast_words`); ring geometry lane_plain_ring_bytes(R) per warp.
__global__ void __launch_bounds__(1024, 1) encode_unigram_lane_plain_kernel(const KModel M, const KBatch B, uint8_t *slabs,
                                                                       uint32_t cap, uint32_t R) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint32_t *s_tab = reinterpret_cast<uint32_t *>(smem);
  fill_lane_tables(M, s_tab);
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp_in_cta = threadIdx.x >> 5;
  const uint32_t warp_global = blockIdx.x * (blockDim.x >> 5) + warp_in_cta;
  const LaneCtx c = lane_ctx(s_tab, slabs, cap, warp_global, lane);
  // ring offsets (see kRingSlot): the lane's score in slot 0, one past the last slot
  const uint32_t ring_lo = static_cast<uint32_t>(__cvta_generic_to_shared(smem)) + kLaneTableBytes +
                           warp_in_cta * lane_plain_ring_bytes(R) + lane * 4u;
  const uint32_t ring_span = lane_plain_ring_bytes(R);
  const uint32_t ring_hi = ring_lo + ring_span;
  const uint2 *node2 = M.trie_node2;
  const uint32_t root = __ldg(&node2[0]).x;
  const bool bf = M.flags & kFlagByteFallback;
  const bool regular = M.flags & kFlagRegularScores;

  uint32_t first = 0;
  while (lane_claim_group(B, lane, &first)) {
    LanePhaseClock clk(B);
    lane_wait_input(B, first, lane);
    const bool have = first + lane < B.n;
    const uint32_t sent = have && B.order ? B.order[first + lane] : first + lane;
    // ---------------- K1 ----------------
    uint32_t n = 0;
    bool defer = false;
    if (have) {
      defer = !lane_k1(M, B, c, sent, cap, &n);
      if (defer) lane_defer(B, sent);
    }
    __syncwarp();
    clk.mark();
    // ---------------- K2: flat state machine, one trie transition per trip (parked-lane schedule) ----------------
    // text window: words w0..w3 = bytes [4*aw, 4*aw+16), aw = s >> 2; ch = the byte at the walk position k and `cur`
    // streams the bytes after it (low byte first).
    uint32_t s = 0, ss = ring_lo /* ring offset of s's slot */, k = 0, l = root, mblen = 1, nlog = 0, ch = 0;
    bool has_single = false, parked = false;  // the lane is done once s reaches n
    float base = 0.f;
    bool base_regular = regular;  // base == 0
    uint32_t w0 = 0, w1 = 0, w2 = 0, w3 = 0;
    unsigned long long cur = 0;
    auto window_low = [&]() -> unsigned long long {  // bytes s .. s+7
      const uint32_t sh = (s & 3u) * 8u;
      return static_cast<unsigned long long>(__funnelshift_r(w0, w1, sh)) |
             (static_cast<unsigned long long>(__funnelshift_r(w1, w2, sh)) << 32);
    };
    auto window_high = [&]() -> unsigned long long {  // bytes s+8 .. (at least s+12)
      const uint32_t sh = (s & 3u) * 8u;
      return static_cast<unsigned long long>(__funnelshift_r(w2, w3, sh)) |
             (static_cast<unsigned long long>(w3 >> sh) << 32);
    };
    if (n != 0) {
      for (uint32_t r = 0; r < R; ++r) ring_st_bp(ring_lo + r * kPlainRingSlot, 0u);  // all positions unset
      ring_st_score(ring_lo, 0.f);
      w0 = slab_ld(c.text_w + 0, c.pol); w1 = slab_ld(c.text_w + 32, c.pol); w2 = slab_ld(c.text_w + 64, c.pol); w3 = slab_ld(c.text_w + 96, c.pol);
      mblen = one_char_len(w0 & 0xFFu);
      if (mblen > n) mblen = n;
      cur = window_low();
      ch = static_cast<uint32_t>(cur) & 0xFFu;
      cur >>= 8;
    }
    // the schedule of encode_unigram_lane_kernel: parked lanes, warp-uniform start steps (park_need)
    uint32_t need = park_need(__popc(__ballot_sync(0xFFFFFFFFu, s < n)));
    while (need != 0) {
      if (__popc(__ballot_sync(0xFFFFFFFFu, parked)) >= need) {
        if (parked) {
          // the walk from s is over (traverse() == -2, or end of text)
          uint32_t sl = ss + mblen * kPlainRingSlot;
          if (sl >= ring_hi) sl -= ring_span;
          if (!has_single) {  // UNK edge, unigram_model.cc:995-1005
            const float cand = __fadd_rn(M.unk_score, base);
            if (ring_ld_bp(sl) == 0u || cand > ring_ld_score(sl)) {
              ring_st_score(sl, cand);
              ring_st_bp(sl, (mblen << 24) | kLaneUnk);
            }
          }
          // position s leaves the window; only character starts are ever targets, so its
          // slot is the only one that has to be cleared for position s + R
          ring_st_bp(ss, 0u);
          s += mblen;
          ss = sl;
          // position s is final: append (plen | previous char length | unit) to the log
          slab_st(c.log + static_cast<size_t>(nlog) * 32, ring_ld_bp(ss) | ((mblen - 1u) << 22), c.pol);
          ++nlog;
          if (s < n) {
            base = ring_ld_score(ss);
            base_regular = regular && score_regular(base);
            // slide the text window so that it is anchored at s; prefetch the new tail word
            if ((s >> 2) != ((s - mblen) >> 2)) {
              w0 = w1; w1 = w2; w2 = w3;
              w3 = slab_ld(c.text_w + static_cast<size_t>((s >> 2) + 3) * 32, c.pol);
            }
            cur = window_low();
            ch = static_cast<uint32_t>(cur) & 0xFFu;  // the first byte of the new walk
            cur >>= 8;
            mblen = one_char_len(ch);
            if (mblen > n - s) mblen = n - s;
            k = s;
            l = root;
            has_single = false;
          }
          parked = false;
        }
        need = park_need(__popc(__ballot_sync(0xFFFFFFFFu, s < n)));
      }
      // walk step: one transition on ch (k < n holds for every live lane here: a walk that reaches n parks)
      if (s < n && !parked) {
        const uint32_t v = (l >> kLinkBaseShift) ^ ch;
        const uint2 nd = __ldg(&node2[v]);  // {link, child mask}: one 8-byte load (L1/L2)
        parked = true;
        if ((nd.x & kLinkLabelMask) == ch) {
          ++k;
          l = nd.x;
          const uint32_t kind = (nd.x >> kLinkKindShift) & 3u;
          if (kind == kKindNormal || kind == kKindUserDefined) {
            const uint32_t plen = k - s;
            uint32_t sl = ss + plen * kPlainRingSlot;
            if (sl >= ring_hi) sl -= ring_span;
            const float curs = ring_ld_score(sl);
            const bool unset = ring_ld_bp(sl) == 0u;
            float ns;
            bool better;
            if (kind == kKindNormal && base_regular) {
              // Exact float formulation of the reference's double comparison (Q1).  With
              // |score|, |base| in {0} U [2^-10, 2^18) the double sum a + b is exact, so
              // (float)cand == fl(a + b) and cand > cur <=> ns > cur || (ns == cur && err > 0),
              // err being the exact rounding error of the float add (Knuth two-sum).
              const float a = __uint_as_float(__ldg(M.trie_val + v));
              ns = __fadd_rn(a, base);
              const float bb = __fsub_rn(ns, a);
              const float err = __fadd_rn(__fsub_rn(a, __fsub_rn(ns, bb)), __fsub_rn(base, bb));
              better = unset || ns > curs || (ns == curs && err > 0.f);
            } else {
              const double sc = kind == kKindNormal
                                    ? static_cast<double>(__uint_as_float(__ldg(M.trie_val + v)))
                                    : static_cast<double>(__fmul_rn(static_cast<float>(plen), M.max_score)) - 0.1;
              const double cand = sc + static_cast<double>(base);
              better = unset || cand > static_cast<double>(curs);
              ns = static_cast<float>(cand);
            }
            if (better) {
              ring_st_score(sl, ns);
              ring_st_bp(sl, (plen << 24) | v);
            }
            has_single |= plen == mblen;
          }
          // read the next byte; early termination: if the node has no child on it, the failing
          // probe (and its cold miss) is skipped and the lane parks now
          if (k < n) {
            const uint32_t d = k - s;
            if (d >= 13u) {  // beyond the register window: long piece, rare
              ch = lane_text_byte(c, k);
            } else {
              if (d == 8u) cur = window_high();
              ch = static_cast<uint32_t>(cur) & 0xFFu;
              cur >>= 8;
            }
            parked = !((nd.y >> (ch & 31u)) & 1u);
          }
        }
      }
    }
    clk.mark();
    lane_finish(M, B, c, n, nlog, lane, have, defer, sent, bf);  // K4
    clk.mark();
    lane_drain(B, sent, have, lane);  // K6 (fused host path only)
    __syncwarp();
    clk.flush(lane);
  }
}


}  // namespace spm_b200
#endif
