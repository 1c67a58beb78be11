// engine.cu -- host side of the engine and the extern "C" boundary (include/spm_b200.h).
//
// Mirrors what SentencePieceProcessor::Load builds on the CPU
// (src/sentencepiece_processor.cc:242-281; ModelInterface::InitializePieces
// src/model_interface.cc:63-151; unigram::Model ctor src/unigram_model.cc:652-670;
// Normalizer::Init src/normalizer.cc:47-69) as flat device tables, and drives the
// kernels of kernels.cuh / bpe_kernel.cuh for a packed batch of sentences.
//
// There is no CPU fallback anywhere in this file: without a CUDA device
// spm_engine_create fails.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cfloat>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <random>
#include <thread>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/spm_b200.h"
#include "bpe_kernel.cuh"
#include "bpe_lane2_kernel.cuh"
#include "device_model.h"
#include "kernels.cuh"
#include "lane_kernel.cuh"
#include "model_reader.h"
#include "order_kernel.cuh"
#include "decode_kernel.cuh"
#include "padded_kernel.cuh"
#include "pieces_kernel.cuh"
#include "nbest_kernel.cuh"
#include "normalize_kernel.cuh"
#include "offsets_kernel.cuh"
#include "chars_kernel.cuh"
#include "lattice_kernel.cuh"
#include "trie_builder.h"

using namespace spm_b200;

namespace {

std::string g_create_error;
std::mutex g_create_mu;

#define CUDA_TRY(expr)                                                                          \
  do {                                                                                          \
    cudaError_t err__ = (expr);                                                                 \
    if (err__ != cudaSuccess) {                                                                 \
      set_error(std::string(#expr) + ": " + cudaGetErrorString(err__));                         \
      return SPM_ERR_CUDA;                                                                      \
    }                                                                                           \
  } while (0)

// passes on the SPM_* code of a call that failed
#define SPM_TRY(...)                                                                            \
  do {                                                                                          \
    const int rc__ = (__VA_ARGS__);                                                             \
    if (rc__ != SPM_OK) return rc__;                                                            \
  } while (0)

// Device and pinned host buffers own their memory: moved, never copied, freed by their destructor.
template <typename T>
struct DevBuf {
  T *p = nullptr;
  size_t cap = 0;  // elements
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  DevBuf(DevBuf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  DevBuf &operator=(DevBuf &&o) noexcept {
    if (this != &o) { release(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; }
    return *this;
  }
  ~DevBuf() { release(); }
  cudaError_t ensure(size_t n, bool keep = false) {
    if (n <= cap) return cudaSuccess;
    size_t want = std::max(n, cap + cap / 2);
    T *np = nullptr;
    cudaError_t e = cudaMalloc(&np, want * sizeof(T) + 256);
    if (e != cudaSuccess) return e;
    if (keep && p && cap) cudaMemcpy(np, p, cap * sizeof(T), cudaMemcpyDeviceToDevice);
    if (p) cudaFree(p);
    p = np;
    cap = want;
    return cudaSuccess;
  }
  cudaError_t upload(const std::vector<T> &v) {
    cudaError_t e = ensure(v.size() ? v.size() : 1);
    if (e != cudaSuccess) return e;
    if (!v.empty()) e = cudaMemcpy(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice);
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

template <typename T>
struct PinBuf {
  T *p = nullptr;
  size_t cap = 0;
  PinBuf() = default;
  PinBuf(const PinBuf &) = delete;
  PinBuf &operator=(const PinBuf &) = delete;
  PinBuf(PinBuf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  PinBuf &operator=(PinBuf &&o) noexcept {
    if (this != &o) { release(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; }
    return *this;
  }
  ~PinBuf() { release(); }
  cudaError_t ensure(size_t n) {
    if (n <= cap) return cudaSuccess;
    size_t want = std::max(n, cap + cap / 2);
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
    cudaError_t e = cudaMallocHost(&p, want * sizeof(T) + 64);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
};

// a copy would free the same memory twice
static_assert(!std::is_copy_constructible<DevBuf<int>>::value && !std::is_copy_constructible<PinBuf<int>>::value,
              "buffers own their memory");

// SPM_B200_TRACE: the chunked host paths print "[trace]" lines to stderr, stamped with the time since the call began.
struct TraceClock {
  const bool on = getenv("SPM_B200_TRACE") != nullptr;
  const std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
  double ms() const { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(); }
};

bool valid_utf8(const char *s, size_t n) {
  size_t i = 0;
  const unsigned char *b = reinterpret_cast<const unsigned char *>(s);
  while (i < n) {
    const unsigned c = b[i];
    size_t l = c < 0x80 ? 1 : (c & 0xE0) == 0xC0 ? 2 : (c & 0xF0) == 0xE0 ? 3 : (c & 0xF8) == 0xF0 ? 4 : 0;
    if (!l || i + l > n) return false;
    uint32_t cp = l == 1 ? c : l == 2 ? c & 0x1F : l == 3 ? c & 0x0F : c & 0x07;
    for (size_t k = 1; k < l; ++k) {
      if ((b[i + k] & 0xC0) != 0x80) return false;
      cp = (cp << 6) | (b[i + k] & 0x3F);
    }
    if ((l == 2 && cp < 0x80) || (l == 3 && cp < 0x800) || (l == 4 && cp < 0x10000) || cp > 0x10FFFF ||
        (cp >= 0xD800 && cp < 0xE000))
      return false;
    i += l;
  }
  return true;
}

// A piece as encode_unigram_lane_kernel spells it: every U+2581 (E2 96 81) becomes the one byte kWsByte.  Pieces are
// valid UTF-8, so E2 96 81 is always that character and the respelling is one to one.
std::string spell_ws_byte(const char *p, size_t n) {
  std::string s;
  s.reserve(n);
  for (size_t i = 0; i < n; ++i) {
    if (i + 2 < n && p[i] == '\xE2' && p[i + 1] == '\x96' && p[i + 2] == '\x81') {
      s.push_back(static_cast<char>(kWsByte));
      i += 2;
    } else {
      s.push_back(p[i]);
    }
  }
  return s;
}

}  // namespace

struct spm_engine {
  int device = 0;
  int sm_count = 0;
  size_t smem_optin = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  std::mutex mu;
  mutable std::string err;
  // Also takes down an engine that create_common gave up on part way.  The buffers free themselves after this body.
  ~spm_engine() {
    cudaSetDevice(device);
    for (cudaStream_t s : {stream, s_h2d, s_d2h})
      if (s) cudaStreamSynchronize(s);
    for (cudaEvent_t x : ev)
      if (x) cudaEventDestroy(x);
    for (int k = 0; k < 2; ++k)
      for (cudaEvent_t x : {ev_in[k], ev_out[k], ev_d2h[k]})
        if (x) cudaEventDestroy(x);
    if (ev_offs) cudaEventDestroy(ev_offs);
    for (cudaStream_t s : {stream, s_h2d, s_d2h})
      if (s) cudaStreamDestroy(s);
  }

  ModelData model;
  DeviceTrie trie, user_trie;
  // unigram: the piece trie with every U+2581 spelled as the one byte kWsByte (lane_kernel.cuh), the key set of
  // encode_unigram_lane_kernel's normalized text; its own unit order, node4 table and unit -> id array
  DeviceTrie trie_ws;
  float min_score = 0.f, max_score = 0.f;
  int32_t unk_id = -1;
  uint32_t max_expand_num = 3, max_expand_den = 1;  // worst-case normalized bytes per input byte
  uint32_t charsmap_units = 0;
  bool bpe_word_split = false;

  // device tables
  DevBuf<uint32_t> d_link, d_val, d_user_link, d_cm_units, d_cm_lead, d_cm_pair, d_node2;
  DevBuf<int32_t> d_id, d_id_ws, d_cm_solo, d_byte_to_id;
  DevBuf<uint8_t> d_cm_targets, d_types;
  DevBuf<float> d_scores;
  DevBuf<uint16_t> d_word_safe;
  DevBuf<uint4> d_node4;
  DevBuf<uint32_t> d_word_fast;
  DevBuf<uint4> d_bpe_cache;
  // SPM_B200_BPE_CACHE: log2 of the word-cache entries (64 bytes each), 0 = no cache.  Measured per step of 1M English
  // sentences with the cache emptied before every step (bench.py, H100 SXM at a 400 W limit, one run each): 2^20
  // 5.80 ms, 2^22 5.73 ms (256 MB of HBM), 2^24 5.93 ms (emptying 1 GB costs more than the extra hits save)
  int bpe_cache_log2 = 22;
  int upload_word_safe();
  KModel km{};

  // tuning
  int G = 1;  // 1: lane kernels (sentence per lane); 32: the general kernels (sentence per warp) for every batch
  int threads = 1024;
  uint32_t ncap = 256;
  static constexpr uint32_t lane_cap = 512;  // normalized-byte capacity per sentence of the lane kernel's slabs
  int ctas_per_sm = 1;

  // per-call buffers (grow only)
  DevBuf<uint8_t> d_bytes, d_tmp_norm, d_norm, d_long_scratch, d_lane_slabs, d_bpe_long;
  DevBuf<uint64_t> d_offsets;
  DevBuf<int32_t> d_tmp_ids, d_ids;
  DevBuf<uint32_t> d_tmp_tok_end, d_tok_end, d_tmp_n2o, d_n2o, d_sent_count, d_norm_len, d_deferred, d_deferred2, d_long_list, d_ctrl32;
  DevBuf<unsigned long long> d_sent_start, d_norm_start, d_id_offsets, d_norm_offsets, d_n2o_offsets, d_block_sums,
      d_ctrl64, d_long_off;
  PinBuf<int32_t> h_ids;
  PinBuf<uint32_t> h_tok_end, h_n2o, h_ctrl32, h_deferred;
  PinBuf<uint64_t> h_id_offsets, h_norm_offsets;
  PinBuf<unsigned long long> h_ctrl64;
  PinBuf<uint8_t> h_norm;
  // pipelined host API: two input slots, two output slots, copy streams
  DevBuf<uint8_t> p_bytes[2];
  DevBuf<uint64_t> p_offsets[2];
  DevBuf<int32_t> p_ids[2];
  DevBuf<unsigned long long> p_id_offsets[2];
  cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
  cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_out[2] = {nullptr, nullptr}, ev_d2h[2] = {nullptr, nullptr};
  int ensure_copy_streams();  // creates the copy streams and the slot events on first use
  // Makes the pinned result buffer `buf` hold `have` + `more` elements (rare), keeping the `have` that have already
  // arrived from s_d2h; the new size extrapolates the elements per item of the first `done` of the batch's n items.
  template <typename T>
  int grow_pinned(PinBuf<T> &buf, unsigned long long have, uint64_t more, size_t done, size_t n) {
    if (have + more + 1 <= buf.cap) return SPM_OK;
    CUDA_TRY(cudaStreamSynchronize(s_d2h));
    PinBuf<T> bigger;
    const double per_item = static_cast<double>(have + more) / static_cast<double>(done);
    CUDA_TRY(bigger.ensure(static_cast<size_t>(per_item * 1.25 * n) + more + 4096));
    if (have) memcpy(bigger.p, buf.p, have * sizeof(T));
    buf = std::move(bigger);
    return SPM_OK;
  }
  size_t pipeline_min_sentences = 300000, pipeline_chunk_sentences = 65536;
  DevBuf<uint32_t> d_order, d_order_hist;  // K0: length-bucketed processing order
  int build_order(const uint64_t *d_offs, size_t n, cudaStream_t st, const uint32_t **order, uint32_t seg);
  bool sort_by_length = true;
  DevBuf<unsigned long long> d_kstats;  // SPM_B200_KSTATS: in-kernel counters of the unigram lane kernel -> stderr
  bool kstats = false;
  // streamed host batches (encode_host_streamed): set around run_device calls
  const uint32_t *cur_ready = nullptr;
  unsigned long long cur_off_lo = 0, cur_off_hi = ~0ull;  // valid offset range of the batch run_device is given
  uint32_t cur_ready_base = 0, cur_piece_shift = 0;
  DevBuf<uint8_t> s_bytes;
  DevBuf<uint64_t> s_offsets;
  DevBuf<uint32_t> d_ready;
  PinBuf<uint32_t> h_marks;
  PinBuf<unsigned long long> h_progress;
  cudaEvent_t ev_offs = nullptr;
  void feed_input(const char *bytes, const uint64_t *offsets, size_t n, size_t piece, std::atomic<int> *rc);
  int encode_host_streamed(const char *bytes, const uint64_t *offsets, size_t n, const int32_t **ids,
                           const uint64_t **id_offsets);
  int encode_host_fused(const char *bytes, const uint64_t *offsets, size_t n, const int32_t **ids, const uint64_t **id_offsets);
  bool fused_host_path = true;
  int fused_skip = 0, fused_backoff = 8;
  DevBuf<uint32_t> d_seg_done, d_sent_rel;
  DevBuf<unsigned long long> d_seg_words;
  // Launch geometry of the lane kernels for an ids-only batch; ok == false: the model / tuning is outside the lane
  // kernels (the general warp-per-sentence kernels take the batch).  Shared memory per warp grows with the longest
  // piece (ring of max(max piece length, 4) + 2 slots), so the warps per CTA shrink until the rings fit.
  struct LaneGeom {
    bool ok = false;
    int version = 1;       // unigram: 2 = encode_unigram_lane_kernel (whole-word shortcut), 1 = the plain instantiation
    int threads = 0;
    uint32_t R = 0, smem = 0;
    uint32_t warp_bytes = 0;  // shared memory per warp: the unigram ring or the BPE symbol arrays and word list
  };
  // unigram: which instantiation takes the next batch -- the whole-word shortcut pays on text made of space-separated
  // words and only costs on text without them (CJK, mixed script).  Decided per call from a sample of the batch's bytes
  // (pick_fast_words); SPM_B200_FASTWORDS=0/1 forces it.
  bool batch_fast_words = true;
  int force_fast_words = -1;
  DevBuf<unsigned long long> d_sample;
  bool pick_fast_words_host(const char *bytes, const uint64_t *offsets, size_t n) const;
  int pick_fast_words_device(const uint8_t *d_bytes_base, const uint64_t *d_offs, size_t n, cudaStream_t st, bool *fast);
  bool any_user_defined = false;
  LaneGeom lane_geometry() const {
    LaneGeom g;
    if (G != 1) return g;
    const size_t avail = smem_optin > kLaneTableBytes ? smem_optin - kLaneTableBytes : 0;
    if (model.model_type == SPM_BPE) {
      if (!((km.flags & kFlagBpeWordSplit) && (km.flags & kFlagEscapeWs) && !(km.flags & (kFlagHasUserSymbols | kFlagHasUnused))))
        return g;
      // (launch bounds: 704 threads -- 22 warps is what the shared-memory arrays allow)
      const int warps = static_cast<int>(std::min<size_t>(std::min(threads, 704) / 32, avail / kBpeLane2WarpBytes));
      if (warps < 4) return g;
      g.ok = true;
      g.threads = warps * 32;
      g.warp_bytes = kBpeLane2WarpBytes;
      g.smem = static_cast<uint32_t>(kLaneTableBytes + static_cast<size_t>(warps) * g.warp_bytes);
      return g;
    }
    if (trie.max_key_len > 62) return g;
    g.version = ((km.flags & kFlagFastWords) && batch_fast_words) ? 2 : 1;  // 2: whole-word shortcut, 1: plain
    // ring of the longest edge + 2 slots: an edge is a piece (version 2 walks the one-byte-U+2581 keys) or the UNK edge
    // over one character, up to 4 bytes -- the kernels step the ring index by an edge length with a single wrap
    const uint32_t longest = g.version == 2 ? trie_ws.max_key_len : trie.max_key_len;
    g.R = std::max<uint32_t>(longest, 4) + 2;
    const uint32_t ring = g.version == 2 ? lane_ring_bytes(g.R) : lane_plain_ring_bytes(g.R);
    const int warps = static_cast<int>(std::min<size_t>(threads / 32, avail / ring));
    if (warps < 4) return g;
    g.ok = true;
    g.threads = warps * 32;
    g.warp_bytes = ring;
    g.smem = static_cast<uint32_t>(kLaneTableBytes + static_cast<size_t>(warps) * ring);
    return g;
  }
  bool uses_lane_kernel() const { return lane_geometry().ok; }
  // Per-warp slabs (normalized text + back-pointer log) of `warps` resident warps of a lane kernel.
  cudaError_t ensure_lane_slabs(size_t warps, uint32_t cap) { return d_lane_slabs.ensure(warps * lane_slab_bytes(cap) + 256); }
  // Launches the lane encode kernel that takes an ids-only batch under `lg` (lg.ok): BPE lane2, or the unigram
  // whole-word (version 2) or plain instantiation.  The slabs (and the BPE long-word scratch) must be in place.
  void launch_lane_encode(const LaneGeom &lg, int grid, const KModel &M, const KBatch &B, cudaStream_t st) {
    if (model.model_type == SPM_BPE)
      encode_bpe_lane2_kernel<<<grid, lg.threads, lg.smem, st>>>(M, B, d_lane_slabs.p, lane_cap, d_bpe_long.p);
    else if (lg.version == 2)
      encode_unigram_lane_kernel<<<grid, lg.threads, lg.smem, st>>>(M, B, d_lane_slabs.p, lane_cap, lg.R);
    else
      encode_unigram_lane_plain_kernel<<<grid, lg.threads, lg.smem, st>>>(M, B, d_lane_slabs.p, lane_cap, lg.R);
  }
  // Decode (K7): per-id decoded strings, built on first use
  DevBuf<uint32_t> d_dec_off, d_dec_info;
  DevBuf<uint8_t> d_dec_bytes, d_dec_tmp, d_dec_text;
  DevBuf<int32_t> d_dec_ids;
  DevBuf<unsigned long long> d_dec_text_offsets;
  DevBuf<uint32_t> d_dec_tok_end;  // spm_decode_offsets: decode_warp_kernel's ENDS mode
  PinBuf<char> h_dec_text;
  PinBuf<uint64_t> h_dec_text_offsets;
  PinBuf<uint32_t> h_dec_tok_end;
  DevBuf<DecStreamState> d_dec_state;  // spm_decode_stream_device: the new states, until the call has succeeded
  uint32_t dec_max_len = 3;            // the longest decoded piece, unk_surface or U+FFFD
  bool dec_ready = false;
  int ensure_decode_tables();
  // decode_warp_kernel's arguments for n id lists (ids indexed by the values of id_offsets), results in d_dec_tmp
  KDecode decode_args(const int32_t *ids, const uint64_t *id_offsets, uint32_t n, unsigned long long tmp_cap) const {
    KDecode D{};
    D.ids = ids;
    D.id_offsets = reinterpret_cast<const unsigned long long *>(id_offsets);
    D.n = n;
    D.vocab = model.vocab_size();
    D.dec_off = d_dec_off.p;
    D.dec_bytes = d_dec_bytes.p;
    D.dec_info = d_dec_info.p;
    D.strip = (model.add_dummy_prefix || model.remove_extra_whitespaces) ? 1u : 0u;
    D.rm = model.remove_extra_whitespaces ? 1u : 0u;
    D.tmp = d_dec_tmp.p;
    D.tmp_cap = tmp_cap;
    D.cursor = d_ctrl64.p;
    D.sent_start = d_sent_start.p;
    D.sent_count = d_sent_count.p;
    D.status = d_ctrl32.p;
    return D;
  }
  // the error behind decode_warp_kernel's status word in h_ctrl32, or SPM_OK; rows: the ROWS mode, which keeps the
  // offending id whole in h_ctrl64[1]
  int decode_error(bool rows = false) const {
    if (h_ctrl32.p[1] == 2u) {  // :915-918
      set_error("Invalid id: " + (rows ? std::to_string(static_cast<long long>(h_ctrl64.p[1]))
                                       : std::to_string(static_cast<int32_t>(h_ctrl32.p[3]))));
      return SPM_ERR_ARG;
    }
    if (h_ctrl32.p[1] == 3u) {  // STREAM mode only
      set_error("Decode: a stream's id count would overflow 2^32 - 1");
      return SPM_ERR_UNSUPPORTED;
    }
    if (h_ctrl32.p[1] == 1u) {
      set_error("Decode: byte piece of id " + std::to_string(h_ctrl32.p[3]) + " is not of the form <0xXX>");
      return SPM_ERR_ENCODE;
    }
    return SPM_OK;
  }
  // large host batches: chunked three-stage pipeline (staged H2D of the ids / decode kernels / D2H of the text)
  DevBuf<int32_t> p_dec_ids[2];
  DevBuf<uint8_t> p_dec_text[2];
  DevBuf<unsigned long long> p_dec_toff[2];
  DevBuf<uint32_t> p_dec_tok_end[2];
  PinBuf<uint8_t> h_stage[2];
  // tok_end != NULL: the ENDS mode, and the token ends are copied back too
  int decode_host_pipelined(const int32_t *ids, const uint64_t *id_offsets, size_t n, const char **text,
                            const uint64_t **text_offsets, const uint32_t **tok_end);
  DevBuf<uint32_t> d_row_len;  // spm_decode_ids_device: the length of every row
  // The decode of n lists on st after the caller's checks: launch(tmp_cap) queues decode_warp_kernel, which is run again
  // with the exact temporary size if it overflowed; then the text is put into list order and copied into the pinned
  // results, and the call waits for it.  rows: launch runs the ROWS mode (for decode_error).  tok_end != NULL: launch
  // runs the ENDS mode into d_dec_tok_end, whose n_tok entries are copied back too.  at_ok (may be empty) queues more
  // work on st once the status words have been read back clean; the call waits for it too.
  template <typename Launch>
  int decode_text(uint32_t n, unsigned long long tmp_cap, bool rows, cudaStream_t st, Launch &&launch, const char **text,
                  const uint64_t **text_offsets, const uint32_t **tok_end = nullptr, uint64_t n_tok = 0,
                  const std::function<int()> &at_ok = {}) {
    CUDA_TRY(d_sent_start.ensure(n));
    CUDA_TRY(d_sent_count.ensure(n));
    CUDA_TRY(d_dec_text_offsets.ensure(n + 1));
    CUDA_TRY(h_dec_text_offsets.ensure(n + 1));
    unsigned long long tot = 0;
    for (int attempt = 0; attempt < 3; ++attempt) {
      CUDA_TRY(d_dec_tmp.ensure(tmp_cap));
      CUDA_TRY(cudaMemsetAsync(d_ctrl32.p, 0, 16 * sizeof(uint32_t), st));
      CUDA_TRY(cudaMemsetAsync(d_ctrl64.p, 0, 8 * sizeof(unsigned long long), st));
      CUDA_TRY(cudaEventRecord(ev[0], st));
      launch(tmp_cap);
      CUDA_TRY(cudaGetLastError());
      CUDA_TRY(cudaEventRecord(ev[1], st));
      ++last_launches;
      SPM_TRY(read_status(st, 16, 8));
      SPM_TRY(decode_error(rows));
      tot = h_ctrl64.p[0];
      if (h_ctrl32.p[2]) { tmp_cap = tot + 1024; continue; }
      break;
    }
    if (h_ctrl32.p[2]) { set_error("Decode: temporary buffer overflow persisted"); return SPM_ERR_CAPACITY; }
    if (at_ok) SPM_TRY(at_ok());
    // offsets (exclusive scan) + gather into list order: the kernels of the encode path
    CUDA_TRY(d_dec_text.ensure(tot + 16));
    SPM_TRY(scan_total(d_sent_count.p, n, 0, d_ctrl64.p + 2, st));
    SPM_TRY(scan_gather<uint8_t>(d_sent_count.p, n, d_dec_text_offsets.p, d_sent_start.p, d_dec_tmp.p, d_dec_text.p,
                                 d_dec_text.cap, 0, 0ull, st));
    CUDA_TRY(cudaEventRecord(ev[2], st));
    CUDA_TRY(h_dec_text.ensure(tot + 1));
    if (tot) CUDA_TRY(cudaMemcpyAsync(h_dec_text.p, d_dec_text.p, tot, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(h_dec_text_offsets.p, d_dec_text_offsets.p, (n + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    if (tok_end) {
      CUDA_TRY(h_dec_tok_end.ensure(n_tok + 1));
      if (n_tok) CUDA_TRY(cudaMemcpyAsync(h_dec_tok_end.p, d_dec_tok_end.p, n_tok * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    }
    CUDA_TRY(cudaStreamSynchronize(st));
    last_d2h = tot + (n + 1) * sizeof(uint64_t) + (tok_end ? n_tok * sizeof(uint32_t) : 0);
    h_dec_text.p[tot] = 0;
    *text = h_dec_text.p;
    *text_offsets = h_dec_text_offsets.p;
    if (tok_end) *tok_end = h_dec_tok_end.p;
    return SPM_OK;
  }
  // EncodeAsPieces (K9): per-id piece bytes, built on first use; the raw ids of the lane kernels, the unknown-surface
  // subset and its spans run, the packed pieces
  DevBuf<uint32_t> d_pc_off, d_pc_flag, d_pc_sub_of, d_pc_sub_len, d_pc_text_len, d_pc_ntok, d_pc_end;
  DevBuf<uint8_t> d_pc_bytes, d_pc_unk, d_pc_sub_bytes, d_pc_text;
  DevBuf<int32_t> d_pc_ids, d_pc_out_ids;
  DevBuf<unsigned long long> d_pc_id_offsets, d_pc_pos, d_pc_sub_start, d_pc_sub_offsets, d_pc_text_offsets,
      d_pc_out_id_offsets;
  PinBuf<char> h_pc_text;
  PinBuf<uint64_t> h_pc_text_offsets;
  PinBuf<uint32_t> h_pc_end;
  bool pc_ready = false;
  int ensure_piece_tables();
  // K9's size pass, scans and write pass over the P.n lists of P (sources and frame set), then the copies of the
  // packed pieces, their ends, the framed ids and both offset arrays into the pinned results; waits for them.
  // *d2h: the bytes copied.
  int write_pieces(KPieces &P, const char *unk_piece, size_t unk_len, const char **text, const uint64_t **text_offsets,
                   const uint32_t **piece_end, const int32_t **ids, const uint64_t **id_offsets, uint64_t *d2h);
  // The raw segmentation of a host batch (n > 0, offsets checked) on the device, for K9 and K11: uploads the input
  // into d_bytes / d_offsets and fills P's sources (ids, id_offsets and, with `detour`, the unknown-surface subset).
  // Sets last_h2d, last_deferred and last_unk_detour; *raw_ids: the ids of the raw segmentation, *main_ms: the encode
  // kernel's time.
  int raw_segmentation(const char *bytes, const uint64_t *offsets, size_t n, bool detour, KPieces *P, uint64_t *raw_ids,
                       float *main_ms);
  // Its device part, for a batch at d_bytes_base + d_offs[i] on st (the unigram kernel choice already made): the encode
  // with the frame off, the unknown flags, the subset pack and the spans run.  at_read (may be empty) is called after
  // the encode, while d_sent_count still holds its raw counts, to queue more work and copies on st; they complete in the
  // status read that gives the detour count, or in a read of their own when no detour count is read.
  int raw_segmentation_device(const uint8_t *d_bytes_base, const uint64_t *d_offs, size_t n, uint64_t total_bytes,
                              bool detour, KPieces *P, uint64_t *raw_ids, float *main_ms, cudaStream_t st,
                              const std::function<int()> &at_read);
  // spm_encode_offsets (K11): begin / end of the framed tokens
  DevBuf<uint32_t> d_off_begin, d_off_end;
  PinBuf<uint32_t> h_off_begin, h_off_end;
  // spm_encode_offsets_device_padded: the longest row, the longest sentence and the K11 chunk plan
  // (offsets_plan_kernel), and their pinned copy
  DevBuf<unsigned long long> d_opad;
  PinBuf<unsigned long long> h_opad;
  // spm_encode_windows_device: the rows R, the longest body, then the first row of each sentence (d_win), their
  // pinned copy (the first two words) and the windows per sentence
  DevBuf<unsigned long long> d_win;
  PinBuf<unsigned long long> h_win;
  DevBuf<uint32_t> d_win_count;
  // spm_encode_pairs_device (which also uses d_win / h_win / d_win_count): the template's ids, each pair's kept ids of
  // A and B per row and the step between its windows
  DevBuf<int32_t> d_pair_tmpl;
  DevBuf<uint2> d_pair_keep;
  DevBuf<uint32_t> d_pair_step;
  // n-best / sampling; pieces: the candidates' token ends and the exported normalized texts (NbestOut)
  DevBuf<uint8_t> d_nb_scratch, d_nb_norm;
  DevBuf<uint32_t> d_nb_end;
  DevBuf<unsigned long long> d_nb_norm_start;
  DevBuf<unsigned long long> d_cand_start, d_cand_offsets;
  DevBuf<uint32_t> d_cand_count, d_n_cands, d_picks;
  DevBuf<float> d_cand_score;
  PinBuf<float> h_cand_score;
  PinBuf<uint32_t> h_n_cands, h_picks;
  PinBuf<uint64_t> h_cand_offsets;
  std::mt19937 rng{5489u};
  // full-lattice operations (lattice_kernel.cuh): exported lattices of one chunk of sentences
  DevBuf<uint8_t> d_lat_scratch;
  DevBuf<uint4> d_lat_nodes;
  DevBuf<uint2> d_lat_pos;
  DevBuf<unsigned long long> d_lat_node_start, d_lat_pos_start;
  DevBuf<uint32_t> d_lat_nchars;
  DevBuf<float> d_lat_entropy;
  PinBuf<uint4> h_lat_nodes;
  PinBuf<uint2> h_lat_pos;
  PinBuf<unsigned long long> h_lat_node_start, h_lat_pos_start;
  PinBuf<uint32_t> h_lat_nchars;
  PinBuf<float> h_lat_entropy;
  std::vector<int32_t> byte_to_id_host;
  std::vector<int32_t> lat_ids;          // results of the last lattice sampling call
  std::vector<uint64_t> lat_offsets;
  std::vector<float> lat_scores;
  std::vector<char> lat_text;            // and its pieces, when asked for (LatPieces)
  std::vector<uint64_t> lat_text_offsets;
  std::vector<uint32_t> lat_piece_end;
  // pieces of the lattice draws, as spm_encode_pieces writes them: unk_piece (null: unknown tokens keep their surface)
  // and sep
  struct LatPieces {
    const char *unk_piece;
    size_t unk_len;
    int sep;
  };
  // mode 0: samples >= 1 draws per sentence from the lattice (ids, offsets[n*samples+1], scores), each with the encode
  // frame -- also the draw of an empty sentence when frame_empty (SampleEncode frames its empty result; an empty
  // sentence has no samples in SampleEncodeAndScore) -- and, with pc, their pieces; mode 1: entropy
  int run_lattice(const char *bytes, const uint64_t *offsets, size_t n, float inv_theta, int mode, int samples,
                  bool frame_empty = false, const LatPieces *pc = nullptr);
  // ends: also the token ends of the candidates (d_nb_end); norm: also the normalized text of every sentence whose
  // lattice holds an UNK node (d_nb_norm, d_nb_norm_start)
  int run_nbest(const char *bytes, const uint64_t *offsets, size_t n, uint32_t nbest, uint64_t *tmp_total,
                bool ends = false, bool norm = false);
  // SampleEncode with nbest_size = K > 1: run_nbest, then the draw on this engine's generator; leaves the picked
  // candidate of every sentence in d_sent_start / d_sent_count.  *d2h: the bytes copied.
  int sample_picks(const char *bytes, const uint64_t *offsets, size_t n, uint32_t K, float alpha, bool ends, bool norm,
                   uint64_t *d2h);
  // Long-sentence path of the lattice and n-best calls: one job per sentence their lane kernels deferred.
  struct LongJob {
    uint32_t sent;     // index in the launch
    uint32_t cap;      // normalized-byte capacity of its slab
    uint32_t hyp_cap;  // n-best: hypothesis pool
  };
  DevBuf<uint32_t> d_long_hyp, d_long_need;
  static constexpr unsigned long long kLongWaveBytes = 1ull << 30;  // scratch of the long jobs of one launch
  int read_deferred(uint32_t n_def, const uint64_t *offs, std::vector<LongJob> *jobs);
  // Runs `jobs` in waves of at most kLongWaveBytes of scratch (a single larger job gets a wave of its own):
  // slab_bytes(job) sizes a job's slab; launch(LB, m) runs the kernel over the m jobs of the wave in LB.long_list /
  // long_scratch_off, their pools in d_long_hyp.  A job whose kernel leaves d_long_need[k] != 0 runs again in a later
  // wave with that pool.  Stops early when the kernel reports an error (h_ctrl32[1]); h_ctrl32 / h_ctrl64 hold the
  // control words after the last wave.
  template <typename SlabBytes, typename Launch>
  int run_long_jobs(std::vector<LongJob> jobs, const KBatch &B, SlabBytes &&slab_bytes, Launch &&launch) {
    cudaStream_t st = stream;
    std::vector<uint32_t> list, hyp, need;
    std::vector<unsigned long long> offs;
    for (size_t lo = 0; lo < jobs.size();) {
      size_t hi = lo;
      offs.assign(1, 0);
      list.clear();
      hyp.clear();
      while (hi < jobs.size() && (hi == lo || offs.back() + slab_bytes(jobs[hi]) <= kLongWaveBytes)) {
        offs.push_back(offs.back() + slab_bytes(jobs[hi]));
        list.push_back(jobs[hi].sent);
        list.push_back(jobs[hi].cap);
        hyp.push_back(jobs[hi].hyp_cap);
        ++hi;
      }
      const uint32_t m = static_cast<uint32_t>(hi - lo);
      CUDA_TRY(d_long_scratch.ensure(offs.back() + 256));
      CUDA_TRY(d_long_list.ensure(2 * static_cast<size_t>(m)));
      CUDA_TRY(d_long_off.ensure(m + 1));
      CUDA_TRY(d_long_hyp.ensure(m));
      CUDA_TRY(d_long_need.ensure(m));
      CUDA_TRY(cudaMemcpyAsync(d_long_list.p, list.data(), 2ull * m * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
      CUDA_TRY(cudaMemcpyAsync(d_long_off.p, offs.data(), (m + 1) * sizeof(unsigned long long), cudaMemcpyHostToDevice, st));
      CUDA_TRY(cudaMemcpyAsync(d_long_hyp.p, hyp.data(), m * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
      CUDA_TRY(cudaMemsetAsync(d_long_need.p, 0, m * sizeof(uint32_t), st));
      KBatch LB = B;
      LB.long_list = d_long_list.p;
      LB.long_n = m;
      LB.long_scratch = d_long_scratch.p;
      LB.long_scratch_off = d_long_off.p;
      launch(LB, m);
      CUDA_TRY(cudaGetLastError());
      ++last_launches;
      need.resize(m);
      CUDA_TRY(cudaMemcpyAsync(need.data(), d_long_need.p, m * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
      SPM_TRY(read_status(st, 16, 4));
      if (h_ctrl32.p[1]) return SPM_OK;
      for (uint32_t k = 0; k < m; ++k)
        if (need[k]) jobs.push_back(LongJob{jobs[lo + k].sent, jobs[lo + k].cap, need[k]});
      lo = hi;
    }
    return SPM_OK;
  }

  // encode frame (spm_engine_set_encode_frame): the ids of P then S, on the host and where the writers read them
  static constexpr uint32_t kMaxFrame = 64;
  std::vector<int32_t> frame_ids;
  uint32_t frame_np = 0, frame_ns = 0;
  bool frame_rev = false;
  DevBuf<int32_t> d_frame;
  KFrame kframe(const uint32_t *n_real = nullptr, uint32_t per = 1) const {
    return KFrame{d_frame.p, frame_np, frame_ns, frame_rev ? 1u : 0u, n_real, per};
  }
  bool framed() const { return frame_np + frame_ns != 0 || frame_rev; }

  // stats of the last call
  uint64_t last_launches = 0, last_h2d = 0, last_d2h = 0, last_deferred = 0, last_unk_detour = 0;
  float last_ms = 0.f, last_main_ms = 0.f;

  void set_error(const std::string &m) const { err = m; }

  // Status words of the kernels (status, counters, cursors, scan totals): d_ctrl32 / d_ctrl64 and their pinned copies,
  // kCtrlWords each, allocated by create_common.  copy_status queues the copy of the first n32 / n64 words on st;
  // read_status also waits for it.
  static constexpr size_t kCtrlWords = 16;
  int copy_status(cudaStream_t st, size_t n32, size_t n64) {
    if (n32) CUDA_TRY(cudaMemcpyAsync(h_ctrl32.p, d_ctrl32.p, n32 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(h_ctrl64.p, d_ctrl64.p, n64 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    return SPM_OK;
  }
  int read_status(cudaStream_t st, size_t n32, size_t n64) {
    SPM_TRY(copy_status(st, n32, n64));
    CUDA_TRY(cudaStreamSynchronize(st));
    return SPM_OK;
  }

  // Exclusive scan of n counts (kernels.cuh), each count plus `extra` and, with F, plus its frame's share.
  // scan_total leaves the block prefixes in d_block_sums and the grand total at d_total (device memory); scan_gather
  // then writes offsets[0..n] (+ off_base) and, when dst is given, copies item i's elements from src + src_start[i]
  // (and src2 into dst2) to dst + offsets[i], within dst_cap.  Between the two a caller may read the total back to size
  // dst.
  int scan_total(const uint32_t *counts, uint32_t n, uint32_t extra, unsigned long long *d_total, cudaStream_t st,
                 const KFrame *F = nullptr) {
    const uint32_t nb = (n + kScanChunk - 1) / kScanChunk;
    CUDA_TRY(d_block_sums.ensure(nb + 1));
    if (F) scan_block_sums_kernel<true><<<nb, 256, 0, st>>>(counts, n, d_block_sums.p, extra, *F);
    else scan_block_sums_kernel<<<nb, 256, 0, st>>>(counts, n, d_block_sums.p, extra);
    scan_block_prefix_kernel<<<1, 1024, 0, st>>>(d_block_sums.p, nb, d_total);
    CUDA_TRY(cudaGetLastError());
    last_launches += 2;
    return SPM_OK;
  }
  template <typename ElemT, bool FRAMED = false>
  int scan_gather(const uint32_t *counts, uint32_t n, unsigned long long *offsets, const unsigned long long *src_start,
                  const ElemT *src, ElemT *dst, unsigned long long dst_cap, uint32_t extra, unsigned long long off_base,
                  cudaStream_t st, const uint32_t *src2 = nullptr, uint32_t *dst2 = nullptr, const KFrame &F = KFrame{}) {
    const uint32_t nb = (n + kScanChunk - 1) / kScanChunk;
    scan_write_gather_kernel<ElemT, FRAMED><<<nb, 256, 0, st>>>(counts, n, d_block_sums.p, offsets, src_start, src, dst,
                                                                src2, dst2, dst_cap, extra, off_base, F);
    CUDA_TRY(cudaGetLastError());
    ++last_launches;
    return SPM_OK;
  }
  int build_tables();
  int upload_types();
  int upload_node2();
  int configure_kernel_attrs();
  // The encode stage of run_device: the encode kernels (lane, second-chance and long-sentence) leave sentence i's raw
  // ids at d_tmp_ids + d_sent_start[i], d_sent_count[i] of them (with spans, also the token ends and the normalized
  // text); its writers follow: run_device's packed one, the padded one of spm_encode_ids_device_padded.
  int encode_stage(const uint8_t *d_bytes_base, const uint64_t *d_offs, size_t n, uint64_t total_bytes, bool spans,
                   cudaStream_t st);
  int run_device(const uint8_t *d_bytes_base, const uint64_t *d_offs, size_t n, uint64_t total_bytes, bool spans,
                 int32_t *user_ids, uint64_t user_ids_cap, unsigned long long *user_id_offsets, uint64_t *total_ids,
                 uint64_t *total_norm, cudaStream_t st, DevBuf<int32_t> *out_ids = nullptr,
                 DevBuf<unsigned long long> *out_offs = nullptr, unsigned long long off_base = 0);
  int encode_host_pipelined(const char *bytes, const uint64_t *offsets, size_t n, const int32_t **ids,
                            const uint64_t **id_offsets);
};

// ---------------------------------------------------------------- model ----

namespace {

// ModelInterface::PieceToId for byte pieces (model_interface.cc:51-61,210-212)
int32_t piece_to_id(const std::unordered_map<std::string, int32_t> &reserved,
                    const std::unordered_map<std::string, int32_t> &pieces, int32_t unk, const std::string &p) {
  auto it = reserved.find(p);
  if (it != reserved.end()) return it->second;
  auto it2 = pieces.find(p);
  if (it2 != pieces.end()) return it2->second;
  return unk;
}

}  // namespace

int spm_engine::build_tables() {
  ModelData &m = model;
  if (m.model_type != SPM_UNIGRAM && m.model_type != SPM_BPE) {
    set_error("only UNIGRAM and BPE models are on the accelerated path (model_factory.cc:25-48)");
    return SPM_ERR_UNSUPPORTED;
  }
  const int V = m.vocab_size();
  // ---- InitializePieces (model_interface.cc:63-151) ----
  std::unordered_map<std::string, int32_t> pieces, reserved;
  std::vector<bool> byte_found(256, false);
  unk_id = -1;
  for (int i = 0; i < V; ++i) {
    const std::string p(m.piece(i), m.piece_len(i));
    if (p.empty()) { set_error("piece must not be empty."); return SPM_ERR_MODEL; }
    const uint8_t t = m.types[i];
    const bool normal = t == SPM_NORMAL || t == SPM_USER_DEFINED || t == SPM_UNUSED;
    if (!(normal ? pieces : reserved).emplace(p, i).second) { set_error(p + " is already defined."); return SPM_ERR_MODEL; }
    if (t == SPM_UNKNOWN) {
      if (unk_id >= 0) { set_error("unk is already defined."); return SPM_ERR_MODEL; }
      unk_id = i;
    }
    if (t == SPM_BYTE) {
      if (!m.byte_fallback) { set_error("byte piece " + p + " is found although `byte_fallback` is false."); return SPM_ERR_MODEL; }
      int b = -1;
      if (p.size() == 6) {
        char canon[8];
        for (int v = 0; v < 256 && b < 0; ++v) {
          snprintf(canon, sizeof canon, "<0x%02X>", v);
          if (p == canon) b = v;
        }
      }
      if (b < 0) { set_error("byte piece " + p + " is invalid."); return SPM_ERR_MODEL; }
      byte_found[b] = true;
    }
  }
  if (unk_id < 0) { set_error("unk is not defined."); return SPM_ERR_MODEL; }
  if (m.byte_fallback && std::find(byte_found.begin(), byte_found.end(), false) != byte_found.end()) {
    set_error("there are not 256 byte pieces although `byte_fallback` is true.");
    return SPM_ERR_MODEL;
  }
  // ---- unigram::Model ctor (unigram_model.cc:657-664): max starts at FLT_MIN (quirk Q3) ----
  min_score = FLT_MAX;
  max_score = FLT_MIN;
  for (int i = 0; i < V; ++i)
    if (m.types[i] == SPM_NORMAL) {
      min_score = std::min(min_score, m.scores[i]);
      max_score = std::max(max_score, m.scores[i]);
    }
  // ---- piece trie over pieces_ (unigram_model.cc:608-650 / bpe pieces_.find) ----
  std::vector<TrieKey> keys, user_keys;
  bool ws_only_at_front = true;
  for (int i = 0; i < V; ++i) {
    const uint8_t t = m.types[i];
    if (!(t == SPM_NORMAL || t == SPM_USER_DEFINED || t == SPM_UNUSED)) continue;
    const float s = m.scores[i];
    const float w = m.model_type == SPM_UNIGRAM ? std::exp(s) : 1.0f / (1.0f + std::fabs(s));
    const uint32_t kind = t == SPM_NORMAL ? kKindNormal : (t == SPM_USER_DEFINED ? kKindUserDefined : kKindUnused);
    keys.push_back({m.piece(i), static_cast<uint32_t>(m.piece_len(i)), i, s, w, kind});
    if (t == SPM_USER_DEFINED) user_keys.push_back({m.piece(i), static_cast<uint32_t>(m.piece_len(i)), i, 0.f, 1.f, kKindNormal});
    if (!valid_utf8(m.piece(i), m.piece_len(i))) {
      set_error("pieces that are not valid UTF-8 are not supported by the device path");
      return SPM_ERR_UNSUPPORTED;
    }
    // U+2581 anywhere but at byte 0 defeats the per-word BPE decomposition
    const std::string p(m.piece(i), m.piece_len(i));
    if (p.find("\xE2\x96\x81", 1) != std::string::npos) ws_only_at_front = false;
  }
  bpe_word_split = ws_only_at_front;
  std::string e;
  if (!BuildDeviceTrie(keys, V, &trie, &e)) { set_error(e); return SPM_ERR_MODEL; }
  if (trie.max_key_len > 255) { set_error("pieces longer than 255 bytes are not supported by the device path"); return SPM_ERR_UNSUPPORTED; }
  if (!user_keys.empty() && !BuildDeviceTrie(user_keys, V, &user_trie, &e)) { set_error(e); return SPM_ERR_MODEL; }
  // the same key set, weights and kinds with U+2581 as one byte (encode_unigram_lane_kernel)
  trie_ws = DeviceTrie();
  if (m.model_type == SPM_UNIGRAM) {
    std::vector<std::string> spelled(keys.size());
    std::vector<TrieKey> ws_keys = keys;
    for (size_t j = 0; j < keys.size(); ++j) {
      spelled[j] = spell_ws_byte(keys[j].data, keys[j].len);
      ws_keys[j].data = spelled[j].data();
      ws_keys[j].len = static_cast<uint32_t>(spelled[j].size());
    }
    if (!BuildDeviceTrie(ws_keys, V, &trie_ws, &e)) { set_error(e); return SPM_ERR_MODEL; }
  }

  // ---- byte fallback ids (sentencepiece_processor.cc:587-588) ----
  std::vector<int32_t> byte_to_id(256, unk_id);
  for (int b = 0; b < 256; ++b) {
    char bp[8];
    snprintf(bp, sizeof bp, "<0x%02X>", b);
    byte_to_id[b] = piece_to_id(reserved, pieces, unk_id, bp);
  }

  // ---- precompiled charsmap (normalizer.cc:274-309) + fast-path tables ----
  std::vector<uint32_t> cm_units, cm_lead(8, 0), cm_pair(128 * 256 / 32, 0);
  std::vector<int32_t> cm_solo(128, -1);
  std::vector<uint8_t> cm_targets(1, 0);
  max_expand_num = m.escape_whitespaces ? 3 : 1;
  max_expand_den = 1;
  if (!m.charsmap.empty()) {
    const std::string &blob = m.charsmap;
    uint32_t trie_bytes = 0;
    if (blob.size() <= 4) { set_error("Blob for normalization rule is broken."); return SPM_ERR_MODEL; }
    memcpy(&trie_bytes, blob.data(), 4);
    if (trie_bytes >= blob.size() - 4 + 4 || trie_bytes + 4 > blob.size()) { set_error("Trie data size exceeds the input blob size."); return SPM_ERR_MODEL; }
    cm_units.resize(trie_bytes / 4);
    memcpy(cm_units.data(), blob.data() + 4, cm_units.size() * 4);
    cm_targets.assign(blob.begin() + 4 + trie_bytes, blob.end());
    cm_targets.push_back(0);  // the blob's last target is NUL-terminated already; be safe
    const size_t NU = cm_units.size();
    auto off = [](uint32_t u) { return (u >> 10) << ((u & (1u << 9)) >> 6); };
    auto label = [](uint32_t u) { return u & ((1u << 31) | 0xFFu); };
    if (NU == 0) { set_error("Blob for normalization rule is broken."); return SPM_ERR_MODEL; }
    // enumerate all keys breadth-first over the double array: (node after the step, depth).  Keys of any length
    // count: a rule set may have keys of hundreds of bytes, and their expansion sizes the long-sentence scratch.  The
    // double array is a DAWG (darts-clone shares common suffixes), so a node can have several parents; breadth-first,
    // a node is first reached at its least depth, where its keys have their highest ratio, and is walked on from there
    // only.  Every edge still sets the lead / pair tables.  At most NU frames, also for a malformed blob.
    struct Fr { uint32_t node; uint32_t depth; uint32_t first; };
    std::vector<Fr> queue;
    std::vector<uint8_t> queued(NU, 0);
    const uint32_t root_next = 0 ^ off(cm_units[0]);
    queue.push_back({root_next, 0, 256});
    for (size_t head = 0; head < queue.size(); ++head) {
      const Fr f = queue[head];
      for (uint32_t c = 0; c < 256; ++c) {
        const uint32_t node = f.node ^ c;
        if (node >= NU) continue;
        const uint32_t unit = cm_units[node];
        if (label(unit) != c) continue;
        const uint32_t first = f.depth == 0 ? c : f.first;
        if (f.depth == 0) cm_lead[c >> 5] |= 1u << (c & 31);
        if (f.depth == 1 && f.first < 128) cm_pair[(f.first * 256 + c) >> 5] |= 1u << (c & 31);
        const uint32_t nxt = node ^ off(unit);
        if ((unit >> 8) & 1u) {
          if (nxt >= NU) { set_error("charsmap trie is malformed"); return SPM_ERR_MODEL; }
          const uint32_t value = cm_units[nxt] & 0x7FFFFFFFu;
          if (value >= cm_targets.size()) { set_error("charsmap target offset out of range"); return SPM_ERR_MODEL; }
          const size_t tl = strlen(reinterpret_cast<const char *>(cm_targets.data()) + value);
          if (!valid_utf8(reinterpret_cast<const char *>(cm_targets.data()) + value, tl)) {
            set_error("charsmap targets that are not valid UTF-8 are not supported by the device path");
            return SPM_ERR_UNSUPPORTED;
          }
          if (f.depth == 0 && c < 128) cm_solo[c] = static_cast<int32_t>(value);
          // expansion: every target byte may be a space that escapes to 3 bytes
          size_t nsp = 0;
          for (size_t k = 0; k < tl; ++k) nsp += cm_targets[value + k] == ' ';
          const uint64_t out_bytes = tl + (m.escape_whitespaces ? 2 * nsp : 0);
          const uint64_t klen = f.depth + 1;
          if (out_bytes * max_expand_den > static_cast<uint64_t>(max_expand_num) * klen) {
            max_expand_num = static_cast<uint32_t>(out_bytes);
            max_expand_den = static_cast<uint32_t>(klen);
          }
        }
        if (queued[node]) continue;
        queued[node] = 1;
        queue.push_back({nxt, f.depth + 1, first});
      }
    }
  }
  // malformed bytes expand 1 -> 3 (U+FFFD)
  if (static_cast<uint64_t>(3) * max_expand_den > max_expand_num) { max_expand_num = 3; max_expand_den = 1; }
  charsmap_units = static_cast<uint32_t>(cm_units.size());

  // ---- upload ----
  if (cudaSetDevice(device) != cudaSuccess) { set_error("cudaSetDevice failed"); return SPM_ERR_CUDA; }
  CUDA_TRY(d_link.upload(trie.link));
  CUDA_TRY(d_val.upload(trie.val));
  CUDA_TRY(d_id.upload(trie.id));
  if (!user_trie.link.empty()) CUDA_TRY(d_user_link.upload(user_trie.link));
  if (cm_units.empty()) cm_units.push_back(0);
  CUDA_TRY(d_cm_units.upload(cm_units));
  CUDA_TRY(d_cm_targets.upload(cm_targets));
  CUDA_TRY(d_cm_lead.upload(cm_lead));
  CUDA_TRY(d_cm_pair.upload(cm_pair));
  CUDA_TRY(d_cm_solo.upload(cm_solo));
  CUDA_TRY(d_byte_to_id.upload(byte_to_id));
  byte_to_id_host = byte_to_id;
  CUDA_TRY(d_scores.upload(m.scores));
  CUDA_TRY(d_types.upload(m.types));

  { const int rc2 = upload_node2(); if (rc2) return rc2; }
  km.trie_link = d_link.p;
  km.trie_val = d_val.p;
  km.trie_id = d_id.p;
  km.trie_units = static_cast<uint32_t>(trie.link.size());
  km.match_slots = trie.max_matches_per_start + 1;
  km.user_link = d_user_link.p;
  km.cm_units = d_cm_units.p;
  km.cm_nunits = charsmap_units;
  km.cm_targets = d_cm_targets.p;
  km.cm_lead = d_cm_lead.p;
  km.cm_pair = d_cm_pair.p;
  km.cm_solo = d_cm_solo.p;
  km.byte_to_id = d_byte_to_id.p;
  km.scores = d_scores.p;
  km.types = d_types.p;
  km.unk_id = unk_id;
  km.unk_score = min_score - 10.0f;  // kUnkPenalty, unigram_model.cc:955
  km.max_score = max_score;
  km.model_type = m.model_type;
  km.flags = (m.add_dummy_prefix ? kFlagAddDummyPrefix : 0) | (m.remove_extra_whitespaces ? kFlagRemoveExtraWs : 0) |
             (m.escape_whitespaces ? kFlagEscapeWs : 0) | (m.treat_whitespace_as_suffix ? kFlagWsSuffix : 0) |
             (m.byte_fallback ? kFlagByteFallback : 0) | (!user_trie.link.empty() ? kFlagHasUserSymbols : 0) |
             (charsmap_units ? kFlagHasCharsmap : 0) | (bpe_word_split ? kFlagBpeWordSplit : 0);
  any_user_defined = false;
  for (uint8_t t : m.types) {
    if (t == SPM_UNUSED) km.flags |= kFlagHasUnused;
    if (t == SPM_USER_DEFINED) any_user_defined = true;
  }
  {
    bool regular = true;
    for (const TrieKey &k : keys) {
      const float a = std::fabs(k.score);
      if (!(k.score == 0.f || (a >= 0.0009765625f && a <= 1024.f))) regular = false;
    }
    if (regular) km.flags |= kFlagRegularScores;
  }
  return upload_word_safe();
}

// whole-word shortcut of the unigram lane kernel (lane_kernel.cuh): for every NORMAL piece P, seen as a word of its own, the largest
// normalized end position e up to which EncodeOptimized (unigram_model.cc:889-1020) is CERTAIN to encode the word
// as P alone, whatever precedes it.
//
// Setting: no piece contains U+2581 past byte 0 and whitespace is escaped, so a word [b, e) -- U+2581 (or the text
// start) up to the next U+2581 -- is only entered through position b and only left through e: the recurrence inside
// the word depends on the rest of the sentence through B = best_path_score[b] alone.  Let S_P be P's score and
// S_alt the best exact (real-number) score of any OTHER segmentation of the word into pieces / UNK edges, built
// with the reference's edge rules (has_single_node, UNUSED skipped, unk_score = min_score - 10).  The reference
// relaxes the whole-word edge first (start b is the earliest start of any edge into e), storing fl(S_P + B).  Every
// float it stores for a position inside the word is within (characters so far) roundings of B + (exact best), and
// every rounding is at most ulp(Vmax) with Vmax >= any |partial score| <= e * maxabs (at most one edge per byte,
// each of magnitude <= maxabs).  So a later candidate into e is at most B + S_alt + c * ulp(Vmax) and cannot
// exceed the stored value (>= B + S_P - ulp(Vmax)) when  S_P - S_alt > (c + 1) * ulp(Vmax).  The table stores the
// largest e for which that holds with a further factor of two of slack on both the margin and Vmax.
//
// The kernel spells U+2581 as the one byte kWsByte, in its normalized text and in its trie (trie_ws), so positions,
// e and the keys here are all in that spelling.  The segmentations of a word, their edges and their scores are the
// same in either spelling, so S_P - S_alt and c do not change.  The bound on Vmax still holds: a path into e has at
// most one edge per character, and every character, U+2581 included, still takes at least one byte, so there are at
// most e edges of magnitude <= maxabs.
int spm_engine::upload_word_safe() {
  std::vector<uint16_t> safe(trie_ws.link.size(), 0);
  const bool eligible = model.model_type == SPM_UNIGRAM && bpe_word_split && model.escape_whitespaces &&
                        !model.treat_whitespace_as_suffix && !any_user_defined && trie.max_key_len <= 62;
  km.flags &= ~kFlagFastWords;
  if (eligible) {
    const int V = model.vocab_size();
    const double unk = static_cast<double>(min_score - 10.0f);
    double maxabs = std::fabs(unk);
    for (int i = 0; i < V; ++i)
      if (model.types[i] == SPM_NORMAL) maxabs = std::max(maxabs, static_cast<double>(std::fabs(model.scores[i])));
    maxabs = std::max(maxabs, 1e-3);
    const double kNegInf = -1e300;
    std::vector<double> E;
    for (int i = 0; i < V; ++i) {
      if (model.types[i] != SPM_NORMAL) continue;
      const uint32_t unit = trie_ws.unit_of_id[i];
      if (unit == 0xFFFFFFFFu) continue;
      const std::string key = spell_ws_byte(model.piece(i), model.piece_len(i));
      const unsigned char *p = reinterpret_cast<const unsigned char *>(key.data());
      const uint32_t L = static_cast<uint32_t>(key.size());
      E.assign(L + 1, kNegInf);
      E[0] = 0.0;
      uint32_t chars = 0;
      for (uint32_t st = 0; st < L;) {
        static const uint8_t kLen[16] = {1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 3, 4};  // OneCharLen, util.h:151-153
        const uint32_t mb = p[st] == kWsByte ? 1u : std::min<uint32_t>(kLen[p[st] >> 4], L - st);
        ++chars;
        if (E[st] > kNegInf) {
          bool has_single = false;
          uint32_t l = trie_ws.link[0];
          for (uint32_t k = st; k < L; ++k) {
            const uint32_t v = (l >> kLinkBaseShift) ^ p[k];
            if (v >= trie_ws.link.size() || (trie_ws.link[v] & kLinkLabelMask) != p[k]) break;
            l = trie_ws.link[v];
            const uint32_t kind = (l >> kLinkKindShift) & 3u;
            if (kind != kKindNormal && kind != kKindUserDefined) continue;
            const uint32_t len = k + 1 - st;
            if (len == mb) has_single = true;
            if (st == 0 && len == L) continue;  // the whole-word edge itself
            float sc;
            memcpy(&sc, &trie_ws.val[v], 4);
            E[st + len] = std::max(E[st + len], E[st] + static_cast<double>(sc));
          }
          if (!has_single) E[st + mb] = std::max(E[st + mb], E[st] + unk);
        }
        st += mb;
      }
      const double margin = E[L] > kNegInf ? static_cast<double>(model.scores[i]) - E[L] : 1e300;
      if (!(margin > 0.0)) continue;
      // (chars + 1) * 2^(kk - 23) < margin / 2   with   Vmax < 2^(kk + 1)
      const double x = margin / (2.0 * (chars + 1));
      const int kk = std::min(40, std::ilogb(x) + 22);
      if (kk < -40) continue;
      const double vmax = std::ldexp(1.0, kk + 1) / (2.0 * maxabs);  // largest admissible e (Vmax = e * maxabs, 2x slack)
      const double e_max = std::floor(vmax) - 1.0;
      if (e_max >= L) safe[unit] = static_cast<uint16_t>(std::min(65535.0, e_max));
    }
    km.flags |= kFlagFastWords;
  }
  // BPE (bpe_lane2_kernel.cuh): word_fast[unit] = id of the piece when the reference's merge loop
  // (bpe_model.cc:38-203: best score, leftmost on ties; candidates are string members of pieces_) run on the piece's
  // own characters ends with the piece as its only symbol; such a word needs no merge loop on the device.
  std::vector<uint32_t> fastw(trie.link.size(), 0xFFFFFFFFu);
  if (model.model_type == SPM_BPE && bpe_word_split && model.escape_whitespaces && !any_user_defined &&
      !(km.flags & kFlagHasUnused)) {
    static const uint8_t kLen[16] = {1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 3, 4};
    auto find = [&](const unsigned char *p, uint32_t len) -> uint32_t {  // exact match: unit of the piece, or ~0
      uint32_t l = trie.link[0], v = 0xFFFFFFFFu;
      for (uint32_t k = 0; k < len; ++k) {
        v = (l >> kLinkBaseShift) ^ p[k];
        if (v >= trie.link.size() || (trie.link[v] & kLinkLabelMask) != p[k]) return 0xFFFFFFFFu;
        l = trie.link[v];
      }
      return ((l >> kLinkKindShift) & 3u) != kKindNone ? v : 0xFFFFFFFFu;
    };
    std::vector<std::pair<uint32_t, uint32_t>> sy;  // (start, length) of the live symbols
    for (int i = 0; i < model.vocab_size(); ++i) {
      const uint32_t unit = trie.unit_of_id[i];
      if (unit == 0xFFFFFFFFu) continue;
      const unsigned char *p = reinterpret_cast<const unsigned char *>(model.piece(i));
      const uint32_t L = static_cast<uint32_t>(model.piece_len(i));
      sy.clear();
      for (uint32_t st = 0; st < L;) {
        const uint32_t mb = std::min<uint32_t>(kLen[p[st] >> 4], L - st);
        sy.emplace_back(st, mb);
        st += mb;
      }
      while (sy.size() > 1) {
        int bi = -1;
        float best = 0.f;
        for (size_t j = 0; j + 1 < sy.size(); ++j) {
          const uint32_t u = find(p + sy[j].first, sy[j].second + sy[j + 1].second);
          if (u == 0xFFFFFFFFu) continue;
          float sc;
          memcpy(&sc, &trie.val[u], 4);
          if (bi < 0 || sc > best) { best = sc; bi = static_cast<int>(j); }
        }
        if (bi < 0) break;
        sy[bi].second += sy[bi + 1].second;
        sy.erase(sy.begin() + bi + 1);
      }
      if (sy.size() == 1) fastw[unit] = static_cast<uint32_t>(i);
    }
  }
  CUDA_TRY(cudaSetDevice(device));
  CUDA_TRY(d_word_safe.upload(safe));
  CUDA_TRY(d_word_fast.upload(fastw));
  km.word_safe = d_word_safe.p;
  km.word_fast = d_word_fast.p;
  // word cache of the BPE lane2 kernel: emptied whenever the tables change (the ids of a word are a function of the
  // vocabulary and the live piece types)
  km.bpe_cache = nullptr;
  km.bpe_cache_mask = 0;
  if (model.model_type == SPM_BPE && bpe_cache_log2 > 0) {
    const size_t entries = size_t{1} << bpe_cache_log2;
    CUDA_TRY(d_bpe_cache.ensure(entries * 4));
    CUDA_TRY(cudaMemset(d_bpe_cache.p, 0, entries * 64));
    CUDA_TRY(cudaDeviceSynchronize());
    km.bpe_cache = d_bpe_cache.p;
    km.bpe_cache_mask = static_cast<uint32_t>(entries - 1);
  }
  {
    std::vector<uint4> n4(trie_ws.link.size());
    for (size_t u = 0; u < trie_ws.link.size(); ++u)
      n4[u] = make_uint4(trie_ws.link[u], trie_ws.cmask[u], trie_ws.val[u], safe[u]);
    CUDA_TRY(d_node4.upload(n4));
    CUDA_TRY(d_id_ws.upload(trie_ws.id));
    km.trie_node4 = d_node4.p;
    km.trie_id_ws = d_id_ws.p;
  }
  return SPM_OK;
}

// {link, child mask} pairs for the lane kernel.
int spm_engine::upload_node2() {
  std::vector<uint32_t> n2(trie.link.size() * 2);
  for (size_t u = 0; u < trie.link.size(); ++u) { n2[2 * u] = trie.link[u]; n2[2 * u + 1] = trie.cmask[u]; }
  CUDA_TRY(d_node2.upload(n2));
  km.trie_node2 = reinterpret_cast<const uint2 *>(d_node2.p);
  return SPM_OK;
}

// Live piece types -> trie link words (kind bits) + types array.
int spm_engine::upload_types() {
  for (int i = 0; i < model.vocab_size(); ++i) {
    const uint32_t u = trie.unit_of_id[i];
    if (u == 0xFFFFFFFFu) continue;
    const uint8_t t = model.types[i];
    const uint32_t kind = t == SPM_NORMAL ? kKindNormal : (t == SPM_USER_DEFINED ? kKindUserDefined : kKindUnused);
    trie.link[u] = (trie.link[u] & ~(3u << kLinkKindShift)) | (kind << kLinkKindShift);
    if (!trie_ws.link.empty()) {
      const uint32_t uw = trie_ws.unit_of_id[i];
      trie_ws.link[uw] = (trie_ws.link[uw] & ~(3u << kLinkKindShift)) | (kind << kLinkKindShift);
    }
  }
  bool any_unused = false;
  any_user_defined = false;
  for (uint8_t t : model.types) { any_unused |= t == SPM_UNUSED; any_user_defined |= t == SPM_USER_DEFINED; }
  km.flags = (km.flags & ~kFlagHasUnused) | (any_unused ? kFlagHasUnused : 0u);
  CUDA_TRY(cudaSetDevice(device));
  CUDA_TRY(d_link.upload(trie.link));
  CUDA_TRY(d_types.upload(model.types));
  { const int rc = upload_node2(); if (rc) return rc; }
  return upload_word_safe();
}

// -------------------------------------------------------------- launches ---

namespace {

struct LaunchGeom {
  uint32_t hot_link, hot_val, tile_bytes, smem_bytes, tiles;
};

// Shared memory of the general (warp-per-sentence) kernels: `tiles` scratch areas of `tile_bytes` first, the rest
// goes to the hot trie prefix (3:1 link:val, both multiples of 4 units for the 16-byte bulk copy).
LaunchGeom plan_geometry(const spm_engine &e, uint32_t tile_bytes, uint32_t tiles) {
  LaunchGeom g{};
  g.tiles = tiles;
  g.tile_bytes = tile_bytes;
  const size_t budget = e.smem_optin / std::max(1, e.ctas_per_sm) - (e.ctas_per_sm > 1 ? 1024 : 0);
  const size_t fixed = 16 + static_cast<size_t>(tiles) * tile_bytes + 128;
  const size_t hot = budget > fixed ? budget - fixed : 0;
  const uint32_t units = e.km.trie_units;
  g.hot_link = static_cast<uint32_t>(std::min<size_t>(units, (hot * 3 / 4) / 4)) & ~3u;
  // if the whole link array fits, the remainder goes to val
  g.hot_val = static_cast<uint32_t>(std::min<size_t>(units, (hot - static_cast<size_t>(g.hot_link) * 4) / 4)) & ~3u;
  g.smem_bytes = static_cast<uint32_t>(16 + static_cast<size_t>(g.hot_link + g.hot_val) * 4 + static_cast<size_t>(tiles) * tile_bytes);
  return g;
}

template <typename KernelT>
cudaError_t set_smem(KernelT k, size_t bytes) {
  return cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
}

}  // namespace

int spm_engine::configure_kernel_attrs() {
  const size_t mx = smem_optin;
  CUDA_TRY(set_smem(encode_unigram_kernel<false>, mx));
  CUDA_TRY(set_smem(encode_unigram_kernel<true>, mx));
  CUDA_TRY(set_smem(encode_unigram_long_kernel<false>, mx));
  CUDA_TRY(set_smem(encode_unigram_long_kernel<true>, mx));
  CUDA_TRY(set_smem(encode_unigram_lane_kernel, mx));
  CUDA_TRY(set_smem(encode_unigram_lane_plain_kernel, mx));
  CUDA_TRY(set_smem(encode_bpe_lane2_kernel, mx));
  CUDA_TRY(set_smem(nbest_lane_kernel<kNbestTop, 1024>, mx));
  CUDA_TRY(set_smem(lattice_lane_kernel, mx));
  CUDA_TRY(set_smem(encode_bpe_kernel<false>, mx));
  CUDA_TRY(set_smem(encode_bpe_kernel<true>, mx));
  CUDA_TRY(set_smem(encode_bpe_long_kernel<false>, mx));
  CUDA_TRY(set_smem(encode_bpe_long_kernel<true>, mx));
  return SPM_OK;
}

// Which instantiation of the unigram lane kernel takes this batch: the whole-word shortcut wants text made of
// space-separated words.  A sample of the batch's bytes decides (one space per <= 16 bytes: words of <= 15 bytes on
// average); results never depend on the choice, only the speed does.
bool spm_engine::pick_fast_words_host(const char *bytes, const uint64_t *offsets, size_t n) const {
  if (force_fast_words >= 0) return force_fast_words != 0;
  if (!(km.flags & kFlagFastWords) || !bytes || n == 0) return true;
  const uint64_t lo = offsets[0], hi = offsets[n];
  if (hi <= lo + 64) return true;
  const uint64_t total = hi - lo, win = std::min<uint64_t>(total, 4096);
  uint64_t spaces = 0, seen = 0;
  for (int w = 0; w < 16; ++w) {
    const uint64_t start = lo + (total - win) * static_cast<uint64_t>(w) / 15;
    for (uint64_t k = 0; k < win; ++k) spaces += bytes[start + k] == ' ';
    seen += win;
  }
  return spaces * 16 >= seen;
}

int spm_engine::pick_fast_words_device(const uint8_t *d_bytes_base, const uint64_t *d_offs, size_t n, cudaStream_t st, bool *fast) {
  *fast = true;
  if (force_fast_words >= 0) { *fast = force_fast_words != 0; return SPM_OK; }
  if (!(km.flags & kFlagFastWords) || n == 0) return SPM_OK;
  CUDA_TRY(d_sample.ensure(2));
  CUDA_TRY(cudaMemsetAsync(d_sample.p, 0, 2 * sizeof(unsigned long long), st));
  sample_spaces_kernel<<<16, 256, 0, st>>>(d_bytes_base, d_offs, static_cast<uint32_t>(n), d_sample.p);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(h_ctrl64.p + 6, d_sample.p, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  const unsigned long long spaces = h_ctrl64.p[6], seen = h_ctrl64.p[7];
  *fast = seen < 64 || spaces * 16 >= seen;
  return SPM_OK;
}

// K0: sentence indices sorted by byte length, longest first, within segments of `seg` sentences (order_kernel.cuh;
// seg = 0: the whole batch is one segment); *order = null for tiny batches
int spm_engine::build_order(const uint64_t *d_offs, size_t n, cudaStream_t st, const uint32_t **order, uint32_t seg) {
  *order = nullptr;
  if (!sort_by_length || n <= 64) return SPM_OK;
  const uint32_t n32 = static_cast<uint32_t>(n);
  if (seg == 0 || seg > n32) seg = n32;
  const uint32_t segs = (n32 + seg - 1) / seg;
  CUDA_TRY(d_order.ensure(n));
  CUDA_TRY(d_order_hist.ensure(static_cast<size_t>(segs) * kOrderBuckets));
  CUDA_TRY(cudaMemsetAsync(d_order_hist.p, 0, static_cast<size_t>(segs) * kOrderBuckets * sizeof(uint32_t), st));
  const uint32_t per_block = kOrderThreads * kOrderPerThread;
  const dim3 grid((seg + per_block - 1) / per_block, segs);
  order_hist_kernel<<<grid, kOrderThreads, 0, st>>>(d_offs, n32, seg, d_order_hist.p);
  order_scan_kernel<<<segs, kOrderBuckets, 0, st>>>(d_order_hist.p);
  order_scatter_kernel<<<grid, kOrderThreads, 0, st>>>(d_offs, n32, seg, d_order_hist.p, d_order.p);
  CUDA_TRY(cudaGetLastError());
  last_launches += 3;
  *order = d_order.p;
  return SPM_OK;
}

int spm_engine::encode_stage(const uint8_t *d_bytes_base, const uint64_t *d_offs, size_t n, uint64_t total_bytes,
                             bool spans, cudaStream_t st) {
  last_launches = 0;
  last_deferred = 0;
  const uint32_t n32 = static_cast<uint32_t>(n);
  const bool bpe = model.model_type == SPM_BPE;
  const int tile_threads = std::min(threads, 512);
  const uint32_t K = km.match_slots;
  // fast path: sentence per lane (lane kernels); else the general kernels, a warp per sentence
  const LaneGeom lg = spans ? LaneGeom{} : lane_geometry();
  const bool lane_path = lg.ok;
  LaunchGeom geom = plan_geometry(*this, bpe ? bpe_tile_bytes(ncap, spans) : tile_bytes_for(ncap, K, spans), tile_threads / 32);
  if (lane_path) {
    geom.tiles = lg.threads / 32;
    geom.tile_bytes = lg.warp_bytes;
    geom.hot_link = geom.hot_val = 0;  // the lane kernels read the trie through L1: rings / word arrays get the shared memory
    geom.smem_bytes = lg.smem;
    const size_t warps_total = static_cast<size_t>(sm_count) * ctas_per_sm * geom.tiles;
    CUDA_TRY(ensure_lane_slabs(warps_total, lane_cap));
    if (bpe) CUDA_TRY(d_bpe_long.ensure(warps_total * bpe_long_bytes(lane_cap)));
  }
  if (geom.smem_bytes > smem_optin) { set_error("shared-memory geometry does not fit; lower smem_norm_cap"); return SPM_ERR_ARG; }
  KModel M = km;
  M.hot_link = geom.hot_link;
  M.hot_val = geom.hot_val;

  // capacities: ids <= normalized bytes; start with one id per input byte (+slack) and
  // retry with the exact requirement when a pathological batch overflows.
  unsigned long long tmp_cap = total_bytes + 4ull * n + 1024;
  unsigned long long norm_cap = spans ? (total_bytes * 2 + 8ull * n + 1024) : 0;
  CUDA_TRY(d_sent_start.ensure(n));
  CUDA_TRY(d_sent_count.ensure(n));
  CUDA_TRY(d_deferred.ensure(2 * n + 2));
  CUDA_TRY(d_deferred2.ensure(2 * n + 2));
  if (spans) {
    CUDA_TRY(d_norm_start.ensure(n));
    CUDA_TRY(d_norm_len.ensure(n));
  }

  const int grid = sm_count * ctas_per_sm;
  for (int attempt = 0; attempt < 3; ++attempt) {
    CUDA_TRY(d_tmp_ids.ensure(tmp_cap));
    if (spans) {
      CUDA_TRY(d_tmp_tok_end.ensure(tmp_cap));
      CUDA_TRY(d_tmp_norm.ensure(norm_cap));
      CUDA_TRY(d_tmp_n2o.ensure(norm_cap));
    }
    CUDA_TRY(cudaMemsetAsync(d_ctrl32.p, 0, 16 * sizeof(uint32_t), st));
    CUDA_TRY(cudaMemsetAsync(d_ctrl64.p, 0, 4 * sizeof(unsigned long long), st));
    KBatch B{};
    B.bytes = d_bytes_base;
    B.offsets = d_offs;
    B.n = n32;
    B.off_lo = cur_off_lo;
    B.off_hi = cur_off_hi;
    B.tmp_ids = d_tmp_ids.p;
    B.tmp_tok_end = d_tmp_tok_end.p;
    B.tmp_cap = tmp_cap;
    B.cursor = d_ctrl64.p;
    B.sent_start = d_sent_start.p;
    B.sent_count = d_sent_count.p;
    B.tmp_norm = d_tmp_norm.p;
    B.tmp_n2o = d_tmp_n2o.p;
    B.tmp_norm_cap = norm_cap;
    B.norm_start = d_norm_start.p;
    B.norm_len = d_norm_len.p;
    B.work_counter = d_ctrl32.p + 4;
    B.deferred = d_deferred.p;
    B.status = d_ctrl32.p;
    B.ncap = ncap;
    B.tile_bytes = geom.tile_bytes;

    CUDA_TRY(cudaEventRecord(ev[0], st));
    if (kstats) {
      CUDA_TRY(d_kstats.ensure(16));
      CUDA_TRY(cudaMemsetAsync(d_kstats.p, 0, 16 * sizeof(unsigned long long), st));
      B.kstats = d_kstats.p;
    }
    if (lane_path) {
      const int rc = build_order(d_offs, n, st, &B.order, cur_ready ? (1u << cur_piece_shift) : 0u);
      if (rc) return rc;
      B.ready = cur_ready;
      B.ready_base = cur_ready_base;
      B.piece_shift = cur_piece_shift;
      launch_lane_encode(lg, grid, M, B, st);
    } else if (bpe) {
      if (spans) encode_bpe_kernel<true><<<grid, tile_threads, geom.smem_bytes, st>>>(M, B);
      else encode_bpe_kernel<false><<<grid, tile_threads, geom.smem_bytes, st>>>(M, B);
    } else if (spans) {
      encode_unigram_kernel<true><<<grid, tile_threads, geom.smem_bytes, st>>>(M, B);
    } else {
      encode_unigram_kernel<false><<<grid, tile_threads, geom.smem_bytes, st>>>(M, B);
    }
    CUDA_TRY(cudaGetLastError());
    ++last_launches;
    CUDA_TRY(cudaEventRecord(ev[1], st));
    SPM_TRY(read_status(st, 16, 4));
    if (kstats) {
      unsigned long long ks[16];
      CUDA_TRY(cudaMemcpy(ks, d_kstats.p, sizeof ks, cudaMemcpyDeviceToHost));
      if (ks[12])
        fprintf(stderr, "[kstats] groups %llu: warp trips/group %.1f, lane trips/sentence %.1f (lane utilisation of K2 %.3f), starts/sentence "
                "%.1f (whole words %.1f), normalized bytes/sentence %.1f (U+2581 as one byte)\n", ks[12], double(ks[8]) / ks[12], double(ks[9]) / n,
                double(ks[9]) / (32.0 * ks[8]), double(ks[10]) / n, double(ks[11]) / n, double(ks[13]) / n);
      if (ks[14])  // K2 runs the end-of-walk block of the parked lanes in warp-uniform start steps
        fprintf(stderr, "[kstats] start steps/group %.1f, lanes per start step %.1f\n", double(ks[14]) / ks[12],
                double(ks[10]) / ks[14]);
      if (ks[4]) {
        const double w = 1e-6 / (static_cast<double>(grid) * geom.tiles);
        fprintf(stderr, "[kstats] M cycles per warp (lane 0): group loop %.2f = K1 %.2f, K2 %.2f, K4 %.2f, rest %.2f\n", ks[4] * w,
                ks[5] * w, ks[6] * w, ks[7] * w, (ks[4] - ks[5] - ks[6] - ks[7]) * w);
      }
    }
    uint32_t n_def = h_ctrl32.p[0];
    const uint32_t *def_list = d_deferred.p;
    // ---- second chance: the sentences a lane kernel could not take (long words, long sentences) go through the
    //      shared-memory warp kernels before the HBM-scratch path -- unless their tiles do not fit in shared memory
    //      (a model with up to 62 piece matches per start), in which case the HBM-scratch path takes them all ----
    const LaunchGeom g2 = n_def && lane_path ? plan_geometry(*this, bpe ? bpe_tile_bytes(ncap, false)
                                                                       : tile_bytes_for(ncap, K, false), tile_threads / 32)
                                             : LaunchGeom{};
    if (n_def && lane_path && g2.smem_bytes <= smem_optin) {
      last_deferred = n_def;
      KModel M2 = km;
      M2.hot_link = g2.hot_link;
      M2.hot_val = g2.hot_val;
      KBatch B2 = B;
      B2.sub_list = d_deferred.p;
      B2.sub_n = n_def;
      B2.deferred = d_deferred2.p;
      B2.status = d_ctrl32.p + 8;
      B2.work_counter = d_ctrl32.p + 12;
      B2.ncap = ncap;
      B2.tile_bytes = g2.tile_bytes;
      const int grid2 = static_cast<int>(std::min<uint32_t>(static_cast<uint32_t>(grid), (n_def + g2.tiles - 1) / g2.tiles));
      if (bpe) encode_bpe_kernel<false><<<grid2, tile_threads, g2.smem_bytes, st>>>(M2, B2);
      else encode_unigram_kernel<false><<<grid2, tile_threads, g2.smem_bytes, st>>>(M2, B2);
      CUDA_TRY(cudaGetLastError());
      ++last_launches;
      SPM_TRY(read_status(st, 16, 4));
      n_def = h_ctrl32.p[8];
      h_ctrl32.p[1] |= h_ctrl32.p[9];
      h_ctrl32.p[2] |= h_ctrl32.p[10];
      def_list = d_deferred2.p;
      M.hot_link = M2.hot_link;  // the long kernels stage the same hot prefix
      M.hot_val = M2.hot_val;
    }
    if (n_def) {
      // ---- long sentences: warp per sentence, scratch slab in HBM ----
      last_deferred = std::max<uint64_t>(last_deferred, n_def);
      CUDA_TRY(h_deferred.ensure(2 * static_cast<size_t>(n_def)));
      CUDA_TRY(cudaMemcpyAsync(h_deferred.p, def_list, 2ull * n_def * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
      // lengths of the deferred sentences whose normalized size is unknown
      std::vector<uint64_t> two(2);
      std::vector<unsigned long long> offs(n_def + 1, 0);
      CUDA_TRY(cudaStreamSynchronize(st));
      for (uint32_t k = 0; k < n_def; ++k) {
        uint32_t need = h_deferred.p[2 * k + 1];
        if (need == 0) {
          const uint32_t s = h_deferred.p[2 * k];
          CUDA_TRY(cudaMemcpy(two.data(), d_offs + s, 16, cudaMemcpyDeviceToHost));
          const uint64_t len = two[1] - two[0];
          const uint64_t bound = (len * max_expand_num + max_expand_den - 1) / max_expand_den + 8;
          if (bound > 0x7FFFFF00ull) { set_error("sentence too long for the device path"); return SPM_ERR_UNSUPPORTED; }
          need = static_cast<uint32_t>(bound);
        }
        need += 8;
        h_deferred.p[2 * k + 1] = need;
        const uint32_t lk = bpe ? 1 : K;
        const unsigned long long bytes = bpe ? bpe_tile_bytes(need, spans) : tile_bytes_for(need, lk, spans);
        offs[k + 1] = offs[k] + ((bytes + 255ull) & ~255ull);
      }
      CUDA_TRY(d_long_scratch.ensure(offs[n_def] + 256));
      CUDA_TRY(d_long_list.ensure(2 * static_cast<size_t>(n_def)));
      CUDA_TRY(d_long_off.ensure(n_def + 1));
      CUDA_TRY(cudaMemcpyAsync(d_long_list.p, h_deferred.p, 2ull * n_def * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
      CUDA_TRY(cudaMemcpyAsync(d_long_off.p, offs.data(), (n_def + 1) * sizeof(unsigned long long), cudaMemcpyHostToDevice, st));
      B.long_list = d_long_list.p;
      B.long_n = n_def;
      B.long_scratch = d_long_scratch.p;
      B.long_scratch_off = d_long_off.p;
      const int lgrid = static_cast<int>(std::min<uint32_t>((n_def + 7) / 8, static_cast<uint32_t>(sm_count) * 4));
      const uint32_t lsmem = 16 + (M.hot_link + M.hot_val) * 4;
      if (bpe) {
        if (spans) encode_bpe_long_kernel<true><<<lgrid, 256, lsmem, st>>>(M, B);
        else encode_bpe_long_kernel<false><<<lgrid, 256, lsmem, st>>>(M, B);
      } else {
        if (spans) encode_unigram_long_kernel<true><<<lgrid, 256, lsmem, st>>>(M, B);
        else encode_unigram_long_kernel<false><<<lgrid, 256, lsmem, st>>>(M, B);
      }
      CUDA_TRY(cudaGetLastError());
      ++last_launches;
      SPM_TRY(read_status(st, 16, 4));
      h_ctrl32.p[1] |= h_ctrl32.p[9];
      h_ctrl32.p[2] |= h_ctrl32.p[10];
    }
    if (h_ctrl32.p[1]) {
      if (h_ctrl32.p[1] & 8u) set_error("encode failed: a long sentence normalized to more bytes than the scratch sized for it");
      else if (h_ctrl32.p[1] & 2u) set_error("encode failed: the host-to-device copy of a streamed batch made no progress for 3 s");
      else set_error("encode failed: internal consistency check (status " + std::to_string(h_ctrl32.p[1]) + ")");
      return SPM_ERR_ENCODE;
    }
    if (h_ctrl32.p[2]) {  // temporary buffers too small: cursors hold the exact requirement
      tmp_cap = h_ctrl64.p[0] + 1024;
      norm_cap = spans ? h_ctrl64.p[1] + 1024 : 0;
      continue;
    }
    break;
  }
  if (h_ctrl32.p[2]) { set_error("temporary buffer overflow persisted"); return SPM_ERR_CAPACITY; }
  return SPM_OK;
}

// Encodes a device-resident batch.  Outputs: ids (+offsets) either into the
// engine's buffers (user_ids == nullptr) or the caller's.
int spm_engine::run_device(const uint8_t *d_bytes_base, const uint64_t *d_offs, size_t n, uint64_t total_bytes,
                           bool spans, int32_t *user_ids, uint64_t user_ids_cap, unsigned long long *user_id_offsets,
                           uint64_t *total_ids, uint64_t *total_norm, cudaStream_t st, DevBuf<int32_t> *out_ids,
                           DevBuf<unsigned long long> *out_offs, unsigned long long off_base) {
  SPM_TRY(encode_stage(d_bytes_base, d_offs, n, total_bytes, spans, st));
  const uint32_t n32 = static_cast<uint32_t>(n);
  // ---- offsets (exclusive scan) + compaction into sentence order; ids (not spans) get the encode frame ----
  const bool framed_ids = !spans && framed();
  SPM_TRY(scan_total(d_sent_count.p, n32, framed_ids ? frame_np + frame_ns : 0u, d_ctrl64.p + 2, st));
  SPM_TRY(read_status(st, 0, 4));
  const unsigned long long tot = h_ctrl64.p[2];  // the cursor over-counts (chunked claims); the scan is exact
  *total_ids = tot;
  if (total_norm) *total_norm = spans ? h_ctrl64.p[1] : 0;
  int32_t *ids_out = user_ids;
  unsigned long long *off_out = user_id_offsets;
  if (!user_ids) {
    DevBuf<int32_t> &ib = out_ids ? *out_ids : d_ids;
    DevBuf<unsigned long long> &ob = out_offs ? *out_offs : d_id_offsets;
    CUDA_TRY(ib.ensure(tot + 1));
    CUDA_TRY(ob.ensure(n + 1));
    ids_out = ib.p;
    off_out = ob.p;
    user_ids_cap = ib.cap;
    if (spans) CUDA_TRY(d_tok_end.ensure(tot + 1));
  } else if (tot > user_ids_cap) {
    set_error("ids_capacity too small: need " + std::to_string(tot));
    return SPM_ERR_CAPACITY;
  }
  if (framed_ids)
    SPM_TRY(scan_gather<int32_t, true>(d_sent_count.p, n32, off_out, d_sent_start.p, d_tmp_ids.p, ids_out, user_ids_cap, 0,
                                       off_base, st, nullptr, nullptr, kframe()));
  else
    SPM_TRY(scan_gather<int32_t>(d_sent_count.p, n32, off_out, d_sent_start.p, d_tmp_ids.p, ids_out, user_ids_cap, 0,
                                 off_base, st, spans ? d_tmp_tok_end.p : nullptr, spans ? d_tok_end.p : nullptr));
  if (spans) {
    const unsigned long long tn = h_ctrl64.p[1];  // sum(n_i + 1)
    CUDA_TRY(d_norm.ensure(tn + 1));
    CUDA_TRY(d_n2o.ensure(tn + 1));
    CUDA_TRY(d_norm_offsets.ensure(n + 1));
    CUDA_TRY(d_n2o_offsets.ensure(n + 1));
    SPM_TRY(scan_total(d_norm_len.p, n32, 0, d_ctrl64.p + 3, st));
    SPM_TRY(scan_gather<uint8_t>(d_norm_len.p, n32, d_norm_offsets.p, d_norm_start.p, d_tmp_norm.p, d_norm.p, d_norm.cap, 0,
                                 0ull, st));
    // norm_to_orig has n_i + 1 entries per sentence: block sums of (len + 1)
    SPM_TRY(scan_total(d_norm_len.p, n32, 1, d_ctrl64.p + 3, st));
    SPM_TRY(scan_gather<uint32_t>(d_norm_len.p, n32, d_n2o_offsets.p, d_norm_start.p, d_tmp_n2o.p, d_n2o.p, d_n2o.cap, 1,
                                  0ull, st));
  }
  CUDA_TRY(cudaEventRecord(ev[2], st));
  return SPM_OK;
}

int spm_engine::ensure_copy_streams() {
  if (s_h2d) return SPM_OK;
  CUDA_TRY(cudaStreamCreateWithFlags(&s_h2d, cudaStreamNonBlocking));
  CUDA_TRY(cudaStreamCreateWithFlags(&s_d2h, cudaStreamNonBlocking));
  for (int k = 0; k < 2; ++k) {
    CUDA_TRY(cudaEventCreateWithFlags(&ev_in[k], cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreateWithFlags(&ev_out[k], cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreateWithFlags(&ev_d2h[k], cudaEventDisableTiming));
  }
  return SPM_OK;
}

// Input feeder of the streamed host paths, run on a helper thread so that the first encode kernel is launched right
// away: the bytes of the batch go to s_bytes in pieces of `piece` sentences, each followed by a 4-byte copy that
// advances the device-side watermark d_ready.  Cuts between the copies sit on 128-byte lines of the device buffer
// (ByteStream in lane_kernel.cuh over-reads within a line).  *rc = 1 when a copy could not be queued.
void spm_engine::feed_input(const char *bytes, const uint64_t *offsets, size_t n, size_t piece, std::atomic<int> *rc) {
  if (cudaSetDevice(device) != cudaSuccess) { *rc = 1; return; }
  const uint64_t total_bytes = offsets[n] - offsets[0];
  const size_t P = (n + piece - 1) / piece;
  uint64_t done_bytes = 0;
  for (size_t p = 0; p < P; ++p) {
    const size_t hi = std::min(n, (p + 1) * piece);
    uint64_t cut = offsets[hi] - offsets[0];
    cut = hi == n ? total_bytes : std::min<uint64_t>(total_bytes, (cut + 127u) & ~uint64_t{127});
    if (cut > done_bytes &&
        cudaMemcpyAsync(s_bytes.p + done_bytes, bytes + offsets[0] + done_bytes, cut - done_bytes, cudaMemcpyHostToDevice,
                        s_h2d) != cudaSuccess) { *rc = 1; return; }
    done_bytes = std::max(done_bytes, cut);
    h_marks.p[p] = static_cast<uint32_t>(hi);
    if (cudaMemcpyAsync(d_ready.p, h_marks.p + p, sizeof(uint32_t), cudaMemcpyHostToDevice, s_h2d) != cudaSuccess) {
      *rc = 1;
      return;
    }
  }
}

// Large host batches: chunked three-stage pipeline.  H2D of chunk c+1 and D2H of chunk c-1
// run on their own streams while chunk c is being encoded; inputs and outputs are double
// buffered, the temporary buffers are only ever touched by the (serial) compute stream.
int spm_engine::encode_host_pipelined(const char *bytes, const uint64_t *offsets, size_t n, const int32_t **ids,
                                      const uint64_t **id_offsets) {
  CUDA_TRY(cudaSetDevice(device));
  for (size_t i = 0; i < n; ++i)
    if (offsets[i + 1] < offsets[i]) { set_error("offsets must be non-decreasing"); return SPM_ERR_ARG; }
  { const int rc = ensure_copy_streams(); if (rc) return rc; }
  // one sentence group (32 sentences) per resident warp and chunk: a launch cannot finish faster than
  // one group, so smaller chunks would only add idle warps
  const bool is_bpe = model.model_type == SPM_BPE;
  const LaneGeom lgw = lane_geometry();
  const size_t warps = static_cast<size_t>(sm_count) * ctas_per_sm * ((lgw.ok ? lgw.threads : std::min(threads, 512)) / 32);
  const size_t groups_per_warp = is_bpe ? 2 : 1;
  const TraceClock trace;
  const size_t chunk = std::max<size_t>(pipeline_chunk_sentences, warps * 32 * groups_per_warp);
  const size_t C = (n + chunk - 1) / chunk;
  const uint64_t total_bytes = offsets[n] - offsets[0];
  CUDA_TRY(h_id_offsets.ensure(n + 1));
  // ids are not known in advance: start from the running average (or 1 id per 3 bytes) and grow
  CUDA_TRY(h_ids.ensure(std::max<size_t>(h_ids.cap, total_bytes / 3 + (2 + frame_np + frame_ns) * n + 4096)));
  uint64_t max_chunk_bytes = 0;
  for (size_t c = 0; c < C; ++c) {
    const size_t lo = c * chunk, hi = std::min(n, lo + chunk);
    max_chunk_bytes = std::max<uint64_t>(max_chunk_bytes, offsets[hi] - offsets[lo]);
  }
  for (int k = 0; k < 2; ++k) {
    CUDA_TRY(p_bytes[k].ensure(max_chunk_bytes + 64));
    CUDA_TRY(p_offsets[k].ensure(chunk + 1));
  }
  auto issue_h2d = [&](size_t c) -> int {
    const int k = static_cast<int>(c & 1);
    const size_t lo = c * chunk, hi = std::min(n, lo + chunk);
    if (c >= 2) CUDA_TRY(cudaStreamWaitEvent(s_h2d, ev_out[k], 0));  // the slot's previous chunk has been encoded
    const uint64_t nb = offsets[hi] - offsets[lo];
    if (nb) CUDA_TRY(cudaMemcpyAsync(p_bytes[k].p, bytes + offsets[lo], nb, cudaMemcpyHostToDevice, s_h2d));
    CUDA_TRY(cudaMemcpyAsync(p_offsets[k].p, offsets + lo, (hi - lo + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, s_h2d));
    CUDA_TRY(cudaEventRecord(ev_in[k], s_h2d));
    return SPM_OK;
  };
  uint64_t launches = 0, deferred = 0;
  float main_ms = 0.f, all_ms = 0.f;
  unsigned long long id_base = 0;
  if (trace.on) fprintf(stderr, "[trace] setup done at %.3f ms\n", trace.ms());
  { const int rc = issue_h2d(0); if (rc) return rc; }
  for (size_t c = 0; c < C; ++c) {
    const int k = static_cast<int>(c & 1);
    const size_t lo = c * chunk, hi = std::min(n, lo + chunk);
    if (c + 1 < C) { const int rc = issue_h2d(c + 1); if (rc) return rc; }
    CUDA_TRY(cudaStreamWaitEvent(stream, ev_in[k], 0));
    if (c >= 2) CUDA_TRY(cudaStreamWaitEvent(stream, ev_d2h[k], 0));  // the slot's previous results have left the GPU
    uint64_t tot = 0;
    const int rc = run_device(p_bytes[k].p - offsets[lo], p_offsets[k].p, hi - lo, offsets[hi] - offsets[lo], false, nullptr, 0,
                              nullptr, &tot, nullptr, stream, &p_ids[k], &p_id_offsets[k], id_base);
    if (rc) { cudaDeviceSynchronize(); return rc; }
    const double t_ret = trace.on ? trace.ms() : 0.0;
    CUDA_TRY(cudaEventRecord(ev_out[k], stream));
    launches += last_launches;
    deferred += last_deferred;
    SPM_TRY(grow_pinned(h_ids, id_base, tot, hi, n));
    CUDA_TRY(cudaStreamWaitEvent(s_d2h, ev_out[k], 0));
    if (tot) CUDA_TRY(cudaMemcpyAsync(h_ids.p + id_base, p_ids[k].p, tot * sizeof(int32_t), cudaMemcpyDeviceToHost, s_d2h));
    CUDA_TRY(cudaMemcpyAsync(h_id_offsets.p + lo, p_id_offsets[k].p, (hi - lo + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, s_d2h));
    CUDA_TRY(cudaEventRecord(ev_d2h[k], s_d2h));
    float a = 0.f;
    if (cudaEventElapsedTime(&a, ev[0], ev[1]) == cudaSuccess) { main_ms += a; all_ms += a; }
    if (trace.on) fprintf(stderr, "[trace] chunk %zu: run_device returned at %.3f ms (encode kernel %.3f ms), D2H issued at %.3f ms\n", c,
                       t_ret, a, trace.ms());
    id_base += tot;
  }
  if (trace.on) fprintf(stderr, "[trace] all chunks issued at %.3f ms\n", trace.ms());
  CUDA_TRY(cudaStreamSynchronize(s_d2h));
  if (trace.on) fprintf(stderr, "[trace] results on host at %.3f ms (%zu chunks of %zu)\n", trace.ms(), C, chunk);
  last_launches = launches;
  last_deferred = deferred;
  last_main_ms = main_ms;
  last_ms = all_ms;
  last_h2d = total_bytes + (n + C) * sizeof(uint64_t);
  last_d2h = id_base * sizeof(int32_t) + (n + C) * sizeof(uint64_t);
  *ids = h_ids.p;
  *id_offsets = h_id_offsets.p;
  return SPM_OK;
}

// Large host batches through the lane kernels: streamed input.  Every H2D copy of the batch is queued up front in
// pieces of 32k sentences, each followed by a 4-byte copy that advances a device-side watermark; the encode kernels
// cover a few large chunks (>= 2 sentence groups per resident warp, so that the length-ordered dynamic schedule can
// balance them) and their warps wait on the watermark for the piece that holds their group.  The kernel of a chunk
// therefore starts as soon as its first piece has landed instead of after the whole chunk, and the D2H of chunk c
// overlaps the encode of chunk c + 1.
int spm_engine::encode_host_streamed(const char *bytes, const uint64_t *offsets, size_t n, const int32_t **ids,
                                     const uint64_t **id_offsets) {
  CUDA_TRY(cudaSetDevice(device));
  { const int rc = ensure_copy_streams(); if (rc) return rc; }
  if (!ev_offs) CUDA_TRY(cudaEventCreateWithFlags(&ev_offs, cudaEventDisableTiming));
  const TraceClock trace;
  constexpr uint32_t kPieceShift = 15;
  constexpr size_t kPiece = size_t{1} << kPieceShift;
  const size_t P = (n + kPiece - 1) / kPiece;
  const bool is_bpe = model.model_type == SPM_BPE;
  const LaneGeom lgw = lane_geometry();
  const size_t warps = static_cast<size_t>(sm_count) * ctas_per_sm * ((lgw.ok ? lgw.threads : std::min(threads, 512)) / 32);
  const size_t groups_per_warp = is_bpe ? 4 : 2;
  const size_t min_chunk = std::max<size_t>(kPiece, warps * 32 * groups_per_warp);
  const size_t want_chunks = std::max<size_t>(1, n / min_chunk);
  const size_t chunk = ((P + want_chunks - 1) / want_chunks) * kPiece;
  const size_t C = (n + chunk - 1) / chunk;
  const uint64_t total_bytes = offsets[n] - offsets[0];
  CUDA_TRY(s_bytes.ensure(total_bytes + 64));
  CUDA_TRY(s_offsets.ensure(n + 1));
  CUDA_TRY(d_ready.ensure(4));
  CUDA_TRY(h_marks.ensure(P + 1));
  CUDA_TRY(h_id_offsets.ensure(n + 1));
  CUDA_TRY(h_ids.ensure(std::max<size_t>(h_ids.cap, total_bytes / 3 + (2 + frame_np + frame_ns) * n + 4096)));
  // ---- queue the whole input ----
  CUDA_TRY(cudaMemsetAsync(d_ready.p, 0, sizeof(uint32_t), s_h2d));
  CUDA_TRY(cudaMemcpyAsync(s_offsets.p, offsets, (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, s_h2d));
  CUDA_TRY(cudaEventRecord(ev_offs, s_h2d));
  {
    uint64_t bad = 0;  // checked while the offsets are on their way
    for (size_t i = 0; i < n; ++i) bad |= static_cast<uint64_t>(offsets[i + 1] < offsets[i]);
    if (bad) {
      cudaStreamSynchronize(s_h2d);
      set_error("offsets must be non-decreasing");
      return SPM_ERR_ARG;
    }
  }
  std::atomic<int> feed_rc{0};
  std::thread feeder([&]() { feed_input(bytes, offsets, n, kPiece, &feed_rc); });
  struct Joiner { std::thread &t; ~Joiner() { if (t.joinable()) t.join(); } } joiner{feeder};
  CUDA_TRY(cudaStreamWaitEvent(stream, ev_offs, 0));
  uint64_t launches = 0, deferred = 0;
  float main_ms = 0.f, all_ms = 0.f;
  unsigned long long id_base = 0;
  for (size_t c = 0; c < C; ++c) {
    const int k = static_cast<int>(c & 1);
    const size_t lo = c * chunk, hi = std::min(n, lo + chunk);
    if (c >= 2) CUDA_TRY(cudaStreamWaitEvent(stream, ev_d2h[k], 0));  // the slot's previous results have left the GPU
    uint64_t tot = 0;
    cur_ready = d_ready.p;
    cur_ready_base = static_cast<uint32_t>(lo);
    cur_piece_shift = kPieceShift;
    const int rc = run_device(s_bytes.p - offsets[0], s_offsets.p + lo, hi - lo, offsets[hi] - offsets[lo], false, nullptr, 0,
                              nullptr, &tot, nullptr, stream, &p_ids[k], &p_id_offsets[k], id_base);
    cur_ready = nullptr;
    if (rc) { cudaDeviceSynchronize(); return rc; }
    const double t_ret = trace.on ? trace.ms() : 0.0;
    CUDA_TRY(cudaEventRecord(ev_out[k], stream));
    launches += last_launches;
    deferred += last_deferred;
    SPM_TRY(grow_pinned(h_ids, id_base, tot, hi, n));
    CUDA_TRY(cudaStreamWaitEvent(s_d2h, ev_out[k], 0));
    if (tot) CUDA_TRY(cudaMemcpyAsync(h_ids.p + id_base, p_ids[k].p, tot * sizeof(int32_t), cudaMemcpyDeviceToHost, s_d2h));
    CUDA_TRY(cudaMemcpyAsync(h_id_offsets.p + lo, p_id_offsets[k].p, (hi - lo + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, s_d2h));
    CUDA_TRY(cudaEventRecord(ev_d2h[k], s_d2h));
    float a = 0.f;
    if (cudaEventElapsedTime(&a, ev[0], ev[1]) == cudaSuccess) { main_ms += a; all_ms += a; }
    if (trace.on) fprintf(stderr, "[trace] chunk %zu (%zu sentences): run_device returned at %.3f ms (encode kernel %.3f ms)\n", c,
                       hi - lo, t_ret, a);
    id_base += tot;
  }
  feeder.join();
  if (feed_rc) { cudaDeviceSynchronize(); set_error("host-to-device copy of a streamed batch failed"); return SPM_ERR_CUDA; }
  CUDA_TRY(cudaStreamSynchronize(s_d2h));
  if (trace.on) fprintf(stderr, "[trace] results on host at %.3f ms\n", trace.ms());
  last_launches = launches;
  last_deferred = deferred;
  last_main_ms = main_ms;
  last_ms = all_ms;
  last_h2d = total_bytes + (n + 1) * sizeof(uint64_t) + P * sizeof(uint32_t);
  last_d2h = id_base * sizeof(int32_t) + (n + C) * sizeof(uint64_t);
  *ids = h_ids.p;
  *id_offsets = h_id_offsets.p;
  return SPM_OK;
}

// Large host batches, fused: ONE launch of a lane kernel for the whole batch.  Input streams in as in
// encode_host_streamed; the results are compacted segment by segment inside the kernel (drain.cuh) straight into the
// pinned host buffers, so the transfer of the ids overlaps the encode and nothing is left to do after the kernel but
// read the status words.  Batches the kernel cannot finish on its own (a sentence deferred to the long path, result
// buffer too small) are redone through encode_host_streamed.
int spm_engine::encode_host_fused(const char *bytes, const uint64_t *offsets, size_t n, const int32_t **ids,
                                  const uint64_t **id_offsets) {
  CUDA_TRY(cudaSetDevice(device));
  { const int rc = ensure_copy_streams(); if (rc) return rc; }
  if (!ev_offs) CUDA_TRY(cudaEventCreateWithFlags(&ev_offs, cudaEventDisableTiming));
  const TraceClock trace;
  constexpr uint32_t kPieceShift = 15;
  constexpr uint32_t kSegShift = 10;
  const size_t kPiece = size_t{1} << kPieceShift;
  const size_t P = (n + kPiece - 1) / kPiece;
  const size_t S = (n + (size_t{1} << kSegShift) - 1) >> kSegShift;
  const uint32_t n32 = static_cast<uint32_t>(n);
  const bool bpe = model.model_type == SPM_BPE;
  const uint64_t total_bytes = offsets[n] - offsets[0];
  cudaStream_t st = stream;
  // ---- buffers ----
  CUDA_TRY(s_bytes.ensure(total_bytes + 64));
  CUDA_TRY(s_offsets.ensure(n + 1));
  CUDA_TRY(d_ready.ensure(4));
  CUDA_TRY(h_marks.ensure(P + 1));
  CUDA_TRY(h_id_offsets.ensure(n + 1));
  CUDA_TRY(h_ids.ensure(std::max<size_t>(h_ids.cap, total_bytes / 2 + (2 + frame_np + frame_ns) * n + 4096)));
  const unsigned long long tmp_cap = total_bytes + 4ull * n + 1024;
  CUDA_TRY(d_tmp_ids.ensure(tmp_cap));
  CUDA_TRY(d_sent_start.ensure(n));
  CUDA_TRY(d_sent_count.ensure(n));
  CUDA_TRY(d_sent_rel.ensure(n));
  CUDA_TRY(d_deferred.ensure(2 * n + 2));
  CUDA_TRY(d_seg_done.ensure(2 * S + 4));   // groups finished [S], copied flags [S], drained counter
  CUDA_TRY(d_seg_words.ensure(2 * S));
  CUDA_TRY(d_ids.ensure(h_ids.cap));
  CUDA_TRY(h_progress.ensure(8));
  *reinterpret_cast<volatile unsigned long long *>(h_progress.p) = 0;
  // ---- launch geometry of the lane kernels (as in run_device) ----
  const LaneGeom lg = lane_geometry();
  if (!lg.ok) { set_error("fused path: the model is outside the lane kernels"); return SPM_ERR_ARG; }
  const int grid = sm_count * ctas_per_sm;
  const size_t warps_total = static_cast<size_t>(grid) * (lg.threads / 32);
  CUDA_TRY(ensure_lane_slabs(warps_total, lane_cap));
  if (bpe) CUDA_TRY(d_bpe_long.ensure(warps_total * bpe_long_bytes(lane_cap)));
  // ---- queue the whole input ----
  CUDA_TRY(cudaMemsetAsync(d_ready.p, 0, sizeof(uint32_t), s_h2d));
  CUDA_TRY(cudaMemcpyAsync(s_offsets.p, offsets, (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, s_h2d));
  CUDA_TRY(cudaEventRecord(ev_offs, s_h2d));
  if (offsets[n] < offsets[0]) { cudaStreamSynchronize(s_h2d); set_error("offsets must be non-decreasing"); return SPM_ERR_ARG; }
  std::atomic<int> feed_rc{0};
  std::thread feeder([&]() { feed_input(bytes, offsets, n, kPiece, &feed_rc); });
  struct Joiner { std::thread &t; ~Joiner() { if (t.joinable()) t.join(); } } joiner{feeder};
  // ---- one launch ----
  last_launches = 0;
  last_deferred = 0;
  CUDA_TRY(cudaStreamWaitEvent(st, ev_offs, 0));
  CUDA_TRY(cudaMemsetAsync(d_ctrl32.p, 0, 16 * sizeof(uint32_t), st));
  CUDA_TRY(cudaMemsetAsync(d_ctrl64.p, 0, 16 * sizeof(unsigned long long), st));
  CUDA_TRY(cudaMemsetAsync(d_seg_done.p, 0, (2 * S + 4) * sizeof(uint32_t), st));
  CUDA_TRY(cudaMemsetAsync(d_seg_words.p, 0, 2 * S * sizeof(unsigned long long), st));
  KModel M = km;
  M.hot_link = M.hot_val = 0;
  KBatch B{};
  B.bytes = s_bytes.p - offsets[0];
  B.offsets = s_offsets.p;
  B.n = n32;
  B.off_lo = offsets[0];
  B.off_hi = offsets[n];
  B.tmp_ids = d_tmp_ids.p;
  B.tmp_cap = tmp_cap;
  B.cursor = d_ctrl64.p;
  B.sent_start = d_sent_start.p;
  B.sent_count = d_sent_count.p;
  B.work_counter = d_ctrl32.p + 4;
  B.deferred = d_deferred.p;
  B.status = d_ctrl32.p;
  B.ready = d_ready.p;
  B.ready_base = 0;
  B.piece_shift = kPieceShift;
  B.seg_shift = kSegShift;
  B.seg_done = d_seg_done.p;
  B.seg_total = d_seg_words.p;
  B.seg_prefix = d_seg_words.p + S;
  B.sent_rel = d_sent_rel.p;
  {
    void *dp = nullptr;
    CUDA_TRY(cudaHostGetDevicePointer(&dp, h_id_offsets.p, 0));
    B.out_offsets = static_cast<unsigned long long *>(dp);
    CUDA_TRY(cudaHostGetDevicePointer(&dp, h_progress.p, 0));
    B.host_progress = static_cast<unsigned long long *>(dp);
  }
  B.out_ids = d_ids.p;
  B.seg_copied = d_seg_done.p + S;
  B.drained_upto = d_seg_done.p + 2 * S;
  B.out_cap = std::min<unsigned long long>(h_ids.cap, d_ids.cap);
  B.out_off_base = 0;
  B.kstats = trace.on ? d_ctrl64.p + 4 : nullptr;
  B.frame = kframe();
  CUDA_TRY(cudaEventRecord(ev[0], st));
  // processing order: sorted within each drain segment.  Sorting whole input pieces instead makes all 32 segments of a
  // piece finish in the same last few groups, whose warps then compact them one after the other, which serializes the
  // drain.
  {
    const int rc = build_order(s_offsets.p, n, st, &B.order, 1u << kSegShift);
    if (rc) return rc;
    if (!B.order) { set_error("fused path needs the segment order"); return SPM_ERR_ARG; }
  }
  launch_lane_encode(lg, grid, M, B, st);
  CUDA_TRY(cudaGetLastError());
  ++last_launches;
  CUDA_TRY(cudaEventRecord(ev[1], st));
  CUDA_TRY(cudaEventRecord(ev[2], st));
  CUDA_TRY(cudaMemcpyAsync(h_ctrl32.p, d_ctrl32.p, 16 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  if (trace.on) CUDA_TRY(cudaMemcpyAsync(h_ctrl64.p, d_ctrl64.p, 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  if (trace.on) fprintf(stderr, "[trace] fused kernel launched at %.3f ms\n", trace.ms());
  // the offsets are checked while the GPU works (a decreasing pair only makes the kernels defer that sentence: the
  // lengths are taken as unsigned); a bad batch is reported after the launch has drained
  uint64_t bad = 0;
  for (size_t i = 0; i < n; ++i) bad |= static_cast<uint64_t>(offsets[i + 1] < offsets[i]);
  // fetch the finished prefix of the ids with the copy engine while the kernel is still encoding
  CUDA_TRY(cudaEventRecord(ev_offs, st));  // (reused) kernel + status copy done
  unsigned long long seen = 0, copied = 0;
  const unsigned long long min_copy = 1ull << 20;  // ids per copy: 4 MB
  for (;;) {
    const cudaError_t q = cudaEventQuery(ev_offs);
    if (q != cudaSuccess && q != cudaErrorNotReady) CUDA_TRY(q);
    const unsigned long long pr = *reinterpret_cast<volatile unsigned long long *>(h_progress.p);
    if (pr > seen && pr <= h_ids.cap) seen = pr;
    if (seen - copied >= min_copy) {
      CUDA_TRY(cudaMemcpyAsync(h_ids.p + copied, d_ids.p + copied, (seen - copied) * sizeof(int32_t), cudaMemcpyDeviceToHost, s_d2h));
      copied = seen;
    }
    if (q == cudaSuccess) break;
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  feeder.join();
  if (trace.on) fprintf(stderr, "[trace] fused kernel done at %.3f ms; warp-cycles: input wait %.1f M, compaction %.1f M (look-back %.1f M), "
                     "%llu groups on %zu warps\n", trace.ms(), h_ctrl64.p[4] * 1e-6, h_ctrl64.p[5] * 1e-6, h_ctrl64.p[6] * 1e-6,
                     static_cast<unsigned long long>(h_ctrl64.p[7]), warps_total);
  if (trace.on) {
    float km = 0.f;
    cudaEventElapsedTime(&km, ev[0], ev[1]);
    const double w = 1e-6 / warps_total;  // M cycles per warp
    fprintf(stderr, "[trace] kernel %.3f ms on the device; M cycles per warp (lane 0): group loop %.2f = K1 + input wait %.2f, K2 %.2f, "
                    "K4 %.2f, drain %.2f\n", km, h_ctrl64.p[8] * w, h_ctrl64.p[9] * w, h_ctrl64.p[10] * w, h_ctrl64.p[11] * w,
            (h_ctrl64.p[8] - h_ctrl64.p[9] - h_ctrl64.p[10] - h_ctrl64.p[11]) * w);
  }
  if (bad) { cudaDeviceSynchronize(); set_error("offsets must be non-decreasing"); return SPM_ERR_ARG; }
  if (feed_rc) { cudaDeviceSynchronize(); set_error("host-to-device copy of a streamed batch failed"); return SPM_ERR_CUDA; }
  if (h_ctrl32.p[1] & 2u) { set_error("encode failed: the host-to-device copy of a streamed batch made no progress for 3 s"); return SPM_ERR_CUDA; }
  if (h_ctrl32.p[1] & 4u) { set_error("encode failed: the in-kernel compaction waited 3 s for an earlier segment"); return SPM_ERR_ENCODE; }
  if (h_ctrl32.p[1]) { set_error("encode failed: internal consistency check (status " + std::to_string(h_ctrl32.p[1]) + ")"); return SPM_ERR_ENCODE; }
  if (h_ctrl32.p[0] || h_ctrl32.p[2]) {
    // deferred sentences or a buffer that was too small: the chunked path has the second-chance and retry logic
    if (trace.on) fprintf(stderr, "[trace] fused path incomplete (deferred %u, overflow %u): redoing the batch in chunks\n",
                       h_ctrl32.p[0], h_ctrl32.p[2]);
    CUDA_TRY(cudaStreamSynchronize(s_d2h));
    // data like this (long words, very long lines) tends to come in runs: go chunked for a while, longer each time
    fused_skip = fused_backoff;
    fused_backoff = std::min(fused_backoff * 4, 1 << 16);
    return encode_host_streamed(bytes, offsets, n, ids, id_offsets);
  }
  fused_backoff = 8;
  const uint64_t tot = h_id_offsets.p[n];
  if (tot > copied) CUDA_TRY(cudaMemcpyAsync(h_ids.p + copied, d_ids.p + copied, (tot - copied) * sizeof(int32_t), cudaMemcpyDeviceToHost, s_d2h));
  CUDA_TRY(cudaStreamSynchronize(s_d2h));
  if (trace.on) fprintf(stderr, "[trace] ids on host at %.3f ms (%llu of %llu fetched while encoding)\n", trace.ms(),
                     static_cast<unsigned long long>(copied), static_cast<unsigned long long>(tot));
  float a = 0.f;
  if (cudaEventElapsedTime(&a, ev[0], ev[1]) != cudaSuccess) a = 0.f;
  last_main_ms = a;
  last_ms = a;
  last_h2d = total_bytes + (n + 1) * sizeof(uint64_t) + P * sizeof(uint32_t);
  last_d2h = tot * sizeof(int32_t) + (n + 1) * sizeof(uint64_t);  // written by the kernel over PCIe
  *ids = h_ids.p;
  *id_offsets = h_id_offsets.p;
  return SPM_OK;
}

// ---- Decode (K7): per-id decoded strings + info words (decode_kernel.cuh) ----
int spm_engine::ensure_decode_tables() {
  if (dec_ready) return SPM_OK;
  const int V = model.vocab_size();
  std::vector<uint32_t> off(V + 1, 0), info(V, 0);
  std::string bytes;
  static const char kSpace[] = "\xE2\x96\x81";
  for (int i = 0; i < V; ++i) {
    const char *p = model.piece(i);
    const size_t len = model.piece_len(i);
    const uint8_t t = model.types[i];
    off[i] = static_cast<uint32_t>(bytes.size());
    if (t == SPM_CONTROL) {
      info[i] = kDecKindControl;
    } else if (t == SPM_UNKNOWN) {
      info[i] = kDecKindUnknown;
      bytes.append(model.unk_surface.c_str());  // the reference takes c_str() (:772-773)
    } else if (t == SPM_BYTE) {
      // PieceToByte (model_interface.cc:214-230): exactly "<0xXX>", upper-case hex
      int v = -1;
      if (len == 6 && p[0] == '<' && p[1] == '0' && p[2] == 'x' && p[5] == '>') {
        auto hex = [](char ch) { return ch >= '0' && ch <= '9' ? ch - '0' : (ch >= 'A' && ch <= 'F' ? ch - 'A' + 10 : -1); };
        const int hi = hex(p[3]), lo = hex(p[4]);
        if (hi >= 0 && lo >= 0) v = hi * 16 + lo;
      }
      info[i] = kDecKindByte | (v < 0 ? kDecBadByte : (static_cast<uint32_t>(v) << kDecByteShift));
      bytes.push_back(static_cast<char>(v < 0 ? 0 : v));
    } else {  // NORMAL, USER_DEFINED, UNUSED: U+2581 -> ' ' (StrReplaceAll, :809)
      info[i] = kDecKindNormal | ((len >= 3 && memcmp(p, kSpace, 3) == 0) ? kDecLeadWs : 0u);
      for (size_t k = 0; k < len;) {
        if (k + 3 <= len && memcmp(p + k, kSpace, 3) == 0) { bytes.push_back(' '); k += 3; }
        else { bytes.push_back(p[k]); k += 1; }
      }
    }
  }
  off[V] = static_cast<uint32_t>(bytes.size());
  dec_max_len = 3;
  for (int i = 0; i < V; ++i) dec_max_len = std::max(dec_max_len, off[i + 1] - off[i]);
  std::vector<uint8_t> b(bytes.begin(), bytes.end());
  b.push_back(0);
  CUDA_TRY(d_dec_off.upload(off));
  CUDA_TRY(d_dec_info.upload(info));
  CUDA_TRY(d_dec_bytes.upload(b));
  dec_ready = true;
  return SPM_OK;
}

// IdToPiece for every id, the raw piece bytes (U+2581 kept).  Piece strings never change after load: SetVocabulary /
// ResetVocabulary only change types (spm_engine_set_types), and the unknown piece is replaced per call.
int spm_engine::ensure_piece_tables() {
  if (pc_ready) return SPM_OK;
  const int V = model.vocab_size();
  std::vector<uint32_t> off(V + 1, 0);
  std::vector<uint8_t> bytes;
  for (int i = 0; i < V; ++i) {
    off[i] = static_cast<uint32_t>(bytes.size());
    bytes.insert(bytes.end(), model.piece(i), model.piece(i) + model.piece_len(i));
  }
  off[V] = static_cast<uint32_t>(bytes.size());
  bytes.push_back(0);
  CUDA_TRY(d_pc_off.upload(off));
  CUDA_TRY(d_pc_bytes.upload(bytes));
  pc_ready = true;
  return SPM_OK;
}

// Host-to-device copy of caller memory: pinned memory goes straight to the copy engine; pageable memory is first
// copied into a pinned staging buffer by a few host threads (the driver's own staging of pageable memory is
// single-threaded and synchronous), then handed to the copy engine.
namespace {
bool is_pinned(const void *p) {
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { (void)cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeHost;
}
void parallel_memcpy(void *dst, const void *src, size_t bytes) {
  const size_t T = bytes < (4u << 20) ? 1 : std::min<size_t>(8, std::max<size_t>(1, std::thread::hardware_concurrency() / 2));
  if (T == 1) { memcpy(dst, src, bytes); return; }
  std::vector<std::thread> th;
  const size_t per = ((bytes + T - 1) / T + 63) & ~size_t{63};
  for (size_t t = 1; t < T; ++t) {
    const size_t lo = std::min(bytes, t * per), hi = std::min(bytes, (t + 1) * per);
    if (hi > lo) th.emplace_back([=]() { memcpy(static_cast<char *>(dst) + lo, static_cast<const char *>(src) + lo, hi - lo); });
  }
  memcpy(dst, src, std::min(bytes, per));
  for (auto &t : th) t.join();
}
}  // namespace

// Decode of a large host batch: chunks of id lists flow through H2D (staged when the caller's memory is pageable),
// decode + scan + gather, and D2H of the text on three streams; inputs and outputs are double buffered.
int spm_engine::decode_host_pipelined(const int32_t *ids, const uint64_t *id_offsets, size_t n, const char **text,
                                      const uint64_t **text_offsets, const uint32_t **tok_end) {
  { const int rc = ensure_copy_streams(); if (rc) return rc; }
  cudaStream_t st = stream;
  const TraceClock trace;
  const size_t chunk = 131072;
  const size_t C = (n + chunk - 1) / chunk;
  const bool pinned_in = is_pinned(ids);
  uint64_t max_ids = 0;
  for (size_t c = 0; c < C; ++c) max_ids = std::max<uint64_t>(max_ids, id_offsets[std::min(n, (c + 1) * chunk)] - id_offsets[c * chunk]);
  const uint64_t total_ids = id_offsets[n] - id_offsets[0];
  for (int k = 0; k < 2; ++k) {
    CUDA_TRY(p_dec_ids[k].ensure(max_ids + 1));
    CUDA_TRY(p_offsets[k].ensure(chunk + 1));
    CUDA_TRY(p_dec_toff[k].ensure(chunk + 1));
    if (tok_end) CUDA_TRY(p_dec_tok_end[k].ensure(max_ids + 1));
    if (!pinned_in) CUDA_TRY(h_stage[k].ensure(max_ids * sizeof(int32_t) + 64));
  }
  CUDA_TRY(h_dec_text_offsets.ensure(n + 1));
  if (tok_end) CUDA_TRY(h_dec_tok_end.ensure(total_ids + 1));
  CUDA_TRY(h_dec_text.ensure(std::max<size_t>(h_dec_text.cap, total_ids * 5 + 16 * n + 4096)));
  CUDA_TRY(d_sent_start.ensure(chunk));
  CUDA_TRY(d_sent_count.ensure(chunk));
  auto issue_h2d = [&](size_t c) -> int {
    const int k = static_cast<int>(c & 1);
    const size_t lo = c * chunk, hi = std::min(n, lo + chunk);
    const uint64_t cnt = id_offsets[hi] - id_offsets[lo];
    if (c >= 2) {
      CUDA_TRY(cudaStreamWaitEvent(s_h2d, ev_out[k], 0));  // the slot's previous chunk has been decoded
      if (!pinned_in) CUDA_TRY(cudaEventSynchronize(ev_in[k]));  // ... and its staging buffer has been read
    }
    const void *src = ids + id_offsets[lo];
    if (cnt && !pinned_in) {
      parallel_memcpy(h_stage[k].p, src, cnt * sizeof(int32_t));
      src = h_stage[k].p;
    }
    if (cnt) CUDA_TRY(cudaMemcpyAsync(p_dec_ids[k].p, src, cnt * sizeof(int32_t), cudaMemcpyHostToDevice, s_h2d));
    CUDA_TRY(cudaMemcpyAsync(p_offsets[k].p, id_offsets + lo, (hi - lo + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, s_h2d));
    CUDA_TRY(cudaEventRecord(ev_in[k], s_h2d));
    return SPM_OK;
  };
  last_launches = 0;
  float main_ms = 0.f, all_ms = 0.f;  // decode kernels; scan + gather kernels
  unsigned long long text_base = 0;
  { const int rc = issue_h2d(0); if (rc) return rc; }
  for (size_t c = 0; c < C; ++c) {
    const int k = static_cast<int>(c & 1);
    const size_t lo = c * chunk, hi = std::min(n, lo + chunk);
    const uint32_t m = static_cast<uint32_t>(hi - lo);
    const uint64_t cnt = id_offsets[hi] - id_offsets[lo];
    CUDA_TRY(cudaStreamWaitEvent(st, ev_in[k], 0));
    if (c >= 2) CUDA_TRY(cudaStreamWaitEvent(st, ev_d2h[k], 0));  // the slot's previous text has left the GPU
    unsigned long long tmp_cap = cnt * 6 + 16ull * m + (1u << 20);
    unsigned long long tot = 0;
    bool staged_next = false;
    for (int attempt = 0; attempt < 3; ++attempt) {
      CUDA_TRY(d_dec_tmp.ensure(tmp_cap));
      CUDA_TRY(cudaMemsetAsync(d_ctrl32.p, 0, 16 * sizeof(uint32_t), st));
      CUDA_TRY(cudaMemsetAsync(d_ctrl64.p, 0, 8 * sizeof(unsigned long long), st));
      CUDA_TRY(cudaEventRecord(ev[0], st));
      const int grid = static_cast<int>(std::min<size_t>(static_cast<size_t>(sm_count) * 8, (m + 7) / 8));
      KDecode D = decode_args(p_dec_ids[k].p - id_offsets[lo], p_offsets[k].p, m, tmp_cap);
      if (tok_end) {
        D.tok_end = p_dec_tok_end[k].p - id_offsets[lo];
        decode_warp_kernel<int32_t, false, true><<<grid, 256, 0, st>>>(D, {});
      } else {
        decode_warp_kernel<<<grid, 256, 0, st>>>(D, {});
      }
      CUDA_TRY(cudaGetLastError());
      CUDA_TRY(cudaEventRecord(ev[1], st));
      ++last_launches;
      SPM_TRY(copy_status(st, 16, 8));
      // the next chunk's ids are staged / queued while this chunk's kernel runs
      if (!staged_next && c + 1 < C) { const int rc = issue_h2d(c + 1); if (rc) { cudaDeviceSynchronize(); return rc; } }
      staged_next = true;
      CUDA_TRY(cudaStreamSynchronize(st));
      float a = 0.f;
      if (cudaEventElapsedTime(&a, ev[0], ev[1]) == cudaSuccess) main_ms += a;
      if (trace.on) fprintf(stderr, "[trace] decode chunk %zu: kernel done at %.3f ms (kernel %.3f ms, input %s)\n", c, trace.ms(), a,
                         pinned_in ? "pinned" : "pageable, staged");
      if (const int rc = decode_error()) { cudaDeviceSynchronize(); return rc; }
      tot = h_ctrl64.p[0];
      if (h_ctrl32.p[2]) { tmp_cap = tot + 1024; continue; }
      break;
    }
    if (h_ctrl32.p[2]) { cudaDeviceSynchronize(); set_error("Decode: temporary buffer overflow persisted"); return SPM_ERR_CAPACITY; }
    CUDA_TRY(p_dec_text[k].ensure(tot + 16));
    if (c > 0) {  // the previous chunk's scan + gather finished before this chunk's kernel did
      float g = 0.f;
      if (cudaEventElapsedTime(&g, ev[2], ev[3]) == cudaSuccess) all_ms += g;
    }
    CUDA_TRY(cudaEventRecord(ev[2], st));
    SPM_TRY(scan_total(d_sent_count.p, m, 0, d_ctrl64.p + 2, st));
    SPM_TRY(scan_gather<uint8_t>(d_sent_count.p, m, p_dec_toff[k].p, d_sent_start.p, d_dec_tmp.p, p_dec_text[k].p,
                                 p_dec_text[k].cap, 0, text_base, st));
    CUDA_TRY(cudaEventRecord(ev[3], st));
    CUDA_TRY(cudaEventRecord(ev_out[k], st));
    SPM_TRY(grow_pinned(h_dec_text, text_base, tot, hi, n));
    CUDA_TRY(cudaStreamWaitEvent(s_d2h, ev_out[k], 0));
    if (tot) CUDA_TRY(cudaMemcpyAsync(h_dec_text.p + text_base, p_dec_text[k].p, tot, cudaMemcpyDeviceToHost, s_d2h));
    CUDA_TRY(cudaMemcpyAsync(h_dec_text_offsets.p + lo, p_dec_toff[k].p, (m + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, s_d2h));
    if (tok_end && cnt)
      CUDA_TRY(cudaMemcpyAsync(h_dec_tok_end.p + (id_offsets[lo] - id_offsets[0]), p_dec_tok_end[k].p, cnt * sizeof(uint32_t),
                               cudaMemcpyDeviceToHost, s_d2h));
    CUDA_TRY(cudaEventRecord(ev_d2h[k], s_d2h));
    text_base += tot;
  }
  CUDA_TRY(cudaStreamSynchronize(s_d2h));
  if (trace.on) fprintf(stderr, "[trace] decode: text on host at %.3f ms (%zu chunks)\n", trace.ms(), C);
  {
    float g = 0.f;
    if (cudaEventElapsedTime(&g, ev[2], ev[3]) == cudaSuccess) all_ms += g;
  }
  h_dec_text.p[text_base] = 0;
  last_main_ms = main_ms;
  last_ms = main_ms + all_ms;
  last_h2d = total_ids * sizeof(int32_t) + (n + C) * sizeof(uint64_t);
  last_d2h = text_base + (n + C) * sizeof(uint64_t) + (tok_end ? total_ids * sizeof(uint32_t) : 0);
  *text = h_dec_text.p;
  *text_offsets = h_dec_text_offsets.p;
  if (tok_end) *tok_end = h_dec_tok_end.p;
  return SPM_OK;
}

// The deferred list of a lattice / n-best lane kernel (n_def {sentence, normalized length or 0} pairs in d_deferred) as
// long-sentence jobs: the slab holds the exact normalized length when the lane kernel measured it, else the bound from
// the input length (offs: the launch's host offsets).
int spm_engine::read_deferred(uint32_t n_def, const uint64_t *offs, std::vector<LongJob> *jobs) {
  cudaStream_t st = stream;
  CUDA_TRY(h_deferred.ensure(2 * static_cast<size_t>(n_def)));
  CUDA_TRY(cudaMemcpyAsync(h_deferred.p, d_deferred.p, 2ull * n_def * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  jobs->clear();
  for (uint32_t k = 0; k < n_def; ++k) {
    const uint32_t s = h_deferred.p[2 * k];
    uint64_t need = h_deferred.p[2 * k + 1];
    if (need == 0) need = ((offs[s + 1] - offs[s]) * max_expand_num + max_expand_den - 1) / max_expand_den + 8;
    if (need > 0x7FFFFF00ull) { set_error("sentence too long for the device path"); return SPM_ERR_UNSUPPORTED; }
    jobs->push_back(LongJob{s, static_cast<uint32_t>(need + 8), 0u});
  }
  return SPM_OK;
}

// ---- n-best (K5): lattice + A* per sentence on the GPU; leaves candidates in the temporary buffers ----
int spm_engine::run_nbest(const char *bytes, const uint64_t *offsets, size_t n, uint32_t nbest, uint64_t *tmp_total,
                          bool ends, bool norm) {
  cudaStream_t st = stream;
  const uint64_t base = offsets[0];
  const uint64_t total_bytes = offsets[n] - base;
  CUDA_TRY(d_bytes.ensure(total_bytes + 64));
  CUDA_TRY(d_offsets.ensure(n + 1));
  if (total_bytes) CUDA_TRY(cudaMemcpyAsync(d_bytes.p, bytes + base, total_bytes, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(d_offsets.p, offsets, (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
  last_h2d = total_bytes + (n + 1) * sizeof(uint64_t);
  NbestGeom G{};
  G.cap = lane_cap;
  G.node_cap = std::min<uint32_t>(65535u, 4 * lane_cap + 64);
  G.hyp_cap = 6144 + nbest * 64;   // typical need: ~60 hypotheses per result; retried with 8x on overflow
  G.heap_cap = 10000 + 1024 + 512;  // even: keeps the child pairs of the agenda 16-byte aligned
  // 32 warps per SM (64 registers per lane): the search is bound by L2 / HBM transactions on the per-lane agendas, so
  // more resident warps hide more of their latency
  const size_t groups = std::max<size_t>(1, (n + 31) / 32);   // one group of 32 sentences per warp pass
  int ctas = static_cast<int>(std::min<size_t>(sm_count, groups));
  int warps_per_cta = static_cast<int>(std::min<size_t>(32, (groups + ctas - 1) / ctas));
  size_t warps_total = static_cast<size_t>(ctas) * warps_per_cta;
  CUDA_TRY(ensure_lane_slabs(warps_total, lane_cap));
  CUDA_TRY(d_nb_scratch.ensure(warps_total * 32 * nbest_lane_bytes(G) + 256));
  CUDA_TRY(d_deferred.ensure(2 * n + 2));
  const size_t nc = n * static_cast<size_t>(nbest);
  CUDA_TRY(d_cand_start.ensure(nc));
  CUDA_TRY(d_cand_count.ensure(nc));
  CUDA_TRY(d_cand_score.ensure(nc));
  CUDA_TRY(d_n_cands.ensure(n));
  // candidates: at most one id per normalized byte each; start from 2 ids per input byte per 8 candidates
  unsigned long long tmp_cap = std::max<unsigned long long>(1u << 20, total_bytes * nbest / 3 + 64ull * n);
  // exported normalized texts: at most the bound of the whole batch's normalized length (as run_lattice's pos_cap)
  unsigned long long norm_cap = (total_bytes * max_expand_num) / max_expand_den + 16ull * n + 1024;
  if (norm) CUDA_TRY(d_nb_norm_start.ensure(n));
  for (int attempt = 0; attempt < 4; ++attempt) {
    CUDA_TRY(d_tmp_ids.ensure(tmp_cap));
    if (ends) CUDA_TRY(d_nb_end.ensure(tmp_cap));
    if (norm) CUDA_TRY(d_nb_norm.ensure(norm_cap));
    CUDA_TRY(cudaMemsetAsync(d_ctrl32.p, 0, 16 * sizeof(uint32_t), st));
    CUDA_TRY(cudaMemsetAsync(d_ctrl64.p, 0, 4 * sizeof(unsigned long long), st));
    KBatch B{};
    B.bytes = d_bytes.p - base;
    B.offsets = d_offsets.p;
    B.n = static_cast<uint32_t>(n);
    B.off_lo = 0;
    B.off_hi = ~0ull;
    B.work_counter = d_ctrl32.p + 4;
    B.status = d_ctrl32.p;
    B.deferred = d_deferred.p;
    NbestOut O{};
    O.tmp_ids = d_tmp_ids.p;
    O.tmp_cap = tmp_cap;
    O.cursor = d_ctrl64.p;
    O.cand_start = d_cand_start.p;
    O.cand_count = d_cand_count.p;
    O.cand_score = d_cand_score.p;
    O.n_cands = d_n_cands.p;
    O.status = d_ctrl32.p;
    if (ends) O.tmp_end = d_nb_end.p;
    if (norm) {
      O.norm = d_nb_norm.p;
      O.norm_cap = norm_cap;
      O.norm_cursor = d_ctrl64.p + 1;
      O.norm_start = d_nb_norm_start.p;
    }
    CUDA_TRY(cudaEventRecord(ev[0], st));
    { const int rc = build_order(d_offsets.p, n, st, &B.order, 0); if (rc) return rc; }
    nbest_lane_kernel<kNbestTop, 1024><<<ctas, warps_per_cta * 32, nbest_smem_bytes<kNbestTop>(warps_per_cta), st>>>(
        km, B, O, d_lane_slabs.p, d_nb_scratch.p, G, nbest);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaEventRecord(ev[1], st));
    ++last_launches;
    SPM_TRY(read_status(st, 16, 4));
    last_deferred = h_ctrl32.p[0];
    if (h_ctrl32.p[0] && !h_ctrl32.p[1]) {
      // ---- sentences the lane kernel deferred (long, large lattice, pool or agenda full): warp per sentence ----
      std::vector<LongJob> jobs;
      { const int rc = read_deferred(h_ctrl32.p[0], offsets, &jobs); if (rc) return rc; }
      const uint32_t mm1 = trie.max_matches_per_start + 1;
      for (LongJob &j : jobs) {
        if (nbest_long_nodes(j.cap, mm1) > 0xFFFFFF00ull) { set_error("sentence too long for the device path"); return SPM_ERR_UNSUPPORTED; }
        j.hyp_cap = static_cast<uint32_t>(std::min<unsigned long long>(4ull * j.cap + 16384ull + 64ull * nbest, 0xFFFFFF00ull));
      }
      const int rc = run_long_jobs(
          jobs, B, [&](const LongJob &j) { return nbest_long_bytes(j.cap, mm1, j.hyp_cap, G.heap_cap); },
          [&](const KBatch &LB, uint32_t m) {
            const int lgrid = static_cast<int>(std::min<uint32_t>((m + 7) / 8, static_cast<uint32_t>(sm_count) * 4));
            nbest_long_kernel<<<lgrid, 256, 0, st>>>(km, LB, O, d_long_hyp.p, d_long_need.p, mm1, G.heap_cap, nbest);
          });
      if (rc) return rc;
    }
    if (h_ctrl32.p[1] & 8u) { set_error("n-best: a long sentence normalized to more bytes than the scratch sized for it"); return SPM_ERR_ENCODE; }
    if (h_ctrl32.p[1] & 16u) { set_error("n-best: a lattice exceeds the sizes the model's trie implies"); return SPM_ERR_ENCODE; }
    if (h_ctrl32.p[1]) { set_error("n-best: internal consistency check failed"); return SPM_ERR_ENCODE; }
    if (h_ctrl32.p[2]) {
      if (h_ctrl32.p[2] & 1u) tmp_cap = h_ctrl64.p[0] + 1024;
      if (h_ctrl32.p[2] & 2u) norm_cap = h_ctrl64.p[1] + 1024;
      continue;
    }
    *tmp_total = h_ctrl64.p[0];
    return SPM_OK;
  }
  set_error("n-best: temporary buffer overflow persisted");
  return SPM_ERR_CAPACITY;
}

// ---- SampleEncode with nbest_size > 1 (sentencepiece_processor.cc:703-718): n-best, then one draw per sentence ----
int spm_engine::sample_picks(const char *bytes, const uint64_t *offsets, size_t n, uint32_t K, float alpha, bool ends,
                             bool norm, uint64_t *d2h) {
  cudaStream_t st = stream;
  uint64_t tmp_total = 0;
  SPM_TRY(run_nbest(bytes, offsets, n, K, &tmp_total, ends, norm));
  const size_t nc = n * static_cast<size_t>(K);
  CUDA_TRY(h_cand_score.ensure(nc + 1));
  CUDA_TRY(h_n_cands.ensure(n + 1));
  CUDA_TRY(h_picks.ensure(n + 1));
  CUDA_TRY(cudaMemcpyAsync(h_cand_score.p, d_cand_score.p, nc * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(h_n_cands.p, d_n_cands.p, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  // ---- the draw (sentencepiece_processor.cc:703-718) ----
  // The uniform of sentence i is generate_canonical<double,53>(mt) exactly as
  // std::discrete_distribution::operator() takes it; a sentence with fewer than two candidates
  // draws nothing.  Generated in sentence order on one generator, then the (independent)
  // log-sum-exp / cumulative tables are evaluated by all host threads.
  std::vector<double> u(n, 0.0);
  for (size_t i = 0; i < n; ++i)
    if (h_n_cands.p[i] >= 2) u[i] = std::generate_canonical<double, std::numeric_limits<double>::digits>(rng);
  const float *sc = h_cand_score.p;
  const uint32_t *kc = h_n_cands.p;
  uint32_t *picks = h_picks.p;
  auto work = [&](size_t lo, size_t hi) {
    std::vector<double> lp(K), cp(K);
    for (size_t i = lo; i < hi; ++i) {
      const uint32_t k = kc[i];
      if (k < 2) { picks[i] = 0; continue; }
      const float *s = sc + i * K;
      for (uint32_t c = 0; c < k; ++c) lp[c] = alpha * s[c];  // float product, widened (:705-706)
      double Z = lp[0];                                       // log_domain::LogSum, util.cc:278-294
      for (uint32_t c = 1; c < k; ++c) {
        double xa = Z, xb = lp[c];
        if (xa > xb) std::swap(xa, xb);
        Z = xb + std::log1p(std::exp(xa - xb));
      }
      double sum = 0.0;
      for (uint32_t c = 0; c < k; ++c) { lp[c] = std::exp(lp[c] - Z); sum += lp[c]; }
      double run = 0.0;  // discrete_distribution::param_type::_M_initialize
      for (uint32_t c = 0; c < k; ++c) { run += lp[c] / sum; cp[c] = run; }
      cp[k - 1] = 1.0;
      picks[i] = static_cast<uint32_t>(std::lower_bound(cp.begin(), cp.begin() + k, u[i]) - cp.begin());
    }
  };
  {
    const size_t T = std::max<size_t>(1, std::min<size_t>(std::thread::hardware_concurrency(), n / 2048 + 1));
    std::vector<std::thread> th;
    const size_t per = (n + T - 1) / T;
    for (size_t t = 1; t < T; ++t) th.emplace_back(work, std::min(n, t * per), std::min(n, (t + 1) * per));
    work(0, std::min(n, per));
    for (auto &t : th) t.join();
  }
  // ---- gather the picked candidates into sentence order ----
  CUDA_TRY(d_picks.ensure(n));
  CUDA_TRY(d_sent_start.ensure(n));
  CUDA_TRY(d_sent_count.ensure(n));
  CUDA_TRY(cudaMemcpyAsync(d_picks.p, picks, n * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  const uint32_t n32 = static_cast<uint32_t>(n);
  pick_candidates_kernel<<<(n32 + 255) / 256, 256, 0, st>>>(d_picks.p, n32, K, d_cand_start.p, d_cand_count.p,
                                                           d_sent_start.p, d_sent_count.p);
  CUDA_TRY(cudaGetLastError());
  ++last_launches;
  *d2h = nc * 4 + n * 4;
  return SPM_OK;
}

// ---- full-lattice operations (SURVEY 8f item 1): lattice + forward algorithm on the GPU (lattice_kernel.cuh), in
//      chunks of sentences; mode 0 then draws on the host exactly as Lattice::Sample (unigram_model.cc:511-542) does
//      -- std::exp in double, std::discrete_distribution<int> over float probabilities, this engine's std::mt19937 --
//      for the sentences in order, which reproduces the reference's single-threaded stream under a seed ----
int spm_engine::run_lattice(const char *bytes, const uint64_t *offsets, size_t n, float inv_theta, int mode, int samples,
                            bool frame_empty, const LatPieces *pc) {
  cudaStream_t st = stream;
  lat_ids.clear();
  lat_scores.clear();
  lat_offsets.assign(1, 0);
  lat_text.clear();
  lat_piece_end.clear();
  lat_text_offsets.assign(1, 0);
  std::string unk_bytes;         // pieces: the normalized bytes of the draw's UNK nodes, in path order
  std::vector<uint32_t> unk_end;  // per body token: the end of its bytes in unk_bytes (known pieces add none)
  LatticeGeom G{};
  G.cap = lane_cap;
  G.node_cap = lane_cap * (trie.max_matches_per_start + 1) + 64;
  constexpr size_t kChunk = 32768;
  const int warps_per_cta = 8;
  const uint32_t mm1 = trie.max_matches_per_start + 1;
  uint64_t deferred = 0;
  CUDA_TRY(d_deferred.ensure(2 * std::min(n, kChunk) + 2));
  last_launches = 0;
  last_h2d = last_d2h = 0;
  float main_ms = 0.f;
  if (mode == 1) CUDA_TRY(h_lat_entropy.ensure(n + 1));
  std::vector<float> probs;
  std::vector<uint32_t> path;
  for (size_t lo = 0; lo < n; lo += kChunk) {
    const size_t m = std::min(kChunk, n - lo);
    const uint64_t base = offsets[lo];
    const uint64_t chunk_bytes = offsets[lo + m] - base;
    CUDA_TRY(d_bytes.ensure(chunk_bytes + 64));
    CUDA_TRY(d_offsets.ensure(m + 1));
    if (chunk_bytes) CUDA_TRY(cudaMemcpyAsync(d_bytes.p, bytes + base, chunk_bytes, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(d_offsets.p, offsets + lo, (m + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
    last_h2d += chunk_bytes + (m + 1) * sizeof(uint64_t);
    const size_t groups = (m + 31) / 32;
    const int ctas = static_cast<int>(std::min<size_t>(sm_count, (groups + warps_per_cta - 1) / warps_per_cta));
    const size_t warps_total = static_cast<size_t>(ctas) * warps_per_cta;
    CUDA_TRY(ensure_lane_slabs(warps_total, G.cap));
    CUDA_TRY(d_lat_scratch.ensure(warps_total * 32 * lattice_lane_bytes(G) + 256));
    CUDA_TRY(d_lat_node_start.ensure(m));
    CUDA_TRY(d_lat_pos_start.ensure(m));
    CUDA_TRY(d_lat_nchars.ensure(m));
    CUDA_TRY(d_lat_entropy.ensure(m));
    // a sentence of b normalized bytes has at most b + 2 position records; nodes: start from 3 per input byte
    unsigned long long node_cap = mode == 0 ? 3ull * chunk_bytes + 64ull * m + 1024 : 1;
    const unsigned long long pos_cap = mode == 0 ? (chunk_bytes * max_expand_num) / max_expand_den + 16ull * m + 1024 : 1;
    for (int attempt = 0;; ++attempt) {
      CUDA_TRY(d_lat_nodes.ensure(node_cap));
      CUDA_TRY(d_lat_pos.ensure(pos_cap));
      CUDA_TRY(cudaMemsetAsync(d_ctrl32.p, 0, 16 * sizeof(uint32_t), st));
      CUDA_TRY(cudaMemsetAsync(d_ctrl64.p, 0, 4 * sizeof(unsigned long long), st));
      KBatch B{};
      B.bytes = d_bytes.p - base;
      B.offsets = d_offsets.p;
      B.n = static_cast<uint32_t>(m);
      B.off_lo = 0;
      B.off_hi = ~0ull;
      B.work_counter = d_ctrl32.p + 4;
      B.status = d_ctrl32.p;
      B.deferred = d_deferred.p;
      LatticeOut O{};
      O.nodes = d_lat_nodes.p;
      O.pos = d_lat_pos.p;
      O.node_cap = node_cap;
      O.pos_cap = pos_cap;
      O.cursor = d_ctrl64.p;
      O.node_start = d_lat_node_start.p;
      O.pos_start = d_lat_pos_start.p;
      O.n_chars = d_lat_nchars.p;
      O.entropy = d_lat_entropy.p;
      O.status = d_ctrl32.p;
      CUDA_TRY(cudaEventRecord(ev[0], st));
      lattice_lane_kernel<<<ctas, warps_per_cta * 32, kLaneTableBytes, st>>>(km, B, O, d_lane_slabs.p, d_lat_scratch.p, G,
                                                                            inv_theta, mode);
      CUDA_TRY(cudaGetLastError());
      CUDA_TRY(cudaEventRecord(ev[1], st));
      ++last_launches;
      SPM_TRY(read_status(st, 16, 4));
      float a = 0.f;
      if (cudaEventElapsedTime(&a, ev[0], ev[1]) == cudaSuccess) main_ms += a;
      const uint32_t n_def = h_ctrl32.p[0];
      if (n_def && !h_ctrl32.p[1]) {
        // ---- sentences the lane kernel deferred (long, large lattice): warp per sentence ----
        std::vector<LongJob> jobs;
        { const int rc = read_deferred(n_def, offsets + lo, &jobs); if (rc) return rc; }
        const int rc = run_long_jobs(
            jobs, B, [&](const LongJob &j) { return lattice_long_bytes(j.cap, mm1); },
            [&](const KBatch &LB, uint32_t nj) {
              const int lgrid = static_cast<int>(std::min<uint32_t>((nj + 7) / 8, static_cast<uint32_t>(sm_count) * 4));
              lattice_long_kernel<<<lgrid, 256, 0, st>>>(km, LB, O, mm1, inv_theta, mode);
            });
        if (rc) return rc;
      }
      if (h_ctrl32.p[1] & 8u) { set_error("lattice: a long sentence normalized to more bytes than the scratch sized for it"); return SPM_ERR_ENCODE; }
      if (h_ctrl32.p[1]) { set_error("lattice: a lattice exceeds the sizes the model's trie implies"); return SPM_ERR_ENCODE; }
      if (h_ctrl32.p[2] && attempt == 0) { node_cap = h_ctrl64.p[0] + 1024; continue; }
      deferred += n_def;
      if (h_ctrl32.p[2]) { set_error("lattice: output buffer overflow persisted"); return SPM_ERR_CAPACITY; }
      break;
    }
    if (mode == 1) {
      CUDA_TRY(cudaMemcpyAsync(h_lat_entropy.p + lo, d_lat_entropy.p, m * sizeof(float), cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaStreamSynchronize(st));
      last_d2h += m * sizeof(float);
      continue;
    }
    const unsigned long long tot_nodes = h_ctrl64.p[0], tot_pos = h_ctrl64.p[1];
    CUDA_TRY(h_lat_nodes.ensure(tot_nodes + 1));
    CUDA_TRY(h_lat_pos.ensure(tot_pos + 1));
    CUDA_TRY(h_lat_node_start.ensure(m));
    CUDA_TRY(h_lat_pos_start.ensure(m));
    CUDA_TRY(h_lat_nchars.ensure(m));
    if (tot_nodes) CUDA_TRY(cudaMemcpyAsync(h_lat_nodes.p, d_lat_nodes.p, tot_nodes * sizeof(uint4), cudaMemcpyDeviceToHost, st));
    if (tot_pos) CUDA_TRY(cudaMemcpyAsync(h_lat_pos.p, d_lat_pos.p, tot_pos * sizeof(uint2), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(h_lat_node_start.p, d_lat_node_start.p, m * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(h_lat_pos_start.p, d_lat_pos_start.p, m * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(h_lat_nchars.p, d_lat_nchars.p, m * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    last_d2h += tot_nodes * sizeof(uint4) + tot_pos * sizeof(uint2) + m * 20;
    // ---- Lattice::Sample per sentence, in order, on one generator ----
    const bool bf = model.byte_fallback;
    for (size_t i = 0; i < m; ++i) {
      const uint32_t L = h_lat_nchars.p[i];
      const uint4 *nodes = h_lat_nodes.p + h_lat_node_start.p[i];
      const uint2 *pos = h_lat_pos.p + h_lat_pos_start.p[i];
      const bool frame_it = framed() && (L || frame_empty);
      for (int sidx = 0; sidx < samples; ++sidx) {
        float score = 0.f;
        if (frame_it) lat_ids.insert(lat_ids.end(), frame_ids.begin(), frame_ids.begin() + frame_np);
        const size_t body = lat_ids.size();
        if (L) {
          auto A = [&](uint32_t p) { float f; memcpy(&f, &pos[p].x, 4); return f; };
          path.clear();
          float Z = A(L);
          uint32_t p = L;
          while (p != 0) {  // at position 0 the only candidate is BOS: no draw (a one-weight distribution)
            const uint32_t q0 = pos[p].y, q1 = pos[p + 1].y;
            probs.clear();
            for (uint32_t q = q0; q < q1; ++q) {
              float sc; memcpy(&sc, &nodes[q].y, 4);
              const float arg = A(nodes[q].z) + inv_theta * sc - Z;   // float expression (:528-529)
              probs.push_back(static_cast<float>(std::exp(static_cast<double>(arg))));
            }
            std::discrete_distribution<int> dist(probs.begin(), probs.end());
            const uint32_t q = q0 + static_cast<uint32_t>(dist(rng));
            path.push_back(q);
            p = nodes[q].z;
            Z = A(p);
          }
          // id path of PopulateSentencePieceText over the sampled nodes, left to right; with pc, also where the
          // surface of each unknown token lies in unk_bytes (a merged run: its nodes' characters in order)
          bool prev_unk = false;
          unk_bytes.clear();
          unk_end.clear();
          for (size_t k = path.size(); k-- > 0;) {
            const uint4 nd = nodes[path[k]];
            float sc; memcpy(&sc, &nd.y, 4);
            score += inv_theta * sc;   // (:846-847)
            const int32_t id = static_cast<int32_t>(nd.x);
            const bool isunk = id == unk_id;
            // an UNK node covers one character of the normalized text, whose bytes it carries; its byte count is the
            // span of the character (a truncated character at the end of the text has fewer bytes: the bytes above
            // it are zero and a zero byte never follows a multi-byte lead in normalized text)
            auto for_char_bytes = [&](auto &&f) {
              static const uint8_t kLen[16] = {1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 3, 4};
              const uint32_t cl = kLen[(nd.w & 0xFFu) >> 4];
              for (uint32_t bq = 0; bq < cl; ++bq) {
                const uint32_t bv = (nd.w >> (8 * bq)) & 0xFFu;
                if (bq > 0 && bv == 0) break;
                f(bv);
              }
            };
            if (isunk && bf) {
              for_char_bytes([&](uint32_t bv) { lat_ids.push_back(byte_to_id_host[bv]); });
            } else {
              if (!(isunk && prev_unk)) {
                lat_ids.push_back(id);
                if (pc) unk_end.push_back(static_cast<uint32_t>(unk_bytes.size()));
              }
              if (pc && isunk) {
                for_char_bytes([&](uint32_t bv) { unk_bytes.push_back(static_cast<char>(bv)); });
                unk_end.back() = static_cast<uint32_t>(unk_bytes.size());
              }
            }
            prev_unk = isunk;
          }
          score -= A(L);  // - marginal (:853)
        }
        const size_t nbody = lat_ids.size() - body;
        if (frame_it) {  // the score stays the raw path's, as in the reference
          if (frame_rev) std::reverse(lat_ids.begin() + body, lat_ids.end());
          lat_ids.insert(lat_ids.end(), frame_ids.begin() + frame_np, frame_ids.end());
        }
        if (pc) {  // the pieces of the framed list, as K9 (pieces_kernel.cuh) writes them
          const size_t first = lat_offsets.back(), T = lat_ids.size() - first;
          const size_t t0 = lat_text.size();
          for (size_t t = 0; t < T; ++t) {
            const int32_t id = lat_ids[first + t];
            const size_t q = first + t - body;  // position in the body, in its final order
            const char *src;
            size_t len;
            if (id == unk_id && pc->unk_piece) {
              src = pc->unk_piece;
              len = pc->unk_len;
            } else if (id == unk_id && !bf && first + t >= body && q < nbody) {
              const size_t r = frame_it && frame_rev ? nbody - 1 - q : q;  // in path order
              const uint32_t b = r ? unk_end[r - 1] : 0u;
              src = unk_bytes.data() + b;
              len = unk_end[r] - b;
            } else {
              src = model.piece(id);
              len = model.piece_len(id);
            }
            lat_text.insert(lat_text.end(), src, src + len);
            lat_piece_end.push_back(static_cast<uint32_t>(lat_text.size() - t0));
            if (pc->sep >= 0 && t + 1 < T) lat_text.push_back(static_cast<char>(pc->sep));
          }
          lat_text_offsets.push_back(lat_text.size());
        }
        lat_offsets.push_back(lat_ids.size());
        lat_scores.push_back(score);
      }
    }
  }
  last_main_ms = main_ms;
  last_ms = main_ms;
  last_deferred = deferred;
  return SPM_OK;
}

// ---------------------------------------------------------------- C ABI ----

extern "C" {

const char *spm_last_error(const spm_engine *e) {
  if (e) return e->err.c_str();
  return g_create_error.c_str();
}

static int create_common(spm_engine *e, int device, spm_engine **out) {
  auto fail = [&](int code, const std::string &msg) {
    std::lock_guard<std::mutex> lk(g_create_mu);
    g_create_error = msg;
    delete e;
    return code;
  };
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(SPM_ERR_CUDA, "no CUDA device available: this engine has no CPU fallback");
  if (device < 0 || device >= ndev) return fail(SPM_ERR_ARG, "invalid device ordinal");
  e->device = device;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(SPM_ERR_CUDA, "cudaGetDeviceProperties failed");
  // sm_90a code runs on compute capability 9.0 only: the 'a' features do not carry over to later architectures.
  if (prop.major != 9 || prop.minor != 0)
    return fail(SPM_ERR_CUDA, "this build targets sm_90a (H100); found compute capability " + std::to_string(prop.major) +
                                  "." + std::to_string(prop.minor));
  e->sm_count = prop.multiProcessorCount;
  if (const char *v = getenv("SPM_B200_SORT")) e->sort_by_length = atoi(v) != 0;
  if (const char *v = getenv("SPM_B200_FUSED")) e->fused_host_path = atoi(v) != 0;
  if (const char *v = getenv("SPM_B200_FASTWORDS")) e->force_fast_words = atoi(v) != 0 ? 1 : 0;
  if (const char *v = getenv("SPM_B200_KSTATS")) e->kstats = atoi(v) != 0;
  if (const char *v = getenv("SPM_B200_BPE_CACHE")) e->bpe_cache_log2 = std::min(24, std::max(0, atoi(v)));
  e->smem_optin = prop.sharedMemPerBlockOptin;
  if (cudaSetDevice(device) != cudaSuccess) return fail(SPM_ERR_CUDA, "cudaSetDevice failed");
  int rc = e->build_tables();
  if (rc) return fail(rc, e->err);
  if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) return fail(SPM_ERR_CUDA, "stream creation failed");
  for (auto &ev : e->ev)
    if (cudaEventCreate(&ev) != cudaSuccess) return fail(SPM_ERR_CUDA, "event creation failed");
  const size_t w = spm_engine::kCtrlWords;
  if (e->d_ctrl32.ensure(w) != cudaSuccess || e->d_ctrl64.ensure(w) != cudaSuccess || e->h_ctrl32.ensure(w) != cudaSuccess ||
      e->h_ctrl64.ensure(w) != cudaSuccess)
    return fail(SPM_ERR_CUDA, "status word allocation failed");
  rc = e->configure_kernel_attrs();
  if (rc) return fail(rc, e->err);
  *out = e;
  return SPM_OK;
}

int spm_engine_create(const spm_model_desc *d, int device, spm_engine **out) {
  if (!d || !out || d->vocab_size <= 0 || !d->piece_bytes || !d->piece_off || !d->scores || !d->types) {
    std::lock_guard<std::mutex> lk(g_create_mu);
    g_create_error = "spm_engine_create: null or empty model description";
    return SPM_ERR_ARG;
  }
  spm_engine *e = new spm_engine();
  ModelData &m = e->model;
  m.model_type = d->model_type;
  m.piece_off.assign(d->piece_off, d->piece_off + d->vocab_size + 1);
  m.piece_bytes.assign(d->piece_bytes, d->piece_off[d->vocab_size]);
  m.scores.assign(d->scores, d->scores + d->vocab_size);
  m.types.assign(d->types, d->types + d->vocab_size);
  m.byte_fallback = d->byte_fallback;
  m.treat_whitespace_as_suffix = d->treat_whitespace_as_suffix;
  m.add_dummy_prefix = d->add_dummy_prefix;
  m.remove_extra_whitespaces = d->remove_extra_whitespaces;
  m.escape_whitespaces = d->escape_whitespaces;
  if (d->charsmap && d->charsmap_bytes) m.charsmap.assign(static_cast<const char *>(d->charsmap), d->charsmap_bytes);
  return create_common(e, device, out);
}

int spm_engine_create_from_serialized(const void *model_proto, size_t len, int device, spm_engine **out) {
  if (!model_proto || !len || !out) {
    std::lock_guard<std::mutex> lk(g_create_mu);
    g_create_error = "spm_engine_create_from_serialized: null argument";
    return SPM_ERR_ARG;
  }
  spm_engine *e = new spm_engine();
  std::string err;
  if (!ParseModelProto(model_proto, len, &e->model, &err)) {
    std::lock_guard<std::mutex> lk(g_create_mu);
    g_create_error = err;
    delete e;
    return SPM_ERR_MODEL;
  }
  return create_common(e, device, out);
}

void spm_engine_destroy(spm_engine *e) { delete e; }

int spm_engine_set_types(spm_engine *e, const uint8_t *types) {
  if (!e || !types) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  // the kinds CONTROL/UNKNOWN/BYTE never change (sentencepiece_processor.cc:311-316)
  for (int i = 0; i < e->model.vocab_size(); ++i) {
    const uint8_t o = e->model.types[i], t = types[i];
    const bool on = o == SPM_NORMAL || o == SPM_USER_DEFINED || o == SPM_UNUSED;
    const bool tn = t == SPM_NORMAL || t == SPM_USER_DEFINED || t == SPM_UNUSED;
    if (on != tn || (!on && o != t)) { e->set_error("spm_engine_set_types: piece class changes are not allowed"); return SPM_ERR_ARG; }
  }
  e->model.types.assign(types, types + e->model.vocab_size());
  return e->upload_types();
}

int spm_engine_cache_reset(spm_engine *e) {
  if (!e) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (e->km.bpe_cache_mask) {
    // (the engine's streams do not synchronize with the legacy stream: the fill runs on the engine's own stream and is
    // complete when the call returns, whatever stream the next batch uses)
    if (cudaSetDevice(e->device) != cudaSuccess ||
        cudaMemsetAsync(e->d_bpe_cache.p, 0, (static_cast<size_t>(e->km.bpe_cache_mask) + 1) * 64, e->stream) != cudaSuccess ||
        cudaStreamSynchronize(e->stream) != cudaSuccess) {
      e->set_error("spm_engine_cache_reset: cudaMemset failed");
      return SPM_ERR_CUDA;
    }
  }
  return SPM_OK;
}

static void finish_timing(spm_engine *e);

int spm_engine_set_encode_frame(spm_engine *e, const int32_t *prefix, uint32_t n_prefix, int reverse, const int32_t *suffix,
                                uint32_t n_suffix) {
  if (!e) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  if (n_prefix > spm_engine::kMaxFrame || n_suffix > spm_engine::kMaxFrame) {
    set_error("spm_engine_set_encode_frame: at most " + std::to_string(spm_engine::kMaxFrame) + " ids before and " +
              std::to_string(spm_engine::kMaxFrame) + " after a sentence");
    return SPM_ERR_ARG;
  }
  if ((n_prefix && !prefix) || (n_suffix && !suffix)) { set_error("spm_engine_set_encode_frame: null ids"); return SPM_ERR_ARG; }
  std::vector<int32_t> ids;
  if (n_prefix) ids.assign(prefix, prefix + n_prefix);
  if (n_suffix) ids.insert(ids.end(), suffix, suffix + n_suffix);
  const int32_t V = e->model.vocab_size();
  for (const int32_t id : ids)
    if (id < 0 || id >= V) {
      set_error("spm_engine_set_encode_frame: id " + std::to_string(id) + " is outside [0, " + std::to_string(V) + ")");
      return SPM_ERR_ARG;
    }
  CUDA_TRY(cudaSetDevice(e->device));
  CUDA_TRY(e->d_frame.ensure(ids.size() + 1));
  if (!ids.empty()) CUDA_TRY(cudaMemcpy(e->d_frame.p, ids.data(), ids.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
  e->frame_ids = std::move(ids);
  e->frame_np = n_prefix;
  e->frame_ns = n_suffix;
  e->frame_rev = reverse != 0;
  return SPM_OK;
}

int spm_engine_set_unk_surface(spm_engine *e, const char *surface, size_t bytes) {
  if (!e || (!surface && bytes)) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  e->model.unk_surface.assign(surface ? surface : "", bytes);
  e->dec_ready = false;
  return SPM_OK;
}

namespace {
// spm_decode_ids and spm_decode_offsets: tok_end == NULL decodes the text only
int decode_host(spm_engine *e, const int32_t *ids, const uint64_t *id_offsets, size_t n, const char **text,
                const uint64_t **text_offsets, const uint32_t **tok_end) {
  if (!e || !id_offsets || !text || !text_offsets) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  if (n >= 0xFFFFFFF0ull) { set_error("too many id lists in one call"); return SPM_ERR_ARG; }
  for (size_t i = 0; i < n; ++i)
    if (id_offsets[i + 1] < id_offsets[i]) { set_error("id_offsets must be non-decreasing"); return SPM_ERR_ARG; }
  const uint64_t base = id_offsets[0];
  const uint64_t total_ids = id_offsets[n] - base;
  if (total_ids && !ids) return SPM_ERR_ARG;
  if (!e->model.denormalizer_charsmap.empty()) {
    set_error("Decode: models with a denormalizer_spec are not on the device path");
    return SPM_ERR_UNSUPPORTED;
  }
  CUDA_TRY(cudaSetDevice(e->device));
  { const int rc = e->ensure_decode_tables(); if (rc) return rc; }
  if (n >= e->pipeline_min_sentences) return e->decode_host_pipelined(ids, id_offsets, n, text, text_offsets, tok_end);
  cudaStream_t st = e->stream;
  e->last_launches = 0;
  CUDA_TRY(e->h_dec_text_offsets.ensure(n + 1));
  if (n == 0) {
    CUDA_TRY(e->h_dec_text.ensure(1));
    e->h_dec_text_offsets.p[0] = 0;
    *text = e->h_dec_text.p;
    *text_offsets = e->h_dec_text_offsets.p;
    if (tok_end) {
      CUDA_TRY(e->h_dec_tok_end.ensure(1));
      *tok_end = e->h_dec_tok_end.p;
    }
    return SPM_OK;
  }
  CUDA_TRY(e->d_dec_ids.ensure(total_ids + 1));
  CUDA_TRY(e->d_offsets.ensure(n + 1));
  if (total_ids) CUDA_TRY(cudaMemcpyAsync(e->d_dec_ids.p, ids + base, total_ids * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(e->d_offsets.p, id_offsets, (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
  e->last_h2d = total_ids * sizeof(int32_t) + (n + 1) * sizeof(uint64_t);
  const uint32_t n32 = static_cast<uint32_t>(n);
  const int grid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (n + 7) / 8));
  if (tok_end) CUDA_TRY(e->d_dec_tok_end.ensure(total_ids + 1));
  SPM_TRY(e->decode_text(n32, total_ids * 6 + 16ull * n + (1u << 20), false, st,  // retried with the exact size on overflow
                         [&](unsigned long long tmp_cap) {
                           KDecode D = e->decode_args(e->d_dec_ids.p - base, e->d_offsets.p, n32, tmp_cap);
                           if (tok_end) {
                             D.tok_end = e->d_dec_tok_end.p - base;
                             decode_warp_kernel<int32_t, false, true><<<grid, 256, 0, st>>>(D, {});
                           } else {
                             decode_warp_kernel<<<grid, 256, 0, st>>>(D, {});
                           }
                         },
                         text, text_offsets, tok_end, total_ids));
  finish_timing(e);
  return SPM_OK;
}
}  // namespace

int spm_decode_ids(spm_engine *e, const int32_t *ids, const uint64_t *id_offsets, size_t n, const char **text,
                   const uint64_t **text_offsets) {
  return decode_host(e, ids, id_offsets, n, text, text_offsets, nullptr);
}

int spm_decode_offsets(spm_engine *e, const int32_t *ids, const uint64_t *id_offsets, size_t n, const char **text,
                       const uint64_t **text_offsets, const uint32_t **tok_end) {
  if (!tok_end) return SPM_ERR_ARG;
  return decode_host(e, ids, id_offsets, n, text, text_offsets, tok_end);
}

int spm_decode_ids_device(spm_engine *e, const void *d_ids, uint32_t id_bytes, uint64_t row_stride, size_t n,
                          uint32_t row_len, const int32_t *d_lengths, int64_t stop_id, const char **text,
                          const uint64_t **text_offsets, void *stream) {
  if (!e || !text || !text_offsets) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  if (id_bytes != 4 && id_bytes != 8) { e->set_error("id_bytes must be 4 or 8"); return SPM_ERR_ARG; }
  if (n && row_len && !d_ids) { e->set_error("null argument"); return SPM_ERR_ARG; }
  if (n >= 0xFFFFFFF0ull) { e->set_error("too many rows in one call"); return SPM_ERR_ARG; }
  if (!e->model.denormalizer_charsmap.empty()) {
    e->set_error("Decode: models with a denormalizer_spec are not on the device path");
    return SPM_ERR_UNSUPPORTED;
  }
  CUDA_TRY(cudaSetDevice(e->device));
  { const int rc = e->ensure_decode_tables(); if (rc) return rc; }
  cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : e->stream;
  e->last_launches = 0;
  e->last_h2d = e->last_d2h = 0;
  if (n == 0) {
    CUDA_TRY(e->h_dec_text.ensure(1));
    CUDA_TRY(e->h_dec_text_offsets.ensure(1));
    CUDA_TRY(cudaStreamSynchronize(st));
    e->h_dec_text_offsets.p[0] = 0;
    *text = e->h_dec_text.p;
    *text_offsets = e->h_dec_text_offsets.p;
    return SPM_OK;
  }
  const uint32_t n32 = static_cast<uint32_t>(n);
  CUDA_TRY(e->d_row_len.ensure(n));
  const int grid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (n + 7) / 8));
  const bool wide = id_bytes == 8;
  if (wide) decode_row_len_kernel<<<grid, 256, 0, st>>>(static_cast<const int64_t *>(d_ids), row_stride, n32, row_len,
                                                         d_lengths, stop_id, e->d_row_len.p);
  else decode_row_len_kernel<<<grid, 256, 0, st>>>(static_cast<const int32_t *>(d_ids), row_stride, n32, row_len,
                                                    d_lengths, stop_id, e->d_row_len.p);
  CUDA_TRY(cudaGetLastError());
  ++e->last_launches;
  // about 6 text bytes per id; the kernel reports the exact size when a batch needs more
  const unsigned long long guess = 6ull * n * std::min<uint32_t>(row_len, 256u) + 16ull * n + (1u << 20);
  SPM_TRY(e->decode_text(n32, guess, true, st,
                         [&](unsigned long long tmp_cap) {
                           KDecode D = e->decode_args(static_cast<const int32_t *>(d_ids), nullptr, n32, tmp_cap);
                           D.row_stride = row_stride;
                           D.row_len = e->d_row_len.p;
                           if (wide) decode_warp_kernel<int64_t, true><<<grid, 256, 0, st>>>(D, {});
                           else decode_warp_kernel<int32_t, true><<<grid, 256, 0, st>>>(D, {});
                         },
                         text, text_offsets));
  finish_timing(e);
  return SPM_OK;
}

static_assert(sizeof(spm_decode_stream_state) == 16 && sizeof(DecStreamState) == 16, "a stream state is 16 bytes");

int spm_decode_stream_device(spm_engine *e, const void *d_ids, uint32_t id_bytes, uint64_t row_stride, size_t n,
                             uint32_t row_len, const int32_t *d_lengths, int64_t stop_id, const int32_t *d_final,
                             spm_decode_stream_state *d_state, const char **text, const uint64_t **text_offsets,
                             void *stream) {
  if (!e || !text || !text_offsets) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  if (id_bytes != 4 && id_bytes != 8) { e->set_error("id_bytes must be 4 or 8"); return SPM_ERR_ARG; }
  if (n && ((row_len && !d_ids) || !d_state)) { e->set_error("null argument"); return SPM_ERR_ARG; }
  if (reinterpret_cast<uintptr_t>(d_state) % 16) { e->set_error("d_state must be 16-byte aligned"); return SPM_ERR_ARG; }
  if (n >= 0xFFFFFFF0ull) { e->set_error("too many rows in one call"); return SPM_ERR_ARG; }
  if (!e->model.denormalizer_charsmap.empty()) {
    e->set_error("Decode: models with a denormalizer_spec are not on the device path");
    return SPM_ERR_UNSUPPORTED;
  }
  CUDA_TRY(cudaSetDevice(e->device));
  { const int rc = e->ensure_decode_tables(); if (rc) return rc; }
  cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : e->stream;
  e->last_launches = 0;
  e->last_h2d = e->last_d2h = 0;
  if (n == 0) {
    CUDA_TRY(e->h_dec_text.ensure(1));
    CUDA_TRY(e->h_dec_text_offsets.ensure(1));
    CUDA_TRY(cudaStreamSynchronize(st));
    e->h_dec_text_offsets.p[0] = 0;
    *text = e->h_dec_text.p;
    *text_offsets = e->h_dec_text_offsets.p;
    return SPM_OK;
  }
  const uint32_t n32 = static_cast<uint32_t>(n);
  CUDA_TRY(e->d_dec_state.ensure(n));
  const int grid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (n + 7) / 8));
  const bool wide = id_bytes == 8;
  DecStreamState *in = reinterpret_cast<DecStreamState *>(d_state);
  // a row's text is at most (its ids + 3 held bytes) surfaces of at most dec_max_len bytes each, so the temporary
  // never overflows below 1 GiB; above that decode_text's retry sizes it exactly (the kernel only reads d_state)
  const unsigned long long bound = (static_cast<unsigned long long>(row_len) + 3ull) * e->dec_max_len * n + 16;
  SPM_TRY(e->decode_text(n32, std::min(bound, 1ull << 30), true, st,
                         [&](unsigned long long tmp_cap) {
                           KDecode D = e->decode_args(static_cast<const int32_t *>(d_ids), nullptr, n32, tmp_cap);
                           D.row_stride = row_stride;
                           const KDecodeStream S{in, e->d_dec_state.p, d_lengths, d_final, stop_id, row_len};
                           if (wide) decode_warp_kernel<int64_t, true, false, true><<<grid, 256, 0, st>>>(D, S);
                           else decode_warp_kernel<int32_t, true, false, true><<<grid, 256, 0, st>>>(D, S);
                         },
                         text, text_offsets, nullptr, 0, [&]() -> int {
                           CUDA_TRY(cudaMemcpyAsync(in, e->d_dec_state.p, n * sizeof(DecStreamState),
                                                    cudaMemcpyDeviceToDevice, st));
                           return SPM_OK;
                         }));
  finish_timing(e);
  return SPM_OK;
}

void *spm_host_alloc(size_t bytes) {
  void *p = nullptr;
  if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) return nullptr;
  return p;
}
void spm_host_free(void *p) { if (p) cudaFreeHost(p); }

int spm_engine_get_info(const spm_engine *e, spm_engine_info *info) {
  if (!e || !info) return SPM_ERR_ARG;
  memset(info, 0, sizeof *info);
  info->device = e->device;
  info->sm_count = e->sm_count;
  info->model_type = e->model.model_type;
  info->vocab_size = e->model.vocab_size();
  info->unk_id = e->unk_id;
  info->min_score = e->min_score;
  info->max_score = e->max_score;
  info->trie_units = e->km.trie_units;
  const uint32_t tile_bytes = e->model.model_type == SPM_BPE ? bpe_tile_bytes(e->ncap, false)
                                                              : tile_bytes_for(e->ncap, e->km.match_slots, false);
  const LaunchGeom g = plan_geometry(*e, tile_bytes, std::min(e->threads, 512) / 32);
  info->trie_hot_units = g.hot_link;
  info->charsmap_units = e->charsmap_units;
  info->last_kernel_launches = e->last_launches;
  info->last_kernel_ms = e->last_ms;
  info->last_main_kernel_ms = e->last_main_ms;
  info->last_h2d_bytes = e->last_h2d;
  info->last_d2h_bytes = e->last_d2h;
  info->last_deferred = e->last_deferred;
  info->last_unk_detour = e->last_unk_detour;
  return SPM_OK;
}

int spm_engine_set_tuning(spm_engine *e, int lanes, int cap, int ctas) {
  if (!e) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (lanes) {
    if (lanes != 1 && lanes != 32) { e->set_error("lanes_per_sentence must be 1 or 32"); return SPM_ERR_ARG; }
    e->G = lanes;
  }
  if (cap) {
    if (cap < 64 || cap > 8192) { e->set_error("smem_norm_cap out of range"); return SPM_ERR_ARG; }
    e->ncap = static_cast<uint32_t>(cap + 15) & ~15u;
  }
  if (ctas) {
    // encoded as threads per CTA when >= 32
    if (ctas >= 32) {
      if (ctas % 32 || ctas > 1024) { e->set_error("threads per CTA must be a multiple of 32, <= 1024"); return SPM_ERR_ARG; }
      e->threads = ctas;
    } else {
      e->ctas_per_sm = ctas;
    }
  }
  return SPM_OK;
}

static void finish_timing(spm_engine *e) {
  float a = 0.f, b = 0.f;
  if (cudaEventElapsedTime(&a, e->ev[0], e->ev[1]) == cudaSuccess) e->last_main_ms = a;
  if (cudaEventElapsedTime(&b, e->ev[0], e->ev[2]) == cudaSuccess) e->last_ms = b;
  else e->last_ms = e->last_main_ms;
  (void)cudaGetLastError();  // an unrecorded event must not leave a stale error behind
}

int spm_encode_ids_device(spm_engine *e, const char *d_bytes, const uint64_t *d_offsets, size_t n, uint64_t total_bytes,
                          int32_t *d_ids, uint64_t ids_capacity, uint64_t *d_id_offsets, uint64_t *total_ids,
                          void *stream) {
  if (!e) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  if (!d_offsets || !d_id_offsets || !total_ids || (n && !d_bytes && total_bytes)) { e->set_error("null argument"); return SPM_ERR_ARG; }
  if (n >= 0xFFFFFFF0ull) { e->set_error("too many sentences in one call"); return SPM_ERR_ARG; }
  CUDA_TRY(cudaSetDevice(e->device));
  cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : e->stream;
  *total_ids = 0;
  if (n == 0) {
    CUDA_TRY(cudaMemsetAsync(d_id_offsets, 0, sizeof(uint64_t), st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return SPM_OK;
  }
  e->last_h2d = e->last_d2h = 0;
  if (e->model.model_type == SPM_UNIGRAM) {
    const int rc0 = e->pick_fast_words_device(reinterpret_cast<const uint8_t *>(d_bytes), d_offsets, n, st, &e->batch_fast_words);
    if (rc0) return rc0;
  }
  const int rc = e->run_device(reinterpret_cast<const uint8_t *>(d_bytes), d_offsets, n, total_bytes, false, d_ids,
                               ids_capacity, reinterpret_cast<unsigned long long *>(d_id_offsets), total_ids, nullptr, st);
  if (rc) return rc;
  CUDA_TRY(cudaStreamSynchronize(st));
  finish_timing(e);
  return SPM_OK;
}

int spm_encode_ids_device_padded(spm_engine *e, const char *d_bytes, const uint64_t *d_offsets, size_t n,
                                 uint64_t total_bytes, int32_t *d_out, uint64_t out_capacity, uint32_t width,
                                 int32_t pad_id, uint32_t flags, int32_t *d_lengths, uint32_t *width_out,
                                 void *stream) {
  if (!e) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  if (!d_offsets || !width_out || (n && (!d_out || !d_lengths)) || (n && !d_bytes && total_bytes)) {
    e->set_error("null argument");
    return SPM_ERR_ARG;
  }
  if (n >= 0xFFFFFFF0ull) { e->set_error("too many sentences in one call"); return SPM_ERR_ARG; }
  if (flags & ~static_cast<uint32_t>(SPM_PAD_TRUNCATE | SPM_PAD_LEFT)) { e->set_error("unknown flags"); return SPM_ERR_ARG; }
  const bool truncate = flags & SPM_PAD_TRUNCATE;
  const uint32_t frame = e->frame_np + e->frame_ns;
  if (truncate && width && width < frame) {
    e->set_error("width " + std::to_string(width) + " is shorter than the encode frame (" + std::to_string(frame) + " ids)");
    return SPM_ERR_ARG;
  }
  CUDA_TRY(cudaSetDevice(e->device));
  cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : e->stream;
  *width_out = 0;
  if (n == 0) {
    CUDA_TRY(cudaStreamSynchronize(st));
    return SPM_OK;
  }
  e->last_h2d = e->last_d2h = 0;
  if (e->model.model_type == SPM_UNIGRAM) {
    const int rc0 = e->pick_fast_words_device(reinterpret_cast<const uint8_t *>(d_bytes), d_offsets, n, st, &e->batch_fast_words);
    if (rc0) return rc0;
  }
  SPM_TRY(e->encode_stage(reinterpret_cast<const uint8_t *>(d_bytes), d_offsets, n, total_bytes, false, st));
  // ---- the longest framed row decides the width, or whether the call fails ----
  const uint32_t n32 = static_cast<uint32_t>(n);
  CUDA_TRY(cudaMemsetAsync(e->d_ctrl64.p + 2, 0, sizeof(unsigned long long), st));
  const int grid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (n + 255) / 256));
  row_max_kernel<<<grid, 256, 0, st>>>(e->d_sent_count.p, n32, frame, e->d_ctrl64.p + 2);
  CUDA_TRY(cudaGetLastError());
  ++e->last_launches;
  SPM_TRY(e->read_status(st, 0, 4));
  const unsigned long long longest = e->h_ctrl64.p[2];
  if (longest > 0xFFFFFFFFull) { e->set_error("a row is longer than 2^32 - 1 ids"); return SPM_ERR_UNSUPPORTED; }
  if (width && !truncate && longest > width) {
    *width_out = static_cast<uint32_t>(longest);
    e->set_error("a row of " + std::to_string(longest) + " ids does not fit width " + std::to_string(width));
    return SPM_ERR_CAPACITY;
  }
  const uint32_t w = width ? width : static_cast<uint32_t>(longest);
  *width_out = w;
  if (static_cast<unsigned long long>(n) * w > out_capacity) {
    e->set_error("out_capacity too small: need " + std::to_string(static_cast<unsigned long long>(n) * w));
    return SPM_ERR_CAPACITY;
  }
  // ---- the padded writer: one warp per row ----
  const int wgrid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (n + 7) / 8));
  write_padded_kernel<<<wgrid, 256, 0, st>>>(e->d_sent_count.p, e->d_sent_start.p, e->d_tmp_ids.p, n32, e->kframe(), w,
                                             pad_id, truncate ? 1u : 0u, (flags & SPM_PAD_LEFT) ? 1u : 0u, d_out,
                                             d_lengths);
  CUDA_TRY(cudaGetLastError());
  ++e->last_launches;
  CUDA_TRY(cudaEventRecord(e->ev[2], st));
  CUDA_TRY(cudaStreamSynchronize(st));
  finish_timing(e);
  return SPM_OK;
}

static int encode_host_locked(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, bool spans,
                              const int32_t **ids, const uint32_t **tok_end, const uint64_t **id_offsets,
                              const char **normalized, const uint64_t **norm_offsets, const uint32_t **n2o) {
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  if (!offsets || !ids || !id_offsets || (n && !bytes && offsets[n] != offsets[0])) { e->set_error("null argument"); return SPM_ERR_ARG; }
  if (n >= 0xFFFFFFF0ull) { e->set_error("too many sentences in one call"); return SPM_ERR_ARG; }
  CUDA_TRY(cudaSetDevice(e->device));
  cudaStream_t st = e->stream;
  CUDA_TRY(e->h_id_offsets.ensure(n + 1));
  CUDA_TRY(e->h_ids.ensure(1));
  if (n == 0) {
    e->h_id_offsets.p[0] = 0;
    *ids = e->h_ids.p;
    *id_offsets = e->h_id_offsets.p;
    if (spans) {
      CUDA_TRY(e->h_norm_offsets.ensure(1)); CUDA_TRY(e->h_norm.ensure(1)); CUDA_TRY(e->h_tok_end.ensure(1)); CUDA_TRY(e->h_n2o.ensure(1));
      e->h_norm_offsets.p[0] = 0;
      *tok_end = e->h_tok_end.p; *normalized = reinterpret_cast<const char *>(e->h_norm.p);
      *norm_offsets = e->h_norm_offsets.p; *n2o = e->h_n2o.p;
    }
    return SPM_OK;
  }
  for (size_t i = 0; i < n; ++i)
    if (offsets[i + 1] < offsets[i]) { e->set_error("offsets must be non-decreasing"); return SPM_ERR_ARG; }
  const uint64_t base = offsets[0];
  const uint64_t total_bytes = offsets[n] - base;
  CUDA_TRY(e->d_bytes.ensure(total_bytes + 64));
  CUDA_TRY(e->d_offsets.ensure(n + 1));
  if (total_bytes) CUDA_TRY(cudaMemcpyAsync(e->d_bytes.p, bytes + base, total_bytes, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(e->d_offsets.p, offsets, (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
  e->last_h2d = total_bytes + (n + 1) * sizeof(uint64_t);
  uint64_t tot = 0, totn = 0;
  const int rc = e->run_device(e->d_bytes.p - base, e->d_offsets.p, n, total_bytes, spans, nullptr, 0, nullptr, &tot, &totn, st);
  if (rc) return rc;
  CUDA_TRY(e->h_ids.ensure(tot + 1));
  if (tot) CUDA_TRY(cudaMemcpyAsync(e->h_ids.p, e->d_ids.p, tot * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(e->h_id_offsets.p, e->d_id_offsets.p, (n + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  e->last_d2h = tot * sizeof(int32_t) + (n + 1) * sizeof(uint64_t);
  if (spans) {
    CUDA_TRY(e->h_tok_end.ensure(tot + 1));
    CUDA_TRY(e->h_norm.ensure(totn + 1));
    CUDA_TRY(e->h_n2o.ensure(totn + 1));
    CUDA_TRY(e->h_norm_offsets.ensure(n + 1));
    if (tot) CUDA_TRY(cudaMemcpyAsync(e->h_tok_end.p, e->d_tok_end.p, tot * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(e->h_norm.p, e->d_norm.p, totn, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(e->h_n2o.p, e->d_n2o.p, totn * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(e->h_norm_offsets.p, e->d_norm_offsets.p, (n + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    e->last_d2h += tot * 4 + totn * 5 + (n + 1) * 8;
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  finish_timing(e);
  *ids = e->h_ids.p;
  *id_offsets = e->h_id_offsets.p;
  if (spans) {
    *tok_end = e->h_tok_end.p;
    *normalized = reinterpret_cast<const char *>(e->h_norm.p);
    *norm_offsets = e->h_norm_offsets.p;
    *n2o = e->h_n2o.p;
  }
  return SPM_OK;
}

// spm_encode_ids with e->mu already held (also used by the n-best / sampling entry points for nbest_size <= 1)
static int encode_ids_locked(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, const int32_t **ids,
                             const uint64_t **id_offsets) {
  if (offsets && bytes && e->model.model_type == SPM_UNIGRAM && n < 0xFFFFFFF0ull && offsets[n] >= offsets[0])
    e->batch_fast_words = e->pick_fast_words_host(bytes, offsets, n);
  if (offsets && ids && id_offsets && bytes && n >= e->pipeline_min_sentences && n < 0xFFFFFFF0ull) {
    if (e->uses_lane_kernel() && e->sort_by_length && e->fused_host_path) {
      if (e->fused_skip > 0) --e->fused_skip;
      else return e->encode_host_fused(bytes, offsets, n, ids, id_offsets);
    }
    if (e->uses_lane_kernel()) return e->encode_host_streamed(bytes, offsets, n, ids, id_offsets);
    return e->encode_host_pipelined(bytes, offsets, n, ids, id_offsets);
  }
  return encode_host_locked(e, bytes, offsets, n, false, ids, nullptr, id_offsets, nullptr, nullptr, nullptr);
}

int spm_encode_ids(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, const int32_t **ids,
                   const uint64_t **id_offsets) {
  if (!e) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  return encode_ids_locked(e, bytes, offsets, n, ids, id_offsets);
}

static int nbest_args_ok(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n) {
  if (e->model.model_type != SPM_UNIGRAM) {
    e->set_error("NBestEncode is not available for the current model.");  // sentencepiece_processor.cc:662-663
    return SPM_ERR_UNSUPPORTED;
  }
  if (!offsets || (n && !bytes && offsets[n] != offsets[0]) || n >= 0x7FFFFFF0ull) { e->set_error("bad argument"); return SPM_ERR_ARG; }
  for (size_t i = 0; i < n; ++i)
    if (offsets[i + 1] < offsets[i]) { e->set_error("offsets must be non-decreasing"); return SPM_ERR_ARG; }
  if (e->trie.max_key_len > 255) { e->set_error("pieces too long for the n-best device path"); return SPM_ERR_UNSUPPORTED; }
  return SPM_OK;
}

int spm_set_random_seed(spm_engine *e, uint32_t seed) {
  if (!e) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  e->rng.seed(seed);
  return SPM_OK;
}

int spm_nbest_encode(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, int nbest_size,
                     const int32_t **ids, const uint64_t **cand_offsets, const float **scores, const uint32_t **n_cands) {
  if (!e || !ids || !cand_offsets || !scores || !n_cands) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  { const int rc = nbest_args_ok(e, bytes, offsets, n); if (rc) return rc; }
  CUDA_TRY(cudaSetDevice(e->device));
  const uint32_t K = static_cast<uint32_t>(std::max(1, std::min(nbest_size, 1024)));  // unigram_model.cc:701
  cudaStream_t st = e->stream;
  const size_t nc = n * static_cast<size_t>(K);
  if (nc >= 0xFFFFFFF0ull) { e->set_error("n-best: sentences x nbest_size must stay below 2^32; split the batch"); return SPM_ERR_ARG; }
  CUDA_TRY(e->h_cand_offsets.ensure(nc + 1));
  CUDA_TRY(e->h_cand_score.ensure(nc + 1));
  CUDA_TRY(e->h_n_cands.ensure(n + 1));
  CUDA_TRY(e->h_ids.ensure(1));
  *ids = e->h_ids.p; *cand_offsets = e->h_cand_offsets.p; *scores = e->h_cand_score.p; *n_cands = e->h_n_cands.p;
  e->h_cand_offsets.p[0] = 0;
  if (n == 0) return SPM_OK;
  e->last_launches = 0;
  if (K == 1) {
    // nbest_size <= 1: {Encode(normalized), 0.0} (unigram_model.cc:703-705)
    const int32_t *pid; const uint64_t *poff;
    const int rc = encode_ids_locked(e, bytes, offsets, n, &pid, &poff);
    if (rc) return rc;
    for (size_t i = 0; i <= n; ++i) e->h_cand_offsets.p[i] = poff[i];
    for (size_t i = 0; i < n; ++i) { e->h_cand_score.p[i] = 0.f; e->h_n_cands.p[i] = 1; }
    *ids = pid;
    return SPM_OK;
  }
  uint64_t tmp_total = 0;
  { const int rc = e->run_nbest(bytes, offsets, n, K, &tmp_total); if (rc) return rc; }
  // candidate-major compaction: the shared scan + gather over n*K counts; every candidate gets the encode frame
  const uint32_t nc32 = static_cast<uint32_t>(nc);
  const bool framed = e->framed();
  const KFrame F = e->kframe(e->d_n_cands.p, K);
  CUDA_TRY(e->d_cand_offsets.ensure(nc + 1));
  SPM_TRY(e->scan_total(e->d_cand_count.p, nc32, 0, e->d_ctrl64.p + 2, st, framed ? &F : nullptr));
  uint64_t total = tmp_total;
  if (framed) {  // the frame's share depends on the candidate counts: read the total
    SPM_TRY(e->read_status(st, 0, 4));
    total = e->h_ctrl64.p[2];
  }
  CUDA_TRY(e->d_ids.ensure(total + 1));
  if (framed)
    SPM_TRY(e->scan_gather<int32_t, true>(e->d_cand_count.p, nc32, e->d_cand_offsets.p, e->d_cand_start.p, e->d_tmp_ids.p,
                                          e->d_ids.p, e->d_ids.cap, 0, 0ull, st, nullptr, nullptr, F));
  else
    SPM_TRY(e->scan_gather<int32_t>(e->d_cand_count.p, nc32, e->d_cand_offsets.p, e->d_cand_start.p, e->d_tmp_ids.p,
                                    e->d_ids.p, e->d_ids.cap, 0, 0ull, st));
  CUDA_TRY(e->h_ids.ensure(total + 1));
  if (total) CUDA_TRY(cudaMemcpyAsync(e->h_ids.p, e->d_ids.p, total * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(e->h_cand_offsets.p, e->d_cand_offsets.p, (nc + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(e->h_cand_score.p, e->d_cand_score.p, nc * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(e->h_n_cands.p, e->d_n_cands.p, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaEventRecord(e->ev[2], st));
  CUDA_TRY(cudaStreamSynchronize(st));
  e->last_d2h = total * 4 + (nc + 1) * 8 + nc * 4 + n * 4;
  finish_timing(e);
  *ids = e->h_ids.p;
  return SPM_OK;
}

int spm_sample_encode_ids(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, int nbest_size,
                          float alpha, const int32_t **ids, const uint64_t **id_offsets) {
  if (!e || !ids || !id_offsets) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (nbest_size > 512) { e->set_error("nbest_size must be nbest_size <= 512"); return SPM_ERR_ARG; }  // :683
  if (e->model.model_type != SPM_UNIGRAM) {
    // models without NBestEncode go to Model::SampleEncode(normalized, alpha) whatever nbest_size is (:689-693): for
    // BPE that is BPE-dropout, which equals Encode only for alpha <= 0 (bpe_model.cc:132-139)
    if (alpha > 0.f) {
      e->set_error("SampleEncode: BPE-dropout (alpha > 0) is not on the accelerated path");
      return SPM_ERR_UNSUPPORTED;
    }
    return encode_ids_locked(e, bytes, offsets, n, ids, id_offsets);
  }
  if (nbest_size < 0) {
    // forward-filtering / backward-sampling over the whole lattice (unigram_model.cc:511-542)
    { const int rc = nbest_args_ok(e, bytes, offsets, n); if (rc) return rc; }
    if (cudaSetDevice(e->device) != cudaSuccess) { e->set_error("cudaSetDevice failed"); return SPM_ERR_CUDA; }
    const int rc = e->run_lattice(bytes, offsets, n, alpha, 0, 1, true);
    if (rc) return rc;
    if (e->lat_ids.empty()) e->lat_ids.reserve(1);
    *ids = e->lat_ids.data();
    *id_offsets = e->lat_offsets.data();
    return SPM_OK;
  }
  if (nbest_size <= 1) return encode_ids_locked(e, bytes, offsets, n, ids, id_offsets);  // :695-698
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  { const int rc = nbest_args_ok(e, bytes, offsets, n); if (rc) return rc; }
  CUDA_TRY(cudaSetDevice(e->device));
  cudaStream_t st = e->stream;
  const uint32_t K = static_cast<uint32_t>(nbest_size);
  CUDA_TRY(e->h_id_offsets.ensure(n + 1));
  CUDA_TRY(e->h_ids.ensure(1));
  *ids = e->h_ids.p; *id_offsets = e->h_id_offsets.p;
  e->h_id_offsets.p[0] = 0;
  if (n == 0) return SPM_OK;
  e->last_launches = 0;
  uint64_t d2h = 0;
  SPM_TRY(e->sample_picks(bytes, offsets, n, K, alpha, false, false, &d2h));
  CUDA_TRY(e->d_id_offsets.ensure(n + 1));
  const uint32_t n32 = static_cast<uint32_t>(n);
  // every sentence's draw gets the encode frame
  SPM_TRY(e->scan_total(e->d_sent_count.p, n32, e->frame_np + e->frame_ns, e->d_ctrl64.p + 2, st));
  SPM_TRY(e->read_status(st, 0, 4));
  const unsigned long long tot = e->h_ctrl64.p[2];
  CUDA_TRY(e->d_ids.ensure(tot + 1));
  if (e->framed())
    SPM_TRY(e->scan_gather<int32_t, true>(e->d_sent_count.p, n32, e->d_id_offsets.p, e->d_sent_start.p, e->d_tmp_ids.p,
                                          e->d_ids.p, e->d_ids.cap, 0, 0ull, st, nullptr, nullptr, e->kframe()));
  else
    SPM_TRY(e->scan_gather<int32_t>(e->d_sent_count.p, n32, e->d_id_offsets.p, e->d_sent_start.p, e->d_tmp_ids.p,
                                    e->d_ids.p, e->d_ids.cap, 0, 0ull, st));
  CUDA_TRY(e->h_ids.ensure(tot + 1));
  if (tot) CUDA_TRY(cudaMemcpyAsync(e->h_ids.p, e->d_ids.p, tot * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(e->h_id_offsets.p, e->d_id_offsets.p, (n + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaEventRecord(e->ev[2], st));
  CUDA_TRY(cudaStreamSynchronize(st));
  e->last_d2h = d2h + tot * 4 + (n + 1) * 8;
  finish_timing(e);
  *ids = e->h_ids.p;
  *id_offsets = e->h_id_offsets.p;
  return SPM_OK;
}

int spm_calculate_entropy(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, float alpha,
                          const float **entropy) {
  if (!e || !entropy) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (e->model.model_type != SPM_UNIGRAM) {
    e->set_error("CalculateEntropy is not available for the current model.");  // sentencepiece_processor.cc:750-751
    return SPM_ERR_UNSUPPORTED;
  }
  { const int rc = nbest_args_ok(e, bytes, offsets, n); if (rc) return rc; }
  if (cudaSetDevice(e->device) != cudaSuccess) { e->set_error("cudaSetDevice failed"); return SPM_ERR_CUDA; }
  if (e->h_lat_entropy.ensure(n + 1) != cudaSuccess) { e->set_error("pinned allocation failed"); return SPM_ERR_CUDA; }
  *entropy = e->h_lat_entropy.p;
  if (n == 0) return SPM_OK;
  return e->run_lattice(bytes, offsets, n, alpha, 1, 1);
}

int spm_sample_encode_and_score(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, int num_samples,
                                float alpha, int wor, int include_best, const int32_t **ids, const uint64_t **cand_offsets,
                                const float **scores) {
  if (!e || !ids || !cand_offsets || !scores) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (e->model.model_type != SPM_UNIGRAM) {
    e->set_error("SampleEncodeAndScore is not available for the current model.");  // sentencepiece_processor.cc:726-727
    return SPM_ERR_UNSUPPORTED;
  }
  if (wor || include_best) {
    // sampling without replacement runs Lattice::NBest with Gumbel-perturbed scores (unigram_model.cc:770-832)
    e->set_error("SampleEncodeAndScore: wor / include_best are not on the accelerated path");
    return SPM_ERR_UNSUPPORTED;
  }
  if (num_samples < 1 || num_samples > 4096) { e->set_error("num_samples must be in [1, 4096]"); return SPM_ERR_ARG; }
  { const int rc = nbest_args_ok(e, bytes, offsets, n); if (rc) return rc; }
  if (cudaSetDevice(e->device) != cudaSuccess) { e->set_error("cudaSetDevice failed"); return SPM_ERR_CUDA; }
  const int rc = e->run_lattice(bytes, offsets, n, alpha, 0, num_samples);
  if (rc) return rc;
  if (e->lat_ids.empty()) e->lat_ids.reserve(1);
  if (e->lat_scores.empty()) e->lat_scores.reserve(1);
  *ids = e->lat_ids.data();
  *cand_offsets = e->lat_offsets.data();
  *scores = e->lat_scores.data();
  return SPM_OK;
}

int spm_encode_spans(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, const int32_t **ids,
                     const uint32_t **tok_end, const uint64_t **id_offsets, const char **normalized,
                     const uint64_t **norm_offsets, const uint32_t **n2o) {
  if (!e || !tok_end || !normalized || !norm_offsets || !n2o) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  return encode_host_locked(e, bytes, offsets, n, true, ids, tok_end, id_offsets, normalized, norm_offsets, n2o);
}

// Slab elements per chunk of spm_normalize: the slabs take this many bytes of text scratch and as many n2o entries,
// the packed chunk at most as much again (1.25 GB of device memory with offsets at most).  A single sentence whose slab
// is larger is a chunk of its own.  Every chunk waits for its totals; at 2^25 the 1M-sentence uni32k/en batch (10
// bytes of slab per input byte) took 40 chunks and spm_normalize with offsets was slower than spm_encode_spans.
static constexpr unsigned long long kNormChunkSlab = 1ull << 27;

// SentencePieceProcessor::Normalize for a host batch, in chunks of at most kNormChunkSlab slab elements: per chunk the
// input goes up, normalize_kernel (K10) fills the slabs, the scan kernels pack them, and the packed chunk comes down
// into the pinned results behind the earlier chunks.
static int normalize_locked(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, bool with_offsets,
                            const char **normalized, const uint64_t **norm_offsets, const uint32_t **n2o) {
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  if (!offsets || !normalized || !norm_offsets || (with_offsets && !n2o) || (n && !bytes && offsets[n] != offsets[0])) {
    e->set_error("null argument");
    return SPM_ERR_ARG;
  }
  if (n >= 0xFFFFFFF0ull) { e->set_error("too many sentences in one call"); return SPM_ERR_ARG; }
  for (size_t i = 0; i < n; ++i)
    if (offsets[i + 1] < offsets[i]) { e->set_error("offsets must be non-decreasing"); return SPM_ERR_ARG; }
  const uint32_t expand = (e->max_expand_num + e->max_expand_den - 1) / e->max_expand_den;
  for (size_t i = 0; i < n; ++i)
    if (norm_slab_start(offsets[i + 1] - offsets[i], 1, expand) > 0x7FFFFF00ull) {
      e->set_error("sentence too long for the device path");
      return SPM_ERR_UNSUPPORTED;
    }
  CUDA_TRY(cudaSetDevice(e->device));
  cudaStream_t st = e->stream;
  e->last_launches = 0;
  e->last_deferred = 0;
  e->last_h2d = 0;
  e->last_d2h = 0;
  e->last_main_ms = 0.f;
  e->last_ms = 0.f;
  const uint64_t total_bytes = n ? offsets[n] - offsets[0] : 0;
  CUDA_TRY(e->h_norm_offsets.ensure(n + 1));
  CUDA_TRY(e->h_norm.ensure(total_bytes + total_bytes / 2 + 64));
  if (with_offsets) CUDA_TRY(e->h_n2o.ensure(total_bytes + total_bytes / 2 + n + 64));
  e->h_norm_offsets.p[0] = 0;
  // the stream is idle when a pinned result grows (after read_status): what has arrived is kept
  auto grow = [&](auto &buf, size_t have, size_t need) -> cudaError_t {
    if (need <= buf.cap) return cudaSuccess;
    std::remove_reference_t<decltype(buf)> bigger;
    const cudaError_t err = bigger.ensure(need + need / 2);
    if (err != cudaSuccess) return err;
    if (have) memcpy(bigger.p, buf.p, have * sizeof(*buf.p));
    buf = std::move(bigger);
    return cudaSuccess;
  };
  KModel M = e->km;
  M.hot_link = M.hot_val = 0;
  unsigned long long done = 0;  // normalized bytes of the earlier chunks
  for (size_t lo = 0; lo < n;) {
    size_t hi = lo + 1;
    while (hi < n && norm_slab_start(offsets[hi + 1] - offsets[lo], static_cast<uint32_t>(hi + 1 - lo), expand) <= kNormChunkSlab)
      ++hi;
    const uint32_t m = static_cast<uint32_t>(hi - lo);
    const uint64_t chunk_bytes = offsets[hi] - offsets[lo];
    const unsigned long long slab = norm_slab_start(chunk_bytes, m, expand);
    CUDA_TRY(e->d_bytes.ensure(chunk_bytes + 64));
    CUDA_TRY(e->d_offsets.ensure(m + 1));
    CUDA_TRY(e->d_tmp_norm.ensure(slab + 16));
    CUDA_TRY(e->d_norm_start.ensure(m));
    CUDA_TRY(e->d_norm_len.ensure(m));
    CUDA_TRY(e->d_norm.ensure(slab + 16));
    CUDA_TRY(e->d_norm_offsets.ensure(m + 1));
    if (with_offsets) {
      CUDA_TRY(e->d_tmp_n2o.ensure(slab + 16));
      CUDA_TRY(e->d_n2o.ensure(slab + 16));
      CUDA_TRY(e->d_n2o_offsets.ensure(m + 1));
    }
    if (chunk_bytes) CUDA_TRY(cudaMemcpyAsync(e->d_bytes.p, bytes + offsets[lo], chunk_bytes, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(e->d_offsets.p, offsets + lo, (m + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
    e->last_h2d += chunk_bytes + (m + 1) * sizeof(uint64_t);
    CUDA_TRY(cudaMemsetAsync(e->d_ctrl32.p, 0, sizeof(uint32_t), st));
    KNormalize A{};
    A.bytes = e->d_bytes.p;
    A.offsets = e->d_offsets.p;
    A.n = m;
    A.expand = expand;
    A.text = e->d_tmp_norm.p;
    A.n2o = with_offsets ? e->d_tmp_n2o.p : nullptr;
    A.slab = e->d_norm_start.p;
    A.len = e->d_norm_len.p;
    A.status = e->d_ctrl32.p;
    const int grid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (m + 7) / 8));
    CUDA_TRY(cudaEventRecord(e->ev[0], st));
    if (with_offsets) normalize_kernel<true><<<grid, 256, 0, st>>>(M, A);
    else normalize_kernel<false><<<grid, 256, 0, st>>>(M, A);
    CUDA_TRY(cudaGetLastError());
    ++e->last_launches;
    CUDA_TRY(cudaEventRecord(e->ev[1], st));
    SPM_TRY(e->scan_total(e->d_norm_len.p, m, 0, e->d_ctrl64.p + 2, st));
    SPM_TRY(e->scan_gather<uint8_t>(e->d_norm_len.p, m, e->d_norm_offsets.p, e->d_norm_start.p, e->d_tmp_norm.p,
                                    e->d_norm.p, e->d_norm.cap, 0, done, st));
    if (with_offsets) {  // n_i + 1 entries per sentence
      SPM_TRY(e->scan_total(e->d_norm_len.p, m, 1, e->d_ctrl64.p + 3, st));
      SPM_TRY(e->scan_gather<uint32_t>(e->d_norm_len.p, m, e->d_n2o_offsets.p, e->d_norm_start.p, e->d_tmp_n2o.p,
                                       e->d_n2o.p, e->d_n2o.cap, 1, 0ull, st));
    }
    CUDA_TRY(cudaEventRecord(e->ev[2], st));
    SPM_TRY(e->read_status(st, 1, 4));
    float k_ms = 0.f, all_ms = 0.f;
    if (cudaEventElapsedTime(&k_ms, e->ev[0], e->ev[1]) == cudaSuccess) e->last_main_ms += k_ms;
    if (cudaEventElapsedTime(&all_ms, e->ev[0], e->ev[2]) == cudaSuccess) e->last_ms += all_ms;
    if (e->h_ctrl32.p[0]) {
      set_error("normalize: a sentence normalized to more bytes than its bound");
      return SPM_ERR_ENCODE;
    }
    const unsigned long long tot = e->h_ctrl64.p[2];
    CUDA_TRY(grow(e->h_norm, done, done + tot + 1));
    if (tot) CUDA_TRY(cudaMemcpyAsync(e->h_norm.p + done, e->d_norm.p, tot, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(e->h_norm_offsets.p + lo, e->d_norm_offsets.p, (m + 1) * sizeof(uint64_t),
                             cudaMemcpyDeviceToHost, st));
    e->last_d2h += tot + (m + 1) * sizeof(uint64_t);
    if (with_offsets) {
      const unsigned long long n2o_done = done + lo;
      CUDA_TRY(grow(e->h_n2o, n2o_done, n2o_done + tot + m + 1));
      CUDA_TRY(cudaMemcpyAsync(e->h_n2o.p + n2o_done, e->d_n2o.p, (tot + m) * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
      e->last_d2h += (tot + m) * sizeof(uint32_t);
    }
    done += tot;
    lo = hi;
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  e->h_norm.p[done] = 0;
  *normalized = reinterpret_cast<const char *>(e->h_norm.p);
  *norm_offsets = e->h_norm_offsets.p;
  if (n2o) *n2o = with_offsets ? e->h_n2o.p : nullptr;
  return SPM_OK;
}

int spm_normalize(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, int with_offsets,
                  const char **normalized, const uint64_t **norm_offsets, const uint32_t **n2o) {
  if (!e) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  return normalize_locked(e, bytes, offsets, n, with_offsets != 0, normalized, norm_offsets, n2o);
}

int spm_engine::write_pieces(KPieces &P, const char *unk_piece, size_t unk_len, const char **text,
                             const uint64_t **text_offsets, const uint32_t **piece_end, const int32_t **ids,
                             const uint64_t **id_offsets, uint64_t *d2h) {
  cudaStream_t st = stream;
  const uint32_t n32 = P.n;
  const size_t n = n32;
  const int wgrid = static_cast<int>(std::min<size_t>(static_cast<size_t>(sm_count) * 8, (n + 7) / 8));
  SPM_TRY(ensure_piece_tables());
  P.pc_off = d_pc_off.p;
  P.pc_bytes = d_pc_bytes.p;
  P.unk_id = unk_id;
  CUDA_TRY(h_pc_text_offsets.ensure(n + 1));
  CUDA_TRY(h_id_offsets.ensure(n + 1));
  if (unk_piece) {
    CUDA_TRY(d_pc_unk.ensure(unk_len + 1));
    if (unk_len) CUDA_TRY(cudaMemcpyAsync(d_pc_unk.p, unk_piece, unk_len, cudaMemcpyHostToDevice, st));
    P.unk_piece = d_pc_unk.p;
    P.unk_len = static_cast<uint32_t>(unk_len);
  }
  CUDA_TRY(d_pc_text_len.ensure(n));
  CUDA_TRY(d_pc_ntok.ensure(n));
  CUDA_TRY(d_pc_text_offsets.ensure(n + 1));
  CUDA_TRY(d_pc_out_id_offsets.ensure(n + 1));
  P.text_len = d_pc_text_len.p;
  P.n_tok = d_pc_ntok.p;
  pieces_warp_kernel<false><<<wgrid, 256, 0, st>>>(P);
  CUDA_TRY(cudaGetLastError());
  ++last_launches;
  SPM_TRY(scan_total(d_pc_text_len.p, n32, 0, d_ctrl64.p + 2, st));
  SPM_TRY(scan_gather<uint8_t>(d_pc_text_len.p, n32, d_pc_text_offsets.p, nullptr, nullptr, nullptr, 0, 0, 0ull, st));
  SPM_TRY(scan_total(d_pc_ntok.p, n32, 0, d_ctrl64.p + 3, st));
  SPM_TRY(scan_gather<uint8_t>(d_pc_ntok.p, n32, d_pc_out_id_offsets.p, nullptr, nullptr, nullptr, 0, 0, 0ull, st));
  SPM_TRY(read_status(st, 0, 4));
  const unsigned long long ttext = h_ctrl64.p[2], tids = h_ctrl64.p[3];
  CUDA_TRY(d_pc_text.ensure(ttext + 1));
  CUDA_TRY(d_pc_end.ensure(tids + 1));
  CUDA_TRY(d_pc_out_ids.ensure(tids + 1));
  P.text_offsets = d_pc_text_offsets.p;
  P.out_id_offsets = d_pc_out_id_offsets.p;
  P.text = d_pc_text.p;
  P.piece_end = d_pc_end.p;
  P.out_ids = d_pc_out_ids.p;
  pieces_warp_kernel<true><<<wgrid, 256, 0, st>>>(P);
  CUDA_TRY(cudaGetLastError());
  ++last_launches;
  CUDA_TRY(h_pc_text.ensure(ttext + 1));
  CUDA_TRY(h_pc_end.ensure(tids + 1));
  CUDA_TRY(h_ids.ensure(tids + 1));
  if (ttext) CUDA_TRY(cudaMemcpyAsync(h_pc_text.p, d_pc_text.p, ttext, cudaMemcpyDeviceToHost, st));
  if (tids) {
    CUDA_TRY(cudaMemcpyAsync(h_pc_end.p, d_pc_end.p, tids * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(h_ids.p, d_pc_out_ids.p, tids * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  }
  CUDA_TRY(cudaMemcpyAsync(h_pc_text_offsets.p, d_pc_text_offsets.p, (n + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(h_id_offsets.p, d_pc_out_id_offsets.p, (n + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaEventRecord(ev[2], st));
  CUDA_TRY(cudaStreamSynchronize(st));
  *d2h = ttext + tids * 8 + (n + 1) * 16;
  h_pc_text.p[ttext] = 0;
  *text = h_pc_text.p;
  *text_offsets = h_pc_text_offsets.p;
  *piece_end = h_pc_end.p;
  *ids = h_ids.p;
  *id_offsets = h_id_offsets.p;
  return SPM_OK;
}

int spm_engine::raw_segmentation(const char *bytes, const uint64_t *offsets, size_t n, bool detour, KPieces *P,
                                 uint64_t *raw_ids, float *main_ms) {
  cudaStream_t st = stream;
  const uint64_t base = offsets[0];
  const uint64_t total_bytes = offsets[n] - base;
  if (model.model_type == SPM_UNIGRAM) batch_fast_words = pick_fast_words_host(bytes, offsets, n);
  CUDA_TRY(d_bytes.ensure(total_bytes + 64));
  CUDA_TRY(d_offsets.ensure(n + 1));
  CUDA_TRY(cudaEventRecord(ev[3], st));
  if (total_bytes) CUDA_TRY(cudaMemcpyAsync(d_bytes.p, bytes + base, total_bytes, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(d_offsets.p, offsets, (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
  const uint64_t h2d = total_bytes + (n + 1) * sizeof(uint64_t);
  SPM_TRY(raw_segmentation_device(d_bytes.p - base, d_offsets.p, n, total_bytes, detour, P, raw_ids, main_ms, st, {}));
  last_h2d = h2d;
  return SPM_OK;
}

// The engine's encode frame switched off for the guard's scope, and restored when it ends.
struct FrameOff {
  spm_engine *e;
  uint32_t np, ns;
  bool rev;
  explicit FrameOff(spm_engine *x) : e(x), np(x->frame_np), ns(x->frame_ns), rev(x->frame_rev) {
    x->frame_np = x->frame_ns = 0;
    x->frame_rev = false;
  }
  ~FrameOff() { e->frame_np = np; e->frame_ns = ns; e->frame_rev = rev; }
};

int spm_engine::raw_segmentation_device(const uint8_t *d_bytes_base, const uint64_t *d_offs, size_t n,
                                        uint64_t total_bytes, bool detour, KPieces *P, uint64_t *raw_ids,
                                        float *main_ms, cudaStream_t st, const std::function<int()> &at_read) {
  // ---- 1. raw ids: the frame is written once, by K9 / K11 ----
  int rc;
  {
    FrameOff off(this);
    rc = run_device(d_bytes_base, d_offs, n, total_bytes, false, nullptr, 0, nullptr, raw_ids, nullptr, st,
                    &d_pc_ids, &d_pc_id_offsets);
  }
  if (rc) return rc;
  if (cudaEventElapsedTime(main_ms, ev[0], ev[1]) != cudaSuccess) *main_ms = 0.f;
  uint64_t deferred = last_deferred;
  const uint32_t n32 = static_cast<uint32_t>(n);
  const int wgrid = static_cast<int>(std::min<size_t>(static_cast<size_t>(sm_count) * 8, (n + 7) / 8));
  P->n = n32;
  P->ids = d_pc_ids.p;
  P->id_offsets = d_pc_id_offsets.p;
  if (at_read) SPM_TRY(at_read());
  // ---- 2. unknown extents: only the sentences that hold the unknown id take the spans path ----
  uint32_t m = 0;
  if (detour && unk_id >= 0) {
    CUDA_TRY(d_pc_flag.ensure(n));
    CUDA_TRY(d_pc_pos.ensure(n + 1));
    pieces_unk_flag_kernel<<<wgrid, 256, 0, st>>>(d_pc_ids.p, d_pc_id_offsets.p, n32, unk_id, d_pc_flag.p);
    CUDA_TRY(cudaGetLastError());
    ++last_launches;
    SPM_TRY(scan_total(d_pc_flag.p, n32, 0, d_ctrl64.p + 2, st));
    SPM_TRY(scan_gather<uint8_t>(d_pc_flag.p, n32, d_pc_pos.p, nullptr, nullptr, nullptr, 0, 0, 0ull, st));
    SPM_TRY(read_status(st, 0, 4));
    m = static_cast<uint32_t>(h_ctrl64.p[2]);
  } else if (at_read) {
    CUDA_TRY(cudaStreamSynchronize(st));
  }
  if (m) {
    CUDA_TRY(d_pc_sub_of.ensure(n));
    CUDA_TRY(d_pc_sub_start.ensure(m));
    CUDA_TRY(d_pc_sub_len.ensure(m));
    CUDA_TRY(d_pc_sub_offsets.ensure(m + 1));
    CUDA_TRY(d_pc_sub_bytes.ensure(total_bytes + 64));
    pieces_sub_list_kernel<<<static_cast<int>(std::min<size_t>(static_cast<size_t>(sm_count) * 8, (n + 255) / 256)), 256, 0, st>>>(
        d_pc_flag.p, d_pc_pos.p, d_offs, n32, d_pc_sub_of.p, d_pc_sub_start.p, d_pc_sub_len.p);
    CUDA_TRY(cudaGetLastError());
    ++last_launches;
    SPM_TRY(scan_total(d_pc_sub_len.p, m, 0, d_ctrl64.p + 2, st));
    SPM_TRY(scan_gather<uint8_t>(d_pc_sub_len.p, m, d_pc_sub_offsets.p, d_pc_sub_start.p, d_bytes_base,
                                 d_pc_sub_bytes.p, d_pc_sub_bytes.cap, 0, 0ull, st));
    // (the whole batch's byte count bounds the subset's: it only sizes the spans run's temporary buffers)
    uint64_t sub_tot = 0, sub_norm = 0;
    const uint64_t launches = last_launches;  // run_device starts its own count
    rc = run_device(d_pc_sub_bytes.p, reinterpret_cast<const uint64_t *>(d_pc_sub_offsets.p), m, total_bytes, true,
                    nullptr, 0, nullptr, &sub_tot, &sub_norm, st);
    if (rc) return rc;
    last_launches += launches;
    deferred += last_deferred;
    P->sub_of = d_pc_sub_of.p;
    P->sub_ids = d_ids.p;
    P->sub_tok_end = d_tok_end.p;
    P->sub_id_offsets = d_id_offsets.p;
    P->norm = d_norm.p;
    P->norm_offsets = d_norm_offsets.p;
  }
  last_deferred = deferred;
  last_unk_detour = m;
  return SPM_OK;
}

// EncodeAsPieces for a host batch:
//   1. raw ids from the kernels spm_encode_ids runs (lane / BPE-lane2 kernels, deferred and long kernels), frame off;
//   2. without unk_piece: the sentences whose raw ids hold the unknown id are packed on the device and run through the
//      spans path, which gives their token ends in the normalized text (the surfaces of their unknown tokens);
//   3. K9 (pieces_kernel.cuh): size pass, scans, write pass -- the frame, reverse, unk_piece and sep applied once, to
//      pieces and ids alike.
// Steps 1 and 2 are spm_engine::raw_segmentation.
static int encode_pieces_locked(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, const char *unk_piece,
                                size_t unk_len, int sep, const char **text, const uint64_t **text_offsets,
                                const uint32_t **piece_end, const int32_t **ids, const uint64_t **id_offsets) {
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  if (!offsets || !text || !text_offsets || !piece_end || !ids || !id_offsets || (unk_len && !unk_piece) ||
      (n && !bytes && offsets[n] != offsets[0])) {
    e->set_error("null argument");
    return SPM_ERR_ARG;
  }
  if (sep < -1 || sep > 255) { e->set_error("sep must be -1 or a byte value"); return SPM_ERR_ARG; }
  if (unk_len > 0xFFFFFFull) { e->set_error("unk_piece too long"); return SPM_ERR_ARG; }
  if (n >= 0xFFFFFFF0ull) { e->set_error("too many sentences in one call"); return SPM_ERR_ARG; }
  CUDA_TRY(cudaSetDevice(e->device));
  e->last_unk_detour = 0;
  CUDA_TRY(e->h_pc_text_offsets.ensure(n + 1));
  CUDA_TRY(e->h_id_offsets.ensure(n + 1));
  if (n == 0) {
    CUDA_TRY(e->h_pc_text.ensure(1)); CUDA_TRY(e->h_pc_end.ensure(1)); CUDA_TRY(e->h_ids.ensure(1));
    e->h_pc_text_offsets.p[0] = 0;
    e->h_id_offsets.p[0] = 0;
    e->h_pc_text.p[0] = 0;
    *text = e->h_pc_text.p; *text_offsets = e->h_pc_text_offsets.p; *piece_end = e->h_pc_end.p;
    *ids = e->h_ids.p; *id_offsets = e->h_id_offsets.p;
    return SPM_OK;
  }
  for (size_t i = 0; i < n; ++i)
    if (offsets[i + 1] < offsets[i]) { e->set_error("offsets must be non-decreasing"); return SPM_ERR_ARG; }
  SPM_TRY(e->ensure_piece_tables());
  KPieces P{};
  uint64_t raw_ids = 0;
  float main_ms = 0.f;
  SPM_TRY(e->raw_segmentation(bytes, offsets, n, !unk_piece, &P, &raw_ids, &main_ms));
  e->last_h2d += unk_len;
  P.sep = sep;
  P.F = e->kframe();
  // ---- 3. K9: sizes, offsets, pieces ----
  uint64_t d2h = 0;
  SPM_TRY(e->write_pieces(P, unk_piece, unk_len, text, text_offsets, piece_end, ids, id_offsets, &d2h));
  e->last_d2h = d2h;
  e->last_main_ms = main_ms;
  float all = 0.f;
  e->last_ms = cudaEventElapsedTime(&all, e->ev[3], e->ev[2]) == cudaSuccess ? all : main_ms;
  (void)cudaGetLastError();
  return SPM_OK;
}

int spm_encode_pieces(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, const char *unk_piece,
                      size_t unk_piece_len, int sep, const char **text, const uint64_t **text_offsets,
                      const uint32_t **piece_end, const int32_t **ids, const uint64_t **id_offsets) {
  if (!e) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  return encode_pieces_locked(e, bytes, offsets, n, unk_piece, unk_piece_len, sep, text, text_offsets, piece_end, ids,
                              id_offsets);
}

// EncodeAsImmutableProto's ids, offsets and (text != NULL) pieces for a host batch:
//   1. the raw segmentation, with the unknown detour whatever unk_piece is: K11 needs the extents of unknown tokens;
//   2. K11 (offsets_kernel.cuh) in chunks of at most kNormChunkSlab slab elements, as spm_normalize: each chunk
//      normalizes its sentences into slabs and writes begin / end (and, without pieces, the framed ids) in place.
//      The chunks need no totals, so they are queued back to back;
//   3. with pieces: K9 as spm_encode_pieces, which also writes the ids.
static int encode_offsets_locked(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, int32_t eos_id,
                                 const char *unk_piece, size_t unk_len, int sep, const int32_t **ids,
                                 const uint64_t **id_offsets, const uint32_t **begin, const uint32_t **end,
                                 const char **text, const uint64_t **text_offsets, const uint32_t **piece_end) {
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  if (!offsets || !ids || !id_offsets || !begin || !end || (text && (!text_offsets || !piece_end)) ||
      (unk_len && !unk_piece) || (n && !bytes && offsets[n] != offsets[0])) {
    e->set_error("null argument");
    return SPM_ERR_ARG;
  }
  if (sep < -1 || sep > 255) { e->set_error("sep must be -1 or a byte value"); return SPM_ERR_ARG; }
  if (unk_len > 0xFFFFFFull) { e->set_error("unk_piece too long"); return SPM_ERR_ARG; }
  if (n >= 0xFFFFFFF0ull) { e->set_error("too many sentences in one call"); return SPM_ERR_ARG; }
  for (size_t i = 0; i < n; ++i)
    if (offsets[i + 1] < offsets[i]) { e->set_error("offsets must be non-decreasing"); return SPM_ERR_ARG; }
  const uint32_t expand = (e->max_expand_num + e->max_expand_den - 1) / e->max_expand_den;
  for (size_t i = 0; i < n; ++i)
    if (norm_slab_start(offsets[i + 1] - offsets[i], 1, expand) > 0x7FFFFF00ull) {
      e->set_error("sentence too long for the device path");
      return SPM_ERR_UNSUPPORTED;
    }
  CUDA_TRY(cudaSetDevice(e->device));
  cudaStream_t st = e->stream;
  e->last_unk_detour = 0;
  if (n == 0) {
    e->last_launches = e->last_deferred = e->last_h2d = e->last_d2h = 0;
    e->last_main_ms = e->last_ms = 0.f;
    CUDA_TRY(e->h_ids.ensure(1)); CUDA_TRY(e->h_id_offsets.ensure(1));
    CUDA_TRY(e->h_off_begin.ensure(1)); CUDA_TRY(e->h_off_end.ensure(1));
    e->h_id_offsets.p[0] = 0;
    *ids = e->h_ids.p; *id_offsets = e->h_id_offsets.p; *begin = e->h_off_begin.p; *end = e->h_off_end.p;
    if (text) {
      CUDA_TRY(e->h_pc_text.ensure(1)); CUDA_TRY(e->h_pc_text_offsets.ensure(1)); CUDA_TRY(e->h_pc_end.ensure(1));
      e->h_pc_text.p[0] = 0;
      e->h_pc_text_offsets.p[0] = 0;
      *text = e->h_pc_text.p; *text_offsets = e->h_pc_text_offsets.p; *piece_end = e->h_pc_end.p;
    }
    return SPM_OK;
  }
  SPM_TRY(e->ensure_piece_tables());
  KPieces P{};
  uint64_t raw_ids = 0;
  float main_ms = 0.f;
  SPM_TRY(e->raw_segmentation(bytes, offsets, n, true, &P, &raw_ids, &main_ms));
  e->last_h2d += unk_len;
  P.sep = sep;
  P.F = e->kframe();
  P.pc_off = e->d_pc_off.p;
  P.pc_bytes = e->d_pc_bytes.p;
  P.unk_id = e->unk_id;
  const uint64_t tids = raw_ids + static_cast<uint64_t>(n) * (P.F.np + P.F.ns);
  // ---- 2. K11 ----
  std::vector<size_t> cut{0};  // chunk c is sentences [cut[c], cut[c + 1])
  unsigned long long slab_max = 0;
  while (cut.back() < n) {
    const size_t lo = cut.back();
    size_t hi = lo + 1;
    while (hi < n && norm_slab_start(offsets[hi + 1] - offsets[lo], static_cast<uint32_t>(hi + 1 - lo), expand) <= kNormChunkSlab)
      ++hi;
    slab_max = std::max(slab_max, norm_slab_start(offsets[hi] - offsets[lo], static_cast<uint32_t>(hi - lo), expand));
    cut.push_back(hi);
  }
  CUDA_TRY(e->d_tmp_norm.ensure(slab_max + 16));
  CUDA_TRY(e->d_tmp_n2o.ensure(slab_max + 16));
  CUDA_TRY(e->d_off_begin.ensure(tids + 1));
  CUDA_TRY(e->d_off_end.ensure(tids + 1));
  if (!text) {
    CUDA_TRY(e->d_pc_out_ids.ensure(tids + 1));
    CUDA_TRY(e->d_pc_out_id_offsets.ensure(n + 1));
  }
  CUDA_TRY(cudaMemsetAsync(e->d_ctrl32.p, 0, sizeof(uint32_t), st));
  KModel M = e->km;
  M.hot_link = M.hot_val = 0;
  KOffsets A{};
  A.P = P;
  A.offsets = e->d_offsets.p;
  A.expand = expand;
  A.slab_text = e->d_tmp_norm.p;
  A.slab_n2o = e->d_tmp_n2o.p;
  A.eos_id = eos_id;
  A.begin = e->d_off_begin.p;
  A.end = e->d_off_end.p;
  A.out_ids = text ? nullptr : e->d_pc_out_ids.p;
  A.out_id_offsets = text ? nullptr : e->d_pc_out_id_offsets.p;
  A.status = e->d_ctrl32.p;
  CUDA_TRY(cudaEventRecord(e->ev[0], st));  // (raw_segmentation has read ev[0] / ev[1])
  for (size_t c = 0; c + 1 < cut.size(); ++c) {
    A.first = static_cast<uint32_t>(cut[c]);
    A.n = static_cast<uint32_t>(cut[c + 1] - cut[c]);
    A.bytes = e->d_bytes.p + (offsets[cut[c]] - offsets[0]);
    const int grid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (A.n + 7) / 8));
    offsets_kernel<<<grid, 256, 0, st>>>(M, A);
    CUDA_TRY(cudaGetLastError());
    ++e->last_launches;
  }
  CUDA_TRY(cudaEventRecord(e->ev[1], st));
  CUDA_TRY(e->h_off_begin.ensure(tids + 1));
  CUDA_TRY(e->h_off_end.ensure(tids + 1));
  if (tids) {
    CUDA_TRY(cudaMemcpyAsync(e->h_off_begin.p, e->d_off_begin.p, tids * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(e->h_off_end.p, e->d_off_end.p, tids * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  }
  SPM_TRY(e->copy_status(st, 1, 0));
  uint64_t d2h = tids * 8;
  // ---- 3. the ids: K9 with the pieces, or K11's ----
  if (text) {
    uint64_t d2h_pieces = 0;
    SPM_TRY(e->write_pieces(P, unk_piece, unk_len, text, text_offsets, piece_end, ids, id_offsets, &d2h_pieces));
    d2h += d2h_pieces;
  } else {
    CUDA_TRY(e->h_ids.ensure(tids + 1));
    CUDA_TRY(e->h_id_offsets.ensure(n + 1));
    if (tids) CUDA_TRY(cudaMemcpyAsync(e->h_ids.p, e->d_pc_out_ids.p, tids * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(e->h_id_offsets.p, e->d_pc_out_id_offsets.p, (n + 1) * sizeof(uint64_t),
                             cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaEventRecord(e->ev[2], st));
    CUDA_TRY(cudaStreamSynchronize(st));
    d2h += tids * 4 + (n + 1) * 8;
    *ids = e->h_ids.p;
    *id_offsets = e->h_id_offsets.p;
  }
  if (e->h_ctrl32.p[0] & 2u) {
    set_error("encode offsets: a sentence normalized to more bytes than its bound");
    return SPM_ERR_ENCODE;
  }
  if (e->h_ctrl32.p[0]) {
    set_error("encode offsets: all normalized characters are not consumed");
    return SPM_ERR_ENCODE;
  }
  *begin = e->h_off_begin.p;
  *end = e->h_off_end.p;
  e->last_d2h = d2h;
  float k_ms = 0.f, all = 0.f;
  e->last_main_ms = main_ms + (cudaEventElapsedTime(&k_ms, e->ev[0], e->ev[1]) == cudaSuccess ? k_ms : 0.f);
  e->last_ms = cudaEventElapsedTime(&all, e->ev[3], e->ev[2]) == cudaSuccess ? all : e->last_main_ms;
  (void)cudaGetLastError();
  return SPM_OK;
}

int spm_encode_offsets(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, int32_t eos_id,
                       const char *unk_piece, size_t unk_piece_len, int sep, const int32_t **ids,
                       const uint64_t **id_offsets, const uint32_t **begin, const uint32_t **end, const char **text,
                       const uint64_t **text_offsets, const uint32_t **piece_end) {
  if (!e) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  return encode_offsets_locked(e, bytes, offsets, n, eos_id, unk_piece, unk_piece_len, sep, ids, id_offsets, begin, end,
                               text, text_offsets, piece_end);
}

// spm_encode_offsets for a device batch, as padded rows:
//   1. the raw segmentation on st, with the unknown detour; behind its encode, row_max_kernel (the longest framed row)
//      and offsets_plan_kernel (the K11 chunk cuts, the longest sentence) fill d_opad, which comes back in the status
//      read of the detour count;
//   2. the width and capacity checks of spm_encode_ids_device_padded;
//   3. offsets_padded_kernel (K11's padded mode) per chunk, writing every cell of the rows;
//   4. with SPM_OFFSETS_CHARS, spans_to_chars_kernel over all rows.
// Host synchronisations: pick_fast_words_device's (unigram), encode_stage's status reads (one, and one more per
// deferral stage that runs), run_device's total, the detour count (with d_opad), the detour's spans run when a
// sentence holds the unknown id (its encode_stage reads and its total), the rest of the cuts when there are more than
// kOpadInlineCuts chunks, and the final one.
static constexpr uint32_t kOpadInlineCuts = 32;
static constexpr size_t kOpadHead = 4;

// offsets_plan_kernel behind a device batch's encode, into d_opad (sized and its head zeroed here); the caller copies
// the head back (into h_opad, sized here too).
static int queue_offsets_plan(spm_engine *e, const uint64_t *d_offsets, uint32_t n32, uint32_t expand, cudaStream_t st) {
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  CUDA_TRY(e->d_opad.ensure(std::max<size_t>(kOpadHead + 2 * kOpadInlineCuts, kOpadHead + 2 * (size_t{n32} + 1))));
  CUDA_TRY(e->h_opad.ensure(e->d_opad.cap));
  CUDA_TRY(cudaMemsetAsync(e->d_opad.p, 0, kOpadHead * sizeof(unsigned long long), st));
  const int grid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (n32 + 255) / 256));
  offsets_plan_kernel<<<grid, 256, 0, st>>>(d_offsets, n32, expand, kNormChunkSlab,
                                            static_cast<uint32_t>((e->d_opad.cap - kOpadHead) / 2), e->d_opad.p);
  CUDA_TRY(cudaGetLastError());
  ++e->last_launches;
  return SPM_OK;
}

// K11 over a device batch in the chunks that offsets_plan_kernel cut (its head already read into h_opad): fetches the
// cuts past the first kOpadInlineCuts, then queues one launch per chunk on st, behind ev[0].  A's outputs (packed or
// padded mode, as `padded` says) are set by the caller; P is the raw segmentation, which gets the frame and the piece
// table here.
static int offsets_device_chunks(spm_engine *e, bool padded, KPieces P, KOffsets &A, const uint8_t *d_base,
                                 const uint64_t *d_offsets, size_t n, uint32_t expand, int32_t eos_id, cudaStream_t st,
                                 uint64_t *d2h) {
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  const size_t head = kOpadHead + 2 * kOpadInlineCuts;
  const unsigned long long *plan = e->h_opad.p;
  const uint64_t chunks = plan[0], slab_max = plan[1];
  if (chunks > kOpadInlineCuts) {  // (over 2^32 slab elements of input)
    const size_t rest = 2 * (chunks - kOpadInlineCuts);
    CUDA_TRY(cudaMemcpyAsync(e->h_opad.p + head, e->d_opad.p + head, rest * sizeof(unsigned long long),
                             cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    *d2h += rest * sizeof(unsigned long long);
  }
  P.F = e->kframe();
  P.pc_off = e->d_pc_off.p;
  P.pc_bytes = e->d_pc_bytes.p;
  P.unk_id = e->unk_id;
  CUDA_TRY(e->d_tmp_norm.ensure(slab_max + 16));
  CUDA_TRY(e->d_tmp_n2o.ensure(slab_max + 16));
  CUDA_TRY(cudaMemsetAsync(e->d_ctrl32.p, 0, sizeof(uint32_t), st));
  KModel M = e->km;
  M.hot_link = M.hot_val = 0;
  A.P = P;
  A.offsets = d_offsets;
  A.expand = expand;
  A.slab_text = e->d_tmp_norm.p;
  A.slab_n2o = e->d_tmp_n2o.p;
  A.eos_id = eos_id;
  A.status = e->d_ctrl32.p;
  CUDA_TRY(cudaEventRecord(e->ev[0], st));  // (raw_segmentation_device has read ev[0] / ev[1])
  for (uint64_t c = 0; c < chunks; ++c) {
    A.first = static_cast<uint32_t>(plan[kOpadHead + 2 * c]);
    A.n = static_cast<uint32_t>((c + 1 < chunks ? plan[kOpadHead + 2 * (c + 1)] : n) - A.first);
    A.bytes = d_base + plan[kOpadHead + 2 * c + 1];
    const int grid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (A.n + 7) / 8));
    if (padded) offsets_padded_kernel<<<grid, 256, 0, st>>>(M, A);
    else offsets_kernel<<<grid, 256, 0, st>>>(M, A);
    CUDA_TRY(cudaGetLastError());
    ++e->last_launches;
  }
  return SPM_OK;
}

// K11's status word, read back: its errors as spm_encode_offsets reports them.
static int offsets_status(spm_engine *e) {
  if (e->h_ctrl32.p[0] & 2u) {
    e->set_error("encode offsets: a sentence normalized to more bytes than its bound");
    return SPM_ERR_ENCODE;
  }
  if (e->h_ctrl32.p[0]) {
    e->set_error("encode offsets: all normalized characters are not consumed");
    return SPM_ERR_ENCODE;
  }
  return SPM_OK;
}

int spm_encode_offsets_device_padded(spm_engine *e, const char *d_bytes, const uint64_t *d_offsets, size_t n,
                                     uint64_t total_bytes, int32_t eos_id, int32_t *d_ids, int32_t *d_spans,
                                     uint64_t out_capacity, uint32_t width, int32_t pad_id, uint32_t flags,
                                     int32_t *d_lengths, uint32_t *width_out, void *stream) {
  if (!e) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  if (!d_offsets || !width_out || (n && (!d_ids || !d_spans || !d_lengths)) || (n && !d_bytes && total_bytes)) {
    e->set_error("null argument");
    return SPM_ERR_ARG;
  }
  if (n >= 0xFFFFFFF0ull) { e->set_error("too many sentences in one call"); return SPM_ERR_ARG; }
  if (reinterpret_cast<uintptr_t>(d_spans) % 8u) {  // (the kernels store (begin, end) as one 8-byte pair)
    e->set_error("d_spans must be 8-byte aligned");
    return SPM_ERR_ARG;
  }
  if (flags & ~static_cast<uint32_t>(SPM_PAD_TRUNCATE | SPM_PAD_LEFT | SPM_OFFSETS_CHARS)) {
    e->set_error("unknown flags");
    return SPM_ERR_ARG;
  }
  const bool truncate = flags & SPM_PAD_TRUNCATE;
  const uint32_t frame = e->frame_np + e->frame_ns;
  if (truncate && width && width < frame) {
    e->set_error("width " + std::to_string(width) + " is shorter than the encode frame (" + std::to_string(frame) + " ids)");
    return SPM_ERR_ARG;
  }
  CUDA_TRY(cudaSetDevice(e->device));
  cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : e->stream;
  *width_out = 0;
  if (n == 0) {
    CUDA_TRY(cudaStreamSynchronize(st));
    return SPM_OK;
  }
  e->last_h2d = e->last_d2h = 0;
  e->last_unk_detour = 0;
  SPM_TRY(e->ensure_piece_tables());
  const uint8_t *d_base = reinterpret_cast<const uint8_t *>(d_bytes);
  if (e->model.model_type == SPM_UNIGRAM) SPM_TRY(e->pick_fast_words_device(d_base, d_offsets, n, st, &e->batch_fast_words));
  const uint32_t n32 = static_cast<uint32_t>(n);
  const uint32_t expand = (e->max_expand_num + e->max_expand_den - 1) / e->max_expand_den;
  const size_t head = kOpadHead + 2 * kOpadInlineCuts;
  uint64_t d2h = 0;
  auto at_read = [&]() -> int {
    SPM_TRY(queue_offsets_plan(e, d_offsets, n32, expand, st));
    const int grid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (n + 255) / 256));
    row_max_kernel<<<grid, 256, 0, st>>>(e->d_sent_count.p, n32, frame, e->d_opad.p + 3);
    CUDA_TRY(cudaGetLastError());
    ++e->last_launches;
    CUDA_TRY(cudaMemcpyAsync(e->h_opad.p, e->d_opad.p, head * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    d2h += head * sizeof(unsigned long long);
    return SPM_OK;
  };
  KPieces P{};
  uint64_t raw_ids = 0;
  float main_ms = 0.f;
  CUDA_TRY(cudaEventRecord(e->ev[3], st));
  SPM_TRY(e->raw_segmentation_device(d_base, d_offsets, n, total_bytes, true, &P, &raw_ids, &main_ms, st, at_read));
  const unsigned long long *plan = e->h_opad.p;
  const uint64_t longest_input = plan[2], longest = plan[3];
  if (norm_slab_start(longest_input, 1, expand) > 0x7FFFFF00ull) {
    set_error("sentence too long for the device path");
    return SPM_ERR_UNSUPPORTED;
  }
  // ---- the longest framed row decides the width, or whether the call fails ----
  if (longest > 0xFFFFFFFFull) { set_error("a row is longer than 2^32 - 1 ids"); return SPM_ERR_UNSUPPORTED; }
  if (width && !truncate && longest > width) {
    *width_out = static_cast<uint32_t>(longest);
    set_error("a row of " + std::to_string(longest) + " ids does not fit width " + std::to_string(width));
    return SPM_ERR_CAPACITY;
  }
  const uint32_t w = width ? width : static_cast<uint32_t>(longest);
  *width_out = w;
  if (static_cast<unsigned long long>(n) * w > out_capacity) {
    set_error("out_capacity too small: need " + std::to_string(static_cast<unsigned long long>(n) * w));
    return SPM_ERR_CAPACITY;
  }
  // ---- K11, padded: the rows ----
  KOffsets A{};
  A.pad_ids = d_ids;
  A.spans = reinterpret_cast<int2 *>(d_spans);
  A.lengths = d_lengths;
  A.w = w;
  A.pad_id = pad_id;
  A.truncate = truncate ? 1u : 0u;
  A.left = (flags & SPM_PAD_LEFT) ? 1u : 0u;
  SPM_TRY(offsets_device_chunks(e, true, P, A, d_base, d_offsets, n, expand, eos_id, st, &d2h));
  if (flags & SPM_OFFSETS_CHARS) {
    const int grid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (n + 7) / 8));
    spans_to_chars_kernel<<<grid, 256, 0, st>>>(d_base, d_offsets, n32, A.spans, d_lengths, w, e->kframe(), eos_id,
                                                A.left);
    CUDA_TRY(cudaGetLastError());
    ++e->last_launches;
  }
  CUDA_TRY(cudaEventRecord(e->ev[1], st));
  SPM_TRY(e->copy_status(st, 1, 0));
  CUDA_TRY(cudaEventRecord(e->ev[2], st));
  CUDA_TRY(cudaStreamSynchronize(st));
  d2h += sizeof(uint32_t);
  SPM_TRY(offsets_status(e));
  e->last_d2h = d2h;
  float k_ms = 0.f, all = 0.f;
  e->last_main_ms = main_ms + (cudaEventElapsedTime(&k_ms, e->ev[0], e->ev[1]) == cudaSuccess ? k_ms : 0.f);
  e->last_ms = cudaEventElapsedTime(&all, e->ev[3], e->ev[2]) == cudaSuccess ? all : e->last_main_ms;
  (void)cudaGetLastError();
  return SPM_OK;
}

// spm_encode_windows_device: a device batch as overlapping windows of one width.
//   1. the encode: encode_stage (ids only), or the raw segmentation with the unknown detour (offsets);
//   2. behind it, while d_sent_count holds the raw counts, windows_plan: the windows per sentence, their exclusive scan
//      (each sentence's first row, R in total) and the longest body, read back in the call's one status read (with
//      offsets, the detour count's, which also brings the K11 chunk plan);
//   3. the checks on the longest body and R, then window_rows_kernel (row_sentence / row_first);
//   4. ids only: write_windows_kernel from the raw ids, as the padded call writes its rows.  Offsets: K11 in packed
//      mode (framed ids, begin, end; each token walked once), lists_to_chars_kernel with SPM_OFFSETS_CHARS, then
//      write_window_spans_kernel gathers every row from the packed lists.
static int windows_plan(spm_engine *e, uint32_t n32, uint32_t B, uint32_t step, cudaStream_t st, uint64_t *d2h) {
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  CUDA_TRY(e->d_win.ensure(size_t{n32} + 3));
  CUDA_TRY(e->h_win.ensure(2));
  CUDA_TRY(e->d_win_count.ensure(n32));
  CUDA_TRY(cudaMemsetAsync(e->d_win.p + 1, 0, sizeof(unsigned long long), st));
  const int grid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (n32 + 255) / 256));
  row_max_kernel<<<grid, 256, 0, st>>>(e->d_sent_count.p, n32, 0u, e->d_win.p + 1);
  window_count_kernel<<<grid, 256, 0, st>>>(e->d_sent_count.p, n32, B, step, e->d_win_count.p);
  CUDA_TRY(cudaGetLastError());
  e->last_launches += 2;
  SPM_TRY(e->scan_total(e->d_win_count.p, n32, 0, e->d_win.p, st));
  SPM_TRY(e->scan_gather<uint8_t>(e->d_win_count.p, n32, e->d_win.p + 2, nullptr, nullptr, nullptr, 0, 0, 0ull, st));
  CUDA_TRY(cudaMemcpyAsync(e->h_win.p, e->d_win.p, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  *d2h += 2 * sizeof(unsigned long long);
  return SPM_OK;
}

int spm_encode_windows_device(spm_engine *e, const char *d_bytes, const uint64_t *d_offsets, size_t n,
                              uint64_t total_bytes, uint32_t width, uint32_t stride, int32_t pad_id, uint32_t flags,
                              int32_t eos_id, int32_t *d_ids, int32_t *d_spans, uint64_t rows_capacity,
                              int32_t *d_lengths, int32_t *d_row_sentence, int32_t *d_row_first, uint64_t *rows_out,
                              void *stream) {
  if (!e) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  if (!d_offsets || !rows_out || (n && (!d_ids || !d_lengths || !d_row_sentence || !d_row_first)) ||
      (n && !d_bytes && total_bytes)) {
    set_error("null argument");
    return SPM_ERR_ARG;
  }
  if (n >= 0xFFFFFFF0ull) { set_error("too many sentences in one call"); return SPM_ERR_ARG; }
  if (reinterpret_cast<uintptr_t>(d_spans) % 8u) {  // (the kernels store (begin, end) as one 8-byte pair)
    set_error("d_spans must be 8-byte aligned");
    return SPM_ERR_ARG;
  }
  if (flags & SPM_PAD_TRUNCATE) { set_error("windows keep every token: SPM_PAD_TRUNCATE does not apply"); return SPM_ERR_ARG; }
  if (flags & ~static_cast<uint32_t>(SPM_PAD_LEFT | SPM_OFFSETS_CHARS)) { set_error("unknown flags"); return SPM_ERR_ARG; }
  if ((flags & SPM_OFFSETS_CHARS) && !d_spans) { set_error("SPM_OFFSETS_CHARS needs d_spans"); return SPM_ERR_ARG; }
  if (width == 0) { set_error("windows need a fixed width"); return SPM_ERR_ARG; }
  const uint32_t frame = e->frame_np + e->frame_ns;
  if (width <= frame) {
    set_error("width " + std::to_string(width) + " leaves no body next to the encode frame (" + std::to_string(frame) +
              " ids)");
    return SPM_ERR_ARG;
  }
  const uint32_t B = width - frame;
  if (stride >= B) {
    set_error("stride " + std::to_string(stride) + " must be less than the window's body of " + std::to_string(B) + " ids");
    return SPM_ERR_ARG;
  }
  const uint32_t step = B - stride;
  const uint32_t left = (flags & SPM_PAD_LEFT) ? 1u : 0u;
  CUDA_TRY(cudaSetDevice(e->device));
  cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : e->stream;
  *rows_out = 0;
  if (n == 0) {
    CUDA_TRY(cudaStreamSynchronize(st));
    return SPM_OK;
  }
  e->last_h2d = e->last_d2h = 0;
  const bool spans = d_spans != nullptr;
  const uint8_t *d_base = reinterpret_cast<const uint8_t *>(d_bytes);
  const uint32_t n32 = static_cast<uint32_t>(n);
  const uint32_t expand = (e->max_expand_num + e->max_expand_den - 1) / e->max_expand_den;
  if (spans) {
    e->last_unk_detour = 0;
    SPM_TRY(e->ensure_piece_tables());
  }
  if (e->model.model_type == SPM_UNIGRAM) SPM_TRY(e->pick_fast_words_device(d_base, d_offsets, n, st, &e->batch_fast_words));
  uint64_t d2h = 0;
  KPieces P{};
  uint64_t raw_ids = 0;
  float main_ms = 0.f;
  if (!spans) {
    SPM_TRY(e->encode_stage(d_base, d_offsets, n, total_bytes, false, st));
    SPM_TRY(windows_plan(e, n32, B, step, st, &d2h));
    CUDA_TRY(cudaStreamSynchronize(st));
  } else {
    const size_t head = kOpadHead + 2 * kOpadInlineCuts;
    auto at_read = [&]() -> int {
      SPM_TRY(queue_offsets_plan(e, d_offsets, n32, expand, st));
      CUDA_TRY(cudaMemcpyAsync(e->h_opad.p, e->d_opad.p, head * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
      d2h += head * sizeof(unsigned long long);
      return windows_plan(e, n32, B, step, st, &d2h);
    };
    CUDA_TRY(cudaEventRecord(e->ev[3], st));
    SPM_TRY(e->raw_segmentation_device(d_base, d_offsets, n, total_bytes, true, &P, &raw_ids, &main_ms, st, at_read));
    if (norm_slab_start(e->h_opad.p[2], 1, expand) > 0x7FFFFF00ull) {
      set_error("sentence too long for the device path");
      return SPM_ERR_UNSUPPORTED;
    }
  }
  // ---- the rows: their number decides whether the call fails ----
  const unsigned long long R = e->h_win.p[0], longest = e->h_win.p[1];
  if (longest > 0x7FFFFFFFull) {
    set_error("a sentence of " + std::to_string(longest) + " ids is longer than 2^31 - 1 ids");
    return SPM_ERR_UNSUPPORTED;
  }
  if (R > 0x7FFFFFFFull) { set_error(std::to_string(R) + " rows do not fit int32"); return SPM_ERR_UNSUPPORTED; }
  *rows_out = R;
  if (R > rows_capacity) {
    set_error("rows_capacity too small: need " + std::to_string(R) + " rows");
    return SPM_ERR_CAPACITY;
  }
  const uint32_t R32 = static_cast<uint32_t>(R);
  const int sgrid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (n + 7) / 8));
  const int rgrid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (R + 7) / 8));
  window_rows_kernel<<<sgrid, 256, 0, st>>>(e->d_win.p + 2, n32, step, nullptr, d_row_sentence, d_row_first);
  CUDA_TRY(cudaGetLastError());
  ++e->last_launches;
  if (!spans) {
    write_windows_kernel<<<rgrid, 256, 0, st>>>(e->d_sent_count.p, e->d_sent_start.p, e->d_tmp_ids.p, R32, e->kframe(),
                                                width, pad_id, left, d_ids, d_lengths, d_row_sentence, d_row_first);
    CUDA_TRY(cudaGetLastError());
    ++e->last_launches;
    CUDA_TRY(cudaEventRecord(e->ev[2], st));
    CUDA_TRY(cudaStreamSynchronize(st));
    e->last_d2h = d2h;
    finish_timing(e);
    return SPM_OK;
  }
  // ---- K11, packed: every token's begin / end once, then the rows ----
  const uint64_t tids = raw_ids + static_cast<uint64_t>(n) * frame;
  CUDA_TRY(e->d_off_begin.ensure(tids + 1));
  CUDA_TRY(e->d_off_end.ensure(tids + 1));
  CUDA_TRY(e->d_pc_out_ids.ensure(tids + 1));
  CUDA_TRY(e->d_pc_out_id_offsets.ensure(n + 1));
  KOffsets A{};
  A.begin = e->d_off_begin.p;
  A.end = e->d_off_end.p;
  A.out_ids = e->d_pc_out_ids.p;
  A.out_id_offsets = e->d_pc_out_id_offsets.p;
  SPM_TRY(offsets_device_chunks(e, false, P, A, d_base, d_offsets, n, expand, eos_id, st, &d2h));
  if (flags & SPM_OFFSETS_CHARS) {
    lists_to_chars_kernel<<<sgrid, 256, 0, st>>>(d_base, d_offsets, n32, A.begin, A.end, A.out_id_offsets, e->kframe(),
                                                 eos_id);
    CUDA_TRY(cudaGetLastError());
    ++e->last_launches;
  }
  write_window_spans_kernel<<<rgrid, 256, 0, st>>>(A.out_ids, A.begin, A.end, A.out_id_offsets, R32, d_row_sentence,
                                                   d_row_first, e->frame_np, frame, width, pad_id, left, d_ids,
                                                   reinterpret_cast<int2 *>(d_spans), d_lengths);
  CUDA_TRY(cudaGetLastError());
  ++e->last_launches;
  CUDA_TRY(cudaEventRecord(e->ev[1], st));
  SPM_TRY(e->copy_status(st, 1, 0));
  CUDA_TRY(cudaEventRecord(e->ev[2], st));
  CUDA_TRY(cudaStreamSynchronize(st));
  d2h += sizeof(uint32_t);
  SPM_TRY(offsets_status(e));
  e->last_d2h = d2h;
  float k_ms = 0.f, all = 0.f;
  e->last_main_ms = main_ms + (cudaEventElapsedTime(&k_ms, e->ev[0], e->ev[1]) == cudaSuccess ? k_ms : 0.f);
  e->last_ms = cudaEventElapsedTime(&all, e->ev[3], e->ev[2]) == cudaSuccess ? all : e->last_main_ms;
  (void)cudaGetLastError();
  return SPM_OK;
}

// spm_encode_pairs_device: 2n sentences as n pair rows (or more, when one member is cut into windows).
//   1. the encode over the 2n sentences with the engine's frame off for the whole call (FrameOff): encode_stage (ids
//      only), or the raw segmentation with the unknown detour (offsets);
//   2. behind it, while d_sent_count holds the raw counts, pairs_plan: pair_plan_kernel (kept ids, rows and step per
//      pair, the least workable width), the exclusive scan of the rows (R in total), read back in the call's one
//      status read (with offsets, the detour count's, which also brings the K11 chunk plan);
//   3. the width and R checks, then window_rows_kernel with the per-pair steps (row_pair / row_first);
//   4. ids only: write_pair_rows_kernel from the raw ids.  Offsets: K11 in packed mode over the 2n sentences,
//      lists_to_chars_kernel with SPM_OFFSETS_CHARS, then write_pair_spans_kernel gathers every row.
static int pairs_plan(spm_engine *e, uint32_t n32, const KPairs &T, uint32_t w, uint32_t trunc, uint32_t overflow,
                      uint32_t stride, cudaStream_t st, uint64_t *d2h) {
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  CUDA_TRY(e->d_win.ensure(size_t{n32} + 3));
  CUDA_TRY(e->h_win.ensure(2));
  CUDA_TRY(e->d_win_count.ensure(n32));
  CUDA_TRY(e->d_pair_keep.ensure(n32));
  CUDA_TRY(e->d_pair_step.ensure(n32));
  CUDA_TRY(cudaMemsetAsync(e->d_win.p + 1, 0, sizeof(unsigned long long), st));
  const int grid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (n32 + 255) / 256));
  pair_plan_kernel<<<grid, 256, 0, st>>>(e->d_sent_count.p, n32, T, w, trunc, overflow, stride, e->d_pair_keep.p,
                                         e->d_win_count.p, e->d_pair_step.p, e->d_win.p + 1);
  CUDA_TRY(cudaGetLastError());
  ++e->last_launches;
  SPM_TRY(e->scan_total(e->d_win_count.p, n32, 0, e->d_win.p, st));
  SPM_TRY(e->scan_gather<uint8_t>(e->d_win_count.p, n32, e->d_win.p + 2, nullptr, nullptr, nullptr, 0, 0, 0ull, st));
  CUDA_TRY(cudaMemcpyAsync(e->h_win.p, e->d_win.p, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  *d2h += 2 * sizeof(unsigned long long);
  return SPM_OK;
}

int spm_encode_pairs_device(spm_engine *e, const char *d_bytes, const uint64_t *d_offsets, size_t n,
                            uint64_t total_bytes, const int32_t *prefix, uint32_t n_prefix, const int32_t *middle,
                            uint32_t n_middle, const int32_t *suffix, uint32_t n_suffix, uint32_t width,
                            uint32_t truncation, uint32_t stride, int32_t pad_id, uint32_t flags, int32_t *d_ids,
                            int32_t *d_type_ids, int32_t *d_spans, uint64_t rows_capacity, uint64_t cells_capacity,
                            int32_t *d_lengths, int32_t *d_row_pair, int32_t *d_row_first, uint64_t *rows_out,
                            uint32_t *width_out, void *stream) {
  if (!e) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  if (!d_offsets || !rows_out || !width_out ||
      (n && (!d_ids || !d_type_ids || !d_lengths || !d_row_pair || !d_row_first)) || (n && !d_bytes && total_bytes) ||
      (n_prefix && !prefix) || (n_middle && !middle) || (n_suffix && !suffix)) {
    set_error("null argument");
    return SPM_ERR_ARG;
  }
  if (n >= 0xFFFFFFF0ull / 2) { set_error("too many sentences in one call"); return SPM_ERR_ARG; }
  if (reinterpret_cast<uintptr_t>(d_spans) % 8u) {  // (the kernels store (begin, end) as one 8-byte pair)
    set_error("d_spans must be 8-byte aligned");
    return SPM_ERR_ARG;
  }
  if (flags & SPM_PAD_TRUNCATE) { set_error("pairs truncate by their strategy: SPM_PAD_TRUNCATE does not apply"); return SPM_ERR_ARG; }
  if (flags & ~static_cast<uint32_t>(SPM_PAD_LEFT | SPM_OFFSETS_CHARS | SPM_PAIR_OVERFLOW)) {
    set_error("unknown flags");
    return SPM_ERR_ARG;
  }
  if ((flags & SPM_OFFSETS_CHARS) && !d_spans) { set_error("SPM_OFFSETS_CHARS needs d_spans"); return SPM_ERR_ARG; }
  if (truncation > SPM_PAIR_TRUNC_ONLY_SECOND) { set_error("unknown truncation strategy"); return SPM_ERR_ARG; }
  const uint32_t overflow = (flags & SPM_PAIR_OVERFLOW) ? 1u : 0u;
  if (overflow && truncation != SPM_PAIR_TRUNC_ONLY_FIRST && truncation != SPM_PAIR_TRUNC_ONLY_SECOND) {
    set_error("SPM_PAIR_OVERFLOW needs SPM_PAIR_TRUNC_ONLY_FIRST or SPM_PAIR_TRUNC_ONLY_SECOND");
    return SPM_ERR_ARG;
  }
  if (stride && !overflow) { set_error("a stride needs SPM_PAIR_OVERFLOW"); return SPM_ERR_ARG; }
  std::vector<int32_t> tmpl;  // prefix, middle, suffix
  const int32_t V = e->model.vocab_size();
  for (const auto &[list, len] : {std::pair{prefix, n_prefix}, std::pair{middle, n_middle}, std::pair{suffix, n_suffix}}) {
    if (len > spm_engine::kMaxFrame) { set_error("a template list holds more than 64 ids"); return SPM_ERR_ARG; }
    for (uint32_t k = 0; k < len; ++k) {
      if (list[k] < 0 || list[k] >= V) {
        set_error("template id " + std::to_string(list[k]) + " is outside [0, " + std::to_string(V) + ")");
        return SPM_ERR_ARG;
      }
      tmpl.push_back(list[k]);
    }
  }
  const uint32_t tsz = n_prefix + n_middle + n_suffix;
  if (truncation != SPM_PAIR_TRUNC_NONE && width <= tsz) {
    set_error("width " + std::to_string(width) + " leaves no room next to the template (" + std::to_string(tsz) +
              " ids)");
    return SPM_ERR_ARG;
  }
  const uint32_t left = (flags & SPM_PAD_LEFT) ? 1u : 0u;
  CUDA_TRY(cudaSetDevice(e->device));
  cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : e->stream;
  *rows_out = 0;
  *width_out = 0;
  if (n == 0) {
    CUDA_TRY(cudaStreamSynchronize(st));
    return SPM_OK;
  }
  e->last_h2d = e->last_d2h = 0;
  FrameOff off(e);  // the template replaces the frame: every stage below sees raw ids
  const bool spans = d_spans != nullptr;
  const uint8_t *d_base = reinterpret_cast<const uint8_t *>(d_bytes);
  const size_t n2 = 2 * n;
  const uint32_t n32 = static_cast<uint32_t>(n), m32 = static_cast<uint32_t>(n2);
  const uint32_t expand = (e->max_expand_num + e->max_expand_den - 1) / e->max_expand_den;
  CUDA_TRY(e->d_pair_tmpl.ensure(std::max<size_t>(tsz, 1)));
  if (tsz) {  // (from pageable memory: the copy is staged before cudaMemcpyAsync returns)
    CUDA_TRY(cudaMemcpyAsync(e->d_pair_tmpl.p, tmpl.data(), tsz * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    e->last_h2d = tsz * sizeof(int32_t);
  }
  const KPairs T{e->d_pair_tmpl.p, n_prefix, n_middle, n_suffix,
                 overflow ? (truncation == SPM_PAIR_TRUNC_ONLY_FIRST ? 1u : 2u) : 0u};
  if (spans) {
    e->last_unk_detour = 0;
    SPM_TRY(e->ensure_piece_tables());
  }
  if (e->model.model_type == SPM_UNIGRAM) SPM_TRY(e->pick_fast_words_device(d_base, d_offsets, n2, st, &e->batch_fast_words));
  uint64_t d2h = 0;
  KPieces P{};
  uint64_t raw_ids = 0;
  float main_ms = 0.f;
  if (!spans) {
    SPM_TRY(e->encode_stage(d_base, d_offsets, n2, total_bytes, false, st));
    SPM_TRY(pairs_plan(e, n32, T, width, truncation, overflow, stride, st, &d2h));
    CUDA_TRY(cudaStreamSynchronize(st));
  } else {
    const size_t head = kOpadHead + 2 * kOpadInlineCuts;
    auto at_read = [&]() -> int {
      SPM_TRY(queue_offsets_plan(e, d_offsets, m32, expand, st));
      CUDA_TRY(cudaMemcpyAsync(e->h_opad.p, e->d_opad.p, head * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
      d2h += head * sizeof(unsigned long long);
      return pairs_plan(e, n32, T, width, truncation, overflow, stride, st, &d2h);
    };
    CUDA_TRY(cudaEventRecord(e->ev[3], st));
    SPM_TRY(e->raw_segmentation_device(d_base, d_offsets, n2, total_bytes, true, &P, &raw_ids, &main_ms, st, at_read));
    if (norm_slab_start(e->h_opad.p[2], 1, expand) > 0x7FFFFF00ull) {
      set_error("sentence too long for the device path");
      return SPM_ERR_UNSUPPORTED;
    }
  }
  // ---- the width, then the rows: each decides whether the call fails ----
  const unsigned long long R = e->h_win.p[0], need = e->h_win.p[1];
  if (need >= 0xFFFFFFFFull) { set_error("a row is longer than 2^32 - 2 ids"); return SPM_ERR_UNSUPPORTED; }
  if (width && need > width) {
    *width_out = static_cast<uint32_t>(need);
    set_error(truncation == SPM_PAIR_TRUNC_NONE
                  ? "a row of " + std::to_string(need) + " ids does not fit width " + std::to_string(width)
                  : "a pair needs width " + std::to_string(need) + " to keep its other member whole and the room " +
                        "above the stride");
    return SPM_ERR_CAPACITY;
  }
  const uint32_t w = width ? width : static_cast<uint32_t>(need);
  if (R > 0x7FFFFFFFull) { set_error(std::to_string(R) + " rows do not fit int32"); return SPM_ERR_UNSUPPORTED; }
  *rows_out = R;
  *width_out = w;
  if (R > rows_capacity || R * w > cells_capacity) {
    set_error("capacity too small: need " + std::to_string(R) + " rows of " + std::to_string(w) + " cells");
    return SPM_ERR_CAPACITY;
  }
  const uint32_t R32 = static_cast<uint32_t>(R);
  const int pgrid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (n + 7) / 8));
  const int rgrid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (R + 7) / 8));
  window_rows_kernel<<<pgrid, 256, 0, st>>>(e->d_win.p + 2, n32, 0u, e->d_pair_step.p, d_row_pair, d_row_first);
  CUDA_TRY(cudaGetLastError());
  ++e->last_launches;
  if (!spans) {
    write_pair_rows_kernel<<<rgrid, 256, 0, st>>>(e->d_sent_count.p, e->d_sent_start.p, e->d_tmp_ids.p, n32, R32, T,
                                                  e->d_pair_keep.p, d_row_pair, d_row_first, w, pad_id, left, d_ids,
                                                  d_type_ids, d_lengths);
    CUDA_TRY(cudaGetLastError());
    ++e->last_launches;
    CUDA_TRY(cudaEventRecord(e->ev[2], st));
    CUDA_TRY(cudaStreamSynchronize(st));
    e->last_d2h = d2h;
    finish_timing(e);
    return SPM_OK;
  }
  // ---- K11, packed over the 2n sentences: every token's begin / end once, then the rows ----
  CUDA_TRY(e->d_off_begin.ensure(raw_ids + 1));
  CUDA_TRY(e->d_off_end.ensure(raw_ids + 1));
  CUDA_TRY(e->d_pc_out_ids.ensure(raw_ids + 1));
  CUDA_TRY(e->d_pc_out_id_offsets.ensure(n2 + 1));
  KOffsets A{};
  A.begin = e->d_off_begin.p;
  A.end = e->d_off_end.p;
  A.out_ids = e->d_pc_out_ids.p;
  A.out_id_offsets = e->d_pc_out_id_offsets.p;
  SPM_TRY(offsets_device_chunks(e, false, P, A, d_base, d_offsets, n2, expand, -1, st, &d2h));
  const int sgrid = static_cast<int>(std::min<size_t>(static_cast<size_t>(e->sm_count) * 8, (n2 + 7) / 8));
  if (flags & SPM_OFFSETS_CHARS) {
    lists_to_chars_kernel<<<sgrid, 256, 0, st>>>(d_base, d_offsets, m32, A.begin, A.end, A.out_id_offsets, e->kframe(),
                                                 -1);
    CUDA_TRY(cudaGetLastError());
    ++e->last_launches;
  }
  write_pair_spans_kernel<<<rgrid, 256, 0, st>>>(A.out_ids, A.begin, A.end, A.out_id_offsets, n32, R32, T,
                                                 e->d_pair_keep.p, d_row_pair, d_row_first, w, pad_id, left, d_ids,
                                                 d_type_ids, reinterpret_cast<int2 *>(d_spans), d_lengths);
  CUDA_TRY(cudaGetLastError());
  ++e->last_launches;
  CUDA_TRY(cudaEventRecord(e->ev[1], st));
  SPM_TRY(e->copy_status(st, 1, 0));
  CUDA_TRY(cudaEventRecord(e->ev[2], st));
  CUDA_TRY(cudaStreamSynchronize(st));
  d2h += sizeof(uint32_t);
  SPM_TRY(offsets_status(e));
  e->last_d2h = d2h;
  float k_ms = 0.f, all = 0.f;
  e->last_main_ms = main_ms + (cudaEventElapsedTime(&k_ms, e->ev[0], e->ev[1]) == cudaSuccess ? k_ms : 0.f);
  e->last_ms = cudaEventElapsedTime(&all, e->ev[3], e->ev[2]) == cudaSuccess ? all : e->last_main_ms;
  (void)cudaGetLastError();
  return SPM_OK;
}

// unk_piece / sep as spm_encode_pieces takes them
static int pieces_args_ok(spm_engine *e, const char *unk_piece, size_t unk_len, int sep) {
  if (unk_len && !unk_piece) { e->set_error("null argument"); return SPM_ERR_ARG; }
  if (sep < -1 || sep > 255) { e->set_error("sep must be -1 or a byte value"); return SPM_ERR_ARG; }
  if (unk_len > 0xFFFFFFull) { e->set_error("unk_piece too long"); return SPM_ERR_ARG; }
  return SPM_OK;
}

// K9 over candidate lists of the n-best buffers (run_nbest with ends; norm unless unk_piece or byte fallback makes the
// unknown surfaces unnecessary): list j is ids [start[j], + count[j]) of sentence j / per.
static KPieces candidate_lists(spm_engine *e, uint32_t lists, const unsigned long long *start, const uint32_t *count,
                               uint32_t per, bool norm, int sep, const KFrame &F) {
  KPieces P{};
  P.n = lists;
  P.ids = e->d_tmp_ids.p;
  P.list_start = start;
  P.list_count = count;
  if (norm) {
    P.tok_end = e->d_nb_end.p;
    P.sent_norm = e->d_nb_norm.p;
    P.sent_norm_start = e->d_nb_norm_start.p;
  }
  P.per = per;
  P.sep = sep;
  P.F = F;
  return P;
}

// Whether the pieces of a batch need the unknown tokens' normalized text (K5 exports it).
static bool needs_unk_surface(const spm_engine *e, const char *unk_piece) {
  return !unk_piece && e->unk_id >= 0 && !e->model.byte_fallback;
}

int spm_nbest_encode_pieces(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, int nbest_size,
                            const char *unk_piece, size_t unk_piece_len, int sep, const char **text,
                            const uint64_t **text_offsets, const uint32_t **piece_end, const int32_t **ids,
                            const uint64_t **cand_offsets, const float **scores, const uint32_t **n_cands) {
  if (!e || !text || !text_offsets || !piece_end || !ids || !cand_offsets || !scores || !n_cands) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  { const int rc = nbest_args_ok(e, bytes, offsets, n); if (rc) return rc; }
  SPM_TRY(pieces_args_ok(e, unk_piece, unk_piece_len, sep));
  CUDA_TRY(cudaSetDevice(e->device));
  const uint32_t K = static_cast<uint32_t>(std::max(1, std::min(nbest_size, 1024)));  // unigram_model.cc:701
  cudaStream_t st = e->stream;
  const size_t nc = n * static_cast<size_t>(K);
  if (nc >= 0xFFFFFFF0ull) { e->set_error("n-best: sentences x nbest_size must stay below 2^32; split the batch"); return SPM_ERR_ARG; }
  CUDA_TRY(e->h_cand_score.ensure(nc + 1));
  CUDA_TRY(e->h_n_cands.ensure(n + 1));
  *scores = e->h_cand_score.p; *n_cands = e->h_n_cands.p;
  if (K == 1 || n == 0) {
    // nbest_size <= 1: {Encode(normalized), 0.0} (unigram_model.cc:703-705)
    SPM_TRY(encode_pieces_locked(e, bytes, offsets, n, unk_piece, unk_piece_len, sep, text, text_offsets, piece_end, ids,
                                 cand_offsets));
    for (size_t i = 0; i < n; ++i) { e->h_cand_score.p[i] = 0.f; e->h_n_cands.p[i] = 1; }
    return SPM_OK;
  }
  e->last_launches = 0;
  e->last_unk_detour = 0;
  const bool norm = needs_unk_surface(e, unk_piece);
  uint64_t tmp_total = 0;
  SPM_TRY(e->run_nbest(bytes, offsets, n, K, &tmp_total, norm, norm));
  // candidate-major lists; every real candidate gets the encode frame, empty slots stay empty
  KPieces P = candidate_lists(e, static_cast<uint32_t>(nc), e->d_cand_start.p, e->d_cand_count.p, K, norm, sep,
                              e->kframe(e->d_n_cands.p, K));
  CUDA_TRY(cudaMemcpyAsync(e->h_cand_score.p, e->d_cand_score.p, nc * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(e->h_n_cands.p, e->d_n_cands.p, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  uint64_t d2h = 0;
  SPM_TRY(e->write_pieces(P, unk_piece, unk_piece_len, text, text_offsets, piece_end, ids, cand_offsets, &d2h));
  e->last_d2h = d2h + nc * 4 + n * 4;
  finish_timing(e);
  return SPM_OK;
}

int spm_sample_encode_pieces(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n, int nbest_size,
                             float alpha, const char *unk_piece, size_t unk_piece_len, int sep, const char **text,
                             const uint64_t **text_offsets, const uint32_t **piece_end, const int32_t **ids,
                             const uint64_t **id_offsets) {
  if (!e || !text || !text_offsets || !piece_end || !ids || !id_offsets) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  auto set_error = [&](const std::string &m) { e->set_error(m); };
  if (nbest_size > 512) { e->set_error("nbest_size must be nbest_size <= 512"); return SPM_ERR_ARG; }  // :683
  SPM_TRY(pieces_args_ok(e, unk_piece, unk_piece_len, sep));
  if (e->model.model_type != SPM_UNIGRAM) {  // as spm_sample_encode_ids
    if (alpha > 0.f) {
      e->set_error("SampleEncode: BPE-dropout (alpha > 0) is not on the accelerated path");
      return SPM_ERR_UNSUPPORTED;
    }
    return encode_pieces_locked(e, bytes, offsets, n, unk_piece, unk_piece_len, sep, text, text_offsets, piece_end, ids,
                                id_offsets);
  }
  if (nbest_size < 0) {
    { const int rc = nbest_args_ok(e, bytes, offsets, n); if (rc) return rc; }
    CUDA_TRY(cudaSetDevice(e->device));
    const spm_engine::LatPieces pc{unk_piece, unk_piece_len, sep};
    SPM_TRY(e->run_lattice(bytes, offsets, n, alpha, 0, 1, true, &pc));
    if (e->lat_ids.empty()) e->lat_ids.reserve(1);
    if (e->lat_text.empty()) e->lat_text.reserve(1);
    if (e->lat_piece_end.empty()) e->lat_piece_end.reserve(1);
    *text = e->lat_text.data(); *text_offsets = e->lat_text_offsets.data(); *piece_end = e->lat_piece_end.data();
    *ids = e->lat_ids.data(); *id_offsets = e->lat_offsets.data();
    return SPM_OK;
  }
  if (nbest_size <= 1)
    return encode_pieces_locked(e, bytes, offsets, n, unk_piece, unk_piece_len, sep, text, text_offsets, piece_end, ids,
                                id_offsets);
  { const int rc = nbest_args_ok(e, bytes, offsets, n); if (rc) return rc; }
  if (n == 0)
    return encode_pieces_locked(e, bytes, offsets, n, unk_piece, unk_piece_len, sep, text, text_offsets, piece_end, ids,
                                id_offsets);
  CUDA_TRY(cudaSetDevice(e->device));
  e->last_launches = 0;
  e->last_unk_detour = 0;
  const bool norm = needs_unk_surface(e, unk_piece);
  uint64_t d2h = 0, d2h_pieces = 0;
  SPM_TRY(e->sample_picks(bytes, offsets, n, static_cast<uint32_t>(nbest_size), alpha, norm, norm, &d2h));
  // every sentence's draw gets the encode frame
  KPieces P = candidate_lists(e, static_cast<uint32_t>(n), e->d_sent_start.p, e->d_sent_count.p, 1, norm, sep, e->kframe());
  SPM_TRY(e->write_pieces(P, unk_piece, unk_piece_len, text, text_offsets, piece_end, ids, id_offsets, &d2h_pieces));
  e->last_d2h = d2h + d2h_pieces;
  finish_timing(e);
  return SPM_OK;
}

int spm_sample_encode_and_score_pieces(spm_engine *e, const char *bytes, const uint64_t *offsets, size_t n,
                                       int num_samples, float alpha, int wor, int include_best, const char *unk_piece,
                                       size_t unk_piece_len, int sep, const char **text, const uint64_t **text_offsets,
                                       const uint32_t **piece_end, const int32_t **ids, const uint64_t **cand_offsets,
                                       const float **scores) {
  if (!e || !text || !text_offsets || !piece_end || !ids || !cand_offsets || !scores) return SPM_ERR_ARG;
  std::lock_guard<std::mutex> lk(e->mu);
  if (e->model.model_type != SPM_UNIGRAM) {
    e->set_error("SampleEncodeAndScore is not available for the current model.");  // sentencepiece_processor.cc:726-727
    return SPM_ERR_UNSUPPORTED;
  }
  if (wor || include_best) {
    e->set_error("SampleEncodeAndScore: wor / include_best are not on the accelerated path");
    return SPM_ERR_UNSUPPORTED;
  }
  if (num_samples < 1 || num_samples > 4096) { e->set_error("num_samples must be in [1, 4096]"); return SPM_ERR_ARG; }
  { const int rc = nbest_args_ok(e, bytes, offsets, n); if (rc) return rc; }
  { const int rc = pieces_args_ok(e, unk_piece, unk_piece_len, sep); if (rc) return rc; }
  if (cudaSetDevice(e->device) != cudaSuccess) { e->set_error("cudaSetDevice failed"); return SPM_ERR_CUDA; }
  const spm_engine::LatPieces pc{unk_piece, unk_piece_len, sep};
  const int rc = e->run_lattice(bytes, offsets, n, alpha, 0, num_samples, false, &pc);
  if (rc) return rc;
  if (e->lat_ids.empty()) e->lat_ids.reserve(1);
  if (e->lat_scores.empty()) e->lat_scores.reserve(1);
  if (e->lat_text.empty()) e->lat_text.reserve(1);
  if (e->lat_piece_end.empty()) e->lat_piece_end.reserve(1);
  *text = e->lat_text.data(); *text_offsets = e->lat_text_offsets.data(); *piece_end = e->lat_piece_end.data();
  *ids = e->lat_ids.data(); *cand_offsets = e->lat_offsets.data(); *scores = e->lat_scores.data();
  return SPM_OK;
}

}  // extern "C"
