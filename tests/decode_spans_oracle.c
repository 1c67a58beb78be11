/* decode_spans_oracle.c -- TEST INFRASTRUCTURE ONLY: a plain-C restatement of the reference's
 * SentencePieceProcessor::Decode(const std::vector<int>&, SentencePieceText*) (src/sentencepiece_processor.cc:766-925)
 * for the text and where every token's surface lies in it, the checker of spm_decode_offsets.  tests/decode_spans_oracle.py
 * compiles it into a temporary directory and calls it through ctypes.  It shares no code with the engine or with
 * oracle/spm_oracle.c.
 *
 * Per id list, in token order (SetSurface, :822-828, appends every surface to the text):
 *   CONTROL -> "", UNKNOWN -> unk_surface (DecodeSentencePiece, :779-790);
 *   any other piece: while no token has produced text and no leading U+2581 has been consumed (is_bos_ws, :879-887),
 *     with add_dummy_prefix or remove_extra_whitespaces one leading U+2581 is dropped, and with
 *     remove_extra_whitespaces the state stays open; then U+2581 -> ' ' (:792-809);
 *   a run of BYTE pieces (ProcessBytePieces, :830-881), flushed before the next other piece and at the end: one
 *     character at a time, a valid c-byte character gives "" to its first c-1 tokens and the character to the last, a
 *     structurally invalid byte gives U+FFFD to its token. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* bytes of one valid UTF-8 character at b[0..len) (IsValidDecodeUTF8: shortest form, no surrogates, <= U+10FFFF), 0 if
 * b[0] does not start one */
static size_t utf8_char(const uint8_t *b, size_t len) {
  if (b[0] < 0x80) return 1;
  size_t need;
  uint32_t cp, min;
  if ((b[0] & 0xE0) == 0xC0) { need = 2; cp = b[0] & 0x1F; min = 0x80; }
  else if ((b[0] & 0xF0) == 0xE0) { need = 3; cp = b[0] & 0x0F; min = 0x800; }
  else if ((b[0] & 0xF8) == 0xF0) { need = 4; cp = b[0] & 0x07; min = 0x10000; }
  else return 0;
  if (len < need) return 0;
  for (size_t k = 1; k < need; ++k) {
    if ((b[k] & 0xC0) != 0x80) return 0;
    cp = (cp << 6) | (b[k] & 0x3F);
  }
  if (cp < min || cp > 0x10FFFF || (cp >= 0xD800 && cp <= 0xDFFF)) return 0;
  return need;
}

/* PieceToByte (model_interface.cc): "<0xXX>" with upper-case hex -> XX, else -1 */
static int piece_byte(const uint8_t *p, size_t len) {
  if (len != 6 || p[0] != '<' || p[1] != '0' || p[2] != 'x' || p[5] != '>') return -1;
  int v = 0;
  for (int k = 3; k < 5; ++k) {
    const int c = p[k];
    const int d = c >= '0' && c <= '9' ? c - '0' : (c >= 'A' && c <= 'F' ? c - 'A' + 10 : -1);
    if (d < 0) return -1;
    v = v * 16 + d;
  }
  return v;
}

enum { kNormal = 1, kUnknown = 2, kControl = 3, kByte = 6 };

/* n lists (list i is ids[ido[i] - ido[0] .. ido[i+1] - ido[0])).  Out: text (cap bytes), text_offsets[n+1],
 * tok_end[ido[n] - ido[0]] relative to the list's text.  Returns 0; 1 for an id out of range, 2 for a BYTE piece that
 * is not <0xXX>, 3 when text does not fit (*bad: the list). */
int decode_spans_batch(const uint8_t *pieces, const uint64_t *piece_off, const uint8_t *types, int32_t vocab,
                       int add_dummy_prefix, int remove_extra_whitespaces, const uint8_t *unk_surface, size_t unk_len,
                       const int32_t *ids, const uint64_t *ido, size_t n, uint8_t *text, uint64_t cap,
                       uint64_t *text_offsets, uint32_t *tok_end, int64_t *bad) {
  static const uint8_t kWs[3] = {0xE2, 0x96, 0x81}, kRepl[3] = {0xEF, 0xBF, 0xBD};
  const int strip = add_dummy_prefix || remove_extra_whitespaces;
  uint64_t out = 0;
  text_offsets[0] = 0;
  uint8_t *bytes = (uint8_t *)malloc((size_t)(ido[n] - ido[0]) + 1); /* the pending BYTE run */
  if (!bytes) { *bad = -1; return 3; }
#define PUT(src, len)                                  \
  do {                                                 \
    if (out + (len) > cap) { free(bytes); *bad = (int64_t)i; return 3; } \
    memcpy(text + out, (src), (len));                  \
    out += (len);                                      \
  } while (0)
  for (size_t i = 0; i < n; ++i) {
    const int32_t *L = ids + (ido[i] - ido[0]);
    uint32_t *E = tok_end + (ido[i] - ido[0]);
    const size_t m = (size_t)(ido[i + 1] - ido[i]);
    const uint64_t start = out;
    for (size_t k = 0; k < m; ++k)
      if (L[k] < 0 || L[k] >= vocab) { free(bytes); *bad = (int64_t)i; return 1; }
    int bos = 1, bos_seen = 0;
    size_t run = 0; /* first token of the pending BYTE run */
    for (size_t k = 0; k <= m; ++k) {
      if (k < m && types[L[k]] == kByte) continue;
      const size_t nb = k - run;
      for (size_t q = 0; q < nb; ++q) { /* ProcessBytePieces(run, k) */
        const int32_t id = L[run + q];
        const int b = piece_byte(pieces + piece_off[id], (size_t)(piece_off[id + 1] - piece_off[id]));
        if (b < 0) { free(bytes); *bad = (int64_t)i; return 2; }
        bytes[q] = (uint8_t)b;
      }
      for (size_t p = 0; p < nb;) {
        const size_t c = utf8_char(bytes + p, nb - p);
        if (c == 0) {
          PUT(kRepl, 3);
          E[run + p] = (uint32_t)(out - start);
          p += 1;
        } else {
          for (size_t j = 0; j + 1 < c; ++j) E[run + p + j] = (uint32_t)(out - start);
          PUT(bytes + p, c);
          E[run + p + c - 1] = (uint32_t)(out - start);
          p += c;
        }
      }
      if (k == m) break;
      run = k + 1;
      if (bos_seen || out != start) bos = 0;
      const int32_t id = L[k];
      const uint8_t *pc = pieces + piece_off[id];
      size_t len = (size_t)(piece_off[id + 1] - piece_off[id]);
      int consumed = 0;
      if (types[id] == kControl) {
        len = 0;
      } else if (types[id] == kUnknown) {
        PUT(unk_surface, unk_len);
        len = 0;
      } else if (bos && strip && len >= 3 && memcmp(pc, kWs, 3) == 0) {
        pc += 3;
        len -= 3;
        consumed = !remove_extra_whitespaces;
      }
      for (size_t q = 0; q < len;) {
        if (q + 3 <= len && memcmp(pc + q, kWs, 3) == 0) { PUT(" ", 1); q += 3; }
        else { PUT(pc + q, 1); q += 1; }
      }
      E[k] = (uint32_t)(out - start);
      bos_seen = consumed;
    }
    text_offsets[i + 1] = out;
  }
#undef PUT
  free(bytes);
  return 0;
}
