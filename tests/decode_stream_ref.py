"""Restatement of spm_decode_stream_device (include/spm_b200.h) over tests/decode_spans_oracle.py, without torch.

A row that has consumed the ids S holds back its held tail: the ids of a trailing BYTE run from the first UTF-8
decision that still lacks bytes.  A call returns Decode(S) from what the row returned before up to the end of the last
settled token, that token's end as Decode(S, SentencePieceText*) sets it.  When the call finishes the row nothing is
held."""
import numpy as np

from decode_spans_oracle import DecodeSpans
from oracle import modelproto


def utf8_need(b0):
    """the bytes the reference's DecodeUTF8 reads to decide at lead byte b0"""
    if b0 & 0xE0 == 0xC0:
        return 2
    if b0 & 0xF0 == 0xE0:
        return 3
    if b0 & 0xF8 == 0xF0:
        return 4
    return 1


def utf8_valid(b):
    """IsValidDecodeUTF8 over the bytes b (at most 4): bytes of one valid character at b[0], 0 if b[0] is invalid"""
    try:
        c = utf8_need(b[0])
        if len(b) < c:
            return 0
        s = bytes(b[:c]).decode("utf-8")
        return c if len(s) == 1 else 0
    except UnicodeDecodeError:
        return 0


class StreamRef:
    def __init__(self, model_bytes):
        self.spans = DecodeSpans(model_bytes)
        m = modelproto.parse_model(model_bytes)
        self.byte = np.full(len(m["pieces"]), -1, np.int64)
        for i, (p, t) in enumerate(zip(m["pieces"], m["types"])):
            if t == modelproto.BYTE and len(p) == 6 and p.startswith(b"<0x") and p.endswith(b">"):
                self.byte[i] = int(p[3:5], 16)

    def held(self, ids):
        """the number of ids at the end of `ids` that a row which has consumed them holds back (0..3)"""
        j = len(ids)
        while j > 0 and self.byte[ids[j - 1]] >= 0:
            j -= 1
        run = [int(self.byte[x]) for x in ids[j:]]
        p = 0
        while p < len(run):
            if len(run) - p < utf8_need(run[p]):
                return len(run) - p
            p += utf8_valid(run[p:p + 4]) or 1
        return 0

    def deltas(self, ids, calls, final=True):
        """The texts (bytes) of successive calls that pass calls[j] more of `ids`; with final, the last call finishes
        the row.  Token ends are those of Decode(ids): a settled token ends where it ends in every longer list."""
        ids = np.asarray(ids, np.int32)
        text, _, te = self.spans.decode_spans_batch(ids, np.array([0, len(ids)], np.uint64))
        out, prev, pos = [], 0, 0
        for j, k in enumerate(calls):
            pos += k
            settled = pos - (0 if final and j == len(calls) - 1 else self.held(ids[:pos]))
            end = int(te[settled - 1]) if settled else 0
            out.append(text[prev:end].tobytes())
            prev = end
        return out

    def deltas_by_prefix(self, ids, calls, final=True):
        """deltas() by the definition: Decode of every prefix the row has consumed, cut at its last settled token"""
        ids = np.asarray(ids, np.int32)
        out, prev, pos = [], 0, 0
        for j, k in enumerate(calls):
            pos += k
            text, _, te = self.spans.decode_spans_batch(ids[:pos], np.array([0, pos], np.uint64))
            settled = pos - (0 if final and j == len(calls) - 1 else self.held(ids[:pos]))
            end = int(te[settled - 1]) if settled else 0
            out.append(text[prev:end].tobytes())
            prev = end
        return out


def random_calls(rng, n, max_step=4):
    """a random splitting of n ids into calls of 0..max_step ids each"""
    calls, left = [], n
    while left:
        k = min(int(rng.integers(0, max_step + 1)), left)
        calls.append(k)
        left -= k
    return calls + [0] * int(rng.integers(0 if calls else 1, 2))
