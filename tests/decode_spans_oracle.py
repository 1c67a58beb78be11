"""ctypes front-end of tests/decode_spans_oracle.c, the restatement of Decode(ids, SentencePieceText*) that
spm_decode_offsets is checked against.  The C file is compiled once per process into a temporary directory (the
repository may be read-only), with $CC or gcc."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

from oracle import modelproto

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "decode_spans_oracle.c")
_lib = None


def _load():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="decode_spans_oracle_"), "decode_spans_oracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-std=c11", "-O2", "-fPIC", "-shared", "-o", so, _SRC])
        L = ctypes.CDLL(so)
        vp = ctypes.c_void_p
        L.decode_spans_batch.argtypes = [vp, vp, vp, ctypes.c_int32, ctypes.c_int, ctypes.c_int, vp, ctypes.c_size_t,
                                         vp, vp, ctypes.c_size_t, vp, ctypes.c_uint64, vp, vp, vp]
        _lib = L
    return _lib


class DecodeSpans:
    """One model's decode restatement: decode_spans_batch(ids, id_offsets) -> (text uint8[], text_offsets uint64[n+1],
    tok_end uint32[]), tok_end[k - id_offsets[0]] the end of token k's surface relative to its list's text."""

    def __init__(self, model_bytes):
        m = modelproto.parse_model(model_bytes)
        self.pieces = np.frombuffer(b"".join(m["pieces"]) + b"\0", np.uint8)
        self.off = np.zeros(len(m["pieces"]) + 1, np.uint64)
        self.off[1:] = np.cumsum([len(p) for p in m["pieces"]])
        self.types = np.asarray(m["types"], np.uint8)
        self.flags = (int(m["add_dummy_prefix"]), int(m["remove_extra_whitespaces"]))
        self.unk = np.frombuffer(bytes(m["unk_surface"]) + b"\0", np.uint8)
        self.unk_len = len(m["unk_surface"])
        # no surface is longer than its piece, unk_surface or U+FFFD
        self.max_surface = max([len(p) for p in m["pieces"]] + [self.unk_len, 3])

    def decode_spans_batch(self, ids, ido):
        L = _load()
        ids = np.ascontiguousarray(ids, np.int32)
        ido = np.ascontiguousarray(ido, np.uint64)
        n = len(ido) - 1
        tot = int(ido[n]) - int(ido[0])
        cap = tot * self.max_surface + 1
        text = np.zeros(cap, np.uint8)
        to = np.zeros(n + 1, np.uint64)
        te = np.zeros(max(tot, 1), np.uint32)
        bad = ctypes.c_int64()
        rc = L.decode_spans_batch(self.pieces.ctypes.data, self.off.ctypes.data, self.types.ctypes.data,
                                  len(self.types), *self.flags, self.unk.ctypes.data, self.unk_len,
                                  ids[int(ido[0]):].ctypes.data if tot else ids.ctypes.data, ido.ctypes.data, n,
                                  text.ctypes.data, cap, to.ctypes.data, te.ctypes.data, ctypes.byref(bad))
        if rc:
            raise RuntimeError(f"decode_spans_batch failed ({rc}) at list {bad.value}")
        return text[:int(to[n])].copy(), to, te[:tot]
