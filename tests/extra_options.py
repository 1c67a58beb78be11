"""SetEncodeExtraOptions in the tests' own terms: ApplyExtraOptions (src/sentencepiece_processor.cc:1019-1064) restated
option by option on id lists, and the digests of what the unmodified reference (oracle/_ref) returned under extra
options, kept in tests/golden/reference_digests_extra.json.  Same digests and the same recording rule as
tests/refstore.py: build oracle/_ref and run tests/test_oracle_extra_options.py with SPM_RECORD_REFERENCE=1."""
import ctypes
import json
import os

import numpy as np

from refstore import digest

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_digests_extra.json")
# option strings every entry point is checked under; "" is the plain output
OPTION_SETS = ["bos", "eos", "bos:eos", "reverse", "bos:reverse:eos", "eos:bos:bos", "reverse:reverse", ""]
# the strings the reference's results are stored for
REFERENCE_SETS = ["bos:eos", "reverse:eos", "bos:reverse:eos", "eos:bos:bos"]
EDGE_LINES = [b"", b"   ", b"a", b"hello world", b"\xe2\x96\x81", b"\xff\xfe"]
_store = None


def apply_extra(ids, options, bos, eos):
    """ApplyExtraOptions on one id list, option by option in order."""
    out = list(ids)
    for o in options.split(":") if options else []:
        if o == "reverse":
            out.reverse()
        elif o == "bos":
            out.insert(0, bos)
        elif o == "eos":
            out.append(eos)
    return out


def apply_packed(ids, offs, options, bos, eos, skip_empty=False):
    """apply_extra over every list of a packed result -> (ids int32[], offsets uint64[]).  skip_empty: empty lists
    stay empty (SampleEncodeAndScore returns no sample for an empty sentence)."""
    lists = []
    for i in range(len(offs) - 1):
        a = ids[int(offs[i]):int(offs[i + 1])].tolist()
        lists.append(a if skip_empty and not a else apply_extra(a, options, bos, eos))
    o = np.zeros(len(lists) + 1, dtype=np.uint64)
    if lists:
        o[1:] = np.cumsum([len(a) for a in lists], dtype=np.uint64)
    flat = np.array([x for a in lists for x in a], dtype=np.int32)
    return flat, o


def set_reference_options(ref, options):
    """SetEncodeExtraOptions on the compiled reference, through the oracle shim's ref_set_encode_extra_options."""
    ref.lib.ref_set_encode_extra_options.argtypes = [ctypes.c_void_p, ctypes.c_char_p]
    assert ref.lib.ref_set_encode_extra_options(ref.h, options.encode()) == 0, options


def reference(key, compute):
    """The stored digest of the reference's result for `key`; with SPM_RECORD_REFERENCE=1, `compute()` is run and its
    digest stored first."""
    global _store
    if _store is None:
        _store = {}
        if os.path.exists(PATH):
            with open(PATH) as f:
                _store = json.load(f)
    if os.environ.get("SPM_RECORD_REFERENCE") == "1":
        r = compute()
        _store[key] = digest(*(r if isinstance(r, tuple) else (r,)))
        with open(PATH, "w") as f:
            json.dump(_store, f, indent=1, sort_keys=True)
            f.write("\n")
    assert key in _store, f"no stored reference result for {key} (see tests/extra_options.py)"
    return _store[key]


def nbest_digest(cands):
    """digest of per-sentence n-best lists (lists of id arrays)"""
    return digest([[np.asarray(c, dtype=np.int32) for c in cs] for cs in cands])
