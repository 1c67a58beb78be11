"""Digests of what the unmodified reference (oracle/_ref) returned for the EncodeAsPieces tests
(tests/test_gpu_pieces.py), kept in tests/golden/reference_digests_pieces.json.  Same digests and the same recording
rule as tests/refstore.py: build oracle/_ref and run the tests with SPM_RECORD_REFERENCE=1 to store them again.  Each
test takes its reference digest before it creates an engine, so the recording also works where no GPU is present."""
import json
import os

import numpy as np

from refstore import digest

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_digests_pieces.json")
_store = None


def pieces_digest(rows, ids=None):
    """digest of per-sentence piece lists (bytes), and of their ids when given"""
    text = b"".join(b"".join(r) for r in rows)
    lens = np.array([len(p) for r in rows for p in r], dtype=np.int64)
    counts = np.array([len(r) for r in rows], dtype=np.int64)
    parts = (text, lens, counts) if ids is None else (text, lens, counts, np.asarray(ids, dtype=np.int64))
    return digest(*parts)


def reference(key, compute):
    """The stored digest of the reference's result for `key`; with SPM_RECORD_REFERENCE=1, `compute()` (which returns
    the digest itself) is run and stored first."""
    global _store
    if _store is None:
        _store = {}
        if os.path.exists(PATH):
            with open(PATH) as f:
                _store = json.load(f)
    if os.environ.get("SPM_RECORD_REFERENCE") == "1":
        _store[key] = compute()
        with open(PATH, "w") as f:
            json.dump(_store, f, indent=1, sort_keys=True)
            f.write("\n")
    assert key in _store, f"no stored reference result for {key} (see tests/refstore_pieces.py)"
    return _store[key]
