"""Digests of what the unmodified reference (oracle/_ref) returned for the long-sentence lattice tests
(tests/test_oracle_lattice_long.py, tests/test_gpu_lattice_long.py), kept in
tests/golden/reference_digests_long.json.  Same digests and the same recording rule as tests/refstore.py: build
oracle/_ref and run the tests with SPM_RECORD_REFERENCE=1 to store them again."""
import json
import os

from refstore import digest

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_digests_long.json")
_store = None


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
    assert key in _store, f"no stored reference result for {key} (see tests/refstore_long.py)"
    return _store[key]
