"""spm_decode_offsets against spm_decode_ids on bench.py's seeded corpora at 1M sentences (uni32k/en,
mix_bf8k/mixed): the corpus is encoded once, and its ids, in pinned host memory, are decoded by both calls.  At this
size both take the chunked three-stage path (pipeline_min_sentences).
End to end: a host clock around each call (the calls return with their results in pinned host memory); best and median
of --steps timed rounds after --warmup rounds, the two calls alternating.  Kernel against copy: the engine's own
timings (spm_engine_info: last_main_kernel_ms for the decode kernels, last_kernel_ms with the scan and gather kernels)
and the bytes each call copied back.  The check: the text and text offsets of spm_decode_offsets equal spm_decode_ids'
for every list, and its token ends equal those of tests/decode_spans_oracle.c on a stride of lists.  One JSON line
per result, the first one with the GPU name and power limit.  Needs an H100; writes nothing.
Usage: python tools/decode_offsets_bench.py [--n 1000000] [--steps 10] [--warmup 2] [--stride 499]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

CORPUS_SEED = 20260922  # bench.py's
WORKLOADS = [("uni32k", "en"), ("mix_bf8k", "mixed")]


def stats(ts):
    return {"best_ms": round(float(np.min(ts)), 3), "median_ms": round(float(np.median(ts)), 3)}


def parity(eng, om, ids, ido, stride):
    text, to = eng.decode_packed(ids, ido)
    t2, to2, te = eng.decode_offsets(ids, ido)
    same_text = bool(np.array_equal(text, t2) and np.array_equal(to, to2))
    bad = 0
    sel = range(0, len(ido) - 1, stride)
    for i in sel:
        a, b = int(ido[i]), int(ido[i + 1])
        _, _, ote = om.decode_spans_batch(ids[a:b], np.array([0, b - a], np.uint64))
        bad += not np.array_equal(te[a:b], ote)
    return {"text_identical_all_lists": same_text, "tok_end_oracle_lists_checked": len(sel), "tok_end_mismatches": bad}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--stride", type=int, default=499)
    a = ap.parse_args()
    import torch
    import corpus
    from decode_spans_oracle import DecodeSpans
    from sentencepiece_b200 import Engine
    if not torch.cuda.is_available():
        raise SystemExit("decode_offsets_bench needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    g = corpus.CorpusGen()
    for model, kind in WORKLOADS:
        mb = open(os.path.join(ROOT, "tests", "golden", "models", model + ".model"), "rb").read()
        buf, offs = g.fill(kind, CORPUS_SEED, a.n)
        eng = Engine(mb)
        ids, ido = eng.encode_packed(buf, offs)
        ids = torch.from_numpy(np.ascontiguousarray(ids)).pin_memory().numpy()
        ido = torch.from_numpy(np.ascontiguousarray(ido).view(np.int64)).pin_memory().numpy().view(np.uint64)
        r = {"model": model, "kind": kind, "n": a.n, "ids": int(ido[-1])}
        r.update(parity(eng, DecodeSpans(mb), ids, ido, a.stride))
        L, h, n = eng._lib, eng._h, a.n
        p = [ctypes.c_void_p() for _ in range(3)]
        ref = [ctypes.byref(x) for x in p]

        def check(rc):
            if rc:
                raise RuntimeError(L.spm_last_error(h).decode())
        fns = {"decode_ids": lambda: check(L.spm_decode_ids(h, ids.ctypes.data, ido.ctypes.data, n, *ref[:2])),
               "decode_offsets": lambda: check(L.spm_decode_offsets(h, ids.ctypes.data, ido.ctypes.data, n, *ref))}
        for _ in range(a.warmup):
            for f in fns.values():
                f()
        ts = {k: [] for k in fns}
        info = {k: [] for k in fns}
        for _ in range(a.steps):
            for k, f in fns.items():
                t0 = time.perf_counter()
                f()
                ts[k].append((time.perf_counter() - t0) * 1e3)
                i = eng.info()
                info[k].append((i.last_main_kernel_ms, i.last_kernel_ms, int(i.last_d2h_bytes)))
        for k in fns:
            best = int(np.argmin(ts[k]))
            km, ka, d2h = info[k][best]
            r[k] = dict(stats(ts[k]), decode_kernel_ms=round(km, 3), kernels_all_ms=round(ka, 3), d2h_bytes=d2h)
        print(json.dumps(r), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
