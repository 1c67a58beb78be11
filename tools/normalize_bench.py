"""spm_normalize on bench.py's seeded corpora at 1M sentences (uni32k/en, mix_bf8k/mixed), inputs in pinned host memory:
  normalize       : spm_normalize with_offsets = 0 (text only);
  normalize+n2o   : spm_normalize with_offsets = 1;
  encode_spans    : spm_encode_spans, the only way to the normalized text before spm_normalize (it also encodes);
  encode_ids      : spm_encode_ids, for scale.
End to end: a host clock around each C call, which returns with its results in pinned host memory.  Kernel: the
engine's own timings of the call (spm_engine_info: last_main_kernel_ms = the normalize kernels, last_kernel_ms = those
plus the packing scans and gathers, summed over the call's chunks), and the bytes each call copied back.  The check:
spm_normalize's text and norm_to_orig equal spm_encode_spans' wherever spans defines them, and the text is the same
without offsets.  Warm-up first, then the variants alternate for --reps rounds; median and min are printed.  One JSON
line per result, the first one with the GPU name and power limit.  Needs an H100; writes nothing.
Usage: python tools/normalize_bench.py [--n 1000000] [--reps 5]"""
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

CORPUS_SEED = 20260922  # bench.py's
WORKLOADS = [("uni32k", "en"), ("mix_bf8k", "mixed")]


def stats(ts):
    return {"median_ms": round(float(np.median(ts)), 3), "min_ms": round(float(np.min(ts)), 3)}


def calls(eng, buf, offs):
    """name -> zero-argument function running the C call once on the pinned batch"""
    L, h, n = eng._lib, eng._h, len(offs) - 1
    b, o = buf.ctypes.data, offs.ctypes.data
    p = [ctypes.c_void_p() for _ in range(6)]
    ref = [ctypes.byref(x) for x in p]

    def check(rc):
        if rc:
            raise RuntimeError(L.spm_last_error(h).decode())
    return {
        "normalize": lambda: check(L.spm_normalize(h, b, o, n, 0, *ref[:3])),
        "normalize+n2o": lambda: check(L.spm_normalize(h, b, o, n, 1, *ref[:3])),
        "encode_spans": lambda: check(L.spm_encode_spans(h, b, o, n, *ref)),
        "encode_ids": lambda: check(L.spm_encode_ids(h, b, o, n, *ref[:2])),
    }


def same_output(eng, buf, offs):
    text, no, n2o = eng.normalize(buf, offs, with_offsets=True)
    t2, no2, _ = eng.normalize(buf, offs)
    r = eng.encode_spans(buf, offs)
    lens = np.diff(no.astype(np.int64))
    keep = np.repeat(lens > 0, lens + 1)
    return bool(np.array_equal(no, r["norm_offsets"]) and text.tobytes() == r["normalized"] and
                np.array_equal(n2o[keep], r["n2o"][keep]) and np.array_equal(no2, no) and np.array_equal(t2, text))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import corpus
    from sentencepiece_b200 import Engine
    if not torch.cuda.is_available():
        raise SystemExit("normalize_bench needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    g = corpus.CorpusGen()
    for model, kind in WORKLOADS:
        mb = open(os.path.join(ROOT, "tests", "golden", "models", model + ".model"), "rb").read()
        buf, offs = g.fill(kind, CORPUS_SEED, a.n)
        buf = torch.from_numpy(np.ascontiguousarray(buf)).pin_memory().numpy()
        offs = torch.from_numpy(np.ascontiguousarray(offs).view(np.int64)).pin_memory().numpy().view(np.uint64)
        eng = Engine(mb)
        r = {"model": model, "kind": kind, "n": a.n, "input_bytes": int(offs[-1] - offs[0]),
             "identical_output": same_output(eng, buf, offs)}
        fns = calls(eng, buf, offs)
        for f in fns.values():  # warm-up: module loads, buffer growth
            f()
        ts = {k: [] for k in fns}
        info = {}
        for _ in range(a.reps):
            for k, f in fns.items():
                t0 = time.perf_counter()
                f()
                ts[k].append((time.perf_counter() - t0) * 1e3)
                i = eng.info()
                info[k] = {"kernel_ms": round(i.last_main_kernel_ms, 3), "kernels_and_packing_ms": round(i.last_kernel_ms, 3),
                           "d2h_bytes": int(i.last_d2h_bytes), "launches": int(i.last_kernel_launches)}
        for k in fns:
            r[k] = dict(stats(ts[k]), **info[k])
        print(json.dumps(r), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
