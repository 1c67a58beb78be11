"""Padded rows with offsets on the device against what a caller does without them, on bench.py's seeded corpora at 1M
sentences (uni32k/en, mix_bf8k/mixed, bpe32k/en), the batch resident in HBM:
  (a) ids      : spm_encode_ids_device_padded at width 0, ids only (the floor);
  (b) bytes    : spm_encode_offsets_device_padded, byte offsets;
  (c) chars    : the same with SPM_OFFSETS_CHARS;
  (d) host     : the batch copied to the host, spm_encode_offsets, processor.unicode_spans, rows padded in numpy and
                 uploaded (ids and character offsets).
Per-call wall time (host clock around calls that end in a device synchronise) and the engine's kernel time.  The
variants are warmed up, then alternate for --reps rounds; median and min are printed, with a check that (b) and (d)
give the ids of (a) and that (c) and (d) give identical offsets.  One JSON line per result, the first one with the
GPU name and power limit.  Needs an H100; writes nothing.
Usage: python tools/padded_offsets_bench.py [--n 1000000] [--reps 5]"""
import argparse
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
WORKLOADS = [("uni32k", "en"), ("mix_bf8k", "mixed"), ("bpe32k", "en")]


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def stats(ts):
    return {"median_ms": round(float(np.median(ts)), 3), "min_ms": round(float(np.min(ts)), 3)}


def host_rows(eng, d_bytes, d_offs, eos_id, pad):
    """(d): what a caller does today for ids and character offsets of a device batch"""
    import torch
    from sentencepiece_b200.processor import unicode_spans
    buf = d_bytes.cpu().numpy()
    offs = d_offs.cpu().numpy().view(np.uint64)
    r = eng.encode_offsets(buf, offs, eos_id=eos_id, pieces=False)
    cb, ce = unicode_spans(buf, offs, r["begin"], r["end"], r["id_offsets"])
    ido = r["id_offsets"].astype(np.int64)
    lens = np.diff(ido)
    n, w = len(lens), int(lens.max(initial=0))
    mask = np.arange(w)[None, :] < lens[:, None]
    ids = np.full((n, w), pad, np.int32)
    ids[mask] = r["ids"]
    spans = np.zeros((n, w, 2), np.int32)
    spans[mask] = np.stack([cb, ce], axis=-1)
    return torch.from_numpy(ids).cuda(), torch.from_numpy(spans).cuda(), torch.from_numpy(lens.astype(np.int32)).cuda()


def run(eng, d_bytes, d_offs, eos_id, reps):
    import torch
    variants = {
        "ids": lambda: eng.encode_device_padded(d_bytes, d_offs, pad_id=-1),
        "bytes": lambda: eng.encode_offsets_device_padded(d_bytes, d_offs, pad_id=-1, eos_id=eos_id),
        "chars": lambda: eng.encode_offsets_device_padded(d_bytes, d_offs, pad_id=-1, unit="char", eos_id=eos_id),
        "host": lambda: host_rows(eng, d_bytes, d_offs, eos_id, -1),
    }
    res = {k: timed(f)[1] for k, f in variants.items()}  # warm-up of every shape, and the results compared
    a, b, c, d = res["ids"], res["bytes"], res["chars"], res["host"]
    same = bool(torch.equal(a[0], b[0]) and torch.equal(a[1], b[2]) and torch.equal(a[0], c[0]) and
                torch.equal(a[0], d[0]) and torch.equal(a[1], d[2]) and torch.equal(c[1], d[1]))
    times = {k: [] for k in variants}
    kern = {k: [] for k in variants}
    for _ in range(reps):
        for k, f in variants.items():
            times[k].append(timed(f)[0])
            kern[k].append(eng.info().last_kernel_ms)
    out = {"width0": int(a[0].shape[1]), "identical": same}
    for k in variants:
        out[k] = dict(stats(times[k]), engine_kernels_ms=round(float(np.median(kern[k])), 3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import corpus
    from sentencepiece_b200 import Engine, _modelinfo
    if not torch.cuda.is_available():
        raise SystemExit("padded_offsets_bench needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    g = corpus.CorpusGen()
    for model, kind in WORKLOADS:
        mb = open(os.path.join(ROOT, "tests", "golden", "models", model + ".model"), "rb").read()
        buf, offs = g.fill(kind, CORPUS_SEED, a.n)
        d_bytes = torch.from_numpy(buf).cuda()
        d_offs = torch.from_numpy(offs.view(np.int64)).cuda()
        eng = Engine(mb)
        r = {"model": model, "kind": kind, "n": a.n}
        r.update(run(eng, d_bytes, d_offs, _modelinfo.special_pieces(mb)["eos_id"], a.reps))
        print(json.dumps(r), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
