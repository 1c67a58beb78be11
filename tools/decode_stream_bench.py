"""Streaming decode (spm_decode_stream_device) against what a serving loop does without it, the ids resident in HBM:
each of n sequences is T ids long (bench.py's corpus encoded and concatenated per row, uni32k / English and mix_bf8k /
mixed), and the ids arrive as generation emits them:
  one  : one id per row per call, an int64 [n, 1] column slice of the [n, T] output tensor;
  multi: 1-8 ids per row per call (speculative decoding), an int64 [n, 8] slice with per-row lengths.
Each is run two ways:
  stream : Engine.decode_stream_device, the state of every row on the device;
  prefix : today's way, spm_decode_ids_device of every row's whole prefix at every call, the new text taken as the
           part after the previous call's text.
Per-call wall time (host clock; every call returns after its text has reached the host) gives the median and p99, and
all ids over the summed time give ids/s.  Both ways must end in the same texts (the stream's are checked against
spm_decode_ids of the whole rows).  One JSON line per result, the first with the GPU name and power limit read in the
same run.  Needs an H100; writes nothing.
Usage: python tools/decode_stream_bench.py [--T 1024] [--ns 256,4096] [--modes one,multi] [--ways stream,prefix]"""
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
PLAN_SEED = 20261019


def rows_of(eng, corpus_gen, kind, n, T):
    """[n, T] int64 ids: the corpus encoded and concatenated, cut into rows of T ids"""
    need, got, parts = n * T, 0, []
    chunk = 0
    while got < need:
        buf, offs = corpus_gen.fill(kind, CORPUS_SEED + chunk, 50000)
        ids, _ = eng.encode_packed(buf, offs)
        parts.append(ids)
        got += len(ids)
        chunk += 1
    return np.concatenate(parts)[:need].astype(np.int64).reshape(n, T)


def plan(mode, n, T):
    """per call, the number of ids every row gets: [calls, n] int32"""
    if mode == "one":
        return np.ones((T, n), np.int32)
    rng = np.random.default_rng(PLAN_SEED)
    steps = rng.integers(1, 9, size=(T, n)).astype(np.int32)  # more calls than needed; cut below
    cum = np.cumsum(steps, axis=0)
    steps = np.clip(steps - np.maximum(cum - T, 0), 0, None).astype(np.int32)
    last = int(np.nonzero(steps.any(axis=1))[0].max()) + 1
    return steps[:last]


def run(eng, d_ids, P, way):
    """-> (per-call ms list, final texts)"""
    import torch
    n, T = d_ids.shape
    K = int(P.max())
    pad = torch.zeros((n, K), dtype=torch.int64, device="cuda")
    d_ids = torch.cat([d_ids, pad], dim=1)  # so that every [n, K] slice exists
    pos = np.zeros(n, np.int64)
    d_lens = [torch.from_numpy(p).cuda() for p in P]
    times = []
    if way == "stream":
        st = torch.zeros((n, 16), dtype=torch.uint8, device="cuda")
        out = [[] for _ in range(n)]
        uniform = bool((P == P[0:1]).all())
        for c, p in enumerate(P):
            final = torch.ones(n, dtype=torch.int32, device="cuda") if c == len(P) - 1 else None
            if uniform:  # every row at the same position: one column slice
                j = int(pos[0])
                t = d_ids[:, j:j + K]
            else:
                # rows at different positions: a gather into [n, K] (part of the serving loop's work)
                idx = torch.from_numpy(pos[:, None] + np.arange(K)[None, :]).cuda()
                t = torch.gather(d_ids, 1, idx)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            texts = eng.decode_stream_device(t, st, lengths=d_lens[c], final=final)
            times.append((time.perf_counter() - t0) * 1e3)
            for i, x in enumerate(texts):
                if x:
                    out[i].append(x)
            pos += p
        return times, ["".join(o) for o in out]
    prev = [""] * n
    upto = np.zeros(n, np.int64)
    for c, p in enumerate(P):
        upto += p
        d_upto = torch.from_numpy(upto.astype(np.int32)).cuda()
        Lmax = int(upto.max())
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        texts = eng.decode_device(d_ids[:, :Lmax], lengths=d_upto)
        _ = [texts[i][len(prev[i]):] for i in range(n)]  # the new text of every row
        times.append((time.perf_counter() - t0) * 1e3)
        prev = texts
    return times, prev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=1024)
    ap.add_argument("--ns", default="256,4096")
    ap.add_argument("--modes", default="one,multi")
    ap.add_argument("--ways", default="stream,prefix")
    a = ap.parse_args()
    import torch
    import corpus
    from sentencepiece_b200 import Engine
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"gpu": gpu, "T": a.T}), flush=True)
    g = corpus.CorpusGen()
    for model, kind in (("uni32k", "en"), ("mix_bf8k", "mixed")):
        with open(os.path.join(ROOT, "tests", "golden", "models", model + ".model"), "rb") as f:
            eng = Engine(f.read())
        nmax = max(int(x) for x in a.ns.split(","))
        all_rows = rows_of(eng, g, kind, nmax, a.T)
        for n in (int(x) for x in a.ns.split(",")):
            rows = all_rows[:n]
            ido = np.arange(n + 1, dtype=np.uint64) * a.T
            text, to = eng.decode_packed(rows.astype(np.int32).ravel(), ido)
            raw = text.tobytes()
            want = [raw[int(to[i]):int(to[i + 1])].decode("utf-8", errors="replace") for i in range(n)]
            d_ids = torch.from_numpy(rows).cuda()
            for mode in a.modes.split(","):
                P = plan(mode, n, a.T)
                finals = {}
                for way in a.ways.split(","):
                    run(eng, d_ids, P[:8], way)  # warm-up
                    times, final = run(eng, d_ids, P, way)
                    finals[way] = final
                    tot = float(np.sum(times))
                    print(json.dumps({"model": model, "kind": kind, "n": n, "T": a.T, "mode": mode, "way": way,
                                      "calls": len(P), "median_ms": round(float(np.median(times)), 4),
                                      "p99_ms": round(float(np.percentile(times, 99)), 4),
                                      "total_s": round(tot / 1e3, 3), "ids_per_s": round(n * a.T / (tot / 1e3)),
                                      "texts_equal_decode_ids": final == want}), flush=True)
                if len(finals) == 2:
                    print(json.dumps({"model": model, "n": n, "mode": mode,
                                      "stream_equals_prefix": finals["stream"] == finals["prefix"]}), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
