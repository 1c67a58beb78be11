"""Padded id tensors on the device against what a caller does without them, on bench.py's seeded corpora at 1M
sentences (uni32k/en, mix_bf8k/mixed), the batch resident in HBM:
  packed+torch : spm_encode_ids_device, then the obvious torch packed-to-padded pass (lengths from the offsets, the
                 longest row read back, a mask, a scatter);
  padded0      : spm_encode_ids_device_padded at width 0 (the longest row);
  padded64     : the same at a fixed width of 64 with truncation.
Per-call wall time (host clock around calls that end in a device synchronise), the engine's kernel times, and a check
that the three give the same rows.  Decode: a generation-shaped int64 [4096, 512] tensor with eos at random positions
and garbage after it, decode_device(stop_id=eos) against .cpu() + a cut at eos + DecodeIds.  Warm-up first, then the
variants alternate for --reps rounds; median and min are printed.  One JSON line per result, the first one with the
GPU name and power limit.  Needs an H100; writes nothing.
Usage: python tools/tensor_io_bench.py [--n 1000000] [--reps 7]"""
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
WORKLOADS = [("uni32k", "en"), ("mix_bf8k", "mixed")]


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def stats(ts):
    return {"median_ms": round(float(np.median(ts)), 3), "min_ms": round(float(np.min(ts)), 3)}


def encode_rows(eng, d_bytes, d_offs, reps):
    import torch
    n = d_offs.numel() - 1
    cap = 2 * d_bytes.numel() + 8 * n + 1024
    d_ids = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_ido = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    col = None

    def packed_torch():
        nonlocal col
        tot = eng.encode_device(d_bytes.data_ptr(), d_offs.data_ptr(), n, d_bytes.numel(), d_ids.data_ptr(), cap,
                                d_ido.data_ptr())
        lens = d_ido[1:] - d_ido[:-1]
        w = int(lens.max())
        if col is None or col.numel() < w:
            col = torch.arange(max(w, 1), device="cuda")
        out = torch.full((n, w), -1, dtype=torch.int32, device="cuda")
        out[col[:w][None, :] < lens[:, None]] = d_ids[:tot]
        return out, lens.int()

    variants = {
        "packed+torch": packed_torch,
        "padded0": lambda: eng.encode_device_padded(d_bytes, d_offs, pad_id=-1),
        "padded64": lambda: eng.encode_device_padded(d_bytes, d_offs, width=64, pad_id=-1, truncate=True),
    }
    results = {k: timed(f)[1] for k, f in variants.items()}  # warm-up of every shape, and the rows compared
    a, la = results["packed+torch"]
    b, lb = results["padded0"]
    c, lc = results["padded64"]
    w = a.shape[1]
    a64 = a[:, :64] if w >= 64 else torch.nn.functional.pad(a, (0, 64 - w), value=-1)
    same = bool(torch.equal(a, b) and torch.equal(la, lb) and torch.equal(a64, c) and torch.equal(torch.clamp(la, max=64), lc))
    times = {k: [] for k in variants}
    kern = {k: [] for k in variants}
    for _ in range(reps):
        for k, f in variants.items():
            times[k].append(timed(f)[0])
            i = eng.info()
            kern[k].append((i.last_kernel_ms, i.last_main_kernel_ms))
    out = {"width0": w, "identical_rows": same}
    for k in variants:
        out[k] = dict(stats(times[k]), engine_kernels_ms=round(float(np.median([x[0] for x in kern[k]])), 3),
                      encode_kernel_ms=round(float(np.median([x[1] for x in kern[k]])), 3))
    return out


def decode_rows(sp, reps, rows=4096, T=512):
    import torch
    eng = sp.engine
    vocab = eng.info().vocab_size
    eos = sp._specials()["eos_id"]
    rng = np.random.default_rng(11)
    gen = rng.integers(3, vocab, size=(rows, T), dtype=np.int64)
    stops = rng.integers(1, T, size=rows)
    for i, p in enumerate(stops):
        gen[i, p] = eos
        gen[i, p + 1:] = rng.integers(-2 ** 40, 2 ** 40, size=T - p - 1)  # garbage after eos
    g = torch.from_numpy(gen).cuda()

    def host():
        h = g.cpu().numpy()
        lists = []
        for r in h:
            hit = np.flatnonzero(r == eos)
            lists.append(r[:hit[0] if len(hit) else T].tolist())
        return sp.DecodeIds(lists)

    def device():
        return eng.decode_device(g, stop_id=eos)

    same = timed(host)[1] == timed(device)[1]
    th, td = [], []
    for _ in range(reps):
        th.append(timed(host)[0])
        td.append(timed(device)[0])
    return {"rows": rows, "T": T, "identical_text": same, "cpu+DecodeIds": stats(th), "decode_device": stats(td),
            "decode_device_kernels_ms": round(eng.info().last_kernel_ms, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    import torch
    import corpus
    from sentencepiece_b200 import Engine, SentencePieceProcessor
    if not torch.cuda.is_available():
        raise SystemExit("tensor_io_bench needs a CUDA device")
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
        r.update(encode_rows(eng, d_bytes, d_offs, a.reps))
        print(json.dumps(r), flush=True)
        eng.close()
    sp = SentencePieceProcessor(model_proto=open(os.path.join(ROOT, "tests", "golden", "models", "uni32k.model"),
                                                 "rb").read())
    print(json.dumps(dict(model="uni32k", decode=decode_rows(sp, a.reps))), flush=True)


if __name__ == "__main__":
    main()
