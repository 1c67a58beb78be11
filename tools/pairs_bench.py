"""Sentence pairs on the device (spm_encode_pairs_device) against what a caller does without them, the batch resident
in HBM:
  rerank: 1M pairs of bench.py's English corpus (sentence i with sentence 1M + i) on uni32k, template
          [CLS] A [SEP] B [SEP], w = 128, longest_first, ids and type ids;
  qa    : 20,000 short questions (bench.py's English sentences cut at 64 bytes) with 4 KB contexts (its sentences joined
          with spaces) on uni32k, the same template, w = 384, only_second with overflow windows, stride = 128, with
          character offsets.
Each is timed two ways:
  pairs : Engine.encode_device_pairs over the stacked batch;
  torch : two device encodes (spm_encode_ids_device, or spm_encode_offsets_device_padded at width 0 for offsets), one
          per member, then a vectorised torch assembly (the truncation or window plan, an index tensor per row and
          gathers for the ids, type ids and offsets).
Both must give identical tensors.  Wall time per call (host clock around calls that end in a device synchronise),
after a warm-up of both; the variants alternate for --reps rounds, median and min printed.  One JSON line per result,
the first with the GPU name and power limit read in the same run.
Needs an H100; writes nothing.
Usage: python tools/pairs_bench.py [--reps 5] [--n 1000000] [--qa 20000]"""
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
QA_SEED = 20261019
TEMPLATE = ((1,), (2,), (2,))  # [CLS] A [SEP] B [SEP] with uni32k's <s> / </s> ids


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def stats(ts):
    return {"median_ms": round(float(np.median(ts)), 3), "min_ms": round(float(np.min(ts)), 3)}


def packed(eng, d_bytes, d_offs):
    """spm_encode_ids_device of one member's batch -> (ids, starts int64 [n], lengths int64 [n]) on the device"""
    import torch
    n = d_offs.numel() - 1
    cap = int(d_bytes.numel()) + 1  # (a byte is at most one id)
    ids = torch.empty(cap, dtype=torch.int32, device="cuda")
    ido = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    eng.encode_device(d_bytes.data_ptr(), d_offs.data_ptr(), n, d_bytes.numel(), ids.data_ptr(), cap, ido.data_ptr(),
                      torch.cuda.current_stream().cuda_stream)
    return ids, ido[:-1], ido[1:] - ido[:-1]


def assemble(rp, fa, ca, fb, cb, A, B, w, pad, spans):
    """the rows prefix ++ A[fa, fa + ca) ++ middle ++ B[fb, fb + cb) ++ suffix of pairs rp; A / B = (ids, starts,
    lengths, spans or None) -> (ids, lengths, type_ids[, spans])"""
    import torch
    np_, nm, ns = (len(x) for x in TEMPLATE)
    tmpl = torch.tensor([i for x in TEMPLATE for i in x], dtype=torch.int32, device="cuda")
    k = torch.arange(w, device="cuda")[None, :]
    e2 = (np_ + ca)[:, None]
    e3 = e2 + nm
    e4 = e3 + cb[:, None]
    real = e4 + ns
    in_a = (k >= np_) & (k < e2)
    in_b = (k >= e3) & (k < e4)
    in_t = (k < real) & ~in_a & ~in_b
    qa = torch.where(in_a, A[1][rp][:, None] + fa[:, None] + k - np_, 0)
    qb = torch.where(in_b, B[1][rp][:, None] + fb[:, None] + k - e3, 0)
    qt = torch.where(k < np_, k, torch.where(k < e4, np_ + k - e2, np_ + nm + k - e4)).clamp(0, len(tmpl) - 1)
    ids = torch.where(in_a, A[0][qa], torch.where(in_b, B[0][qb], torch.where(in_t, tmpl[qt], pad)))
    types = ((k >= e3) & (k < real)).int()
    res = (ids.int(), real[:, 0].int(), types)
    if spans:
        sp = torch.where(in_a[..., None], A[3][qa], torch.where(in_b[..., None], B[3][qb], 0))
        res += (sp.int(),)
    return res


def torch_rerank(eng, d_bytes, d_offs, n, w):
    import torch
    A = packed(eng, d_bytes, d_offs[:n + 1]) + (None,)
    B = packed(eng, d_bytes, d_offs[n:]) + (None,)
    a, b = A[2], B[2]
    bt = w - sum(len(x) for x in TEMPLATE)
    ka = torch.minimum(a, torch.clamp(bt - b, min=(bt + 1) // 2))  # longest-first, closed form
    kb = torch.minimum(b, bt - ka)
    rp = torch.arange(n, device="cuda")
    zero = torch.zeros_like(a)
    ids, real, types = assemble(rp, zero, ka, zero, kb, A, B, w, -1, False)
    return ids, real, types, rp.int(), zero.int()


def torch_qa(eng, d_bytes, d_offs, n, w, stride):
    import torch

    def member(offs):
        pi, psp, pl = eng.encode_offsets_device_padded(d_bytes, offs, pad_id=-1, unit="char", eos_id=-1)
        W = pi.shape[1]
        return pi.reshape(-1), torch.arange(pl.numel(), device="cuda") * W, pl.long(), psp.reshape(-1, 2)
    A, B = member(d_offs[:n + 1]), member(d_offs[n:])
    a, b = A[2], B[2]
    room = w - sum(len(x) for x in TEMPLATE) - a
    step = room - stride
    m = torch.where(b <= room, 1, 1 + (torch.clamp(b - room, min=0) + step - 1) // step)
    rp = torch.repeat_interleave(torch.arange(n, device="cuda"), m)
    first = (torch.arange(len(rp), device="cuda") - (torch.cumsum(m, 0) - m)[rp]) * step[rp]
    cb = torch.minimum(b[rp] - first, room[rp])
    zero = torch.zeros_like(rp)
    ids, real, types, sp = assemble(rp, zero, a[rp], first, cb, A, B, w, -1, True)
    return ids, real, types, rp.int(), first.int(), sp


def compare_run(variants, reps):
    import torch
    res = {k: timed(f)[1] for k, f in variants.items()}
    same = all(torch.equal(x, y) for x, y in zip(res["pairs"], res["torch"]))
    times = {k: [] for k in variants}
    for _ in range(reps):
        for k, f in variants.items():
            times[k].append(timed(f)[0])
    out = {"rows": int(res["pairs"][0].shape[0]), "identical": same}
    for k in variants:
        out[k] = stats(times[k])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--qa", type=int, default=20000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import corpus
    from sentencepiece_b200 import Engine
    if not torch.cuda.is_available():
        raise SystemExit("pairs_bench needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    g = corpus.CorpusGen()
    mb = open(os.path.join(ROOT, "tests", "golden", "models", "uni32k.model"), "rb").read()
    eng = Engine(mb)
    p, m_, s = TEMPLATE
    # rerank / NLI: sentence i paired with sentence n + i of one seeded batch
    buf, offs = g.fill("en", CORPUS_SEED, 2 * a.n)
    d_bytes, d_offs = torch.from_numpy(buf).cuda(), torch.from_numpy(offs.view(np.int64)).cuda()
    w = 128
    variants = {
        "pairs": lambda: eng.encode_device_pairs(d_bytes, d_offs, p, m_, s, width=w, truncation="longest_first",
                                                 pad_id=-1),
        "torch": lambda: torch_rerank(eng, d_bytes, d_offs, a.n, w),
    }
    r = {"workload": "rerank", "model": "uni32k", "n_pairs": a.n, "w": w, "truncation": "longest_first",
         "offsets": None}
    r.update(compare_run(variants, a.reps))
    print(json.dumps(r), flush=True)
    del d_bytes, d_offs
    # extractive QA: short questions, 4 KB contexts
    qs = [x[:64] for x in g.lines("en", QA_SEED, a.qa)]
    lines = g.lines("en", QA_SEED + 1, a.qa * 4096 // 60)
    ctx, cur, j = [], [], 0
    for x in lines:
        cur.append(x)
        j += len(x) + 1
        if j > 4096:
            ctx.append(b" ".join(cur)[:4096])
            cur, j = [], 0
            if len(ctx) == a.qa:
                break
    assert len(ctx) == a.qa, len(ctx)
    items = qs + ctx
    buf = np.frombuffer(b"".join(items), np.uint8)
    offs = np.concatenate([[0], np.cumsum([len(x) for x in items])]).astype(np.int64)
    d_bytes, d_offs = torch.from_numpy(buf.copy()).cuda(), torch.from_numpy(offs).cuda()
    w, stride = 384, 128
    variants = {
        "pairs": lambda: eng.encode_device_pairs(d_bytes, d_offs, p, m_, s, width=w, truncation="only_second",
                                                 overflow=True, stride=stride, pad_id=-1, unit="char"),
        "torch": lambda: torch_qa(eng, d_bytes, d_offs, a.qa, w, stride),
    }
    r = {"workload": "qa", "model": "uni32k", "n_pairs": a.qa, "w": w, "truncation": "only_second", "stride": stride,
         "offsets": "char"}
    r.update(compare_run(variants, a.reps))
    print(json.dumps(r), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
