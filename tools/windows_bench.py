"""Overlapping windows on the device (spm_encode_windows_device) against what a caller does without them, the batch
resident in HBM:
  en1m  : 1M sentences of bench.py's English corpus on uni32k at w = 64, stride = 16 (most sentences fit: the cost
          over the padded call), ids only;
  doc64k: 2,000 seeded 64 KB documents (bench.py's English generator) on uni32k at w = 512, stride = 128, ids only
          and with character offsets.
Each is timed three ways:
  windows : Engine.encode_device_windows;
  torch   : the packed source on the device (spm_encode_ids_device; for offsets, spm_encode_offsets_device_padded at
            width 0) and a torch windowing gather (the window plan, a repeat, an index tensor and a gather);
  host    : copy the batch to the host, spm_encode_ids / spm_encode_offsets (+ unicode_spans), cut the windows in
            numpy and upload them.
The three must give identical tensors.  Wall time per call (host clock around calls that end in a device
synchronise), after a warm-up of every variant; the variants alternate for --reps rounds, median and min printed.
One JSON line per result, the first with the GPU name and power limit.  --padded-only times just the padded calls
(ids and character offsets at w = 64) whose kernels the windows share code with, so that two builds of the
project can be compared.
Needs an H100; writes nothing.
Usage: python tools/windows_bench.py [--reps 5] [--docs 2000]"""
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
DOC_SEED = 20261018


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def stats(ts):
    return {"median_ms": round(float(np.median(ts)), 3), "min_ms": round(float(np.min(ts)), 3)}


def plan(xp, starts, lens, w, stride, np_, ns):
    """the window plan over framed lists src[starts[i] : starts[i] + lens[i]] -> (row_sentence, row_first, body, src
    index [R, w], valid [R, w]); xp is numpy or torch"""
    fr = np_ + ns
    B = w - fr
    step = B - stride
    L = lens - fr
    m = xp.where(L <= B, 1, 1 + (xp.clip(L - B, 0, None) + step - 1) // step)
    if xp is np:
        rs = np.repeat(np.arange(len(L)), m)
        cum = np.cumsum(m) - m
        first = (np.arange(len(rs)) - np.repeat(cum, m)) * step
        k = np.arange(w)[None, :]
    else:
        import torch
        rs = torch.repeat_interleave(torch.arange(len(L), device=L.device), m)
        cum = torch.cumsum(m, 0) - m
        first = (torch.arange(len(rs), device=L.device) - cum[rs]) * step
        k = torch.arange(w, device=L.device)[None, :]
    body = xp.minimum(L[rs] - first, xp.full_like(first, B) if xp is not np else B)
    real = body + fr
    valid = k < real[:, None]
    src = xp.where(k < np_, k, xp.where(k < np_ + body[:, None], k + first[:, None], k + (L[rs] - body)[:, None]))
    src = src + starts[rs][:, None]
    return rs, first, real, xp.where(valid, src, 0), valid


def torch_windows(eng, d_bytes, d_offs, w, stride, np_, ns, eos_id, chars):
    import torch
    n = d_offs.numel() - 1
    if not chars:
        cap = int(d_bytes.numel()) + n * (np_ + ns) + 1  # (a byte is at most one id)
        ids = torch.empty(cap, dtype=torch.int32, device="cuda")
        ido = torch.empty(n + 1, dtype=torch.int64, device="cuda")
        eng.encode_device(d_bytes.data_ptr(), d_offs.data_ptr(), n, d_bytes.numel(), ids.data_ptr(), cap,
                          ido.data_ptr(), torch.cuda.current_stream().cuda_stream)
        starts, lens = ido[:-1], ido[1:] - ido[:-1]
        src_ids, src_sp = ids, None
    else:
        pi, psp, pl = eng.encode_offsets_device_padded(d_bytes, d_offs, pad_id=-1, unit="char", eos_id=eos_id)
        W = pi.shape[1]
        starts = torch.arange(n, device="cuda", dtype=torch.int64) * W
        lens = pl.long()
        src_ids, src_sp = pi.reshape(-1), psp.reshape(-1, 2)
    rs, first, real, src, valid = plan(torch, starts, lens, w, stride, np_, ns)
    out = torch.where(valid, src_ids[src], torch.full_like(src, -1, dtype=torch.int32))
    res = (out.int(), real.int(), rs.int(), first.int())
    if chars:
        res += (torch.where(valid[..., None], src_sp[src], 0).int(),)
    return res


def host_windows(eng, d_bytes, d_offs, w, stride, np_, ns, eos_id, chars):
    import torch
    from sentencepiece_b200.processor import unicode_spans
    buf = d_bytes.cpu().numpy()
    offs = d_offs.cpu().numpy().view(np.uint64)
    if chars:
        r = eng.encode_offsets(buf, offs, eos_id=eos_id, pieces=False)
        ids, ido = r["ids"], r["id_offsets"].astype(np.int64)
        cb, ce = unicode_spans(buf, offs, r["begin"], r["end"], r["id_offsets"])
    else:
        ids, ido = eng.encode_packed(buf, offs)
        ido = ido.astype(np.int64)
    rs, first, real, src, valid = plan(np, ido[:-1], np.diff(ido), w, stride, np_, ns)
    res = [np.where(valid, ids[src], -1).astype(np.int32), real.astype(np.int32), rs.astype(np.int32),
           first.astype(np.int32)]
    if chars:
        res.append(np.where(valid[..., None], np.stack([cb[src], ce[src]], -1), 0).astype(np.int32))
    return tuple(torch.from_numpy(x).cuda() for x in res)


def compare_run(eng, d_bytes, d_offs, w, stride, np_, ns, eos_id, chars, reps):
    import torch
    unit = "char" if chars else None
    variants = {
        "windows": lambda: eng.encode_device_windows(d_bytes, d_offs, w, stride=stride, pad_id=-1, unit=unit,
                                                     eos_id=eos_id),
        "torch": lambda: torch_windows(eng, d_bytes, d_offs, w, stride, np_, ns, eos_id, chars),
        "host": lambda: host_windows(eng, d_bytes, d_offs, w, stride, np_, ns, eos_id, chars),
    }
    res = {k: timed(f)[1] for k, f in variants.items()}
    same = all(torch.equal(a, b) and torch.equal(a, c)
               for a, b, c in zip(res["windows"], res["torch"], res["host"]))
    times = {k: [] for k in variants}
    for _ in range(reps):
        for k, f in variants.items():
            times[k].append(timed(f)[0])
    out = {"rows": int(res["windows"][0].shape[0]), "identical": same}
    for k in variants:
        out[k] = stats(times[k])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--docs", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--padded-only", action="store_true")
    a = ap.parse_args()
    import torch
    import corpus
    from sentencepiece_b200 import Engine, _modelinfo
    from sentencepiece_b200.processor import extra_frame
    if not torch.cuda.is_available():
        raise SystemExit("windows_bench needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    g = corpus.CorpusGen()
    mb = open(os.path.join(ROOT, "tests", "golden", "models", "uni32k.model"), "rb").read()
    sp = _modelinfo.special_pieces(mb)
    eng = Engine(mb)
    prefix, rev, suffix = extra_frame(["bos", "eos"], sp["bos_id"], sp["eos_id"])
    eng.set_encode_frame(prefix, rev, suffix)
    buf, offs = g.fill("en", CORPUS_SEED, a.n)
    d_bytes, d_offs = torch.from_numpy(buf).cuda(), torch.from_numpy(offs.view(np.int64)).cuda()
    if a.padded_only:
        variants = {"padded_ids_w64": lambda: eng.encode_device_padded(d_bytes, d_offs, width=64, pad_id=-1,
                                                                        truncate=True),
                    "padded_chars_w64": lambda: eng.encode_offsets_device_padded(
                        d_bytes, d_offs, width=64, pad_id=-1, truncate=True, unit="char", eos_id=sp["eos_id"])}
        for f in variants.values():
            timed(f)
        times = {k: [] for k in variants}
        for _ in range(a.reps):
            for k, f in variants.items():
                times[k].append(timed(f)[0])
        print(json.dumps({"workload": "uni32k/en", "n": a.n, **{k: stats(v) for k, v in times.items()}}), flush=True)
        return
    r = {"workload": "en1m", "model": "uni32k", "n": a.n, "w": 64, "stride": 16, "offsets": None}
    r.update(compare_run(eng, d_bytes, d_offs, 64, 16, 1, 1, sp["eos_id"], False, a.reps))
    print(json.dumps(r), flush=True)
    del d_bytes, d_offs
    # 64 KB documents: bench.py's English sentences joined with spaces, cut at 65,536 bytes
    lines = g.lines("en", DOC_SEED, a.docs * 65536 // 60)
    docs, cur, j = [], [], 0
    for s in lines:
        cur.append(s)
        j += len(s) + 1
        if j > 65536:  # (the joined document is j - 1 bytes)
            docs.append(b" ".join(cur)[:65536])
            cur, j = [], 0
            if len(docs) == a.docs:
                break
    assert len(docs) == a.docs, len(docs)
    buf = np.frombuffer(b"".join(docs), np.uint8)
    offs = np.concatenate([[0], np.cumsum([len(d) for d in docs])]).astype(np.int64)
    assert (np.diff(offs) == 65536).all()
    d_bytes, d_offs = torch.from_numpy(buf.copy()).cuda(), torch.from_numpy(offs).cuda()
    for chars in (False, True):
        r = {"workload": "doc64k", "model": "uni32k", "n": a.docs, "w": 512, "stride": 128,
             "offsets": "char" if chars else None}
        r.update(compare_run(eng, d_bytes, d_offs, 512, 128, 1, 1, sp["eos_id"], chars, max(a.reps - 2, 3)))
        print(json.dumps(r), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
