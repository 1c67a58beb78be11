"""spm_encode_offsets on bench.py's seeded corpora at 1M sentences (uni32k/en, bpe32k/en, mix_bf8k/mixed), inputs in
pinned host memory:
  encode_ids        : spm_encode_ids, for scale;
  offsets           : spm_encode_offsets without pieces (ids + begin / end);
  offsets+pieces    : spm_encode_offsets with pieces (as spm_encode_pieces writes them);
  spans+numpy       : the route without this call: spm_encode_spans, then begin / end derived from its tok_end,
                      normalized text and norm_to_orig in numpy (offsets_from_spans).
End to end: a host clock around each call; the C calls return with their results in pinned host memory, the spans
route includes its Python copies and the numpy pass.  Kernel: the engine's own timings (spm_engine_info:
last_main_kernel_ms, last_kernel_ms) and the bytes each call copied back.  The check: all routes give the same ids,
begin and end, and the pieces equal spm_encode_pieces'.  Warm-up first, then the variants alternate for --reps rounds;
median and min are printed.  One JSON line per result, the first one with the GPU name and power limit.  Needs an H100;
writes nothing.
Usage: python tools/offsets_bench.py [--n 1000000] [--reps 5]"""
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
WORKLOADS = [("uni32k", "en"), ("bpe32k", "en"), ("mix_bf8k", "mixed")]
BYTE = 6  # SPM_BYTE


def offsets_from_spans(r, types):
    """begin / end of every token from Engine.encode_spans' result (no encode frame), as spm_encode_offsets returns
    them: n2o at the token's start and end in the normalized text; byte-fallback tokens of one character all begin at
    the character and only the last one ends after it."""
    ids = r["ids"]
    if len(ids) == 0:
        return np.zeros(0, np.uint32), np.zeros(0, np.uint32)
    te = r["tok_end"].astype(np.int64)
    ido = r["id_offsets"].astype(np.int64)
    no = r["norm_offsets"].astype(np.int64)
    n = len(ido) - 1
    cnt = np.diff(ido)
    sent = np.repeat(np.arange(n), cnt)
    first = np.zeros(len(ids), bool)
    first[ido[:-1][cnt > 0]] = True
    start = np.where(first, 0, np.roll(te, 1))
    base = (no[:-1] + np.arange(n))[sent]
    n2o = r["n2o"]
    b, e = n2o[base + start], n2o[base + te]
    byte = np.asarray(types)[ids] == BYTE
    norm = np.frombuffer(r["normalized"], np.uint8)
    at = np.minimum(no[:-1][sent] + start, max(len(norm) - 1, 0))
    cont = byte & ((norm[at] & 0xC0) == 0x80) if len(norm) else np.zeros(len(ids), bool)
    head = np.maximum.accumulate(np.where(cont, 0, np.arange(len(ids))))
    b = b[head]
    e = np.where(byte & np.append(cont[1:], False), b, e)
    return b.astype(np.uint32), e.astype(np.uint32)


def stats(ts):
    return {"median_ms": round(float(np.median(ts)), 3), "min_ms": round(float(np.min(ts)), 3)}


def calls(eng, buf, offs, types):
    """name -> zero-argument function running the route once on the pinned batch"""
    L, h, n = eng._lib, eng._h, len(offs) - 1
    b, o = buf.ctypes.data, offs.ctypes.data
    p = [ctypes.c_void_p() for _ in range(7)]
    ref = [ctypes.byref(x) for x in p]

    def check(rc):
        if rc:
            raise RuntimeError(L.spm_last_error(h).decode())
    return {
        "encode_ids": lambda: check(L.spm_encode_ids(h, b, o, n, *ref[:2])),
        "offsets": lambda: check(L.spm_encode_offsets(h, b, o, n, -1, None, 0, -1, *ref[:4], None, None, None)),
        "offsets+pieces": lambda: check(L.spm_encode_offsets(h, b, o, n, -1, None, 0, -1, *ref)),
        "spans+numpy": lambda: offsets_from_spans(eng.encode_spans(buf, offs), types),
    }


def same_output(eng, buf, offs, types):
    r = eng.encode_offsets(buf, offs)
    q = eng.encode_offsets(buf, offs, pieces=False)
    ids, ido = eng.encode_packed(buf, offs)
    pc = eng.encode_pieces(buf, offs)
    sb, se = offsets_from_spans(eng.encode_spans(buf, offs), types)
    same = [np.array_equal(x["ids"], ids) and np.array_equal(x["id_offsets"], ido) for x in (r, q)]
    same += [np.array_equal(r[k], q[k]) for k in ("begin", "end")]
    same += [np.array_equal(r["begin"], sb), np.array_equal(r["end"], se)]
    same += [np.array_equal(r[k], pc[k]) for k in ("text", "text_offsets", "piece_end")]
    return bool(all(same))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    import corpus
    from oracle import modelproto
    from sentencepiece_b200 import Engine
    if not torch.cuda.is_available():
        raise SystemExit("offsets_bench needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    g = corpus.CorpusGen()
    for model, kind in WORKLOADS:
        mb = open(os.path.join(ROOT, "tests", "golden", "models", model + ".model"), "rb").read()
        types = np.asarray(modelproto.parse_model(mb)["types"], np.uint8)
        buf, offs = g.fill(kind, CORPUS_SEED, a.n)
        buf = torch.from_numpy(np.ascontiguousarray(buf)).pin_memory().numpy()
        offs = torch.from_numpy(np.ascontiguousarray(offs).view(np.int64)).pin_memory().numpy().view(np.uint64)
        eng = Engine(mb)
        r = {"model": model, "kind": kind, "n": a.n, "input_bytes": int(offs[-1] - offs[0]),
             "identical_output": same_output(eng, buf, offs, types)}
        fns = calls(eng, buf, offs, types)
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
                info[k] = {"kernel_ms": round(i.last_main_kernel_ms, 3), "kernels_all_ms": round(i.last_kernel_ms, 3),
                           "d2h_bytes": int(i.last_d2h_bytes), "launches": int(i.last_kernel_launches),
                           "unk_detour": int(i.last_unk_detour)}
        for k in fns:
            r[k] = dict(stats(ts[k]), **info[k])
        print(json.dumps(r), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
