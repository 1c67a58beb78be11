"""EncodeAsPieces on the device (spm_encode_pieces, K9) against what it replaces, on bench.py's seeded corpora at 1M
sentences: uni32k/en, bpe32k/en, mix_bf8k/mixed (byte pieces) and uni32k/mixed (many unknown runs, so the
unknown-surface path).  Best-of-N wall time per call of
  ids      : spm_encode_ids (the lane kernels / fused host path);
  pieces   : spm_encode_pieces, sep = -1 and sep = ' ';
  spans    : spm_encode_spans alone (the device half of the old pieces path; its host half built one string per token
             on top of this);
  cli      : spm_encode_b200 --output_format=piece on a file of the same sentences (one --batch_lines batch).
plus the fraction of sentences that took the unknown-surface detour and the engine's kernel times (spm_engine_info).
Prints one JSON line per workload and one with the GPU name and power limit.  Needs an H100; writes only to a
temporary directory.
Usage: python tools/pieces_bench.py [--n 1000000] [--reps 5]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

CORPUS_SEED = 20260922  # bench.py's
WORKLOADS = [("uni32k", "en"), ("bpe32k", "en"), ("mix_bf8k", "mixed"), ("uni32k", "mixed")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import corpus
    from sentencepiece_b200 import Engine
    g = corpus.CorpusGen()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    cli = os.path.join(ROOT, "sentencepiece_b200", "lib", "spm_encode_b200")
    for model, kind in WORKLOADS:
        mpath = os.path.join(ROOT, "tests", "golden", "models", model + ".model")
        mb = open(mpath, "rb").read()
        buf, offs = g.fill(kind, CORPUS_SEED, a.n)
        eng = Engine(mb)
        L = eng._lib
        bp, op = buf.ctypes.data, offs.ctypes.data
        vp = ctypes.c_void_p

        def best(fn):
            fn()
            ts = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                fn()
                ts.append(time.perf_counter() - t0)
            return min(ts) * 1e3

        def ids():
            o = [vp() for _ in range(2)]
            eng._check(L.spm_encode_ids(eng._h, bp, op, a.n, *[ctypes.byref(x) for x in o]))

        def pieces(sep):
            def run():
                o = [vp() for _ in range(5)]
                eng._check(L.spm_encode_pieces(eng._h, bp, op, a.n, None, 0, sep, *[ctypes.byref(x) for x in o]))
            return run

        def spans():
            o = [vp() for _ in range(6)]
            eng._check(L.spm_encode_spans(eng._h, bp, op, a.n, *[ctypes.byref(x) for x in o]))

        r = {"model": model, "kind": kind, "n": a.n}
        r["ids_ms"] = best(ids)
        r["pieces_ms"] = best(pieces(-1))
        i = eng.info()
        r["pieces_kernel_ms"] = i.last_kernel_ms
        r["pieces_main_kernel_ms"] = i.last_main_kernel_ms
        r["pieces_launches"] = i.last_kernel_launches
        r["unk_detour_fraction"] = i.last_unk_detour / a.n
        r["pieces_d2h_mb"] = i.last_d2h_bytes / 1e6
        r["pieces_sep_ms"] = best(pieces(ord(" ")))
        r["spans_ms"] = best(spans)
        i = eng.info()
        r["spans_kernel_ms"] = i.last_kernel_ms
        r["spans_d2h_mb"] = i.last_d2h_bytes / 1e6
        eng.close()
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "in.txt")
            raw = buf.tobytes()
            o = offs.tolist()
            with open(path, "wb") as f:
                f.write(b"".join(raw[o[k]:o[k + 1]] + b"\n" for k in range(a.n)))
            args = [cli, f"--model={mpath}", "--output_format=piece", f"--input={path}", f"--output={os.path.join(d, 'out.txt')}",
                    f"--batch_lines={a.n}"]
            subprocess.run(args, check=True)
            t0 = time.perf_counter()
            subprocess.run(args, check=True)
            r["cli_piece_s"] = time.perf_counter() - t0
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
