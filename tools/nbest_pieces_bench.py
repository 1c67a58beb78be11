"""N-best and sampled pieces on the device against their ids calls, on bench.py's seeded corpus (config 5: 256k
sentences).  Best-of-N wall time per call of
  nbest    : spm_nbest_encode against spm_nbest_encode_pieces, uni32k/en at nbest_size 64 and uni32k/mixed at 16
             (nearly every mixed-script sentence holds an unknown run, so the normalized-text export runs);
  lattice  : spm_sample_encode_ids against spm_sample_encode_pieces at nbest_size -1 (the host draw), same corpora;
  class    : SentencePieceProcessor::NBestEncode(inputs, nbest_size, pieces) of the C++ host class on the first
             --class-n sentences, built from this tree and from --parent-tree (another checkout, already built),
             alternated in this process.
Every compared pair is checked for identical outputs: the ids, offsets, scores and candidate counts of the pieces calls
against the ids calls (the lattice pair under the same seed), and the class's pieces of both builds by hash.  Prints one
JSON line with the GPU name and power limit, then one per workload.  Needs an H100; writes only to a temporary
directory.
Usage: python tools/nbest_pieces_bench.py [--n 262144] [--class-n 32768] [--reps 3] [--parent-tree DIR]"""
import argparse
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
WORKLOADS = [("uni32k", "en", 64), ("uni32k", "mixed", 16)]


def best(fn, reps):
    out = fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return min(ts) * 1e3, out


def build_driver(tree, d, tag):
    """the class timing driver linked against the build in `tree`"""
    lib = os.path.join(tree, "sentencepiece_b200", "lib")
    exe = os.path.join(d, "class_bench_" + tag)
    subprocess.run(["g++", "-O2", "-std=c++17", "-pthread"] + (["-DHAS_PACKED"] if tag == "this" else []) + ["-I", os.path.join(tree, "sentencepiece_b200", "csrc"),
                    "-I", os.path.join(tree, "include"), os.path.join(ROOT, "tools", "nbest_pieces_class_bench.cc"),
                    os.path.join(lib, "sentencepiece_processor.o"), os.path.join(lib, "model_reader.o"),
                    "-L" + os.path.join(lib, "stdcxx"), "-L" + lib, "-lspm_b200", "-Wl,-rpath," + lib, "-o", exe], check=True)
    return exe


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=262144)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--class-n", type=int, default=32768)
    ap.add_argument("--parent-tree", default=None)
    a = ap.parse_args()
    import corpus
    from sentencepiece_b200 import Engine
    g = corpus.CorpusGen()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    with tempfile.TemporaryDirectory() as d:
        drivers = {"this": build_driver(ROOT, d, "this")}
        if a.parent_tree:
            drivers["parent"] = build_driver(os.path.abspath(a.parent_tree), d, "parent")
        for model, kind, nb in WORKLOADS:
            mpath = os.path.join(ROOT, "tests", "golden", "models", model + ".model")
            buf, offs = g.fill(kind, CORPUS_SEED, a.n)
            eng = Engine(open(mpath, "rb").read())
            r = {"model": model, "kind": kind, "n": a.n, "nbest_size": nb}
            r["nbest_ids_ms"], ids = best(lambda: eng.nbest_encode(buf, offs, nb), a.reps)
            r["nbest_pieces_ms"], pcs = best(lambda: eng.nbest_encode_pieces(buf, offs, nb), a.reps)
            i = eng.info()
            r["nbest_pieces_kernel_ms"], r["nbest_pieces_launches"] = i.last_kernel_ms, i.last_kernel_launches
            r["nbest_pieces_d2h_mb"] = i.last_d2h_bytes / 1e6
            r["nbest_identical"] = all(np.array_equal(ids[k], pcs[k]) for k in ("ids", "cand_offsets", "scores", "n_cands"))

            def seeded(fn):
                def run():
                    eng.set_random_seed(4242)
                    return fn()
                return run
            r["lattice_ids_ms"], lids = best(seeded(lambda: eng.sample_encode(buf, offs, -1, 0.5)), a.reps)
            r["lattice_pieces_ms"], lpcs = best(seeded(lambda: eng.sample_encode_pieces(buf, offs, -1, 0.5)), a.reps)
            r["lattice_identical"] = np.array_equal(lids[0], lpcs["ids"]) and np.array_equal(lids[1], lpcs["id_offsets"])
            eng.close()
            bf, of = os.path.join(d, "bytes"), os.path.join(d, "offs")
            cn = min(a.class_n, a.n)
            buf[:int(offs[cn])].tofile(bf)
            offs[:cn + 1].astype(np.uint64).tofile(of)
            r["class_n"] = cn
            res = {k: [] for k in drivers}
            for _ in range(2):  # alternated
                for k, exe in drivers.items():
                    out = subprocess.run([exe, mpath, bf, of, str(nb), str(a.reps)], capture_output=True, text=True,
                                         check=True).stdout.split()
                    res[k].append((float(out[0]), out[1]))
                    if len(out) > 2:
                        r["class_packed_call_this_ms"] = min(float(out[2]), r.get("class_packed_call_this_ms", 1e300))
            for k, v in res.items():
                r[f"class_nbest_pieces_{k}_ms"] = min(t for t, _ in v)
            hashes = {h for v in res.values() for _, h in v}
            r["class_identical"] = len(hashes) == 1
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
