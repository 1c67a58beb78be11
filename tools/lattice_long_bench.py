"""Throughput of the lattice operations on long documents (the long-sentence path: nbest_long_kernel,
lattice_long_kernel): NBestEncode, SampleEncode at nbest 8 and -1, SampleEncodeAndScore and CalculateEntropy on batches
of 8 KB - 1 MB documents, in sentences/s and MB/s of input, with the same calls of the reference (oracle/_ref, one host
thread) when it is built.  Prints the card name and power limit first, since they are part of every number.

    python tools/lattice_long_bench.py [--sizes 8000,64000,256000,1000000] [--batch-bytes 2000000] [--nbest 64]
"""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

import corpus  # noqa: E402
from oracle import oracle_py  # noqa: E402


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                                       text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        import torch
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def documents(gen, kind, size, count, seed):
    docs = []
    for d in range(count):
        out, n = [], 0
        for s in gen.lines(kind, seed + d, size // 20 + 100):
            if n + len(s) + 1 > size:
                break
            out.append(s)
            n += len(s) + 1
        docs.append(b" ".join(out))
    return docs


def timed(f):
    t = time.perf_counter()
    f()
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="uni32k")
    ap.add_argument("--kind", default="en")
    ap.add_argument("--sizes", default="8000,64000,256000,1000000")
    ap.add_argument("--batch-bytes", type=int, default=2_000_000, help="input bytes per batch (at least one document)")
    ap.add_argument("--nbest", type=int, default=64)
    ap.add_argument("--nbest-max-size", type=int, default=256_000, help="largest document size for the n-best calls")
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()
    from sentencepiece_b200 import Engine
    mb = open(os.path.join(ROOT, "tests", "golden", "models", args.model + ".model"), "rb").read()
    eng = Engine(mb)
    ref = oracle_py.RefModel(mb) if oracle_py.ref_available() and not args.no_reference else None
    gen = corpus.CorpusGen()
    print(f"card: {card()}; model {args.model}/{args.kind}", flush=True)
    warm = oracle_py.pack(documents(gen, args.kind, 20_000, 2, 1))
    eng.nbest_encode(*warm, 8)
    eng.sample_encode(*warm, -1, 0.3)
    for size in [int(s) for s in args.sizes.split(",")]:
        docs = documents(gen, args.kind, size, max(1, args.batch_bytes // size), 500 + size % 997)
        buf, offs = oracle_py.pack(docs)
        mbytes = len(buf) / 1e6
        calls = [("sample -1", lambda: eng.sample_encode(buf, offs, -1, 0.3),
                  ref and (lambda: ref.sample_encode_batch(buf, offs, -1, 0.3, 1))),
                 ("sample_score x3", lambda: eng.sample_encode_and_score(buf, offs, 3, 0.3),
                  ref and (lambda: ref.sample_score_batch(buf, offs, 3, 0.3, 1))),
                 ("entropy", lambda: eng.calculate_entropy(buf, offs, 0.3),
                  ref and (lambda: ref.entropy_batch(buf, offs, 0.3)))]
        if size <= args.nbest_max_size:
            calls += [("sample 8", lambda: eng.sample_encode(buf, offs, 8, 0.3),
                       ref and (lambda: ref.sample_encode_batch(buf, offs, 8, 0.3, 1))),
                      (f"nbest {args.nbest}", lambda: eng.nbest_encode(buf, offs, args.nbest),
                       ref and (lambda: [ref.nbest_encode(d, args.nbest) for d in docs]))]
        for name, dev, host in calls:
            t = timed(dev)
            deferred = eng.info().last_deferred
            line = (f"{size:>8} B x {len(docs):>3}  {name:<16} device {len(docs) / t:9.2f} sent/s {mbytes / t:8.3f} MB/s "
                    f"(long path: {deferred})")
            if host:
                th = timed(host)
                line += f"  reference {len(docs) / th:9.2f} sent/s {mbytes / th:8.3f} MB/s"
            print(line, flush=True)
    eng.close()


if __name__ == "__main__":
    main()
