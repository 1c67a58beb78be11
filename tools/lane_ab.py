"""A/B of the lane-kernel generations on an H100: ids must be identical, times are printed.

usage: python tools/lane_ab.py [model:kind ...] [--n N] [--variants "FW=0;FW=1;T=512"]
Each variant is a ';'-separated item of ','-separated KEY=VALUE knobs:
  FW whole-word shortcut (SPM_B200_FASTWORDS), S length ordering (SPM_B200_SORT), T threads per CTA,
  CR=1 empties the BPE word cache before every launch, C log2 of its entries (SPM_B200_BPE_CACHE).
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import corpus  # noqa: E402
from sentencepiece_b200 import Engine  # noqa: E402

ENV = {"FW": "SPM_B200_FASTWORDS", "C": "SPM_B200_BPE_CACHE", "S": "SPM_B200_SORT"}

ap = argparse.ArgumentParser()
ap.add_argument("workloads", nargs="*", default=["uni32k:en"])
ap.add_argument("--n", type=int, default=1_000_000)
ap.add_argument("--reps", type=int, default=4)
ap.add_argument("--variants", default="FW=0;FW=1")
args = ap.parse_args()

g = corpus.CorpusGen()
dev = torch.device("cuda", 0)
rc = 0
for wl in args.workloads:
    model, kind = wl.split(":")
    mb = open(os.path.join(ROOT, "tests", "golden", "models", model + ".model"), "rb").read()
    n = args.n
    buf, offs = g.fill(kind, 20260922, n)
    total = int(offs[-1])
    d_bytes = torch.from_numpy(buf.copy()).to(dev)
    d_offs = torch.from_numpy(offs.astype(np.int64)).to(dev)
    cap = total + 4 * n + 1024
    d_ids = torch.empty(cap, dtype=torch.int32, device=dev)
    d_ido = torch.empty(n + 1, dtype=torch.int64, device=dev)
    ref = None
    for variant in args.variants.split(";"):
        knobs = dict(kv.split("=") for kv in variant.split(",") if kv)
        for k in ENV.values():
            os.environ.pop(k, None)
        for k, v in knobs.items():
            if k in ENV:
                os.environ[ENV[k]] = v
        try:
            eng = Engine(mb)
            if "T" in knobs:
                eng.set_tuning(0, 0, int(knobs["T"]))
            ms = []
            for _ in range(args.reps):
                if knobs.get("CR") == "1":
                    eng.cache_reset()  # BPE: every launch starts with an empty word cache
                tot = eng.encode_device(d_bytes.data_ptr(), d_offs.data_ptr(), n, total, d_ids.data_ptr(), cap,
                                        d_ido.data_ptr(), None)
                info = eng.info()
                ms.append(info.last_main_kernel_ms)
            ids = d_ids[:tot].cpu().numpy()
            ido = d_ido.cpu().numpy()
            if ref is None:
                ref = (ids.copy(), ido.copy())
                same = "reference"
            else:
                ok = ids.shape == ref[0].shape and np.array_equal(ids, ref[0]) and np.array_equal(ido, ref[1])
                same = "same ids" if ok else "DIFFERENT IDS"
                if not ok:
                    rc = 1
                    bad = np.nonzero(np.diff(ido) != np.diff(ref[1]))[0]
                    print(f"   first sentences with a different id count: {bad[:5]}", flush=True)
            print(f"{wl} n={n} [{variant}]: main {min(ms[1:]):.3f} ms (first {ms[0]:.3f}) all {info.last_kernel_ms:.3f} ms "
                  f"{n / min(ms[1:]) / 1e3:.1f} M sent/s deferred={info.last_deferred} ids={tot} {same}", flush=True)
            eng.close()
        except Exception as e:  # noqa: BLE001
            rc = 1
            print(f"{wl} [{variant}]: FAILED {e}", flush=True)
sys.exit(rc)
