"""Tuning sweep on an H100: encode-kernel time for the device-resident workload under different
kernels (lanes per sentence 1 or 32), CTA sizes and shared-memory caps.
usage: python tools/sweep.py [workload] [n] [lanes,threads,cap ...]"""
import itertools
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import corpus  # noqa: E402
from sentencepiece_b200 import Engine  # noqa: E402

workload = sys.argv[1] if len(sys.argv) > 1 else "uni32k:en"
n = int(sys.argv[2]) if len(sys.argv) > 2 else 1_000_000
configs = sys.argv[3:] or None
model, kind = workload.split(":")
mb = open(os.path.join(ROOT, "tests", "golden", "models", model + ".model"), "rb").read()
g = corpus.CorpusGen()
buf, offs = g.fill(kind, 20260922, n)
total = int(offs[-1])
dev = torch.device("cuda", 0)
d_bytes = torch.from_numpy(buf.copy()).to(dev)
d_offs = torch.from_numpy(offs.astype(np.int64)).to(dev)
cap = total + 4 * n + 1024
d_ids = torch.empty(cap, dtype=torch.int32, device=dev)
d_ido = torch.empty(n + 1, dtype=torch.int64, device=dev)
if configs:
    grid = [tuple(int(x) for x in c.split(",")) for c in configs]
else:
    grid = [(1, 512, 0), (1, 768, 0), (1, 1024, 0)]
ref = None
for G, thr, capn in grid:
    try:
        eng = Engine(mb)
        eng.set_tuning(G, capn, thr)
        ms = []
        for _ in range(4):
            tot = eng.encode_device(d_bytes.data_ptr(), d_offs.data_ptr(), n, total, d_ids.data_ptr(), cap,
                                    d_ido.data_ptr(), None)
            info = eng.info()
            ms.append(info.last_main_kernel_ms)
        chk = int(d_ids[:tot].to(torch.int64).sum().item())
        if ref is None:
            ref = (tot, chk)
        print(f"G={G:2d} threads={thr} ncap={capn}: main {min(ms[1:]):.3f} ms  all {info.last_kernel_ms:.3f} ms  "
              f"{n / min(ms[1:]) / 1e3:.1f} M sent/s  deferred={info.last_deferred} hot={info.trie_hot_units} "
              f"ids={tot} {'same' if (tot, chk) == ref else 'DIFFERENT RESULT'}", flush=True)
        eng.close()
    except Exception as e:
        print(f"G={G} threads={thr} ncap={capn}: {e}", flush=True)
