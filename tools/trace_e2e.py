"""Host-path traces of the fused path (SPM_B200_TRACE=1: timeline + per-phase cycles per warp) for the bench corpora.
usage: python tools/trace_e2e.py [model:kind ...]   (env: T threads per CTA)"""
import os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools"))
import corpus
from sentencepiece_b200 import Engine
g = corpus.CorpusGen()
todo = [a.split(":") for a in sys.argv[1:]] or [("uni32k", "en"), ("mix_bf8k", "mixed"), ("bpe32k", "en")]
for model, kind in todo:
    mb = open(os.path.join(ROOT, "tests", "golden", "models", model + ".model"), "rb").read()
    buf, offs = g.fill(kind, 20260922, 1_000_000)
    eng = Engine(mb)
    if os.environ.get("T"):
        eng.set_tuning(0, 0, int(os.environ["T"]))
    import torch
    pb = torch.from_numpy(buf).pin_memory().numpy(); po = torch.from_numpy(offs.view(np.int64)).pin_memory().numpy().view(np.uint64)
    for rep in range(4):
        if rep == 3: os.environ["SPM_B200_TRACE"] = "1"
        t0 = time.perf_counter()
        try:
            ids, ido = eng.encode_packed(pb, po, copy=False)
        except Exception as e:  # noqa: BLE001
            ids, ido = np.zeros(0), np.zeros(1)
            print("   (call failed:", str(e)[:80], ")")
        dt = time.perf_counter() - t0
        print(f"{model}/{kind} rep {rep}: {dt*1e3:.2f} ms, device kernel {eng.info().last_main_kernel_ms:.3f} ms, {len(offs)-1} sentences, {len(ids)} ids, bytes {int(offs[-1])}", flush=True)
    os.environ.pop("SPM_B200_TRACE", None)
    eng.close()
