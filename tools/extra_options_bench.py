"""Cost of the encode frame (SetEncodeExtraOptions "bos:eos") on bench.py's headline batch: 1M English sentences,
uni32k.  Times, per step:
  host : spm_encode_ids with the frame written by the engine, against the plain call plus the framing a C ABI caller
         does on the host (a vectorised numpy pass over the returned ids: new offsets, P / S, body copy);
  device: spm_encode_ids_device with the frame, against the plain call plus a framing pass on the device
         (torch index ops into a second buffer).
Prints one JSON line with the GPU name and power limit.  Needs an H100; writes nothing into the tree.
Usage: python tools/extra_options_bench.py [--n 1000000] [--reps 10]"""
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

CORPUS_SEED = 20240607  # any fixed seed; the batch only has to be the same for every arm


def frame_host(ids, ido, p, s):
    n = len(ido) - 1
    c = np.diff(ido.astype(np.int64))
    F = len(p) + len(s)
    no = ido.astype(np.int64) + np.arange(n + 1, dtype=np.int64) * F
    out = np.empty(int(no[-1]), dtype=np.int32)
    for k, v in enumerate(p):
        out[no[:-1] + k] = v
    for k, v in enumerate(s):
        out[no[1:] - len(s) + k] = v
    sid = np.repeat(np.arange(n), c)
    out[no[sid] + len(p) + (np.arange(len(ids), dtype=np.int64) - ido[sid].astype(np.int64))] = ids
    return out, no


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    import torch
    import corpus
    from sentencepiece_b200 import Engine, _modelinfo
    mb = open(os.path.join(ROOT, "tests", "golden", "models", "uni32k.model"), "rb").read()
    sp = _modelinfo.special_pieces(mb)
    P, S = [sp["bos_id"]], [sp["eos_id"]]
    buf, offs = corpus.CorpusGen().fill("en", CORPUS_SEED, a.n)
    eng = Engine(mb)
    n = a.n

    def best(fn):
        fn()
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            fn()
            ts.append(time.perf_counter() - t0)
        return min(ts) * 1e3, float(np.median(ts)) * 1e3

    res = {}
    eng.set_encode_frame()
    res["host_plain_ms"] = best(lambda: eng.encode_packed(buf, offs, copy=False))
    res["host_plain_plus_host_framing_ms"] = best(lambda: frame_host(*eng.encode_packed(buf, offs, copy=False), P, S))
    eng.set_encode_frame(P, False, S)
    res["host_engine_frame_ms"] = best(lambda: eng.encode_packed(buf, offs, copy=False))
    framed = eng.encode_packed(buf, offs)
    eng.set_encode_frame()
    ref = frame_host(*eng.encode_packed(buf, offs), P, S)
    assert np.array_equal(framed[0], ref[0]) and np.array_equal(framed[1], ref[1].astype(np.uint64))

    d_bytes = torch.from_numpy(buf.copy()).cuda()
    d_offs = torch.from_numpy(offs.astype(np.int64)).cuda()
    tot = int(framed[1][-1])
    d_ids = torch.empty(tot + 16, dtype=torch.int32, device="cuda")
    d_ido = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    d_out = torch.empty(tot + 16, dtype=torch.int32, device="cuda")
    ar = torch.arange(n + 1, device="cuda", dtype=torch.int64)
    Pt, St = torch.tensor(P, device="cuda", dtype=torch.int32), torch.tensor(S, device="cuda", dtype=torch.int32)

    def dev():
        return eng.encode_device(d_bytes.data_ptr(), d_offs.data_ptr(), n, len(buf), d_ids.data_ptr(), tot + 16, d_ido.data_ptr())

    def dev_plus_framing():
        t = dev()
        no = d_ido + ar * (len(P) + len(S))
        c = d_ido[1:] - d_ido[:-1]
        sid = torch.repeat_interleave(torch.arange(n, device="cuda"), c, output_size=t)
        d_out[no[:-1]] = Pt[0]
        d_out[no[1:] - 1] = St[0]
        d_out[no[sid] + len(P) + torch.arange(t, device="cuda") - d_ido[sid]] = d_ids[:t]
        torch.cuda.synchronize()

    eng.set_encode_frame()
    res["device_plain_ms"] = best(dev)
    res["device_plain_plus_device_framing_ms"] = best(dev_plus_framing)
    eng.set_encode_frame(P, False, S)
    res["device_engine_frame_ms"] = best(dev)
    assert np.array_equal(d_ids[:tot].cpu().numpy(), framed[0])
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"what": "bos:eos frame on %d sentences, uni32k; (best, median) ms of %d steps" % (n, a.reps),
                      "gpu": gpu, **res}))
    eng.close()


if __name__ == "__main__":
    main()
