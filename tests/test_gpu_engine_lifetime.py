"""Destroying an engine gives its device memory back.  Twenty uni32k engines in turn each run every entry point once --
encode of a small batch and of a 300k-sentence batch (the chunked host path), spans, pieces, decode of both batches
(the second through the pipelined decode), n-best, the three sampling modes and entropy, on a batch with documents
far longer than the lane kernels take, so that the n-best and lattice calls also run their long-sentence jobs -- and
are destroyed.  The device's free memory must come back to where it was, within a tolerance far below what one
engine holds.  Needs an H100."""
import numpy as np
import pytest

from conftest import model_bytes
from oracle import oracle_py

pytestmark = pytest.mark.gpu

CYCLES = 20
# device memory the CYCLES engines together may leave behind: a few of the driver's 2 MiB allocation pages
TOLERANCE = 16 << 20


def batches(corpus_gen):
    short = corpus_gen.lines("en", 901, 60)
    # documents of a few KB: longer than the 512 normalized bytes a lane kernel takes, so they become long jobs
    docs = [b" ".join(corpus_gen.lines("en", 902 + k, 60)) for k in range(3)]
    lines = short[:20] + [docs[0]] + short[20:40] + [docs[1]] + short[40:] + [docs[2]]
    return oracle_py.pack(lines), corpus_gen.fill("en", 905, 300_000)


def run_every_entry_point(eng, small, large):
    buf, offs = small
    ids, ido = eng.encode_packed(buf, offs)
    eng.encode_spans(buf, offs)
    eng.encode_pieces(buf, offs)
    eng.decode_packed(ids, ido)
    big_ids, big_ido = eng.encode_packed(*large)
    eng.decode_packed(big_ids, big_ido)
    eng.nbest_encode(buf, offs, 4)
    assert eng.info().last_deferred >= 3, "the documents did not take the long n-best path"
    eng.sample_encode(buf, offs, 4, 0.5)
    eng.sample_encode(buf, offs, -1, 0.5)
    eng.sample_encode_and_score(buf, offs, 2, 0.5)
    eng.calculate_entropy(buf, offs, 0.5)
    assert eng.info().last_deferred >= 3, "the documents did not take the long lattice path"


def test_destroy_returns_device_memory(corpus_gen):
    import torch
    from sentencepiece_b200 import Engine

    mb = model_bytes("uni32k")
    small, large = batches(corpus_gen)

    def cycle():
        eng = Engine(mb)
        eng.set_random_seed(7)
        run_every_entry_point(eng, small, large)
        held = torch.cuda.mem_get_info()[0]
        eng.close()
        return held

    cycle()  # the first engine loads the kernels, which stay with the process
    start = torch.cuda.mem_get_info()[0]
    footprint = start - cycle()
    assert footprint > 8 * TOLERANCE, f"one engine holds only {footprint >> 20} MiB: too little to tell a leak from noise"
    for _ in range(CYCLES - 1):
        cycle()
    left = start - torch.cuda.mem_get_info()[0]
    print(f"one engine holds {footprint >> 20} MiB; {CYCLES} engines left {left / 2**20:.1f} MiB behind")
    assert left <= TOLERANCE, f"{CYCLES} engines left {left >> 20} MiB behind (one engine holds {footprint >> 20} MiB)"
