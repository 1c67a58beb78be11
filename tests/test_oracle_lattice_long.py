"""Pins the oracle's lattice operations on long sentences against the reference (the digests of its results,
tests/refstore_long.py): n-best lists at 64 and 512 (ids and score bits; a long sentence shrinks the agenda many times),
seeded SampleEncode at nbest 8 and -1, and CalculateEntropy, on 9 KB, 70 KB (over 65,535 characters) and 300 KB
documents, English on uni32k and mixed-script on mix_bf8k.  tests/test_gpu_lattice_long.py compares the device with
the oracle on such documents.  CPU only."""
import pytest

from conftest import model_bytes
from oracle import oracle_py
from refstore import digest
from refstore_long import reference

SIZES = [9_000, 70_000, 300_000]
CASES = [("uni32k", "en"), ("mix_bf8k", "mixed")]


def document(corpus_gen, kind, seed, size):
    """corpus lines joined by spaces, cut to `size` bytes at a line boundary"""
    out, n = [], 0
    for s in corpus_gen.lines(kind, seed, size // 20 + 100):
        if n + len(s) + 1 > size:
            break
        out.append(s)
        n += len(s) + 1
    return b" ".join(out)


def batch(corpus_gen, kind):
    """the three documents, each followed by a short line"""
    lines = []
    for k, size in enumerate(SIZES):
        lines += [document(corpus_gen, kind, 9700 + k, size), corpus_gen.lines(kind, 9710 + k, 1)[0]]
    return lines


@pytest.mark.parametrize("model,kind", CASES)
def test_nbest_long_vs_reference(model, kind, corpus_gen):
    mb = model_bytes(model)
    docs = batch(corpus_gen, kind)[0::2]
    om = oracle_py.OracleModel(mb)
    for nbest, sizes in ((64, SIZES), (512, SIZES[:2])):
        for size, s in zip(SIZES, docs):
            if size not in sizes:
                continue
            want = reference(f"oracle_lattice_long/nbest/{model}/{kind}/{size}/{nbest}",
                             lambda: oracle_py.RefModel(mb).nbest_encode(s, nbest))
            got = om.nbest_encode(s, nbest)
            assert len(got[0]) == nbest
            assert digest(*got) == want, (size, nbest)


@pytest.mark.parametrize("model,kind", CASES)
def test_sampling_and_entropy_long_vs_reference(model, kind, corpus_gen):
    mb = model_bytes(model)
    buf, offs = oracle_py.pack(batch(corpus_gen, kind))
    om = oracle_py.OracleModel(mb)
    for nbest in (8, -1):
        want = reference(f"oracle_lattice_long/sample/{model}/{kind}/{nbest}",
                         lambda: oracle_py.RefModel(mb).sample_encode_batch(buf, offs, nbest, 0.3, 606))
        assert digest(*om.sample_encode_batch(buf, offs, nbest, 0.3, 606)) == want, nbest
    want = reference(f"oracle_lattice_long/entropy/{model}/{kind}",
                     lambda: oracle_py.RefModel(mb).entropy_batch(buf, offs, 0.3))
    assert digest(om.entropy_batch(buf, offs, 0.3)) == want
