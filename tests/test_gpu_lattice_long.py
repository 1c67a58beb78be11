"""The lattice operations on sentences of any length: NBestEncode, SampleEncode with nbest_size > 1 and < 0,
SampleEncodeAndScore(wor=False) and CalculateEntropy on documents of 9 KB to 1 MB placed among short sentences, which
the lane kernels defer to nbest_long_kernel / lattice_long_kernel.  Short sentences follow the long ones, so the seeded
draws check that one generator walks the batch in sentence order across both paths.  Every n-best list (ids and score
bits), every seeded draw bit-exact against the oracle; entropies and sample scores within 2e-5.  The rule sets of
tests/charsmap_rules.py and the model families of tests/score_edges.py run with no sentence refused.  Needs an H100."""
import numpy as np
import pytest

import charsmap_rules as cr
import score_edges as se
from conftest import model_bytes
from oracle import modelproto as mp
from oracle import oracle_py
from refstore import digest
from refstore_long import reference

pytestmark = pytest.mark.gpu


def document(corpus_gen, kind, seed, size):
    """corpus lines joined by spaces, cut to `size` bytes at a line boundary"""
    out, n = [], 0
    for s in corpus_gen.lines(kind, seed, size // 20 + 100):
        if n + len(s) + 1 > size:
            break
        out.append(s)
        n += len(s) + 1
    return b" ".join(out)


def long_batch(corpus_gen, kind, seed, sizes):
    """short lines, then each long document followed by short lines: (lines, number of long documents)"""
    short = corpus_gen.lines(kind, seed, 12 * (len(sizes) + 1))
    lines = short[:12]
    for k, size in enumerate(sizes):
        lines += [document(corpus_gen, kind, seed + 1 + k, size)] + short[12 * (k + 1):12 * (k + 2)]
    return lines, len(sizes)


@pytest.fixture
def engine():
    from sentencepiece_b200 import Engine
    made = []

    def make(mb):
        made.append(Engine(mb))
        return made[-1]
    yield make
    for e in made:
        e.close()


def check_nbest(eng, om, lines, nbest, what):
    buf, offs = oracle_py.pack(lines)
    r = eng.nbest_encode(buf, offs, nbest)
    for i, s in enumerate(lines):
        cands, scores = om.nbest_encode(s, nbest)
        assert int(r["n_cands"][i]) == len(cands), (what, i)
        base = i * nbest
        for c, (ids, sc) in enumerate(zip(cands, scores)):
            a, b = int(r["cand_offsets"][base + c]), int(r["cand_offsets"][base + c + 1])
            assert r["ids"][a:b].tolist() == ids.tolist(), (what, i, c)
            assert np.float32(r["scores"][base + c]).view(np.uint32) == np.float32(sc).view(np.uint32), (what, i, c)


def assert_same(got, want, what):
    assert np.array_equal(np.asarray(got[1], np.uint64), np.asarray(want[1], np.uint64)), f"offsets differ: {what}"
    assert np.array_equal(got[0], want[0]), f"ids differ: {what}"


CASES = [("uni32k", "en"), ("mix_bf8k", "mixed")]


@pytest.mark.parametrize("model,kind", CASES)
def test_lattice_calls_on_long_documents(model, kind, corpus_gen, engine):
    """lattice sampling, SampleEncodeAndScore and entropy with 9 KB, 70 KB, 300 KB and 1 MB documents in the batch"""
    mb = model_bytes(model)
    lines, n_long = long_batch(corpus_gen, kind, 9300, [9_000, 70_000, 300_000, 1_000_000])
    buf, offs = oracle_py.pack(lines)
    om = oracle_py.OracleModel(mb)
    eng = engine(mb)
    eng.set_random_seed(4242)
    assert_same(eng.sample_encode(buf, offs, -1, 0.3), om.sample_encode_batch(buf, offs, -1, 0.3, 4242), "sample -1")
    assert eng.info().last_deferred == n_long
    ent = eng.calculate_entropy(buf, offs, 0.3)
    assert eng.info().last_deferred == n_long
    np.testing.assert_allclose(ent, om.entropy_batch(buf, offs, 0.3), rtol=2e-5, atol=2e-5)
    eng.set_random_seed(77)
    ids, co, sc = eng.sample_encode_and_score(buf, offs, 3, 0.2)
    oids, oco, osc = om.sample_score_batch(buf, offs, 3, 0.2, 77)
    assert np.array_equal(co, oco) and np.array_equal(ids, oids)
    np.testing.assert_allclose(sc, osc, rtol=2e-5, atol=2e-5)


@pytest.mark.parametrize("model,kind", CASES)
def test_nbest_on_long_documents(model, kind, corpus_gen, engine):
    """n-best lists at 2 (up to 300 KB), 64 (up to 70 KB) and 512 (9 KB: many agenda shrinks), seeded SampleEncode at
    nbest 8"""
    mb = model_bytes(model)
    om = oracle_py.OracleModel(mb)
    eng = engine(mb)
    for nbest, sizes in ((2, [9_000, 70_000, 300_000]), (64, [9_000, 70_000]), (512, [9_000])):
        lines, n_long = long_batch(corpus_gen, kind, 9400 + nbest, sizes)
        check_nbest(eng, om, lines, nbest, (model, nbest))
        assert eng.info().last_deferred >= n_long
    lines, n_long = long_batch(corpus_gen, kind, 9500, [9_000, 70_000])
    buf, offs = oracle_py.pack(lines)
    eng.set_random_seed(808)
    assert_same(eng.sample_encode(buf, offs, 8, 0.3), om.sample_encode_batch(buf, offs, 8, 0.3, 808), "sample 8")


def test_deep_keys_repeated():
    """the 100-byte key of test_gpu_normalizer_rules.py::test_deep_keys_size_the_lattice repeated 100 times: about 80 KB
    of normalized text, eight bytes per input byte, which the host sizes from the input length"""
    from sentencepiece_b200 import Engine
    mb = mp.replace_flags(model_bytes("uni32k"), charsmap=cr.blob("long_keys"))
    k = [k for k in cr.keys("long_keys") if len(k) == 100][0]
    lines = [b"a short one", k * 100, b"and after it"]
    buf, offs = oracle_py.pack(lines)
    om = oracle_py.OracleModel(mb)
    assert len(om.normalize(k * 100)[0]) > 80_000
    eng = Engine(mb)
    eng.set_random_seed(8081)
    assert_same(eng.sample_encode(buf, offs, -1, 0.3), om.sample_encode_batch(buf, offs, -1, 0.3, 8081), "sample -1")
    assert eng.info().last_deferred == 1
    np.testing.assert_allclose(eng.calculate_entropy(buf, offs, 0.3), om.entropy_batch(buf, offs, 0.3), rtol=2e-5,
                               atol=2e-5)
    check_nbest(eng, om, lines, 8, "deep keys")
    eng.close()


@pytest.mark.parametrize("name", [f.__name__ for f in se.UNIGRAM])
def test_score_edges_whole(name, engine):
    """the first 20 sentences of every unigram family and their first three words at nbest 2, 8, 16 and 64, one
    sentence per call: none refused"""
    fam = se.family(name)
    lines = fam.lines[:20]
    lines = lines + [b" ".join(s.split()[:3]) for s in lines]
    om = oracle_py.OracleModel(fam.model)
    eng = engine(fam.model)
    for nbest in (2, 8, 16, 64):
        for i, s in enumerate(lines):
            check_nbest(eng, om, [s], nbest, (name, nbest, i))


@pytest.mark.parametrize("name", cr.ALL)
def test_charsmaps_whole(name, corpus_gen, engine):
    """the first 40 corpus lines of every rule set at nbest 2 and 16 and seeded SampleEncode at 8, one sentence per
    call: none refused"""
    mb = mp.replace_flags(model_bytes("uni32k"), charsmap=cr.blob(name))
    om = oracle_py.OracleModel(mb)
    eng = engine(mb)
    for i, s in enumerate(cr.lines(name, corpus_gen, 5200, 800)[:40]):
        for nbest in (2, 16):
            check_nbest(eng, om, [s], nbest, (name, nbest, i))
        buf, offs = oracle_py.pack([s])
        eng.set_random_seed(8081 + i)
        assert_same(eng.sample_encode(buf, offs, 8, 0.3), om.sample_encode_batch(buf, offs, 8, 0.3, 8081 + i), (name, i))


def test_long_batch_vs_reference(corpus_gen, engine):
    """a batch with a 70 KB document against the digest of the reference's seeded lattice samples"""
    mb = model_bytes("uni32k")
    lines, _ = long_batch(corpus_gen, "en", 9600, [70_000])
    buf, offs = oracle_py.pack(lines)
    want = reference("gpu_lattice_long/sample/uni32k/en",
                     lambda: oracle_py.RefModel(mb).sample_encode_batch(buf, offs, -1, 0.5, 4711))
    eng = engine(mb)
    eng.set_random_seed(4711)
    assert digest(*eng.sample_encode(buf, offs, -1, 0.5)) == want
