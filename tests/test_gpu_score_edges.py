"""Every scoring kernel on the model families of tests/score_edges.py, where float rounding and score ties decide the
ids: the unigram lane kernels with and without the whole-word shortcut, the general unigram and BPE kernels (ids and
spans), the deferred pass and the long-sentence kernels, the BPE lane2 kernel with and without its word cache, the
n-best lane kernel and the lattice kernel with the host sampler.  Ids and offsets bit-exact against the oracle (which
tests/test_oracle_score_edges.py pins to the reference); the default path also against the reference's digest.
Needs an H100."""
import re

import numpy as np
import pytest

import score_edges as se
from oracle import oracle_py
from refstore import digest, reference

pytestmark = pytest.mark.gpu
UNIGRAM = [f.__name__ for f in se.UNIGRAM]
BPE = [f.__name__ for f in se.BPE]
ALL = UNIGRAM + BPE
NBEST_LINES = 80
# The n-best kernel refuses some of these sentences ("exceeds the device path's capacity"): on an agenda shrink it
# rebuilds the heap but never compacts its hypothesis pool (the reference clones the surviving hypotheses into a fresh
# allocator, unigram_model.cc:483-505), so on lattices with many near-equal paths the pool runs out.  The tests accept
# that refusal and nothing else, sentence by sentence, and compare every sentence the kernel takes bit for bit.
CAPACITY = "exceeds the device path's capacity"
# (family, nbest) pairs the n-best kernel takes whole; elsewhere a refusal is accepted
NBEST_WHOLE = {(n, nb) for n in ("u_flat", "u_overflow", "u_nearword") for nb in (2, 8, 16, 64)} | \
              {("u_chain", 2), ("u_chain", 8)}


def nbest_lines(fam):
    """the first sentences of the corpus and, to keep the lattices small, their first three words"""
    lines = fam.lines[:NBEST_LINES]
    return lines + [b" ".join(s.split()[:3]) for s in lines]


_want = {}


def batch(name):
    fam = se.family(name)
    buf, offs = oracle_py.pack(fam.lines)
    if name not in _want:
        _want[name] = oracle_py.OracleModel(fam.model).encode_batch(buf, offs)
    return fam, buf, offs, _want[name]


@pytest.fixture
def engine(monkeypatch):
    """Engine(fam.model) with the environment variables `env` set; closed at teardown, also when the test fails"""
    from sentencepiece_b200 import Engine
    made = []

    def make(fam, **env):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        made.append(Engine(fam.model))
        return made[-1]
    yield make
    for e in made:
        e.close()


def assert_same(got, want, what):
    assert np.array_equal(np.asarray(got[1], np.uint64), np.asarray(want[1], np.uint64)), f"offsets differ: {what}"
    assert np.array_equal(got[0], want[0]), f"ids differ: {what}"


@pytest.mark.parametrize("name", ALL)
def test_default_path_vs_reference(name, engine):
    fam, buf, offs, want = batch(name)
    eng = engine(fam)
    got = eng.encode_packed(buf, offs)
    assert_same(got, want, name)
    assert digest(*got) == reference(f"score_edges/encode/{name}",
                                     lambda: oracle_py.RefModel(fam.model).encode_batch(buf, offs))


@pytest.mark.parametrize("name", UNIGRAM)
def test_unigram_lane_kernels(name, engine, monkeypatch, capfd):
    """SPM_B200_FASTWORDS=1: the lane kernel with the whole-word shortcut (its counters on stderr prove it ran; every
    family but U-userdef is eligible); =0: the plain lane kernel (no counters)"""
    fam, buf, offs, want = batch(name)
    monkeypatch.setenv("SPM_B200_KSTATS", "1")
    for force in ("1", "0"):
        eng = engine(fam, SPM_B200_FASTWORDS=force)
        capfd.readouterr()
        got = eng.encode_packed(buf, offs)
        err = capfd.readouterr().err
        assert_same(got, want, f"{name} SPM_B200_FASTWORDS={force}")
        whole_word_kernel = force == "1" and name != "u_userdef"
        assert ("[kstats] groups" in err) == whole_word_kernel, err
        if whole_word_kernel and name == "u_nearword":
            m = re.search(r"whole words ([0-9.]+)\)", err)
            assert m and float(m.group(1)) > 0, err


@pytest.mark.parametrize("name", ALL)
def test_general_kernels(name, engine):
    """set_tuning(32, 0, 0): the warp-per-sentence kernel (encode_unigram_kernel<false> / encode_bpe_kernel<false>);
    encode_spans: the spans instantiation (<true>), ids and token ends against the oracle's"""
    fam, buf, offs, want = batch(name)
    eng = engine(fam)
    eng.set_tuning(32, 0, 0)
    threads = 0
    if name == "u_chain":
        # 63 match slots per start: at the default CTA size the general kernels' per-warp tiles do not fit in shared
        # memory, and the engine says so instead of encoding; 128 threads (4 tiles) fit
        with pytest.raises(RuntimeError, match="shared-memory geometry does not fit"):
            eng.encode_packed(buf, offs)
        threads = 128
        eng.set_tuning(32, 0, threads)
    assert_same(eng.encode_packed(buf, offs), want, f"{name} general kernel")
    eng = engine(fam)
    if threads:
        eng.set_tuning(32, 0, threads)
    r = eng.encode_spans(buf, offs)
    om = oracle_py.OracleModel(fam.model)
    for i, s in enumerate(fam.lines):
        ids, te = om.encode(s)
        a, b = int(r["id_offsets"][i]), int(r["id_offsets"][i + 1])
        assert r["ids"][a:b].tolist() == ids.tolist(), (name, i)
        assert r["tok_end"][a:b].tolist() == te.tolist(), (name, i)


@pytest.mark.parametrize("name", ALL)
def test_deferred_and_long_sentences(name, engine):
    """sentences of about 600 bytes (past the lane kernels' cap: the deferred pass) and about 20 KB (the long kernels
    with HBM scratch) in one batch with the short ones"""
    fam = se.family(name)
    mid, long_ = b"", b""
    for s in fam.lines:
        if len(mid) < 600:
            mid += (b" " if mid else b"") + s
        long_ += (b" " if long_ else b"") + s
        if len(long_) >= 20000:
            break
    while len(long_) < 20000:
        long_ += b" " + long_
    lines = fam.lines[:100] + [mid[:620], long_[:20500]] + fam.lines[100:200]
    buf, offs = oracle_py.pack(lines)
    want = oracle_py.OracleModel(fam.model).encode_batch(buf, offs)
    eng = engine(fam)
    assert_same(eng.encode_packed(buf, offs), want, name)
    assert eng.info().last_deferred > 0


@pytest.mark.parametrize("name", BPE)
@pytest.mark.parametrize("cache", ["0", "8", None])
def test_bpe_word_cache(name, cache, engine):
    """the BPE lane2 kernel without the word cache, with a small one (2^8 entries: collisions) and with the default;
    each cold, then warm on the same engine"""
    fam, buf, offs, want = batch(name)
    eng = engine(fam, **({} if cache is None else {"SPM_B200_BPE_CACHE": cache}))
    for run in ("cold", "warm"):
        assert_same(eng.encode_packed(buf, offs), want, f"{name} SPM_B200_BPE_CACHE={cache} {run}")


@pytest.mark.parametrize("nbest", [2, 16, 64])
@pytest.mark.parametrize("name", UNIGRAM)
def test_nbest(name, nbest, engine):
    """n-best lists, one sentence per call: ids and score bits against the oracle, or the capacity refusal"""
    fam = se.family(name)
    om = oracle_py.OracleModel(fam.model)
    eng = engine(fam)
    compared = 0
    for i, s in enumerate(nbest_lines(fam)):
        buf, offs = oracle_py.pack([s])
        try:
            r = eng.nbest_encode(buf, offs, nbest)
        except RuntimeError as e:
            assert CAPACITY in str(e) and (name, nbest) not in NBEST_WHOLE, (i, str(e))
            continue
        cands, scores = om.nbest_encode(s, nbest)
        assert int(r["n_cands"][0]) == len(cands), i
        for c, (ids, sc) in enumerate(zip(cands, scores)):
            a, b = int(r["cand_offsets"][c]), int(r["cand_offsets"][c + 1])
            assert r["ids"][a:b].tolist() == ids.tolist(), (i, c)
            assert np.float32(r["scores"][c]).view(np.uint32) == np.float32(sc).view(np.uint32), (i, c)
        compared += 1
    assert compared > 0


@pytest.mark.parametrize("name", UNIGRAM)
def test_sample_nbest(name, engine):
    """seeded SampleEncode with nbest 8 (the n-best kernel + the host draw), one sentence per call, against the oracle
    with the same seed, or the capacity refusal"""
    fam = se.family(name)
    om = oracle_py.OracleModel(fam.model)
    eng = engine(fam)
    compared = 0
    for i, s in enumerate(nbest_lines(fam)):
        buf, offs = oracle_py.pack([s])
        eng.set_random_seed(8081 + i)
        try:
            ids, ido = eng.sample_encode(buf, offs, 8, 0.3)
        except RuntimeError as e:
            assert CAPACITY in str(e) and (name, 8) not in NBEST_WHOLE, (i, str(e))
            continue
        oids, oido = om.sample_encode_batch(buf, offs, 8, 0.3, 8081 + i)
        assert np.array_equal(ido, oido) and np.array_equal(ids, oids), i
        compared += 1
    assert compared > 0


@pytest.mark.parametrize("name", [n for n in UNIGRAM if n != "u_overflow"])
def test_lattice_sampling_and_entropy(name, engine):
    """seeded SampleEncode with nbest -1 (lattice kernel + host sampler) on the whole corpus; CalculateEntropy within
    float rounding (the device's exp / log differ from glibc's in the last place)"""
    fam = se.family(name)
    buf, offs = oracle_py.pack(fam.lines)
    om = oracle_py.OracleModel(fam.model)
    eng = engine(fam)
    eng.set_random_seed(8081)
    ids, ido = eng.sample_encode(buf, offs, -1, 0.3)
    oids, oido = om.sample_encode_batch(buf, offs, -1, 0.3, 8081)
    assert np.array_equal(ido, oido) and np.array_equal(ids, oids)
    ent = eng.calculate_entropy(buf, offs, 0.3)
    np.testing.assert_allclose(ent, om.entropy_batch(buf, offs, 0.3), rtol=2e-5, atol=2e-5)
