"""Every device normalizer (K1) on the rule sets of tests/charsmap_rules.py: the unigram lane kernels with and without
the whole-word shortcut, the general kernels at two shared-memory caps, the deferred pass and the long-sentence
kernels, the spans API (ids, token ends, normalized text, norm_to_orig), BPE lane2 and the general BPE kernel, n-best,
seeded sampling, lattice sampling and entropy, and the fused host path.  Every rule set runs under the default
normalizer flags and five variants on the encode paths, under three flag sets on n-best and the lattice.  Ids bit-exact
against the oracle (which tests/test_oracle_charsmaps.py pins to the reference).  Needs an H100."""
import numpy as np
import pytest

import charsmap_rules as cr
from conftest import model_bytes
from oracle import modelproto as mp
from oracle import oracle_py

pytestmark = pytest.mark.gpu
SEED, N = 5200, 800
FLAGS = list(zip(cr.FLAG_IDS, cr.FLAGS))
SAMPLE_FLAGS = [FLAGS[0], FLAGS[2], FLAGS[3]]  # default, keep_ws, no_escape
CAPACITY = "exceeds the device path's capacity"

_lines = {}


def corpus(name, corpus_gen):
    if name not in _lines:
        _lines[name] = cr.lines(name, corpus_gen, SEED, N)
    return _lines[name]


def model(base, name, flags):
    return mp.replace_flags(model_bytes(base), charsmap=cr.blob(name), **flags)


@pytest.fixture
def engine(monkeypatch):
    """Engine(mb) with the environment variables `env` set; closed at teardown, also when the test fails"""
    from sentencepiece_b200 import Engine
    made = []

    def make(mb, **env):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        made.append(Engine(mb))
        return made[-1]
    yield make
    for e in made:
        e.close()


def assert_same(got, want, what):
    assert np.array_equal(np.asarray(got[1], np.uint64), np.asarray(want[1], np.uint64)), f"offsets differ: {what}"
    assert np.array_equal(got[0], want[0]), f"ids differ: {what}"


def assert_spans(r, om, lines, what):
    for i, s in enumerate(lines):
        ids, te = om.encode(s)
        nrm, n2o = om.normalize(s)
        a, b = int(r["id_offsets"][i]), int(r["id_offsets"][i + 1])
        assert r["ids"][a:b].tolist() == ids.tolist(), (what, i)
        assert r["tok_end"][a:b].tolist() == te.tolist(), (what, i)
        na, nb = int(r["norm_offsets"][i]), int(r["norm_offsets"][i + 1])
        assert r["normalized"][na:nb] == nrm, (what, i)
        if len(nrm):
            assert r["n2o"][na + i: nb + i + 1].tolist() == n2o, (what, i)


@pytest.mark.parametrize("fid,flags", FLAGS, ids=cr.FLAG_IDS)
@pytest.mark.parametrize("name", cr.ALL)
def test_unigram_lane_kernels(name, fid, flags, corpus_gen, engine, monkeypatch, capfd):
    """SPM_B200_FASTWORDS=1: the lane kernel with the whole-word shortcut where the model is eligible (escaped
    whitespace, no suffix; its counters on stderr prove it ran); =0: the plain lane kernel"""
    mb = model("uni32k", name, flags)
    buf, offs = oracle_py.pack(corpus(name, corpus_gen))
    want = oracle_py.OracleModel(mb).encode_batch(buf, offs)
    monkeypatch.setenv("SPM_B200_KSTATS", "1")
    for force in ("1", "0"):
        eng = engine(mb, SPM_B200_FASTWORDS=force)
        capfd.readouterr()
        got = eng.encode_packed(buf, offs)
        err = capfd.readouterr().err
        assert_same(got, want, f"{name}/{fid} SPM_B200_FASTWORDS={force}")
        whole_word = force == "1" and flags.get("escape_whitespaces", True) and not flags.get("treat_whitespace_as_suffix")
        assert ("[kstats] groups" in err) == whole_word, err


@pytest.mark.parametrize("fid,flags", FLAGS, ids=cr.FLAG_IDS)
@pytest.mark.parametrize("name", cr.ALL)
def test_general_kernels_and_spans(name, fid, flags, corpus_gen, engine):
    """set_tuning(32, cap, 0): the warp-per-sentence kernel at the default cap and at 128 normalized bytes (more
    sentences go on to the long kernels); encode_spans: ids, token ends, normalized text and norm_to_orig"""
    mb = model("uni32k", name, flags)
    lines = corpus(name, corpus_gen)
    buf, offs = oracle_py.pack(lines)
    om = oracle_py.OracleModel(mb)
    want = om.encode_batch(buf, offs)
    for cap in (0, 128):
        eng = engine(mb)
        eng.set_tuning(32, cap, 0)
        assert_same(eng.encode_packed(buf, offs), want, f"{name}/{fid} general kernel, cap {cap}")
    assert_spans(engine(mb).encode_spans(buf, offs), om, lines, f"{name}/{fid}")


@pytest.mark.parametrize("fid,flags", FLAGS, ids=cr.FLAG_IDS)
@pytest.mark.parametrize("name", cr.ALL)
def test_bpe_kernels(name, fid, flags, corpus_gen, engine):
    """bpe32k: the BPE lane2 kernel (default tuning) and the general BPE kernel (set_tuning(32, 0, 0))"""
    mb = model("bpe32k", name, flags)
    buf, offs = oracle_py.pack(corpus(name, corpus_gen))
    want = oracle_py.OracleModel(mb).encode_batch(buf, offs)
    assert_same(engine(mb).encode_packed(buf, offs), want, f"{name}/{fid} BPE lane2")
    eng = engine(mb)
    eng.set_tuning(32, 0, 0)
    assert_same(eng.encode_packed(buf, offs), want, f"{name}/{fid} general BPE")


@pytest.mark.parametrize("base", ["uni32k", "bpe32k"])
@pytest.mark.parametrize("fid,flags", FLAGS, ids=cr.FLAG_IDS)
@pytest.mark.parametrize("name", cr.ALL)
def test_deferred_and_long_sentences(name, fid, flags, base, corpus_gen, engine):
    """sentences of about 600 bytes (past the lane kernels' cap: the deferred pass) and about 6 KB (past the general
    kernel's staging cap: the long kernels), in one batch with short ones"""
    lines = corpus(name, corpus_gen)
    mid, long_ = b" ".join(lines[:12])[:620], b" ".join(lines[:100])
    while len(long_) < 6000:
        long_ += b" " + long_
    lines = lines[:100] + [mid, long_[:6000]] + lines[100:200]
    buf, offs = oracle_py.pack(lines)
    mb = model(base, name, flags)
    eng = engine(mb)
    assert_same(eng.encode_packed(buf, offs), oracle_py.OracleModel(mb).encode_batch(buf, offs), f"{name}/{fid}")
    assert eng.info().last_deferred > 0


def deep_key_lines():
    """sentences made of the 66- and 100-byte keys, whose targets are more than 3x as long: KBs of input with no exact
    normalized length (past the general kernel's staging cap) go to the long kernels with scratch sized from the
    model's worst-case expansion"""
    ks = [k for k in cr.keys("long_keys") if len(k) in (66, 100)]
    return [k * (2600 // len(k)) for k in ks] + [b" ".join([k] * 30) for k in ks] + [b"a b", b""]


@pytest.mark.parametrize("base", ["uni32k", "bpe32k"])
def test_deep_keys_size_the_long_scratch(base, engine):
    mb = model(base, "long_keys", {})
    buf, offs = oracle_py.pack(deep_key_lines())
    om = oracle_py.OracleModel(mb)
    want = om.encode_batch(buf, offs)
    eng = engine(mb)
    assert_same(eng.encode_packed(buf, offs), want, base)
    assert eng.info().last_deferred >= 4
    r = eng.encode_spans(buf, offs)
    assert_spans(r, om, deep_key_lines(), base)


def test_deep_keys_size_the_lattice():
    """the lattice kernel's position buffer is sized from the worst-case expansion: one sentence of ten 100-byte keys
    normalizes to about 8 KB, 8 bytes per input byte"""
    from sentencepiece_b200 import Engine
    mb = model("uni32k", "long_keys", {})
    k = [k for k in cr.keys("long_keys") if len(k) == 100][0]
    buf, offs = oracle_py.pack([k * 10])
    om = oracle_py.OracleModel(mb)
    assert len(om.normalize(k * 10)[0]) > 8000
    eng = Engine(mb)
    eng.set_random_seed(8081)
    got = eng.sample_encode(buf, offs, -1, 0.3)
    assert_same(got, om.sample_encode_batch(buf, offs, -1, 0.3, 8081), "lattice sampling")
    np.testing.assert_allclose(eng.calculate_entropy(buf, offs, 0.3), om.entropy_batch(buf, offs, 0.3), rtol=2e-5,
                               atol=2e-5)
    eng.close()


def short_lines(name, om, corpus_gen, n):
    """n corpus lines whose normalized text fits the n-best and lattice kernels comfortably"""
    return [s for s in corpus(name, corpus_gen)[:300] if len(om.normalize(s)[0]) <= 400][:n]


@pytest.mark.parametrize("fid,flags", SAMPLE_FLAGS, ids=[f[0] for f in SAMPLE_FLAGS])
@pytest.mark.parametrize("name", cr.ALL)
def test_nbest_and_sample(name, fid, flags, corpus_gen, engine):
    """n-best lists at 2 and 16 and seeded SampleEncode at nbest 8, one sentence per call: ids and score bits against
    the oracle.  The n-best kernel may refuse a sentence for capacity (it does not compact its hypothesis pool); that
    refusal is accepted on at most a tenth of the sentences and nothing else is"""
    mb = model("uni32k", name, flags)
    om = oracle_py.OracleModel(mb)
    eng = engine(mb)
    lines = short_lines(name, om, corpus_gen, 40)
    refused = 0
    for i, s in enumerate(lines):
        buf, offs = oracle_py.pack([s])
        try:
            for nbest in (2, 16):
                r = eng.nbest_encode(buf, offs, nbest)
                cands, scores = om.nbest_encode(s, nbest)
                assert int(r["n_cands"][0]) == len(cands), (i, nbest)
                for c, (ids, sc) in enumerate(zip(cands, scores)):
                    a, b = int(r["cand_offsets"][c]), int(r["cand_offsets"][c + 1])
                    assert r["ids"][a:b].tolist() == ids.tolist(), (i, nbest, c)
                    assert np.float32(r["scores"][c]).view(np.uint32) == np.float32(sc).view(np.uint32), (i, nbest, c)
            eng.set_random_seed(8081 + i)
            got = eng.sample_encode(buf, offs, 8, 0.3)
        except RuntimeError as e:
            assert CAPACITY in str(e), (i, str(e))
            refused += 1
            continue
        assert_same(got, om.sample_encode_batch(buf, offs, 8, 0.3, 8081 + i), (name, fid, i))
    assert refused * 10 <= len(lines), f"{refused} of {len(lines)} sentences refused"


@pytest.mark.parametrize("fid,flags", SAMPLE_FLAGS, ids=[f[0] for f in SAMPLE_FLAGS])
@pytest.mark.parametrize("name", cr.ALL)
def test_lattice_sampling_and_entropy(name, fid, flags, corpus_gen, engine):
    """seeded SampleEncode with nbest -1 (lattice kernel + host sampler); CalculateEntropy within float rounding"""
    mb = model("uni32k", name, flags)
    om = oracle_py.OracleModel(mb)
    lines = short_lines(name, om, corpus_gen, 120)
    buf, offs = oracle_py.pack(lines)
    eng = engine(mb)
    eng.set_random_seed(8081)
    assert_same(eng.sample_encode(buf, offs, -1, 0.3), om.sample_encode_batch(buf, offs, -1, 0.3, 8081), name)
    np.testing.assert_allclose(eng.calculate_entropy(buf, offs, 0.3), om.entropy_batch(buf, offs, 0.3), rtol=2e-5,
                               atol=2e-5)


def test_fused_host_path(corpus_gen, engine, capfd):
    """a batch of more than 300k sentences takes the fused host path (one kernel, streamed input); nfkc_cf on uni32k"""
    mb = model("uni32k", "nfkc_cf", {})
    lines = cr.transform(corpus_gen.lines("en", 5300, 320_000), cr.keys("nfkc_cf"), 5300)
    buf, offs = oracle_py.pack(lines)
    eng = engine(mb, SPM_B200_TRACE="1")
    capfd.readouterr()
    got = eng.encode_packed(buf, offs)
    assert "[trace] fused kernel done" in capfd.readouterr().err
    assert_same(got, oracle_py.OracleModel(mb).encode_batch(buf, offs), "fused host path")


def user_symbol_models():
    """USER_DEFINED pieces that overlap rule keys: `ﬁx` against nmt_nfkc's rule for `ﬁ` (uni32k's own charsmap), and
    `thx`, `abc`, `zzz`-style pieces against the ascii_keys and ladder rules"""
    out = []
    for base in ("uni32k", "bpe32k"):
        m = mp.parse_model(model_bytes(base))
        pieces = list(zip(m["pieces"], m["scores"], m["types"]))
        have = set(m["pieces"])
        users = ["ﬁx", "thx", "abc", "the.", "zzz", "zzzzzq", "Ⅷx"]
        pieces += [(u.encode(), 0.0, mp.USER_DEFINED) for u in users if u.encode() not in have]
        for name in (None, "ascii_keys", "ladder"):
            kw = {} if name is None else dict(charsmap=cr.blob(name))
            out.append((base, name, mp.replace_flags(model_bytes(base), pieces=pieces, **kw)))
    return out


def user_symbol_lines(corpus_gen):
    ks = [u.encode() for u in ("ﬁx", "ﬁ", "thx", "abc", "the.", "zzz", "zzzzzq", "Ⅷx", "the", "th", "a", "zz")]
    return cr.transform(corpus_gen.lines("en", 5400, 1500), ks, 5400) + cr.edge_lines(ks) + \
        [b"\xef\xac\x81x", b"\xef\xac\x81", b"\xef\xac\x81xx \xef\xac\x81 x", b"thxthe.abcd", b"zzzzzzzzq", b"abcx"]


def test_user_symbols_win_over_rules(corpus_gen, engine):
    """a user symbol is matched before the charsmap (normalizer.cc:201-205): the plain lane kernel, the general kernel
    and the spans API on uni32k, the general BPE kernel on bpe32k"""
    lines = user_symbol_lines(corpus_gen)
    buf, offs = oracle_py.pack(lines)
    models = user_symbol_models()
    om = oracle_py.OracleModel(models[0][2])  # uni32k with nmt_nfkc: `ﬁ` alone folds to `fi`, `ﬁx` stays
    assert om.normalize("ﬁ ﬁx".encode())[0] == "▁fi▁ﬁx".encode()
    for base, name, mb in models:
        om = oracle_py.OracleModel(mb)
        want = om.encode_batch(buf, offs)
        what = f"{base}/{name}"
        if base == "uni32k":
            assert_same(engine(mb, SPM_B200_FASTWORDS="0").encode_packed(buf, offs), want, f"{what} plain lane")
            eng = engine(mb)
            eng.set_tuning(32, 0, 0)
            assert_same(eng.encode_packed(buf, offs), want, f"{what} general")
            assert_spans(engine(mb).encode_spans(buf, offs), om, lines, what)
        else:
            eng = engine(mb)
            eng.set_tuning(32, 0, 0)
            assert_same(eng.encode_packed(buf, offs), want, f"{what} general BPE")
