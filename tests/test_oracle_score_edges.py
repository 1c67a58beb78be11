"""Pins the oracle against the reference (the digests of its results, tests/refstore.py) on the model families of
tests/score_edges.py, where float rounding and score ties decide the ids: encode ids and offsets, n-best lists with
their score bits, seeded SampleEncode (n-best and full lattice) and CalculateEntropy bit for bit.  Also checks that
every family's corpus reaches the regime it is built for, measured by the exact-arithmetic instrument.  CPU only."""
import numpy as np
import pytest

import score_edges as se
from oracle import oracle_py
from refstore import digest, reference

UNIGRAM = [f.__name__ for f in se.UNIGRAM]
ALL = [f.__name__ for f in se.ALL]
NBEST_LINES = 40  # n-best lists of the first sentences of each corpus (the reference's A* search is slow on U-chain)


@pytest.mark.parametrize("name", ALL)
def test_regime(name):
    fam = se.family(name)
    st = se.measure(fam)
    for k, least in fam.regime.items():
        assert getattr(st, k) >= least, f"{name}: {k} = {getattr(st, k)}, the corpus is built for >= {least}"


def test_instrument_finds_rounding_decisions():
    """two relaxations into one position whose float sums are equal but whose exact sums differ: the strict `>` on the
    double candidate takes the later one"""
    x = se.f32(-1000.5)
    pcs = se.base_pieces() + [("▁", -1.0, se.mp.NORMAL), ("x", x, se.mp.NORMAL), ("q", 2.0 ** -12, se.mp.NORMAL),
                              ("xq", x, se.mp.NORMAL)]
    um = se.UnigramModel(pcs)
    st = se.Stats()
    text = se.normalize(b"x" * 300 + b"q")
    path = um.viterbi(text, st)
    assert st.rounding >= 1 and st.double_vs_float >= 1
    assert path[-1][2] == len(se.base_pieces()) + 2  # "q": fl(B + x) + 2^-12 > fl(B + x) exactly


@pytest.mark.parametrize("name", ALL)
def test_encode_vs_reference(name):
    fam = se.family(name)
    buf, offs = oracle_py.pack(fam.lines)
    want = reference(f"score_edges/encode/{name}", lambda: oracle_py.RefModel(fam.model).encode_batch(buf, offs))
    assert digest(*oracle_py.OracleModel(fam.model).encode_batch(buf, offs)) == want


@pytest.mark.parametrize("name", UNIGRAM)
def test_nbest_vs_reference(name):
    fam = se.family(name)
    calls = [(s, nb) for nb in (2, 16, 64) for s in fam.lines[:NBEST_LINES]]

    def run(m):
        return tuple(m.nbest_encode(s, nb) for s, nb in calls)
    want = reference(f"score_edges/nbest/{name}", lambda: run(oracle_py.RefModel(fam.model)))
    assert digest(*run(oracle_py.OracleModel(fam.model))) == want


@pytest.mark.parametrize("name", [n for n in UNIGRAM if n != "u_overflow"])
def test_sample_and_entropy_vs_reference(name):
    """(U-overflow is left out: LogSumExp of two -inf is NaN, whose bits are not portable)"""
    fam = se.family(name)
    buf, offs = oracle_py.pack(fam.lines)
    om = oracle_py.OracleModel(fam.model)
    for nb in (8, -1):
        want = reference(f"score_edges/sample/{name}/{nb}",
                         lambda: oracle_py.RefModel(fam.model).sample_encode_batch(buf, offs, nb, 0.3, 8081))
        assert digest(*om.sample_encode_batch(buf, offs, nb, 0.3, 8081)) == want, nb
    want = reference(f"score_edges/entropy/{name}", lambda: oracle_py.RefModel(fam.model).entropy_batch(buf, offs, 0.3))
    ent = om.entropy_batch(buf, offs, 0.3)
    assert digest(ent) == want
