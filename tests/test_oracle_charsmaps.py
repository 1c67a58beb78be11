"""Pins the oracle against the reference (the digests of its results, tests/refstore.py) on the rule sets of
tests/charsmap_rules.py: Normalize (text and norm_to_orig) and encode ids on a unigram and a BPE model, under the
default normalizer flags and five variants.  Also checks that each synthetic family's corpus reaches every rule it is
built for.  CPU only."""
import pytest

import charsmap_rules as cr
from conftest import model_bytes
from oracle import modelproto as mp
from oracle import oracle_py
from refstore import digest, reference

SEED, N = 5100, 400
FIRES = {"ascii_keys": 20, "ladder": 10, "long_keys": 20, "delete_expand": 50, "glue": 1000}


def corpus(name, corpus_gen):
    return cr.lines(name, corpus_gen, SEED, N)


@pytest.mark.parametrize("name", cr.SYNTHETIC)
def test_every_rule_fires(name, corpus_gen):
    fired = cr.fires(name, corpus(name, corpus_gen))
    rare = {k: v for k, v in fired.items() if v < FIRES[name]}
    assert not rare, f"{name}: rules chosen fewer than {FIRES[name]} times: {rare}"


def test_long_keys_cross_every_window():
    lens = sorted(len(k) for k in cr.keys("long_keys"))
    assert set(lens) == set(cr.LONG) and lens.count(100) == 2
    ratio = {len(k.encode()): (len(t.encode()) + 2 * t.count(" ")) / len(k.encode()) for k, t in cr.RULES["long_keys"]}
    assert min(ratio[66], ratio[100]) > 3 and max(ratio, key=ratio.get) in (66, 100)


@pytest.mark.parametrize("flags", cr.FLAGS, ids=cr.FLAG_IDS)
@pytest.mark.parametrize("name", cr.ALL)
def test_normalize_vs_reference(name, flags, corpus_gen):
    mb = mp.replace_flags(model_bytes("uni32k"), charsmap=cr.blob(name), **flags)
    lines = corpus(name, corpus_gen)

    def run(m):
        return [m.normalize(s) for s in lines]
    fid = cr.FLAG_IDS[cr.FLAGS.index(flags)]
    want = reference(f"charsmaps/normalize/{name}/{fid}", lambda: run(oracle_py.RefModel(mb)))
    assert digest(run(oracle_py.OracleModel(mb))) == want


@pytest.mark.parametrize("model", ["uni32k", "bpe32k"])
@pytest.mark.parametrize("flags", cr.FLAGS, ids=cr.FLAG_IDS)
@pytest.mark.parametrize("name", cr.ALL)
def test_encode_vs_reference(name, flags, model, corpus_gen):
    mb = mp.replace_flags(model_bytes(model), charsmap=cr.blob(name), **flags)
    buf, offs = oracle_py.pack(corpus(name, corpus_gen))
    fid = cr.FLAG_IDS[cr.FLAGS.index(flags)]
    want = reference(f"charsmaps/encode/{model}/{name}/{fid}", lambda: oracle_py.RefModel(mb).encode_batch(buf, offs))
    assert digest(*oracle_py.OracleModel(mb).encode_batch(buf, offs)) == want
