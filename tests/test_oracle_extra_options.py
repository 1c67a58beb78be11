"""The restatement of ApplyExtraOptions in tests/extra_options.py, over the oracle's results, against the reference's
own results under SetEncodeExtraOptions (stored digests): Encode, NBestEncode, seeded SampleEncode and
SampleEncodeAndScore, empty sentences included.  These pin what the device's encode frame must reproduce
(tests/test_gpu_extra_options.py).  Runs on the CPU."""
import numpy as np
import pytest

from conftest import model_bytes
from extra_options import EDGE_LINES, REFERENCE_SETS, apply_extra, apply_packed, nbest_digest, reference, set_reference_options
from oracle import oracle_py
from refstore import digest
from sentencepiece_b200 import _modelinfo
from sentencepiece_b200.processor import extra_frame


def _ref(model, options):
    r = oracle_py.RefModel(model_bytes(model))
    set_reference_options(r, options)
    return r


def _lines(corpus_gen, kind, n):
    return EDGE_LINES + corpus_gen.lines(kind, 6061, n)


def _special(model):
    sp = _modelinfo.special_pieces(model_bytes(model))
    return sp["bos_id"], sp["eos_id"]


@pytest.mark.parametrize("model,kind", [("uni32k", "en"), ("bpe32k", "en"), ("mix_bf8k", "mixed")])
@pytest.mark.parametrize("options", REFERENCE_SETS)
def test_encode(model, kind, options, corpus_gen):
    buf, offs = oracle_py.pack(_lines(corpus_gen, kind, 300))
    want = reference(f"encode/{model}/{kind}/{options}", lambda: _ref(model, options).encode_batch(buf, offs))
    ids, ido = oracle_py.OracleModel(model_bytes(model)).encode_batch(buf, offs)
    assert digest(*apply_packed(ids, ido, options, *_special(model))) == want


@pytest.mark.parametrize("options", REFERENCE_SETS)
def test_nbest(options, corpus_gen):
    """Every candidate is framed; an empty sentence has one empty candidate, which is framed as well."""
    lines = _lines(corpus_gen, "en", 40)

    def live():
        ref = _ref("uni32k", options)
        return [[np.asarray(c, dtype=np.int32) for c in ref.nbest_encode(s, 8)[0]] for s in lines]

    want = reference(f"nbest/uni32k/{options}", live)
    om = oracle_py.OracleModel(model_bytes("uni32k"))
    bos, eos = _special("uni32k")
    got = [[apply_extra(c.tolist(), options, bos, eos) for c in om.nbest_encode(s, 8)[0]] for s in lines]
    assert nbest_digest(got) == want


@pytest.mark.parametrize("nbest", [-1, 8, 1])
@pytest.mark.parametrize("options", REFERENCE_SETS)
def test_sample_encode(nbest, options, corpus_gen):
    buf, offs = oracle_py.pack(_lines(corpus_gen, "en", 200))
    want = reference(f"sample/uni32k/{nbest}/{options}",
                     lambda: _ref("uni32k", options).sample_encode_batch(buf, offs, nbest, 0.5, 77))
    ids, ido = oracle_py.OracleModel(model_bytes("uni32k")).sample_encode_batch(buf, offs, nbest, 0.5, 77)
    assert digest(*apply_packed(ids, ido, options, *_special("uni32k"))) == want


@pytest.mark.parametrize("options", REFERENCE_SETS)
def test_sample_encode_and_score(options, corpus_gen):
    """Samples are framed and keep the raw path's score; an empty sentence has no sample (the reference returns an
    error for it), so its slots stay empty."""
    buf, offs = oracle_py.pack(_lines(corpus_gen, "en", 100))
    want = reference(f"sample_score/uni32k/{options}",
                     lambda: _ref("uni32k", options).sample_score_batch(buf, offs, 3, 0.5, 78))
    ids, co, sc = oracle_py.OracleModel(model_bytes("uni32k")).sample_score_batch(buf, offs, 3, 0.5, 78)
    fids, fco = apply_packed(ids, co, options, *_special("uni32k"), skip_empty=True)
    assert digest(fids, fco, sc) == want


@pytest.mark.parametrize("options", ["bos", "eos", "bos:eos", "reverse", "bos:reverse:eos", "eos:bos:bos",
                                     "reverse:reverse", "reverse:bos:reverse:eos:reverse", ""])
def test_canonical_form(options):
    """The engine's form prefix ++ (r or reversed r) ++ suffix equals applying the options one by one."""
    r = list(range(10, 17))
    p, rev, s = extra_frame(options.split(":") if options else [], 1, 2)
    assert p + (r[::-1] if rev else r) + s == apply_extra(r, options, 1, 2)


def test_special_pieces():
    sp = _modelinfo.special_pieces(model_bytes("uni32k"))
    pieces, _ = _modelinfo.pieces_and_unk(model_bytes("uni32k"))
    assert pieces[sp["bos_id"]] == sp["bos_piece"] == "<s>" and pieces[sp["eos_id"]] == sp["eos_piece"] == "</s>"
