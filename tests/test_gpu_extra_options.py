"""The encode frame (spm_engine_set_encode_frame): every entry point that returns encode ids returns exactly
ApplyExtraOptions (tests/extra_options.py) over the same engine's unframed output, for several option strings, on the
small, fused, chunked-fallback and device paths, with empty and long sentences; the reference's own results under
SetEncodeExtraOptions (stored digests) are matched; bad frames and undefined bos pieces fail like the reference.
Needs an H100."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, model_bytes
from extra_options import EDGE_LINES, OPTION_SETS, REFERENCE_SETS, apply_packed, nbest_digest, reference
from oracle import modelproto, oracle_py
from refstore import digest

pytestmark = pytest.mark.gpu
MODELS = [("uni32k", "en"), ("bpe32k", "en"), ("mix_bf8k", "mixed")]


def _engine(model):
    from sentencepiece_b200 import Engine
    return Engine(model_bytes(model))


def _special(model):
    from sentencepiece_b200 import _modelinfo
    sp = _modelinfo.special_pieces(model_bytes(model))
    return sp["bos_id"], sp["eos_id"]


def _set(eng, model, options):
    from sentencepiece_b200.processor import extra_frame
    p, rev, s = extra_frame(options.split(":") if options else [], *_special(model))
    eng.set_encode_frame(p, rev, s)


def _long_doc(corpus_gen, kind, seed, nbytes):
    return b" ".join(corpus_gen.lines(kind, seed, nbytes // 20))[:nbytes]


@pytest.fixture(scope="module")
def small_batches(corpus_gen):
    """short sentences, the edge cases and two documents long enough for the deferred (long-sentence) kernels"""
    out = {}
    for model, kind in MODELS:
        lines = EDGE_LINES + corpus_gen.lines(kind, 7071, 3000) + [_long_doc(corpus_gen, kind, 7072, 9000),
                                                                   _long_doc(corpus_gen, kind, 7073, 20000)]
        out[model] = oracle_py.pack(lines)
    return out


def _check_encode(eng, model, buf, offs, options):
    _set(eng, model, "")
    raw = eng.encode_packed(buf, offs)
    _set(eng, model, options)
    ids, ido = eng.encode_packed(buf, offs)
    want = apply_packed(*raw, options, *_special(model))
    assert np.array_equal(ido, want[1]) and np.array_equal(ids, want[0]), options
    return ids, ido


@pytest.mark.parametrize("model,kind", MODELS)
def test_encode_small(model, kind, small_batches):
    buf, offs = small_batches[model]
    eng = _engine(model)
    for options in OPTION_SETS:
        _check_encode(eng, model, buf, offs, options)
    assert eng.info().last_deferred > 0  # the long documents took the long-sentence path
    eng.close()


def _frame_vectorized(ids, ido, options, bos, eos):
    """the canonical form over a large packed result (numpy), checked against apply_extra by test_canonical_form"""
    from sentencepiece_b200.processor import extra_frame
    p, rev, s = extra_frame(options.split(":") if options else [], bos, eos)
    n = len(ido) - 1
    c = np.diff(ido.astype(np.int64))
    F = len(p) + len(s)
    no = ido.astype(np.int64) + np.arange(n + 1, dtype=np.int64) * F
    out = np.zeros(int(no[-1]), dtype=np.int32)
    for k, v in enumerate(p):
        out[no[:-1] + k] = v
    for k, v in enumerate(s):
        out[no[1:] - len(s) + k] = v
    sid = np.repeat(np.arange(n), c)
    j = np.arange(len(ids), dtype=np.int64) - ido[sid].astype(np.int64)
    if rev:
        j = c[sid] - 1 - j
    out[no[sid] + len(p) + j] = ids
    return out, no.astype(np.uint64)


@pytest.mark.parametrize("model,kind", MODELS)
@pytest.mark.parametrize("fallback", [False, True])
def test_encode_large(model, kind, fallback, corpus_gen):
    """>= 300k sentences: the fused path (in-kernel compaction) and, with one long document, the chunked fallback"""
    lines = corpus_gen.lines(kind, 7074, 320000) + EDGE_LINES
    if fallback:
        lines.insert(150000, _long_doc(corpus_gen, kind, 7075, 12000))
    buf, offs = oracle_py.pack(lines)
    eng = _engine(model)
    _set(eng, model, "")
    raw = eng.encode_packed(buf, offs)
    for options in ["bos:eos", "reverse", "bos:reverse:eos", "eos:bos:bos"]:
        _set(eng, model, options)
        ids, ido = eng.encode_packed(buf, offs)
        want = _frame_vectorized(*raw, options, *_special(model))
        assert np.array_equal(ido, want[1]) and np.array_equal(ids, want[0]), options
    eng.close()


@pytest.mark.parametrize("model,kind", MODELS)
def test_encode_device(model, kind, small_batches):
    import torch
    buf, offs = small_batches[model]
    n = len(offs) - 1
    d_bytes = torch.from_numpy(buf.copy()).cuda()
    d_offs = torch.from_numpy(offs.astype(np.int64)).cuda()
    eng = _engine(model)
    _set(eng, model, "")
    raw = eng.encode_packed(buf, offs)
    for options in OPTION_SETS:
        _set(eng, model, options)
        want = apply_packed(*raw, options, *_special(model))
        tot = int(want[1][-1])
        d_ids = torch.zeros(tot + 1, dtype=torch.int32, device="cuda")
        d_ido = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
        got = eng.encode_device(d_bytes.data_ptr(), d_offs.data_ptr(), n, len(buf), d_ids.data_ptr(), tot, d_ido.data_ptr())
        assert got == tot
        assert np.array_equal(d_ido.cpu().numpy().astype(np.uint64), want[1])
        assert np.array_equal(d_ids[:tot].cpu().numpy(), want[0]), options
        if tot > int(raw[1][-1]):  # room for the ids but not for the frame
            with pytest.raises(RuntimeError, match=f"need {tot}"):
                eng.encode_device(d_bytes.data_ptr(), d_offs.data_ptr(), n, len(buf), d_ids.data_ptr(), tot - 1,
                                  d_ido.data_ptr())
    eng.close()


@pytest.mark.parametrize("model,kind", [("uni32k", "en"), ("mix_bf8k", "mixed")])
def test_nbest(model, kind, small_batches):
    buf, offs = small_batches[model]
    eng = _engine(model)
    _set(eng, model, "")
    raw = eng.nbest_encode(buf, offs, 8)
    for options in OPTION_SETS:
        _set(eng, model, options)
        r = eng.nbest_encode(buf, offs, 8)
        want = apply_packed(raw["ids"], raw["cand_offsets"], options, *_special(model))
        # the empty slots (c >= n_cands) stay empty
        real = (np.arange(len(raw["cand_offsets"]) - 1) % 8) < np.repeat(raw["n_cands"], 8)
        lens = np.where(real, np.diff(want[1].astype(np.int64)), 0)
        wo = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
        wids = np.concatenate([want[0][int(want[1][j]):int(want[1][j + 1])] for j in np.nonzero(real)[0]])
        assert np.array_equal(r["n_cands"], raw["n_cands"]) and np.array_equal(r["scores"], raw["scores"])
        assert np.array_equal(r["cand_offsets"], wo) and np.array_equal(r["ids"], wids), options
    eng.close()


@pytest.mark.parametrize("model,kind", [("uni32k", "en"), ("mix_bf8k", "mixed")])
@pytest.mark.parametrize("nbest", [-1, 8, 1])
def test_sample_encode(model, kind, nbest, small_batches):
    buf, offs = small_batches[model]
    eng = _engine(model)
    for options in OPTION_SETS:
        _set(eng, model, "")
        eng.set_random_seed(99)
        raw = eng.sample_encode(buf, offs, nbest, 0.3)
        _set(eng, model, options)
        eng.set_random_seed(99)
        ids, ido = eng.sample_encode(buf, offs, nbest, 0.3)
        want = apply_packed(*raw, options, *_special(model))
        assert np.array_equal(ido, want[1]) and np.array_equal(ids, want[0]), options
    eng.close()


def test_sample_encode_and_score(small_batches):
    buf, offs = small_batches["uni32k"]
    eng = _engine("uni32k")
    for options in OPTION_SETS:
        _set(eng, "uni32k", "")
        eng.set_random_seed(5)
        raw = eng.sample_encode_and_score(buf, offs, 3, 0.5)
        _set(eng, "uni32k", options)
        eng.set_random_seed(5)
        ids, co, sc = eng.sample_encode_and_score(buf, offs, 3, 0.5)
        want = apply_packed(raw[0], raw[1], options, *_special("uni32k"), skip_empty=True)
        assert np.array_equal(co, want[1]) and np.array_equal(ids, want[0]) and np.array_equal(sc, raw[2]), options
    eng.close()


# ---- the reference's results under SetEncodeExtraOptions (digests recorded by tests/test_oracle_extra_options.py) ----

@pytest.mark.parametrize("model,kind", MODELS)
@pytest.mark.parametrize("options", REFERENCE_SETS)
def test_reference_digests(model, kind, options, corpus_gen):
    lines = EDGE_LINES + corpus_gen.lines(kind, 6061, 300)
    eng = _engine(model)
    _set(eng, model, options)
    assert digest(*eng.encode_packed(*oracle_py.pack(lines))) == reference(f"encode/{model}/{kind}/{options}", None)
    if model == "uni32k":
        nb_lines = EDGE_LINES + corpus_gen.lines(kind, 6061, 40)
        r = eng.nbest_encode(*oracle_py.pack(nb_lines), 8)
        co = r["cand_offsets"]
        got = [[r["ids"][int(co[i * 8 + c]):int(co[i * 8 + c + 1])] for c in range(int(r["n_cands"][i]))]
               for i in range(len(nb_lines))]
        assert nbest_digest(got) == reference(f"nbest/uni32k/{options}", None)
        buf, offs = oracle_py.pack(EDGE_LINES + corpus_gen.lines(kind, 6061, 200))
        for nbest in (-1, 8, 1):
            eng.set_random_seed(77)
            assert digest(*eng.sample_encode(buf, offs, nbest, 0.5)) == reference(f"sample/uni32k/{nbest}/{options}", None)
        buf, offs = oracle_py.pack(EDGE_LINES + corpus_gen.lines(kind, 6061, 100))
        eng.set_random_seed(78)
        assert digest(*eng.sample_encode_and_score(buf, offs, 3, 0.5)) == reference(f"sample_score/uni32k/{options}", None)
    eng.close()


# ---- errors ----

def test_bad_frames():
    eng = _engine("uni32k")
    V = eng.info().vocab_size
    for prefix, suffix in (([V], []), ([], [-1]), ([1] * 65, []), ([], [2] * 65)):
        with pytest.raises(RuntimeError, match="spm_b200 error 1: spm_engine_set_encode_frame"):
            eng.set_encode_frame(prefix, False, suffix)
    eng.set_encode_frame([1] * 64, True, [2] * 64)  # the largest frame
    eng.close()


def _toy_without_bos():
    """a unigram model whose trainer_spec names the default <s>, which is not among its pieces"""
    pieces = [("<unk>", 0.0, modelproto.UNKNOWN), ("</s>", 0.0, modelproto.CONTROL), ("▁", -1.0, modelproto.NORMAL),
              ("a", -2.0, modelproto.NORMAL), ("b", -2.0, modelproto.NORMAL)]
    return modelproto.build_model(pieces)


def test_undefined_bos_python():
    from sentencepiece_b200 import SentencePieceProcessor
    sp = SentencePieceProcessor(model_proto=_toy_without_bos())
    with pytest.raises(RuntimeError, match="id for `<s>` is not defined."):
        sp.SetEncodeExtraOptions("bos:eos")
    with pytest.raises(RuntimeError, match="id for `<s>` is not defined."):
        sp.encode("ab", add_bos=True)
    assert sp.encode("ab ba", add_eos=True, reverse=True) == apply_packed(
        np.array(sp.encode("ab ba"), np.int32), np.array([0, len(sp.encode("ab ba"))], np.uint64), "reverse:eos", -1, 1)[0].tolist()


def test_undefined_bos_cli(tmp_path):
    cli = os.path.join(ROOT, "sentencepiece_b200", "lib", "spm_encode_b200")
    mpath = str(tmp_path / "toy.model")
    with open(mpath, "wb") as f:
        f.write(_toy_without_bos())
    inp = tmp_path / "in.txt"
    inp.write_bytes(b"ab\n")
    r = subprocess.run([cli, f"--model={mpath}", "--extra_options=bos", f"--input={inp}"], capture_output=True)
    assert r.returncode != 0 and b"id for `<s>` is not defined." in r.stderr
    r = subprocess.run([cli, f"--model={mpath}", "--extra_options=eos:reverse", "--output_format=id", f"--input={inp}"],
                       capture_output=True, check=True)
    ids = [int(x) for x in r.stdout.split()]
    assert ids[0] == 1 and len(ids) >= 2  # eos, then the reversed sentence


def test_python_mirror(small_batches):
    """encode / NBestEncodeAsIds / SampleEncodeAsIds with add_bos, add_eos, reverse after SetEncodeExtraOptions"""
    from sentencepiece_b200 import SentencePieceProcessor
    sp = SentencePieceProcessor(model_proto=model_bytes("uni32k"))
    bos, eos = _special("uni32k")
    text = ["hello world", "", "a b c"]
    plain = sp.encode(text)
    sp.SetEncodeExtraOptions("eos")
    got = sp.encode(text, add_bos=True, reverse=True)
    assert got == [apply_packed(np.array(p, np.int32), np.array([0, len(p)], np.uint64), "eos:reverse:bos", bos, eos)[0].tolist()
                   for p in plain]
    nb = sp.NBestEncodeAsIds("hello world", 4, add_eos=True)
    sp.SetEncodeExtraOptions("")
    nb_plain = sp.NBestEncodeAsIds("hello world", 4)
    assert nb == [c + [eos, eos] for c in nb_plain]
    sp.SetRandomGeneratorSeed(3)
    s1 = sp.SampleEncodeAsIds(text, -1, 0.5, add_bos=True)
    sp.SetRandomGeneratorSeed(3)
    s0 = sp.SampleEncodeAsIds(text, -1, 0.5)
    assert s1 == [[bos] + s for s in s0]
    pcs = sp.encode("hello world", out_type=str, add_bos=True, add_eos=True, emit_unk_piece=True)
    assert pcs[0] == "<s>" and pcs[-1] == "</s>" and pcs[1:-1] == sp.encode("hello world", out_type=str)
    with pytest.raises(RuntimeError, match='option "foo" is not available.'):
        sp.SetEncodeExtraOptions("bos:foo")
    assert sp.encode(text) == plain  # a failed parse keeps no option
