"""spm_decode_offsets (K7's token-end mode, decode_kernel.cuh) and the layers on it: the C++ class's
DecodeWithOffsets and Python's decode / Decode / DecodeIds / DecodeIdsAsImmutableProto.  Checked against digests of the
unmodified reference's Decode(ids, SentencePieceText*) (tests/decode_offsets_cases.py), a plain-C restatement of its
rules (tests/decode_spans_oracle.c) and spm_decode_ids.  Needs an H100."""
import os
import subprocess

import numpy as np
import pytest

import decode_offsets_cases as dc
from conftest import ROOT, model_bytes
from decode_spans_oracle import DecodeSpans
from oracle import modelproto as mp
from test_decode_offsets_host import _byte_model, byte_fallback_kat

pytestmark = pytest.mark.gpu
WS = "▁"
N, U, C, B = mp.NORMAL, mp.UNKNOWN, mp.CONTROL, mp.BYTE


def _engine(mb):
    from sentencepiece_b200 import Engine
    return Engine(mb)


def _check_against(eng, om, ids, ido, what):
    text, to, te = eng.decode_offsets(ids, ido)
    t2, to2 = eng.decode_packed(ids, ido)
    assert np.array_equal(text, t2) and np.array_equal(to, to2), f"{what}: text differs from spm_decode_ids"
    otext, oto, ote = om.decode_spans_batch(ids, ido)
    assert np.array_equal(to, oto) and np.array_equal(text, otext), f"{what}: text differs from the restatement"
    assert np.array_equal(te, ote), f"{what}: token ends differ from the restatement"


@pytest.mark.parametrize("model", dc.MODELS)
def test_reference_digests(model, corpus_gen):
    want = dc.stored()
    base = model_bytes(model)
    for variant in dc.VARIANTS:
        mb = dc.model_variant(base, variant)
        eng = _engine(mb)
        pieces = dc.piece_bytes(mb)
        for name in dc.INPUTS:
            ids, ido = dc.packed(dc.lists_of(corpus_gen, name, mb))
            rows = dc.rows(pieces, ids, ido, *eng.decode_offsets(ids, ido))
            assert dc.digest(rows) == want[dc.key(model, variant, name)], (model, variant, name)
        eng.close()


@pytest.mark.parametrize("model,kind", [("uni32k", "en"), ("mix_bf8k", "mixed"), ("bpe32k", "en"), ("botchan8k", "en"),
                                        ("mix_bpe4k", "mixed")])
def test_scale_round_trip_and_random_lists(model, kind, corpus_gen):
    base = model_bytes(model)
    for variant in dc.VARIANTS:
        mb = dc.model_variant(base, variant)
        eng = _engine(mb)
        om = DecodeSpans(mb)
        buf, offs = corpus_gen.fill(kind, 9301, 20000)
        ids, ido = eng.encode_packed(buf, offs)
        _check_against(eng, om, ids, ido, f"{model}/{variant} round trip")
        lists = sum((dc.random_lists(mb, seed) for seed in range(9302, 9310)), [])[:3200]
        ids2, ido2 = dc.packed(lists)
        _check_against(eng, om, ids2, ido2, f"{model}/{variant} random lists")
        # a nonzero id_offsets[0]: tok_end is indexed from it
        ido3 = ido2[5:].copy()
        te_all = eng.decode_offsets(ids2, ido2)[2]
        text, to, te = eng.decode_offsets(ids2, ido3)
        assert np.array_equal(te, te_all[int(ido3[0]):]), f"{model}/{variant} nonzero first offset"
        eng.close()


def test_toy_known_answers():
    from sentencepiece_b200 import SentencePieceProcessor
    pieces = [("<unk>", 0.0, U), ("<s>", 0.0, C), ("</s>", 0.0, C), (WS + "ABC", 0.0, N), (WS + "DE", 0.0, N),
              ("F", 0.0, N), ("G" + WS + "H", 0.0, N), ("I", 0.0, N)]
    sp = SentencePieceProcessor(model_proto=mp.build_model(pieces))
    p = sp.DecodeIdsAsImmutableProto([1, 3, 0, 4, 5, 6, 7, 2])  # sentencepiece_processor_test.cc:575-620
    assert p.text == "ABC ⁇  DEFG HI"
    assert [(x.piece, x.id, x.surface, x.begin, x.end) for x in p] == [
        ("<s>", 1, "", 0, 0), (WS + "ABC", 3, "ABC", 0, 3), ("<unk>", 0, " ⁇ ", 3, 6), (WS + "DE", 4, " DE", 6, 9),
        ("F", 5, "F", 9, 10), ("G" + WS + "H", 6, "G H", 10, 13), ("I", 7, "I", 13, 14), ("</s>", 2, "", 14, 14)]
    eng = _engine(mp.build_model(pieces))
    text, to, te = eng.decode_offsets(np.array([1, 3, 0, 4, 5, 6, 7, 2], np.int32), np.array([0, 8], np.uint64))
    assert te.tolist() == [0, 3, 8, 11, 12, 15, 16, 16]  # the byte offsets of the C++ test
    eng.close()
    ids, text, want = byte_fallback_kat()  # :843-
    eng = _engine(_byte_model())
    t, to, te = eng.decode_offsets(np.asarray(ids, np.int32), np.array([0, len(ids)], np.uint64))
    assert t.tobytes().decode() == text
    assert te.tolist() == [e for _, _, e in want]
    sp = SentencePieceProcessor(model_proto=_byte_model())
    p = sp.decode(ids, out_type="immutable_proto")
    raw = text.encode()
    assert [(x.surface_as_bytes, x.begin, x.end) for x in p] == [
        (s.encode(), len(raw[:b].decode()), len(raw[:e].decode())) for s, b, e in want]
    eng.close()


def test_pipelined_path(corpus_gen):
    from sentencepiece_b200 import Engine
    mb = model_bytes("mix_bf8k")
    eng = Engine(mb)
    om = DecodeSpans(mb)
    buf, offs = corpus_gen.fill("mixed", 9303, 300000)
    ids, ido = eng.encode_packed(buf, offs)
    text, to, te = eng.decode_offsets(ids, ido)  # n >= pipeline_min_sentences: the chunked three-stage path
    assert eng.info().last_d2h_bytes >= len(te) * 4 + len(text)  # the token ends are counted with the text
    assert np.array_equal(text, eng.decode_packed(ids, ido)[0])
    step = 100000
    for lo in range(0, 300000, step):
        part = ido[lo:lo + step + 1]
        t2, to2, te2 = eng.decode_offsets(ids, part)
        assert np.array_equal(t2, text[int(to[lo]):int(to[lo + len(part) - 1])]), lo
        assert np.array_equal(te2, te[int(part[0]):int(part[-1])]), lo
    sel = np.arange(0, 300000, 97)
    for i in sel.tolist():
        a, b = int(ido[i]), int(ido[i + 1])
        ot, _, ote = om.decode_spans_batch(ids[a:b], np.array([0, b - a], np.uint64))
        assert np.array_equal(te[a:b], ote) and text[int(to[i]):int(to[i + 1])].tobytes() == ot.tobytes(), i
    eng.close()


def test_errors():
    import ctypes
    from sentencepiece_b200 import Engine, _capi
    mb = model_bytes("mix_bf8k")
    eng = Engine(mb)
    om = DecodeSpans(mb)
    good = (np.array([5, 6, 7], np.int32), np.array([0, 3], np.uint64))
    for n in (3, 300000):  # the plain path and the pipelined one
        lists = [[5, 6]] * (n - 1) + [[5, 999999]]
        ids, ido = dc.packed(lists)
        with pytest.raises(RuntimeError, match="Invalid id: 999999"):
            eng.decode_offsets(ids, ido)
        ids[-1] = -3
        with pytest.raises(RuntimeError, match="Invalid id: -3"):
            eng.decode_offsets(ids, ido)
        _check_against(eng, om, *good, "after an error")  # still usable
    # n == 0
    text, to, te = eng.decode_offsets(np.zeros(0, np.int32), np.array([0], np.uint64))
    assert len(text) == 0 and to.tolist() == [0] and len(te) == 0
    text, to, te = eng.decode_offsets(np.zeros(0, np.int32), np.array([7], np.uint64))
    assert to.tolist() == [0] and len(te) == 0
    # id_offsets must be non-decreasing; null outputs
    with pytest.raises(RuntimeError, match="non-decreasing"):
        eng.decode_offsets(np.array([5, 6], np.int32), np.array([0, 2, 1], np.uint64))
    L = _capi.load()
    p = [ctypes.c_void_p() for _ in range(3)]
    ids, ido = good
    assert L.spm_decode_offsets(eng._h, ids.ctypes.data, ido.ctypes.data, 1, ctypes.byref(p[0]), ctypes.byref(p[1]),
                                None) == 1
    assert L.spm_decode_offsets(None, ids.ctypes.data, ido.ctypes.data, 1, *[ctypes.byref(x) for x in p]) == 1
    _check_against(eng, om, *good, "after the argument errors")
    eng.close()
    # a BYTE piece that is not <0xXX> never reaches the decoder: the engine refuses the model
    bad = [("<unk>", 0.0, U), ("A", 0.0, N)] + [("<0x%02X>" % i, 0.0, B) for i in range(255)] + [("<0xzz>", 0.0, B)]
    with pytest.raises(RuntimeError, match="invalid"):
        Engine(mp.build_model(bad, byte_fallback=True))
    # a model with a denormalizer_spec: SPM_ERR_UNSUPPORTED, as spm_decode_ids
    with open(os.path.join(ROOT, "tests", "golden", "charsmaps", "nmt_nfkc_cf.bin"), "rb") as f:
        cm = f.read()
    dm = model_bytes("uni32k") + mp._ld(5, mp._ld(2, cm))
    eng = Engine(dm)
    with pytest.raises(RuntimeError, match="denormalizer"):
        eng.decode_offsets(*good)
    with pytest.raises(RuntimeError, match="denormalizer"):
        eng.decode_packed(*good)
    eng.close()


def test_cpp_class(corpus_gen, tmp_path):
    lib = os.path.join(ROOT, "sentencepiece_b200", "lib")
    exe = str(tmp_path / "decode_offsets_class_check")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(ROOT, "sentencepiece_b200", "csrc"),
                           "-I" + os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "decode_offsets_class_check.cc"),
                           os.path.join(lib, "sentencepiece_processor.o"), os.path.join(lib, "model_reader.o"),
                           "-L" + os.path.join(lib, "stdcxx"), "-L" + lib, "-lspm_b200", "-Wl,-rpath," + lib])
    for model in ("uni32k", "mix_bf8k", "bpe32k"):
        mb = model_bytes(model)
        lists = dc.lists_of(corpus_gen, "mixed", mb)[:300] + dc.random_lists(mb, 9304)[-200:]
        inp = tmp_path / "in.txt"
        inp.write_text("".join(" ".join(map(str, x)) + "\n" for x in lists))
        out = subprocess.check_output([exe, os.path.join(ROOT, "tests", "golden", "models", model + ".model"), str(inp)])
        rows = out.decode().splitlines()
        assert len(rows) == len(lists) + 2
        ids, ido = dc.packed(lists)
        om = DecodeSpans(mb)
        want = dc.rows(dc.piece_bytes(mb), ids, ido, *om.decode_spans_batch(ids, ido))
        assert rows[:len(lists)] == want, model
        assert rows[len(lists)] == want[-1]  # the single-list overload on the last list
        assert rows[-1] == "error: Invalid id: " + str(len(dc.piece_bytes(mb))), model


def test_python_api():
    from sentencepiece_b200 import SentencePieceProcessor
    from sentencepiece_b200.processor import ImmutableSentencePiece, ImmutableSentencePieceText
    sp = SentencePieceProcessor(model_file=os.path.join(ROOT, "tests", "golden", "models", "mix_bf8k.model"))
    texts = ["Hello world.", "こんにちは、世界", "emoji 😀 and 한국어", "ǅ ₩ ﬁ", ""]
    lists = sp.EncodeAsIds(texts)
    plain = sp.DecodeIds(lists)
    assert sp.decode(lists) == plain and sp.Decode(lists) == plain
    assert sp.decode(lists[0]) == plain[0] and sp.DecodeIds(lists[0]) == plain[0]
    assert sp.decode(lists, out_type=bytes) == [s.encode() for s in plain]
    assert sp.DecodeIds(lists[1], out_type=bytes) == plain[1].encode()
    assert sp.decode(lists[0][0]) == sp.DecodeIds([lists[0][0]])  # one int
    assert sp.decode([]) == "" and sp.Decode([], out_type="immutable_proto") == ""
    assert sp.decode([[]]) == [""]
    assert sp.decode(np.asarray(lists[1])) == plain[1]
    protos = sp.decode(lists, out_type="immutable_proto")
    assert protos == sp.DecodeIdsAsImmutableProto(lists) == sp.decode_ids_as_immutable_proto(lists)
    assert sp.DecodeIds(lists, out_type="immutable_proto") == protos
    assert sp.decode(lists[2], out_type="immutable_proto") == protos[2]
    pieces = sp.EncodeAsPieces(texts)
    for pr, text, ids, pcs in zip(protos, plain, lists, pieces):
        assert isinstance(pr, ImmutableSentencePieceText) and pr.text == text and len(pr) == len(ids)
        assert [x.id for x in pr] == ids
        prev = 0
        for x in pr:
            assert isinstance(x, ImmutableSentencePiece)
            assert x.surface == pr.text[x.begin:x.end] and x.begin == prev
            prev = x.end
        assert prev == len(pr.text)
    # byte fallback: the bytes of a character share its begin, only the last token gets the character
    assert any(x.piece.startswith("<0x") for pr in protos for x in pr)
    # CJK surfaces are whole characters in character offsets
    cjk = protos[1]
    assert "".join(x.surface for x in cjk) == cjk.text
    # equality, read-only behaviour, comparison with other types
    assert protos[0] != protos[1] and protos[0] != "x" and protos[0][0] != 1
    with pytest.raises(AttributeError):
        protos[0].text = "x"
    with pytest.raises(AttributeError):
        protos[0][0].begin = 3
    # pieces are not on the device path; unknown out_type
    with pytest.raises(NotImplementedError):
        sp.decode("▁Hello")
    with pytest.raises(NotImplementedError):
        sp.decode(["▁Hello", "▁world"])
    with pytest.raises(NotImplementedError):
        sp.decode([["▁Hello"]], out_type="immutable_proto")
    with pytest.raises(RuntimeError):
        sp.decode(lists, out_type=float)
    with pytest.raises(RuntimeError, match="Invalid id"):
        sp.decode([[1], [10 ** 6]], out_type="immutable_proto")
