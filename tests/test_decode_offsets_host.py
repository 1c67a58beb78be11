"""Decode with offsets without a GPU: the restatement of Decode(ids, SentencePieceText*) (tests/decode_spans_oracle.c)
against the reference's own known answers (sentencepiece_processor_test.cc DecodeTest :575-620 and
ByteFallbackDecodeTest :843-, restated over ids) and against every stored digest of the unmodified reference
(tests/golden/reference_digests_decode_offsets.json); ConvertToUnicodeSpans over decoded text; and the loud failure of
the Python entry points without a device."""
import numpy as np
import pytest

import decode_offsets_cases as dc
from conftest import model_bytes
from decode_spans_oracle import DecodeSpans
from oracle import modelproto as mp
from oracle import oracle_py
from sentencepiece_b200.processor import decode_protos, unicode_spans

WS = "▁"
N, U, C, B = mp.NORMAL, mp.UNKNOWN, mp.CONTROL, mp.BYTE


def _spans(om, ids):
    text, to, te = om.decode_spans_batch(np.asarray(ids, dtype=np.int32), np.array([0, len(ids)], dtype=np.uint64))
    t = text.tobytes()
    out, b = [], 0
    for e in te.tolist():
        out.append((t[b:e].decode("utf-8"), b, e))
        b = e
    return t.decode("utf-8"), out


def _toy(**kw):
    pieces = [("<unk>", 0.0, U), ("<s>", 0.0, C), ("</s>", 0.0, C), (WS + "ABC", 0.0, N), (WS + "DE", 0.0, N),
              ("F", 0.0, N), ("G" + WS + "H", 0.0, N), ("I", 0.0, N)]
    return DecodeSpans(mp.build_model(pieces, **kw))


def test_kat_decode_test():
    # :575-620; "I" is a normal piece here (the mock model's out-of-vocabulary piece decodes to itself)
    text, sp = _spans(_toy(), [1, 3, 0, 4, 5, 6, 7, 2])
    assert text == "ABC ⁇  DEFG HI"
    assert sp == [("", 0, 0), ("ABC", 0, 3), (" ⁇ ", 3, 8), (" DE", 8, 11), ("F", 11, 12), ("G H", 12, 15),
                  ("I", 15, 16), ("", 16, 16)]


def test_kat_leading_whitespace():
    pieces = [("<unk>", 0.0, U), (WS, 0.0, N), (WS + WS, 0.0, N), (WS + "a", 0.0, N), ("b", 0.0, N)]
    rm = DecodeSpans(mp.build_model(pieces))
    assert _spans(rm, [1, 1, 3, 3]) == ("a a", [("", 0, 0), ("", 0, 0), ("a", 0, 1), (" a", 1, 3)])
    norm = DecodeSpans(mp.build_model(pieces, remove_extra_whitespaces=False))
    assert _spans(norm, [1, 1, 3]) == ("  a", [("", 0, 0), (" ", 0, 1), (" a", 1, 3)])


def _byte_model():
    pieces = [("<unk>", 0.0, U), ("<s>", 0.0, C), ("</s>", 0.0, C), ("A", 0.0, N), ("B", 0.0, N), ("C", 0.0, N)]
    pieces += [("<0x%02X>" % i, 0.0, B) for i in range(256)]
    return mp.build_model(pieces, byte_fallback=True)


def byte_fallback_kat():
    """ByteFallbackDecodeTest (:843-) over ids: the ids, the text and every token's (surface, begin, end)"""
    b = lambda x: 6 + x  # noqa: E731
    ids = [1, 3, 4, b(0xE3), b(0x81), b(0x82), b(0x5A), b(0xCE), b(0xA9), 5, b(0xE0), b(0x80), b(0xE3), b(0x81), b(0x84),
           b(0xEF), b(0xBF), b(0xBD)]
    R = "�"
    want = [("", 0, 0), ("A", 0, 1), ("B", 1, 2), ("", 2, 2), ("", 2, 2), ("あ", 2, 5), ("Z", 5, 6), ("", 6, 6),
            ("Ω", 6, 8), ("C", 8, 9), (R, 9, 12), (R, 12, 15), ("", 15, 15), ("", 15, 15), ("い", 15, 18), ("", 18, 18),
            ("", 18, 18), (R, 18, 21)]
    return ids, "ABあZΩC" + R + R + "い" + R, want


def test_kat_byte_fallback_decode():
    ids, text, want = byte_fallback_kat()
    assert _spans(DecodeSpans(_byte_model()), ids) == (text, want)
    # a run that ends inside a character: one U+FFFD per byte, then the piece
    R = "�"
    assert _spans(DecodeSpans(_byte_model()), [6 + 0xE3, 6 + 0x81, 3]) == \
        (R + R + "A", [(R, 0, 3), (R, 3, 6), ("A", 6, 7)])


def test_text_equals_decode_ids(corpus_gen):
    mb = model_bytes("mix_bf8k")
    lists = dc.random_lists(mb, 5)
    ids, ido = dc.packed(lists)
    text, to, _ = DecodeSpans(mb).decode_spans_batch(ids, ido)
    t2, to2 = oracle_py.OracleModel(mb).decode_batch(ids, ido)  # oracle/spm_oracle.c's Decode(ids)
    assert np.array_equal(text, t2) and np.array_equal(to, to2)


@pytest.mark.parametrize("model", dc.MODELS)
def test_oracle_matches_reference_digests(model, corpus_gen):
    want = dc.stored()
    base = model_bytes(model)
    for variant in dc.VARIANTS:
        mb = dc.model_variant(base, variant)
        om = DecodeSpans(mb)
        pieces = dc.piece_bytes(mb)
        for name in dc.INPUTS:
            ids, ido = dc.packed(dc.lists_of(corpus_gen, name, mb))
            rows = dc.rows(pieces, ids, ido, *om.decode_spans_batch(ids, ido))
            assert dc.digest(rows) == want[dc.key(model, variant, name)], (model, variant, name)


def test_unicode_spans_on_decoded_text():
    R = "�".encode()
    # lists: "aあ😀" + U+FFFD + "b", then "" , then "é" + U+FFFD
    t0 = b"a" + "あ".encode() + "😀".encode() + R + b"b"
    t1 = "é".encode() + R
    text = np.frombuffer(t0 + t1, np.uint8)
    to = np.array([0, len(t0), len(t0), len(t0) + len(t1)], np.uint64)
    ends0 = [1, 1, 4, 8, 11, 12]  # a, "", あ, 😀, U+FFFD, b
    ends2 = [0, 2, 5]
    te = np.array(ends0 + ends2, np.uint32)
    ido = np.array([0, 6, 6, 9], np.uint64)
    pieces = [b"p%d" % i for i in range(10)]
    ids = np.arange(9, dtype=np.int32)
    protos = decode_protos(pieces, ids, ido, text, to, te)
    assert [(p.begin, p.end) for p in protos[0]] == [(0, 1), (1, 1), (1, 2), (2, 3), (3, 4), (4, 5)]
    assert len(protos[1]) == 0 and protos[1].text == ""
    assert [(p.begin, p.end) for p in protos[2]] == [(0, 0), (0, 1), (1, 2)]
    for pr in protos:
        for p in pr:
            assert p.surface == pr.text[p.begin:p.end]
    tb = np.array([0, 1, 1, 4, 8, 11, 0, 0, 2])
    cb, ce = unicode_spans(text, to, tb, te, ido)
    assert cb.tolist() == [0, 1, 1, 2, 3, 4, 0, 0, 1] and ce.tolist() == [1, 1, 2, 3, 4, 5, 0, 1, 2]


def test_python_entry_points_fail_without_device(monkeypatch):
    from sentencepiece_b200 import _capi
    from sentencepiece_b200 import processor
    monkeypatch.setattr(_capi, "LIB_PATH", "/nonexistent/libspm_b200.so")
    monkeypatch.setattr(_capi, "_lib", None)
    with pytest.raises(RuntimeError):
        processor.Engine(model_bytes("uni32k"))
    sp = processor.SentencePieceProcessor()
    for call in (lambda: sp.decode([1, 2]), lambda: sp.Decode([[1]], out_type="immutable_proto"),
                 lambda: sp.DecodeIdsAsImmutableProto([1]), lambda: sp.decode_ids_as_immutable_proto([1]),
                 lambda: sp.DecodeIds([1], out_type=bytes)):
        with pytest.raises(RuntimeError, match="not initialized"):
            call()
