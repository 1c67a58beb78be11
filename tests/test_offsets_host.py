"""Host side of EncodeAsImmutableProto, CPU only: the vectorised ConvertToUnicodeSpans against the reference's rule
and its own expectations, the clip, the read-only result objects, the call failing loudly where no device is present,
and the restatement of PopulateSentencePieceText / ApplyExtraOptions that tests/test_gpu_offsets.py checks every
sentence against, pinned here to the unmodified reference's digests."""
import numpy as np
import pytest

import offsets_cases as oc
from conftest import model_bytes
from sentencepiece_b200.processor import (ImmutableSentencePiece, ImmutableSentencePieceText, immutable_protos,
                                          pack_sentences, unicode_spans)


def restated(text, spans):
    """ConvertToUnicodeSpans (sentencepiece_processor.cc:63-91), line by line; a last character whose lead byte claims
    more bytes than remain ends at the end"""
    if not text:
        return list(spans)
    m, prev, ulen = [0] * (len(text) + 1), 0, 0
    while prev < len(text):
        ln = min(max(1, ([1] * 12 + [2, 2, 3, 4])[text[prev] >> 4]), len(text) - prev)
        for i in range(prev, prev + ln):
            m[i] = ulen
        ulen, prev = ulen + 1, prev + ln
    m[prev] = ulen
    clip = lambda s: min(max(0, s), len(m) - 1)
    return [(m[clip(b)], m[clip(e)]) for b, e in spans]


def convert(items):
    """[(text bytes, [(begin, end)])] -> character spans per item through the batch helper"""
    buf, offs = pack_sentences([t for t, _ in items])
    ido = np.zeros(len(items) + 1, np.uint64)
    ido[1:] = np.cumsum([len(s) for _, s in items])
    b = np.array([x for _, s in items for x, _ in s], np.uint32)
    e = np.array([y for _, s in items for _, y in s], np.uint32)
    cb, ce = unicode_spans(buf, offs, b, e, ido)
    out = []
    for i in range(len(items)):
        a, z = int(ido[i]), int(ido[i + 1])
        out.append(list(zip(cb[a:z].tolist(), ce[a:z].tolist())))
    return out


def tokens(toks):
    """ConvertToUnicodeSpansTest's make_spt: consecutive tokens, byte spans"""
    spans, prev = [], 0
    for t in toks:
        b = t.encode()
        spans.append((prev, prev + len(b)))
        prev += len(b)
    return "".join(toks).encode(), spans


def test_reference_expectations():
    """sentencepiece_processor_test.cc:1657-1710"""
    cases = [(["hello", "_world", "."], [(0, 5), (5, 11), (11, 12)]),
             (["これは", "test", "です"], [(0, 3), (3, 7), (7, 9)]),
             (["いABは", "にほCD", "へと"], [(0, 4), (4, 8), (8, 10)])]
    got = convert([tokens(t) for t, _ in cases])
    assert got == [w for _, w in cases]


def test_against_rule():
    items = [
        (b"", [(0, 0), (0, 0)]),                                  # empty text: left as is
        (b"abc", [(0, 0), (0, 1), (1, 3), (3, 3)]),
        ("日本語".encode(), [(0, 3), (3, 3), (3, 9), (9, 9)]),       # byte tokens: begin == end
        ("é x".encode(), [(0, 2), (2, 4)]),
        (b"a\xffb", [(0, 1), (1, 2), (2, 3)]),                      # a malformed byte is one character
        (b"\x80\x80x", [(0, 1), (1, 2), (2, 3)]),
        (b"ab\xe3", [(0, 2), (2, 3), (3, 3)]),                      # truncated lead byte at the end
        (b"ab\xf0c", [(0, 2), (2, 4)]),
        ("ｈｅｌｌｏ".encode(), [(0, 6), (6, 15)]),
    ]
    assert convert(items) == [restated(t, s) for t, s in items]
    # the clip: offsets past the end map to the character count
    buf, offs = pack_sentences([b"abc"])
    cb, ce = unicode_spans(buf, offs, np.array([7], np.uint32), np.array([9], np.uint32), np.array([0, 1], np.uint64))
    assert (cb.tolist(), ce.tolist()) == ([3], [3])


def test_objects():
    text = "a é".encode()
    r = dict(ids=np.array([5, 9, 7], np.int32), id_offsets=np.array([0, 3], np.uint64),
             begin=np.array([0, 1, 2], np.uint32), end=np.array([1, 2, 4], np.uint32),
             text=np.frombuffer("▁a▁é".encode(), np.uint8), text_offsets=np.array([0, 9], np.uint64),
             piece_end=np.array([4, 7, 9], np.uint32))
    buf, offs = pack_sentences([text])
    (t,) = immutable_protos([text], buf, offs, r)
    assert isinstance(t, ImmutableSentencePieceText) and t.text == "a é" and t.text_as_bytes == text
    assert len(t) == 3 and [p.piece for p in t] == ["▁a", "▁", "é"]
    assert [(p.id, p.begin, p.end, p.surface) for p in t.pieces] == [(5, 0, 1, "a"), (9, 1, 2, " "), (7, 2, 3, "é")]
    assert t[-1].surface_as_bytes == "é".encode() and t[1:] == t.pieces[1:]
    assert t[0] == ImmutableSentencePiece("▁a".encode(), 5, b"a", 0, 1)
    for attr in ("piece", "id", "surface", "begin", "end"):
        with pytest.raises(AttributeError):
            setattr(t[0], attr, 1)
    with pytest.raises(AttributeError):
        t.text = "x"
    assert "begin: 2" in repr(t)
    assert t != None and t[0] != None and t != "a é" and t[0] != (5, 0, 1)  # noqa: E711


def test_fail_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible here; the failure path is for GPU-less boxes")
    from sentencepiece_b200 import Engine, SentencePieceProcessor
    buf, offs = np.frombuffer(b"hello", np.uint8), np.array([0, 5], np.uint64)
    with pytest.raises(RuntimeError, match="no CPU fallback|CUDA"):
        Engine(model_bytes("uni32k")).encode_offsets(buf, offs)
    with pytest.raises(RuntimeError, match="no CPU fallback|CUDA"):
        SentencePieceProcessor(model_proto=model_bytes("uni32k")).EncodeAsImmutableProto("hello")
    with pytest.raises(RuntimeError, match="not initialized"):
        SentencePieceProcessor().encode("hello", out_type="immutable_proto")


@pytest.mark.parametrize("model", oc.MODELS)
def test_restatement_matches_reference(model, corpus_gen):
    """ids and surfaces from the oracle's encode, pieces from the model (the normalized surface for unknown runs),
    begin / end from offsets_cases.restated / framed: equal to the reference's SentencePieceText in every case"""
    from oracle import oracle_py
    from sentencepiece_b200 import _modelinfo
    mb = model_bytes(model)
    om = oracle_py.OracleModel(mb)
    sp = _modelinfo.special_pieces(mb)
    pieces = om.proto["pieces"]
    unk_piece = sp["unk_piece"].encode() if isinstance(sp["unk_piece"], str) else sp["unk_piece"]
    want = oc.stored()
    for name in oc.INPUTS:
        lines = oc.inputs(corpus_gen, name)
        base = []
        for s in lines:
            norm, _ = om.normalize(s)
            ids, te = om.encode(s)
            spans = oc.restated(om, s)
            assert len(spans) == len(ids)
            toks, c = [], 0
            for i, e, (b, en) in zip(ids.tolist(), te.tolist(), spans):
                toks.append((i, norm[c:e] if i == om.unk_id else pieces[i], s[b:en], b, en))
                c = e
            base.append(toks)
        for fr in oc.FRAMES:
            opts = oc.options_of(fr)
            rows = []
            for s, toks in zip(lines, base):
                spans = oc.framed([(b, e) for *_, b, e in toks], len(s), opts, sp)
                t = list(toks)
                for o in opts:
                    if o == "reverse":
                        t.reverse()
                    elif o == "bos":
                        t.insert(0, (sp["bos_id"], pieces[sp["bos_id"]]))
                    elif o == "eos":
                        t.append((sp["eos_id"], pieces[sp["eos_id"]]))
                unk = "unk" in opts
                rows.append(oc.row([(x[0], unk_piece if unk and x[0] == om.unk_id else x[1], s[b:e], b, e)
                                    for x, (b, e) in zip(t, spans)]))
            assert oc.digest(rows) == want[oc.key(model, name, fr)], (model, name, fr)
