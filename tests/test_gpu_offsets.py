"""spm_encode_offsets (K11, offsets_kernel.cuh) and EncodeAsImmutableProto: ids against spm_encode_ids, pieces against
spm_encode_pieces, and every token's begin / end against a restatement of PopulateSentencePieceText and
ApplyExtraOptions (src/sentencepiece_processor.cc:547-636, 1019-1064) over the oracle's normalize and model_encode,
which tests/test_oracle_golden.py pins to the reference; ids, pieces, surfaces and begin / end also against digests
of the unmodified reference's SentencePieceText (tests/offsets_cases.py).  Golden models under every frame, rule sets and normalizer
flags, user-defined and UNUSED pieces, edge lines, long sentences, chunked batches, the spans-derived route, the C++
class and the Python API.  Needs an H100."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import charsmap_rules as cr
from conftest import ROOT, model_bytes
from oracle import modelproto as mp
from oracle import oracle_py
from sentencepiece_b200 import Engine, SentencePieceProcessor, _modelinfo
from sentencepiece_b200.processor import extra_frame
from offsets_cases import framed, options_of, restated
from test_gpu_normalize import edge_lines, u2u
import offsets_cases as oc
from offsets_bench import offsets_from_spans

pytestmark = pytest.mark.gpu
MODELS = ["uni32k", "botchan8k", "mix_bf8k", "bpe32k", "mix_bpe4k"]
FRAMES = ["", "bos:eos", "reverse", "eos:reverse:bos", "unk", "reverse:unk:eos"]
_engines = {}


def engine(mb):
    if mb not in _engines:
        _engines[mb] = Engine(mb)
    return _engines[mb]


def set_frame(eng, sp, options):
    prefix, rev, suffix = extra_frame(options, sp["bos_id"], sp["eos_id"])
    eng.set_encode_frame(prefix, rev, suffix)
    return sp["unk_piece"] if "unk" in options else None


def check(mb, lines, what, frames=FRAMES, om=None, eng=None):
    om = om or oracle_py.OracleModel(mb)
    eng = eng or engine(mb)
    sp = _modelinfo.special_pieces(mb)
    want = [restated(om, s) for s in lines]
    buf, offs = oracle_py.pack(lines)
    try:
        for fr in frames:
            opts = options_of(fr)
            unk = set_frame(eng, sp, opts)
            r = eng.encode_offsets(buf, offs, eos_id=sp["eos_id"], unk_piece=unk)
            ids, ido = eng.encode_packed(buf, offs)
            assert np.array_equal(r["ids"], ids) and np.array_equal(r["id_offsets"], ido), (what, fr)
            p = eng.encode_pieces(buf, offs, unk_piece=unk)
            for k in ("text", "text_offsets", "piece_end"):
                assert np.array_equal(r[k], p[k]), (what, fr, k)
            q = eng.encode_offsets(buf, offs, eos_id=sp["eos_id"], unk_piece=unk, pieces=False)
            assert "text" not in q
            for k in ("ids", "id_offsets", "begin", "end"):
                assert np.array_equal(q[k], r[k]), (what, fr, k)
            b, e = r["begin"].tolist(), r["end"].tolist()
            for i, s in enumerate(lines):
                a, z = int(ido[i]), int(ido[i + 1])
                got = list(zip(b[a:z], e[a:z]))
                assert got == framed(want[i], len(s), opts, sp), (what, fr, i, s[:80])
    finally:
        eng.set_encode_frame()


@pytest.mark.parametrize("kind", ["en", "mixed"])
@pytest.mark.parametrize("model", MODELS)
def test_golden_models(model, kind, corpus_gen):
    check(model_bytes(model), corpus_gen.lines(kind, 7100, 20000), f"{model}/{kind}")


@pytest.mark.parametrize("model", oc.MODELS)
def test_reference_digests(model, corpus_gen):
    """ids, pieces, surfaces and begin / end of every sentence equal the unmodified reference's SentencePieceText
    (tests/offsets_cases.py, recorded by tools/record_offsets_reference.py) under every option mix"""
    mb = model_bytes(model)
    eng = engine(mb)
    sp = _modelinfo.special_pieces(mb)
    want = oc.stored()
    try:
        for name in oc.INPUTS:
            lines = oc.inputs(corpus_gen, name)
            buf, offs = oracle_py.pack(lines)
            for fr in oc.FRAMES:
                unk = set_frame(eng, sp, options_of(fr))
                r = eng.encode_offsets(buf, offs, eos_id=sp["eos_id"], unk_piece=unk)
                assert oc.digest(oc.engine_rows(lines, r)) == want[oc.key(model, name, fr)], (model, name, fr)
    finally:
        eng.set_encode_frame()


def test_unknown_runs_and_byte_fallback(corpus_gen):
    """uni32k on mixed text has unknown runs (the detour runs with and without unk_piece); mix_bf8k splits unknown
    characters into byte tokens, whose surfaces sit on the last byte"""
    lines = corpus_gen.lines("mixed", 7150, 3000)
    buf, offs = oracle_py.pack(lines)
    eng = engine(model_bytes("uni32k"))
    for unk in (None, "<unk>"):
        eng.encode_offsets(buf, offs, unk_piece=unk, pieces=unk is None)
        assert eng.info().last_unk_detour > 0
    r = engine(model_bytes("mix_bf8k")).encode_offsets(buf, offs)
    zero = r["begin"] == r["end"]
    assert zero.any() and (~zero).any()


@pytest.mark.parametrize("name", ["delete_expand"] + [n for n in cr.ALL if n != "delete_expand"][:2])
@pytest.mark.parametrize("fid", ["default", "no_prefix", "suffix"])
def test_rule_sets(name, fid, corpus_gen):
    flags = cr.FLAGS[cr.FLAG_IDS.index(fid)]
    # (delete_expand turns a character into 200 bytes: BPE over such sentences takes minutes)
    for base in ("uni32k",) if name == "delete_expand" else ("uni32k", "bpe32k"):
        mb = mp.replace_flags(model_bytes(base), charsmap=cr.blob(name), **flags)
        check(mb, cr.lines(name, corpus_gen, 7200, 600), f"{base}/{name}/{fid}", frames=["", "eos:reverse:bos"],
              eng=Engine(mb))


def test_user_defined_and_unused(corpus_gen):
    from test_gpu_normalizer_rules import user_symbol_lines, user_symbol_models
    lines = user_symbol_lines(corpus_gen)
    for base, name, mb in user_symbol_models():
        check(mb, lines, f"{base}/{name} user symbols", frames=["", "reverse:unk:eos"], eng=Engine(mb))
    base, name, mb = user_symbol_models()[0]
    om = oracle_py.OracleModel(mb)
    eng = Engine(mb)
    t = om.types.copy()
    t[(t == mp.NORMAL) & (np.arange(len(t)) % 2 == 0)] = mp.UNUSED
    eng.set_types(t)
    om.set_types(t)
    check(mb, lines, "set_types UNUSED", frames=["", "bos:eos"], om=om, eng=eng)


@pytest.mark.parametrize("model", ["uni32k", "mix_bf8k", "bpe32k"])
def test_edges(model, corpus_gen):
    """empty, whitespace-only, NUL and malformed lines, 600 B / 64 KB / 1 MB sentences"""
    # (BPE merges over the 64 KB and 1 MB one-line documents take minutes; the BPE model gets the others)
    lines = edge_lines()[:-2 if model == "bpe32k" else None] + corpus_gen.lines("mixed", 7300, 200)
    check(model_bytes(model), lines, f"{model} edges", frames=["", "eos:reverse:bos"])
    check(mp.replace_flags(model_bytes("uni32k"), charsmap=cr.blob("delete_expand")), lines, "delete_expand edges",
          frames=[""])


def test_empty_batch_and_first_offset():
    mb = model_bytes("uni32k")
    eng = engine(mb)
    for pieces in (True, False):
        r = eng.encode_offsets(np.zeros(0, np.uint8), np.zeros(1, np.uint64), pieces=pieces)
        assert r["id_offsets"].tolist() == [0] and len(r["ids"]) == 0 and len(r["begin"]) == 0
        i = eng.info()  # nothing left over from the previous call
        assert (i.last_h2d_bytes, i.last_d2h_bytes, i.last_kernel_launches, i.last_kernel_ms) == (0, 0, 0, 0.0)
        eng.encode_offsets(np.frombuffer(b"hello", np.uint8), np.array([0, 5], np.uint64))
    om = oracle_py.OracleModel(mb)
    raw = b"XXXXhello  world  \xe3\x81\x82 x\xe2\x80\xbb"
    buf = np.frombuffer(raw, np.uint8)
    offs = np.array([4, 9, 9, 18, len(raw)], np.uint64)
    r = eng.encode_offsets(buf, offs)
    for i in range(4):
        a, z = int(r["id_offsets"][i]), int(r["id_offsets"][i + 1])
        s = raw[int(offs[i]):int(offs[i + 1])]
        assert list(zip(r["begin"][a:z].tolist(), r["end"][a:z].tolist())) == restated(om, s)


@pytest.mark.parametrize("model", ["uni32k", "mix_bf8k"])
def test_chunked_batch_and_spans_route(model, corpus_gen):
    """300k sentences span several K11 chunks: ids as spm_encode_ids, offsets as derived from spm_encode_spans"""
    mb = model_bytes(model)
    buf, offs = corpus_gen.fill("en" if model == "uni32k" else "mixed", 7400, 300000)
    eng = engine(mb)
    r = eng.encode_offsets(buf, offs, pieces=False)
    ids, ido = eng.encode_packed(buf, offs)
    assert np.array_equal(r["ids"], ids) and np.array_equal(r["id_offsets"], ido)
    sp = eng.encode_spans(buf, offs)
    b, e = offsets_from_spans(sp, oracle_py.OracleModel(mb).types)
    assert np.array_equal(r["begin"], b) and np.array_equal(r["end"], e)
    om = oracle_py.OracleModel(mb)
    o = offs.astype(np.int64)
    for i in range(0, 300000, 1499):
        a, z = int(ido[i]), int(ido[i + 1])
        assert list(zip(r["begin"][a:z].tolist(), r["end"][a:z].tolist())) == restated(om, buf[o[i]:o[i + 1]].tobytes())


def test_errors():
    eng = engine(model_bytes("uni32k"))
    buf = np.frombuffer(b"abc", np.uint8)
    with pytest.raises(RuntimeError, match="non-decreasing"):
        eng.encode_offsets(buf, np.array([0, 2, 1], np.uint64))
    with pytest.raises(RuntimeError, match="sep"):
        eng.encode_offsets(buf, np.array([0, 3], np.uint64), sep=300)
    L = eng._lib
    offs = np.array([0, 3], np.uint64)
    p = [ctypes.c_void_p() for _ in range(7)]
    ref = [ctypes.byref(x) for x in p]
    assert L.spm_encode_offsets(eng._h, buf.ctypes.data, offs.ctypes.data, 1, -1, None, 3, -1, *ref) == 1  # len, no piece
    assert L.spm_encode_offsets(eng._h, buf.ctypes.data, offs.ctypes.data, 1, -1, None, 0, -1, None, *ref[1:]) == 1
    assert L.spm_encode_offsets(eng._h, buf.ctypes.data, offs.ctypes.data, 1, -1, None, 0, -1, *ref[:4], ref[4], None,
                                ref[6]) == 1  # text without text_offsets
    assert L.spm_encode_offsets(None, buf.ctypes.data, offs.ctypes.data, 1, -1, None, 0, -1, *ref) == 1


def test_cpp_class(corpus_gen, tmp_path):
    lib = os.path.join(ROOT, "sentencepiece_b200", "lib")
    exe = str(tmp_path / "offsets_class_check")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(ROOT, "sentencepiece_b200", "csrc"),
                           "-I" + os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "offsets_class_check.cc"),
                           os.path.join(lib, "sentencepiece_processor.o"), os.path.join(lib, "model_reader.o"),
                           "-L" + os.path.join(lib, "stdcxx"), "-L" + lib, "-lspm_b200", "-Wl,-rpath," + lib])
    lines = edge_lines()[:-2] + corpus_gen.lines("mixed", 7500, 300)  # (no one-line documents: BPE takes minutes)
    inp = tmp_path / "in.txt"
    inp.write_text("".join(s.hex() + "\n" for s in lines))
    buf, offs = oracle_py.pack(lines)
    for model, frame in (("uni32k", "bos:eos"), ("mix_bf8k", "reverse:unk:eos"), ("bpe32k", "")):
        mb = model_bytes(model)
        out = subprocess.check_output([exe, os.path.join(ROOT, "tests", "golden", "models", model + ".model"), str(inp),
                                       frame or "-"])
        rows = out.decode().splitlines()
        assert len(rows) == len(lines) + 1
        eng = engine(mb)
        sp = _modelinfo.special_pieces(mb)
        try:
            unk = set_frame(eng, sp, options_of(frame))
            r = eng.encode_offsets(buf, offs, eos_id=sp["eos_id"], unk_piece=unk)
        finally:
            eng.set_encode_frame()
        ido, pe, text, to = r["id_offsets"], r["piece_end"], r["text"].tobytes(), r["text_offsets"]
        for i, s in enumerate(lines):
            want = []
            t = text[int(to[i]):int(to[i + 1])]
            for k in range(int(ido[i]), int(ido[i + 1])):
                b, e = int(r["begin"][k]), int(r["end"][k])
                p0 = int(pe[k - 1]) if k > int(ido[i]) else 0
                want.append(f"{t[p0:int(pe[k])].hex()}:{int(r['ids'][k])}:{s[b:e].hex()}:{b}:{e}")
            assert rows[i] == " ".join(want), (model, i)
        assert rows[-1] == rows[len(lines) - 1]  # the single-sentence overload


def chars(s, spans):
    m = u2u(s)
    clip = lambda x: m[min(max(0, x), len(s))]
    return [(clip(b), clip(e)) for b, e in spans]


def test_python_api(corpus_gen):
    mb = model_bytes("mix_bf8k")
    spp = SentencePieceProcessor(model_proto=mb)
    om = oracle_py.OracleModel(mb)
    sp = _modelinfo.special_pieces(mb)
    lines = edge_lines()[:-2] + corpus_gen.lines("mixed", 7600, 300)
    strs = [s.decode("utf-8", "replace") for s in lines]
    got = spp.EncodeAsImmutableProto(strs)
    ids = spp.EncodeAsIds(strs)
    pieces = spp.EncodeAsPieces(strs)
    for s, g, i, p in zip(strs, got, ids, pieces):
        raw = s.encode()
        want = chars(raw, restated(om, raw))
        assert [(x.begin, x.end) for x in g] == want, s[:60]
        assert [x.id for x in g] == i and [x.piece for x in g] == p
        assert all(x.surface_as_bytes == raw[x2b(raw, x.begin):x2b(raw, x.end)] for x in g)
        assert g.text == s and len(g) == len(g.pieces) == len(i)
    assert spp.encode_as_immutable_proto(strs[30]) == got[30]
    assert spp.encode(strs[30], out_type="immutable_proto") == got[30]
    assert spp.encode(strs[:5], out_type="immutable_proto") == got[:5]
    assert list(iter(got[30])) == list(got[30].pieces) and got[30][-1] == got[30].pieces[-1]
    with pytest.raises(AttributeError):
        got[30][0].begin = 3
    bgot = spp.EncodeAsImmutableProto(lines)
    for s, g in zip(lines, bgot):
        assert [(x.begin, x.end) for x in g] == chars(s, restated(om, s))
        assert g.text_as_bytes == s
    # SetEncodeExtraOptions' options apply before the conversion
    spp.SetEncodeExtraOptions("bos:eos")
    g = spp.EncodeAsImmutableProto("héllo wörld")
    n = len("héllo wörld")
    assert (g[0].id, g[0].begin, g[0].end) == (sp["bos_id"], 0, 0) and (g[-1].id, g[-1].begin, g[-1].end) == (sp["eos_id"], n, n)
    spp.SetEncodeExtraOptions("")
    for kw in ("add_bos", "add_eos", "reverse", "emit_unk_piece"):
        with pytest.raises(RuntimeError, match="not supported in proto API"):
            spp.EncodeAsImmutableProto("x", **{kw: True})
    with pytest.raises(NotImplementedError):
        spp.encode("x", out_type="immutable_proto", enable_sampling=True)


def x2b(raw, ci):
    """the byte offset of character index ci (the inverse of u2u on character starts)"""
    m = u2u(raw)
    return m.index(ci) if ci < m[-1] else len(raw)
