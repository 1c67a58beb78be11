"""spm_normalize (K10, normalize_kernel.cuh) and the Normalize wrappers: the normalized text and norm_to_orig of every
sentence against the oracle (which tests/test_oracle_golden.py and tests/test_oracle_charsmaps.py pin to the
reference) and against the reference's own stored result, on the golden models, every rule set of
tests/charsmap_rules.py, edge cases, chunked batches, spm_encode_spans and the C++ / Python wrappers.  Needs an H100."""
import os
import subprocess

import numpy as np
import pytest

import charsmap_rules as cr
from conftest import ROOT, model_bytes
from oracle import modelproto as mp
from oracle import oracle_py
from refstore import digest, reference
from sentencepiece_b200 import Engine, SentencePieceProcessor, _capi
from sentencepiece_b200.processor import char_index

pytestmark = pytest.mark.gpu
MODELS = ["uni32k", "botchan8k", "mix_bf8k", "bpe32k", "mix_bpe4k"]
EMPTY = _capi.NORM_TO_ORIG_EMPTY
_engines = {}


def engine(mb):
    if mb not in _engines:
        _engines[mb] = Engine(mb)
    return _engines[mb]


def split(text, no, n2o, n):
    """spm_normalize's packed result -> [(bytes, norm_to_orig list as the reference returns it)]"""
    raw = text.tobytes()
    out = []
    for i in range(n):
        a, b = int(no[i]), int(no[i + 1])
        m = None if n2o is None else n2o[a + i:b + i + 1].tolist()
        out.append((raw[a:b], None if m is None else ([] if m == [EMPTY] else m)))
    return out


def check(mb, lines, what, om=None):
    """both modes of spm_normalize == the oracle, sentence by sentence"""
    om = om or oracle_py.OracleModel(mb)
    buf, offs = oracle_py.pack(lines)
    eng = engine(mb)
    got = split(*eng.normalize(buf, offs, with_offsets=True), len(lines))
    text, no, none = eng.normalize(buf, offs)
    assert none is None
    plain = split(text, no, None, len(lines))
    for i, s in enumerate(lines):
        want = om.normalize(s)
        assert got[i] == want, (what, i, s[:80])
        assert plain[i][0] == want[0], (what, i, "with_offsets=0")
    return got


@pytest.mark.parametrize("kind", ["en", "mixed"])
@pytest.mark.parametrize("model", MODELS)
def test_golden_models(model, kind, corpus_gen):
    check(model_bytes(model), corpus_gen.lines(kind, 6100, 20000), f"{model}/{kind}")


def test_reference_result(corpus_gen):
    """the reference's own Normalize of these lines, stored by tests/test_oracle_golden.py"""
    mb = model_bytes("mix_bf8k")
    lines = corpus_gen.lines("mixed", 779, 400)
    want = reference("oracle_golden/normalize/mix_bf8k", lambda: None)
    buf, offs = oracle_py.pack(lines)
    got = split(*engine(mb).normalize(buf, offs, with_offsets=True), len(lines))
    assert digest(*((t, m) for t, m in got)) == want


@pytest.mark.parametrize("fid,flags", list(zip(cr.FLAG_IDS, cr.FLAGS)), ids=cr.FLAG_IDS)
@pytest.mark.parametrize("name", cr.ALL)
def test_rule_sets(name, fid, flags, corpus_gen):
    for base in ("uni32k", "bpe32k"):
        mb = mp.replace_flags(model_bytes(base), charsmap=cr.blob(name), **flags)
        check(mb, cr.lines(name, corpus_gen, 5200, 800), f"{base}/{name}/{fid}")


def test_user_symbols_win_over_rules(corpus_gen):
    from test_gpu_normalizer_rules import user_symbol_lines, user_symbol_models
    lines = user_symbol_lines(corpus_gen)
    for base, name, mb in user_symbol_models():
        check(mb, lines, f"{base}/{name} user symbols")


def test_set_types_user_defined(corpus_gen):
    """after spm_engine_set_types the output follows the live types, as encode's normalizer does: USER_DEFINED pieces
    stay verbatim while other pieces turn UNUSED and back"""
    from test_gpu_normalizer_rules import user_symbol_lines, user_symbol_models
    lines = user_symbol_lines(corpus_gen)
    base, name, mb = user_symbol_models()[0]
    om = oracle_py.OracleModel(mb)
    eng = Engine(mb)
    t = om.types.copy()
    t[(t == mp.NORMAL) & (np.arange(len(t)) % 2 == 0)] = mp.UNUSED
    eng.set_types(t)
    om.set_types(t)
    buf, offs = oracle_py.pack(lines)
    got = split(*eng.normalize(buf, offs, with_offsets=True), len(lines))
    assert got == [om.normalize(s) for s in lines]
    r = eng.encode_spans(buf, offs)
    for i, (txt, m) in enumerate(got):
        na, nb = int(r["norm_offsets"][i]), int(r["norm_offsets"][i + 1])
        assert r["normalized"][na:nb] == txt
    eng.close()


def edge_lines():
    return [b"", b" ", b"   ", b"\t \n", b"a", b" a ", b"  a  b  ", b"\x00", b"a\x00b", b"\x00 \x00",
            b"\xff", b"\xe3\x81", b"a\xe3\x81b\xff\xfe", b"\xc0\x80", b"\xed\xa0\x80", b"\xf4\x90\x80\x80",
            "　　x　".encode(), "ｈｅｌｌｏ　ｗｏｒｌｄ".encode(), "▁".encode(), b"x" * 600,
            ("word " * 13107).encode()[:65536], ("été " * 90000).encode()[:1 << 20]]


@pytest.mark.parametrize("model", ["uni32k", "mix_bf8k", "bpe32k"])
def test_edges(model, corpus_gen):
    lines = edge_lines() + corpus_gen.lines("mixed", 6200, 200)
    check(model_bytes(model), lines, f"{model} edges")
    got = check(mp.replace_flags(model_bytes("uni32k"), charsmap=cr.blob("delete_expand")), lines, "delete_expand")
    assert got[0] == (b"", [])


def test_empty_batch_and_first_offset():
    eng = engine(model_bytes("uni32k"))
    text, no, n2o = eng.normalize(np.zeros(0, np.uint8), np.zeros(1, np.uint64), with_offsets=True)
    assert len(text) == 0 and no.tolist() == [0]
    om = oracle_py.OracleModel(model_bytes("uni32k"))
    raw = b"XXXXhello  world  \xe3\x81\x82 x"
    buf = np.frombuffer(raw, np.uint8)
    offs = np.array([4, 9, 9, 18, len(raw)], np.uint64)
    got = split(*eng.normalize(buf, offs, with_offsets=True), 4)
    assert got == [om.normalize(raw[int(offs[i]):int(offs[i + 1])]) for i in range(4)]


def test_chunked_batch_and_spans(corpus_gen):
    """300k sentences span several chunks; spm_encode_spans' text and norm_to_orig are the same wherever it defines
    them (a sentence that normalizes to nothing has no norm_to_orig there)"""
    mb = model_bytes("uni32k")
    buf, offs = corpus_gen.fill("en", 6300, 300000)
    eng = engine(mb)
    text, no, n2o = eng.normalize(buf, offs, with_offsets=True)
    r = eng.encode_spans(buf, offs)
    assert np.array_equal(no, r["norm_offsets"]) and text.tobytes() == r["normalized"]
    lens = np.diff(no.astype(np.int64))
    keep = np.repeat(lens > 0, lens + 1)
    assert np.array_equal(n2o[keep], r["n2o"][keep])
    t2, no2, _ = eng.normalize(buf, offs)
    assert np.array_equal(no2, no) and np.array_equal(t2, text)
    om = oracle_py.OracleModel(mb)
    o = offs.astype(np.int64)
    got = split(text, no, n2o, 300000)
    for i in range(0, 300000, 997):
        assert got[i] == om.normalize(buf[o[i]:o[i + 1]].tobytes()), i


def test_errors():
    eng = engine(model_bytes("uni32k"))
    buf = np.frombuffer(b"abc", np.uint8)
    with pytest.raises(RuntimeError, match="non-decreasing"):
        eng.normalize(buf, np.array([0, 2, 1], np.uint64))


def test_cpp_class(corpus_gen, tmp_path):
    lib = os.path.join(ROOT, "sentencepiece_b200", "lib")
    exe = str(tmp_path / "normalize_class_check")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-pthread", "-I" + os.path.join(ROOT, "sentencepiece_b200", "csrc"),
                           "-I" + os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "normalize_class_check.cc"),
                           os.path.join(lib, "sentencepiece_processor.o"), os.path.join(lib, "model_reader.o"),
                           "-L" + os.path.join(lib, "stdcxx"), "-L" + lib, "-lspm_b200", "-Wl,-rpath," + lib])
    lines = edge_lines()[:-1] + corpus_gen.lines("mixed", 6400, 300)
    inp = tmp_path / "in.txt"
    inp.write_text("".join(s.hex() + "\n" for s in lines))
    for model in ("uni32k", "bpe32k"):
        out = subprocess.check_output([exe, os.path.join(ROOT, "tests", "golden", "models", model + ".model"), str(inp)])
        om = oracle_py.OracleModel(model_bytes(model))
        rows = out.decode().splitlines()
        assert len(rows) == len(lines)
        for s, row in zip(lines, rows):
            h, *m = row.split(" ")
            t, want = om.normalize(s)
            assert bytes.fromhex(h) == t
            assert ([] if m == ["-"] else [int(x) for x in m]) == want, s[:60]
    assert rows[0].endswith(" -")  # empty input: empty norm_to_orig


def u2u(s):
    """utf8_to_unicode_offsets of ConvertToUnicodeAlignment (sentencepiece_trainer.cc:369-385); a last step past the end
    of malformed input stops at the end"""
    out, prev, ulen = [0] * (len(s) + 1), 0, 0
    while prev < len(s):
        ln = min(([1] * 12 + [2, 2, 3, 4])[s[prev] >> 4], len(s) - prev)
        for i in range(prev, prev + ln):
            out[i] = ulen
        ulen, prev = ulen + 1, prev + ln
    out[prev] = ulen
    return out


def unicode_restated(orig, norm, n2o):
    """ConvertToUnicodeAlignment (sentencepiece_trainer.cc:369-397), line by line"""
    oo, no = u2u(orig), u2u(norm)
    res = [0] * (no[-1] + 1)
    for i, v in enumerate(n2o):
        res[no[i]] = oo[v]
    return res


def test_python_api(corpus_gen):
    mb = model_bytes("mix_bf8k")
    sp = SentencePieceProcessor(model_proto=mb)
    om = oracle_py.OracleModel(mb)
    lines = [s for s in edge_lines()[:-2] + corpus_gen.lines("mixed", 6500, 300)]
    strs = [s.decode("utf-8", "replace") for s in lines]
    got = sp.Normalize(strs, with_offsets=True)
    for s, (t, m) in zip(strs, got):
        wt, wm = om.normalize(s.encode())
        assert t == wt.decode() and m == unicode_restated(s.encode(), wt, wm), s[:60]
    assert sp.normalize(strs) == [t for t, _ in got]
    assert sp.Normalize(strs[30]) == got[30][0]
    assert sp.Normalize(strs[30], with_offsets=True) == got[30]
    assert sp.Normalize("") == "" and sp.Normalize("", with_offsets=True) == ("", [0])
    bgot = sp.Normalize(lines, with_offsets=True)
    for s, (t, m) in zip(lines, bgot):
        assert (t, m) == om.normalize(s)
    assert sp.Normalize(b"", with_offsets=True) == (b"", [])
    assert sp.Normalize(lines[40]) == bgot[40][0]
    # the vectorised character table against the restatement, malformed sentences included
    buf, offs = oracle_py.pack(lines)
    ci = char_index(buf, offs)
    for i, s in enumerate(lines):
        a = int(offs[i]) + i
        assert ci[a:a + len(s) + 1].tolist() == u2u(s), i
