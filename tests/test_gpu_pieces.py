"""spm_encode_pieces (EncodeAsPieces on the device, K9): piece strings and framed ids against the reference's
EncodeAsPieces (stored digests, tests/refstore_pieces.py), against the spans path plus host assembly it replaces, and
through every layer above it -- Python mirror, C++ class, spm_encode_b200 --output_format=piece.  Needs an H100."""
import itertools
import os
import subprocess

import numpy as np
import pytest

from conftest import MODELS_DIR, ROOT, model_bytes
from extra_options import set_reference_options
from oracle import modelproto as mp
from oracle import oracle_py
from refstore import digest
from refstore_pieces import pieces_digest, reference

pytestmark = pytest.mark.gpu
ALL_MODELS = ["uni32k", "mix_bf8k", "botchan8k", "bpe32k", "mix_bpe4k"]
CLI = os.path.join(ROOT, "sentencepiece_b200", "lib", "spm_encode_b200")
REF_CLI = os.path.join(ROOT, "oracle", "_ref", "spm_encode")
U2581 = "▁".encode()


def _engine(mb):
    from sentencepiece_b200 import Engine
    return Engine(mb)


def _special(mb):
    from sentencepiece_b200 import _modelinfo
    return _modelinfo.special_pieces(mb)


def _rows(r):
    """packed spm_encode_pieces output (sep = -1) -> list of lists of piece bytes"""
    raw = r["text"].tobytes()
    to, ido, pe = r["text_offsets"].tolist(), r["id_offsets"].tolist(), r["piece_end"].tolist()
    out = []
    for i in range(len(to) - 1):
        s = raw[to[i]:to[i + 1]]
        ends = pe[ido[i]:ido[i + 1]]
        out.append([s[b:e] for b, e in zip([0] + ends[:-1], ends)])
    return out


def _ref_rows(mb, lines, options=""):
    ref = oracle_py.RefModel(mb)
    if options:
        set_reference_options(ref, options)
    return [ref.encode_pieces(s) for s in lines]


def _ref_digest(mb, lines, options=""):
    ref = oracle_py.RefModel(mb)
    if options:
        set_reference_options(ref, options)
    rows = [ref.encode_pieces(s) for s in lines]
    ids = np.concatenate([ref.encode(s) for s in lines] + [np.zeros(0, np.int32)])
    return pieces_digest(rows, ids)


def _old_rows(eng, mb, buf, offs, options=""):
    """what EncodeAsPieces did before: spm_encode_spans (raw segmentation), IdToPiece / the normalized surface of
    unknown tokens on the host, then ApplyExtraOptions on (piece, id) pairs"""
    from sentencepiece_b200 import _modelinfo
    pieces, unk = _modelinfo.pieces_and_unk(mb)
    pieces = [p.encode() for p in pieces]
    sp = _special(mb)
    r = eng.encode_spans(buf, offs)
    ids, te, ido, no, norm = r["ids"].tolist(), r["tok_end"].tolist(), r["id_offsets"].tolist(), r["norm_offsets"].tolist(), r["normalized"]
    rows, id_rows = [], []
    for i in range(len(offs) - 1):
        pairs, begin = [], 0
        for k in range(ido[i], ido[i + 1]):
            pairs.append((norm[no[i] + begin:no[i] + te[k]] if ids[k] == unk else pieces[ids[k]], ids[k]))
            begin = te[k]
        for o in options.split(":") if options else []:
            if o == "reverse":
                pairs.reverse()
            elif o == "bos":
                pairs.insert(0, (sp["bos_piece"].encode(), sp["bos_id"]))
            elif o == "eos":
                pairs.append((sp["eos_piece"].encode(), sp["eos_id"]))
            elif o == "unk":
                pairs = [(sp["unk_piece"].encode(), d) if d == unk else (p, d) for p, d in pairs]
        rows.append([p for p, _ in pairs])
        id_rows.append([d for _, d in pairs])
    return rows, id_rows


def _set_options(eng, mb, options):
    from sentencepiece_b200.processor import extra_frame
    sp = _special(mb)
    opts = options.split(":") if options else []
    p, rev, s = extra_frame(opts, sp["bos_id"], sp["eos_id"])
    eng.set_encode_frame(p, rev, s)
    return sp["unk_piece"] if "unk" in opts else None


def _check(eng, mb, buf, offs, options="", sep_too=False):
    """spm_encode_pieces == the old path, and its ids == spm_encode_ids under the same frame; returns the pieces"""
    unk = _set_options(eng, mb, options)
    r = eng.encode_pieces(buf, offs, unk_piece=unk)
    ids, ido = eng.encode_packed(buf, offs)
    assert np.array_equal(r["id_offsets"], ido) and np.array_equal(r["ids"], ids), options
    _set_options(eng, mb, "")
    want, want_ids = _old_rows(eng, mb, buf, offs, options)
    got = _rows(r)
    assert got == want, options
    assert [r["ids"][int(ido[i]):int(ido[i + 1])].tolist() for i in range(len(got))] == want_ids
    if sep_too:
        _set_options(eng, mb, options)
        j = eng.encode_pieces(buf, offs, unk_piece=unk, sep=ord(" "))
        raw = j["text"].tobytes()
        to = j["text_offsets"].tolist()
        assert [raw[to[i]:to[i + 1]] for i in range(len(got))] == [b" ".join(row) for row in got]
        assert np.array_equal(j["ids"], r["ids"])
    _set_options(eng, mb, "")
    return got


# ---- 1. reference parity ----

@pytest.mark.parametrize("kind", ["en", "mixed"])
@pytest.mark.parametrize("model", ALL_MODELS)
def test_reference_parity(model, kind, corpus_gen):
    mb = model_bytes(model)
    lines = corpus_gen.lines(kind, 9191, 20000)
    want = reference(f"parity/{model}/{kind}", lambda: _ref_digest(mb, lines))
    buf, offs = oracle_py.pack(lines)
    eng = _engine(mb)
    r = eng.encode_pieces(buf, offs)
    assert pieces_digest(_rows(r), r["ids"]) == want
    ids, ido = eng.encode_packed(buf, offs)
    assert np.array_equal(r["ids"], ids) and np.array_equal(r["id_offsets"], ido)
    if model in ("uni32k", "botchan8k") and kind == "mixed":
        assert eng.info().last_unk_detour > 0  # unknown runs took the spans path
    if model == "mix_bf8k":
        assert eng.info().last_unk_detour == 0  # byte fallback: no unknown id survives
    eng.close()


# ---- 2. the unknown-surface subset ----

def _unknown_chars(mb, n):
    """characters uni32k has no piece for (each encodes to the unknown id)"""
    om = oracle_py.OracleModel(mb)
    unk = om.unk_id
    out = []
    for cp in range(0x4E00, 0x9FFF):
        ch = chr(cp).encode()
        if om.encode(b"a" + ch + b"b")[0].tolist().count(unk) == 1:
            out.append(ch)
            if len(out) == n:
                return out
    raise AssertionError("no unknown characters found")


def _unknown_lines(mb, corpus_gen):
    u = _unknown_chars(mb, 4)
    long_words = b" ".join(corpus_gen.lines("en", 9301, 200))
    return [
        u[0] + b" start", b"mid " + u[1] + u[2] + b" dle", b"the end " + u[3], u[0] + u[1] + u[2] + u[3],
        b" " + u[0] + b" after a space", b"word" + u[1] + b"word", ("▁" + u[2].decode()).encode(),
        long_words[:290] + u[0] + long_words[290:600], b"", b"   ", b"\x00", b"a\x00" + u[1], b"\xff\xfe",
        b"\xc3" + u[2] + b"\x80", u[3] * 40,
    ]


def test_unknown_subset_fractions(corpus_gen):
    mb = model_bytes("uni32k")
    u = _unknown_chars(mb, 8)
    om = oracle_py.OracleModel(mb)
    plain = [s for s in corpus_gen.lines("en", 9201, 3000) if om.unk_id not in om.encode(s)[0].tolist()]
    rng = np.random.default_rng(5)
    few = list(plain)
    for k in rng.choice(len(few), size=len(few) // 30, replace=False):
        few[k] = few[k] + b" " + u[k % 8]
    every = [s + u[i % 8] for i, s in enumerate(plain)]
    eng = _engine(mb)
    for lines, frac in ((plain, 0), (few, 1), (every, 2)):
        buf, offs = oracle_py.pack(lines)
        _check(eng, mb, buf, offs)
        flagged = eng.info().last_unk_detour
        if frac == 0:
            assert flagged == 0
        elif frac == 1:
            assert 0 < flagged < len(lines)
        else:
            assert flagged == len(lines)
        # unk_piece replaces every unknown piece: no sentence takes the detour
        _check(eng, mb, buf, offs, "unk")
        assert eng.info().last_unk_detour == 0
    eng.close()


def test_unknown_runs_and_edges(corpus_gen):
    """unknown runs at the start, middle and end, next to U+2581, inside 600-byte and 1 MB sentences (deferred and long
    kernels), and empty, whitespace-only, NUL and malformed-UTF-8 sentences"""
    mb = model_bytes("uni32k")
    lines = _unknown_lines(mb, corpus_gen)
    u = _unknown_chars(mb, 2)
    doc = b" ".join(corpus_gen.lines("mixed", 9302, 40000))[:1 << 20]
    big = doc[:1000] + u[0] * 3 + doc[1000:(1 << 20) - 1000] + b" " + u[1]
    lines = lines + [big] + corpus_gen.lines("mixed", 9303, 500)
    # the oracle shim hands the reference's pieces over NUL-separated, so a piece holding NUL (an unknown run over a
    # NUL byte) cannot come back whole: those sentences are checked against the spans path only
    keep = [i for i, s in enumerate(lines) if b"\x00" not in s]
    want = reference("edges/uni32k/without-nul", lambda: _ref_digest(mb, [lines[i] for i in keep]))
    buf, offs = oracle_py.pack(lines)
    eng = _engine(mb)
    got = _check(eng, mb, buf, offs, sep_too=True)
    assert eng.info().last_deferred > 0
    r = eng.encode_pieces(buf, offs)
    ido = r["id_offsets"]
    kept_ids = np.concatenate([r["ids"][int(ido[i]):int(ido[i + 1])] for i in keep])
    assert pieces_digest([got[i] for i in keep], kept_ids) == want
    eng.close()


# ---- 3. extra options ----

PERMS = [":".join(p) for k in range(1, 5) for p in itertools.permutations(["bos", "eos", "reverse", "unk"], k)]


def test_extra_options(corpus_gen):
    mb = model_bytes("uni32k")
    u = _unknown_chars(mb, 2)
    lines = [b"", b"an " + u[0] + b" unknown and " + u[1] + u[0], b"plain words only"]
    wants = {o: reference(f"options/uni32k/{o}", lambda o=o: _ref_digest(mb, lines, o)) for o in PERMS}
    buf, offs = oracle_py.pack(lines)
    eng = _engine(mb)
    for o in PERMS:
        unk = _set_options(eng, mb, o)
        r = eng.encode_pieces(buf, offs, unk_piece=unk)
        ids, ido = eng.encode_packed(buf, offs)
        assert np.array_equal(r["ids"], ids) and np.array_equal(r["id_offsets"], ido), o
        assert pieces_digest(_rows(r), r["ids"]) == wants[o], o
        _set_options(eng, mb, "")
        _check(eng, mb, buf, offs, o)
    eng.close()


# ---- 4. agreement with the old path ----

@pytest.mark.parametrize("flags", [dict(add_dummy_prefix=False), dict(remove_extra_whitespaces=False),
                                   dict(escape_whitespaces=False, add_dummy_prefix=False),
                                   dict(treat_whitespace_as_suffix=True),
                                   dict(escape_whitespaces=False, remove_extra_whitespaces=False)])
def test_normalizer_flag_variants(flags, corpus_gen):
    mb = mp.replace_flags(model_bytes("uni32k"), **flags)
    buf, offs = oracle_py.pack(corpus_gen.lines("mixed", 9401, 2000) + [b"", b"  a  b ", b"x\ty"])
    eng = _engine(mb)
    _check(eng, mb, buf, offs, sep_too=True)
    _check(eng, mb, buf, offs, "bos:reverse:eos")
    eng.close()


def test_toy_models_and_set_types():
    """the synthetic models of the reference's unigram / BPE tests with USER_DEFINED and UNUSED pieces, before and
    after spm_engine_set_types (piece strings do not change with the types)"""
    from test_oracle_kat import BASE, ENCODE_PIECES, UNUSED_PIECES
    texts = [b"abc", b"AB", b"abcd", b"abcc", b"xabcabaabcdd", "xyz東京".encode(), b"ABC", b"abABCcd",
             b"ababcdabcdcd", b"abqrcd", b"", b"  ab  cd "]
    buf, offs = oracle_py.pack(texts)
    for mt in (mp.UNIGRAM, mp.BPE):
        pcs = BASE + [(p, s, mp.NORMAL) for p, s in ENCODE_PIECES]
        for i in (9, 10, 11, 12):
            pcs[i] = (pcs[i][0], pcs[i][1], mp.USER_DEFINED)
        up = BASE + [(p, s, mp.NORMAL) for p, s in UNUSED_PIECES]
        for plist in (pcs, up):
            mb = mp.build_model(plist, model_type=mt, charsmap=b"", add_dummy_prefix=False)
            types = np.array([t for _, _, t in plist], dtype=np.uint8)
            eng = _engine(mb)
            _check(eng, mb, buf, offs)
            t2 = types.copy()
            t2[(t2 == mp.NORMAL) & (np.arange(len(t2)) % 2 == 1)] = mp.UNUSED
            eng.set_types(t2)
            _check(eng, mb, buf, offs)
            eng.set_types(types)
            _check(eng, mb, buf, offs)
            eng.close()


@pytest.mark.parametrize("model,kind", [("uni32k", "mixed"), ("bpe32k", "en")])
def test_large_batch(model, kind, corpus_gen):
    """a batch above pipeline_min_sentences: ids equal spm_encode_ids' (the fused host path), pieces equal the old path
    on a sample of sentences"""
    mb = model_bytes(model)
    N = 320000
    buf, offs = corpus_gen.fill(kind, 9501, N)
    eng = _engine(mb)
    _set_options(eng, mb, "bos:eos")
    r = eng.encode_pieces(buf, offs)
    ids, ido = eng.encode_packed(buf, offs)
    assert np.array_equal(r["id_offsets"], ido) and np.array_equal(r["ids"], ids)
    _set_options(eng, mb, "")
    rows = _rows(r)
    pick = list(range(0, N, 997))
    raw = buf.tobytes()
    sb, so = oracle_py.pack([raw[int(offs[i]):int(offs[i + 1])] for i in pick])
    want, _ = _old_rows(eng, mb, sb, so, "bos:eos")
    assert [rows[i] for i in pick] == want
    eng.close()


# ---- 5. layers ----

def test_python_mirror(corpus_gen):
    from sentencepiece_b200 import SentencePieceProcessor
    mb = model_bytes("uni32k")
    lines = corpus_gen.lines("mixed", 9601, 300) + [b""]
    strs = [s.decode("utf-8", errors="replace") for s in lines]
    cases = (("", {}), ("bos:eos:unk", dict(add_bos=True, add_eos=True, emit_unk_piece=True)),
             ("reverse:bos", dict(reverse=True, add_bos=True)), ("eos:unk", None))
    wants = {o: reference(f"python/uni32k/{o}", lambda o=o: _ref_digest(mb, [s.encode() for s in strs], o)) for o, _ in cases}
    for opts, kw in cases[:3]:
        want = wants[opts]
        sp = SentencePieceProcessor(model_proto=mb)
        got = sp.encode(strs, out_type=str, **kw)
        assert got == sp.EncodeAsPieces(strs, **kw)
        ids = sp.encode(strs, out_type=int, **kw)
        assert pieces_digest([[p.encode() for p in row] for row in got], np.concatenate([np.asarray(i, np.int32) for i in ids])) == want
        assert sp.EncodeAsPieces(strs[0], **kw) == got[0]
    sp = SentencePieceProcessor(model_proto=mb)
    sp.SetEncodeExtraOptions("eos:unk")
    want = wants["eos:unk"]
    got = sp.EncodeAsPieces(strs)
    ids = sp.EncodeAsIds(strs)
    assert pieces_digest([[p.encode() for p in row] for row in got], np.concatenate([np.asarray(i, np.int32) for i in ids])) == want


@pytest.mark.parametrize("model,kind,extra,n", [("uni32k", "mixed", "bos:eos:unk", 3000), ("uni32k", "mixed", "reverse", 3000),
                                                ("bpe32k", "en", "", 2500), ("mix_bf8k", "mixed", "eos", 2500)])
def test_cli_piece(model, kind, extra, n, corpus_gen, tmp_path):
    """spm_encode_b200 --output_format=piece (C++ class, spm_encode_pieces with sep ' ') prints what the reference's
    spm_encode prints, over more lines than one --batch_lines"""
    path = str(tmp_path / "in.txt")
    corpus_gen.write_file(path, kind, 9701, n)
    mpath = os.path.join(MODELS_DIR, model + ".model")
    args = [f"--model={mpath}", "--output_format=piece", f"--input={path}"]
    if extra:
        args.append(f"--extra_options={extra}")
    want = reference(f"cli/{model}/{kind}/{extra}/{n}",
                     lambda: digest(subprocess.run([REF_CLI] + args, capture_output=True, check=True).stdout))
    assert os.path.exists(CLI), "spm_encode_b200 has not been built (__graft_entry__.build())"
    ours = subprocess.run([CLI, "--batch_lines=1000"] + args, capture_output=True, check=True).stdout
    assert digest(ours) == want


# ---- 6. errors ----

def test_errors_leave_engine_usable(corpus_gen):
    mb = model_bytes("uni32k")
    buf, offs = corpus_gen.fill("mixed", 9801, 5000)
    eng = _engine(mb)
    good = eng.encode_pieces(buf, offs)
    bad = offs.copy()
    bad[100] = bad[101] + 5
    with pytest.raises(RuntimeError, match=r"error 1: offsets must be non-decreasing"):
        eng.encode_pieces(buf, bad)
    wild = offs.copy()
    wild[200] = np.uint64(10 ** 12)
    wild[201] = np.uint64(10 ** 12 + 5)
    with pytest.raises(RuntimeError, match=r"error 1: offsets must be non-decreasing"):
        eng.encode_pieces(buf, wild)
    with pytest.raises(RuntimeError, match="error 1"):
        eng.encode_pieces(buf, offs, sep=256)
    again = eng.encode_pieces(buf, offs)
    for k in good:
        assert np.array_equal(good[k], again[k]), k
    e = eng.encode_pieces(np.zeros(0, np.uint8), np.zeros(1, np.uint64))
    assert len(e["ids"]) == 0 and e["text_offsets"].tolist() == [0]
    eng.close()
