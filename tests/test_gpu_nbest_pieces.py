"""spm_nbest_encode_pieces, spm_sample_encode_pieces and spm_sample_encode_and_score_pieces: n-best and sampled piece
strings written by K9 from the n-best kernels' token ends and exported normalized text (no second encode), and by the
host loop of the lattice draws.  Checked against the ids calls bit for bit, against the normalized text, against the
reference's spm_encode (nbest_piece / sample_piece, stored digests in tests/golden/reference_digests_nbest_pieces.json)
and through the Python mirror, the C++ class and spm_encode_b200.  Needs an H100."""
import itertools
import json
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import MODELS_DIR, ROOT, model_bytes
from oracle import oracle_py
from refstore import digest

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "sentencepiece_b200", "lib", "spm_encode_b200")
REF_CLI = os.path.join(ROOT, "oracle", "_ref", "spm_encode")
STORE = os.path.join(ROOT, "tests", "golden", "reference_digests_nbest_pieces.json")
MODELS = ["uni32k", "botchan8k", "mix_bf8k"]
_store = None


def reference(key, compute):
    """the stored digest of the reference's output for `key`; SPM_RECORD_REFERENCE=1 runs compute() and stores it"""
    global _store
    if _store is None:
        _store = json.load(open(STORE)) if os.path.exists(STORE) else {}
    if os.environ.get("SPM_RECORD_REFERENCE") == "1":
        _store[key] = compute()
        with open(STORE, "w") as f:
            json.dump(_store, f, indent=1, sort_keys=True)
            f.write("\n")
    assert key in _store, f"no stored reference result for {key}"
    return _store[key]


def _engine(mb):
    from sentencepiece_b200 import Engine
    return Engine(mb)


def _lists(r, offs_key):
    """packed pieces (sep = -1) -> list of lists of piece bytes, one per list"""
    raw = r["text"].tobytes()
    to, ido, pe = r["text_offsets"].tolist(), r[offs_key].tolist(), r["piece_end"].tolist()
    out = []
    for j in range(len(to) - 1):
        s = raw[to[j]:to[j + 1]]
        ends = pe[ido[j]:ido[j + 1]]
        out.append([s[b:e] for b, e in zip([0] + ends[:-1], ends)])
    return out


def _surface(mb):
    """piece bytes -> its bytes in the normalized text (byte pieces <0xXX> stand for one byte)"""
    from sentencepiece_b200 import _modelinfo
    pieces, _ = _modelinfo.pieces_and_unk(mb)
    byte = re.compile(rb"<0x([0-9A-F]{2})>")

    def f(p, i):
        m = byte.fullmatch(p)
        return bytes.fromhex(m.group(1).decode()) if m and pieces[i].encode() == p else p
    return f


def _check_structure(eng, mb, buf, offs, lists, ids, id_offs, per):
    """without frame or unk_piece, the pieces of every list concatenate to its sentence's normalized text, and each
    known id's piece is its vocabulary piece"""
    from sentencepiece_b200 import _modelinfo
    pieces, unk = _modelinfo.pieces_and_unk(mb)
    sp = eng.encode_spans(buf, offs)
    norm, no = sp["normalized"], sp["norm_offsets"].tolist()
    surf = _surface(mb)
    ids, io = ids.tolist(), id_offs.tolist()
    for j, row in enumerate(lists):
        if not row:
            continue
        i = j // per
        t = ids[io[j]:io[j + 1]]
        assert len(t) == len(row)
        assert b"".join(surf(p, k) for p, k in zip(row, t)) == norm[no[i]:no[i + 1]], (j, row)
        for p, k in zip(row, t):
            if k != unk:
                assert p == pieces[k].encode()


def _unknown_chars(mb, n):
    om = oracle_py.OracleModel(mb)
    out = []
    for cp in range(0x4E00, 0x9FFF):
        ch = chr(cp).encode()
        if om.encode(b"a" + ch + b"b")[0].tolist().count(om.unk_id) == 1:
            out.append(ch)
            if len(out) == n:
                return out
    raise AssertionError("no unknown characters found")


def _edge_lines(mb, corpus_gen):
    u = _unknown_chars(mb, 4)
    words = b" ".join(corpus_gen.lines("en", 9301, 3000))
    return [
        u[0] + b" start", b"mid " + u[1] + u[2] + b" dle", b"the end " + u[3], u[0] + u[1] + u[2] + u[3],
        b" " + u[0] + b" after a space", ("▁" + u[2].decode()).encode(), b"", b"   ", b"\x00", b"a\x00" + u[1],
        b"\xff\xfe", b"\xc3" + u[2] + b"\x80", u[3] * 40,
        words[:4500] + u[0] + words[4500:9000],                   # 9 KB: the long-sentence kernels
        (words * 3)[:30000] + u[1] + u[2] + (words * 3)[30000:64000],  # 64 KB
    ]


# ---- n-best ----

@pytest.mark.parametrize("kind", ["en", "mixed"])
@pytest.mark.parametrize("model", MODELS)
def test_nbest_pieces_equal_ids(model, kind, corpus_gen):
    mb = model_bytes(model)
    buf, offs = corpus_gen.fill(kind, 9411, 1500)
    eng = _engine(mb)
    for nb in (1, 2, 16, 64):
        r = eng.nbest_encode_pieces(buf, offs, nb)
        want = eng.nbest_encode(buf, offs, nb)
        for k in ("ids", "cand_offsets", "scores", "n_cands"):
            assert np.array_equal(r[k], want[k]), (nb, k)
        lists = _lists(r, "cand_offsets")
        _check_structure(eng, mb, buf, offs, lists, r["ids"], r["cand_offsets"], r["K"])
        if nb == 1:
            p = eng.encode_pieces(buf, offs)
            assert np.array_equal(p["text"], r["text"]) and np.array_equal(p["piece_end"], r["piece_end"])
    eng.close()


@pytest.mark.parametrize("model", ["uni32k", "mix_bf8k"])
def test_nbest_edges_and_long_documents(model, corpus_gen):
    mb = model_bytes(model)
    lines = _edge_lines(model_bytes("uni32k"), corpus_gen)
    buf, offs = oracle_py.pack(lines)
    eng = _engine(mb)
    r = eng.nbest_encode_pieces(buf, offs, 8)
    assert eng.info().last_deferred > 0
    want = eng.nbest_encode(buf, offs, 8)
    for k in ("ids", "cand_offsets", "scores", "n_cands"):
        assert np.array_equal(r[k], want[k]), k
    _check_structure(eng, mb, buf, offs, _lists(r, "cand_offsets"), r["ids"], r["cand_offsets"], 8)
    s = eng.sample_encode_and_score_pieces(buf, offs, 2, 0.5)
    assert eng.info().last_deferred > 0
    _check_structure(eng, mb, buf, offs, _lists(s, "cand_offsets"), s["ids"], s["cand_offsets"], 2)
    eng.close()


def _framed(rows, ids, real, options, sp, unk):
    """ApplyExtraOptions on the unframed (piece, id) lists; empty n-best slots (not real) stay empty"""
    out = []
    for row, t, is_real in zip(rows, ids, real):
        pairs = list(zip(row, t))
        if not is_real:
            out.append([])
            continue
        for o in options:
            if o == "reverse":
                pairs.reverse()
            elif o == "bos":
                pairs.insert(0, (sp["bos_piece"].encode(), sp["bos_id"]))
            elif o == "eos":
                pairs.append((sp["eos_piece"].encode(), sp["eos_id"]))
            elif o == "unk":
                pairs = [(sp["unk_piece"].encode() if k == unk else p, k) for p, k in pairs]
        out.append(pairs)
    return out


def test_extra_option_orderings(corpus_gen):
    from sentencepiece_b200 import _modelinfo
    from sentencepiece_b200.processor import extra_frame
    mb = model_bytes("uni32k")
    sp = _modelinfo.special_pieces(mb)
    _, unk = _modelinfo.pieces_and_unk(mb)
    buf, offs = corpus_gen.fill("mixed", 9511, 600)
    eng = _engine(mb)
    base = eng.nbest_encode_pieces(buf, offs, 4)
    rows, io, ids = _lists(base, "cand_offsets"), base["cand_offsets"].tolist(), base["ids"].tolist()
    raw_ids = [ids[io[j]:io[j + 1]] for j in range(len(rows))]
    real = [j % 4 < int(base["n_cands"][j // 4]) for j in range(len(rows))]
    for n in range(1, 5):
        for perm in itertools.permutations(["bos", "eos", "reverse", "unk"], n):
            p, rev, s = extra_frame(perm, sp["bos_id"], sp["eos_id"])
            eng.set_encode_frame(p, rev, s)
            r = eng.nbest_encode_pieces(buf, offs, 4, unk_piece=sp["unk_piece"] if "unk" in perm else None)
            want = _framed(rows, raw_ids, real, perm, sp, unk)
            got = _lists(r, "cand_offsets")
            assert got == [[q for q, _ in w] for w in want], perm
            assert r["ids"].tolist() == [k for w in want for _, k in w], perm
    eng.close()


# ---- sampling ----

@pytest.mark.parametrize("model", ["uni32k", "mix_bf8k"])
def test_sample_pieces_equal_ids(model, corpus_gen):
    mb = model_bytes(model)
    buf, offs = corpus_gen.fill("mixed", 9611, 2000)
    eng = _engine(mb)
    for nb, seed, alpha in itertools.product((8, -1), (1, 77), (0.1, 0.5)):
        eng.set_random_seed(seed)
        r = eng.sample_encode_pieces(buf, offs, nb, alpha)
        eng.set_random_seed(seed)
        ids, ido = eng.sample_encode(buf, offs, nb, alpha)
        assert np.array_equal(r["ids"], ids) and np.array_equal(r["id_offsets"], ido), (nb, seed, alpha)
        _check_structure(eng, mb, buf, offs, _lists(r, "id_offsets"), r["ids"], r["id_offsets"], 1)
        # the generator: a pieces call then an ids call draws what two ids calls draw
        eng.set_random_seed(seed)
        eng.sample_encode_pieces(buf, offs, nb, alpha)
        second = eng.sample_encode(buf, offs, nb, alpha)
        eng.set_random_seed(seed)
        eng.sample_encode(buf, offs, nb, alpha)
        again = eng.sample_encode(buf, offs, nb, alpha)
        assert np.array_equal(second[0], again[0]) and np.array_equal(second[1], again[1])
    eng.close()


def test_sample_encode_and_score_pieces(corpus_gen):
    mb = model_bytes("uni32k")
    lines = corpus_gen.lines("mixed", 9711, 1500) + [b"", b"  "]
    buf, offs = oracle_py.pack(lines)
    eng = _engine(mb)
    eng.set_encode_frame([1], True, [2])
    for ns in (1, 5):
        eng.set_random_seed(5)
        r = eng.sample_encode_and_score_pieces(buf, offs, ns, 0.3)
        eng.set_random_seed(5)
        ids, co, sc = eng.sample_encode_and_score(buf, offs, ns, 0.3)
        assert np.array_equal(r["ids"], ids) and np.array_equal(r["cand_offsets"], co)
        assert np.array_equal(r["scores"].view(np.uint32), sc.view(np.uint32))
        lists = _lists(r, "cand_offsets")
        n = len(lines)
        for j in range((n - 2) * ns, n * ns):  # empty sentences: empty, unframed slots
            assert lists[j] == [] and r["text_offsets"][j] == r["text_offsets"][j + 1]
    eng.close()


def test_bpe():
    mb = model_bytes("bpe32k")
    buf, offs = oracle_py.pack([b"hello world", b"", "日本語 text".encode()])
    eng = _engine(mb)
    want = eng.encode_pieces(buf, offs)
    r = eng.sample_encode_pieces(buf, offs, 8, 0.0)
    for k in want:
        assert np.array_equal(r[k], want[k]), k
    with pytest.raises(RuntimeError, match="error 6"):
        eng.sample_encode_pieces(buf, offs, 8, 0.5)
    with pytest.raises(RuntimeError, match="error 6"):
        eng.nbest_encode_pieces(buf, offs, 8)
    eng.close()


# ---- layers ----

def test_python_mirror(corpus_gen):
    from sentencepiece_b200 import SentencePieceProcessor, _modelinfo
    mb = model_bytes("uni32k")
    strs = [s.decode("utf-8", "replace") for s in corpus_gen.lines("mixed", 9811, 300)] + [""]
    sp = SentencePieceProcessor(model_proto=mb)
    eng = _engine(mb)
    buf, offs = oracle_py.pack([s.encode() for s in strs])
    r = eng.nbest_encode_pieces(buf, offs, 4)
    rows = [[p.decode("utf-8", "replace") for p in row] for row in _lists(r, "cand_offsets")]
    nb = sp.NBestEncodeAsPieces(strs, 4)
    assert nb == [rows[4 * i:4 * i + int(r["n_cands"][i])] for i in range(len(strs))]
    assert sp.NBestEncode(strs, out_type=str, nbest_size=4) == nb
    assert sp.NBestEncode(strs[0], out_type=int, nbest_size=4) == sp.NBestEncodeAsIds(strs[0], 4)
    for nbs in (8, -1):
        sp.SetRandomGeneratorSeed(3)
        a = sp.SampleEncodeAsPieces(strs, nbs, 0.2, add_bos=True, reverse=True, emit_unk_piece=True)
        sp.SetRandomGeneratorSeed(3)
        b = sp.encode(strs, out_type=str, enable_sampling=True, nbest_size=nbs, alpha=0.2, add_bos=True, reverse=True,
                      emit_unk_piece=True)
        assert a == b
        sp.SetRandomGeneratorSeed(3)
        ids = sp.SampleEncodeAsIds(strs, nbs, 0.2, add_bos=True, reverse=True)
        assert [len(x) for x in a] == [len(x) for x in ids]
        unk_piece, unk = sp._specials()["unk_piece"], _modelinfo.pieces_and_unk(mb)[1]
        assert all(p == unk_piece for row, t in zip(a, ids) for p, k in zip(row, t) if k == unk)
    sp.SetRandomGeneratorSeed(9)
    sc = sp.SampleEncodeAndScoreAsPieces(strs, 3, 0.5)
    sp.SetRandomGeneratorSeed(9)
    si = sp.SampleEncodeAndScoreAsIds(strs, 3, 0.5)
    assert [[s for _, s in x] for x in sc] == [[s for _, s in x] for x in si]
    assert sc[-1] == [] and si[-1] == []
    assert all(len(x) == 3 for x in sc[:-1])
    eng.close()


CLI_CASES = [("uni32k", "mixed", "nbest_piece", "8", ""), ("uni32k", "mixed", "nbest_piece", "3", "bos:eos:unk"),
             ("mix_bf8k", "mixed", "nbest_piece", "16", "reverse"), ("botchan8k", "en", "nbest_piece", "64", ""),
             ("uni32k", "mixed", "sample_piece", "8", ""), ("uni32k", "mixed", "sample_piece", "-1", ""),
             ("uni32k", "mixed", "sample_piece", "-1", "reverse:bos:unk"), ("mix_bf8k", "en", "sample_piece", "-1", "eos")]


@pytest.mark.parametrize("model,kind,fmt,nbest,extra", CLI_CASES)
def test_cli_against_reference(model, kind, fmt, nbest, extra, corpus_gen, tmp_path):
    """spm_encode_b200 (the C++ class over the new calls, sep ' ') prints what the reference's spm_encode prints for
    the same seed, over more lines than one --batch_lines"""
    path = str(tmp_path / "in.txt")
    corpus_gen.write_file(path, kind, 9901, 1500)
    mpath = os.path.join(MODELS_DIR, model + ".model")
    args = [f"--model={mpath}", f"--output_format={fmt}", f"--nbest_size={nbest}", "--alpha=0.3", "--random_seed=11",
            f"--input={path}"]
    if extra:
        args.append(f"--extra_options={extra}")
    want = reference(f"cli/{model}/{kind}/{fmt}/{nbest}/{extra}",
                     lambda: digest(subprocess.run([REF_CLI] + args, capture_output=True, check=True).stdout))
    assert os.path.exists(CLI), "spm_encode_b200 has not been built (__graft_entry__.build())"
    ours = subprocess.run([CLI, "--batch_lines=1000"] + args, capture_output=True, check=True).stdout
    assert digest(ours) == want


def test_errors_leave_engine_usable(corpus_gen):
    mb = model_bytes("uni32k")
    buf, offs = corpus_gen.fill("mixed", 9951, 2000)
    eng = _engine(mb)
    good = eng.nbest_encode_pieces(buf, offs, 8)
    bad = offs.copy()
    bad[100] = bad[101] + 5
    with pytest.raises(RuntimeError, match="error 1"):
        eng.nbest_encode_pieces(buf, bad, 8)
    with pytest.raises(RuntimeError, match="error 1"):
        eng.sample_encode_pieces(buf, offs, 8, 0.1, sep=300)
    with pytest.raises(RuntimeError, match="error 1"):
        eng.sample_encode_pieces(buf, offs, 600, 0.1)
    with pytest.raises(RuntimeError, match="error 1"):
        eng.sample_encode_and_score_pieces(buf, offs, 0, 0.1)
    with pytest.raises(RuntimeError, match="error 6"):
        eng.sample_encode_and_score_pieces(buf, offs, 2, 0.1, wor=True)
    again = eng.nbest_encode_pieces(buf, offs, 8)
    for k in ("text", "text_offsets", "piece_end", "ids", "cand_offsets", "scores", "n_cands"):
        assert np.array_equal(good[k], again[k]), k
    eng.close()


# ---- the reference's NBestEncodeAsPieces / SampleEncodeAsPieces over the matrix of models, corpora and sizes ----
# spm_encode prints these piece lists (one line per candidate / draw, pieces joined by ' ') from a seeded generator on
# one thread, which is the stream the engine reproduces for a batch.

MATRIX = ([(m, k, "nbest_piece", str(nb), "0.5", "11", "") for m in MODELS for k in ("en", "mixed") for nb in (1, 2, 16, 64)]
          + [(m, "mixed", "sample_piece", str(nb), a, s, "") for m in ("uni32k", "mix_bf8k") for nb in (8, -1)
             for a in ("0.1", "0.5") for s in ("11", "12")]
          + [("uni32k", "mixed", fmt, nb, "0.3", "13", "reverse") for fmt, nb in
             (("nbest_piece", "8"), ("sample_piece", "8"), ("sample_piece", "-1"))])


@pytest.mark.parametrize("model,kind,fmt,nbest,alpha,seed,extra", MATRIX)
def test_reference_matrix(model, kind, fmt, nbest, alpha, seed, extra, corpus_gen, tmp_path):
    path = str(tmp_path / "in.txt")
    corpus_gen.write_file(path, kind, 9931, 600)
    mpath = os.path.join(MODELS_DIR, model + ".model")
    args = [f"--model={mpath}", f"--output_format={fmt}", f"--nbest_size={nbest}", f"--alpha={alpha}",
            f"--random_seed={seed}", f"--input={path}"]
    if extra:
        args.append(f"--extra_options={extra}")
    want = reference(f"matrix/{model}/{kind}/{fmt}/{nbest}/{alpha}/{seed}/{extra}",
                     lambda: digest(subprocess.run([REF_CLI] + args, capture_output=True, check=True).stdout))
    ours = subprocess.run([CLI, "--batch_lines=250"] + args, capture_output=True, check=True).stdout
    assert digest(ours) == want


def test_sample_encode_and_score_reversed_unknown_surfaces(corpus_gen):
    """SampleEncodeAndScore pieces under a reversed frame without unk_piece: ids and scores are the reference's under
    the same options and seed, and each sample's pieces are those of the unframed call, reversed, whose unknown
    surfaces lie in the normalized text"""
    from extra_options import set_reference_options
    mb = model_bytes("uni32k")
    lines = corpus_gen.lines("mixed", 9961, 400) + [b"", b" "]
    buf, offs = oracle_py.pack(lines)

    def ref_digest():
        ref = oracle_py.RefModel(mb)
        set_reference_options(ref, "reverse")
        ids, co, sc = ref.sample_score_batch(buf, offs, 3, 0.4, 21)
        return digest(ids, co, sc)
    want = reference("score/uni32k/mixed/reverse/3/0.4/21", ref_digest)
    eng = _engine(mb)
    eng.set_random_seed(21)
    plain = eng.sample_encode_and_score_pieces(buf, offs, 3, 0.4)
    _check_structure(eng, mb, buf, offs, _lists(plain, "cand_offsets"), plain["ids"], plain["cand_offsets"], 3)
    eng.set_encode_frame([], True, [])
    eng.set_random_seed(21)
    r = eng.sample_encode_and_score_pieces(buf, offs, 3, 0.4)
    assert digest(r["ids"], r["cand_offsets"], r["scores"]) == want
    got, base = _lists(r, "cand_offsets"), _lists(plain, "cand_offsets")
    assert got == [b[::-1] for b in base]
    from sentencepiece_b200 import _modelinfo
    unk = _modelinfo.pieces_and_unk(mb)[1]
    assert int(np.count_nonzero(r["ids"] == unk)) > 100  # the mixed corpus holds many unknown runs
    eng.close()
