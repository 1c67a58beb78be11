"""spm_encode_pairs_device (Engine.encode_device_pairs, SentencePieceProcessor.encode_pairs): 2n sentences as n pair
rows prefix ++ A ++ middle ++ B ++ suffix with type ids, truncation strategies, overflow windows and offsets.  The rows
are checked against pairs_ref, a numpy restatement of the semantics in include/spm_b200.h, applied to packed lists
that other tests pin: the reference's own ids (tests/golden/ids), spm_encode_ids_device and spm_encode_offsets (bytes,
and characters through unicode_spans).  Needs an H100."""
import ctypes
import os

import numpy as np
import pytest

import charsmap_rules as cr
from conftest import model_bytes
from oracle import modelproto as mp
from oracle import oracle_py
from pairs_ref import pairs_ref
from sentencepiece_b200 import Engine, SentencePieceProcessor, _capi
from sentencepiece_b200.processor import unicode_spans
from test_gpu_normalize import edge_lines
from test_gpu_padded import _long_doc, _packed_device
from test_gpu_padded_offsets import Batch, _device, _frame

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN = [("uni32k", "en"), ("uni32k", "mixed"), ("botchan8k", "en"), ("mix_bf8k", "mixed"), ("bpe32k", "en"),
          ("mix_bpe4k", "mixed")]
CORPUS_SEED = 20260922  # bench.py's
# (prefix, middle, suffix): none, "[CLS] A [SEP] B [SEP]", "<s> A </s></s> B </s>", and 64-id lists
TEMPLATES = [((), (), ()), ((1,), (2,), (2,)), ((1,), (2, 2), (2,)),
             (tuple(range(3, 67)), tuple(range(100, 164)), tuple(range(200, 264)))]
NAMES = ("ids", "lengths", "type_ids", "row_pair", "row_first", "spans")


def run(eng, d_bytes, d_offs, tmpl, w, trunc, overflow=False, stride=0, pad=-1, left=False, unit=None):
    p, m, s = tmpl
    return eng.encode_device_pairs(d_bytes, d_offs, prefix=p, middle=m, suffix=s, width=w, truncation=trunc,
                                   overflow=overflow, stride=stride, pad_id=pad, pad_left=left, unit=unit)


def check(eng, d_bytes, d_offs, ids, ido, tmpl, w, trunc, overflow=False, stride=0, pad=-1, left=False, unit=None,
          begin=None, end=None, what=()):
    """the call against pairs_ref of the packed raw lists; a pair that cannot be laid out must raise ValueError with
    the least width -> pairs_ref's answer"""
    want = pairs_ref(ids, ido, *tmpl, w, trunc, overflow, stride, pad, left, begin, end)
    what = what + (tmpl[0][:2], w, trunc, overflow, stride, left, unit)
    if "error" in want:
        with pytest.raises(ValueError, match=str(want["width"])):
            run(eng, d_bytes, d_offs, tmpl, w, trunc, overflow, stride, pad, left, unit)
        return want
    got = run(eng, d_bytes, d_offs, tmpl, w, trunc, overflow, stride, pad, left, unit)
    for name, g in zip(NAMES, got):
        g = g.cpu().numpy()
        x = want[name]
        assert g.shape == x.shape, (what, name, g.shape, x.shape)
        if not np.array_equal(g, x):
            bad = np.argwhere(g != x)[0]
            raise AssertionError(f"{what}: {name} differs at {bad.tolist()}: {g[tuple(bad)]} != {x[tuple(bad)]}")
    return want


def _stacked(z):
    """the first 2 * (n // 2) stored lists: a stacked batch of n // 2 pairs"""
    m = 2 * (int(z["n"]) // 2)
    ido = z["id_offsets"].astype(np.int64)[:m + 1]
    return z["ids"][:ido[-1]], ido, m


@pytest.mark.parametrize("model,kind", GOLDEN)
def test_reference_ids(model, kind, corpus_gen):
    """the reference's stored ids: every strategy, widths that cut often and rarely, four templates, both paddings"""
    z = np.load(os.path.join(GOLD, "ids", f"{model}__{kind}.npz"))
    ids, ido, m = _stacked(z)
    buf, offs = corpus_gen.fill(kind, int(z["seed"]), int(z["n"]))
    d_bytes, d_offs = _device(buf, np.asarray(offs)[:m + 1])
    eng = Engine(model_bytes(model))
    for j, tmpl in enumerate(TEMPLATES):
        T = sum(len(x) for x in tmpl)
        left = j % 2 == 1
        check(eng, d_bytes, d_offs, ids, ido, tmpl, 0, "none", left=left, what=(model, kind))
        longest = int(pairs_ref(ids, ido, *tmpl, 0, "none")["width"])
        check(eng, d_bytes, d_offs, ids, ido, tmpl, longest, "none", pad=0, left=not left, what=(model, kind))
        check(eng, d_bytes, d_offs, ids, ido, tmpl, longest - 1, "none", what=(model, kind))
        for w in (T + 1, T + 16, T + 48, T + 160):
            for trunc in ("longest_first", "only_first", "only_second"):
                check(eng, d_bytes, d_offs, ids, ido, tmpl, w, trunc, pad=7, left=left, what=(model, kind))
        for w, stride in ((T + 40, 0), (T + 64, 16), (T + 160, 100)):
            for trunc in ("only_first", "only_second"):
                check(eng, d_bytes, d_offs, ids, ido, tmpl, w, trunc, True, stride, left=not left, what=(model, kind))
    eng.close()


def _qa_lines(corpus_gen, kind, long=True):
    """short questions, then contexts: a 9 KB and (long) a 64 KB document, edge lines (empty, whitespace-only,
    malformed UTF-8) and corpus lines"""
    docs = [_long_doc(corpus_gen, kind, 9400, 9000)] + ([_long_doc(corpus_gen, kind, 9401, 65536)] if long else [])
    ctx = docs + edge_lines()[:-2] + corpus_gen.lines(kind, 9403, 200) + [b""]
    q = [x[:40] for x in corpus_gen.lines(kind, 9404, len(ctx))]
    q[3] = b""
    return q, ctx


@pytest.mark.parametrize("model", ["uni32k", "botchan8k", "mix_bf8k"])
def test_overflow(model, corpus_gen):
    """only_second / only_first with overflow over long contexts and edge lines, strides 0, 16 and r - 1 for the
    shortest room: rows, row_pair, row_first (hence each pair's step) against pairs_ref over spm_encode_ids_device"""
    eng = Engine(model_bytes(model))
    kind = "mixed" if model.startswith("mix") else "en"
    q, ctx = _qa_lines(corpus_gen, kind)
    for trunc, lines in (("only_second", q + ctx), ("only_first", ctx + q)):
        d_bytes, d_offs = _device(*oracle_py.pack(lines))
        ids, ido = _packed_device(eng, d_bytes, d_offs)
        n = len(lines) // 2
        other = np.diff(ido)[n:] if trunc == "only_first" else np.diff(ido)[:n]
        for tmpl in TEMPLATES[:3]:
            T = sum(len(x) for x in tmpl)
            w = 128
            shortest_room = w - T - int(other.max())
            for stride in (0, 16, shortest_room - 1):
                want = check(eng, d_bytes, d_offs, ids, ido, tmpl, w, trunc, True, stride, left=stride == 16,
                             what=(model,))
                assert "error" not in want and len(want["lengths"]) > n + 100
            # a room at the stride: pairs that need cutting cannot be laid out, and the least width comes back
            check(eng, d_bytes, d_offs, ids, ido, tmpl, w, trunc, True, shortest_room, what=(model,))
    eng.close()


def _offsets_check(eng, lines, shapes, what=()):
    b = Batch(eng, lines, -1)
    r, byte_spans, char_spans = b.reference()
    ids, ido = r["ids"], r["id_offsets"].astype(np.int64)
    for tmpl, w, trunc, overflow, stride in shapes:
        for unit, (be, en) in (("byte", byte_spans), ("char", char_spans)):
            check(eng, b.d_bytes, b.d_offs, ids, ido, tmpl, w, trunc, overflow, stride, -1, w % 2 == 1, unit, be, en,
                  what)


OFFSET_SHAPES = [(TEMPLATES[1], 0, "none", False, 0), (TEMPLATES[2], 24, "longest_first", False, 0),
                 (TEMPLATES[0], 33, "only_second", True, 8), (TEMPLATES[1], 40, "only_second", False, 0)]


@pytest.mark.parametrize("model", ["uni32k", "botchan8k", "mix_bf8k", "bpe32k", "mix_bpe4k"])
def test_offsets_golden_models(model, corpus_gen):
    """offsets in bytes and characters against spm_encode_offsets (+ unicode_spans), with edge and malformed lines"""
    eng = Engine(model_bytes(model))
    kind = "mixed" if model.startswith("mix") else "en"
    q, ctx = _qa_lines(corpus_gen, kind, long=False)
    _offsets_check(eng, q + ctx, OFFSET_SHAPES, (model,))
    _offsets_check(eng, ctx + q, [(TEMPLATES[1], 40, "only_first", True, 5)], (model,))
    eng.close()


def test_offsets_rule_set_and_user_defined(corpus_gen):
    from test_gpu_normalizer_rules import user_symbol_lines, user_symbol_models
    mb = mp.replace_flags(model_bytes("uni32k"), charsmap=cr.blob("delete_expand"))
    eng = Engine(mb)
    lines = cr.lines("delete_expand", corpus_gen, 9300, 600) + edge_lines()[:-2]
    _offsets_check(eng, lines[:2 * (len(lines) // 2)], OFFSET_SHAPES, ("delete_expand",))
    eng.close()
    lines = user_symbol_lines(corpus_gen)
    base, name, mb = user_symbol_models()[0]
    om = oracle_py.OracleModel(mb)
    eng = Engine(mb)
    t = om.types.copy()
    t[(t == mp.NORMAL) & (np.arange(len(t)) % 2 == 0)] = mp.UNUSED
    eng.set_types(t)
    _offsets_check(eng, lines[:2 * (len(lines) // 2)], OFFSET_SHAPES, (name,))
    eng.close()


def test_invariants_against_existing_calls(corpus_gen):
    """every B empty and no middle: the padded calls with frame (prefix, suffix) and eos_id = -1, type ids 1 exactly on
    the suffix; every A empty: only_second + overflow equals spm_encode_windows_device over the B sentences"""
    import torch
    mb = model_bytes("mix_bf8k")
    eng = Engine(mb)
    lines = edge_lines()[:-3] + corpus_gen.lines("mixed", 9150, 1500)
    pre, suf = (5, 6), (7,)
    n = len(lines)
    solo = Batch(eng, lines, -1)
    a_only = _device(*oracle_py.pack(lines + [b""] * n))
    b_only = _device(*oracle_py.pack([b""] * n + lines))
    for left in (False, True):
        for w, trunc in ((0, "none"), (12, "longest_first")):
            eng.set_encode_frame(list(pre), False, list(suf))
            want_ids, want_len = eng.encode_device_padded(solo.d_bytes, solo.d_offs, width=w, pad_id=0,
                                                          truncate=bool(w), pad_left=left)
            oi, osp, ol = eng.encode_offsets_device_padded(solo.d_bytes, solo.d_offs, width=w, pad_id=0,
                                                           truncate=bool(w), pad_left=left, unit="char", eos_id=-1)
            eng.set_encode_frame([], False, [])
            ids, lens, types, rp, rf, spans = run(eng, *a_only, (pre, (), suf), w, trunc, pad=0, left=left,
                                                  unit="char")
            assert torch.equal(ids, want_ids) and torch.equal(lens, want_len) and torch.equal(spans, osp)
            assert torch.equal(ids, oi) and torch.equal(lens, ol)
            cells = torch.arange(ids.shape[1], device="cuda")[None, :]
            start = (ids.shape[1] - lens)[:, None] if left else 0
            suffix_cells = (cells - start == (lens[:, None] - 1))
            assert torch.equal(types, suffix_cells.to(torch.int32))
            assert torch.equal(rp.cpu(), torch.arange(n, dtype=torch.int32)) and bool((rf == 0).all())
        for w, stride in ((16, 4), (40, 0)):
            eng.set_encode_frame(list(pre), False, list(suf))
            wi, wl, ws, wf, wsp = eng.encode_device_windows(solo.d_bytes, solo.d_offs, w, stride=stride, pad_id=0,
                                                            pad_left=left, unit="byte", eos_id=-1)
            eng.set_encode_frame([], False, [])
            ids, lens, types, rp, rf, spans = run(eng, *b_only, (pre, (), suf), w, "only_second", True, stride, pad=0,
                                                  left=left, unit="byte")
            assert torch.equal(ids, wi) and torch.equal(lens, wl) and torch.equal(rp, ws) and torch.equal(rf, wf)
            assert torch.equal(spans, wsp)
            k = torch.arange(w, device="cuda")[None, :] - ((w - lens)[:, None] if left else 0)
            assert torch.equal(types == 1, (k >= len(pre)) & (k < lens[:, None]))
    eng.close()


def test_engine_frame_does_not_apply(corpus_gen):
    """a bos:eos:reverse frame on the engine leaves the pair rows unchanged, and spm_encode_ids_device still applies it
    after the pair call"""
    import torch
    mb = model_bytes("uni32k")
    lines = corpus_gen.lines("en", 9600, 400) + edge_lines()[:-2]
    lines = lines[:2 * (len(lines) // 2)]
    d_bytes, d_offs = _device(*oracle_py.pack(lines))
    plain = Engine(mb)
    eng = Engine(mb)
    _frame(eng, mb, "bos:eos:reverse")
    framed_before = _packed_device(eng, d_bytes, d_offs)
    for args in ((TEMPLATES[1], 24, "longest_first"), (TEMPLATES[2], 128, "only_second", True, 6, -1, False, "char")):
        got, want = run(eng, d_bytes, d_offs, *args), run(plain, d_bytes, d_offs, *args)
        assert all(torch.equal(x, y) for x, y in zip(got, want))
    framed_after = _packed_device(eng, d_bytes, d_offs)
    assert all(np.array_equal(x, y) for x, y in zip(framed_before, framed_after))
    assert not np.array_equal(framed_after[1], _packed_device(plain, d_bytes, d_offs)[1])
    eng.close()
    plain.close()


def _raw(eng, d_bytes, d_offs, tmpl, width, trunc, stride, flags, bufs, rows_cap, cells_cap, n=None, stream=None,
         lens=None):
    (ids, types, spans, lengths, rp, rf) = bufs
    p = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    arr = lambda x: (ctypes.c_int32 * len(x))(*x)  # noqa: E731
    rows, w = ctypes.c_uint64(12345), ctypes.c_uint32(54321)
    pl, ml, sl = lens or tuple(len(x) for x in tmpl)
    rc = eng._lib.spm_encode_pairs_device(
        eng._h, p(d_bytes), p(d_offs), (d_offs.numel() - 1) // 2 if n is None else n,
        d_bytes.numel() if d_bytes is not None else 0, arr(tmpl[0]) if tmpl[0] is not None else None, pl,
        arr(tmpl[1]), ml, arr(tmpl[2]), sl, width, trunc, stride, -1, flags, p(ids), p(types), p(spans), rows_cap,
        cells_cap, p(lengths), p(rp), p(rf), ctypes.byref(rows), ctypes.byref(w), stream)
    return rc, rows.value, w.value


def _bufs(R, w, spans_on, fill=-7):
    import torch
    c = lambda k: torch.full((k,), fill, dtype=torch.int32, device="cuda")  # noqa: E731
    return (c(R * w), c(R * w), c(2 * R * w) if spans_on else None, c(R), c(R), c(R))


def test_capacity_and_retry(corpus_gen):
    """the width failure and the rows / cells failure report the exact width and R and write nothing; a retry at the
    reported size succeeds, and the Python wrapper retries on its own"""
    import torch
    eng = Engine(model_bytes("uni32k"))
    q, ctx = _qa_lines(corpus_gen, "en")
    d_bytes, d_offs = _device(*oracle_py.pack(q + ctx))
    ids, ido = _packed_device(eng, d_bytes, d_offs)
    tmpl = TEMPLATES[1]
    w, stride = 64, 16
    want = pairs_ref(ids, ido, *tmpl, w, "only_second", True, stride)
    R = len(want["lengths"])
    for spans_on in (False, True):
        flags = _capi.PAIR_OVERFLOW | (_capi.OFFSETS_CHARS if spans_on else 0)
        bufs = _bufs(R, w, spans_on)
        assert _raw(eng, d_bytes, d_offs, tmpl, w, 3, stride, flags, bufs, R - 1, R * w) == (_capi.SPM_ERR_CAPACITY, R, w)
        assert _raw(eng, d_bytes, d_offs, tmpl, w, 3, stride, flags, bufs, R, R * w - 1) == (_capi.SPM_ERR_CAPACITY, R, w)
        need = pairs_ref(ids, ido, *tmpl, 20, "only_second", True, stride)["width"]
        assert _raw(eng, d_bytes, d_offs, tmpl, 20, 3, stride, flags, bufs, R, R * w) == (_capi.SPM_ERR_CAPACITY, 0,
                                                                                           need)
        # NONE at a fixed width below the longest row: the longest row comes back
        longest = pairs_ref(ids, ido, *tmpl, 0, "none")["width"]
        assert _raw(eng, d_bytes, d_offs, tmpl, 300, 0, 0, flags & ~_capi.PAIR_OVERFLOW, bufs, R, R * w) == \
            (_capi.SPM_ERR_CAPACITY, 0, longest)
        assert all(t is None or bool((t == -7).all()) for t in bufs)
        assert _raw(eng, d_bytes, d_offs, tmpl, w, 3, stride, flags, bufs, R, R * w) == (0, R, w)
        assert np.array_equal(bufs[0].view(R, w).cpu().numpy(), want["ids"])
        R2 = len(pairs_ref(ids, ido, *tmpl, need, "only_second", True, stride)["lengths"])
        assert _raw(eng, d_bytes, d_offs, tmpl, need, 3, stride, flags, _bufs(R2, need, spans_on), R2, R2 * need) == \
            (0, R2, need)

    class Counting:
        def __init__(self, lib):
            self.lib, self.calls = lib, 0

        def __getattr__(self, name):
            if name == "spm_encode_pairs_device":
                self.calls += 1
            return getattr(self.lib, name)
    fresh = Engine(model_bytes("uni32k"))
    fresh._lib = Counting(fresh._lib)
    got = run(fresh, d_bytes, d_offs, tmpl, w, "only_second", True, stride)  # the first guess (n rows) is short
    assert fresh._lib.calls == 2 and np.array_equal(got[0].cpu().numpy(), want["ids"])
    got = run(fresh, d_bytes, d_offs, tmpl, w, "only_second", True, stride)  # the guess has grown: no retry
    assert fresh._lib.calls == 3 and np.array_equal(got[0].cpu().numpy(), want["ids"])
    got = run(fresh, d_bytes, d_offs, tmpl, 0, "none")  # width 0: the guessed width is short
    assert fresh._lib.calls == 5 and got[0].shape[1] == longest
    fresh._lib = fresh._lib.lib
    fresh.close()
    with pytest.raises(ValueError, match=str(need)):
        run(eng, d_bytes, d_offs, tmpl, 20, "only_second", True, stride)
    out = torch.empty(R * (2 * w + 3), dtype=torch.int32, device="cuda")
    got = eng.encode_device_pairs(d_bytes, d_offs, *tmpl, width=w, truncation="only_second", overflow=True,
                                  stride=stride, pad_id=-1, out=out)
    assert got[0].data_ptr() == out.data_ptr() and np.array_equal(got[0].cpu().numpy(), want["ids"])
    with pytest.raises(ValueError, match="capacity too small"):
        eng.encode_device_pairs(d_bytes, d_offs, *tmpl, width=w, truncation="only_second", overflow=True,
                                stride=stride, pad_id=-1, out=out[:(R - 1) * (2 * w + 3)])
    eng.close()


def test_errors_and_edge_cases(corpus_gen):
    import torch
    eng = Engine(model_bytes("uni32k"))
    lines = corpus_gen.lines("en", 9700, 400)
    d_bytes, d_offs = _device(*oracle_py.pack(lines))
    n, w = 200, 64
    bufs = _bufs(8 * n, w, True, 0)
    tmpl = TEMPLATES[1]
    T = 3

    def rc(tmpl=tmpl, width=w, trunc=1, stride=0, flags=0, bufs=bufs, **kw):
        return _raw(eng, kw.get("d_bytes", d_bytes), kw.get("d_offs", d_offs), tmpl, width, trunc, stride, flags,
                    bufs, 8 * n, 8 * n * w, n=n, lens=kw.get("lens"))[0]
    assert rc() == 0 and rc(flags=_capi.OFFSETS_CHARS) == 0 and rc(trunc=3, stride=2, flags=_capi.PAIR_OVERFLOW) == 0
    nospans = bufs[:2] + (None,) + bufs[3:]
    bad = [dict(flags=_capi.PAD_TRUNCATE), dict(flags=16), dict(trunc=4), dict(tmpl=((1,) * 65, (), ())),
           dict(tmpl=((), (32000,), ())), dict(tmpl=((), (), (-1,))), dict(width=0), dict(width=T),
           dict(trunc=0, flags=_capi.PAIR_OVERFLOW), dict(trunc=1, flags=_capi.PAIR_OVERFLOW), dict(stride=4),
           dict(trunc=2, stride=4), dict(flags=_capi.OFFSETS_CHARS, bufs=nospans), dict(d_offs=None),
           dict(tmpl=(None, (), ()), lens=(2, 0, 0))]
    bad += [dict(bufs=tuple(None if j == k else t for j, t in enumerate(bufs))) for k in (0, 1, 3, 4, 5)]
    assert rc(width=T + 1) == 0 and rc(trunc=0, width=0) == 0
    for b in bad:
        assert rc(**b) == 1, b
    misaligned = bufs[:2] + (bufs[2][1:],) + bufs[3:]
    assert rc(flags=_capi.OFFSETS_CHARS, bufs=misaligned) == 1
    with pytest.raises(ValueError, match="truncation"):
        run(eng, d_bytes, d_offs, tmpl, w, "first")
    with pytest.raises(ValueError, match="2n"):
        run(eng, d_bytes, d_offs[:-1], tmpl, w, "longest_first")
    # n == 0
    empty = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert _raw(eng, d_bytes, empty, tmpl, w, 1, 0, 0, (None,) * 6, 0, 0) == (0, 0, 0)
    for unit in (None, "char"):
        got = run(eng, d_bytes, empty, tmpl, w, "longest_first", unit=unit)
        assert got[0].shape[0] == 0 and all(t.numel() == 0 for t in got[1:])
    # a caller stream
    want = run(eng, d_bytes, d_offs, tmpl, 96, "only_first", True, 4, unit="char")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = run(eng, d_bytes, d_offs, tmpl, 96, "only_first", True, 4, unit="char")
        flat = torch.cat([t.reshape(-1) for t in got])  # work queued behind the call on s
    torch.cuda.current_stream().wait_stream(s)
    assert all(torch.equal(x, y) for x, y in zip(got, want))
    assert torch.equal(flat, torch.cat([t.reshape(-1) for t in want]))
    # no per-token traffic: the template up, the same few status words back for 10 and 20,000 pairs
    d2h = []
    for k in (20, 40000):
        db, do = _device(*oracle_py.pack(corpus_gen.lines("mixed", 9800, k)))
        for unit in (None, "char"):
            run(eng, db, do, tmpl, 128, "only_second", True, 4, unit=unit)
            i = eng.info()
            assert i.last_h2d_bytes == 4 * T
            d2h.append(i.last_d2h_bytes)
    assert d2h[0] == d2h[2] and d2h[1] == d2h[3] and d2h[1] < 1024
    eng.close()


def test_large_batch(corpus_gen):
    """300,000 pairs of bench.py's corpus at w = 128, longest_first, ids and character offsets, checked in slices"""
    eng = Engine(model_bytes("uni32k"))
    n = 300000
    buf, offs = corpus_gen.fill("en", CORPUS_SEED, 2 * n)
    d_bytes, d_offs = _device(buf, offs)
    r = eng.encode_offsets(buf, offs, eos_id=-1, pieces=False)
    cb, ce = unicode_spans(buf, offs, r["begin"], r["end"], r["id_offsets"])
    tmpl = TEMPLATES[1]
    got = [t.cpu().numpy() for t in run(eng, d_bytes, d_offs, tmpl, 32, "longest_first", unit="char")]
    ido = r["id_offsets"].astype(np.int64)
    for lo in range(0, n, 60000):
        hi = lo + 60000
        parts = [(ido[lo], ido[hi]), (ido[n + lo], ido[n + hi])]  # the slice's A lists, then its B lists
        sub = [np.concatenate([a[x:y] for x, y in parts]) for a in (r["ids"], cb, ce)]
        sub_ido = np.concatenate([ido[lo:hi] - ido[lo], ido[n + lo:n + hi + 1] - ido[n + lo] + ido[hi] - ido[lo]])
        want = pairs_ref(sub[0], sub_ido, *tmpl, 32, "longest_first", begin=sub[1], end=sub[2])
        for name, g in zip(NAMES, got):
            x = g[lo:hi]
            if name == "row_pair":
                x = x - lo
            assert np.array_equal(x, want[name]), (lo, name)
    ids = run(eng, d_bytes, d_offs, tmpl, 32, "longest_first")
    assert all(np.array_equal(a.cpu().numpy(), b) for a, b in zip(ids, got[:5]))
    eng.close()


def test_python_api(corpus_gen):
    """encode_pairs on str lists: EncodeAsIds of each member assembled by pairs_ref; with return_offsets,
    EncodeAsImmutableProto's begin / end; the (bytes, offsets) pairs give the same"""
    import torch
    mb = model_bytes("mix_bf8k")
    spp = SentencePieceProcessor(model_proto=mb)
    q, ctx = _qa_lines(corpus_gen, "mixed")
    first = [s.decode("utf-8", "replace") for s in q]
    second = [s.decode("utf-8", "replace") for s in ctx]
    lists = spp.EncodeAsIds(first + second)
    protos = spp.EncodeAsImmutableProto(first + second)
    ido = np.cumsum([0] + [len(x) for x in lists])
    flat = [t for x in lists for t in x]
    begin = [p.begin for g in protos for p in g]
    end = [p.end for g in protos for p in g]
    tmpl = TEMPLATES[2]
    for kw, want in (
            (dict(max_len=48), pairs_ref(flat, ido, *tmpl, 48, "longest_first", pad=0, begin=begin, end=end)),
            (dict(max_len=64, truncation="only_second", stride=16, pad_left=True),
             pairs_ref(flat, ido, *tmpl, 64, "only_second", True, 16, 0, True, begin, end)),
            (dict(), pairs_ref(flat, ido, *tmpl, 0, "none", pad=0, begin=begin, end=end))):
        got = spp.encode_pairs(first, second, prefix=tmpl[0], middle=tmpl[1], suffix=tmpl[2], pad_id=0,
                               return_offsets=True, **kw)
        names = ("ids", "lengths", "type_ids") + (("row_pair", "row_first") if "stride" in kw else ()) + ("spans",)
        assert len(got) == len(names)
        for name, g in zip(names, got):
            assert np.array_equal(g.cpu().numpy(), want[name]), (kw, name)
        plain = spp.encode_pairs(first, second, prefix=tmpl[0], middle=tmpl[1], suffix=tmpl[2], pad_id=0, **kw)
        assert len(plain) == len(names) - 1 and all(torch.equal(x, y) for x, y in zip(plain, got))
    enc1, enc2 = [s.encode() for s in first], [s.encode() for s in second]
    pair1, pair2 = _device(*oracle_py.pack(enc1)), _device(*oracle_py.pack(enc2))
    got = spp.encode_pairs(pair2, pair1, max_len=64, truncation="only_first", stride=3, pad_id=0)
    want = spp.encode_pairs(enc2, enc1, max_len=64, truncation="only_first", stride=3, pad_id=0)
    assert got[0].shape[0] > len(enc1) + 100
    assert all(torch.equal(x, y) for x, y in zip(got, want))
    with pytest.raises(ValueError, match="same number"):
        spp.encode_pairs(first, second[:-1])
