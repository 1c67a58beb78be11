"""spm_encode_windows_device (Engine.encode_device_windows, SentencePieceProcessor.encode_windows): a device batch as
overlapping windows of one width with a stride, each row's sentence and first body token, and optionally every token's
begin / end.  The rows are checked against windows_ref, a numpy restatement of the semantics in include/spm_b200.h
applied to packed, framed results that other tests pin: the reference's own ids (tests/golden/ids), spm_encode_ids_device
and spm_encode_offsets (bytes, and characters through unicode_spans).  Needs an H100."""
import ctypes
import os

import numpy as np
import pytest

import charsmap_rules as cr
from conftest import model_bytes
from oracle import modelproto as mp
from oracle import oracle_py
from sentencepiece_b200 import Engine, SentencePieceProcessor, _capi
from sentencepiece_b200.processor import extra_frame, unicode_spans
from test_gpu_normalize import edge_lines
from test_gpu_offsets import FRAMES
from test_gpu_padded import _long_doc, _packed_device
from test_gpu_padded_offsets import Batch, _device, _frame

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN = [("uni32k", "en"), ("uni32k", "mixed"), ("botchan8k", "en"), ("mix_bf8k", "mixed"), ("bpe32k", "en"),
          ("mix_bpe4k", "mixed")]
CORPUS_SEED = 20260922  # bench.py's


def windows_ref(ids, begin, end, id_offsets, w, stride, np_, ns, pad, left):
    """The windows of the framed, packed lists ids[id_offsets[i]:id_offsets[i + 1]] (prefix of np_, body, suffix of
    ns) -> (rows int32 [R, w], spans int64 [R, w, 2] or None, lengths, row_sentence, row_first int32 [R]).  begin /
    end: the lists' offsets, or None."""
    ido = np.asarray(id_offsets, np.int64)
    fr = np_ + ns
    B = w - fr
    step = B - stride
    L = np.diff(ido) - fr
    m = np.where(L <= B, 1, 1 + (np.maximum(L - B, 0) + step - 1) // step)
    R = int(m.sum())
    rs = np.repeat(np.arange(len(L)), m)
    first = (np.arange(R) - np.repeat(np.cumsum(m) - m, m)) * step
    body = np.minimum(L[rs] - first, B)
    real = body + fr
    k = np.arange(w, dtype=np.int64)[None, :] - ((w - real)[:, None] if left else 0)
    valid = (k >= 0) & (k < real[:, None])
    src = np.where(k < np_, k, np.where(k < np_ + body[:, None], k + first[:, None], k + (L[rs] - body)[:, None]))
    src = np.clip(src + ido[rs][:, None], 0, max(int(ido[-1]) - 1, 0))

    def take(a, fill):
        a = np.asarray(a, np.int64)
        return np.where(valid, a[src] if len(a) else 0, fill)
    spans = None if begin is None else np.stack([take(begin, 0), take(end, 0)], axis=-1)
    return (take(ids, pad).astype(np.int32), spans, real.astype(np.int32), rs.astype(np.int32),
            first.astype(np.int32))


def frame_packed(ids, ido, prefix, rev, suffix):
    """the framed lists prefix ++ (body, reversed when rev) ++ suffix of packed raw lists"""
    ido = np.asarray(ido, np.int64)
    out, offs = [], [0]
    for i in range(len(ido) - 1):
        b = np.asarray(ids[ido[i]:ido[i + 1]], np.int32)
        out.append(np.concatenate([np.asarray(prefix, np.int32), b[::-1] if rev else b, np.asarray(suffix, np.int32)]))
        offs.append(offs[-1] + len(out[-1]))
    return (np.concatenate(out) if out else np.zeros(0, np.int32)), np.asarray(offs, np.int64)


def compare(got, want, what):
    names = ("ids", "lengths", "row_sentence", "row_first", "spans")
    order = (0, 2, 3, 4, 1)  # windows_ref's order -> the wrapper's
    for name, g, j in zip(names, got, order):
        w_ = want[j]
        g = g.cpu().numpy()
        assert g.shape == w_.shape, (what, name, g.shape, w_.shape)
        if not np.array_equal(g, w_):
            bad = np.argwhere(g != w_)[0]
            raise AssertionError(f"{what}: {name} differs at {bad.tolist()}: {g[tuple(bad)]} != {w_[tuple(bad)]}")


def run(eng, d_bytes, d_offs, w, stride, pad, left, unit=None, eos_id=-1):
    return eng.encode_device_windows(d_bytes, d_offs, w, stride=stride, pad_id=pad, pad_left=left, unit=unit,
                                     eos_id=eos_id)


@pytest.mark.parametrize("model,kind", GOLDEN)
def test_reference_ids(model, kind, corpus_gen):
    """the reference's stored ids, framed by extra_frame and cut by windows_ref, under every frame, both paddings and
    (w, stride) in (16, 0), (16, 15 - np - ns), (64, 16), (512, 128)"""
    from sentencepiece_b200 import _modelinfo
    from offsets_cases import options_of
    from test_gpu_offsets import set_frame
    z = np.load(os.path.join(GOLD, "ids", f"{model}__{kind}.npz"))
    buf, offs = corpus_gen.fill(kind, int(z["seed"]), int(z["n"]))
    d_bytes, d_offs = _device(buf, offs)
    mb = model_bytes(model)
    eng = Engine(mb)
    sp = _modelinfo.special_pieces(mb)
    for fr in FRAMES:
        set_frame(eng, sp, options_of(fr))
        prefix, rev, suffix = extra_frame(options_of(fr), sp["bos_id"], sp["eos_id"])
        fids, fido = frame_packed(z["ids"], z["id_offsets"], prefix, rev, suffix)
        np_, ns = len(prefix), len(suffix)
        for w, stride in ((16, 0), (16, 15 - np_ - ns), (64, 16), (512, 128)):
            for left in (False, True):
                want = windows_ref(fids, None, None, fido, w, stride, np_, ns, -1, left)
                compare(run(eng, d_bytes, d_offs, w, stride, -1, left), want, (model, kind, fr, w, stride, left))
    eng.close()


def _long_lines(corpus_gen, kind):
    return (edge_lines() + [_long_doc(corpus_gen, kind, 9400, 9000), _long_doc(corpus_gen, kind, 9401, 65536),
                            _long_doc(corpus_gen, "mixed", 9402, 70000)] + corpus_gen.lines(kind, 9403, 300)
            + corpus_gen.lines("mixed", 9404, 300) + [b""] * 2)


@pytest.mark.parametrize("model", ["uni32k", "botchan8k", "mix_bf8k"])
def test_long_inputs(model, corpus_gen):
    """edge lines (empty, whitespace-only, malformed UTF-8, the 64 KB and 1 MB documents), byte fallback and unknown
    runs with 9 KB / 64 KB documents: ids against spm_encode_ids_device, spans against spm_encode_offsets"""
    mb = model_bytes(model)
    eng = Engine(mb)
    kind = "mixed" if model.startswith("mix") else "en"
    lines = _long_lines(corpus_gen, kind)
    for fr in ("bos:eos", "eos:reverse:bos", ""):
        sp, np_, ns = _frame(eng, mb, fr)
        b = Batch(eng, lines, sp["eos_id"])
        pids, pido = _packed_device(eng, b.d_bytes, b.d_offs)
        r, byte_spans, char_spans = b.reference()
        assert np.array_equal(pids, r["ids"]) and np.array_equal(pido, r["id_offsets"].astype(np.int64))
        for w, stride, left in ((512, 128, False), (64, 16, True), (np_ + ns + 1, 0, False)):
            what = (model, fr, w, stride, left)
            compare(run(eng, b.d_bytes, b.d_offs, w, stride, -1, left),
                    windows_ref(pids, None, None, pido, w, stride, np_, ns, -1, left), what)
            if w == 64 or fr == "bos:eos":
                for unit, (be, en) in (("byte", byte_spans), ("char", char_spans)):
                    got = run(eng, b.d_bytes, b.d_offs, w, stride, -1, left, unit, sp["eos_id"])
                    compare(got, windows_ref(r["ids"], be, en, r["id_offsets"], w, stride, np_, ns, -1, left),
                            what + (unit,))
        if fr == "bos:eos":  # eos in every window of the 1 MB document holds its length
            ids, lens, rs, rf, spans = run(eng, b.d_bytes, b.d_offs, 64, 16, -1, False, "char", sp["eos_id"])
            doc = len(edge_lines()) - 1
            rows = (rs == doc).nonzero().flatten()
            assert rows.numel() > 1000
            nchars = len(lines[doc].decode("utf-8", "replace"))  # (ends inside a character: one U+FFFD)
            last = spans[rows, lens[rows].long() - 1].cpu().numpy()
            assert (last == nchars).all()
    eng.close()


@pytest.mark.parametrize("model", ["uni32k", "botchan8k", "mix_bf8k", "bpe32k", "mix_bpe4k"])
def test_offsets_golden_models(model, corpus_gen):
    """offsets in bytes and characters under every frame, with edge and malformed lines"""
    mb = model_bytes(model)
    eng = Engine(mb)
    kind = "mixed" if model.startswith("mix") else "en"
    lines = edge_lines()[:-2] + [b""] * 3 + corpus_gen.lines(kind, 9100, 1500)
    for fr in FRAMES:
        sp, np_, ns = _frame(eng, mb, fr)
        b = Batch(eng, lines, sp["eos_id"])
        r, byte_spans, char_spans = b.reference()
        for w, stride, left in ((16, 15 - np_ - ns, False), (24, 5, True)):
            for unit, (be, en) in (("byte", byte_spans), ("char", char_spans)):
                compare(run(eng, b.d_bytes, b.d_offs, w, stride, 0, left, unit, sp["eos_id"]),
                        windows_ref(r["ids"], be, en, r["id_offsets"], w, stride, np_, ns, 0, left),
                        (model, fr, w, stride, left, unit))
    eng.close()


def _offsets_check(eng, mb, lines, frames, shapes):
    for fr in frames:
        sp, np_, ns = _frame(eng, mb, fr)
        b = Batch(eng, lines, sp["eos_id"])
        r, byte_spans, char_spans = b.reference()
        for w, stride in shapes:
            for unit, (be, en) in (("byte", byte_spans), ("char", char_spans)):
                compare(run(eng, b.d_bytes, b.d_offs, w, stride, -1, True, unit, sp["eos_id"]),
                        windows_ref(r["ids"], be, en, r["id_offsets"], w, stride, np_, ns, -1, True), (fr, w, unit))


@pytest.mark.parametrize("name", ["nfkc_cf", "delete_expand"])
def test_offsets_rule_sets(name, corpus_gen):
    mb = mp.replace_flags(model_bytes("uni32k"), charsmap=cr.blob(name))
    eng = Engine(mb)
    _offsets_check(eng, mb, cr.lines(name, corpus_gen, 9300, 600) + edge_lines()[:-2], ("eos:reverse:bos",),
                   ((12, 3), (40, 10)))
    eng.close()


def test_offsets_user_defined_and_unused(corpus_gen):
    from test_gpu_normalizer_rules import user_symbol_lines, user_symbol_models
    lines = user_symbol_lines(corpus_gen)
    for base, name, mb in user_symbol_models():
        eng = Engine(mb)
        _offsets_check(eng, mb, lines, ("", "reverse:unk:eos"), ((10, 2),))
        eng.close()
    base, name, mb = user_symbol_models()[0]
    om = oracle_py.OracleModel(mb)
    eng = Engine(mb)
    t = om.types.copy()
    t[(t == mp.NORMAL) & (np.arange(len(t)) % 2 == 0)] = mp.UNUSED
    eng.set_types(t)
    _offsets_check(eng, mb, lines, ("bos:eos",), ((10, 2),))
    eng.close()


def test_invariant_rows_that_fit(corpus_gen):
    """every sentence fits: the windows are the padded rows cell for cell, R = n, row_sentence = 0..n-1, row_first = 0"""
    import torch
    mb = model_bytes("mix_bf8k")
    eng = Engine(mb)
    sp, np_, ns = _frame(eng, mb, "bos:eos")
    b = Batch(eng, edge_lines()[:-3] + corpus_gen.lines("mixed", 9150, 3000), sp["eos_id"])
    n = len(b.lines)
    w = int(eng.encode_device_padded(b.d_bytes, b.d_offs, pad_id=0)[0].shape[1]) + 3
    for left in (False, True):
        want_ids, want_len = eng.encode_device_padded(b.d_bytes, b.d_offs, width=w, pad_id=0, pad_left=left)
        ids, lens, rs, rf = run(eng, b.d_bytes, b.d_offs, w, 7, 0, left)
        assert torch.equal(ids, want_ids) and torch.equal(lens, want_len)
        assert torch.equal(rs.cpu(), torch.arange(n, dtype=torch.int32)) and bool((rf == 0).all())
        for unit in ("byte", "char"):
            pi, psp, pl = eng.encode_offsets_device_padded(b.d_bytes, b.d_offs, width=w, pad_id=0, pad_left=left,
                                                           unit=unit, eos_id=sp["eos_id"])
            ids, lens, rs, rf, spans = run(eng, b.d_bytes, b.d_offs, w, 7, 0, left, unit, sp["eos_id"])
            assert torch.equal(ids, pi) and torch.equal(lens, pl) and torch.equal(spans, psp)
            assert torch.equal(rs.cpu(), torch.arange(n, dtype=torch.int32)) and bool((rf == 0).all())
    eng.close()


def _raw(eng, d_bytes, d_offs, width, stride, flags, ids, spans, cap, lengths, rs, rf, n=None, stream=None):
    rows = ctypes.c_uint64(12345)
    p = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    rc = eng._lib.spm_encode_windows_device(eng._h, p(d_bytes), p(d_offs), d_offs.numel() - 1 if n is None else n,
                                            d_bytes.numel() if d_bytes is not None else 0, width, stride, -1, flags, 2,
                                            p(ids), p(spans), cap, p(lengths), p(rs), p(rf), ctypes.byref(rows), stream)
    return rc, rows.value


def test_capacity_and_retry(corpus_gen):
    """rows_capacity = R - 1: SPM_ERR_CAPACITY with *rows_out = R and nothing written, with and without spans; the
    retry with room succeeds.  The Python wrapper retries on its own and grows its guess"""
    import torch
    mb = model_bytes("uni32k")
    eng = Engine(mb)
    _frame(eng, mb, "bos:eos")
    lines = [_long_doc(corpus_gen, "en", 9500, 20000)] + corpus_gen.lines("en", 9501, 500)
    d_bytes, d_offs = _device(*oracle_py.pack(lines))
    w, stride = 32, 8
    R = run(eng, d_bytes, d_offs, w, stride, -1, False)[0].shape[0]
    n = len(lines)
    assert R > n + 100
    for spans_on in (False, True):
        ids = torch.full((R * w,), -7, dtype=torch.int32, device="cuda")
        spans = torch.full((2 * R * w,), -7, dtype=torch.int32, device="cuda") if spans_on else None
        lengths, rs, rf = (torch.full((R,), -7, dtype=torch.int32, device="cuda") for _ in range(3))
        flags = _capi.OFFSETS_CHARS if spans_on else 0
        assert _raw(eng, d_bytes, d_offs, w, stride, flags, ids, spans, R - 1, lengths, rs, rf) == \
            (_capi.SPM_ERR_CAPACITY, R)
        for t in (ids, spans, lengths, rs, rf):
            assert t is None or bool((t == -7).all())
        assert _raw(eng, d_bytes, d_offs, w, stride, flags, ids, spans, R, lengths, rs, rf) == (0, R)
        assert bool((lengths > 0).all()) and int(rs[-1]) == n - 1

    class Counting:
        def __init__(self, lib):
            self.lib, self.calls = lib, 0

        def __getattr__(self, name):
            if name == "spm_encode_windows_device":
                self.calls += 1
            return getattr(self.lib, name)
    fresh = Engine(mb)
    _frame(fresh, mb, "bos:eos")
    fresh._lib = Counting(fresh._lib)
    want = run(eng, d_bytes, d_offs, w, stride, -1, False)
    got = run(fresh, d_bytes, d_offs, w, stride, -1, False)  # the first guess (n rows) is short: one retry
    assert fresh._lib.calls == 2 and all(torch.equal(x, y) for x, y in zip(got, want))
    assert fresh._win_ratio == pytest.approx(R / n)
    got = run(fresh, d_bytes, d_offs, w, stride, -1, False)  # the guess has grown: no retry
    assert fresh._lib.calls == 3 and all(torch.equal(x, y) for x, y in zip(got, want))
    fresh._lib = fresh._lib.lib
    fresh.close()
    # `out`: exactly enough, then one row short
    out = torch.empty(R * (w + 3), dtype=torch.int32, device="cuda")
    got = eng.encode_device_windows(d_bytes, d_offs, w, stride=stride, pad_id=-1, out=out)
    assert all(torch.equal(x, y) for x, y in zip(got, want)) and got[0].data_ptr() == out.data_ptr()
    with pytest.raises(ValueError, match="rows_capacity too small"):
        eng.encode_device_windows(d_bytes, d_offs, w, stride=stride, pad_id=-1, out=out[:(R - 1) * (w + 3)])
    eng.close()


def test_errors_and_edge_cases(corpus_gen):
    import torch
    mb = model_bytes("uni32k")
    eng = Engine(mb)
    _frame(eng, mb, "bos:eos")
    d_bytes, d_offs = _device(*oracle_py.pack(corpus_gen.lines("en", 9700, 200)))
    n = 200
    ids = torch.zeros(n * 4 * 64, dtype=torch.int32, device="cuda")
    spans = torch.zeros(2 * ids.numel() + 2, dtype=torch.int32, device="cuda")
    lengths, rs, rf = (torch.zeros(4 * n, dtype=torch.int32, device="cuda") for _ in range(3))
    cap = 4 * n

    def rc(**kw):
        a = dict(d_bytes=d_bytes, d_offs=d_offs, width=64, stride=16, flags=0, ids=ids, spans=None, cap=cap,
                 lengths=lengths, rs=rs, rf=rf)
        a.update(kw)
        return _raw(eng, a["d_bytes"], a["d_offs"], a["width"], a["stride"], a["flags"], a["ids"], a["spans"],
                    a["cap"], a["lengths"], a["rs"], a["rf"], n=n)[0]
    assert rc() == 0 and rc(spans=spans, flags=_capi.OFFSETS_CHARS) == 0
    for bad in (dict(width=0), dict(flags=_capi.PAD_TRUNCATE), dict(flags=_capi.OFFSETS_CHARS), dict(flags=8),
                dict(ids=None), dict(lengths=None), dict(rs=None), dict(rf=None), dict(d_offs=None),
                dict(spans=spans[1:]), dict(width=2), dict(width=3, stride=1), dict(width=64, stride=62),
                dict(width=64, stride=100)):
        assert rc(**bad) == 1, bad
    one = eng.encode_device_windows(d_bytes, d_offs, 3, pad_id=0)  # one body id per window next to bos / eos
    assert bool((one[1] == 3).all()) and one[0].shape[0] > 4 * n
    with pytest.raises(RuntimeError, match="stride"):
        eng.encode_device_windows(d_bytes, d_offs, 10, stride=8, pad_id=0)
    with pytest.raises(ValueError, match="unit"):
        eng.encode_device_windows(d_bytes, d_offs, 10, pad_id=0, unit="word")
    with pytest.raises(ValueError, match="engine's device"):
        eng.encode_device_windows(d_bytes.cpu(), d_offs, 10, pad_id=0)
    # n == 0
    empty = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert _raw(eng, d_bytes, empty, 16, 0, 0, None, None, 0, None, None, None) == (0, 0)
    for unit in (None, "char"):
        got = eng.encode_device_windows(d_bytes, empty, 16, pad_id=0, unit=unit)
        assert tuple(got[0].shape) == (0, 16) and all(t.numel() == 0 for t in got[1:])
    # a caller stream
    want = eng.encode_device_windows(d_bytes, d_offs, 12, stride=3, pad_id=0, unit="char")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = eng.encode_device_windows(d_bytes, d_offs, 12, stride=3, pad_id=0, unit="char")
        flat = torch.cat([t.reshape(-1) for t in got])  # work queued behind the call on s
    torch.cuda.current_stream().wait_stream(s)
    assert all(torch.equal(x, y) for x, y in zip(got, want))
    assert torch.equal(flat, torch.cat([t.reshape(-1) for t in want]))
    # no per-token traffic: nothing up, the same few status words back for 10 and 20,000 sentences
    d2h = []
    for k in (10, 20000):
        db, do = _device(*oracle_py.pack(corpus_gen.lines("mixed", 9800, k)))
        for unit in (None, "char"):
            eng.encode_device_windows(db, do, 16, stride=4, pad_id=0, unit=unit)
            i = eng.info()
            assert i.last_h2d_bytes == 0
            d2h.append(i.last_d2h_bytes)
    assert d2h[0] == d2h[2] and d2h[1] == d2h[3] and d2h[1] < 1024
    eng.close()


def test_large_batch(corpus_gen):
    """300,000 sentences of bench.py's corpus at w = 64, stride = 16, ids and character offsets, checked in slices"""
    mb = model_bytes("uni32k")
    eng = Engine(mb)
    sp, np_, ns = _frame(eng, mb, "bos:eos")
    buf, offs = corpus_gen.fill("en", CORPUS_SEED, 300000)
    d_bytes, d_offs = _device(buf, offs)
    r = eng.encode_offsets(buf, offs, eos_id=sp["eos_id"], pieces=False)
    cb, ce = unicode_spans(buf, offs, r["begin"], r["end"], r["id_offsets"])
    pids, pido = _packed_device(eng, d_bytes, d_offs)
    assert np.array_equal(pids, r["ids"])
    got = [t.cpu().numpy() for t in run(eng, d_bytes, d_offs, 64, 16, -1, False, "char", sp["eos_id"])]
    ido = r["id_offsets"].astype(np.int64)
    for lo in range(0, 300000, 50000):
        hi = lo + 50000
        want = windows_ref(r["ids"], cb, ce, ido[lo:hi + 1], 64, 16, np_, ns, -1, False)
        sel = (got[2] >= lo) & (got[2] < hi)
        for g, j in zip(got, (0, 2, 3, 4, 1)):
            x = g[sel]
            if j == 3:
                x = x - lo
            assert np.array_equal(x, want[j]), (lo, j)
    ids = run(eng, d_bytes, d_offs, 64, 16, -1, False)
    assert all(np.array_equal(a.cpu().numpy(), b) for a, b in zip(ids, got[:4]))
    eng.close()


def _cut(items, B, stride):
    """the windows of per-sentence lists, in the test: (sentence, first, body slice)"""
    step = B - stride
    out = []
    for i, body in enumerate(items):
        m = 1 if len(body) <= B else 1 + -(-(len(body) - B) // step)
        out += [(i, j * step, body[j * step:j * step + B]) for j in range(m)]
    return out


def test_python_api(corpus_gen):
    """encode_windows on str input: row r is the window of EncodeAsIds / EncodeAsImmutableProto of its sentence, with
    bos / eos around every window; the (bytes, offsets) pair gives the same"""
    import torch
    mb = model_bytes("mix_bf8k")
    spp = SentencePieceProcessor(model_proto=mb)
    lines = edge_lines()[:-2] + [_long_doc(corpus_gen, "mixed", 9900, 5000)] + corpus_gen.lines("mixed", 9901, 300)
    strs = [s.decode("utf-8", "replace") for s in lines]
    protos = spp.EncodeAsImmutableProto(strs)
    from sentencepiece_b200 import _modelinfo
    special = _modelinfo.special_pieces(mb)
    bos, eos = special["bos_id"], special["eos_id"]
    for add, w, stride in ((False, 16, 4), (True, 40, 10)):
        ids, lens, rs, rf, offs = spp.encode_windows(strs, w, stride=stride, pad_id=-1, add_bos=add, add_eos=add,
                                                     return_offsets=True)
        f = 2 if add else 0
        cut = _cut([[(x.id, x.begin, x.end) for x in g] for g in protos], w - f, stride)
        assert ids.shape[0] == len(cut)
        ids, lens, rs, rf, offs = (t.cpu().tolist() for t in (ids, lens, rs, rf, offs))
        for r, (i, first, win) in enumerate(cut):
            n_ = len(strs[i])
            want_ids = ([bos] if add else []) + [t[0] for t in win] + ([eos] if add else [])
            want_sp = ([[0, 0]] if add else []) + [[t[1], t[2]] for t in win] + ([[n_, n_]] if add else [])
            assert (rs[r], rf[r], lens[r]) == (i, first, len(want_ids))
            assert ids[r] == want_ids + [-1] * (w - len(want_ids))
            assert offs[r] == want_sp + [[0, 0]] * (w - len(want_sp))
        plain = spp.encode_windows(strs, w, stride=stride, pad_id=-1, add_bos=add, add_eos=add)
        assert len(plain) == 4 and torch.equal(plain[0].cpu(), torch.tensor(ids, dtype=torch.int32))
    cut = _cut(spp.EncodeAsIds(strs), 8, 2)
    enc = [s.encode() for s in strs]
    pair = _device(*oracle_py.pack(enc))
    got = spp.encode_windows(pair, 8, stride=2, pad_id=0, pad_left=True)
    assert all(torch.equal(x, y) for x, y in zip(got, spp.encode_windows(enc, 8, stride=2, pad_id=0, pad_left=True)))
    rows = got[0].cpu().tolist()
    assert [row[8 - len(c[2]):] for row, c in zip(rows, cut)] == [list(c[2]) for c in cut]
