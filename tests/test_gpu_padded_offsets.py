"""spm_encode_offsets_device_padded (Engine.encode_offsets_device_padded, encode_padded(return_offsets=True)): padded
id rows of a device batch with every token's begin / end, in bytes or characters.  The ids, lengths and width equal
spm_encode_ids_device_padded's on the same arguments; the offsets equal spm_encode_offsets' packed begin / end (pinned
to the reference by tests/test_gpu_offsets.py), laid out in rows by pad_ref3 and, for characters, converted by
processor.unicode_spans.  Golden models under every frame, fixed widths with truncation, left padding, edge and
malformed lines, byte fallback, unknown runs, user-defined and UNUSED pieces, rule sets, long documents and a batch of
bench size.  Needs an H100."""
import ctypes

import numpy as np
import pytest

import charsmap_rules as cr
from conftest import model_bytes
from extra_options import EDGE_LINES
from offsets_cases import options_of
from oracle import modelproto as mp
from oracle import oracle_py
from sentencepiece_b200 import Engine, SentencePieceProcessor, _capi, _modelinfo
from sentencepiece_b200.processor import extra_frame, unicode_spans
from test_gpu_normalize import edge_lines
from test_gpu_offsets import FRAMES, set_frame

pytestmark = pytest.mark.gpu
MODELS = ["uni32k", "botchan8k", "mix_bf8k", "bpe32k", "mix_bpe4k"]
CORPUS_SEED = 20260922  # bench.py's


def pad_ref3(ids, begin, end, ido, w, pad, ns, truncate=False, left=False):
    """test_gpu_padded.pad_ref over three parallel arrays: the framed lists ids / begin / end[ido[i]:ido[i+1]] as rows
    of width w -> (ids int32 [n, w], spans int64 [n, w, 2], lengths int32 [n]); pad cells hold pad / (0, 0)"""
    ido = ido.astype(np.int64)
    lens = np.diff(ido)
    real = np.minimum(lens, w) if truncate else lens
    assert (real <= w).all()
    k = np.arange(w, dtype=np.int64)[None, :] - ((w - real)[:, None] if left else 0)
    valid = (k >= 0) & (k < real[:, None])
    src = np.clip(np.where(k < (real - ns)[:, None], k, k + (lens - real)[:, None]) + ido[:-1, None], 0,
                  max(len(ids) - 1, 0))

    def take(a, fill):
        a = np.asarray(a, np.int64)
        return np.where(valid, a[src] if len(a) else 0, fill)
    spans = np.stack([take(begin, 0), take(end, 0)], axis=-1)
    return take(ids, pad).astype(np.int32), spans, real.astype(np.int32)


def _device(buf, offs):
    import torch
    return torch.from_numpy(np.ascontiguousarray(buf, np.uint8).copy()).cuda(), \
        torch.from_numpy(np.asarray(offs, np.uint64).view(np.int64).copy()).cuda()


class Batch:
    """one batch on the host and the device, with spm_encode_offsets' packed result under the engine's frame"""

    def __init__(self, eng, lines, eos_id):
        self.lines = lines
        self.buf, self.offs = oracle_py.pack(lines)
        self.d_bytes, self.d_offs = _device(self.buf, self.offs)
        self.eos_id = eos_id
        self.eng = eng

    def reference(self):
        r = self.eng.encode_offsets(self.buf, self.offs, eos_id=self.eos_id, pieces=False)
        cb, ce = unicode_spans(self.buf, self.offs, r["begin"], r["end"], r["id_offsets"])
        return r, (r["begin"], r["end"]), (cb, ce)


def check(b, ns, width, pad, truncate=False, left=False, units=("byte", "char"), ref=None):
    """every unit: ids, spans and lengths against pad_ref3 of the host result, ids / lengths / width against
    spm_encode_ids_device_padded"""
    eng = b.eng
    r, byte_spans, char_spans = ref or b.reference()
    w = width or int(np.diff(r["id_offsets"].astype(np.int64)).max(initial=0))
    want_ids, want_len = eng.encode_device_padded(b.d_bytes, b.d_offs, width=width, pad_id=pad, truncate=truncate,
                                                  pad_left=left)
    for unit in units:
        ids, spans, lens = eng.encode_offsets_device_padded(b.d_bytes, b.d_offs, width=width, pad_id=pad,
                                                             truncate=truncate, pad_left=left, unit=unit,
                                                             eos_id=b.eos_id)
        be = byte_spans if unit == "byte" else char_spans
        rows, sp, real = pad_ref3(r["ids"], be[0], be[1], r["id_offsets"], w, pad, ns, truncate, left)
        what = (width, pad, truncate, left, unit)
        assert tuple(ids.shape) == (len(b.lines), w) and tuple(spans.shape) == (len(b.lines), w, 2), what
        assert np.array_equal(ids.cpu().numpy(), rows), what
        assert np.array_equal(lens.cpu().numpy(), real), what
        got = spans.cpu().numpy()
        if not np.array_equal(got, sp):
            i, j = (int(x[0]) for x in np.nonzero((got != sp).any(-1)))
            raise AssertionError(f"{what}: row {i} cell {j}: {got[i, j].tolist()} != {sp[i, j].tolist()} "
                                 f"({b.lines[i][:80]!r})")
        assert np.array_equal(ids.cpu().numpy(), want_ids.cpu().numpy()), what
        assert np.array_equal(lens.cpu().numpy(), want_len.cpu().numpy()), what


def sweep(b, np_, ns, pads=(-1, 0, 2 ** 31 - 1)):
    """width 0, left padding, fixed widths with truncation down to the bare frame, three pad ids, both units"""
    ref = b.reference()
    check(b, ns, 0, pads[0], ref=ref)
    check(b, ns, 0, pads[1], left=True, ref=ref)
    for j, width in enumerate(sorted({np_ + ns, np_ + ns + 1, 5, 17, 64})):
        if width >= np_ + ns:
            check(b, ns, width, pads[j % 3], truncate=True, left=width % 2 == 1, ref=ref)


def _frame(eng, mb, fr):
    """sets the frame of the option string fr -> (special pieces, prefix size, suffix size)"""
    sp = _modelinfo.special_pieces(mb)
    set_frame(eng, sp, options_of(fr))
    p, _, s = extra_frame(options_of(fr), sp["bos_id"], sp["eos_id"])
    return sp, len(p), len(s)


def _lines(corpus_gen, kind, seed, n):
    return EDGE_LINES + edge_lines()[:-2] + [b""] * 3 + corpus_gen.lines(kind, seed, n)


@pytest.mark.parametrize("model", MODELS)
def test_golden_models(model, corpus_gen):
    """every frame of test_gpu_offsets.FRAMES; edge, empty, whitespace-only and malformed lines among the corpus"""
    mb = model_bytes(model)
    eng = Engine(mb)
    kind = "mixed" if model.startswith("mix") else "en"
    lines = _lines(corpus_gen, kind, 9100, 2000)
    for fr in FRAMES:
        sp, np_, ns = _frame(eng, mb, fr)
        sweep(Batch(eng, lines, sp["eos_id"]), np_, ns)
    eng.close()


def test_unknown_detour_none_and_all(corpus_gen):
    """uni32k on mixed text: a batch in which no sentence holds the unknown id, and one in which every sentence does"""
    mb = model_bytes("uni32k")
    eng = Engine(mb)
    unk = eng.info().unk_id
    lines = corpus_gen.lines("mixed", 9200, 3000)
    ids, ido = eng.encode_packed(*oracle_py.pack(lines))
    has = [bool((ids[int(ido[i]):int(ido[i + 1])] == unk).any()) for i in range(len(lines))]
    sp, _, ns = _frame(eng, mb, "bos:eos")
    for holds in (False, True):
        part = [s for s, h in zip(lines, has) if h == holds]
        assert part
        check(Batch(eng, part, sp["eos_id"]), ns, 0, -1)
        assert eng.info().last_unk_detour == (len(part) if holds else 0)
    eng.close()


def test_user_defined_and_unused(corpus_gen):
    from test_gpu_normalizer_rules import user_symbol_lines, user_symbol_models
    lines = user_symbol_lines(corpus_gen)
    for base, name, mb in user_symbol_models():
        eng = Engine(mb)
        for fr in ("", "reverse:unk:eos"):
            sp, np_, ns = _frame(eng, mb, fr)
            b = Batch(eng, lines, sp["eos_id"])
            check(b, ns, 0, -1)
            check(b, ns, np_ + ns + 3, 0, truncate=True, left=True)
        eng.close()
    base, name, mb = user_symbol_models()[0]
    om = oracle_py.OracleModel(mb)
    eng = Engine(mb)
    t = om.types.copy()
    t[(t == mp.NORMAL) & (np.arange(len(t)) % 2 == 0)] = mp.UNUSED
    eng.set_types(t)
    sp, np_, ns = _frame(eng, mb, "bos:eos")
    sweep(Batch(eng, lines, sp["eos_id"]), np_, ns)
    eng.close()


@pytest.mark.parametrize("name", ["nfkc_cf", "delete_expand"])
def test_rule_sets(name, corpus_gen):
    mb = mp.replace_flags(model_bytes("uni32k"), charsmap=cr.blob(name))
    eng = Engine(mb)
    sp, _, ns = _frame(eng, mb, "eos:reverse:bos")
    b = Batch(eng, cr.lines(name, corpus_gen, 9300, 600) + edge_lines()[:-2], sp["eos_id"])
    check(b, ns, 0, -1)
    check(b, ns, 9, 0, truncate=True, left=True)
    eng.close()


def _long_doc(corpus_gen, kind, seed, nbytes):
    return b" ".join(corpus_gen.lines(kind, seed, nbytes // 20))[:nbytes]


@pytest.mark.parametrize("model", ["uni32k", "botchan8k", "mix_bf8k"])
def test_long_documents(model, corpus_gen):
    """9 KB and 64 KB documents (the long-sentence kernels, and many sweep blocks per row), with the 64 KB and 1 MB
    one-line documents of test_gpu_normalize.edge_lines, the last of which ends inside a character"""
    mb = model_bytes(model)
    eng = Engine(mb)
    kind = "mixed" if model.startswith("mix") else "en"
    lines = [_long_doc(corpus_gen, kind, 9400, 9000), _long_doc(corpus_gen, kind, 9401, 65536),
             _long_doc(corpus_gen, "mixed", 9402, 70000)] + edge_lines()[-2:] + corpus_gen.lines(kind, 9403, 300)
    sp, _, ns = _frame(eng, mb, "bos:eos")
    b = Batch(eng, lines, sp["eos_id"])
    check(b, ns, 0, -1)
    assert eng.info().last_deferred > 0
    check(b, ns, 100, 0, truncate=True, left=True)
    sp, _, ns = _frame(eng, mb, "eos:reverse:bos")
    check(b, ns, 0, 7, units=("char",))
    eng.close()


def test_bench_size_batch(corpus_gen):
    """1M sentences of bench.py's English corpus on uni32k (several K11 chunks): every real cell against the host
    result, every pad cell against the pad id and (0, 0)"""
    import torch
    mb = model_bytes("uni32k")
    eng = Engine(mb)
    sp, _, _ = _frame(eng, mb, "bos:eos")
    buf, offs = corpus_gen.fill("en", CORPUS_SEED, 1000000)
    d_bytes, d_offs = _device(buf, offs)
    r = eng.encode_offsets(buf, offs, eos_id=sp["eos_id"], pieces=False)
    cb, ce = unicode_spans(buf, offs, r["begin"], r["end"], r["id_offsets"])
    want_ids, want_len = eng.encode_device_padded(d_bytes, d_offs, pad_id=-1)
    for unit, (b, e) in (("byte", (r["begin"], r["end"])), ("char", (cb, ce))):
        ids, spans, lens = eng.encode_offsets_device_padded(d_bytes, d_offs, pad_id=-1, unit=unit, eos_id=sp["eos_id"])
        assert torch.equal(ids, want_ids) and torch.equal(lens, want_len)
        assert torch.equal(lens.cpu().long(), torch.from_numpy(np.diff(r["id_offsets"].astype(np.int64))))
        mask = torch.arange(ids.shape[1], device="cuda")[None, :] < lens[:, None]
        assert torch.equal(ids[mask].cpu(), torch.from_numpy(r["ids"]))
        real = spans[mask].cpu().numpy()
        assert np.array_equal(real[:, 0], np.asarray(b, np.int64)) and np.array_equal(real[:, 1], np.asarray(e, np.int64))
        assert bool((ids[~mask] == -1).all()) and bool((spans[~mask] == 0).all())
    eng.close()


def test_python_api(corpus_gen):
    """encode_padded(return_offsets=True) on str and bytes lists: row i is EncodeAsImmutableProto(input i)'s ids and
    begin / end, then pads; truncation and left padding as the id rows; a (bytes, offsets) pair of CUDA tensors"""
    import torch
    mb = model_bytes("mix_bf8k")
    spp = SentencePieceProcessor(model_proto=mb)
    lines = edge_lines()[:-2] + corpus_gen.lines("mixed", 9500, 400)
    strs = [s.decode("utf-8", "replace") for s in lines]
    for items in (strs, lines):
        for opts in ("", "bos:eos"):
            spp.SetEncodeExtraOptions(opts)
            protos = spp.EncodeAsImmutableProto(items)
            ids, lens, offs = spp.encode_padded(items, pad_id=-1, return_offsets=True)
            assert offs.dtype == torch.int32 and tuple(offs.shape) == tuple(ids.shape) + (2,)
            ids, lens, offs = ids.cpu().tolist(), lens.cpu().tolist(), offs.cpu().tolist()
            for i, g in enumerate(protos):
                assert lens[i] == len(g)
                assert ids[i][:lens[i]] == [x.id for x in g] and set(ids[i][lens[i]:]) <= {-1}
                assert offs[i][:lens[i]] == [[x.begin, x.end] for x in g], items[i][:60]
                assert all(c == [0, 0] for c in offs[i][lens[i]:])
            # truncated to 6 with eos kept, left-padded: the same cells as the id rows
            a, la = spp.encode_padded(items, max_len=6, pad_id=0, truncate=True, pad_left=True)
            b, lb, ob = spp.encode_padded(items, max_len=6, pad_id=0, truncate=True, pad_left=True, return_offsets=True)
            assert torch.equal(a, b) and torch.equal(la, lb)
            for i, g in enumerate(protos):
                keep = [[x.begin, x.end] for x in g]
                keep = keep if len(keep) <= 6 else keep[:6 - (opts != "")] + keep[len(keep) - (opts != ""):]
                assert ob[i].cpu().tolist() == [[0, 0]] * (6 - len(keep)) + keep
    spp.SetEncodeExtraOptions("")
    s = "héllo wörld ▁ x"
    ids, lens, offs = spp.encode_padded([s], pad_id=0, add_eos=True, return_offsets=True)
    assert offs[0, int(lens[0]) - 1].tolist() == [len(s), len(s)]
    # the (bytes, offsets) pair: characters of each input's bytes
    buf, o = oracle_py.pack(lines)
    pair = _device(buf, o)
    got = spp.encode_padded(pair, pad_id=-1, return_offsets=True)
    want = spp.encode_padded(lines, pad_id=-1, return_offsets=True)
    assert all(torch.equal(x, y) for x, y in zip(got, want))
    # the default return value is unchanged
    assert len(spp.encode_padded(strs[:3], pad_id=0)) == 2


def test_caller_stream(corpus_gen):
    import torch
    mb = model_bytes("bpe32k")
    eng = Engine(mb)
    sp, _, _ = _frame(eng, mb, "bos:eos")
    b = Batch(eng, corpus_gen.lines("en", 9600, 3000), sp["eos_id"])
    want = eng.encode_offsets_device_padded(b.d_bytes, b.d_offs, pad_id=-1, unit="char")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = eng.encode_offsets_device_padded(b.d_bytes, b.d_offs, pad_id=-1, unit="char")
        flat = torch.cat([got[0].reshape(-1), got[1].reshape(-1), got[2]])  # work queued behind the call on s
    torch.cuda.current_stream().wait_stream(s)
    assert all(torch.equal(x, y) for x, y in zip(got, want))
    assert torch.equal(flat, torch.cat([want[0].reshape(-1), want[1].reshape(-1), want[2]]))
    eng.close()


def _raw(eng, d_bytes, d_offs, ids, spans, cap, width, flags, lengths, n=None, eos=-1):
    w = ctypes.c_uint32(12345)
    rc = eng._lib.spm_encode_offsets_device_padded(
        eng._h, d_bytes.data_ptr() if d_bytes is not None else None, d_offs.data_ptr() if d_offs is not None else None,
        d_offs.numel() - 1 if n is None else n, d_bytes.numel() if d_bytes is not None else 0, eos,
        ids.data_ptr() if ids is not None else None, spans.data_ptr() if spans is not None else None, cap, width, -1,
        flags, lengths.data_ptr() if lengths is not None else None, ctypes.byref(w), None)
    return rc, w.value


def test_errors(corpus_gen):
    import torch
    mb = model_bytes("uni32k")
    eng = Engine(mb)
    _frame(eng, mb, "bos:eos")
    b = Batch(eng, corpus_gen.lines("en", 9700, 500), 2)
    n = len(b.lines)
    longest = int(eng.encode_device_padded(b.d_bytes, b.d_offs, pad_id=0)[0].shape[1])
    ids = torch.full((n * (longest + 1),), -7, dtype=torch.int32, device="cuda")
    spans = torch.full((2 * ids.numel(),), -7, dtype=torch.int32, device="cuda")
    lengths = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    C = _capi.OFFSETS_CHARS
    # a row longer than a fixed width without truncation; too small a capacity (width 0 and fixed): nothing written
    assert _raw(eng, b.d_bytes, b.d_offs, ids, spans, ids.numel(), 10, C, lengths) == (_capi.SPM_ERR_CAPACITY, longest)
    assert _raw(eng, b.d_bytes, b.d_offs, ids, spans, n * longest - 1, 0, C, lengths) == (_capi.SPM_ERR_CAPACITY, longest)
    assert _raw(eng, b.d_bytes, b.d_offs, ids, spans, n * 8 - 1, 8, 1, lengths) == (_capi.SPM_ERR_CAPACITY, 8)
    assert bool((ids == -7).all()) and bool((spans == -7).all()) and bool((lengths == -7).all())
    assert _raw(eng, b.d_bytes, b.d_offs, ids, spans, n * longest, 0, C, lengths) == (0, longest)
    # unknown flags, null pointers, truncating below the frame
    assert _raw(eng, b.d_bytes, b.d_offs, ids, spans, ids.numel(), 0, 8, lengths)[0] == 1
    assert _raw(eng, b.d_bytes, b.d_offs, ids, None, ids.numel(), 0, 0, lengths)[0] == 1
    assert _raw(eng, b.d_bytes, b.d_offs, None, spans, ids.numel(), 0, 0, lengths)[0] == 1
    assert _raw(eng, b.d_bytes, b.d_offs, ids, spans, ids.numel(), 0, 0, None)[0] == 1
    assert _raw(eng, b.d_bytes, None, ids, spans, ids.numel(), 0, 0, lengths, n=n)[0] == 1
    assert _raw(eng, b.d_bytes, b.d_offs, ids, spans, ids.numel(), 1, 1, lengths)[0] == 1
    assert _raw(eng, b.d_bytes, b.d_offs, ids, spans[1:], ids.numel() - 1, 0, 0, lengths)[0] == 1  # spans misaligned
    with pytest.raises(RuntimeError, match="shorter than the encode frame"):
        eng.encode_offsets_device_padded(b.d_bytes, b.d_offs, width=1, pad_id=0, truncate=True)
    # the ids call keeps refusing the new bit
    w = ctypes.c_uint32()
    assert eng._lib.spm_encode_ids_device_padded(eng._h, b.d_bytes.data_ptr(), b.d_offs.data_ptr(), n,
                                                 b.d_bytes.numel(), ids.data_ptr(), ids.numel(), 0, -1, C,
                                                 lengths.data_ptr(), ctypes.byref(w), None) == 1
    # Python: a fixed width too small, a small `out`, tensors on the host, a bad unit
    with pytest.raises(ValueError, match="does not fit width 10"):
        eng.encode_offsets_device_padded(b.d_bytes, b.d_offs, width=10, pad_id=0)
    with pytest.raises(ValueError, match="out_capacity too small"):
        eng.encode_offsets_device_padded(b.d_bytes, b.d_offs, pad_id=0, out=ids[:3 * n + 1])
    with pytest.raises(ValueError, match="engine's device"):
        eng.encode_offsets_device_padded(b.d_bytes.cpu(), b.d_offs, pad_id=0)
    with pytest.raises(ValueError, match="unit"):
        eng.encode_offsets_device_padded(b.d_bytes, b.d_offs, pad_id=0, unit="word")
    # n == 0
    empty = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert _raw(eng, b.d_bytes, empty, None, None, 0, 0, C, None) == (0, 0)
    i, s, l = eng.encode_offsets_device_padded(b.d_bytes, empty, pad_id=0, unit="char")
    assert tuple(i.shape) == (0, 0) and tuple(s.shape) == (0, 0, 2) and l.numel() == 0
    eng.close()


def test_transfers(corpus_gen):
    """nothing goes up, and the same fixed number of bytes comes back for 10 and for 20,000 sentences"""
    mb = model_bytes("uni32k")
    eng = Engine(mb)
    sp, _, _ = _frame(eng, mb, "bos:eos")
    d2h = []
    for n in (10, 20000):
        lines = corpus_gen.lines("mixed", 9800, n)
        b = Batch(eng, lines, sp["eos_id"])
        eng.encode_offsets_device_padded(b.d_bytes, b.d_offs, pad_id=-1, unit="char")
        i = eng.info()
        assert i.last_h2d_bytes == 0
        d2h.append(i.last_d2h_bytes)
    assert d2h[0] == d2h[1] and 0 < d2h[0] < 1024
    eng.close()
