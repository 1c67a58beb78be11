"""Padded id tensors on the device: spm_encode_ids_device_padded (Engine.encode_device_padded) writes row i as sentence
i of spm_encode_ids_device under the encode frame, truncated and padded; spm_decode_ids_device (Engine.decode_device)
gives every row exactly the text spm_decode_ids gives its id list.  Batches hold the edge lines, empty sentences,
corpus lines and two documents long enough for the long-sentence kernels.  Needs an H100."""
import ctypes

import numpy as np
import pytest

from conftest import model_bytes
from extra_options import EDGE_LINES, OPTION_SETS
from oracle import oracle_py
from sentencepiece_b200.processor import extra_frame

pytestmark = pytest.mark.gpu
MODELS = [("uni32k", "en"), ("bpe32k", "en"), ("mix_bf8k", "mixed")]


def _engine(model):
    from sentencepiece_b200 import Engine
    return Engine(model_bytes(model))


def _frame(eng, model, options):
    from sentencepiece_b200 import _modelinfo
    from sentencepiece_b200.processor import extra_frame
    sp = _modelinfo.special_pieces(model_bytes(model))
    p, rev, s = extra_frame(options.split(":") if options else [], sp["bos_id"], sp["eos_id"])
    eng.set_encode_frame(p, rev, s)
    return len(p), len(s)


def _long_doc(corpus_gen, kind, seed, nbytes):
    return b" ".join(corpus_gen.lines(kind, seed, nbytes // 20))[:nbytes]


@pytest.fixture(scope="module")
def batches(corpus_gen):
    out = {}
    for model, kind in MODELS:
        lines = EDGE_LINES + [b""] * 3 + corpus_gen.lines(kind, 8081, 2000) + [b""] + \
            [_long_doc(corpus_gen, kind, 8082, 9000), _long_doc(corpus_gen, kind, 8083, 6000)]
        out[model] = oracle_py.pack(lines)
    return out


def _device(buf, offs):
    import torch
    return torch.from_numpy(buf.copy()).cuda(), torch.from_numpy(offs.astype(np.int64)).cuda()


def _packed_device(eng, d_bytes, d_offs):
    """spm_encode_ids_device of the batch -> (ids int32[], id_offsets int64[n+1]) on the host"""
    import torch
    n = d_offs.numel() - 1
    cap = 4 * d_bytes.numel() + 64 * n + 1024
    d_ids = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_ido = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    tot = eng.encode_device(d_bytes.data_ptr(), d_offs.data_ptr(), n, d_bytes.numel(), d_ids.data_ptr(), cap,
                            d_ido.data_ptr())
    return d_ids[:tot].cpu().numpy(), d_ido.cpu().numpy()


def pad_ref(ids, ido, w, pad, ns, truncate=False, left=False):
    """Rows of the framed lists ids[ido[i]:ido[i+1]] at width w: prefix ++ body[:w - np - ns] ++ suffix when truncating
    (the list's first real - ns ids, then its last ns), pad elsewhere -> (rows int32 [n, w], lengths int32 [n])"""
    ido = ido.astype(np.int64)
    lens = np.diff(ido)
    real = np.minimum(lens, w) if truncate else lens
    assert (real <= w).all()
    k = np.arange(w, dtype=np.int64)[None, :] - ((w - real)[:, None] if left else 0)
    valid = (k >= 0) & (k < real[:, None])
    src = np.where(k < (real - ns)[:, None], k, k + (lens - real)[:, None]) + ido[:-1, None]
    vals = ids[np.clip(src, 0, len(ids) - 1)] if len(ids) else np.zeros(src.shape, np.int32)
    return np.where(valid, vals, np.int32(pad)).astype(np.int32), real.astype(np.int32)


def _check(eng, d_bytes, d_offs, want_ids, want_ido, ns, width, pad, truncate=False, left=False):
    ids, lens = eng.encode_device_padded(d_bytes, d_offs, width=width, pad_id=pad, truncate=truncate, pad_left=left)
    w = width or int(np.diff(want_ido).max())
    rows, real = pad_ref(want_ids, want_ido, w, pad, ns, truncate, left)
    assert tuple(ids.shape) == rows.shape
    assert np.array_equal(lens.cpu().numpy(), real)
    assert np.array_equal(ids.cpu().numpy(), rows), (width, pad, truncate, left)


@pytest.mark.parametrize("model,kind", MODELS)
def test_rows_equal_encode_device(model, kind, batches):
    """width 0, fixed widths with truncation (down to the bare frame), left padding and pad ids -1 / 0 / a large id,
    under every frame of OPTION_SETS"""
    d_bytes, d_offs = _device(*batches[model])
    eng = _engine(model)
    for j, options in enumerate(OPTION_SETS):
        np_, ns = _frame(eng, model, options)
        want = _packed_device(eng, d_bytes, d_offs)
        pad = (-1, 0, 2 ** 31 - 1)[j % 3]
        _check(eng, d_bytes, d_offs, *want, ns, 0, pad)
        assert eng.info().last_deferred > 0
        _check(eng, d_bytes, d_offs, *want, ns, 0, pad, left=True)
        for width in sorted({np_ + ns, np_ + ns + 1, 5, 17, 64}):
            if width >= np_ + ns:
                _check(eng, d_bytes, d_offs, *want, ns, width, pad, truncate=True, left=width % 2 == 1)
        if np_ + ns > 1:  # (width 0 is the longest row)
            with pytest.raises(RuntimeError, match="shorter than the encode frame"):
                eng.encode_device_padded(d_bytes, d_offs, width=np_ + ns - 1, pad_id=0, truncate=True)
    # a fixed width that every row fits needs no truncation
    _frame(eng, model, "bos:eos")
    want = _packed_device(eng, d_bytes, d_offs)
    _check(eng, d_bytes, d_offs, *want, 1, int(np.diff(want[1]).max()) + 3, -1, left=True)
    eng.close()


def _raw_padded(eng, d_bytes, d_offs, out, cap, width, flags, lengths):
    w = ctypes.c_uint32(12345)
    rc = eng._lib.spm_encode_ids_device_padded(eng._h, d_bytes.data_ptr(), d_offs.data_ptr(), d_offs.numel() - 1,
                                               d_bytes.numel(), out.data_ptr(), cap, width, -1, flags,
                                               lengths.data_ptr(), ctypes.byref(w), None)
    return rc, w.value


def test_capacity_errors_write_nothing(batches):
    import torch
    from sentencepiece_b200 import _capi
    d_bytes, d_offs = _device(*batches["uni32k"])
    n = d_offs.numel() - 1
    eng = _engine("uni32k")
    _frame(eng, "uni32k", "bos:eos")
    longest = int(np.diff(_packed_device(eng, d_bytes, d_offs)[1]).max())
    out = torch.full((n * (longest + 1),), -7, dtype=torch.int32, device="cuda")
    lengths = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    # a row longer than a fixed width without truncation: the longest row length comes back
    assert _raw_padded(eng, d_bytes, d_offs, out, out.numel(), 40, 0, lengths) == (_capi.SPM_ERR_CAPACITY, longest)
    # room for fewer than n * w cells: w comes back, for width 0 and for a fixed width
    assert _raw_padded(eng, d_bytes, d_offs, out, n * longest - 1, 0, 0, lengths) == (_capi.SPM_ERR_CAPACITY, longest)
    assert _raw_padded(eng, d_bytes, d_offs, out, n * 30 - 1, 30, 1, lengths) == (_capi.SPM_ERR_CAPACITY, 30)
    assert bool((out == -7).all()) and bool((lengths == -7).all())
    assert _raw_padded(eng, d_bytes, d_offs, out, n * longest, 0, 0, lengths) == (0, longest)
    assert int(lengths.max()) == longest
    # the Python method: a longer row fails, a small `out` fails, width 0 grows its own buffer
    with pytest.raises(ValueError, match="does not fit width 40"):
        eng.encode_device_padded(d_bytes, d_offs, width=40, pad_id=0)
    with pytest.raises(ValueError, match="out_capacity too small"):
        eng.encode_device_padded(d_bytes, d_offs, pad_id=0, out=out[:n])
    eng._pad_guess = 2
    ids, _ = eng.encode_device_padded(d_bytes, d_offs, pad_id=0)
    assert tuple(ids.shape) == (n, longest) and eng._pad_guess == longest
    ids2, _ = eng.encode_device_padded(d_bytes, d_offs, pad_id=0, out=out)
    assert ids2.data_ptr() == out.data_ptr() and torch.equal(ids, ids2)
    eng.close()


def test_caller_stream_and_empty_batch(batches):
    import torch
    d_bytes, d_offs = _device(*batches["bpe32k"])
    eng = _engine("bpe32k")
    want = _packed_device(eng, d_bytes, d_offs)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ids, lens = eng.encode_device_padded(d_bytes, d_offs, pad_id=3)
        text = eng.decode_device(ids, lens)
    torch.cuda.current_stream().wait_stream(s)
    rows, real = pad_ref(*want, ids.shape[1], 3, 0)
    assert np.array_equal(ids.cpu().numpy(), rows) and np.array_equal(lens.cpu().numpy(), real)
    t, o = eng.decode_packed(*want)
    raw = t.tobytes()
    assert text == [raw[int(o[i]):int(o[i + 1])].decode("utf-8", errors="replace") for i in range(len(o) - 1)]
    empty_offs = torch.zeros(1, dtype=torch.int64, device="cuda")
    ids, lens = eng.encode_device_padded(d_bytes, empty_offs, pad_id=0)
    assert tuple(ids.shape) == (0, 0) and lens.numel() == 0
    assert eng.decode_device(torch.zeros((0, 8), dtype=torch.int64, device="cuda")) == []
    eng.close()


def test_large_batch(corpus_gen):
    buf, offs = corpus_gen.fill("en", 8084, 300000)
    d_bytes, d_offs = _device(buf, offs)
    eng = _engine("uni32k")
    _frame(eng, "uni32k", "bos:eos")
    want = _packed_device(eng, d_bytes, d_offs)
    _check(eng, d_bytes, d_offs, *want, 1, 0, -1)
    _check(eng, d_bytes, d_offs, *want, 1, 24, -1, truncate=True, left=True)
    eng.close()


def _texts(eng, lists):
    ido = np.zeros(len(lists) + 1, dtype=np.uint64)
    ido[1:] = np.cumsum([len(x) for x in lists])
    ids = np.concatenate([np.asarray(x, dtype=np.int32) for x in lists]) if int(ido[-1]) else np.zeros(0, np.int32)
    t, o = eng.decode_packed(ids, ido)
    raw = t.tobytes()
    return [raw[int(o[i]):int(o[i + 1])].decode("utf-8", errors="replace") for i in range(len(lists))]


@pytest.mark.parametrize("model,kind", MODELS)
def test_decode_rows(model, kind, batches):
    """int32 and int64 rows, with lengths, with a stop id and garbage after it (out-of-range ids included), and a
    column slice; mix_bf8k's rows hold BYTE pieces"""
    import torch
    d_bytes, d_offs = _device(*batches[model])
    eng = _engine(model)
    vocab = eng.info().vocab_size
    _frame(eng, model, "bos:eos")
    ids, lens = eng.encode_device_padded(d_bytes, d_offs, pad_id=-1)
    rows = ids.cpu().numpy()
    lists = [rows[i, :int(k)].tolist() for i, k in enumerate(lens.cpu().numpy())]
    want = _texts(eng, lists)
    assert eng.decode_device(ids, lens) == want
    assert eng.decode_device(ids.long(), lens) == want
    # a generation-shaped tensor: row i = list i, stop id, garbage; wider than its slice
    rng = np.random.default_rng(5)
    n, T = len(lists), ids.shape[1] + 1
    stop = 2  # </s>
    body = [[x for x in l if x != stop] for l in lists]
    gen = rng.integers(-2 ** 40, 2 ** 40, size=(n, T + 9), dtype=np.int64)
    for i, l in enumerate(body):
        gen[i, :len(l)] = l
        gen[i, len(l)] = stop
    g = torch.from_numpy(gen).cuda()
    want_body = _texts(eng, body)
    assert eng.decode_device(g[:, :T], stop_id=stop) == want_body
    assert eng.decode_device(g[:, :T].int(), stop_id=stop) == want_body  # (garbage wraps; it is never read)
    k = torch.tensor([len(l) for l in body], dtype=torch.int32, device="cuda")
    assert eng.decode_device(g[:, :T], lengths=k) == want_body
    short = torch.clamp(k - 2, min=0)
    assert eng.decode_device(g, lengths=short, stop_id=stop) == _texts(eng, [l[:max(len(l) - 2, 0)] for l in body])
    # an out-of-range id inside a row fails the call with its whole value; after the stop it is never read
    bad = g[:, :T].clone()
    j = max(range(n), key=lambda i: len(body[i]))
    bad[j, 1] = 2 ** 40 + 5
    with pytest.raises(RuntimeError, match=f"Invalid id: {2 ** 40 + 5}"):
        eng.decode_device(bad, stop_id=stop)
    bad32 = ids.clone()
    bad32[j, 0] = vocab
    with pytest.raises(RuntimeError, match=f"Invalid id: {vocab}"):
        eng.decode_device(bad32, lens)
    bad[j, 1] = body[j][1]
    bad[j, len(body[j]) + 1] = -5
    assert eng.decode_device(bad, stop_id=stop) == want_body
    eng.close()


def test_python_api(corpus_gen):
    import torch
    from sentencepiece_b200 import SentencePieceProcessor
    sp = SentencePieceProcessor(model_proto=model_bytes("uni32k"))
    lines = [l.decode() for l in corpus_gen.lines("en", 8085, 500)] + ["", "hello world", "▁"]
    for kw in ({}, dict(add_bos=True, add_eos=True), dict(reverse=True, add_eos=True)):
        want = sp.EncodeAsIds(lines, **kw)
        w = max(len(x) for x in want)
        ids, lens = sp.encode_padded(lines, pad_id=-1, **kw)
        assert ids.device.type == "cuda" and tuple(ids.shape) == (len(lines), w)
        assert ids.cpu().tolist() == [x + [-1] * (w - len(x)) for x in want]
        assert lens.cpu().tolist() == [len(x) for x in want]
        # truncated to 8 (the frame's suffix kept, as its first ids are), left-padded with 0
        ns = len(extra_frame(sp._options(kw.get("add_bos"), kw.get("add_eos"), kw.get("reverse")), 1, 2)[2])
        cut = [x if len(x) <= 8 else x[:8 - ns] + x[len(x) - ns:] for x in want]
        ids, lens = sp.encode_padded(lines, max_len=8, pad_id=0, truncate=True, pad_left=True, **kw)
        assert ids.cpu().tolist() == [[0] * (8 - len(x)) + x for x in cut]
        assert lens.cpu().tolist() == [len(x) for x in cut]
        assert sp.decode_padded(*sp.encode_padded(lines, pad_id=0, **kw)) == sp.DecodeIds(want)
    eos = sp._specials()["eos_id"]
    ids, lens = sp.encode_padded(lines, pad_id=5, add_eos=True)
    assert sp.decode_padded(ids.long(), stop_id=eos) == sp.DecodeIds(sp.EncodeAsIds(lines))
    # a (bytes, offsets) pair of CUDA tensors
    buf, offs = oracle_py.pack([l.encode() for l in lines])
    pair = (torch.from_numpy(buf.copy()).cuda(), torch.from_numpy(offs.view(np.int64)).cuda())
    assert torch.equal(sp.encode_padded(pair, pad_id=-1)[0], sp.encode_padded(lines, pad_id=-1)[0])
    with pytest.raises(ValueError, match="pad_id"):
        sp.encode_padded(lines)
    with pytest.raises(ValueError, match="engine's device"):
        sp.decode_padded(ids.cpu())


def test_default_width_after_empty_batches():
    """an empty batch, or one whose rows are all empty, leaves the width-0 path of the same engine working"""
    from sentencepiece_b200 import SentencePieceProcessor
    sp = SentencePieceProcessor(model_proto=model_bytes("uni32k"))
    for empty in ([], ["", ""]):
        ids, lens = sp.encode_padded(empty, pad_id=0)
        assert tuple(ids.shape) == (len(empty), 0) and lens.tolist() == [0] * len(empty)
        want = sp.EncodeAsIds(["hello", "hello world"])
        ids, lens = sp.encode_padded(["hello", "hello world"], pad_id=0)
        w = max(len(x) for x in want)
        assert ids.cpu().tolist() == [x + [0] * (w - len(x)) for x in want]


def test_model_pad_id_is_read_once(monkeypatch):
    """pad_id=None takes the model's CONTROL <pad> piece; the ModelProto is parsed once per engine, not per call"""
    from oracle import modelproto
    from sentencepiece_b200 import SentencePieceProcessor, _modelinfo
    C, N = modelproto.CONTROL, modelproto.NORMAL
    mb = modelproto.build_model([("<unk>", 0.0, modelproto.UNKNOWN), ("<s>", 0.0, C), ("</s>", 0.0, C), ("<pad>", 0.0, C),
                                 ("\u2581a", -1.0, N), ("a", -2.0, N), ("b", -2.5, N), ("\u2581", -3.0, N)])
    sp = SentencePieceProcessor(model_proto=mb)
    want = sp.EncodeAsIds(["a", "ab ba b", ""])  # (the processor reads bos / eos here, once)
    calls = []
    real = _modelinfo.special_pieces
    monkeypatch.setattr(_modelinfo, "special_pieces", lambda data: calls.append(1) or real(data))
    for _ in range(3):
        ids, _ = sp.encode_padded(["a", "ab ba b", ""])
        w = max(len(x) for x in want)
        assert ids.cpu().tolist() == [x + [3] * (w - len(x)) for x in want]
    assert sp.engine.pad_id() == 3 and len(calls) == 1
