"""spm_decode_stream_device (Engine.decode_stream_device, SentencePieceProcessor.decode_stream) call by call against
the restatement in tests/decode_stream_ref.py, the reference's stored round-trip digests, and its rules for finishing,
slot reuse and errors.  Needs an H100."""
import numpy as np
import pytest

from conftest import model_bytes
from decode_stream_ref import StreamRef, random_calls
from oracle import modelproto as mp
from refstore import digest, reference

pytestmark = pytest.mark.gpu
WS = "▁"
N, U, C, B = mp.NORMAL, mp.UNKNOWN, mp.CONTROL, mp.BYTE


def _byte_model():
    bp = [("<unk>", 0.0, U), ("<s>", 0.0, C), ("</s>", 0.0, C), ("A", 0.0, N), ("B", 0.0, N), ("C", 0.0, N)]
    bp += [("<0x%02X>" % i, 0.0, B) for i in range(256)]
    return mp.build_model(bp, byte_fallback=True)


def _state(n):
    import torch
    return torch.zeros((n, 16), dtype=torch.uint8, device="cuda")


def _one_per_call(eng, lists, final_extra=True, dtype=None):
    """feeds row i's list one id per call ([n, 1] int64 column slices; rows that ran out pass length 0) and finishes
    every row in one more call -> each row's texts"""
    import torch
    n, T = len(lists), max([len(x) for x in lists] + [1])
    full = torch.full((n, T + 1), -7, dtype=dtype or torch.int64)
    for i, x in enumerate(lists):
        full[i, :len(x)] = torch.tensor(x, dtype=full.dtype)
    full = full.cuda()
    lens = torch.tensor([len(x) for x in lists], dtype=torch.int32, device="cuda")
    st = _state(n)
    out = [[] for _ in range(n)]
    for j in range(T + (1 if final_extra else 0)):
        k = (lens > j).int()
        fin = (lens <= j).int() if j == T else None
        for i, t in enumerate(eng.decode_stream_device(full[:, j:j + 1], st, lengths=k, final=fin)):
            if j < len(lists[i]) or j == T:
                out[i].append(t)
    return out


def test_known_answers():
    from sentencepiece_b200 import Engine
    eng = Engine(_byte_model())
    b = lambda x: 6 + x  # noqa: E731
    ids = [1, 3, 4, b(0xE3), b(0x81), b(0x82), b(0x5A), b(0xCE), b(0xA9), 5, b(0xE0), b(0x80), b(0xE3), b(0x81),
           b(0x84), b(0xEF), b(0xBF), b(0xBD)]
    want = ["", "A", "B", "", "", "あ", "Z", "", "Ω", "C", "", "", "��", "", "い", "", "", "�"]
    got = _one_per_call(eng, [ids, [b(0xE3), b(0x81)], [b(0xE3), b(0x81), 3]])
    assert got[0] == want + [""]
    assert got[1] == ["", "", "��"]
    assert got[2] == ["", "", "��A", ""]
    eng.close()
    # the leading-U+2581 rule crosses call boundaries
    pieces = [("<unk>", 0.0, U), ("<s>", 0.0, C), ("</s>", 0.0, C), (WS + "ABC", 0.0, N), (WS + "DE", 0.0, N),
              ("F", 0.0, N), ("G" + WS + "H", 0.0, N), (WS, 0.0, N), (WS + WS, 0.0, N)]
    lists = [[1, 3, 0, 4, 5, 6, 2], [], [1, 2], [7, 7, 3, 3], [8, 5], [0, 3], [7], [8], [1, 7, 2, 8, 3], [1, 1, 7, 4]]
    for kw in ({}, dict(remove_extra_whitespaces=False), dict(add_dummy_prefix=False, remove_extra_whitespaces=False)):
        eng = Engine(mp.build_model(pieces, **kw))
        ido = np.zeros(len(lists) + 1, np.uint64)
        ido[1:] = np.cumsum([len(x) for x in lists])
        text, to = eng.decode_packed(np.concatenate([np.asarray(x, np.int32) for x in lists]), ido)
        raw = text.tobytes()
        got = _one_per_call(eng, lists)
        assert ["".join(g) for g in got] == [raw[int(to[i]):int(to[i + 1])].decode() for i in range(len(lists))], kw
        eng.close()


def _random_lists(m, rng, n, maxlen):
    vocab = len(m["pieces"])
    special = np.nonzero(np.asarray(m["types"]) != mp.NORMAL)[0]
    out = []
    for _ in range(n):
        a = rng.integers(0, vocab, size=int(rng.integers(0, maxlen)))
        msk = rng.random(len(a)) < 0.35
        if len(special) and msk.any():
            a[msk] = rng.choice(special, size=int(msk.sum()))
        out.append(a.astype(np.int32))
    return out


def _run_plan(eng, ref, lists, rng, dtype, slice_cols, max_step=4):
    """every row gets its own random splitting (0 ids per call included) and is finished with `final` in its last
    call; done rows then get garbage.  Each call's texts are compared with the restatement."""
    import torch
    n = len(lists)
    plans = [random_calls(rng, len(x), max_step) for x in lists]
    want = [ref.deltas(x, p) for x, p in zip(lists, plans)]
    steps = max(len(p) for p in plans) + 1
    K = max_step
    st = _state(n)
    pos = [0] * n
    for j in range(steps):
        wide = rng.integers(-2 ** 40, 2 ** 40, size=(n, K + slice_cols), dtype=np.int64)
        lens = np.zeros(n, np.int32)
        fin = np.zeros(n, np.int32)
        for i in range(n):
            if j < len(plans[i]):
                k = plans[i][j]
                wide[i, :k] = lists[i][pos[i]:pos[i] + k]
                lens[i] = k
                pos[i] += k
                fin[i] = j == len(plans[i]) - 1
            else:
                lens[i] = K  # a done row: its ids are neither read nor validated
        t = torch.from_numpy(wide).to(dtype).cuda()[:, :K]
        got = eng.decode_stream_device(t, st, lengths=torch.from_numpy(lens).cuda(), final=torch.from_numpy(fin).cuda())
        for i in range(n):
            w = want[i][j].decode() if j < len(plans[i]) else ""
            assert got[i] == w, (i, j)
    assert bool(((st[:, 12] & 1) == 1).all())


@pytest.mark.parametrize("model,kind", [("uni32k", "en"), ("mix_bf8k", "mixed"), ("bpe32k", "en"), ("botchan8k", "en"),
                                        ("mix_bpe4k", "mixed")])
def test_against_restatement(model, kind, corpus_gen):
    import torch
    from sentencepiece_b200 import Engine
    rng = np.random.default_rng(31)
    base = model_bytes(model)
    variants = [base, mp.replace_flags(base, remove_extra_whitespaces=False),
                mp.replace_flags(base, add_dummy_prefix=False, remove_extra_whitespaces=False)]
    for vi, mb in enumerate(variants):
        eng = Engine(mb)
        ref = StreamRef(mb)
        buf, offs = corpus_gen.fill(kind, 9301 + vi, 300)
        ids, ido = eng.encode_packed(buf, offs)
        lists = [ids[int(ido[i]):int(ido[i + 1])] for i in range(len(ido) - 1)]
        lists += _random_lists(mp.parse_model(mb), rng, 300, 40)
        _run_plan(eng, ref, lists, rng, torch.int64 if vi != 1 else torch.int32, slice_cols=3 * vi)
        eng.close()


@pytest.mark.parametrize("model,kind", [("uni32k", "en"), ("mix_bf8k", "mixed")])
def test_reference_digests(model, kind, corpus_gen):
    """the concatenated texts of 200k streamed round trips equal the reference's stored Decode results"""
    import torch
    from sentencepiece_b200 import Engine
    mb = model_bytes(model)
    want = reference(f"gpu_decode/round_trip/{model}/{kind}", None)
    buf, offs = corpus_gen.fill(kind, 9202, 200000)
    eng = Engine(mb)
    ids, ido = eng.encode_packed(buf, offs)
    n = len(ido) - 1
    lens = np.diff(ido.astype(np.int64))
    W, K = int(lens.max()), 5
    rows = np.zeros((n, W + K), np.int32)
    col = np.arange(W)[None, :]
    rows[:, :W][col < lens[:, None]] = ids
    t = torch.from_numpy(rows).cuda()
    dl = torch.from_numpy(lens.astype(np.int32)).cuda()
    st = _state(n)
    parts = [[] for _ in range(n)]
    for j in range(0, W + 1, K):
        k = torch.clamp(dl - j, 0, K).int()
        fin = (dl <= j + K).int()
        for i, x in enumerate(eng.decode_stream_device(t[:, j:j + K], st, lengths=k, final=fin)):
            if x:
                parts[i].append(x)
    texts = [("".join(p)).encode() for p in parts]
    to = np.zeros(n + 1, np.uint64)
    to[1:] = np.cumsum([len(x) for x in texts])
    text = np.frombuffer(b"".join(texts), np.uint8)
    assert digest((ids, ido), (text, to)) == want
    assert bool(((st[:, 12] & 1) == 1).all())
    eng.close()


def test_stop_final_done_and_reuse():
    import torch
    from sentencepiece_b200 import Engine
    eng = Engine(_byte_model())
    b = lambda x: 6 + x  # noqa: E731
    stop = 2
    st = _state(4)
    # row 0: ids then the stop id and out-of-range garbage; row 1: a held byte finished by final; row 2: runs on;
    # row 3: finished by final with nothing held
    t = torch.tensor([[3, b(0xE3), stop, 2 ** 40, -5], [4, b(0xE3), b(0x81), 0, 0], [b(0xCE), 0, 0, 0, 0],
                      [5, 5, 0, 0, 0]], dtype=torch.int64, device="cuda")
    lens = torch.tensor([5, 3, 1, 2], dtype=torch.int32, device="cuda")
    fin = torch.tensor([0, 1, 0, 1], dtype=torch.int32, device="cuda")
    assert eng.decode_stream_device(t, st, lengths=lens, stop_id=stop, final=fin) == ["A�", "B��", "", "CC"]
    assert (st[:, 12] & 1).tolist() == [1, 1, 0, 1]
    # done rows ignore later ids, even invalid ones; the live row continues
    t2 = torch.tensor([[2 ** 40], [-1], [b(0xA9)], [10 ** 6]], dtype=torch.int64, device="cuda")
    assert eng.decode_stream_device(t2, st, stop_id=stop) == ["", "", "Ω", ""]
    # a zeroed slot starts a new sequence mid-batch
    st[1] = 0
    t3 = torch.tensor([[3], [b(0xCE)], [4], [5]], dtype=torch.int64, device="cuda")
    assert eng.decode_stream_device(t3, st, stop_id=stop) == ["", "", "B", ""]
    t4 = torch.tensor([[3], [b(0xA9)], [stop], [5]], dtype=torch.int64, device="cuda")
    assert eng.decode_stream_device(t4, st, stop_id=stop) == ["", "Ω", "", ""]
    assert (st[:, 12] & 1).tolist() == [1, 0, 1, 1]
    eng.close()


def test_errors_leave_state_untouched():
    import torch
    from sentencepiece_b200 import Engine
    eng = Engine(_byte_model())
    b = lambda x: 6 + x  # noqa: E731
    st = _state(3)
    t = torch.tensor([[3, b(0xE3)], [b(0xF0), b(0x9F)], [1, 4]], dtype=torch.int64, device="cuda")
    assert eng.decode_stream_device(t, st) == ["A", "", "B"]
    snap = st.clone()
    bad = torch.tensor([[b(0x81)], [2 ** 40 + 5], [5]], dtype=torch.int64, device="cuda")
    with pytest.raises(RuntimeError, match=f"Invalid id: {2 ** 40 + 5}"):
        eng.decode_stream_device(bad, st)
    assert torch.equal(st, snap)
    bad32 = torch.tensor([[b(0x81)], [262], [5]], dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="Invalid id: 262"):
        eng.decode_stream_device(bad32, st)
    assert torch.equal(st, snap)
    # a row whose id count would pass 2^32 - 1
    over = snap.clone()
    over[2, 8:12] = 255
    with pytest.raises(RuntimeError, match="error 6"):
        eng.decode_stream_device(torch.tensor([[3], [3], [3]], device="cuda"), over)
    assert torch.equal(over[:2], snap[:2]) and bool((over[2, 8:12] == 255).all())
    # the same call with the bad id fixed
    good = torch.tensor([[b(0x81)], [b(0x98)], [5]], dtype=torch.int64, device="cuda")
    assert eng.decode_stream_device(good, st) == ["", "", "C"]
    assert eng.decode_stream_device(torch.tensor([[b(0x82)], [b(0x80)], [2]], device="cuda"), st) == ["あ", "😀", ""]
    # n == 0; argument errors
    assert eng.decode_stream_device(torch.zeros((0, 1), dtype=torch.int64, device="cuda"), _state(0)) == []
    with pytest.raises(ValueError):
        eng.decode_stream_device(good, _state(2))
    with pytest.raises(ValueError):
        eng.decode_stream_device(good, st, final=torch.zeros(3, dtype=torch.int64, device="cuda"))
    eng.close()
    # a model with a denormalizer_spec: SPM_ERR_UNSUPPORTED
    import os
    from conftest import ROOT
    with open(os.path.join(ROOT, "tests", "golden", "charsmaps", "nmt_nfkc_cf.bin"), "rb") as f:
        cm = f.read()
    eng = Engine(model_bytes("uni32k") + mp._ld(5, mp._ld(2, cm)))
    with pytest.raises(RuntimeError, match="denormalizer"):
        eng.decode_stream_device(torch.tensor([[5]], device="cuda"), _state(1))
    eng.close()


def test_caller_stream_large_batch_and_python_api(corpus_gen):
    import torch
    from sentencepiece_b200 import Engine, SentencePieceProcessor
    mb = model_bytes("mix_bf8k")
    eng = Engine(mb)
    buf, offs = corpus_gen.fill("mixed", 9303, 100000)
    ids, ido = eng.encode_packed(buf, offs)
    n = len(ido) - 1
    text, to = eng.decode_packed(ids, ido)
    raw = text.tobytes()
    want = [raw[int(to[i]):int(to[i + 1])].decode() for i in range(n)]
    lens = np.diff(ido.astype(np.int64))
    W = int(lens.max())
    rows = np.zeros((n, W + 1), np.int64)
    rows[:, :W][np.arange(W)[None, :] < lens[:, None]] = ids
    dl = torch.from_numpy(lens.astype(np.int32)).cuda()
    t = torch.from_numpy(rows).cuda()
    st = _state(n)
    parts = [[] for _ in range(n)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for j in range(0, W + 1, 7):
            k = torch.clamp(dl - j, 0, 7).int()
            fin = (dl <= j + 7).int()
            for i, x in enumerate(eng.decode_stream_device(t[:, j:j + 7], st, lengths=k, final=fin)):
                parts[i].append(x)
    torch.cuda.current_stream().wait_stream(s)
    assert ["".join(p) for p in parts] == want
    eng.close()
    # the Python API: one id per step from a [n] tensor, stop at eos, slot reuse
    sp = SentencePieceProcessor(model_proto=mb)
    lines = ["Hello world", "日本語のテキスト 😀", "", "naïve café"]
    enc = sp.EncodeAsIds(lines)
    from sentencepiece_b200 import _modelinfo
    eos = _modelinfo.special_pieces(mb)["eos_id"]
    T = max(len(x) for x in enc) + 2
    gen = torch.full((len(lines), T), 5, dtype=torch.int64)
    for i, x in enumerate(enc):
        gen[i, :len(x)] = torch.tensor(x)
        gen[i, len(x)] = eos
    gen = gen.cuda()
    ds = sp.decode_stream(len(lines), stop_id=eos)
    out = [""] * len(lines)
    for j in range(T):
        for i, x in enumerate(ds.step(gen[:, j])):
            out[i] += x
    assert out == [sp.DecodeIds(x) for x in enc]
    assert ds.done.dtype == torch.bool and ds.done.tolist() == [True] * len(lines)
    ds.reset([2])
    assert ds.done.tolist() == [True, True, False, True]
    first = gen[:, 0].clone()
    first[2] = enc[1][0]
    assert ds.step(first, final=torch.ones(len(lines), dtype=torch.int32, device="cuda")) == \
        ["", "", sp.DecodeIds(enc[1][:1]), ""]
    assert ds.done.tolist() == [True] * len(lines)
