"""Host-buffer C ABI on large batches: the fused path (one kernel launch, streamed input, in-kernel
compaction, engine.cu encode_host_fused), its chunked fallback (encode_host_streamed) and the plain
path must return identical ids; checked against the oracle on a sample.  Needs an H100."""
import os

import numpy as np
import pytest

from conftest import model_bytes
from oracle import oracle_py

pytestmark = pytest.mark.gpu
N = 420_000  # > pipeline_min_sentences (300k): spm_encode_ids takes the large-batch paths


def _engine(model, **env):
    """engine created under the given SPM_B200_* environment settings (read at engine creation)"""
    from sentencepiece_b200 import Engine
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return Engine(model_bytes(model))
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _ragged(buf, offs, rng, extra):
    """insert empty sentences and the `extra` byte strings at random positions"""
    raw = buf.tobytes()[: int(offs[-1])]
    sents = [raw[int(offs[i]):int(offs[i + 1])] for i in range(len(offs) - 1)]
    for pos in sorted(rng.integers(0, len(sents), size=200).tolist(), reverse=True):
        sents.insert(pos, b"")
    for e in extra:
        sents.insert(int(rng.integers(0, len(sents))), e)
    lens = np.fromiter((len(s) for s in sents), dtype=np.uint64, count=len(sents))
    o = np.zeros(len(sents) + 1, dtype=np.uint64)
    np.cumsum(lens, out=o[1:])
    return np.frombuffer(b"".join(sents), dtype=np.uint8).copy(), o


@pytest.mark.parametrize("model,kind", [("uni32k", "en"), ("mix_bf8k", "mixed"), ("bpe32k", "en")])
def test_fused_equals_chunked_equals_plain(model, kind, corpus_gen):
    buf, offs = corpus_gen.fill(kind, 7001, N)
    fused = _engine(model)
    a, ao = fused.encode_packed(buf, offs)
    chunked = _engine(model, SPM_B200_FUSED=0)
    b, bo = chunked.encode_packed(buf, offs)
    plain = _engine(model, SPM_B200_FUSED=0, SPM_B200_SORT=0)
    c, co = plain.encode_packed(buf, offs)
    assert np.array_equal(ao, bo) and np.array_equal(a, b)
    assert np.array_equal(ao, co) and np.array_equal(a, c)
    # twice through the same engine: buffers are reused
    a2, ao2 = fused.encode_packed(buf, offs)
    assert np.array_equal(ao, ao2) and np.array_equal(a, a2)
    om = oracle_py.OracleModel(model_bytes(model))
    raw = buf.tobytes()
    for i in range(0, N, 4999):
        assert a[int(ao[i]):int(ao[i + 1])].tolist() == om.encode(raw[int(offs[i]):int(offs[i + 1])])[0].tolist(), i
    for e in (fused, chunked, plain):
        e.close()


def test_fused_falls_back_on_long_sentences(corpus_gen):
    """sentences the lane kernel defers (longer than its slab) make the fused attempt incomplete: the
    batch is redone in chunks and the result is still exact; empty sentences in between."""
    rng = np.random.default_rng(5)
    buf, offs = corpus_gen.fill("en", 7002, N)
    raw = buf.tobytes()
    long1 = raw[: 6000]
    long2 = (b"x" * 3000) + b" " + raw[100:2000]
    rb, ro = _ragged(buf, offs, rng, [long1, long2])
    eng = _engine("uni32k")
    a, ao = eng.encode_packed(rb, ro)
    ref = _engine("uni32k", SPM_B200_FUSED=0, SPM_B200_SORT=0)
    b, bo = ref.encode_packed(rb, ro)
    assert np.array_equal(ao, bo) and np.array_equal(a, b)
    om = oracle_py.OracleModel(model_bytes("uni32k"))
    rraw = rb.tobytes()
    lens = np.diff(ro)
    check = list(np.nonzero(lens > 2500)[0]) + list(np.nonzero(lens == 0)[0][:5]) + list(range(0, len(lens), 9001))
    assert len([i for i in check if lens[i] > 2500]) == 2
    for i in check:
        i = int(i)
        assert a[int(ao[i]):int(ao[i + 1])].tolist() == om.encode(rraw[int(ro[i]):int(ro[i + 1])])[0].tolist(), i
    # the next plain batch goes through the fused path again (or its back-off) and is still exact
    a3, ao3 = eng.encode_packed(buf, offs)
    b3, bo3 = ref.encode_packed(buf, offs)
    assert np.array_equal(ao3, bo3) and np.array_equal(a3, b3)
    eng.close()
    ref.close()


def test_bpe_long_words_stay_in_the_lane_kernel(corpus_gen):
    """words of more symbols than the lane kernel's shared arrays hold (URLs, digit runs, unspaced CJK) are merged in
    the same kernel with HBM scratch: nothing is deferred, so the fused path completes, and the ids are exact."""
    rng = np.random.default_rng(11)
    buf, offs = corpus_gen.fill("en", 7003, N)
    extra = [b"see https://example.org/a/very/long/path/with-many-segments_and_underscores?query=1234567890&k=v#frag now",
             b"1234567890" * 30,
             ("\u6771\u4eac\u90fd\u5343\u4ee3\u7530\u533a" * 12).encode("utf-8"),
             b"a" * 25, b"ab" * 13 + b" " + b"z" * 24, b"x" * 500,
             ("caf\u00e9" * 40).encode("utf-8") + b" tail"]
    rb, ro = _ragged(buf, offs, rng, extra * 3)
    eng = _engine("bpe32k")
    a, ao = eng.encode_packed(rb, ro)
    assert eng.info().last_deferred == 0
    ref = _engine("bpe32k", SPM_B200_FUSED=0, SPM_B200_SORT=0)
    ref.set_tuning(32, 0, 0)  # the general BPE kernel (bpe_kernel.cuh) as the reference
    b, bo = ref.encode_packed(rb, ro)
    assert np.array_equal(ao, bo) and np.array_equal(a, b)
    om = oracle_py.OracleModel(model_bytes("bpe32k"))
    rraw = rb.tobytes()
    lens = np.diff(ro)
    raws = [rraw[int(ro[i]):int(ro[i + 1])] for i in range(len(lens))]
    check = [i for i, r in enumerate(raws) if r in extra] + list(range(0, len(lens), 9001))
    assert len(check) >= len(extra) * 3
    for i in check:
        assert a[int(ao[i]):int(ao[i + 1])].tolist() == om.encode(raws[i])[0].tolist(), i
    # the small-batch (device) path takes the same kernel
    sb, so = _ragged(*corpus_gen.fill("en", 7004, 3000), rng, extra)
    c, co = eng.encode_packed(sb, so)
    assert eng.info().last_deferred == 0
    oc, oco = om.encode_batch(sb, so)
    assert np.array_equal(co, oco) and np.array_equal(c, oc)
    eng.close()
    ref.close()


def test_large_batch_rejects_decreasing_offsets(corpus_gen):
    buf, offs = corpus_gen.fill("en", 7003, N)
    bad = offs.copy()
    bad[1000] = bad[1001] + 5  # offsets[1000] > offsets[1001]
    eng = _engine("uni32k")
    with pytest.raises(RuntimeError, match="non-decreasing"):
        eng.encode_packed(buf, bad)
    a, ao = eng.encode_packed(buf, offs)  # the engine is still usable
    assert len(ao) == N + 1 and int(ao[-1]) == len(a)
    # offsets that point far outside the batch's buffer (the fused path launches before the host has validated them):
    # the kernels must not touch those sentences, the call fails with the same error, and the context stays healthy
    wild = offs.copy()
    wild[2000] = np.uint64(10 ** 12)
    wild[2001] = np.uint64(10 ** 12 + 5)
    with pytest.raises(RuntimeError, match="non-decreasing"):
        eng.encode_packed(buf, wild)
    a2, ao2 = eng.encode_packed(buf, offs)
    assert np.array_equal(ao2, ao) and np.array_equal(a2, a)
    eng.close()


@pytest.mark.parametrize("model,kind", [("uni32k", "en"), ("mix_bf8k", "mixed")])
def test_decode_pipelined_equals_plain(model, kind, corpus_gen):
    """spm_decode_ids on >= 300k lists takes the chunked three-stage pipeline (staged H2D of pageable ids, decode,
    D2H of the text); the same lists in two halves take the plain path.  Both must agree, pageable and pinned input
    alike, and match the oracle on a sample."""
    import ctypes
    buf, offs = corpus_gen.fill(kind, 7005, N)
    eng = _engine(model)
    ids, ido = eng.encode_packed(buf, offs)
    text, to = eng.decode_packed(ids, ido)                    # pageable numpy arrays -> staged
    h = N // 3                                                # < 300k lists: plain path
    parts, base = [], 0
    for lo, hi in ((0, h), (h, 2 * h), (2 * h, N)):
        t, o = eng.decode_packed(ids, ido[lo:hi + 1])
        assert int(o[0]) == 0
        assert np.array_equal(o + np.uint64(base), to[lo:hi + 1]), (lo, hi)
        parts.append(t)
        base += int(o[-1])
    assert np.array_equal(np.concatenate(parts), text)
    # pinned input goes straight to the copy engine
    lib = eng._lib
    p_ids = lib.spm_host_alloc(ids.nbytes + 64)
    pin = np.ctypeslib.as_array(ctypes.cast(p_ids, ctypes.POINTER(ctypes.c_int32)), (ids.size,))
    pin[:] = ids
    t2, o2 = eng.decode_packed(pin, ido)
    lib.spm_host_free(p_ids)
    assert np.array_equal(o2, to) and np.array_equal(t2, text)
    om = oracle_py.OracleModel(model_bytes(model))
    k = 3000
    ot, oto = om.decode_batch(ids[: int(ido[k])], ido[: k + 1])
    assert np.array_equal(oto, to[: k + 1]) and np.array_equal(ot, text[: int(to[k])])
    # an id out of range fails the call like the reference (sentencepiece_processor.cc:915-918), also mid-pipeline
    bad = ids.copy()
    bad[int(ido[N - 5])] = 10 ** 8
    with pytest.raises(RuntimeError, match="Invalid id"):
        eng.decode_packed(bad, ido)
    t3, o3 = eng.decode_packed(ids, ido)                      # and the engine is usable afterwards
    assert np.array_equal(o3, to) and np.array_equal(t3, text)
    eng.close()
