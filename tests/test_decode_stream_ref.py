"""The restatement of spm_decode_stream_device (tests/decode_stream_ref.py) against its own contract: for random
splittings of random id lists on the golden models, the texts of a row's calls concatenate to Decode of the whole
list, no call holds back more than 3 ids, every text decodes as strict UTF-8, and the fast form (token ends of the
whole list) equals the definition (Decode of every prefix).  CPU only."""
import numpy as np
import pytest

from conftest import model_bytes
from decode_stream_ref import StreamRef, random_calls
from oracle import modelproto as mp

MODELS = ["uni32k", "mix_bf8k", "bpe32k", "botchan8k", "mix_bpe4k"]


def _random_lists(m, rng, n, maxlen):
    """ids with many control / unknown / byte pieces: byte runs are often broken UTF-8"""
    vocab = len(m["pieces"])
    special = np.nonzero(np.asarray(m["types"]) != mp.NORMAL)[0]
    out = []
    for _ in range(n):
        a = rng.integers(0, vocab, size=int(rng.integers(0, maxlen)))
        msk = rng.random(len(a)) < 0.5
        if len(special) and msk.any():
            a[msk] = rng.choice(special, size=int(msk.sum()))
        out.append(a.astype(np.int32))
    return out


@pytest.mark.parametrize("model", MODELS)
def test_random_splits(model):
    rng = np.random.default_rng(77)
    mb = model_bytes(model)
    for variant in (mb, mp.replace_flags(mb, remove_extra_whitespaces=False),
                    mp.replace_flags(mb, add_dummy_prefix=False, remove_extra_whitespaces=False)):
        ref = StreamRef(variant)
        m = mp.parse_model(variant)
        for ids in _random_lists(m, rng, 60, 40) + [np.zeros(0, np.int32)]:
            text, _, _ = ref.spans.decode_spans_batch(ids, np.array([0, len(ids)], np.uint64))
            calls = random_calls(rng, len(ids))
            d = ref.deltas(ids, calls)
            assert d == ref.deltas_by_prefix(ids, calls)
            assert b"".join(d) == text.tobytes()
            for x in d:
                x.decode("utf-8")
            pos = 0
            for k in calls:
                pos += k
                assert ref.held(ids[:pos]) <= 3


def test_byte_fallback_known_answers():
    U, C, N, B = mp.UNKNOWN, mp.CONTROL, mp.NORMAL, mp.BYTE
    bp = [("<unk>", 0.0, U), ("<s>", 0.0, C), ("</s>", 0.0, C), ("A", 0.0, N), ("B", 0.0, N), ("C", 0.0, N)]
    bp += [("<0x%02X>" % i, 0.0, B) for i in range(256)]
    ref = StreamRef(mp.build_model(bp, byte_fallback=True))
    b = lambda x: 6 + x  # noqa: E731
    ids = [1, 3, 4, b(0xE3), b(0x81), b(0x82), b(0x5A), b(0xCE), b(0xA9), 5, b(0xE0), b(0x80), b(0xE3), b(0x81),
           b(0x84), b(0xEF), b(0xBF), b(0xBD)]
    want = ["", "A", "B", "", "", "あ", "Z", "", "Ω", "C", "", "", "��", "", "い", "", "", "�"]
    assert [x.decode() for x in ref.deltas(ids, [1] * len(ids))] == want
    assert [x.decode() for x in ref.deltas([b(0xE3), b(0x81)], [1, 1, 0])] == ["", "", "��"]
    assert [x.decode() for x in ref.deltas([b(0xE3), b(0x81), 3], [1, 1, 1])] == ["", "", "��A"]
