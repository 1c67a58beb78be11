"""Host side of Normalize, CPU only: the vectorised ConvertToUnicodeAlignment on hand-made cases and on the
reference's own expectations, the empty-input rule, and the call failing loudly where no device is present."""
import numpy as np
import pytest

from conftest import model_bytes
from sentencepiece_b200 import _capi
from sentencepiece_b200.processor import char_index, pack_sentences, unicode_alignment

EMPTY = _capi.NORM_TO_ORIG_EMPTY


def align(pairs):
    """[(orig bytes, normalized bytes, byte norm_to_orig)] -> character norm_to_orig per pair, as the batch helper
    computes them from spm_normalize's layout"""
    buf, offs = pack_sentences([o for o, _, _ in pairs])
    nbuf, noffs = pack_sentences([t for _, t, _ in pairs])
    n2o = np.concatenate([np.asarray(m if m else [EMPTY], np.int64) for _, _, m in pairs])
    uo, uv = unicode_alignment(buf, offs, nbuf, noffs, n2o)
    return [uv[int(uo[i]):int(uo[i + 1])].tolist() for i in range(len(pairs))]


def test_reference_expectations():
    """sentencepiece_trainer_test.cc:379-393: the byte offsets of "ＫＡＤＯＫＡＷＡ   ABC " and their conversion"""
    orig = "ＫＡＤＯＫＡＷＡ   ABC ".encode()
    norm = "▁KADOKAWA▁ABC".encode()
    n2o = [0, 0, 0, 0, 3, 6, 9, 12, 15, 18, 21, 24, 24, 24, 27, 28, 29, 30]
    assert align([(orig, norm, n2o)]) == [[0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 11, 12, 13, 14]]


def test_hand_made():
    cases = [
        (b"abc", b"abc", [0, 1, 2, 3], [0, 1, 2, 3]),
        ("日本".encode(), "日本".encode(), [0, 0, 0, 3, 3, 3, 6], [0, 1, 2]),
        ("é".encode(), b"e\xcc\x81", [0, 0, 0, 2], [0, 0, 1]),         # one input character, two normalized
        (b"\xff", "�".encode(), [0, 0, 0, 1], [0, 1]),           # a malformed byte is one character
        (b"x \xe3A", b"x\xe2\x96\x81\xe3\x81\x82", [0, 1, 1, 1, 2, 2, 2, 4], [0, 1, 2, 3]),
        (b"", b"", [], [0]),                                          # empty input: [0] after the conversion
        (b"   ", b"", [], [0]),
        (b"x", b"", [1], [1]),                                        # normalizes to nothing: {consumed}
    ]
    assert align([(o, t, m) for o, t, m, _ in cases]) == [w for *_, w in cases]


def test_char_index_malformed():
    sents = [b"", b"\xe3A", b"\x80\x80x", b"abc\xf0", "aé".encode(), b"\xc3"]
    buf, offs = pack_sentences(sents)
    assert char_index(buf, offs).tolist() == [0, 0, 0, 1, 0, 1, 2, 3, 0, 1, 2, 3, 4, 0, 1, 1, 2, 0, 1]


def test_fail_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible here; the failure path is for GPU-less boxes")
    from sentencepiece_b200 import Engine, SentencePieceProcessor
    buf, offs = np.frombuffer(b"hello", np.uint8), np.array([0, 5], np.uint64)
    with pytest.raises(RuntimeError, match="no CPU fallback|CUDA"):
        Engine(model_bytes("uni32k")).normalize(buf, offs, with_offsets=True)
    with pytest.raises(RuntimeError, match="no CPU fallback|CUDA"):
        SentencePieceProcessor(model_proto=model_bytes("uni32k")).Normalize("hello")
    with pytest.raises(RuntimeError, match="not initialized"):
        SentencePieceProcessor().Normalize("hello", with_offsets=True)
