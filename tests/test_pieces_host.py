"""Host side of spm_encode_pieces, CPU only: the Python list builder over packed output, and a loud failure where no
device is present."""
import numpy as np
import pytest

from conftest import model_bytes


def test_split_pieces():
    from sentencepiece_b200.processor import split_pieces
    rows = [["▁he", "llo", "▁", "世界"], [], ["<s>", "a\x00b", ""], ["x"]]
    blobs = [b"".join(p.encode() for p in r) for r in rows]
    text = np.frombuffer(b"".join(blobs), dtype=np.uint8)
    to = np.concatenate([[0], np.cumsum([len(b) for b in blobs])]).astype(np.uint64)
    ido = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.uint64)
    ends = np.array([e for r in rows for e in np.cumsum([len(p.encode()) for p in r]).tolist()], dtype=np.uint32)
    assert split_pieces(text, to, ends, ido) == rows
    assert split_pieces(np.zeros(0, np.uint8), np.zeros(1, np.uint64), np.zeros(0, np.uint32), np.zeros(1, np.uint64)) == []


def test_pieces_fail_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible here; the failure path is for GPU-less boxes")
    from sentencepiece_b200 import Engine, SentencePieceProcessor
    with pytest.raises(RuntimeError, match="no CPU fallback|CUDA"):
        Engine(model_bytes("uni32k")).encode_pieces(np.zeros(1, np.uint8), np.array([0, 1], np.uint64))
    with pytest.raises(RuntimeError, match="no CPU fallback|CUDA"):
        SentencePieceProcessor(model_proto=model_bytes("uni32k")).EncodeAsPieces("hello")
    with pytest.raises(RuntimeError, match="not initialized"):
        SentencePieceProcessor().encode("hello", out_type=str)
