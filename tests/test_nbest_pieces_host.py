"""Host side of the n-best and sampled pieces, CPU only: the new calls fail loudly where no device is present, and the
C++ class builds these pieces from the engine alone, with no second encode."""
import os
import re

import numpy as np
import pytest

from conftest import ROOT, model_bytes


def test_fail_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible here; the failure path is for GPU-less boxes")
    from sentencepiece_b200 import Engine, SentencePieceProcessor
    buf, offs = np.frombuffer(b"hello", np.uint8), np.array([0, 5], np.uint64)
    with pytest.raises(RuntimeError, match="no CPU fallback|CUDA"):
        Engine(model_bytes("uni32k")).nbest_encode_pieces(buf, offs, 4)
    with pytest.raises(RuntimeError, match="no CPU fallback|CUDA"):
        Engine(model_bytes("uni32k")).sample_encode_pieces(buf, offs, -1, 0.1)
    with pytest.raises(RuntimeError, match="no CPU fallback|CUDA"):
        Engine(model_bytes("uni32k")).sample_encode_and_score_pieces(buf, offs, 2, 0.1)
    with pytest.raises(RuntimeError, match="no CPU fallback|CUDA"):
        SentencePieceProcessor(model_proto=model_bytes("uni32k")).NBestEncodeAsPieces("hello", 4)
    with pytest.raises(RuntimeError, match="not initialized"):
        SentencePieceProcessor().encode("hello", out_type=str, enable_sampling=True)
    with pytest.raises(RuntimeError, match="not initialized"):
        SentencePieceProcessor().SampleEncodeAndScoreAsPieces("hello", 2, 0.1)


def test_class_sampling_paths_run_no_second_encode():
    src = open(os.path.join(ROOT, "sentencepiece_b200", "csrc", "host", "sentencepiece_processor.cc")).read()
    bodies = re.split(r"\n(?=\S[^\n]*SentencePieceProcessor::)", src)
    sampling = [b for b in bodies if re.search(r"SentencePieceProcessor::(NBestEncode|SampleEncode)", b.split("\n")[0] + b[:400])]
    assert sampling, "no n-best / sampling functions found"
    for b in sampling:
        assert "spm_encode_spans" not in b
    assert "PiecesFromIds" not in src and "RawIds" not in src and "ApplyExtraPieces" not in src
