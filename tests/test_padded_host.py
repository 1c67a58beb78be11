"""Host side of the padded tensors, CPU only: the pad id that encode_padded uses by default is the reference's pad_id()
(sentencepiece_processor.cc:1011-1015: PieceToId(trainer_spec.pad_piece), kept only when that piece is CONTROL), for
every golden model and for models whose pad piece is a CONTROL piece, another type, renamed or missing."""
import pytest

from conftest import model_bytes
from oracle import modelproto

GOLDEN = ["uni32k", "bpe32k", "mix_bf8k", "mix_bpe4k", "botchan8k"]


def reference_pad_id(data, pad_piece="<pad>"):
    """pad_id() restated on the oracle's parse of the model: the first piece spelled pad_piece, if it is CONTROL"""
    m = modelproto.parse_model(data)
    for i, p in enumerate(m["pieces"]):
        if p == pad_piece.encode():
            return i if m["types"][i] == modelproto.CONTROL else -1
    return -1


def _toy(pad_type=None, pad_piece=None):
    C, N = modelproto.CONTROL, modelproto.NORMAL
    pieces = [("<unk>", 0.0, modelproto.UNKNOWN), ("<s>", 0.0, C), ("</s>", 0.0, C), ("a", -1.0, N), ("b", -2.0, N)]
    if pad_type is not None:
        pieces.append((pad_piece or "<pad>", 0.0, pad_type))
    data = modelproto.build_model(pieces)
    if pad_piece:  # a second TrainerSpec message: its fields merge into the first (field 48 = pad_piece)
        data += modelproto._ld(2, modelproto._ld(48, pad_piece.encode()))
    return data


@pytest.mark.parametrize("model", GOLDEN)
def test_golden_models(model):
    from sentencepiece_b200 import _modelinfo
    sp = _modelinfo.special_pieces(model_bytes(model))
    assert sp["pad_piece"] == "<pad>"
    assert sp["pad_id"] == reference_pad_id(model_bytes(model))


@pytest.mark.parametrize("pad_type,pad_piece,want", [
    (modelproto.CONTROL, None, 5),        # <pad> defined as a control piece
    (modelproto.USER_DEFINED, None, -1),  # defined, but not CONTROL: pad_id() is -1
    (modelproto.NORMAL, None, -1),
    (None, None, -1),                     # not defined: PieceToId gives the unknown id
    (modelproto.CONTROL, "[PAD]", 5),     # trainer_spec.pad_piece renamed
])
def test_toy_models(pad_type, pad_piece, want):
    from sentencepiece_b200 import _modelinfo
    data = _toy(pad_type, pad_piece)
    sp = _modelinfo.special_pieces(data)
    assert sp["pad_id"] == want == reference_pad_id(data, pad_piece or "<pad>")
    assert sp["bos_id"] == 1 and sp["eos_id"] == 2
