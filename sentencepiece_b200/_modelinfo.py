"""Piece strings of a serialized ModelProto (sentencepiece_model.proto:293-332) for the Python mirror's piece
output: a minimal wire-format reader (field 1 = repeated SentencePiece {1: piece, 2: score, 3: type})."""


def _varint(b, p):
    v = s = 0
    while True:
        c = b[p]
        p += 1
        v |= (c & 0x7F) << s
        if c < 0x80:
            return v, p
        s += 7


def pieces_and_unk(data):
    pieces, types = pieces_and_types(data)
    return pieces, _unk_id(types)


def _unk_id(types):
    """the last UNKNOWN piece, -1 when there is none"""
    return max((i for i, t in enumerate(types) if t == 2), default=-1)


def pieces_and_types(data):
    """Piece strings and their types (ModelProto.SentencePiece.Type, NORMAL = 1 when absent)."""
    pieces, types, p, n = [], [], 0, len(data)
    while p < n:
        key, p = _varint(data, p)
        fno, wt = key >> 3, key & 7
        if wt == 2:
            ln, p = _varint(data, p)
            if fno == 1:
                q, end, piece, typ = p, p + ln, b"", 1
                while q < end:
                    k2, q = _varint(data, q)
                    f2, w2 = k2 >> 3, k2 & 7
                    if w2 == 2:
                        l2, q = _varint(data, q)
                        if f2 == 1:
                            piece = data[q:q + l2]
                        q += l2
                    elif w2 == 0:
                        v, q = _varint(data, q)
                        if f2 == 3:
                            typ = v
                    elif w2 == 5:
                        q += 4
                    elif w2 == 1:
                        q += 8
                    else:
                        raise ValueError("unsupported wire type in SentencePiece")
                types.append(typ)
                pieces.append(piece.decode("utf-8", errors="replace"))
            p += ln
        elif wt == 0:
            _, p = _varint(data, p)
        elif wt == 5:
            p += 4
        elif wt == 1:
            p += 8
        else:
            raise ValueError("unsupported wire type in ModelProto")
    return pieces, types


def _fields(b, p, end):
    """(field number, wire type, value) of a message: bytes for length-delimited fields, int for varints."""
    while p < end:
        key, p = _varint(b, p)
        fno, wt = key >> 3, key & 7
        if wt == 2:
            ln, p = _varint(b, p)
            yield fno, wt, b[p:p + ln]
            p += ln
        elif wt == 0:
            v, p = _varint(b, p)
            yield fno, wt, v
        elif wt == 5:
            p += 4
        elif wt == 1:
            p += 8
        else:
            raise ValueError("unsupported wire type in ModelProto")


def special_pieces(data):
    """TrainerSpec unk_piece / bos_piece / eos_piece (sentencepiece_model.proto:220-222, field 2 of ModelProto) and
    their ids as the reference's bos_id() / eos_id() see them: PieceToId of the piece (the first definition wins,
    model_interface.cc:51-61), -1 when that is the unknown id (the piece is not defined).  pad_piece (field 48) and
    pad_id as the reference's pad_id() (sentencepiece_processor.cc:1011-1015): PieceToId of the piece when that is a
    CONTROL piece, else -1."""
    names = {45: "<unk>", 46: "<s>", 47: "</s>", 48: "<pad>"}
    for fno, wt, v in _fields(data, 0, len(data)):
        if fno == 2 and wt == 2:
            for f2, w2, v2 in _fields(v, 0, len(v)):
                if f2 in names and w2 == 2:
                    names[f2] = v2.decode("utf-8", errors="replace")
    pieces, types = pieces_and_types(data)
    unk = _unk_id(types)
    first = {}
    for i, p in enumerate(pieces):
        first.setdefault(p, i)

    def piece_id(p):
        i = first.get(p, unk)
        return -1 if i == unk else i

    pad = piece_id(names[48])
    return dict(unk_piece=names[45], bos_piece=names[46], eos_piece=names[47], pad_piece=names[48],
                bos_id=piece_id(names[46]), eos_id=piece_id(names[47]),
                pad_id=pad if pad >= 0 and types[pad] == 3 else -1)  # 3 = CONTROL
