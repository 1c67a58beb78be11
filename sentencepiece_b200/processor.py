"""Host-side mirror of the reference interface for the batched-encode path."""
import ctypes

import numpy as np

from . import _capi


# SetEncodeExtraOptions names (sentencepiece_processor.cc:1077-1082)
_EXTRA_OPTIONS = {"bos": "bos", "eos": "eos", "reverse": "reverse", "unk": "unk", "unk_piece": "unk"}


def extra_frame(options, bos_id, eos_id):
    """The id effect of ApplyExtraOptions (sentencepiece_processor.cc:1019-1064) for options applied in order, in the
    canonical form the engine writes: (prefix, reverse, suffix), ids -> prefix ++ (ids or reversed ids) ++ suffix."""
    prefix, suffix, rev = [], [], False
    for o in options:
        if o == "reverse":
            prefix, suffix, rev = suffix[::-1], prefix[::-1], not rev
        elif o == "bos":
            prefix.insert(0, bos_id)
        elif o == "eos":
            suffix.append(eos_id)
    return prefix, rev, suffix


def split_pieces(text, text_offsets, piece_end, id_offsets):
    """The packed output of spm_encode_pieces (sep = -1) as one list of piece strings per sentence: piece k of sentence i is
    text[text_offsets[i] + (piece_end[id_offsets[i] + k - 1] or 0) : text_offsets[i] + piece_end[id_offsets[i] + k]]."""
    raw = bytes(np.ascontiguousarray(text, dtype=np.uint8))
    to = np.asarray(text_offsets, dtype=np.uint64).tolist()
    ido = np.asarray(id_offsets, dtype=np.uint64).tolist()
    ends = np.asarray(piece_end, dtype=np.uint32).tolist()
    out = []
    for i in range(len(to) - 1):
        s = raw[to[i]:to[i + 1]]
        row, begin = [], 0
        for end in ends[ido[i]:ido[i + 1]]:
            row.append(s[begin:end].decode("utf-8", errors="replace"))
            begin = end
        out.append(row)
    return out


def _one_char_len(b):
    """string_util::OneCharLen (util.h:151-153) of every byte of a uint8 array"""
    return np.array([1] * 12 + [2, 2, 3, 4], np.int64)[b >> 4]


def char_index(buf, offs):
    """The utf8_to_unicode_offsets table of ConvertToUnicodeAlignment (sentencepiece_trainer.cc:369-388) for every
    sentence of a packed batch, in the n2o layout: entry offs[i] - offs[0] + i + p is the index of the character that
    holds byte p of sentence i (p = its length: the number of characters).  Characters are stepped by their lead byte's
    OneCharLen; a step past the end of a malformed sentence, which the reference does not guard, stops at the end."""
    buf = np.asarray(buf, np.uint8)
    offs = np.asarray(offs, np.int64) - int(offs[0])
    n = len(offs) - 1
    lens = np.diff(offs)
    # every byte that is not a trail byte starts a character, and so does the first byte of a sentence; that is the
    # chain of OneCharLen steps wherever each step lands on the next such byte (always, for valid UTF-8)
    start = (buf & 0xC0) != 0x80
    start[offs[:-1][lens > 0]] = True
    sid = np.repeat(np.arange(n), lens)
    pos = np.flatnonzero(start)
    nxt = np.append(pos[1:], len(buf))
    ends = offs[1:][sid[pos]]
    nxt = np.minimum(nxt, ends)
    good = np.ones(n, bool)
    step = np.minimum(pos + _one_char_len(buf[pos]), ends)
    good[sid[pos[step != nxt]]] = False
    for i in np.flatnonzero(~good):  # malformed sentences only: follow the steps
        s = np.zeros(lens[i], bool)
        p, lead = 0, _one_char_len(buf[offs[i]:offs[i + 1]])
        while p < lens[i]:
            s[p] = True
            p += int(lead[p])
        start[offs[i]:offs[i + 1]] = s
    # one more slot per sentence (its end), counted as a start: the running count minus one is the character index
    ext = np.insert(start.astype(np.int64), offs[1:], 1)
    csum = np.cumsum(ext)
    first = offs[:-1] + np.arange(n)
    before = np.where(first > 0, csum[np.maximum(first - 1, 0)], 0)
    return csum - np.repeat(before, lens + 1) - 1


def unicode_alignment(orig, orig_offs, norm, norm_offs, n2o):
    """ConvertToUnicodeAlignment (sentencepiece_trainer.cc:369-397) of spm_normalize's byte offsets, for a whole batch
    -> (uint64 offsets[n+1], int64 values): sentence i's character offsets are values[offsets[i]:offsets[i+1]], one
    per normalized character and one for the end.  Where the byte offsets are empty (n2o entry NORM_TO_ORIG_EMPTY) the
    reference's table of one zero is left as it is: [0]."""
    n = len(norm_offs) - 1
    norm_offs = np.asarray(norm_offs, np.int64)
    n2o = np.asarray(n2o, np.int64)
    ni = char_index(norm, norm_offs)
    oi = char_index(orig, orig_offs)
    sent = np.repeat(np.arange(n), np.diff(norm_offs) + 1)
    last = np.zeros(len(ni), bool)  # the last byte of each normalized character wins, and every sentence's end
    last[:-1] = ni[:-1] != ni[1:]
    last[norm_offs[1:] - norm_offs[0] + np.arange(n)] = True
    sel = np.flatnonzero(last)
    empty = n2o[sel] == _capi.NORM_TO_ORIG_EMPTY
    orig_base = np.asarray(orig_offs, np.int64)[:-1] - int(orig_offs[0]) + np.arange(n)
    values = np.where(empty, 0, oi[np.where(empty, 0, orig_base[sent[sel]] + n2o[sel])])
    offsets = np.zeros(n + 1, np.uint64)
    offsets[1:] = np.cumsum(np.bincount(sent[sel], minlength=n))
    return offsets, values


def unicode_spans(buf, offs, begin, end, id_offsets):
    """ConvertToUnicodeSpans (sentencepiece_processor.cc:63-91) of spm_encode_offsets' byte offsets, for a whole batch ->
    (begin, end) int64 character indices.  Each offset is clipped to [0, len(input)] and mapped through char_index; an
    empty input keeps its offsets, which are all 0, as the reference does.  A malformed input whose last character's
    lead byte claims more bytes than remain ends at its length instead of reading past it."""
    offs = np.asarray(offs, np.int64)
    n = len(offs) - 1
    ci = char_index(buf, offs)
    sent = np.repeat(np.arange(n), np.diff(np.asarray(id_offsets, np.int64)))
    lens = np.diff(offs)[sent]
    base = (offs[:-1] - offs[0] + np.arange(n))[sent]

    def conv(x):
        return ci[base + np.minimum(np.asarray(x, np.int64), lens)]
    return conv(begin), conv(end)


class ImmutableSentencePiece:
    """One token of an ImmutableSentencePieceText: piece, id, surface (input[begin:end]), begin, end (read-only)."""
    __slots__ = ("_piece", "_id", "_surface", "_begin", "_end")

    def __init__(self, piece, id, surface, begin, end):
        self._piece, self._id, self._surface, self._begin, self._end = piece, id, surface, begin, end

    piece_as_bytes = property(lambda self: self._piece)
    piece = property(lambda self: self._piece.decode("utf-8", errors="replace"))
    surface_as_bytes = property(lambda self: self._surface)
    surface = property(lambda self: self._surface.decode("utf-8", errors="replace"))
    id = property(lambda self: self._id)
    begin = property(lambda self: self._begin)
    end = property(lambda self: self._end)

    def __eq__(self, other):
        if not isinstance(other, ImmutableSentencePiece):
            return NotImplemented
        return (self.piece, self.id, self.surface, self.begin, self.end) == \
            (other.piece, other.id, other.surface, other.begin, other.end)

    def __hash__(self):
        return hash((self._piece, self._id, self._surface, self._begin, self._end))

    def __repr__(self):
        return f'piece: "{self.piece}"\nid: {self.id}\nsurface: "{self.surface}"\nbegin: {self.begin}\nend: {self.end}\n'


class ImmutableSentencePieceText:
    """EncodeAsImmutableProto's result for one input: text, pieces (a tuple of ImmutableSentencePiece); len(),
    indexing and iteration go over the pieces (read-only)."""
    __slots__ = ("_text", "_pieces")

    def __init__(self, text, pieces):
        self._text, self._pieces = text, tuple(pieces)

    text_as_bytes = property(lambda self: self._text)
    text = property(lambda self: self._text.decode("utf-8", errors="replace"))
    pieces = property(lambda self: self._pieces)

    def __len__(self):
        return len(self._pieces)

    def __getitem__(self, k):
        return self._pieces[k]

    def __iter__(self):
        return iter(self._pieces)

    def __eq__(self, other):
        if not isinstance(other, ImmutableSentencePieceText):
            return NotImplemented
        return self.text_as_bytes == other.text_as_bytes and self.pieces == other.pieces

    def __hash__(self):
        return hash((self._text, self._pieces))

    def __repr__(self):
        return "".join(f"pieces {{\n{p!r}}}\n" for p in self._pieces) + f'text: "{self.text}"\n'


def immutable_protos(items, buf, offs, r):
    """The ImmutableSentencePieceText of every input from spm_encode_offsets' result r (with pieces): offsets in
    characters (unicode_spans), surfaces cut from the input by byte offsets."""
    raw = bytes(np.ascontiguousarray(buf, np.uint8))
    text = bytes(r["text"])
    ob = np.asarray(offs, np.int64) - int(offs[0])
    ido, to = r["id_offsets"].tolist(), r["text_offsets"].tolist()
    cb, ce = unicode_spans(buf, offs, r["begin"], r["end"], r["id_offsets"])
    ids, pe, bb, be = r["ids"].tolist(), r["piece_end"].tolist(), r["begin"].tolist(), r["end"].tolist()
    cb, ce = cb.tolist(), ce.tolist()
    out = []
    for i in range(len(items)):
        s = raw[ob[i]:ob[i + 1]]
        t = text[to[i]:to[i + 1]]
        pieces, prev = [], 0
        for k in range(ido[i], ido[i + 1]):
            pieces.append(ImmutableSentencePiece(t[prev:pe[k]], ids[k], s[bb[k]:be[k]], cb[k], ce[k]))
            prev = pe[k]
        out.append(ImmutableSentencePieceText(s, pieces))
    return out


def decode_protos(pieces, ids, id_offsets, text, text_offsets, tok_end):
    """The ImmutableSentencePieceText of every list from spm_decode_offsets' result: .text is the decoded text, piece
    is pieces[id], surface is text[begin:end], begin / end in characters of the text (unicode_spans)."""
    raw = bytes(np.ascontiguousarray(text, np.uint8))
    ido = np.asarray(id_offsets, np.int64)
    ido = ido - ido[0]
    te = np.asarray(tok_end, np.int64)
    tb = te.copy()  # each token begins where the one before it in its list ends, the first one at 0
    if len(tb):
        tb[1:] = te[:-1]
        tb[ido[:-1][ido[:-1] < ido[1:]]] = 0
    cb, ce = unicode_spans(text, text_offsets, tb, te, ido)
    to, ido = np.asarray(text_offsets, np.int64).tolist(), ido.tolist()
    ids, tb, te, cb, ce = np.asarray(ids).tolist(), tb.tolist(), te.tolist(), cb.tolist(), ce.tolist()
    out = []
    for i in range(len(to) - 1):
        t = raw[to[i]:to[i + 1]]
        out.append(ImmutableSentencePieceText(t, [ImmutableSentencePiece(pieces[ids[k]], ids[k], t[tb[k]:te[k]], cb[k], ce[k])
                                                  for k in range(ido[i], ido[i + 1])]))
    return out


def pack_sentences(sentences):
    """list[bytes|str] -> (uint8[total], uint64[n+1])"""
    bs = [s.encode("utf-8") if isinstance(s, str) else bytes(s) for s in sentences]
    offs = np.zeros(len(bs) + 1, dtype=np.uint64)
    if bs:
        offs[1:] = np.cumsum([len(b) for b in bs], dtype=np.uint64)
    buf = np.frombuffer(b"".join(bs), dtype=np.uint8) if bs else np.zeros(0, np.uint8)
    return buf, offs


class Engine:
    """One engine = one model on one GPU (spm_engine in include/spm_b200.h)."""

    def __init__(self, model_bytes, device=0):
        self._lib = _capi.load()
        h = ctypes.c_void_p()
        rc = self._lib.spm_engine_create_from_serialized(model_bytes, len(model_bytes), device, ctypes.byref(h))
        if rc:
            raise RuntimeError(f"spm_engine_create failed ({rc}): {self._lib.spm_last_error(None).decode()}")
        self._h = h
        self.device = device
        self._model_bytes = model_bytes
        self._pad_guess = 64  # cells per row encode_device_padded(width=0) allocates first: the last such call's width
        self._win_ratio = 1.0  # rows per sentence encode_device_windows allocates first: the last call's R / n
        self._pair_guess = (1.0, 64)  # encode_device_pairs' first allocation: the last call's R / n and width
        self._pad = None  # pad_id(), read from the model on first use

    def close(self):
        if getattr(self, "_h", None):
            self._lib.spm_engine_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc:
            raise RuntimeError(f"spm_b200 error {rc}: {self._lib.spm_last_error(self._h).decode()}")

    def info(self):
        i = _capi.EngineInfo()
        self._check(self._lib.spm_engine_get_info(self._h, ctypes.byref(i)))
        return i

    def set_tuning(self, lanes=0, cap=0, ctas=0):
        self._check(self._lib.spm_engine_set_tuning(self._h, lanes, cap, ctas))

    def set_types(self, types):
        t = np.ascontiguousarray(types, dtype=np.uint8)
        self._check(self._lib.spm_engine_set_types(self._h, t.ctypes.data))

    def cache_reset(self):
        """empties the engine's memo tables (the BPE word cache); results never depend on them"""
        self._check(self._lib.spm_engine_cache_reset(self._h))

    def set_encode_frame(self, prefix=(), reverse=False, suffix=()):
        """spm_engine_set_encode_frame: every later id result is prefix ++ (ids, reversed when `reverse`) ++ suffix;
        no arguments restore the plain output."""
        p = np.ascontiguousarray(prefix, dtype=np.int32)
        q = np.ascontiguousarray(suffix, dtype=np.int32)
        self._check(self._lib.spm_engine_set_encode_frame(self._h, p.ctypes.data if len(p) else None, len(p), int(bool(reverse)),
                                                          q.ctypes.data if len(q) else None, len(q)))

    def encode_packed(self, buf, offs, copy=True):
        """Batch encode of a packed host buffer -> (ids int32[], id_offsets uint64[n+1])."""
        n = len(offs) - 1
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        ids = ctypes.c_void_p()
        ido = ctypes.c_void_p()
        self._check(self._lib.spm_encode_ids(self._h, buf.ctypes.data, offs.ctypes.data, n, ctypes.byref(ids),
                                             ctypes.byref(ido)))
        o = np.ctypeslib.as_array(ctypes.cast(ido, ctypes.POINTER(ctypes.c_uint64)), (n + 1,))
        tot = int(o[n])
        a = np.ctypeslib.as_array(ctypes.cast(ids, ctypes.POINTER(ctypes.c_int32)), (max(tot, 1),))[:tot]
        return (a.copy(), o.copy()) if copy else (a, o)

    def encode_packed_ptr(self, bytes_ptr, offs_ptr, n):
        """Raw-pointer variant for benchmarks (pinned host memory): returns total ids."""
        ids = ctypes.c_void_p()
        ido = ctypes.c_void_p()
        self._check(self._lib.spm_encode_ids(self._h, bytes_ptr, offs_ptr, n, ctypes.byref(ids), ctypes.byref(ido)))
        o = np.ctypeslib.as_array(ctypes.cast(ido, ctypes.POINTER(ctypes.c_uint64)), (n + 1,))
        return int(o[n]), ids.value, ido.value

    def encode_spans(self, buf, offs):
        """-> dict(ids, tok_end, id_offsets, normalized(bytes), norm_offsets, n2o)"""
        n = len(offs) - 1
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        p = [ctypes.c_void_p() for _ in range(6)]
        self._check(self._lib.spm_encode_spans(self._h, buf.ctypes.data, offs.ctypes.data, n, *[ctypes.byref(x) for x in p]))
        ido = np.ctypeslib.as_array(ctypes.cast(p[2], ctypes.POINTER(ctypes.c_uint64)), (n + 1,)).copy()
        tot = int(ido[n])
        no = np.ctypeslib.as_array(ctypes.cast(p[4], ctypes.POINTER(ctypes.c_uint64)), (n + 1,)).copy()
        tn = int(no[n])
        ids = np.ctypeslib.as_array(ctypes.cast(p[0], ctypes.POINTER(ctypes.c_int32)), (max(tot, 1),))[:tot].copy()
        te = np.ctypeslib.as_array(ctypes.cast(p[1], ctypes.POINTER(ctypes.c_uint32)), (max(tot, 1),))[:tot].copy()
        norm = ctypes.string_at(p[3], tn) if tn else b""
        n2o = np.ctypeslib.as_array(ctypes.cast(p[5], ctypes.POINTER(ctypes.c_uint32)), (tn + n,)).copy()
        return dict(ids=ids, tok_end=te, id_offsets=ido, normalized=norm, norm_offsets=no, n2o=n2o)

    def normalize(self, buf, offs, with_offsets=False):
        """spm_normalize: the model's normalizer over a packed batch -> (normalized uint8[], norm_offsets uint64[n+1],
        n2o uint32[] or None).  With offsets, sentence i's norm_to_orig is n2o[norm_offsets[i] + i : norm_offsets[i+1] +
        i + 1], the one entry _capi.NORM_TO_ORIG_EMPTY where the reference's is empty."""
        n = len(offs) - 1
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        p = [ctypes.c_void_p() for _ in range(3)]
        self._check(self._lib.spm_normalize(self._h, buf.ctypes.data, offs.ctypes.data, n, int(bool(with_offsets)),
                                            *[ctypes.byref(x) for x in p]))
        no = np.ctypeslib.as_array(ctypes.cast(p[1], ctypes.POINTER(ctypes.c_uint64)), (n + 1,)).copy()
        tn = int(no[n])
        text = np.ctypeslib.as_array(ctypes.cast(p[0], ctypes.POINTER(ctypes.c_uint8)), (max(tn, 1),))[:tn].copy()
        if not with_offsets:
            return text, no, None
        n2o = np.ctypeslib.as_array(ctypes.cast(p[2], ctypes.POINTER(ctypes.c_uint32)), (max(tn + n, 1),))[:tn + n].copy()
        return text, no, n2o

    def encode_pieces(self, buf, offs, unk_piece=None, sep=-1):
        """spm_encode_pieces: EncodeAsPieces over a packed batch, the encode frame applied ->
        dict(text uint8[], text_offsets uint64[n+1], piece_end uint32[], ids int32[], id_offsets uint64[n+1]).
        unk_piece (str | bytes | None) replaces the piece of every unknown token; sep = -1 or the byte written between
        consecutive pieces of a sentence."""
        n = len(offs) - 1
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        p = [ctypes.c_void_p() for _ in range(5)]
        self._check(self._lib.spm_encode_pieces(self._h, buf.ctypes.data, offs.ctypes.data, n, *self._unk(unk_piece), sep,
                                                *[ctypes.byref(x) for x in p]))
        return self._pieces_result(p, n)

    def encode_offsets(self, buf, offs, eos_id=-1, unk_piece=None, sep=-1, pieces=True):
        """spm_encode_offsets: the ids of every token and its byte range in the input, the encode frame applied ->
        dict(ids int32[], id_offsets uint64[n+1], begin uint32[], end uint32[]), begin / end relative to the sentence's
        start; frame entries equal to eos_id get (len, len), the others (0, 0).  pieces: also text, text_offsets and
        piece_end, exactly as encode_pieces with the same unk_piece and sep."""
        n = len(offs) - 1
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        p = [ctypes.c_void_p() for _ in range(7)]
        self._check(self._lib.spm_encode_offsets(self._h, buf.ctypes.data, offs.ctypes.data, n, eos_id, *self._unk(unk_piece),
                                                 sep, *[ctypes.byref(x) for x in p[:4]],
                                                 *([ctypes.byref(x) for x in p[4:]] if pieces else [None] * 3)))
        ido = np.ctypeslib.as_array(ctypes.cast(p[1], ctypes.POINTER(ctypes.c_uint64)), (n + 1,)).copy()
        tot = int(ido[n])

        def arr(ptr, ct):
            return np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ct)), (max(tot, 1),))[:tot].copy()
        r = dict(ids=arr(p[0], ctypes.c_int32), id_offsets=ido, begin=arr(p[2], ctypes.c_uint32),
                 end=arr(p[3], ctypes.c_uint32))
        if pieces:
            to = np.ctypeslib.as_array(ctypes.cast(p[5], ctypes.POINTER(ctypes.c_uint64)), (n + 1,)).copy()
            tt = int(to[n])
            r["text"] = np.ctypeslib.as_array(ctypes.cast(p[4], ctypes.POINTER(ctypes.c_uint8)), (max(tt, 1),))[:tt].copy()
            r["text_offsets"] = to
            r["piece_end"] = arr(p[6], ctypes.c_uint32)
        return r

    @staticmethod
    def _pieces_result(p, lists):
        """text, text_offsets, piece_end, ids and the id offsets of `lists` packed piece lists (pointers p[0..4])"""
        to = np.ctypeslib.as_array(ctypes.cast(p[1], ctypes.POINTER(ctypes.c_uint64)), (lists + 1,)).copy()
        ido = np.ctypeslib.as_array(ctypes.cast(p[4], ctypes.POINTER(ctypes.c_uint64)), (lists + 1,)).copy()
        tt, tot = int(to[lists]), int(ido[lists])
        # (not ctypes.string_at: its size is a C int, and n-best text passes 2 GB at config 5's sizes)
        text = np.ctypeslib.as_array(ctypes.cast(p[0], ctypes.POINTER(ctypes.c_uint8)), (max(tt, 1),))[:tt].copy()
        pe = np.ctypeslib.as_array(ctypes.cast(p[2], ctypes.POINTER(ctypes.c_uint32)), (max(tot, 1),))[:tot].copy()
        ids = np.ctypeslib.as_array(ctypes.cast(p[3], ctypes.POINTER(ctypes.c_int32)), (max(tot, 1),))[:tot].copy()
        return dict(text=text, text_offsets=to, piece_end=pe, ids=ids, id_offsets=ido)

    @staticmethod
    def _unk(unk_piece):
        if isinstance(unk_piece, str):
            unk_piece = unk_piece.encode("utf-8")
        return unk_piece, len(unk_piece) if unk_piece is not None else 0

    def nbest_encode_pieces(self, buf, offs, nbest_size, unk_piece=None, sep=-1):
        """spm_nbest_encode_pieces: NBestEncodeAsPieces over a packed batch -> dict(text, text_offsets uint64[n*K+1],
        piece_end, ids, cand_offsets uint64[n*K+1], scores float32[n*K], n_cands uint32[n], K); candidate c of sentence
        i is list i*K + c, laid out as encode_pieces lays out a sentence."""
        n = len(offs) - 1
        K = max(1, min(nbest_size, 1024))
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        p = [ctypes.c_void_p() for _ in range(7)]
        self._check(self._lib.spm_nbest_encode_pieces(self._h, buf.ctypes.data, offs.ctypes.data, n, nbest_size,
                                                      *self._unk(unk_piece), sep, *[ctypes.byref(x) for x in p]))
        nc = n * K
        r = self._pieces_result(p[:5], nc)
        r["cand_offsets"] = r.pop("id_offsets")
        r["scores"] = np.ctypeslib.as_array(ctypes.cast(p[5], ctypes.POINTER(ctypes.c_float)), (max(nc, 1),))[:nc].copy()
        r["n_cands"] = np.ctypeslib.as_array(ctypes.cast(p[6], ctypes.POINTER(ctypes.c_uint32)), (max(n, 1),))[:n].copy()
        r["K"] = K
        return r

    def sample_encode_pieces(self, buf, offs, nbest_size, alpha, unk_piece=None, sep=-1):
        """spm_sample_encode_pieces: SampleEncodeAsPieces over a packed batch -> the dict of encode_pieces"""
        n = len(offs) - 1
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        p = [ctypes.c_void_p() for _ in range(5)]
        self._check(self._lib.spm_sample_encode_pieces(self._h, buf.ctypes.data, offs.ctypes.data, n, nbest_size, alpha,
                                                       *self._unk(unk_piece), sep, *[ctypes.byref(x) for x in p]))
        return self._pieces_result(p, n)

    def sample_encode_and_score_pieces(self, buf, offs, num_samples, alpha, wor=False, include_best=False,
                                       unk_piece=None, sep=-1):
        """spm_sample_encode_and_score_pieces -> dict(text, text_offsets, piece_end, ids, cand_offsets, scores) over
        n*num_samples lists, sample c of sentence i being list i*num_samples + c"""
        n = len(offs) - 1
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        p = [ctypes.c_void_p() for _ in range(6)]
        self._check(self._lib.spm_sample_encode_and_score_pieces(self._h, buf.ctypes.data, offs.ctypes.data, n, num_samples,
                                                                 alpha, int(wor), int(include_best), *self._unk(unk_piece),
                                                                 sep, *[ctypes.byref(x) for x in p]))
        nc = n * num_samples
        r = self._pieces_result(p[:5], nc)
        r["cand_offsets"] = r.pop("id_offsets")
        r["scores"] = np.ctypeslib.as_array(ctypes.cast(p[5], ctypes.POINTER(ctypes.c_float)), (max(nc, 1),))[:nc].copy()
        return r

    def decode_packed(self, ids, id_offsets):
        """Batch Decode of packed id lists -> (text uint8[], text_offsets uint64[n+1])."""
        n = len(id_offsets) - 1
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        ido = np.ascontiguousarray(id_offsets, dtype=np.uint64)
        text = ctypes.c_void_p()
        to = ctypes.c_void_p()
        self._check(self._lib.spm_decode_ids(self._h, ids.ctypes.data, ido.ctypes.data, n, ctypes.byref(text), ctypes.byref(to)))
        o = np.ctypeslib.as_array(ctypes.cast(to, ctypes.POINTER(ctypes.c_uint64)), (n + 1,)).copy()
        tot = int(o[n])
        t = np.frombuffer(ctypes.string_at(text, tot), dtype=np.uint8) if tot else np.zeros(0, np.uint8)
        return t, o

    def decode_offsets(self, ids, id_offsets):
        """spm_decode_offsets: Decode of packed id lists with every token's surface -> (text uint8[], text_offsets
        uint64[n+1], tok_end uint32[]): text and text_offsets as decode_packed, tok_end[k - id_offsets[0]] the end of
        token k's surface relative to its list's text; token k begins where token k-1 of its list ends, the first at 0."""
        n = len(id_offsets) - 1
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        ido = np.ascontiguousarray(id_offsets, dtype=np.uint64)
        p = [ctypes.c_void_p() for _ in range(3)]
        self._check(self._lib.spm_decode_offsets(self._h, ids.ctypes.data, ido.ctypes.data, n, *[ctypes.byref(x) for x in p]))
        to = np.ctypeslib.as_array(ctypes.cast(p[1], ctypes.POINTER(ctypes.c_uint64)), (n + 1,)).copy()
        tt, tot = int(to[n]), int(ido[n]) - int(ido[0])
        text = np.ctypeslib.as_array(ctypes.cast(p[0], ctypes.POINTER(ctypes.c_uint8)), (max(tt, 1),))[:tt].copy()
        te = np.ctypeslib.as_array(ctypes.cast(p[2], ctypes.POINTER(ctypes.c_uint32)), (max(tot, 1),))[:tot].copy()
        return text, to, te

    def set_random_seed(self, seed):
        self._check(self._lib.spm_set_random_seed(self._h, seed))

    def nbest_encode(self, buf, offs, nbest_size):
        """-> dict(ids, cand_offsets uint64[n*K+1], scores float32[n*K], n_cands uint32[n], K)"""
        n = len(offs) - 1
        K = max(1, min(nbest_size, 1024))
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        p = [ctypes.c_void_p() for _ in range(4)]
        self._check(self._lib.spm_nbest_encode(self._h, buf.ctypes.data, offs.ctypes.data, n, nbest_size,
                                               *[ctypes.byref(x) for x in p]))
        nc = n * K
        co = np.ctypeslib.as_array(ctypes.cast(p[1], ctypes.POINTER(ctypes.c_uint64)), (nc + 1,)).copy()
        tot = int(co[nc])
        ids = np.ctypeslib.as_array(ctypes.cast(p[0], ctypes.POINTER(ctypes.c_int32)), (max(tot, 1),))[:tot].copy()
        sc = np.ctypeslib.as_array(ctypes.cast(p[2], ctypes.POINTER(ctypes.c_float)), (max(nc, 1),))[:nc].copy()
        nk = np.ctypeslib.as_array(ctypes.cast(p[3], ctypes.POINTER(ctypes.c_uint32)), (max(n, 1),))[:n].copy()
        return dict(ids=ids, cand_offsets=co, scores=sc, n_cands=nk, K=K)

    def sample_encode(self, buf, offs, nbest_size, alpha):
        """SampleEncode over a packed batch -> (ids, id_offsets)"""
        n = len(offs) - 1
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        ids = ctypes.c_void_p()
        ido = ctypes.c_void_p()
        self._check(self._lib.spm_sample_encode_ids(self._h, buf.ctypes.data, offs.ctypes.data, n, nbest_size, alpha,
                                                    ctypes.byref(ids), ctypes.byref(ido)))
        o = np.ctypeslib.as_array(ctypes.cast(ido, ctypes.POINTER(ctypes.c_uint64)), (n + 1,)).copy()
        tot = int(o[n])
        a = np.ctypeslib.as_array(ctypes.cast(ids, ctypes.POINTER(ctypes.c_int32)), (max(tot, 1),))[:tot].copy()
        return a, o

    def calculate_entropy(self, buf, offs, alpha):
        """CalculateEntropy per sentence of a packed batch -> float32[n]"""
        n = len(offs) - 1
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        ent = ctypes.c_void_p()
        self._check(self._lib.spm_calculate_entropy(self._h, buf.ctypes.data, offs.ctypes.data, n, alpha, ctypes.byref(ent)))
        return np.ctypeslib.as_array(ctypes.cast(ent, ctypes.POINTER(ctypes.c_float)), (max(n, 1),))[:n].copy()

    def sample_encode_and_score(self, buf, offs, num_samples, alpha, wor=False, include_best=False):
        """-> (ids, cand_offsets uint64[n*num_samples+1], scores float32[n*num_samples])"""
        n = len(offs) - 1
        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        p = [ctypes.c_void_p() for _ in range(3)]
        self._check(self._lib.spm_sample_encode_and_score(self._h, buf.ctypes.data, offs.ctypes.data, n, num_samples, alpha,
                                                          int(wor), int(include_best), *[ctypes.byref(x) for x in p]))
        nc = n * num_samples
        co = np.ctypeslib.as_array(ctypes.cast(p[1], ctypes.POINTER(ctypes.c_uint64)), (nc + 1,)).copy()
        tot = int(co[nc])
        ids = np.ctypeslib.as_array(ctypes.cast(p[0], ctypes.POINTER(ctypes.c_int32)), (max(tot, 1),))[:tot].copy()
        sc = np.ctypeslib.as_array(ctypes.cast(p[2], ctypes.POINTER(ctypes.c_float)), (max(nc, 1),))[:nc].copy()
        return ids, co, sc

    def encode_device(self, d_bytes_ptr, d_offs_ptr, n, total_bytes, d_ids_ptr, ids_cap, d_id_offs_ptr, stream=None):
        """Device-resident batch (pointers are CUDA device pointers, e.g. torch data_ptr())."""
        tot = ctypes.c_uint64()
        self._check(self._lib.spm_encode_ids_device(self._h, d_bytes_ptr, d_offs_ptr, n, total_bytes, d_ids_ptr,
                                                    ids_cap, d_id_offs_ptr, ctypes.byref(tot), stream))
        return tot.value


    # ---- torch CUDA tensors on this engine's device, on torch's current stream ----
    def _stream(self, *tensors):
        import torch
        for t in tensors:
            if t is not None and (not t.is_cuda or t.device.index != self.device):
                raise ValueError(f"tensors must live on cuda:{self.device}, the engine's device (got {t.device})")
        return torch.cuda.current_stream(self.device).cuda_stream

    def pad_id(self):
        """The reference's pad_id(): the id of trainer_spec.pad_piece when that is a CONTROL piece, else -1."""
        if self._pad is None:  # (parsing the ModelProto takes tens of milliseconds: once per engine)
            from . import _modelinfo
            self._pad = _modelinfo.special_pieces(self._model_bytes)["pad_id"]
        return self._pad

    def encode_device_padded(self, d_bytes, d_offsets, width=0, pad_id=None, truncate=False, pad_left=False, out=None):
        """spm_encode_ids_device_padded: a batch already on the GPU (d_bytes uint8 [total], d_offsets int64 or uint64
        [n+1], byte offsets into d_bytes) -> (ids int32 [n, w], lengths int32 [n]).  Row i is sentence i's ids under the
        encode frame, then pad_id (None = the model's pad_id(); a model without a pad piece needs an explicit one);
        pad_left puts the ids at the end of their rows.  width = 0: w is the longest row; a fixed width fails on a
        longer row (ValueError) unless truncate, which keeps the frame and cuts the body.
        Without `out`, the ids go to n * guess new cells, guess being the width of this engine's previous width = 0 call
        (64 at first); when the longest row is wider, the call is repeated into n * w cells, which encodes the batch a
        second time.  out: a contiguous int32 tensor whose first n * w cells take the rows (ValueError when too small).
        The result is a [n, w] view of the cells."""
        import torch
        if pad_id is None:
            pad_id = self.pad_id()
            if pad_id < 0:
                raise ValueError("the model defines no pad piece (trainer_spec.pad_piece): pass pad_id explicitly")
        st = self._stream(d_bytes, d_offsets, out)
        if d_bytes.dtype != torch.uint8 or d_bytes.dim() != 1 or not d_bytes.is_contiguous():
            raise ValueError("d_bytes must be a contiguous 1-D uint8 tensor")
        if d_offsets.dtype not in (torch.int64, torch.uint64) or d_offsets.dim() != 1 or not d_offsets.is_contiguous():
            raise ValueError("d_offsets must be a contiguous 1-D int64 or uint64 tensor of n + 1 offsets")
        if out is not None and (out.dtype != torch.int32 or not out.is_contiguous()):
            raise ValueError("out must be a contiguous int32 tensor")
        n = d_offsets.numel() - 1
        flags = (_capi.PAD_TRUNCATE if truncate else 0) | (_capi.PAD_LEFT if pad_left else 0)
        lengths = torch.empty(n, dtype=torch.int32, device=d_bytes.device)

        def call(cells):
            w = ctypes.c_uint32()
            rc = self._lib.spm_encode_ids_device_padded(self._h, d_bytes.data_ptr(), d_offsets.data_ptr(), n,
                                                        d_bytes.numel(), cells.data_ptr(), cells.numel(), width, pad_id,
                                                        flags, lengths.data_ptr(), ctypes.byref(w), st)
            return rc, w.value

        cells = out if out is not None else torch.empty(n * (width or self._pad_guess), dtype=torch.int32,
                                                        device=d_bytes.device)
        rc, w = call(cells)
        too_long = width and not truncate and w > width
        if rc == _capi.SPM_ERR_CAPACITY and out is None and not too_long:
            cells = torch.empty(n * w, dtype=torch.int32, device=d_bytes.device)
            rc, w = call(cells)
        if rc == _capi.SPM_ERR_CAPACITY:
            raise ValueError(self._lib.spm_last_error(self._h).decode())
        self._check(rc)
        if not width and n:
            self._pad_guess = max(w, 1)  # (an all-empty batch gives 0, and zero cells have no device pointer)
        return cells.view(-1)[:n * w].view(n, w), lengths

    def encode_offsets_device_padded(self, d_bytes, d_offsets, width=0, pad_id=None, truncate=False, pad_left=False,
                                     unit="byte", eos_id=None, out=None):
        """spm_encode_offsets_device_padded: the rows of encode_device_padded with every token's begin / end in its
        input -> (ids int32 [n, w], spans int32 [n, w, 2], lengths int32 [n]).  spans[i, j] is (begin, end) of the
        token in ids[i, j], as encode_offsets gives it; frame entries equal to eos_id (None = the model's eos_id())
        get (len, len), other frame entries and pad cells (0, 0).  unit "byte": offsets in bytes of the sentence's
        input; "char": in characters, as ConvertToUnicodeSpans converts them (EncodeAsImmutableProto's begin / end).
        Arguments, errors and the width-0 retry as encode_device_padded; out: a contiguous int32 tensor of at least
        3 * n * w + 1 cells, which take the ids and then the spans (at an even cell, as the spans must be 8-byte
        aligned)."""
        import torch
        if unit not in ("byte", "char"):
            raise ValueError('unit must be "byte" or "char"')
        if pad_id is None:
            pad_id = self.pad_id()
            if pad_id < 0:
                raise ValueError("the model defines no pad piece (trainer_spec.pad_piece): pass pad_id explicitly")
        if eos_id is None:
            from . import _modelinfo
            eos_id = _modelinfo.special_pieces(self._model_bytes)["eos_id"]
        st = self._stream(d_bytes, d_offsets, out)
        if d_bytes.dtype != torch.uint8 or d_bytes.dim() != 1 or not d_bytes.is_contiguous():
            raise ValueError("d_bytes must be a contiguous 1-D uint8 tensor")
        if d_offsets.dtype not in (torch.int64, torch.uint64) or d_offsets.dim() != 1 or not d_offsets.is_contiguous():
            raise ValueError("d_offsets must be a contiguous 1-D int64 or uint64 tensor of n + 1 offsets")
        if out is not None and (out.dtype != torch.int32 or not out.is_contiguous()):
            raise ValueError("out must be a contiguous int32 tensor")
        n = d_offsets.numel() - 1
        flags = (_capi.PAD_TRUNCATE if truncate else 0) | (_capi.PAD_LEFT if pad_left else 0) | \
            (_capi.OFFSETS_CHARS if unit == "char" else 0)
        lengths = torch.empty(n, dtype=torch.int32, device=d_bytes.device)

        def call(cells):
            cap = max(cells.numel() - 1, 0) // 3
            at = cap + (cap & 1)  # first cell of the spans
            w = ctypes.c_uint32()
            rc = self._lib.spm_encode_offsets_device_padded(self._h, d_bytes.data_ptr(), d_offsets.data_ptr(), n,
                                                            d_bytes.numel(), eos_id, cells.data_ptr(),
                                                            cells.data_ptr() + 4 * at, cap, width, pad_id, flags,
                                                            lengths.data_ptr(), ctypes.byref(w), st)
            return rc, w.value, at

        cells = out if out is not None else torch.empty(3 * n * (width or self._pad_guess) + 1, dtype=torch.int32,
                                                        device=d_bytes.device)
        rc, w, at = call(cells)
        too_long = width and not truncate and w > width
        if rc == _capi.SPM_ERR_CAPACITY and out is None and not too_long:
            cells = torch.empty(3 * n * w + 1, dtype=torch.int32, device=d_bytes.device)
            rc, w, at = call(cells)
        if rc == _capi.SPM_ERR_CAPACITY:
            raise ValueError(self._lib.spm_last_error(self._h).decode())
        self._check(rc)
        if not width and n:
            self._pad_guess = max(w, 1)
        flat = cells.view(-1)
        return flat[:n * w].view(n, w), flat[at:at + 2 * n * w].view(n, w, 2), lengths

    def encode_device_windows(self, d_bytes, d_offsets, width, stride=0, pad_id=None, pad_left=False, unit=None,
                              eos_id=None, out=None):
        """spm_encode_windows_device: a batch already on the GPU as overlapping windows of `width` cells, each holding
        the encode frame and up to B = width - np - ns body ids; every window after a sentence's first starts
        B - stride ids later, so long sentences keep every token -> (ids int32 [R, w], lengths int32 [R],
        row_sentence int32 [R], row_first int32 [R]), plus spans int32 [R, w, 2] when unit is "byte" or "char" (None:
        no offsets).  row_sentence[r] is the sentence of row r, row_first[r] the index of its first body id in the
        sentence's body.  Cells, pad_id, pad_left, eos_id and the spans as encode_offsets_device_padded gives them.
        Without `out`, the rows go to max(n, guess) new rows, guess scaling the previous call's R / n; when R is larger,
        the call is repeated into exactly R rows, which encodes the batch a second time.  out: a contiguous int32 tensor
        of at least R * w cells (3 * R * w + 1 with spans: the ids, then the spans at an even cell) plus 3 * R for the
        lengths and the two row maps (ValueError when too small)."""
        import torch
        if unit not in (None, "byte", "char"):
            raise ValueError('unit must be None, "byte" or "char"')
        if pad_id is None:
            pad_id = self.pad_id()
            if pad_id < 0:
                raise ValueError("the model defines no pad piece (trainer_spec.pad_piece): pass pad_id explicitly")
        if eos_id is None:
            from . import _modelinfo
            eos_id = _modelinfo.special_pieces(self._model_bytes)["eos_id"]
        st = self._stream(d_bytes, d_offsets, out)
        if d_bytes.dtype != torch.uint8 or d_bytes.dim() != 1 or not d_bytes.is_contiguous():
            raise ValueError("d_bytes must be a contiguous 1-D uint8 tensor")
        if d_offsets.dtype not in (torch.int64, torch.uint64) or d_offsets.dim() != 1 or not d_offsets.is_contiguous():
            raise ValueError("d_offsets must be a contiguous 1-D int64 or uint64 tensor of n + 1 offsets")
        if out is not None and (out.dtype != torch.int32 or not out.is_contiguous()):
            raise ValueError("out must be a contiguous int32 tensor")
        n = d_offsets.numel() - 1
        flags = (_capi.PAD_LEFT if pad_left else 0) | (_capi.OFFSETS_CHARS if unit == "char" else 0)
        per_row = 3 * width + 3 if unit else width + 3  # cells a row takes: ids (and spans), length, sentence, first

        def layout(cells):
            rows = max(cells.numel() - (1 if unit else 0), 0) // per_row
            sp_at = rows * width + ((rows * width) & 1)  # the spans start at an even cell (8-byte aligned)
            len_at = sp_at + 2 * rows * width if unit else rows * width
            return rows, sp_at, len_at

        def call(cells):
            rows, sp_at, len_at = layout(cells)
            p = cells.data_ptr()
            r = ctypes.c_uint64()
            rc = self._lib.spm_encode_windows_device(self._h, d_bytes.data_ptr(), d_offsets.data_ptr(), n,
                                                     d_bytes.numel(), width, stride, pad_id, flags, eos_id, p,
                                                     p + 4 * sp_at if unit else None, rows, p + 4 * len_at,
                                                     p + 4 * (len_at + rows), p + 4 * (len_at + 2 * rows),
                                                     ctypes.byref(r), st)
            return rc, r.value

        def alloc(rows):
            return torch.empty(rows * per_row + (1 if unit else 0), dtype=torch.int32, device=d_bytes.device)

        cells = out if out is not None else alloc(max(n, int(n * self._win_ratio + 0.5), 1))
        rc, R = call(cells)
        if rc == _capi.SPM_ERR_CAPACITY and out is None:
            cells = alloc(R)
            rc, R = call(cells)
        if rc == _capi.SPM_ERR_CAPACITY:
            raise ValueError(self._lib.spm_last_error(self._h).decode())
        self._check(rc)
        if n:
            self._win_ratio = R / n
        rows, sp_at, len_at = layout(cells)
        flat = cells.view(-1)
        res = (flat[:R * width].view(R, width), flat[len_at:len_at + R], flat[len_at + rows:len_at + rows + R],
               flat[len_at + 2 * rows:len_at + 2 * rows + R])
        if unit:
            res += (flat[sp_at:sp_at + 2 * R * width].view(R, width, 2),)
        return res

    def encode_device_pairs(self, d_bytes, d_offsets, prefix=(), middle=(), suffix=(), width=0,
                            truncation="longest_first", overflow=False, stride=0, pad_id=None, pad_left=False,
                            unit=None, out=None):
        """spm_encode_pairs_device: a batch of 2n sentences already on the GPU (d_offsets: the 2n + 1 offsets of the
        stacked batch) as n pair rows prefix ++ A_i ++ middle ++ B_i ++ suffix, A_i = sentence i, B_i = sentence n + i,
        cut by `truncation` ("none", "longest_first", "only_first", "only_second") to `width` cells (0: the longest row,
        "none" only) -> (ids int32 [R, w], lengths int32 [R], type_ids int32 [R, w], row_pair int32 [R], row_first
        int32 [R]), plus spans int32 [R, w, 2] when unit is "byte" or "char" (None: no offsets).  overflow (with
        "only_first" / "only_second"): the cut member is split into windows that overlap by `stride` ids instead of
        being dropped; row_pair[r] is the pair of row r and row_first[r] the window's first id in that member.  The
        engine's encode frame does not apply.  A pair that cannot be laid out at `width` raises ValueError naming the
        width it needs.  Without `out`, the rows go to new tensors sized by a guess, and when R or w is larger the call
        is repeated into exactly R rows of w cells, which encodes the batch a second time.  out (fixed widths only): a
        contiguous int32 tensor of at least R * (2 * w + 3) cells (R * (4 * w + 3) with spans), 8-byte aligned, that
        takes the ids, the type ids, the spans, then the lengths and the two row maps (ValueError when too small)."""
        import torch
        if unit not in (None, "byte", "char"):
            raise ValueError('unit must be None, "byte" or "char"')
        if truncation not in _capi.PAIR_TRUNCATION:
            raise ValueError("truncation must be one of " + ", ".join(_capi.PAIR_TRUNCATION))
        if out is not None and not width:
            raise ValueError("out needs a fixed width")
        if pad_id is None:
            pad_id = self.pad_id()
            if pad_id < 0:
                raise ValueError("the model defines no pad piece (trainer_spec.pad_piece): pass pad_id explicitly")
        st = self._stream(d_bytes, d_offsets, out)
        if d_bytes.dtype != torch.uint8 or d_bytes.dim() != 1 or not d_bytes.is_contiguous():
            raise ValueError("d_bytes must be a contiguous 1-D uint8 tensor")
        if d_offsets.dtype not in (torch.int64, torch.uint64) or d_offsets.dim() != 1 or not d_offsets.is_contiguous():
            raise ValueError("d_offsets must be a contiguous 1-D int64 or uint64 tensor of 2n + 1 offsets")
        if (d_offsets.numel() - 1) % 2:
            raise ValueError("d_offsets must hold 2n + 1 offsets: the first members, then the second")
        if out is not None and (out.dtype != torch.int32 or not out.is_contiguous()):
            raise ValueError("out must be a contiguous int32 tensor")
        n = (d_offsets.numel() - 1) // 2
        flags = (_capi.PAD_LEFT if pad_left else 0) | (_capi.OFFSETS_CHARS if unit == "char" else 0) | \
            (_capi.PAIR_OVERFLOW if overflow else 0)
        lists = [(ctypes.c_int32 * len(x))(*x) for x in (prefix, middle, suffix)]

        per_cell = 4 if unit else 2  # int32 per cell: id, type id (and begin, end)

        def layout(total, w):
            """a flat buffer of `total` cells as rows of w: (rows, cells, type ids at, spans at, lengths at); the spans
            start at an even cell, 8-byte aligned"""
            rows = total // (per_cell * w + 3)
            cells = rows * w
            return rows, cells, cells, 2 * cells, per_cell * cells

        def call(buf, w):
            rows, cells, ty_at, sp_at, len_at = layout(buf.numel(), w)
            p = buf.data_ptr()
            r, wo = ctypes.c_uint64(), ctypes.c_uint32()
            rc = self._lib.spm_encode_pairs_device(
                self._h, d_bytes.data_ptr(), d_offsets.data_ptr(), n, d_bytes.numel(), lists[0], len(prefix), lists[1],
                len(middle), lists[2], len(suffix), width, _capi.PAIR_TRUNCATION[truncation], stride, pad_id, flags, p,
                p + 4 * ty_at, p + 4 * sp_at if unit else None, rows, cells, p + 4 * len_at, p + 4 * (len_at + rows),
                p + 4 * (len_at + 2 * rows), ctypes.byref(r), ctypes.byref(wo), st)
            return rc, r.value, wo.value

        def alloc(rows, w):
            return torch.empty(rows * (per_cell * w + 3), dtype=torch.int32, device=d_bytes.device)

        ratio, w_alloc = self._pair_guess
        w_alloc = width or w_alloc
        buf = out if out is not None else alloc(max(n, int(n * ratio + 0.5), 1), w_alloc)
        rc, R, w = call(buf, w_alloc)
        if rc == _capi.SPM_ERR_CAPACITY and out is None and R:
            w_alloc = w
            buf = alloc(R, w)
            rc, R, w = call(buf, w_alloc)
        if rc == _capi.SPM_ERR_CAPACITY:
            raise ValueError(self._lib.spm_last_error(self._h).decode())
        self._check(rc)
        if n:
            self._pair_guess = (R / n, max(w, 1))
        rows, cells, ty_at, sp_at, len_at = layout(buf.numel(), w_alloc)
        flat = buf.view(-1)
        res = (flat[:R * w].view(R, w), flat[len_at:len_at + R], flat[ty_at:ty_at + R * w].view(R, w),
               flat[len_at + rows:len_at + rows + R], flat[len_at + 2 * rows:len_at + 2 * rows + R])
        if unit:
            res += (flat[sp_at:sp_at + 2 * R * w].view(R, w, 2),)
        return res

    def decode_device(self, ids2d, lengths=None, stop_id=-1):
        """spm_decode_ids_device: the rows of an int32 or int64 [n, L] CUDA tensor (any row stride, e.g. a column slice;
        each row contiguous) -> list of n str.  Row i holds min(L, lengths[i]) ids (lengths: int32 [n], or None for L),
        cut before its first stop_id when stop_id >= 0; its text is DecodeIds of that list."""
        import torch
        if ids2d.dim() != 2 or ids2d.dtype not in (torch.int32, torch.int64):
            raise ValueError("ids2d must be a 2-D int32 or int64 tensor")
        n, L = ids2d.shape
        if L > 1 and ids2d.stride(1) != 1:
            raise ValueError("the ids of a row must be contiguous")
        if lengths is not None and (lengths.dtype != torch.int32 or lengths.shape != (n,) or not lengths.is_contiguous()):
            raise ValueError("lengths must be a contiguous int32 tensor of n entries")
        st = self._stream(ids2d, lengths)
        text = ctypes.c_void_p()
        to = ctypes.c_void_p()
        self._check(self._lib.spm_decode_ids_device(self._h, ids2d.data_ptr(), ids2d.element_size(), ids2d.stride(0), n,
                                                    L, lengths.data_ptr() if lengths is not None else None, stop_id,
                                                    ctypes.byref(text), ctypes.byref(to), st))
        o = np.ctypeslib.as_array(ctypes.cast(to, ctypes.POINTER(ctypes.c_uint64)), (n + 1,)).tolist()
        raw = np.ctypeslib.as_array(ctypes.cast(text, ctypes.POINTER(ctypes.c_uint8)), (max(o[n], 1),))[:o[n]].tobytes()
        return [raw[o[i]:o[i + 1]].decode("utf-8", errors="replace") for i in range(n)]

    def decode_stream_device(self, ids2d, state, lengths=None, stop_id=-1, final=None):
        """spm_decode_stream_device: the next ids of n streamed sequences -> list of n str, each the text these ids
        settle.  ids2d, lengths and stop_id are read as decode_device reads them; state: the n rows' states, a
        contiguous CUDA tensor of n * 16 bytes (all zeros for a fresh row), updated in place when the call succeeds;
        final: None or a contiguous int32 [n] CUDA tensor, non-zero for rows to finish in this call."""
        import torch
        if ids2d.dim() != 2 or ids2d.dtype not in (torch.int32, torch.int64):
            raise ValueError("ids2d must be a 2-D int32 or int64 tensor")
        n, L = ids2d.shape
        if L > 1 and ids2d.stride(1) != 1:
            raise ValueError("the ids of a row must be contiguous")
        if lengths is not None and (lengths.dtype != torch.int32 or lengths.shape != (n,) or not lengths.is_contiguous()):
            raise ValueError("lengths must be a contiguous int32 tensor of n entries")
        if final is not None and (final.dtype != torch.int32 or final.shape != (n,) or not final.is_contiguous()):
            raise ValueError("final must be a contiguous int32 tensor of n entries")
        if (not state.is_cuda or not state.is_contiguous()
                or state.numel() * state.element_size() != n * _capi.STREAM_STATE_BYTES):
            raise ValueError("state must be a contiguous CUDA tensor of n * 16 bytes")
        st = self._stream(ids2d, lengths, state, final)
        text = ctypes.c_void_p()
        to = ctypes.c_void_p()
        self._check(self._lib.spm_decode_stream_device(
            self._h, ids2d.data_ptr(), ids2d.element_size(), ids2d.stride(0), n, L,
            lengths.data_ptr() if lengths is not None else None, stop_id,
            final.data_ptr() if final is not None else None, state.data_ptr(), ctypes.byref(text), ctypes.byref(to), st))
        o = np.ctypeslib.as_array(ctypes.cast(to, ctypes.POINTER(ctypes.c_uint64)), (n + 1,)).tolist()
        raw = np.ctypeslib.as_array(ctypes.cast(text, ctypes.POINTER(ctypes.c_uint8)), (max(o[n], 1),))[:o[n]].tobytes()
        # every text is whole UTF-8 characters, so strict decoding cannot fail
        return [raw[o[i]:o[i + 1]].decode("utf-8") for i in range(n)]


class DecodeStream:
    """Streaming Decode for a batch of generated sequences (SentencePieceProcessor.decode_stream): each step() takes the
    next ids of every slot and returns the text they settle, so the texts of a slot's steps concatenate to DecodeIds
    of all its ids.  A slot finishes at stop_id or when final says so; then it ignores further ids until reset()."""

    def __init__(self, engine, batch_size, stop_id=-1):
        import torch
        self._engine = engine
        self._stop_id = stop_id
        self.state = torch.zeros((batch_size, _capi.STREAM_STATE_BYTES), dtype=torch.uint8,
                                 device=torch.device("cuda", engine.device))

    def step(self, ids, lengths=None, final=None):
        """ids: int32 / int64 CUDA tensor [batch_size, k] (k ids per slot, e.g. a column slice of the output), or
        [batch_size] for one id per slot; lengths: int32 [batch_size] ids to take per slot; final: int32
        [batch_size], non-zero to finish a slot after its ids -> list of batch_size str."""
        if ids.dim() == 1:
            ids = ids.unsqueeze(1)
        return self._engine.decode_stream_device(ids, self.state, lengths, self._stop_id, final)

    def reset(self, rows):
        """Zeroes the given slots (indices, a slice or a bool mask), which start new sequences at the next step."""
        self.state[rows] = 0

    @property
    def done(self):
        """bool [batch_size]: the slots that have finished"""
        return (self.state[:, _capi.STREAM_FLAGS_BYTE] & _capi.STREAM_DONE) != 0


def _id_lists(input):
    """One id list or a list of id lists -> (single, (ids int32[], id_offsets uint64[n+1]))"""
    single = len(input) == 0 or not isinstance(input[0], (list, tuple, np.ndarray))
    lists = [input] if single else list(input)
    ido = np.zeros(len(lists) + 1, dtype=np.uint64)
    if lists:
        ido[1:] = np.cumsum([len(x) for x in lists], dtype=np.uint64)
    ids = np.concatenate([np.asarray(x, dtype=np.int32) for x in lists]) if int(ido[-1]) else np.zeros(0, np.int32)
    return single, (ids, ido)


class SentencePieceProcessor:
    """Mirror of the reference's encode API (same method names / argument meaning as
    python/src/sentencepiece/__init__.py and src/sentencepiece_processor.h for this path)."""

    def __init__(self, model_file=None, model_proto=None, device=0):
        self._engine = None
        if model_file is not None:
            self.Load(model_file, device=device)
        elif model_proto is not None:
            self.LoadFromSerializedProto(model_proto, device=device)

    # sentencepiece_processor.h:245
    def Load(self, model_file, device=0):
        with open(model_file, "rb") as f:
            return self.LoadFromSerializedProto(f.read(), device=device)

    # sentencepiece_processor.h:261
    def LoadFromSerializedProto(self, serialized, device=0):
        self._model_bytes = bytes(serialized)
        self._engine = Engine(self._model_bytes, device=device)
        self._special = None
        self._pieces = None
        self._extra = []
        return True

    def _specials(self):
        if self._special is None:
            from . import _modelinfo
            self._special = _modelinfo.special_pieces(self._model_bytes)
        return self._special

    def _check_defined(self, option):
        sp = self._specials()
        if option in ("bos", "eos") and sp[option + "_id"] < 0:
            raise RuntimeError(f"id for `{sp[option + '_piece']}` is not defined.")  # sentencepiece_processor.cc:1088-1097

    # sentencepiece_processor.h:267, parse of sentencepiece_processor.cc:1067-1101; on an error no option is kept
    def SetEncodeExtraOptions(self, extra_option):
        self._require()
        self._extra = []
        opts = []
        for s in extra_option.split(":") if extra_option else []:
            if s not in _EXTRA_OPTIONS:
                raise RuntimeError(f'option "{s}" is not available.')
            opts.append(_EXTRA_OPTIONS[s])
            self._check_defined(opts[-1])
        self._extra = opts
        return True

    def _options(self, add_bos, add_eos, reverse):
        """SetEncodeExtraOptions' options, then the Python binding's reverse, bos, eos (sentencepiece.i:138-145)."""
        opts = list(self._extra) + ["reverse"] * bool(reverse) + ["bos"] * bool(add_bos) + ["eos"] * bool(add_eos)
        for o in opts:
            self._check_defined(o)
        return opts

    def _set_frame(self, add_bos, add_eos, reverse):
        """Makes the engine write the options' ids around every id list of the next call."""
        sp = self._specials()
        prefix, rev, suffix = extra_frame(self._options(add_bos, add_eos, reverse), sp["bos_id"], sp["eos_id"])
        self._engine.set_encode_frame(prefix, rev, suffix)

    def _require(self):
        if self._engine is None:
            raise RuntimeError("Model is not initialized.")  # sentencepiece_processor.cc:293-299

    # sentencepiece_processor.h:458 + python batch entry sentencepiece.i:439-446
    def DecodeIds(self, input, out_type=str):
        """Decode(ids) (src/sentencepiece_processor.h, python __init__.py DecodeIds): one id list or a list of lists;
        out_type str, bytes or 'immutable_proto' as in Decode."""
        self._require()
        if out_type is str:
            return self._decode(input, str)
        return self.Decode(input, out_type=out_type)

    # python/src/sentencepiece/__init__.py Decode (:776-868)
    def Decode(self, input, out_type=str):
        """An id, a list of ids or a list of id lists -> str, bytes or ImmutableSentencePieceText (out_type str, bytes or
        'immutable_proto'), one or a list.  Empty input returns '' as in the reference, whose `if not input` test also
        catches the single id 0.  Pieces (str input) are not decoded by the device path: NotImplementedError."""
        self._require()
        if not isinstance(input, np.ndarray) and not input:
            return ""
        if out_type is not str and out_type is not bytes and out_type != "immutable_proto":
            raise RuntimeError("unknown output or input type")
        first = input
        while isinstance(first, (list, tuple, np.ndarray)) and len(first):
            first = first[0]
        if isinstance(first, str):
            raise NotImplementedError("Decode of piece strings (DecodePieces) is not offered by the device path")
        if isinstance(input, (int, np.integer)):
            input = [int(input)]
        return self._decode(input, out_type)

    decode = Decode

    # sentencepiece.i _DecodeIdsAsImmutableProto (:506-512, 541-545): Decode(ids, SentencePieceText*), then
    # ConvertToUnicodeSpans over the decoded text
    def DecodeIdsAsImmutableProto(self, input):
        """One id list or a list of lists -> ImmutableSentencePieceText (or a list): the decoded text and every token's
        piece, id, surface (text[begin:end]) and begin / end in characters of that text."""
        return self.Decode(input, out_type="immutable_proto")

    decode_ids_as_immutable_proto = DecodeIdsAsImmutableProto

    def _decode(self, input, out_type):
        single, (ids, ido) = _id_lists(input)
        if out_type == "immutable_proto":
            text, to, te = self._engine.decode_offsets(ids, ido)
            if self._pieces is None:
                from . import _modelinfo
                self._pieces = [p.encode("utf-8") for p in _modelinfo.pieces_and_types(self._model_bytes)[0]]
            out = decode_protos(self._pieces, ids, ido, text, to, te)
        else:
            text, to = self._engine.decode_packed(ids, ido)
            raw = text.tobytes()
            out = [raw[int(to[i]):int(to[i + 1])] for i in range(len(ido) - 1)]
            if out_type is str:
                out = [o.decode("utf-8", errors="replace") for o in out]
        return out[0] if single else out

    def EncodeAsIds(self, input, add_bos=False, add_eos=False, reverse=False, emit_unk_piece=False):
        """emit_unk_piece changes piece strings only: it has no effect on ids."""
        self._require()
        single = isinstance(input, (str, bytes))
        buf, offs = pack_sentences([input] if single else input)
        self._set_frame(add_bos, add_eos, reverse)
        ids, ido = self._engine.encode_packed(buf, offs)
        out = [ids[int(ido[i]):int(ido[i + 1])].tolist() for i in range(len(offs) - 1)]
        return out[0] if single else out

    # ---- pieces (spm_encode_pieces): IdToPiece, unknown tokens keep their surface (sentencepiece_processor.cc:609-621);
    #      bos / eos / reverse through the encode frame, UNK_PIECE through unk_piece ----
    def EncodeAsPieces(self, input, add_bos=False, add_eos=False, reverse=False, emit_unk_piece=False):
        self._require()
        single, (buf, offs) = self._split(input)
        unk = self._pieces_frame(add_bos, add_eos, reverse, emit_unk_piece)
        r = self._engine.encode_pieces(buf, offs, unk_piece=unk)
        out = split_pieces(r["text"], r["text_offsets"], r["piece_end"], r["id_offsets"])
        return out[0] if single else out

    # sentencepiece.i _EncodeAsImmutableProto (:420-434): SetEncodeExtraOptions' options apply, then ConvertToUnicodeSpans
    def EncodeAsImmutableProto(self, input, enable_sampling=False, nbest_size=-1, alpha=0.1, add_bos=False,
                               add_eos=False, reverse=False, emit_unk_piece=False):
        """One str / bytes or a list of them -> ImmutableSentencePieceText (or a list): every token's piece, id,
        surface and begin / end in characters of the input.  add_bos / add_eos / reverse / emit_unk_piece are refused
        as in the reference (RewriteIds, sentencepiece.i:167-182); sampled protos are not offered."""
        self._require()
        if add_bos or add_eos or reverse or emit_unk_piece:
            raise RuntimeError("add_bos, add_eos, reverse, and emit_unk_piece is not supported in proto API")
        if enable_sampling:
            raise NotImplementedError("EncodeAsImmutableProto with enable_sampling is not offered by the device path")
        single = not isinstance(input, list)
        items = [input] if single else input
        buf, offs = pack_sentences(items)
        unk = self._pieces_frame(False, False, False, False)
        r = self._engine.encode_offsets(buf, offs, eos_id=self._specials()["eos_id"], unk_piece=unk)
        out = immutable_protos(items, buf, offs, r)
        return out[0] if single else out

    encode_as_immutable_proto = EncodeAsImmutableProto

    def encode(self, input, out_type=int, enable_sampling=False, nbest_size=-1, alpha=0.1, add_bos=False, add_eos=False,
               reverse=False, emit_unk_piece=False):
        """python/src/sentencepiece/__init__.py Encode: out_type int | str | 'immutable_proto'; enable_sampling uses
        SampleEncode.  add_bos / add_eos / reverse apply after SetEncodeExtraOptions' options, in the order reverse,
        bos, eos."""
        kw = dict(add_bos=add_bos, add_eos=add_eos, reverse=reverse, emit_unk_piece=emit_unk_piece)
        if out_type == "immutable_proto":
            return self.EncodeAsImmutableProto(input, enable_sampling, nbest_size, alpha, **kw)
        if enable_sampling:
            if out_type is int:
                return self.SampleEncodeAsIds(input, nbest_size, alpha, **kw)
            return self.SampleEncodeAsPieces(input, nbest_size, alpha, **kw)
        return self.EncodeAsIds(input, **kw) if out_type is int else self.EncodeAsPieces(input, **kw)

    Encode = encode

    def _split(self, input):
        single = isinstance(input, (str, bytes))
        return single, pack_sentences([input] if single else input)

    # sentencepiece_processor.h:481; the draws of a batch are taken in order on one generator (SetRandomGeneratorSeed)
    def SampleEncodeAsIds(self, input, nbest_size, alpha, add_bos=False, add_eos=False, reverse=False, emit_unk_piece=False):
        self._require()
        single, (buf, offs) = self._split(input)
        self._set_frame(add_bos, add_eos, reverse)
        ids, ido = self._engine.sample_encode(buf, offs, nbest_size, alpha)
        out = [ids[int(ido[i]):int(ido[i + 1])].tolist() for i in range(len(offs) - 1)]
        return out[0] if single else out

    def SampleEncodeAsPieces(self, input, nbest_size, alpha, add_bos=False, add_eos=False, reverse=False,
                             emit_unk_piece=False):
        self._require()
        single, (buf, offs) = self._split(input)
        unk = self._pieces_frame(add_bos, add_eos, reverse, emit_unk_piece)
        r = self._engine.sample_encode_pieces(buf, offs, nbest_size, alpha, unk_piece=unk)
        out = split_pieces(r["text"], r["text_offsets"], r["piece_end"], r["id_offsets"])
        return out[0] if single else out

    def _pieces_frame(self, add_bos, add_eos, reverse, emit_unk_piece):
        """Sets the frame for a pieces call and returns its unk_piece argument."""
        opts = self._options(add_bos, add_eos, reverse) + ["unk"] * bool(emit_unk_piece)
        self._set_frame(add_bos, add_eos, reverse)
        return self._specials()["unk_piece"] if "unk" in opts else None

    # sentencepiece_processor.h:471
    def NBestEncodeAsIds(self, input, nbest_size, add_bos=False, add_eos=False, reverse=False, emit_unk_piece=False):
        self._require()
        single, (buf, offs) = self._split(input)
        self._set_frame(add_bos, add_eos, reverse)
        r = self._engine.nbest_encode(buf, offs, nbest_size)
        K, co = r["K"], r["cand_offsets"]
        out = [[r["ids"][int(co[i * K + c]):int(co[i * K + c + 1])].tolist() for c in range(int(r["n_cands"][i]))]
               for i in range(len(offs) - 1)]
        return out[0] if single else out

    def NBestEncodeAsPieces(self, input, nbest_size, add_bos=False, add_eos=False, reverse=False, emit_unk_piece=False):
        self._require()
        single, (buf, offs) = self._split(input)
        unk = self._pieces_frame(add_bos, add_eos, reverse, emit_unk_piece)
        r = self._engine.nbest_encode_pieces(buf, offs, nbest_size, unk_piece=unk)
        K = r["K"]
        lists = split_pieces(r["text"], r["text_offsets"], r["piece_end"], r["cand_offsets"])
        out = [lists[i * K:i * K + int(r["n_cands"][i])] for i in range(len(offs) - 1)]
        return out[0] if single else out

    # python/src/sentencepiece/__init__.py NBestEncode
    def NBestEncode(self, input, out_type=int, nbest_size=-1, add_bos=False, add_eos=False, reverse=False,
                    emit_unk_piece=False):
        f = self.NBestEncodeAsIds if out_type is int else self.NBestEncodeAsPieces
        return f(input, nbest_size, add_bos=add_bos, add_eos=add_eos, reverse=reverse, emit_unk_piece=emit_unk_piece)

    # sentencepiece_processor.h:500-510: (list, score) pairs, num_samples per sentence; wor / include_best are not on
    # the device path
    def SampleEncodeAndScore(self, input, out_type=int, num_samples=-1, alpha=0.1, wor=False, include_best=False,
                             add_bos=False, add_eos=False, reverse=False, emit_unk_piece=False):
        self._require()
        single, (buf, offs) = self._split(input)
        if out_type is int:
            self._set_frame(add_bos, add_eos, reverse)
            ids, co, sc = self._engine.sample_encode_and_score(buf, offs, num_samples, alpha, wor, include_best)
            lists = [ids[int(co[j]):int(co[j + 1])].tolist() for j in range(len(co) - 1)]
        else:
            unk = self._pieces_frame(add_bos, add_eos, reverse, emit_unk_piece)
            r = self._engine.sample_encode_and_score_pieces(buf, offs, num_samples, alpha, wor, include_best, unk_piece=unk)
            co, sc = r["cand_offsets"], r["scores"]
            lists = split_pieces(r["text"], r["text_offsets"], r["piece_end"], co)
        out = []
        for i in range(len(offs) - 1):
            js = range(i * num_samples, (i + 1) * num_samples)
            # a sentence that normalizes to nothing has no samples (unigram_model.cc:745-747); only its slots are empty
            out.append([(lists[j], float(sc[j])) for j in js] if int(co[js[-1] + 1]) > int(co[js[0]]) else [])
        return out[0] if single else out

    def SampleEncodeAndScoreAsIds(self, input, num_samples=-1, alpha=0.1, wor=False, include_best=False, **kw):
        return self.SampleEncodeAndScore(input, int, num_samples, alpha, wor, include_best, **kw)

    def SampleEncodeAndScoreAsPieces(self, input, num_samples=-1, alpha=0.1, wor=False, include_best=False, **kw):
        return self.SampleEncodeAndScore(input, str, num_samples, alpha, wor, include_best, **kw)

    # ---- padded id tensors on the device (no reference counterpart): a model's [batch, seq_len] input, and the text
    #      of a [batch, T] generation output ----
    def encode_padded(self, input, max_len=None, pad_id=None, truncate=False, pad_left=False, add_bos=False,
                      add_eos=False, reverse=False, return_offsets=False):
        """EncodeAsIds of a batch as padded rows on the GPU -> (ids int32 [n, w], lengths int32 [n]) on the engine's
        device.  input: a list of str / bytes (packed and uploaded through pinned memory) or a (bytes, offsets) pair of
        CUDA tensors as Engine.encode_device_padded takes them.  max_len = None: w is the longest row; otherwise rows
        longer than max_len fail (ValueError) unless truncate, which keeps bos / eos and cuts the ids between them.
        pad_id = None: the model's pad_id(), and ValueError when it has none.
        return_offsets: -> (ids, lengths, offsets int32 [n, w, 2]), offsets[i, j] the (begin, end) of the token in
        ids[i, j] in characters of input i, as ConvertToUnicodeSpans counts them (EncodeAsImmutableProto's begin /
        end; eos gets (len, len), bos and pad cells (0, 0))."""
        self._require()
        d_bytes, d_offs = self._device_batch(input)
        self._set_frame(add_bos, add_eos, reverse)
        if return_offsets:
            ids, spans, lengths = self._engine.encode_offsets_device_padded(
                d_bytes, d_offs, width=max_len or 0, pad_id=pad_id, truncate=truncate, pad_left=pad_left, unit="char",
                eos_id=self._specials()["eos_id"])
            return ids, lengths, spans
        return self._engine.encode_device_padded(d_bytes, d_offs, width=max_len or 0, pad_id=pad_id, truncate=truncate,
                                                 pad_left=pad_left)

    def _device_batch(self, input):
        """A list of str / bytes packed and uploaded through pinned memory, or a (bytes, offsets) pair of CUDA tensors
        as it is."""
        if isinstance(input, tuple):
            return input
        import torch
        buf, offs = pack_sentences(input)
        dev = torch.device("cuda", self._engine.device)
        d_bytes = torch.from_numpy(np.require(buf, requirements="W")).pin_memory().to(dev, non_blocking=True)
        d_offs = torch.from_numpy(offs.view(np.int64)).pin_memory().to(dev, non_blocking=True)
        return d_bytes, d_offs

    def encode_windows(self, input, max_len, stride=0, pad_id=None, pad_left=False, add_bos=False, add_eos=False,
                       reverse=False, return_offsets=False):
        """EncodeAsIds of a batch as overlapping windows of max_len cells on the GPU, for inputs longer than a model's
        width: each window holds bos / eos and up to B = max_len - (bos + eos) ids, and a sentence's windows start
        B - stride ids apart, so no token is dropped -> (ids int32 [R, w], lengths int32 [R], row_sentence int32 [R],
        row_first int32 [R]) on the engine's device.  row_sentence[r] is the input row r comes from, row_first[r] the
        index of its first id in the sentence's ids (without bos / eos).  input, pad_id and pad_left as
        encode_padded.  return_offsets: -> (ids, lengths, row_sentence, row_first, offsets int32 [R, w, 2]), the
        offsets in characters as encode_padded(return_offsets=True) gives them."""
        self._require()
        d_bytes, d_offs = self._device_batch(input)
        self._set_frame(add_bos, add_eos, reverse)
        return self._engine.encode_device_windows(d_bytes, d_offs, max_len, stride=stride, pad_id=pad_id,
                                                  pad_left=pad_left, unit="char" if return_offsets else None,
                                                  eos_id=self._specials()["eos_id"])

    def encode_pairs(self, first, second, max_len=None, truncation=None, stride=None, prefix=(), middle=(), suffix=(),
                     pad_id=None, pad_left=False, return_offsets=False):
        """EncodeAsIds of a batch of sentence pairs as padded rows prefix ++ first[i] ++ middle ++ second[i] ++ suffix
        on the GPU (cross-encoders, NLI, extractive QA) -> (ids int32 [R, w], lengths int32 [R], type_ids int32
        [R, w]) on the engine's device; type ids are 1 from second[i]'s first cell through the suffix.  first /
        second: equal-length lists of str / bytes, or two (bytes, offsets) pairs of CUDA tensors as
        Engine.encode_device_pairs takes one batch; they are stacked into one batch on the device.  max_len = None:
        w is the longest row and nothing is cut; otherwise truncation ("longest_first" when None, "only_first",
        "only_second" or "none") fits the pairs to max_len.  stride (an int; with "only_first" / "only_second"): the
        cut member is split into windows overlapping by stride ids, every row repeating the other member, and the
        result also holds (row_pair int32 [R], row_first int32 [R]).  return_offsets: offsets int32 [R, w, 2] last, each
        token's (begin, end) in characters of its own member (EncodeAsImmutableProto's begin / end), (0, 0) on template
        and pad cells.  The add_bos / add_eos / reverse options do not apply: the template places the special ids."""
        self._require()
        if isinstance(first, tuple) != isinstance(second, tuple):
            raise ValueError("first and second must both be lists or both be (bytes, offsets) pairs")
        if isinstance(first, tuple):
            import torch
            (b1, o1), (b2, o2) = first, second
            if o1.numel() != o2.numel():
                raise ValueError("first and second must hold the same number of sentences")
            o1, o2 = o1.view(torch.int64), o2.view(torch.int64)
            end1, start2 = int(o1[-1]), int(o2[0])
            d_bytes = torch.cat([b1[:end1], b2[start2:]])
            d_offs = torch.cat([o1, o2[1:] - start2 + end1])
        else:
            if len(first) != len(second):
                raise ValueError("first and second must hold the same number of sentences")
            d_bytes, d_offs = self._device_batch(list(first) + list(second))
        if truncation is None:
            truncation = "none" if max_len is None else "longest_first"
        res = self._engine.encode_device_pairs(d_bytes, d_offs, prefix=prefix, middle=middle, suffix=suffix,
                                               width=max_len or 0, truncation=truncation, overflow=stride is not None,
                                               stride=stride or 0, pad_id=pad_id, pad_left=pad_left,
                                               unit="char" if return_offsets else None)
        out = (res[0], res[1], res[2])
        if stride is not None:
            out += (res[3], res[4])
        return out + (res[5],) if return_offsets else out

    def decode_padded(self, ids, lengths=None, stop_id=None):
        """DecodeIds of every row of an int32 / int64 [n, L] CUDA tensor -> list of n str: row i holds lengths[i] ids
        (all L when lengths is None), cut before its first stop_id (e.g. eos_id()) when one is given."""
        self._require()
        return self._engine.decode_device(ids, lengths, -1 if stop_id is None else stop_id)

    def decode_stream(self, batch_size, stop_id=None):
        """A DecodeStream of batch_size slots for a generation loop: step(ids) returns each slot's new text as the ids
        arrive; a slot finishes at stop_id (e.g. eos_id()) when one is given."""
        self._require()
        return DecodeStream(self._engine, batch_size, -1 if stop_id is None else stop_id)

    # python/src/sentencepiece/__init__.py Normalize, sentencepiece.i _Normalize / _NormalizeWithOffsets
    def Normalize(self, input, with_offsets=None):
        """The model's normalizer (SentencePieceProcessor::Normalize) on one str / bytes or a list of them: the same type
        back, with with_offsets a (text, offsets) pair per item.  Offsets map each normalized position, and the end, to
        the input: in characters for str input (ConvertToUnicodeAlignment), in bytes for bytes input."""
        self._require()
        single = not isinstance(input, list)
        items = [input] if single else input
        buf, offs = pack_sentences(items)
        text, no, n2o = self._engine.normalize(buf, offs, with_offsets=bool(with_offsets))
        raw = text.tobytes()
        outs = [raw[int(no[i]):int(no[i + 1])] for i in range(len(items))]
        outs = [o.decode("utf-8") if isinstance(x, str) else o for o, x in zip(outs, items)]
        if not with_offsets:
            return outs[0] if single else outs
        uo, uv = unicode_alignment(buf, offs, text, no, n2o)
        res = []
        for i, x in enumerate(items):
            if isinstance(x, str):
                res.append((outs[i], uv[int(uo[i]):int(uo[i + 1])].tolist()))
            else:
                m = n2o[int(no[i]) + i:int(no[i + 1]) + i + 1]
                res.append((outs[i], [] if m[0] == _capi.NORM_TO_ORIG_EMPTY else m.tolist()))
        return res[0] if single else res

    normalize = Normalize

    # sentencepiece_processor.h:521-526
    def CalculateEntropy(self, input, alpha):
        self._require()
        single, (buf, offs) = self._split(input)
        ent = self._engine.calculate_entropy(buf, offs, alpha).tolist()
        return ent[0] if single else ent

    def SetRandomGeneratorSeed(self, seed):
        self._require()
        self._engine.set_random_seed(seed)

    @property
    def engine(self):
        self._require()
        return self._engine
