"""The id lists on which spm_decode_offsets is pinned to the unmodified reference, and the digest both sides are
compared by.  tools/record_decode_offsets_reference.py runs the reference's Decode(const std::vector<int>&,
SentencePieceText*) on them and stores the digests in tests/golden/reference_digests_decode_offsets.json;
tests/test_gpu_decode_offsets.py computes the same digest from the engine's result and tests/test_decode_offsets_host.py
from tests/decode_spans_oracle.c's.

A case is one of the five golden models under one normalizer-flag variant (as trained; remove_extra_whitespaces off;
add_dummy_prefix and remove_extra_whitespaces off) and one input set: the oracle's ids of 2000 English or mixed-script
corpus lines or of tests/golden/edge_cases.json, or seeded random lists in which 35 % of the ids are CONTROL, UNKNOWN or
BYTE pieces, with broken UTF-8 byte runs, empty lists and lists of more than 32 and more than 64 ids.  A list is one row:
the decoded text in hex, then one "id:piece:surface:begin:end" field per token (piece and surface in hex, begin / end
in bytes of the text); the digest is the md5 of the rows."""
import base64
import hashlib
import json
import os

import numpy as np

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PATH = os.path.join(GOLD, "reference_digests_decode_offsets.json")
MODELS = ["uni32k", "botchan8k", "mix_bf8k", "bpe32k", "mix_bpe4k"]
VARIANTS = {"trained": {}, "keep_ws": {"remove_extra_whitespaces": False},
            "no_prefix": {"add_dummy_prefix": False, "remove_extra_whitespaces": False}}
INPUTS = ["en", "mixed", "edge", "random"]


def model_variant(base, variant):
    """The serialized model of one flag variant"""
    from oracle import modelproto as mp
    kw = VARIANTS[variant]
    return mp.replace_flags(base, **kw) if kw else base


def random_lists(mb, seed):
    """Seeded id lists of the model mb: 35 % CONTROL / UNKNOWN / BYTE ids, runs of byte pieces from valid, truncated
    and corrupted UTF-8, empty lists, and lists of up to 150 ids"""
    from oracle import modelproto as mp
    m = mp.parse_model(mb)
    types = np.asarray(m["types"])
    vocab = len(types)
    special = np.flatnonzero(types != mp.NORMAL)
    byte_ids = {bytes(p).decode() if isinstance(p, bytes) else p: i for i, p in enumerate(m["pieces"]) if types[i] == mp.BYTE}
    rng = np.random.default_rng(seed)
    lists = []
    for n, maxlen in ((400, 24), (40, 70), (40, 150)):
        for _ in range(n):
            a = rng.integers(0, vocab, size=int(rng.integers(0, maxlen)))
            sel = rng.random(len(a)) < 0.35
            if len(special) and sel.any():
                a[sel] = rng.choice(special, size=int(sel.sum()))
            lists.append(a.tolist())
    if byte_ids:
        chars = "aZあΩい€😀ࠀ\U0010FFFF"
        for _ in range(120):
            raw = bytearray("".join(rng.choice(list(chars), size=int(rng.integers(1, 6)))).encode())
            cut = int(rng.integers(0, 3))
            if cut == 1:
                raw = raw[:-1]  # ends inside a character
            elif cut == 2 and raw:
                raw[int(rng.integers(0, len(raw)))] = int(rng.integers(0x80, 0x100))  # a stray byte
            lists.append([byte_ids["<0x%02X>" % b] for b in raw] + ([int(rng.choice(special))] if rng.random() < 0.5 else []))
    lists += [[], [], []]
    return lists


def lists_of(corpus_gen, name, mb):
    """The id lists of input set `name` for the model mb"""
    if name == "random":
        return random_lists(mb, 8800)
    from oracle import oracle_py
    from sentencepiece_b200.processor import pack_sentences
    if name == "edge":
        with open(os.path.join(GOLD, "edge_cases.json")) as f:
            buf, offs = pack_sentences([base64.b64decode(s) for s in json.load(f)["inputs"]])
    else:
        buf, offs = corpus_gen.fill(name, 7800 if name == "en" else 7801, 2000)
    ids, ido = oracle_py.OracleModel(mb).encode_batch(buf, offs)
    return [ids[int(ido[i]):int(ido[i + 1])].tolist() for i in range(len(ido) - 1)]


def packed(lists):
    ido = np.zeros(len(lists) + 1, dtype=np.uint64)
    ido[1:] = np.cumsum([len(x) for x in lists])
    ids = np.asarray([i for x in lists for i in x], dtype=np.int32)
    return ids, ido


def key(model, variant, name):
    return f"{model}/{variant}/{name}"


def digest(rows):
    return hashlib.md5("\n".join(rows).encode()).hexdigest()


def rows(pieces, ids, ido, text, text_offsets, tok_end):
    """The rows of a decode with offsets: pieces[id] as bytes, tok_end[k - ido[0]] the end of token k in its list"""
    raw = bytes(np.asarray(text, np.uint8))
    ids, to, te = np.asarray(ids).tolist(), np.asarray(text_offsets).tolist(), np.asarray(tok_end).tolist()
    ido = (np.asarray(ido, np.int64) - int(ido[0])).tolist()
    out = []
    for i in range(len(ido) - 1):
        t = raw[to[i]:to[i + 1]]
        f, b = [t.hex()], 0
        for k in range(ido[i], ido[i + 1]):
            f.append(f"{ids[k]}:{pieces[ids[k]].hex()}:{t[b:te[k]].hex()}:{b}:{te[k]}")
            b = te[k]
        out.append(" ".join(f))
    return out


def piece_bytes(mb):
    from sentencepiece_b200 import _modelinfo
    return [p.encode("utf-8") for p in _modelinfo.pieces_and_types(mb)[0]]


def stored():
    with open(PATH) as f:
        return json.load(f)
