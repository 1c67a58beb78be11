"""The inputs on which spm_encode_offsets is pinned to the unmodified reference, and the digest both sides are
compared by.  tools/record_offsets_reference.py runs the reference's Encode(absl::string_view, SentencePieceText*) on
them and stores the digests in tests/golden/reference_digests_offsets.json; tests/test_gpu_offsets.py computes the
same digest from the engine's result.

A case is one model, one SetEncodeExtraOptions string and one input set: 2000 English or mixed-script corpus lines, or
the inputs of tests/golden/edge_cases.json (empty, whitespace-only, NUL, malformed UTF-8, user symbols, sentences up
to 5000 bytes).  Mixed script covers byte fallback (mix_bf8k, mix_bpe4k) and runs of unknown characters (uni32k,
botchan8k, bpe32k).  Every piece is one "id:piece:surface:begin:end" field (piece and surface in hex, begin / end in
bytes of the input), a sentence one line, and the digest is the md5 of the lines."""
import base64
import hashlib
import json
import os

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PATH = os.path.join(GOLD, "reference_digests_offsets.json")
MODELS = ["uni32k", "botchan8k", "mix_bf8k", "bpe32k", "mix_bpe4k"]
FRAMES = ["", "bos:eos", "reverse", "eos:reverse:bos", "unk", "reverse:unk:eos"]
INPUTS = ["en", "mixed", "edge"]


def inputs(corpus_gen, name):
    if name == "edge":
        with open(os.path.join(GOLD, "edge_cases.json")) as f:
            return [base64.b64decode(s) for s in json.load(f)["inputs"]]
    return corpus_gen.lines(name, 7700 if name == "en" else 7701, 2000)


def key(model, name, frame):
    return f"{model}/{name}/{frame or '-'}"


def digest(rows):
    return hashlib.md5("\n".join(rows).encode()).hexdigest()


def row(tokens):
    """tokens: (id, piece bytes, surface bytes, begin, end) of one sentence"""
    return " ".join(f"{i}:{p.hex()}:{s.hex()}:{b}:{e}" for i, p, s, b, e in tokens)


def engine_rows(lines, r):
    """The rows of spm_encode_offsets' result r (with pieces, sep -1) for the inputs `lines`"""
    text = bytes(r["text"])
    ido, to = r["id_offsets"].tolist(), r["text_offsets"].tolist()
    ids, pe, bb, be = r["ids"].tolist(), r["piece_end"].tolist(), r["begin"].tolist(), r["end"].tolist()
    rows = []
    for i, s in enumerate(lines):
        t = text[to[i]:to[i + 1]]
        toks = []
        for k in range(ido[i], ido[i + 1]):
            p0 = pe[k - 1] if k > ido[i] else 0
            toks.append((ids[k], t[p0:pe[k]], s[bb[k]:be[k]], bb[k], be[k]))
        rows.append(row(toks))
    return rows


def stored():
    with open(PATH) as f:
        return json.load(f)


def restated(om, s):
    """PopulateSentencePieceText's (begin, end) of every token of s, before the extra options"""
    norm, n2o = om.normalize(s)
    ids, te = om.model_encode(norm)
    bf = bool(om.proto["byte_fallback"])
    out, c, prev_unk = [], 0, False
    for i, e in zip(ids.tolist(), te.tolist()):
        unk = i == om.unk_id
        if unk and bf:  # one byte token per byte; only the last carries the end
            b = n2o[c]
            out += [(b, b)] * (e - c - 1) + [(b, n2o[e])]
        elif unk and prev_unk:  # merged unknown run
            out[-1] = (out[-1][0], n2o[e])
        else:
            out.append((n2o[c], n2o[e]))
        c, prev_unk = e, unk
    assert c == len(norm)
    return out


def framed(spans, length, options, sp):
    """ApplyExtraOptions' offsets: bos (0, 0) first, eos (len, len) last, reverse reverses; unk leaves them alone"""
    out = list(spans)
    for o in options:
        if o == "reverse":
            out.reverse()
        elif o == "bos":
            out.insert(0, (0, 0))
        elif o == "eos":
            out.append((length, length))
    return out


def options_of(frame):
    return [{"unk_piece": "unk"}.get(o, o) for o in frame.split(":")] if frame else []
