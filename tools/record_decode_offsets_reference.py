"""Records tests/golden/reference_digests_decode_offsets.json: the unmodified reference's SentencePieceText (text, ids,
pieces, surfaces, begin, end) of Decode(ids) for every case of tests/decode_offsets_cases.py, as digests.

Needs the reference library that oracle/Makefile builds (`make -C oracle _ref/libsentencepiece.a REF=<sentencepiece
checkout>`) and the reference's sources for their headers; no GPU.  tools/decode_offsets_reference.cc is compiled
against them into a temporary directory and run once per case; it fails if a piece's id is not the input id, its
surface is not text[begin, end) or the surfaces do not tile the text.  The flag-variant models are written to the same
temporary directory.
Usage: python tools/record_decode_offsets_reference.py [--ref /path/to/sentencepiece]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import corpus  # noqa: E402
import decode_offsets_cases as dc  # noqa: E402


def build(ref, tmp):
    lib = os.path.join(ROOT, "oracle", "_ref")
    exe = os.path.join(tmp, "decode_offsets_reference")
    inc = [os.path.join(lib, "gen"), ref, os.path.join(ref, "src"), os.path.join(ref, "src", "builtin_pb"),
           os.path.join(ref, "third_party", "protobuf-lite"), os.path.join(ref, "third_party")]
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-w", "-D_USE_INTERNAL_STRING_VIEW", "-DHAVE_PTHREAD=1", "-pthread"] +
                          ["-I" + i for i in inc] +
                          ["-o", exe, os.path.join(ROOT, "tools", "decode_offsets_reference.cc"),
                           os.path.join(lib, "libsentencepiece.a")])
    return exe


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default=os.environ.get("SPM_REFERENCE_SRC", "/root/reference"))
    a = ap.parse_args()
    g = corpus.CorpusGen()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        exe = build(a.ref, tmp)
        for model in dc.MODELS:
            with open(os.path.join(ROOT, "tests", "golden", "models", model + ".model"), "rb") as f:
                base = f.read()
            for variant in dc.VARIANTS:
                mb = dc.model_variant(base, variant)
                mpath = os.path.join(tmp, f"{model}.{variant}.model")
                with open(mpath, "wb") as f:
                    f.write(mb)
                for name in dc.INPUTS:
                    lists = dc.lists_of(g, name, mb)
                    inp = os.path.join(tmp, "lists.txt")
                    with open(inp, "w") as f:
                        f.writelines(" ".join(map(str, x)) + "\n" for x in lists)
                    rows = subprocess.check_output([exe, mpath, inp]).decode().split("\n")[:-1]
                    assert len(rows) == len(lists), (model, variant, name)
                    out[dc.key(model, variant, name)] = dc.digest(rows)
    with open(dc.PATH, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"{len(out)} digests -> {dc.PATH}")


if __name__ == "__main__":
    main()
