"""Records tests/golden/reference_digests_offsets.json: the unmodified reference's SentencePieceText (ids, pieces,
surfaces, begin, end) for every case of tests/offsets_cases.py, as digests.

Needs the reference library that oracle/Makefile builds (`make -C oracle _ref/libsentencepiece.a REF=<sentencepiece
checkout>`) and the reference's sources for their headers; no GPU.  tools/offsets_reference.cc is compiled against
them into a temporary directory, run once per case, and fails if any piece's surface is not input[begin, end).
Usage: python tools/record_offsets_reference.py [--ref /path/to/sentencepiece]"""
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
import offsets_cases as oc  # noqa: E402


def build(ref, tmp):
    lib = os.path.join(ROOT, "oracle", "_ref")
    exe = os.path.join(tmp, "offsets_reference")
    inc = [os.path.join(lib, "gen"), ref, os.path.join(ref, "src"), os.path.join(ref, "src", "builtin_pb"),
           os.path.join(ref, "third_party", "protobuf-lite"), os.path.join(ref, "third_party")]
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-w", "-D_USE_INTERNAL_STRING_VIEW", "-DHAVE_PTHREAD=1", "-pthread"] +
                          ["-I" + i for i in inc] +
                          ["-o", exe, os.path.join(ROOT, "tools", "offsets_reference.cc"),
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
        for name in oc.INPUTS:
            lines = oc.inputs(g, name)
            inp = os.path.join(tmp, name + ".hex")
            with open(inp, "w") as f:
                f.writelines(s.hex() + "\n" for s in lines)
            for model in oc.MODELS:
                mpath = os.path.join(ROOT, "tests", "golden", "models", model + ".model")
                for frame in oc.FRAMES:
                    rows = subprocess.check_output([exe, mpath, frame or "-", inp]).decode().split("\n")[:-1]
                    assert len(rows) == len(lines), (model, name, frame)
                    out[oc.key(model, name, frame)] = oc.digest(rows)
    with open(oc.PATH, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"{len(out)} digests -> {oc.PATH}")


if __name__ == "__main__":
    main()
