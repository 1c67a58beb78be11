#!/usr/bin/env python3
"""Dev-container-only: regenerates the committed golden fixtures from the UNMODIFIED
reference compiled under oracle/_ref (needs /root/reference for that build).

  tests/golden/ids/<model>__<kind>.npz      ids/offsets of seeded corpora (reference output)
  tests/golden/edge_cases.json              ids of hand-picked edge inputs per model
  tests/golden/charsmap_space_rules.bin     the space-containing rule set of
                                            src/normalizer_test.cc:149-164 compiled with the
                                            reference's own Builder::CompileCharsMap
  tests/golden/charsmaps/<name>.bin         the rule sets of tests/charsmap_rules.py: the real ones
                                            from Builder::GetPrecompiledCharsMap, the synthetic ones
                                            compiled by Builder::CompileCharsMap
"""
import base64
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import charsmap_rules  # noqa: E402
import corpus  # noqa: E402
from oracle import oracle_py  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
SETS = [("uni32k", "en", 1234, 2000), ("uni32k", "mixed", 1235, 1000), ("mix_bf8k", "mixed", 1236, 2000),
        ("botchan8k", "en", 1237, 1000), ("bpe32k", "en", 1238, 2000), ("mix_bpe4k", "mixed", 1239, 1000)]

EDGE = [b"", b" ", b"   ", b"\t", b"a", b"hello world", b"  hello   world  ", b"\xe3\x80\x80\xe3\x80\x80ABC",
        "①②③".encode(), "㍿".encode(), " ｸﾞｰｸﾞﾙ ".encode(), "▁▁a▁".encode(), b"abc\x80xy", b"abc\xc3",
        b"ab\xe3\x81xy", b"a\xf3\x81\x81xy", b"ab\xc0\x82xy", b"\xef\xbf\xbd", b"a\x00b", b"\x00", b"\x7f\x01\x02",
        "😀😀 dog 吾輩は猫 cat".encode(), "éè é".encode(), "ﬁ ™ ½ Ⅷ ㎒".encode(),
        "ﷺ ﷺ".encode(), b"<sep>hello<mask> <sep>", b"<unk> <s> </s>", b"<0x41><0xE3>",
        ("long " * 400).encode(), ("長い文" * 300).encode(), b"x" * 5000, (b" " * 600) + b"end", b"\xe2\x96",
        b"\xf0\x9f\x98", "a　　b  c\t\td".encode(), "Ａｐｐｌｅ　ｐｉｅ".encode()]


def build_charsmap_tool():
    """a small program linked against the reference's Builder: `mk_charsmap OUT --rules FILE` compiles the rules of
    FILE (one "<hex key> <hex target>" line each) with CompileCharsMap, `mk_charsmap OUT --real NAME` writes the
    precompiled rule set NAME"""
    src = os.path.join("/tmp", "mk_charsmap.cc")
    with open(src, "w") as f:
        f.write(r"""
#include <cstdio>
#include <fstream>
#include <string>
#include "builder.h"
#include "util.h"
using namespace sentencepiece;
static std::string unhex(const std::string &h) {
  std::string s;
  for (size_t i = 0; i + 1 < h.size(); i += 2) s += static_cast<char>(std::stoi(h.substr(i, 2), nullptr, 16));
  return s;
}
int main(int argc, char **argv) {
  if (argc != 4) return 2;
  std::string out, mode = argv[2];
  if (mode == "--real") {
    if (!normalizer::Builder::GetPrecompiledCharsMap(argv[3], &out).ok()) return 1;
  } else {
    normalizer::Builder::CharsMap cm;
    std::ifstream in(argv[3]);
    std::string hk, ht;
    while (in >> hk >> ht) {
      normalizer::Builder::Chars a, b;
      for (const char32 c : string_util::UTF8ToUnicodeText(unhex(hk))) a.push_back(c);
      for (const char32 c : string_util::UTF8ToUnicodeText(unhex(ht == "-" ? "" : ht))) b.push_back(c);
      cm[a] = b;
    }
    if (!normalizer::Builder::CompileCharsMap(cm, &out).ok()) return 1;
  }
  FILE *f = fopen(argv[1], "wb"); fwrite(out.data(), 1, out.size(), f); fclose(f);
  return 0;
}
""")
    ref = "/root/reference"
    out = os.path.join("/tmp", "mk_charsmap")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-w", "-D_USE_INTERNAL_STRING_VIEW", "-DHAVE_PTHREAD=1", "-pthread",
                           f"-I{ROOT}/oracle/_ref/gen", f"-I{ref}", f"-I{ref}/src", f"-I{ref}/src/builtin_pb",
                           f"-I{ref}/third_party/protobuf-lite", f"-I{ref}/third_party", src,
                           f"{ROOT}/oracle/_ref/libsentencepiece_train.a", f"{ROOT}/oracle/_ref/libsentencepiece.a",
                           "-o", out])
    return out


def compile_rules(tool, rules, path):
    txt = os.path.join("/tmp", "mk_charsmap_rules.txt")
    with open(txt, "w") as f:
        for k, t in rules:
            f.write(f"{k.encode().hex()} {t.encode().hex() or '-'}\n")
    subprocess.check_call([tool, path, "--rules", txt])


def build_charsmaps():
    tool = build_charsmap_tool()
    # src/normalizer_test.cc:149-164
    compile_rules(tool, [("a", " A"), ("b", "B"), ("c", "D E"), ("d", " F G ")],
                  os.path.join(GOLD, "charsmap_space_rules.bin"))
    os.makedirs(charsmap_rules.DIR, exist_ok=True)
    for name in charsmap_rules.REAL:
        subprocess.check_call([tool, os.path.join(charsmap_rules.DIR, name + ".bin"), "--real", name])
    for name, rules in charsmap_rules.RULES.items():
        compile_rules(tool, rules, os.path.join(charsmap_rules.DIR, name + ".bin"))


def main():
    g = corpus.CorpusGen()
    for model, kind, seed, n in SETS:
        mb = open(os.path.join(GOLD, "models", model + ".model"), "rb").read()
        rm = oracle_py.RefModel(mb)
        buf, offs = g.fill(kind, seed, n)
        ids, ido = rm.encode_batch(buf, offs, threads=8)
        np.savez_compressed(os.path.join(GOLD, "ids", f"{model}__{kind}.npz"), ids=ids.astype(np.int32),
                            id_offsets=ido.astype(np.uint32), seed=seed, n=n)
    edge = {"inputs": [base64.b64encode(s).decode() for s in EDGE], "models": {}}
    for model in sorted({m for m, *_ in SETS}):
        mb = open(os.path.join(GOLD, "models", model + ".model"), "rb").read()
        rm = oracle_py.RefModel(mb)
        edge["models"][model] = {
            "ids": [rm.encode(s).tolist() for s in EDGE],
            "normalized": [base64.b64encode(rm.normalize(s)[0]).decode() for s in EDGE],
            "n2o": [rm.normalize(s)[1] if len(s) <= 80 else None for s in EDGE],
            "pieces": [[base64.b64encode(p).decode() for p in rm.encode_pieces(s)] if len(s) <= 80 else None for s in EDGE],
        }
    with open(os.path.join(GOLD, "edge_cases.json"), "w") as f:
        json.dump(edge, f)
    build_charsmaps()
    print("golden fixtures regenerated")


if __name__ == "__main__":
    if sys.argv[1:] == ["charsmaps"]:
        build_charsmaps()
    else:
        main()
