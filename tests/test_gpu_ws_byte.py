"""The unigram lane kernel with the whole-word shortcut spells U+2581 as one byte, in its normalized text and in its
trie (lane_kernel.cuh, kWsByte).  These cases put U+2581 where both spellings have to agree: literal U+2581 in the
input (next to spaces and malformed bytes), charsmap rules whose targets contain spaces or a literal U+2581, runs of
spaces, the length limit of the lane kernel, an UNK U+2581 under byte fallback, and a model whose respelled pieces are
shorter than the longest UNK character.  Compared with the oracle.  Needs an H100."""
import numpy as np
import pytest

from conftest import model_bytes
from oracle import modelproto as mp
from oracle import oracle_py
from test_oracle_kat import space_rules_blob

pytestmark = pytest.mark.gpu
WS = "▁".encode()


def edge_lines(corpus_gen, seed, n):
    lines = []
    for i, s in enumerate(corpus_gen.lines("en", seed, n)):
        words = s.split(b" ")
        k = i % 8
        if k == 0:
            s = WS.join(words)                                  # a literal U+2581 for every space
        elif k == 1:
            s = b" " + WS + b" ".join(words) + WS               # literal U+2581 at both ends
        elif k == 2:
            s = b"   ".join(words) + b"    "                    # runs of spaces
        elif k == 3:
            s = (WS + b" " + WS + WS + b"  ").join(words)       # runs of literal and escaped U+2581
        elif k == 4:
            s = b" \xff ".join(words)                           # malformed byte between spaces
        elif k == 5:
            s = b"\xe2\x96 ".join(words)                        # truncated U+2581 before a space
        elif k == 6:
            s = WS + WS + b" " + s + b" " + WS + b"\xe2"
        lines.append(s)
    return lines + [WS, WS * 3, b" " + WS + b" ", WS + b"a", b"a" + WS, b"", b"   ", (WS + b" ") * 40,
                    b"\xe2\x96\x81\xe2\x96", b"x" + WS * 20 + b"y", b"\xe2\x96\x81 \xe2\x96\x81 a b"]


def encode_whole_word_kernel(mb, buf, offs, monkeypatch, capfd, force="1", expect_kernel=True):
    """Encodes with SPM_B200_FASTWORDS=force; the in-kernel counters of the lane kernel with the whole-word shortcut
    (printed to stderr) show whether it is the kernel that ran."""
    from sentencepiece_b200 import Engine
    monkeypatch.setenv("SPM_B200_FASTWORDS", force)
    monkeypatch.setenv("SPM_B200_KSTATS", "1")
    eng = Engine(mb)
    capfd.readouterr()
    got = eng.encode_packed(buf, offs)
    ran = "[kstats] groups" in capfd.readouterr().err
    assert ran == expect_kernel, "the whole-word lane kernel ran" if ran else "the whole-word lane kernel did not run"
    return eng, got


def assert_same(got, want, what):
    assert np.array_equal(np.asarray(got[1], np.uint64), np.asarray(want[1], np.uint64)), f"offsets differ: {what}"
    assert np.array_equal(got[0], want[0]), f"ids differ: {what}"


def test_literal_u2581_spaces_and_malformed_bytes(corpus_gen, monkeypatch, capfd):
    mb = model_bytes("uni32k")
    buf, offs = oracle_py.pack(edge_lines(corpus_gen, 4201, 4000))
    eng, got = encode_whole_word_kernel(mb, buf, offs, monkeypatch, capfd)
    assert_same(got, oracle_py.OracleModel(mb).encode_batch(buf, offs), "uni32k")
    eng.close()


@pytest.mark.parametrize("flags", [dict(), dict(remove_extra_whitespaces=False), dict(add_dummy_prefix=False)])
def test_charsmap_targets_with_spaces(flags, corpus_gen, monkeypatch, capfd):
    """rules "a" -> " A", "b" -> "B", "c" -> "D E", "d" -> " F G " (normalizer_test.cc:149-264) on a 32k vocabulary"""
    mb = mp.replace_flags(model_bytes("uni32k"), charsmap=space_rules_blob(), **flags)
    lines = edge_lines(corpus_gen, 4202, 2000) + [b"a", b"ba", b"c", b"da", b"ad", b"adb", b"d d  d", b" d" + WS + b"d "]
    buf, offs = oracle_py.pack(lines)
    eng, got = encode_whole_word_kernel(mb, buf, offs, monkeypatch, capfd)
    assert_same(got, oracle_py.OracleModel(mb).encode_batch(buf, offs), str(flags))
    eng.close()


def test_charsmap_target_with_literal_u2581(monkeypatch, capfd, corpus_gen):
    """the space rules with two targets respelled: "c" -> "U+2581", "d" -> "U+2581 FG" (same byte lengths, so the
    compiled double array is unchanged)"""
    blob = space_rules_blob().replace(b" F G \x00", WS + b"FG\x00").replace(b"D E\x00", WS + b"\x00")
    for flags in (dict(), dict(remove_extra_whitespaces=False)):
        mb = mp.replace_flags(model_bytes("uni32k"), charsmap=blob, **flags)
        om = oracle_py.OracleModel(mb)
        assert om.normalize(b"d")[0] == WS + WS + b"FG"
        lines = edge_lines(corpus_gen, 4205, 1000) + [b"c", b"cc", b"dc", b"cd", b"a c", b"c  a", b"d d", b"xc", b"cx",
                                                      b" c ", b"dd  cc"]
        buf, offs = oracle_py.pack(lines)
        eng, got = encode_whole_word_kernel(mb, buf, offs, monkeypatch, capfd)
        assert_same(got, om.encode_batch(buf, offs), str(flags))
        eng.close()


def test_whitespace_as_suffix(corpus_gen, monkeypatch, capfd):
    """suffix models are outside the whole-word shortcut (engine.cu upload_word_safe), so they never reach the one-byte
    spelling, even when the shortcut is forced; the plain lane kernel keeps three bytes"""
    mb = mp.replace_flags(model_bytes("uni32k"), treat_whitespace_as_suffix=True)
    buf, offs = oracle_py.pack(edge_lines(corpus_gen, 4203, 2000))
    eng, got = encode_whole_word_kernel(mb, buf, offs, monkeypatch, capfd, expect_kernel=False)
    assert_same(got, oracle_py.OracleModel(mb).encode_batch(buf, offs), "suffix")
    eng.close()


def test_pieces_shorter_than_an_unk_character(monkeypatch, capfd):
    """single-character pieces + "U+2581": one byte long when respelled, while the UNK edge over a 4-byte character is
    4 bytes long -- the ring must hold the longer of the two.  2-, 3- and 4-byte characters land on every ring slot."""
    chars = "abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789.,!?'"
    base = [("<unk>", 0.0, mp.UNKNOWN), ("<s>", 0.0, mp.CONTROL), ("</s>", 0.0, mp.CONTROL), ("▁", -2.0, mp.NORMAL)]
    mb = mp.build_model(base + [(ch, -3.0 - 0.01 * i, mp.NORMAL) for i, ch in enumerate(chars)], charsmap=b"")
    lines = []
    for x in ("é", "中", "😀", "😀😀", "é中😀", "中 😀", " 😀", "😀 ", "😀é", "a😀b"):
        for k in range(16):
            lines.append(("a" * k + x + "bc").encode())
            lines.append((" ".join(["ab"] * k) + " " + x + " cd").encode())
            lines.append(("é" * k + x + "中" * (k % 5)).encode())
    buf, offs = oracle_py.pack(lines)
    want = oracle_py.OracleModel(mb).encode_batch(buf, offs)
    for force, whole_words in (("1", True), ("0", False)):
        eng, got = encode_whole_word_kernel(mb, buf, offs, monkeypatch, capfd, force=force, expect_kernel=whole_words)
        assert_same(got, want, f"SPM_B200_FASTWORDS={force}")
        eng.close()


def test_unk_u2581_byte_fallback(corpus_gen, monkeypatch, capfd):
    """with the piece "U+2581" UNUSED, a U+2581 that no longer piece covers is an UNK character and falls back to the
    byte pieces of E2 96 81"""
    m = mp.parse_model(model_bytes("uni32k"))
    pieces = list(zip(m["pieces"], m["scores"], m["types"])) + [(b"<0x%02X>" % b, 0.0, mp.BYTE) for b in range(256)]
    mb = mp.replace_flags(model_bytes("uni32k"), byte_fallback=True, pieces=pieces)
    om = oracle_py.OracleModel(mb)
    t = om.types.copy()
    t[m["pieces"].index(WS)] = mp.UNUSED
    om.set_types(t)
    lines = edge_lines(corpus_gen, 4204, 2000) + [b"9 9 9", b"\xe4\xb8\x80 \xe4\xb8\x80" + WS, WS * 5 + b"  "]
    buf, offs = oracle_py.pack(lines)
    from sentencepiece_b200 import Engine
    monkeypatch.setenv("SPM_B200_FASTWORDS", "1")
    monkeypatch.setenv("SPM_B200_KSTATS", "1")
    eng = Engine(mb)
    eng.set_types(t)
    capfd.readouterr()
    got = eng.encode_packed(buf, offs)
    assert "[kstats] groups" in capfd.readouterr().err, "the whole-word lane kernel did not run"
    want = om.encode_batch(buf, offs)
    assert_same(got, want, "byte fallback, U+2581 unused")
    x, y, z = (len(m["pieces"]) + b for b in (0xE2, 0x96, 0x81))
    ids = got[0]
    assert np.any((ids[:-2] == x) & (ids[1:-1] == y) & (ids[2:] == z)), "no U+2581 fell back to bytes"
    eng.close()


def test_length_limit_counts_u2581_as_three_bytes(monkeypatch, capfd):
    """the lane kernel takes sentences of up to 512 normalized bytes; U+2581 counts three bytes there whatever the
    spelling and before the trailing strip, so the same sentences move on to the long-sentence kernels"""
    mb = model_bytes("uni32k")
    om = oracle_py.OracleModel(mb)
    # dummy prefix + "a" x words: 4 bytes per word; two trailing literal U+2581 (stripped) still count before the strip
    for words, tail, deferred in ((128, b"", 0), (129, b"", 1), (128, WS * 2, 1), (127, WS, 0)):
        buf, offs = oracle_py.pack([b" ".join([b"a"] * words) + tail])
        eng, got = encode_whole_word_kernel(mb, buf, offs, monkeypatch, capfd)
        assert_same(got, om.encode_batch(buf, offs), f"{words} words + {tail}")
        assert eng.info().last_deferred == deferred, words
        eng.close()
