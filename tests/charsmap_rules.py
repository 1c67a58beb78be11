"""Normalization rule sets (charsmaps) beyond the trained models' nmt_nfkc, and inputs that reach every rule.  No GPU;
not a test module.

The compiled charsmaps are committed under tests/golden/charsmaps/<name>.bin.  tools/make_golden.py writes them with
the reference's own Builder: GetPrecompiledCharsMap for the real rule sets, CompileCharsMap on `RULES` for the
synthetic ones.  The device normalizers pick their fast paths from tables built from the charsmap (the ASCII bytes
that start no rule of one byte or of two ASCII bytes, the longest-match walk from a register window, the tile's 32-byte
window and its carry into the next one, the worst-case expansion ratio that sizes buffers); each family below puts
rules on the far side of one of those choices:

  nfkc_cf, nmt_nfkc_cf  the reference's case-folding sets: A-Z are one-byte ASCII rules (nmt_nfkc has none)
  ascii_keys            keys of two and three ASCII bytes, `abcd` next to `a` (`abcx` falls back to `a`), ASCII +
                        combining mark keys, a rule on two spaces
  ladder                31 nested keys of `z`: the longest match backs off at every depth
  long_keys             keys of 9 to 100 bytes, ASCII and multi-byte; the 66- and 100-byte ones expand more than 3x
  delete_expand         an ASCII letter and a format character deleted, a CJK character -> 200 bytes, targets that are
                        only spaces or start or end with them
  glue                  " " -> "": a whole sentence is one word

`fires` counts, by NormalizePrefix's longest match (normalizer.cc:195-253), how often each rule key is the chunk chosen
at a position of the input, so that each family can show its corpus reaches the rules it is built for."""
import os
import random

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIR = os.path.join(ROOT, "tests", "golden", "charsmaps")

# the flag sets of the normalizer tests (src/normalizer_test.cc:77-147): the defaults and five variants
FLAGS = [dict(), dict(add_dummy_prefix=False), dict(remove_extra_whitespaces=False),
         dict(escape_whitespaces=False, add_dummy_prefix=False), dict(treat_whitespace_as_suffix=True),
         dict(escape_whitespaces=False, remove_extra_whitespaces=False)]
FLAG_IDS = ["default", "no_prefix", "keep_ws", "no_escape", "suffix", "no_escape_keep_ws"]

REAL = ["nfkc_cf", "nmt_nfkc_cf"]
LONG = (9, 16, 33, 40, 64, 65, 66, 100)  # the lane window is 5..8 bytes, the tile's 32, the old DFS depth cap 65


def key_of(n, ascii_only):
    """a key of exactly n UTF-8 bytes, unique per (n, ascii_only)"""
    if ascii_only:
        return (f"k{n}-" + "abcdefghijklmnopqrstuvwxyz0123456789" * 3)[:n]
    s = f"μ{n}·"
    for ch in "éあ😀ñ中ü" * 20:
        if len((s + ch).encode()) > n:
            break
        s += ch
    return s + "x" * (n - len(s.encode()))


def _long_keys():
    rules = []
    for n in LONG:
        for ascii_only in (True, False):
            if n == 66:
                tgt = "v " * 150                         # 300 bytes, 150 spaces: 600 escaped, ratio 9.1
            elif n == 100:
                tgt = "x" * 500 + " " + "y" * 300        # 801 bytes: 803 escaped, ratio 8.0
            else:
                tgt = f"<{n}{'a' if ascii_only else 'm'}>"  # shorter than the key
            rules.append((key_of(n, ascii_only), tgt))
    return rules


LADDER = list(range(1, 25)) + [26, 28, 30, 33, 36, 40, 45]  # 31 keys: fewer than 32 shared prefixes
RULES = {
    "ascii_keys": [("th", "Þ"), ("the", "ðe"), ("...", "…"), ("ff", "ﬀ"), (" .", "."), ("abcd", "ABCD"), ("a", "α"),
                   ("ing", "iŋ"), ("ou", "o u"), ("n\u0303", "\u00f1"), ("e\u0301", "\u00e9"), ("o\u0308", "\u00f6"),
                   ("  ", " ")],
    "ladder": [("z" * k, ("Z", "zz ", " ζ", "ŻŻ")[k % 4] + str(k)) for k in LADDER],
    "long_keys": _long_keys(),
    "delete_expand": [("q", ""), ("\u200b", ""), ("語", ("big target " * 19)[:200]), ("#", "   "), ("~", " "),
                      ("%", "  pct"), ("@", "at  "), ("&", " and "), ("·", " "), ("\t", " ")],
    "glue": [(" ", "")],
}
SYNTHETIC = list(RULES)
ALL = REAL + SYNTHETIC

# characters the real sets map, to inject next to the case changes of the corpus
REAL_KEYS = ["ﬁ", "Ⅷ", "①", "㍿", "Ａ", "ß", "İ", "Σ", "ǅ", "ｶﾞ", "½", "™", "　", "Ω", "Å", "µ"]


def blob(name):
    with open(os.path.join(DIR, name + ".bin"), "rb") as f:
        return f.read()


def keys(name):
    """the rule keys (UTF-8) that the corpus of `name` injects"""
    if name in RULES:
        return [k.encode() for k, _ in RULES[name]]
    return [k.encode() for k in REAL_KEYS]


def transform(lines, ks, seed):
    """corpus lines changed so that they hit the rules: title and upper case, keys at word starts, word ends and the
    sentence end, a key cut off by the end of the sentence, malformed UTF-8 and NUL right before or after a key"""
    rng = random.Random(seed)
    out = []
    for i, s in enumerate(lines):
        words = s.split(b" ")
        k = rng.choice(ks)
        m = i % 9
        if m == 0:
            s = s.title()
        elif m == 1:
            s = s.upper()
        elif m == 2:
            s = b" ".join(rng.choice(ks) + w if rng.random() < 0.4 else w for w in words)
        elif m == 3:
            s = b" ".join(w + rng.choice(ks) if rng.random() < 0.4 else w for w in words)
        elif m == 4:
            s = s + k
        elif m == 5:
            s = s + b" " + k[:max(1, len(k) - 1 - rng.randrange(3))]
        elif m == 6:
            s = s + rng.choice([b"\xff", b"\x00", b"\xc3", b"\xe2\x96"]) + k + rng.choice([b"\x80", b"\x00", b"\xf0\x9f"])
        elif m == 7:
            w = rng.randrange(len(words))
            words[w] = words[w] + b"".join(rng.choice(ks) for _ in range(rng.randrange(1, 4)))
            s = b" ".join(words)
        out.append(s)
    return out


def edge_lines(ks):
    """the empty and whitespace-only lines, and lengths on both sides of the lane kernels' 512 normalized bytes and of
    the general kernel's staging cap (2048 + 32 input bytes at the default tuning)"""
    lines = [b"", b" ", b"   ", b"\t", b"\t \t", b"\x00", b"  \x00  "]
    for k in ks[:6]:
        lines += [k, b" " + k + b" ", k + k, b"  " + k + b"   " + k + b"  ", k[:-1]]
    unit = b" ".join(ks[:4])
    for n in (120, 127, 129, 250, 500, 510, 512, 514, 530, 1000, 2040, 2048, 2049, 2100):
        lines.append((unit + b" ") * (n // (len(unit) + 1)) + b"a" * (n % (len(unit) + 1)))
    return lines


def family_lines(name):
    """inputs written for the rules of one family"""
    if name == "ascii_keys":  # `abcd` vs `a`; combining marks right after four simple ASCII bytes
        return [b"abcx", b"abcd", b"abc", b"abcdabcx", b"wxyzn\xcc\x83", b"kwxyzn\xcc\x83 o\xcc\x88", b"xyzwe\xcc\x81",
                b"the...", b"th the thee", b" . .  .", b"ff fff ffff", b"wxyz", b"wxyzn", b"wxyzn\xcc"]
    if name == "ladder":
        return [b"z" * k + b"y" for k in range(1, 50)] + [b"z" * k for k in (46, 60, 91)]
    if name == "long_keys":
        out = []
        for k in keys(name):
            out += [k, k[:-1] + b"!", k + k, b"word " + k + b" word", k[:len(k) // 2], b"ab" + k + b"\xff" + k]
        return out
    if name == "delete_expand":
        return [b"q", b"qqq", b" q ", b"q q", b"#", b" # ", b"a#b", b"~~", b"%", b"@@", b"a @ b", b"&&", b"\xe8\xaa\x9e",
                b"\xe8\xaa\x9e\xe8\xaa\x9e q", b"\t", b"\xe2\x80\x8b", b" \xe2\x80\x8b "]
    return []


def lines(name, corpus_gen, seed, n):
    """seeded corpus lines for the rule set `name`, transformed to hit its rules, plus the edge lines"""
    ks = keys(name)
    return (transform(corpus_gen.lines("en" if name != "nmt_nfkc_cf" else "mixed", seed, n), ks, seed) +
            edge_lines(ks) + family_lines(name))


def fires(name, corpus):
    """{rule key: how often NormalizePrefix's longest match chooses it}, over the lines of `corpus`"""
    ks = keys(name)
    by_len = sorted({len(k) for k in ks}, reverse=True)
    kset = set(ks)
    count = dict.fromkeys(ks, 0)
    for s in corpus:
        p = 0
        while p < len(s):
            for ln in by_len:
                if s[p:p + ln] in kset:
                    count[s[p:p + ln]] += 1
                    p += ln
                    break
            else:
                p += one_char(s, p)
    return count


def one_char(s, p):
    """bytes of the valid UTF-8 character at s[p], 1 for a malformed byte (util.cc:51-84)"""
    b = s[p]
    n = 1 if b < 0x80 else 2 if b >> 5 == 6 else 3 if b >> 4 == 14 else 4 if b >> 3 == 30 else 0
    if n == 0:
        return 1
    try:
        s[p:p + n].decode("utf-8")
        return n
    except UnicodeDecodeError:
        return 1
