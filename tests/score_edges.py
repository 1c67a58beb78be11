"""Model families whose ids are decided by float rounding and score ties, their corpora, and an exact-arithmetic
instrument that proves each corpus reaches the regime its family is built for.  No GPU; not a test module.

The reference's unigram Viterbi (EncodeOptimized, unigram_model.cc:950-1020) adds a float score to a float path
score in double, compares with the stored float on a strict `>` and stores the sum rounded to float; the UNK edge is a
float + float sum; a USER_DEFINED edge scores `length * max_score - 0.1` (the product in float, the difference in
double).  BPE (bpe_model.cc:51-57) merges the best-scored live pair, leftmost on ties.  The kernels reproduce these
decisions through rewrites that each hold only under a condition (the two-sum fold of the lane kernels, the whole-word
shortcut and its word_safe bound, the BPE tie order); the families below put a corpus on both sides of each.

`viterbi` restates the unigram recurrence with the reference's types (numpy float32 stores) and, next to it, the
exact optimum in integers (every double is an integer multiple of 2^-1074); `bpe_ties` restates the merge loop.
Both are written from the reference's algorithm, not from the oracle, so the oracle's digests and these counts are
two independent views of the same models."""
import math
from fractions import Fraction

import numpy as np

from oracle import modelproto as mp

WS = "▁".encode()
F32 = np.float32
SCALE = 1 << 1074  # every finite double times SCALE is an integer
LANE_CAP = 512     # normalized bytes of the longest sentence the lane kernels take


def f32(x):
    return float(F32(x))


def next_f32(x, k=1):
    """the float k ulps above x (k < 0: below)"""
    v = F32(x)
    to = F32(np.inf) if k > 0 else F32(-np.inf)
    for _ in range(abs(k)):
        v = np.nextafter(v, to)
    return float(v)


def exact(x):
    """a finite double as an integer multiple of 2^-1074"""
    fr = Fraction(x)
    return fr.numerator * (SCALE // fr.denominator)


def base_pieces():
    return [("<unk>", 0.0, mp.UNKNOWN), ("<s>", 0.0, mp.CONTROL), ("</s>", 0.0, mp.CONTROL)]


def one_char_len(b):
    return (1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 3, 4)[b >> 4]


def normalize(line, add_dummy_prefix=True):
    """the reference's normalization for these models (empty charsmap, extra whitespace removed, spaces escaped)"""
    words = line.split()
    if not words:
        return b""
    return (WS if add_dummy_prefix else b"") + WS.join(words)


class Family:
    """A model, its corpus and what the instrument must find in it.  `regime` maps a count name of `Stats` to the
    least value the corpus is designed to reach."""

    def __init__(self, name, pieces, lines, regime, model_type=mp.UNIGRAM, add_dummy_prefix=True, doc=""):
        self.name = name
        self.pieces = pieces
        self.lines = lines
        self.regime = regime
        self.model_type = model_type
        self.add_dummy_prefix = add_dummy_prefix
        self.model = mp.build_model(pieces, model_type=model_type, add_dummy_prefix=add_dummy_prefix)
        self.doc = doc

    @property
    def unigram(self):
        return self.model_type == mp.UNIGRAM

    def normalized(self):
        return [normalize(s, self.add_dummy_prefix) for s in self.lines]


# ------------------------------------------------------------------------------------------------ instrument --

class Stats:
    def __init__(self):
        self.exact_ties = 0        # a later candidate equal to the stored value: kept out by the strict `>`
        self.rounding = 0          # float-equal to the stored value but exactly different: the two-sum term decides
        self.off_optimum = 0       # sentences whose reference path scores below the exact optimum
        self.userdef_float = 0     # sentences whose path changes when USER_DEFINED scores are computed in float
        self.crosses_2_18 = 0      # sentences of <= LANE_CAP bytes whose path score passes 2^18 in magnitude
        self.double_vs_float = 0   # decisions a float-only candidate (no two-sum term) would reverse
        self.word_alone = 0        # U-nearword: words the reference ends with the whole-word piece alone
        self.word_split = 0        # U-nearword: S_P > S_alt exactly, yet the reference splits the word
        # (both in sentences of <= LANE_CAP bytes, the ones the lane kernel with the shortcut takes)
        self.bpe_ties = 0          # BPE merges with two or more live best-scored pairs
        self.bpe_ties_distinct = 0 # ... of which at least two are different pieces

    def add(self, o):
        for k, v in vars(o).items():
            setattr(self, k, getattr(self, k) + v)


class UnigramModel:
    def __init__(self, pieces):
        self.piece = {}
        normal = []
        for i, (p, s, t) in enumerate(pieces):
            p = p.encode() if isinstance(p, str) else p
            s = f32(s)
            if t in (mp.NORMAL, mp.USER_DEFINED, mp.UNUSED):
                self.piece[p] = (i, s, t)
            if t == mp.NORMAL:
                normal.append(s)
            if t == mp.UNKNOWN:
                self.unk_id = i
        self.min_score = min(normal)
        # unigram_model.cc:657-664: max starts at FLT_MIN
        self.max_score = max(normal + [f32(np.finfo(np.float32).tiny)])
        self.unk_score = f32(F32(self.min_score) - F32(10.0))
        self.maxlen = max(len(p) for p in self.piece)
        self.userdef_in_float = False

    def userdef_score(self, length):
        prod = F32(F32(length) * F32(self.max_score))
        if self.userdef_in_float:
            return float(F32(prod - F32(0.1)))
        return float(prod) - 0.1

    def edges(self, text, s):
        """(end, id, score as a double, piece type) of the pieces starting at s, shortest first"""
        for L in range(1, min(self.maxlen, len(text) - s) + 1):
            hit = self.piece.get(text[s:s + L])
            if hit is None or hit[2] == mp.UNUSED:
                continue
            i, sc, t = hit
            yield s + L, i, (self.userdef_score(L) if t == mp.USER_DEFINED else sc), t

    def viterbi(self, text, st=None):
        """The reference's recurrence on normalized `text`.  Returns [(start, end, id)] and adds counts to `st`."""
        n = len(text)
        best = [None] * (n + 1)  # (float score, start, id)
        best[0] = (0.0, -1, -1)
        s = 0
        while s < n:
            base = best[s][0]
            mblen = min(one_char_len(text[s]), n - s)
            single = False
            for e, i, sc, t in self.edges(text, s):
                cand = sc + base
                cur = best[e]
                if st is not None and cur is not None:
                    self._count(st, cand, cur[0], t)
                if cur is None or cand > cur[0]:
                    best[e] = (f32(cand), s, i)
                single |= e - s == mblen
            if not single:
                e = s + mblen
                cand = f32(F32(self.unk_score) + F32(base))
                cur = best[e]
                if st is not None and cur is not None and cand == cur[0]:
                    st.exact_ties += 1
                if cur is None or cand > cur[0]:
                    best[e] = (cand, s, self.unk_id)
            s += mblen
        path, e = [], n
        while e > 0:
            _, b, i = best[e]
            path.append((b, e, i))
            e = b
        return path[::-1]

    def _count(self, st, cand, cur, t):
        if cand == cur:
            st.exact_ties += 1
        elif math.isfinite(cand) and f32(cand) == cur:
            st.rounding += 1
        ref = cand > cur
        if t == mp.NORMAL and math.isfinite(cand) and ref != (f32(cand) > cur):
            st.double_vs_float += 1

    def exact_best(self, text, skip=None):
        """the exact optimum over all segmentations (the reference's edge set); `skip` = (start, end) of an edge to
        leave out.  Integers scaled by 2^1074; None when no path exists."""
        n = len(text)
        best = [None] * (n + 1)
        best[0] = 0
        unk = exact(self.unk_score)
        s = 0
        while s < n:
            mblen = min(one_char_len(text[s]), n - s)
            if best[s] is not None:
                single = False
                for e, _, sc, _ in self.edges(text, s):
                    single |= e - s == mblen
                    if (s, e) == skip:
                        continue
                    v = best[s] + exact(sc)
                    if best[e] is None or v > best[e]:
                        best[e] = v
                if not single:
                    v = best[s] + unk
                    if best[s + mblen] is None or v > best[s + mblen]:
                        best[s + mblen] = v
            s += mblen
        return best[n]

    def path_exact(self, text, path):
        tot = 0
        for b, e, i in path:
            if i == self.unk_id:
                tot += exact(self.unk_score)
            else:
                hit = self.piece[text[b:e]]
                tot += exact(self.userdef_score(e - b) if hit[2] == mp.USER_DEFINED else hit[1])
        return tot


def measure_unigram(fam, words=()):
    """Counts of the family's corpus.  `words`: whole-word pieces (normalized bytes) whose occurrences are sorted
    into word_alone / word_split."""
    um = UnigramModel(fam.pieces)
    st = Stats()
    wordset = set(words)
    for text in fam.normalized():
        path = um.viterbi(text, st)
        opt = um.exact_best(text)
        if opt is not None and um.path_exact(text, path) < opt:
            st.off_optimum += 1
        if len(text) <= LANE_CAP and abs(path_float(um, text, path)) >= 2.0 ** 18:
            st.crosses_2_18 += 1
        if any(t == mp.USER_DEFINED for _, _, t in um.piece.values()):
            um.userdef_in_float = True
            st.userdef_float += um.viterbi(text) != path
            um.userdef_in_float = False
        if wordset and len(text) <= LANE_CAP:
            edges = {(b, e) for b, e, _ in path}
            for b, e in word_spans(text):
                w = text[b:e]
                if w not in wordset:
                    continue
                if (b, e) in edges:
                    st.word_alone += 1
                else:
                    sp = exact(um.piece[w][1])
                    alt = um.exact_best(w, skip=(0, len(w)))
                    if alt is None or sp > alt:
                        st.word_split += 1
    return st


def path_float(um, text, path):
    """the float path score the reference stores at the end of `path`"""
    v = 0.0
    for b, e, i in path:
        if i == um.unk_id:
            v = f32(F32(um.unk_score) + F32(v))
        else:
            hit = um.piece[text[b:e]]
            v = f32((um.userdef_score(e - b) if hit[2] == mp.USER_DEFINED else hit[1]) + v)
    return v


def word_spans(text):
    """[b, e) of every word: U+2581 up to the next U+2581"""
    starts = [i for i in range(len(text)) if text.startswith(WS, i)]
    return [(b, e) for b, e in zip(starts, starts[1:] + [len(text)])]


def bpe_ties(pieces, text):
    """The reference's merge loop (bpe_model.cc:110-173) on normalized `text`; counts merges with tied best pairs."""
    score = {}
    for p, s, t in pieces:
        if t == mp.NORMAL:
            score[p.encode() if isinstance(p, str) else p] = f32(s)
    syms, i = [], 0
    while i < len(text):
        L = min(one_char_len(text[i]), len(text) - i)
        syms.append(text[i:i + L])
        i += L
    ties = distinct = 0
    while True:
        cands = [(score[a + b], j, a + b) for j, (a, b) in enumerate(zip(syms, syms[1:])) if a + b in score]
        if not cands:
            break
        top = max(c[0] for c in cands)
        tied = [c for c in cands if c[0] == top]
        ties += len(tied) > 1
        distinct += len({c[2] for c in tied}) > 1
        j = tied[0][1]
        syms[j:j + 2] = [syms[j] + syms[j + 1]]
    return ties, distinct


def measure_bpe(fam):
    st = Stats()
    for text in fam.normalized():
        t, d = bpe_ties(fam.pieces, text)
        st.bpe_ties += t
        st.bpe_ties_distinct += d
    return st


def measure(fam):
    if not fam.unigram:
        return measure_bpe(fam)
    with np.errstate(over="ignore"):  # U-overflow: float path scores reach -inf on purpose
        return measure_unigram(fam, getattr(fam, "words", ()))


# -------------------------------------------------------------------------------------------------- families --

def _words(rng, alphabet, lo, hi, count):
    return ["".join(rng.choice(list(alphabet), rng.randint(lo, hi + 1))) for _ in range(count)]


def _line(rng, alphabet, lo, hi, nwords):
    return " ".join(_words(rng, alphabet, lo, hi, nwords)).encode()


def _near_sums(rng, singles, count, jitter, keep):
    """multi-character pieces scored within `jitter` ulps of the sum of their characters' scores: the split and the
    piece reach the same end with float-close path scores, so rounding decides"""
    out, seen = [], set()
    keys = sorted(singles)
    while len(out) < count:
        w = "".join(rng.choice(keys, rng.randint(2, 4)))
        if w in seen:
            continue
        seen.add(w)
        s = next_f32(f32(sum(singles[c] for c in w)), int(rng.randint(-jitter, jitter + 1)))
        if keep(s):
            out.append((w, s, mp.NORMAL))
    return out


def u_flat():
    """Every NORMAL piece scores -1: all segmentations with the same number of pieces tie exactly, so every decision
    is the strict `>` (Q2: the earliest start wins) or the first relaxation into a position."""
    rng = np.random.RandomState(101)
    al = "abcde"
    pcs = base_pieces() + [("▁", -1.0, mp.NORMAL)] + [(c, -1.0, mp.NORMAL) for c in al]
    pcs += [(a + b, -1.0, mp.NORMAL) for a in al for b in al]
    pcs += [(w, -1.0, mp.NORMAL) for w in sorted(set(_words(rng, al, 3, 5, 40)))]
    pcs += [("▁" + c, -1.0, mp.NORMAL) for c in "abc"]
    lines = [_line(rng, al, 1, 12, rng.randint(3, 30)) for _ in range(300)]
    return Family("u_flat", pcs, lines, dict(exact_ties=5000), doc=u_flat.__doc__)


def u_chain():
    """Pieces a, aa, ... up to 62 bytes of a, plus b, c, d and U+2581, all scored -1: the most matches per start
    (match_slots 63), the largest lane ring (R = 64) and more lattice nodes than the n-best kernel's first attempt
    holds for a 512-byte sentence, so its retry with roomy slabs runs."""
    rng = np.random.RandomState(102)
    pcs = base_pieces() + [("▁", -1.0, mp.NORMAL)] + [("a" * k, -1.0, mp.NORMAL) for k in range(1, 63)]
    pcs += [(c, -1.0, mp.NORMAL) for c in "bcd"]
    lines = []
    for i in range(60):
        parts = []
        while sum(len(p) + 1 for p in parts) < rng.randint(60, 500):
            parts.append("a" * rng.randint(1, 200) + "".join(rng.choice(list("abcd"), rng.randint(0, 4))))
        lines.append(" ".join(parts).encode())
    lines += [b"a" * 62, b"a" * 63, b"a" * 124, b"a" * 125, b"a" * 508, b"a" * 511, b"ab" * 100, b"a"]
    return Family("u_chain", pcs, lines, dict(exact_ties=20000), doc=u_chain.__doc__)


def u_round():
    """Random float32 scores with full mantissas in [-20, -1], multi-character pieces within a few ulps of the sum of
    their characters, sentences long enough that the path score reaches about -2000: many relaxations are
    float-equal to the stored score but exactly different, and the two-sum term of the lane kernels decides them."""
    rng = np.random.RandomState(103)
    al = "abcdefghijklmnop"
    singles = {c: f32(-1.0 - 8.0 * rng.rand()) for c in al}
    pcs = base_pieces() + [("▁", f32(-1.0 - 3.0 * rng.rand()), mp.NORMAL)] + [(c, s, mp.NORMAL) for c, s in singles.items()]
    pcs += _near_sums(rng, singles, 150, 3, lambda s: -20.0 <= s <= -1.0)
    lines = [_line(rng, al, 2, 9, rng.randint(30, 80)) for _ in range(200)]
    return Family("u_round", pcs, lines, dict(rounding=300, off_optimum=20, double_vs_float=100), doc=u_round.__doc__)


def u_irregular():
    """Scores outside the two-sum fold's range, so every NORMAL relaxation of the lane kernels takes the double branch:
    tiny (|s| < 2^-10), subnormal, -0.0 next to 0.0, large (-5000, -1e6), near-sum pieces of large scores (rounding
    decides), and a min_score so large that min_score - 10 == min_score (UNK edges tie with the worst piece)."""
    rng = np.random.RandomState(104)
    singles = {c: f32(-1500.0 - 900.0 * rng.rand()) for c in "abcdefgh"}
    pcs = base_pieces() + [("▁", -0.0, mp.NORMAL)] + [(c, s, mp.NORMAL) for c, s in singles.items()]
    pcs += [("i", 0.0, mp.NORMAL), ("j", -0.0, mp.NORMAL), ("ij", 0.0, mp.NORMAL), ("ji", -0.0, mp.NORMAL),
            ("k", -1e-4, mp.NORMAL), ("l", -3e-5, mp.NORMAL), ("kl", f32(F32(-1e-4) + F32(-3e-5)), mp.NORMAL),
            ("m", -1e-42, mp.NORMAL), ("mm", -2e-42, mp.NORMAL), ("n", -5000.0, mp.NORMAL), ("o", -1e6, mp.NORMAL),
            ("no", f32(F32(-5000.0) + F32(-1e6)), mp.NORMAL), ("z", -1e9, mp.NORMAL)]
    pcs += _near_sums(rng, singles, 120, 2, lambda s: True)
    al = "abcdefghijklmnoyz"  # y has no piece: UNK edges of min_score - 10 == min_score
    lines = [_line(rng, al, 1, 8, rng.randint(5, 60)) for _ in range(200)]
    lines += [b"ij ji iijj", b"m mm mmm", b"k l kl lk", b"z y zy yz", b"no on nno"]
    return Family("u_irregular", pcs, lines, dict(rounding=100, exact_ties=100, double_vs_float=50),
                  doc=u_irregular.__doc__)


def u_boundary():
    """Scores at the limits of the regular range (exactly 2^-10 and 1024; the model stays regular), letters scored
    near -1000 and sentences of 300-500 letters: the path score crosses 2^18 inside one sentence, so the lane kernels
    switch from the two-sum fold to the double branch mid-sentence.  Pieces `x` + `q` (q scored 2^-10) next to `xq`
    scored within an ulp of the sum keep rounding-decided relaxations on both sides of the switch."""
    rng = np.random.RandomState(105)
    singles = {c: f32(-900.0 - 120.0 * rng.rand()) for c in "abcdefgh"}
    tiny = 2.0 ** -10
    pcs = base_pieces() + [("▁", -tiny, mp.NORMAL), ("q", tiny, mp.NORMAL), ("z", -1024.0, mp.NORMAL)]
    pcs += [(c, s, mp.NORMAL) for c, s in singles.items()]
    pcs += [(c + "q", next_f32(s + tiny, int(rng.randint(-1, 2))), mp.NORMAL) for c, s in singles.items()]
    pcs += [("q" + c, next_f32(s + tiny, int(rng.randint(-1, 2))), mp.NORMAL) for c, s in singles.items()]
    al = "abcdefghqqz"
    lines = []
    for _ in range(120):
        target = rng.randint(300, 500)  # letters; U+2581 makes the normalized sentence at most LANE_CAP bytes
        ws = []
        while sum(len(w) for w in ws) < target and len(normalize(" ".join(ws).encode())) < LANE_CAP - 40:
            ws.append("".join(rng.choice(list(al), rng.randint(12, 25))))
        lines.append(" ".join(ws).encode())
    return Family("u_boundary", pcs, lines, dict(rounding=200, double_vs_float=50, crosses_2_18=30),
                  doc=u_boundary.__doc__)


def u_boundary_out():
    """As u_boundary with the scores one ulp past the limits (nextafter(2^-10, 0), nextafter(1024, inf)): the model is
    not regular and every NORMAL relaxation takes the double branch."""
    fam = u_boundary()
    tiny_out, big_out = next_f32(2.0 ** -10, -1), next_f32(-1024.0, -1)
    pcs = [(p, (-tiny_out if s == -2.0 ** -10 else tiny_out if s == 2.0 ** -10 else big_out if s == -1024.0 else s), t)
           for p, s, t in fam.pieces]
    return Family("u_boundary_out", pcs, fam.lines, dict(rounding=200, double_vs_float=50, crosses_2_18=30),
                  doc=u_boundary_out.__doc__)


def u_userdef():
    """Positive NORMAL scores (max_score > FLT_MIN) and USER_DEFINED pieces of lengths 1-20, each made of one letter
    whose NORMAL score times the length lands near `length * max_score - 0.1`: the edge's product is rounded in
    float and the subtraction done in double, and a float-only computation reverses some decisions."""
    rng = np.random.RandomState(106)
    M = f32(3.0 + rng.rand())
    pcs = base_pieces() + [("▁", f32(-0.5 - rng.rand()), mp.NORMAL), ("top", M, mp.NORMAL)]
    letters = "abcdefghijklmnopqrst"
    users = []
    for L, c in enumerate(letters, start=1):
        ud = float(F32(F32(L) * F32(M))) - 0.1
        a = next_f32(ud / L, int(rng.randint(-2, 3)))
        pcs.append((c, min(a, M), mp.NORMAL))
        users.append(c * L if L > 1 else "u")  # (a piece is either NORMAL or USER_DEFINED)
    pcs += [(u, 0.0, mp.USER_DEFINED) for u in users]
    lines = []
    for _ in range(300):
        ws = []
        for _ in range(rng.randint(2, 12)):
            c = letters[rng.randint(len(letters))]
            ws.append(c * rng.randint(1, 2 * (letters.index(c) + 1) + 1))
        lines.append(" ".join(ws).encode())
    lines += [u.encode() for u in users] + [" ".join(users).encode(), b"uau aua uuu"]
    return Family("u_userdef", pcs, lines, dict(userdef_float=50), doc=u_userdef.__doc__)


def u_overflow():
    """Scores near -1e38: float path scores overflow to -inf partway through a sentence (the double candidate stays
    finite and is stored as -inf), after which every candidate ties at -inf and the strict `>` keeps the first
    relaxation."""
    rng = np.random.RandomState(107)
    pcs = base_pieces() + [("▁", -1e38, mp.NORMAL)]
    pcs += [(c, f32(-1e38 * (1 + rng.rand())), mp.NORMAL) for c in "abcdef"]
    pcs += [(a + b, f32(-1e38 * (1 + rng.rand())), mp.NORMAL) for a in "abc" for b in "abc"]
    lines = [_line(rng, "abcdefg", 1, 6, rng.randint(1, 12)) for _ in range(400)]
    return Family("u_overflow", pcs, lines, dict(exact_ties=500), doc=u_overflow.__doc__)


NEARWORD_K = [1, 2, 3, 5, 8, 16, 64, 256, 1024, 4096, 1 << 16, 1 << 20]


def u_nearword():
    """A model eligible for the whole-word shortcut (escaped whitespace, no suffix mode, no USER_DEFINED, U+2581 only
    at the front of a piece) whose whole-word pieces U+2581 w score S_P = S_alt + k ulps, S_alt being the exact best
    split of the word, k from 1 ulp to 2^20 ulps.  Each word follows 0-120 other words, so the path score at its
    start takes many magnitudes: some words the reference ends with the piece alone (the shortcut may take them),
    others it splits although S_P > S_alt exactly -- a shortcut without the word_safe rounding bound gets those
    wrong."""
    rng = np.random.RandomState(108)
    al = "abcdefghijklmnopqrstuvwxyz"
    singles = {c: f32(-3.0 - 6.0 * rng.rand()) for c in al}
    pcs = base_pieces() + [("▁", f32(-2.5), mp.NORMAL)] + [(c, s, mp.NORMAL) for c, s in singles.items()]
    pcs += [(w, f32(-4.0 - 8.0 * rng.rand()), mp.NORMAL) for w in sorted(set(_words(rng, al, 2, 3, 60)))]
    um = UnigramModel(pcs)
    targets = sorted(set(_words(rng, al, 3, 8, 48)))
    words = []
    for j, w in enumerate(targets):
        key = WS + w.encode()
        alt = um.exact_best(key, skip=(0, len(key)))
        s = f32(Fraction(alt, SCALE))
        if exact(s) <= alt:
            s = next_f32(s, 1)
        s = next_f32(s, NEARWORD_K[j % len(NEARWORD_K)] - 1)
        assert exact(s) > alt
        pcs.append(("▁" + w, s, mp.NORMAL))
        words.append(key)
    lines = []
    tset = set(targets)
    for rep in range(6):
        for j, w in enumerate(targets):
            npre = (j * 7 + rep * 23) % 121
            pre = [x for x in _words(rng, al, 1, 5, npre) if x not in tset]
            post = [x for x in _words(rng, al, 2, 7, rng.randint(0, 3)) if x not in tset]
            lines.append(" ".join(pre + [w] + post).encode())
    fam = Family("u_nearword", pcs, lines, dict(word_alone=50, word_split=10), doc=u_nearword.__doc__)
    fam.words = words
    return fam


def _bpe(name, score_of, seed, doc):
    rng = np.random.RandomState(seed)
    al = "abcd"
    vocab = [c for c in al] + ["▁"]
    vocab += [a + b for a in al for b in al]
    vocab += ["▁" + c for c in al] + ["▁" + a + b for a in al for b in al[:2]]
    vocab += sorted({w for w in _words(rng, al, 3, 4, 40)})
    whole = sorted({w for w in _words(rng, al, 3, 6, 20)})
    vocab += ["▁" + w for w in whole]
    seen, pcs = set(), base_pieces()
    for i, p in enumerate(vocab):
        if p not in seen:
            seen.add(p)
            pcs.append((p, score_of(i, p, rng), mp.NORMAL))
    lines = [b"aaaa", b"aaaaa aaaaaaa", b"abab ababab abababab", b"a" * 40, b"ab" * 30, b"abcd" * 12]
    for _ in range(300):
        ws = []
        for _ in range(rng.randint(1, 15)):
            r = rng.rand()
            if r < 0.3:
                ws.append(whole[rng.randint(len(whole))])
            elif r < 0.4:
                ws.append("".join(rng.choice(list(al), rng.randint(25, 70))))  # longer than the lane2 word arrays
            elif r < 0.5:
                ws.append(rng.choice(["ab", "aa", "ba"]) * rng.randint(2, 9))
            else:
                ws.append("".join(rng.choice(list(al), rng.randint(1, 9))))
        lines.append(" ".join(ws).encode())
    return Family(name, pcs, lines, dict(bpe_ties=2000, bpe_ties_distinct=500), model_type=mp.BPE, doc=doc)


def b_flat():
    """BPE, every NORMAL piece scored 0: every merge is decided by "leftmost on ties"."""
    return _bpe("b_flat", lambda i, p, rng: 0.0, 201, b_flat.__doc__)


def b_groups():
    """BPE, scores in groups of equal value, 0.0 and -0.0 in the same group: ties between different pieces decided by
    position, and a signed zero that must compare equal."""
    return _bpe("b_groups", lambda i, p, rng: [0.0, -0.0, -1.0, -2.5][rng.randint(4)], 202, b_groups.__doc__)


def b_positive():
    """BPE with some positive scores next to grouped negative ones."""
    return _bpe("b_positive", lambda i, p, rng: [1.5, 1.5, 0.25, -0.0, -3.0][rng.randint(5)], 203, b_positive.__doc__)


UNIGRAM = [u_flat, u_chain, u_round, u_irregular, u_boundary, u_boundary_out, u_userdef, u_overflow, u_nearword]
BPE = [b_flat, b_groups, b_positive]
ALL = UNIGRAM + BPE

_cache = {}


def family(name):
    if name not in _cache:
        _cache[name] = next(f for f in ALL if f.__name__ == name)()
    return _cache[name]
