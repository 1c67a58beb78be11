"""pairs_ref: a numpy restatement of spm_encode_pairs_device's semantics as include/spm_b200.h states them, written
from the header and not from the kernels.  It imports no torch, so that CPU tests can check the truncation rules."""
import numpy as np

TRUNCATION = ("none", "longest_first", "only_first", "only_second")


def longest_first_loop(a, b, bt):
    """the rule as the header states it: while a + b > Bt, drop the last id of the longer body, B's on ties"""
    while a + b > bt:
        if a > b:
            a -= 1
        else:
            b -= 1
    return a, b


def longest_first(a, b, bt):
    """the header's closed form of longest_first_loop"""
    a2 = min(a, max(bt - b, -(-bt // 2)))
    return a2, min(b, bt - a2)


def pair_rows(a, b, T, w, truncation, overflow=False, stride=0):
    """The rows of one pair of sizes (a, b) -> (rows, least width): rows is a list of (fa, ca, fb, cb), the first id and
    the count of A and of B each row holds, or None when the pair cannot be laid out at w; the least width is the
    smallest w at which it can (None under longest_first, where every w > T works)."""
    if truncation == "none":
        return ([(0, a, 0, b)] if not w or T + a + b <= w else None), T + a + b
    bt = w - T
    if truncation == "longest_first":
        a2, b2 = longest_first(a, b, bt)
        return [(0, a2, 0, b2)], None
    first = truncation == "only_first"
    L, other = (a, b) if first else (b, a)
    least = T + min(a + b, other + 1 + stride)
    if a + b <= bt:
        return [(0, a, 0, b)], least
    room = bt - other
    if room < 1 or (overflow and room <= stride):
        return None, least
    if not overflow:
        starts, keep = [0], room
    else:
        step = room - stride
        starts, keep = [j * step for j in range(1 + -(-(L - room) // step))], room
    rows = []
    for f in starts:
        c = min(L - f, keep)
        rows.append((f, c, 0, other) if first else (0, other, f, c))
    return rows, least


def pairs_ref(ids, id_offsets, prefix, middle, suffix, w, truncation, overflow=False, stride=0, pad=-1, left=False,
              begin=None, end=None):
    """The pair rows of the 2n packed raw lists ids[id_offsets[k]:id_offsets[k + 1]] (pair i: lists i and n + i) ->
    dict(ids int32 [R, w], lengths, type_ids int32 [R, w], row_pair, row_first int32 [R], spans int64 [R, w, 2] when
    begin / end are given, width w, steps: per pair, the step between its windows or 0), or dict(error="width",
    width=the least width at which every pair passes)."""
    ido = np.asarray(id_offsets, np.int64)
    ids = np.asarray(ids, np.int64)
    if begin is not None:
        begin, end = np.asarray(begin, np.int64), np.asarray(end, np.int64)
    n = (len(ido) - 1) // 2
    prefix, middle, suffix = (list(x) for x in (prefix, middle, suffix))
    T = len(prefix) + len(middle) + len(suffix)
    plans, need, failed = [], 0, False
    for i in range(n):
        a = int(ido[i + 1] - ido[i])
        b = int(ido[n + i + 1] - ido[n + i])
        rows, least = pair_rows(a, b, T, w, truncation, overflow, stride)
        failed |= rows is None
        need = max(need, least or 0)
        plans.append(rows)
    if failed:
        return dict(error="width", width=need)
    if truncation == "none" and not w:
        w = need
    R = sum(len(p) for p in plans)
    out_ids = np.full((R, w), pad, np.int32)
    types = np.zeros((R, w), np.int32)
    spans = np.zeros((R, w, 2), np.int64) if begin is not None else None
    lengths, row_pair, row_first, steps = (np.zeros(R, np.int32), np.zeros(R, np.int32), np.zeros(R, np.int32),
                                           np.zeros(n, np.int64))
    r = 0
    for i, rows in enumerate(plans):
        if len(rows) > 1:
            steps[i] = rows[1][0] if truncation == "only_first" else rows[1][2]
        for fa, ca, fb, cb in rows:
            qa = np.arange(ido[i] + fa, ido[i] + fa + ca)
            qb = np.arange(ido[n + i] + fb, ido[n + i] + fb + cb)
            cell_ids = np.concatenate([prefix, ids[qa], middle, ids[qb], suffix]).astype(np.int32)
            cell_types = np.concatenate([np.zeros(len(prefix) + ca + len(middle), np.int32),
                                         np.ones(cb + len(suffix), np.int32)])
            real = len(cell_ids)
            at = w - real if left else 0
            out_ids[r, at:at + real] = cell_ids
            types[r, at:at + real] = cell_types
            if spans is not None:
                be = np.zeros((real, 2), np.int64)
                a0, b0 = len(prefix), len(prefix) + ca + len(middle)
                be[a0:a0 + ca, 0] = begin[qa]
                be[a0:a0 + ca, 1] = end[qa]
                be[b0:b0 + cb, 0] = begin[qb]
                be[b0:b0 + cb, 1] = end[qb]
                spans[r, at:at + real] = be
            lengths[r] = real
            row_pair[r] = i
            row_first[r] = fa if truncation == "only_first" else fb
            r += 1
    return dict(ids=out_ids, lengths=lengths, type_ids=types, row_pair=row_pair, row_first=row_first, spans=spans,
                width=w, steps=steps)
