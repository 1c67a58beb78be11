"""pairs_ref's truncation rules on the CPU: the closed form of longest-first equals the rule it restates, one id at a
time, and the windows of one member cover it with the stated room and step."""
from pairs_ref import longest_first, longest_first_loop, pair_rows


def test_longest_first_closed_form():
    for bt in range(1, 40):
        for a in range(60):
            for b in range(60):
                assert longest_first(a, b, bt) == longest_first_loop(a, b, bt), (a, b, bt)


def test_overflow_windows_cover_the_member():
    T, w = 3, 20
    for stride in (0, 4, 9):
        for other in range(0, 10):
            for L in range(0, 80):
                rows, least = pair_rows(other, L, T, w, "only_second", True, stride)
                room = w - T - other
                if other + L > w - T and room <= stride:
                    assert rows is None and least > w
                    continue
                assert least <= w
                firsts = [r[2] for r in rows]
                assert all(r[:2] == (0, other) for r in rows)
                assert firsts[0] == 0 and (len(rows) == 1 or firsts[1] == room - stride)
                covered = set()
                for _, _, f, c in rows:
                    assert 1 <= c <= room or L == 0
                    covered |= set(range(f, f + c))
                assert covered == set(range(L))
                assert rows[-1][2] + rows[-1][3] == L
