"""--chimeras_denovo without a GPU: the case generator reproduces the input digests of
tests/golden/chimeras_denovo_reference.json, and a plain-Python restatement of scan_matches / find_best_parents_long
(core/chimera.cpp:439-624), the selection parents_long_kernel implements, makes the reference's choices on hand-made
match and insert rows: ties, the position that ends a segment, and the doubles of --chimeras_diff_pct 0.3."""
from fractions import Fraction

import numpy as np
import pytest

import chimeras_denovo_cases as D
import uchime_cases as U


@pytest.mark.parametrize("name", sorted(D.CASES))
def test_generator_reproduces_golden_inputs(tmp_path, name):
    q = D.CASES[name][0](str(tmp_path))
    assert U.sha(q) == D.golden()[name]["query_sha256"]


def scan_matches(m, pct):
    """the reference's scan_matches: (start, length) of the first longest window with score sum >= 0, or None"""
    n = len(m)
    p = [0.0] * (n + 1)
    for i in range(n):
        p[i + 1] = p[i] + (pct if m[i] else pct - 100.0)
    q = [0.0] * (n + 1)
    q[n] = p[n]
    for i in range(n - 1, -1, -1):
        q[i] = max(q[i + 1], p[i])
    bi, bd, bc = 0, -1, -1.0
    i = j = 1
    while j <= n:
        c = q[j] - p[i - 1]
        if c >= 0.0:
            if j - i + 1 > bd:
                bi, bd, bc = i, j - i + 1, c
            j += 1
        else:
            i += 1
    return (bi - 1, bd) if bc >= 0.0 else None


def find_best_parents_long(match, insert, parents_max=3, length_min=10, pct=0.0):
    """the reference's find_best_parents_long over rows match[c][p], insert[c][p]: (chimeric, [(cand, start, len)] by start)"""
    qlen = len(match[0]) if match else 0
    used = [False] * qlen
    found = []
    for _ in range(parents_max):
        best = (0, -1, 0)   # len, cand, start
        for c in range(len(match)):
            j = 0
            while j < qlen:
                start, n = j, 0
                while j < qlen and not used[j] and (n == 0 or insert[c][j] == 0):
                    n += 1
                    j += 1
                if n > best[0]:
                    r = scan_matches(match[c][start:start + n], pct)
                    if r is not None and r[1] > best[0]:
                        best = (r[1], c, start + r[0])
                j += 1
        if best[0] < length_min:
            break
        found.append((best[1], best[2], best[0]))
        for p in range(best[2], best[2] + best[0]):
            used[p] = True
    found.sort(key=lambda x: x[1])
    return len(found) > 1 and sum(f[2] for f in found) == qlen, found


def test_scan_matches_longest_first_window():
    assert scan_matches([1] * 8, 0.0) == (0, 8)
    assert scan_matches([0, 1, 1, 0, 1, 1, 1, 0], 0.0) == (4, 3)
    assert scan_matches([1, 1, 0, 1, 1], 0.0) == (0, 2)     # two windows of 2: the first
    assert scan_matches([0, 0], 0.0) == (1, 0)              # nothing matches: an empty window, never chosen
    assert scan_matches([1, 0, 1], 50.0) == (0, 3)          # 50 - 50 + 50 >= 0


def test_scan_matches_diff_pct_03_doubles():
    # one mismatch costs 99.7: 333 matches at 0.3 pay for it (0.2 left), 332 do not (-0.1)
    assert scan_matches([0] + [1] * 333, 0.3) == (0, 334)
    assert scan_matches([0] + [1] * 332, 0.3) == (1, 332)
    assert scan_matches([1] * 200 + [0] + [1] * 133, 0.3) == (0, 334)
    assert scan_matches([1] * 200 + [0] + [1] * 132, 0.3) == (0, 200)


def test_scan_matches_against_exact_brute_force():
    """with diff_pct 0, 1.5 and 50 every prefix sum is exact, so a brute force over fractions must agree"""
    rng = np.random.default_rng(4)
    for pct in (0.0, 1.5, 50.0):
        fp = Fraction(pct)
        for _ in range(300):
            n = int(rng.integers(1, 60))
            m = [int(x) for x in rng.random(n) < rng.uniform(0.5, 1.0)]
            best = None
            for length in range(n, 0, -1):
                for s in range(n - length + 1):
                    if sum(fp if x else fp - 100 for x in m[s:s + length]) >= 0:
                        best = (s, length)
                        break
                if best:
                    break
            got = scan_matches(m, pct)
            assert got == (best if best else (got[0], 0)), (m, pct)


def test_tie_goes_to_the_first_candidate():
    row = [1] * 40
    chim, par = find_best_parents_long([row, row], [[0] * 40, [0] * 40])
    assert par == [(0, 0, 40)] and not chim


def test_tie_in_length_goes_to_lower_candidate_not_lower_start():
    a = [0] * 20 + [1] * 20    # window [20, 40) on candidate 0
    b = [1] * 20 + [0] * 20    # window [0, 20) on candidate 1: same length, earlier start
    chim, par = find_best_parents_long([a, b], [[0] * 40, [0] * 40], length_min=5)
    assert par == [(1, 0, 20), (0, 20, 20)] and chim


def test_position_ending_a_segment_is_skipped():
    """an insert before position 12 ends the segment [0, 12); 12 is skipped, so the next segment is [13, 30), and 12 is
    covered only by a later round that starts a segment there"""
    ins = [0] * 30
    ins[12] = 1
    chim, par = find_best_parents_long([[1] * 30], [ins], length_min=5)
    assert par == [(0, 0, 12), (0, 13, 17)] and not chim
    chim, par = find_best_parents_long([[1] * 30], [ins], length_min=1)
    assert par == [(0, 0, 12), (0, 12, 1), (0, 13, 17)] and chim


def test_insert_after_a_used_position_starts_a_segment():
    m0 = [1] * 20 + [0] * 20
    ins1 = [0] * 40
    ins1[25] = 1
    chim, par = find_best_parents_long([m0, [1] * 40], [[0] * 40, ins1], length_min=3)
    assert par == [(1, 0, 25), (1, 25, 15)] and chim


def test_mismatch_between_windows_leaves_the_query_uncovered():
    m0 = [1] * 12 + [0] + [1] * 17
    chim, par = find_best_parents_long([m0], [[0] * 30], length_min=5)
    assert par == [(0, 0, 12), (0, 13, 17)] and not chim


def test_length_min_stops_the_search():
    m = [1] * 15 + [0] + [1] * 8
    chim, par = find_best_parents_long([m], [[0] * 24], parents_max=5, length_min=9)
    assert par == [(0, 0, 15)] and not chim
