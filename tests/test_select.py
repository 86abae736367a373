"""The seeded feature selection's specification on the CPU (tests/select_reference.py): the Philox stream against numpy's, the
equivalence of the reference's shuffle-based selections with the sampler (exhaustively, over every shuffle the reference can
draw), and the size rules of the three selection functions (Estimator.cpp:3894-4116)."""
import itertools
from collections import Counter
from fractions import Fraction
from math import factorial

import numpy as np
import pytest

from tests import select_reference as sr


@pytest.mark.parametrize("seed,domain,stream,nonce", [(0, 0, 0, 0), (1, 2, 3, 4), (2**64 - 1, 1, (7 << 32) | 11, 9),
                                                      (0x0123456789ABCDEF, 2, 2**63 + 5, 2**64 - 2)])
def test_philox_words_equal_numpy(seed, domain, stream, nonce):
    count = 23                                                    # six blocks, the last one partly used
    key = np.array([seed, domain], np.uint64); counter = np.array([0, stream, nonce, 0], np.uint64)
    ref = np.random.Philox(key=key, counter=counter).random_raw(count)
    assert sr.words(seed, domain, stream, nonce, count) == [int(x) for x in ref]


def test_draws_are_mulhi_of_the_words():
    u = sr.words(5, 0, 12, 3, 40)
    r = sr.draws(5, 0, 12, 3, 1000, 40)
    assert r == [(u[j] * (999 - j)) >> 64 for j in range(40)]
    assert all(0 <= r[j] < 999 - j for j in range(40))


# ---- equivalence: the reference's shuffles give exactly the sampler's distribution ------------------------------------------

def _sampler_distribution(n, k):
    """P(ordered sample) when r_j is uniform on [0, n-1-j): every r sequence, each with probability prod 1/(n-1-j)."""
    dist = Counter()
    p = Fraction(1)
    for j in range(k):
        p /= n - 1 - j
    for r in itertools.product(*[range(n - 1 - j) for j in range(k)]):
        dist[tuple(sr.sample_from_draws(n, list(r)))] += p
    return dist


def _window_reference_distribution(n, F, R):
    """featureSelection as written: F times, shuffle 0 .. len(pool)-2 (every permutation), take element R'-1, erase it from the pool."""
    Rp = min(R, n - 1)
    if n - F < Rp:
        Rp = n - F - 1
    assert Rp >= 1
    dist = Counter()

    def walk(pool, kept, p):
        if len(kept) == F:
            dist[tuple(kept)] += p
            return
        perms = list(itertools.permutations(range(len(pool) - 1)))
        picks = Counter(perm[Rp - 1] for perm in perms)           # rand_ids[R'-1] of every shuffle
        for sel, cnt in picks.items():
            walk(pool[:sel] + pool[sel + 1:], kept + [pool[sel]], p * Fraction(cnt, len(perms)))

    walk(list(range(n)), [], Fraction(1))
    return dist


def _batch_reference_distribution(n, B, BR):
    """One pass of the batch selections: rand_ids[0 .. B) of a shuffle of 0 .. n-2 (every permutation)."""
    perms = list(itertools.permutations(range(n - 1)))
    assert BR >= B
    c = Counter(tuple(perm[:B]) for perm in perms)
    return {k: Fraction(v, len(perms)) for k, v in c.items()}


def test_window_reference_equals_sampler_exhaustively():
    checked = 0
    for n in range(3, 7):
        for F in range(1, n - 1):                                 # n - 1 >= F; n = F + 1 is the undefined size
            for R in (1, 2, 3, 300):
                Rp = min(R, n - 1)
                if n - F < Rp:
                    Rp = n - F - 1
                if Rp < 1:
                    continue
                ref = _window_reference_distribution(n, F, R)
                assert ref == _sampler_distribution(n, F), (n, F, R)
                checked += 1
    assert checked >= 20


def test_batch_reference_equals_sampler_exhaustively():
    for n in range(3, 8):
        for B in range(1, n):                                     # n > B: incremental; start/end with BR' >= B
            ref = _batch_reference_distribution(n, B, B)
            assert ref == _sampler_distribution(n, B), (n, B)
            assert sum(ref.values()) == 1 and len(ref) == factorial(n - 1) // factorial(n - 1 - B)


def test_window_oracle_loop_equals_sampler():
    """The transliterated loop (pool, erase) picks sample_from_draws of the same draws."""
    for n in (102, 150, 1000, 100_000):
        keep, undef = sr.window_select(n, stream=17, seed=3, nonce=1)
        assert not undef and len(keep) == 100 and len(set(keep)) == 100 and max(keep) <= n - 2
        assert keep == sr.sample_from_draws(n, sr.draws(3, sr.DOMAIN_WINDOW, 17, 1, n, 100))


# ---- rules -------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,expect", [(0, None), (1, None), (100, None), (101, "undefined"), (102, 100), (301, 100), (5000, 100)])
def test_window_sizes(n, expect):
    keep, undef = sr.window_select(n, stream=4, seed=9, nonce=0)
    if expect is None:
        assert keep is None and not undef
    else:
        assert len(keep) == 100 and max(keep) <= n - 2
        assert undef == (expect == "undefined")


def test_window_without_random_select_keeps_nothing():
    assert sr.window_select(101, 0, 0, 0, random_select=False) == ([], False)
    assert sr.window_select(5000, 0, 0, 0, random_select=False) == ([], False)
    assert sr.window_select(100, 0, 0, 0, random_select=False) == (None, False)     # returns before the loop


def test_window_sample_does_not_depend_on_the_slot():
    a, _ = sr.window_select(3000, stream=41, seed=1, nonce=2)
    b, _ = sr.window_select(3000, stream=41, seed=1, nonce=2)
    c, _ = sr.window_select(3000, stream=42, seed=1, nonce=2)
    assert a == b and a != c


@pytest.mark.parametrize("n,expect", [(0, None), (1, None), (24, None), (25, None), (26, None), (49, None), (50, "undefined"),
                                      (51, 25), (425, 25), (426, 25), (100_000, 25)])
def test_startend_sizes(n, expect):
    (keep, undef), = sr.batch_select([(3, 4)], [n], 0, seed=1, nonce=0)
    if expect is None:
        assert keep is None and not undef
    else:
        assert len(keep) == 25 and len(set(keep)) == 25 and max(keep) <= n - 2 and undef == (expect == "undefined")


@pytest.mark.parametrize("n,expect", [(0, None), (1, None), (24, None), (25, None), (26, 25), (27, 25), (49, 25), (50, 25), (51, 25)])
def test_incremental_sizes(n, expect):
    (keep, undef), = sr.batch_select([(3, 4)], [n], 1, seed=1, nonce=0)
    assert not undef
    assert keep is None if expect is None else (len(keep) == 25 and max(keep) <= n - 2)


def test_return_versus_continue_across_a_run():
    pairs = [(5, 2), (5, 3), (5, 4), (5, 6), (6, 3), (6, 4)]
    n = [500, 40, 500, 500, 500, 500]
    se = sr.batch_select(pairs, n, 0, seed=2, nonce=0)
    assert [k is None for k, _ in se] == [False, True, True, True, False, False]    # return: the rest of keyframe 5's pairs
    inc = sr.batch_select(pairs, n, 1, seed=2, nonce=0)
    assert [k is None for k, _ in inc] == [False, False, False, False, False, False]  # 40 > 25: incremental samples it
    inc = sr.batch_select(pairs, [500, 20, 500, 500, 500, 500], 1, seed=2, nonce=0)
    assert [k is None for k, _ in inc] == [False, True, False, False, False, False]  # continue: only that pair


def test_batch_streams_and_domains_differ():
    (a, _), (b, _) = sr.batch_select([(1, 2), (2, 1)], [1000, 1000], 1, seed=0, nonce=0)
    (c, _), = sr.batch_select([(1, 2)], [1000], 0, seed=0, nonce=0)
    assert a != b and a != c
    assert sr.stream_of_pair(1, 2) == (1 << 32) | 2
