"""The expected-duration statistics without a GPU: the Python restatements (oracle.expected_durations_for_window,
oracle_durations.window_documents / canonical_stats) against a from-scratch exact reference -- Fraction mean and
variance, an integer square root for the deviation -- on every edge set of duration_edge_cases, and the one
saturating time.Duration(float64) truncation every restatement uses."""
import copy
import math

import numpy as np
import pytest

import duration_edge_cases as E
import oracle_durations as OD
from evergreen_b200 import model as M
from evergreen_b200 import soa as S
from oracle import oracle as O

NOW = 1_800_000_000 * 10 ** 9
SMALL = 5000  # cases up to this many rows also go through the Task-document restatements
ALL = E.CASES + [E.contention_case()]


@pytest.mark.parametrize("case", ALL, ids=[c.name for c in ALL])
def test_canonical_stats_against_exact(case):
    assert case.edge(case), "the case does not reach its edge"
    mean, std = OD.canonical_stats(case.n, case.s, case.s2)
    assert E.close_mean(mean, E.exact_mean(case)), (mean, float(E.exact_mean(case)))
    assert E.close(std, E.exact_std(case)), (std, float(E.exact_std(case)))
    if E.exact_variance(case) == 0:
        assert std == 0.0


def finished_rows(case, project="p", bv="bv", name="n"):
    return [M.Task(id=f"{name}{i}", project=project, build_variant=bv, display_name=name, status="success",
                   time_taken=int(x), start_time=NOW - M.HOUR, finish_time=NOW - M.MINUTE)
            for i, x in enumerate(case.values())]


@pytest.mark.parametrize("case", [c for c in E.CASES if c.n <= SMALL], ids=lambda c: c.name)
def test_restatements_agree_bit_for_bit(case):
    want = OD.canonical_stats(case.n, case.s, case.s2)
    rows = finished_rows(case)
    (n, mean, std, _), = O.expected_durations_for_window(rows, NOW - OD.WINDOW, NOW).values()
    assert (n, mean, std) == (case.n,) + want
    (_, dmean, dstd), = OD.window_documents(rows, "n", "p", "bv", NOW - OD.WINDOW, NOW)
    assert (dmean, dstd) == want


def test_edges_the_rounding_cases_pin():
    """The tie cases land exactly halfway and round to the even neighbour; the case whose low word alone rounds to
    the tie is the one where S2 rounded as hi * 2^64 + lo (twice) goes the wrong way."""
    c = E.by_name(E.CASES)
    assert float(c["sum 2^65 + 2^12: a tie, rounds down to even"].s) == 2.0 ** 65
    assert float(c["sum 2^65 + 3 * 2^12: a tie, rounds up to even"].s) == 2.0 ** 65 + 2.0 ** 14
    assert float(c["sum -(2^65 + 3 * 2^12): a negative tie, rounds to even"].s) == -(2.0 ** 65 + 2.0 ** 14)
    assert float(c["sum 2^65 + 2^12 + 1: just above a tie"].s) == 2.0 ** 65 + 2.0 ** 13
    assert float(c["sum 2^65 + 2^12 - 1: just below a tie"].s) == 2.0 ** 65
    assert float(c["S2 2^128 + 2^75: a tie, rounds down to even"].s2) == 2.0 ** 128
    assert float(c["S2 2^128 + 3 * 2^75: a tie, rounds up to even"].s2) == 2.0 ** 128 + 2.0 ** 77
    s2 = c["S2 2^116 + 2^63 + 1: its low word alone rounds to the tie"].s2
    twice = float(s2 >> 64) * 2.0 ** 64 + float(s2 & (2 ** 64 - 1))
    assert float(s2) == 2.0 ** 116 + 2.0 ** 64 and twice == 2.0 ** 116


EDGES = [  # x, time.Duration(x) under DESIGN.md §3 (iv)
    (2.0 ** 63 - 1024, 2 ** 63 - 1024),  # the largest double below 2^63
    (float(2 ** 63 - 1), 2 ** 63 - 1),   # rounds to 2^63
    (2.0 ** 63, 2 ** 63 - 1),
    (1e300, 2 ** 63 - 1),
    (math.inf, 2 ** 63 - 1),
    (-2.0 ** 63, -2 ** 63),              # fits exactly
    (-2.0 ** 63 - 2.0 ** 11, -2 ** 63),  # the next double below
    (-math.inf, -2 ** 63),
    (math.nan, 0),
    (0.999, 0), (-0.999, 0), (-0.0, 0), (-1.0, -1), (-1.5, -1), (2.5, 2),
]


@pytest.mark.parametrize("x,want", EDGES, ids=[repr(x) for x, _ in EDGES])
def test_duration_from_float_saturates(x, want):
    assert M.duration_from_float(x) == want
    assert OD.duration_from_float_np(np.array([x]))[0] == want


def test_every_restatement_saturates_a_mean_of_2_63():
    """A key of [MAX]: $avg = double(MAX) = 2^63, which no int64 holds.  The model's host route, the oracle's C++
    decision, the Task-document restatement and the numpy restatement all give INT64_MAX."""
    stale = M.CachedDurationValue(0, 0, 0, M.ZERO_TIME)
    t = M.Task(id="t", project="p", build_variant="bv", display_name="n", duration_prediction=stale)
    hist = (2.0 ** 63, 2.0 ** 63)
    assert M.fetch_expected_duration(copy.deepcopy(t), NOW, hist) == (E.I64_MAX, E.I64_MAX)
    assert O.fetch_expected_duration(t, NOW, hist) == (E.I64_MAX, E.I64_MAX)
    finished = finished_rows(E.Multiset("[MAX]", [(E.I64_MAX, 1)], lambda m: True))
    got = OD.fetch_expected_duration(t, NOW, finished)
    assert (got["avg"], got["std"], got["source"]) == (E.I64_MAX, 0, OD.HISTORY)
    hs, codes = S.marshal_duration_history(finished, [t], NOW)
    r = OD.resolve_np(hs.rows, hs.pair_key_off, S.marshal_duration_cache([t], hs), NOW)
    assert (int(r["avg_ns"][0]), int(r["std_ns"][0]), int(r["source"][0])) == (E.I64_MAX, 0, OD.HISTORY)
