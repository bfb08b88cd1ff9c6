"""Edge sets of the expected-duration statistics ($avg / $stdDevPop of one key's matched TimeTaken), shared by the
host and device tests.  A case is a multiset of int64 values -- (value, count) pairs, so that a key of 2^24 rows has an
exact reference without 2^24 Python integers -- with a plain name and the edge it has to reach.  The exact
statistics come from integers and Fractions; the canonical roundings (include/evg_sched.h) are
oracle_durations.canonical_stats."""
import math
from dataclasses import dataclass
from fractions import Fraction
from typing import Callable, List, Sequence, Tuple

import numpy as np

I64_MAX, I64_MIN = 2 ** 63 - 1, -2 ** 63
H3 = 3 * 3600 * 10 ** 9  # 3 h in ns


@dataclass
class Multiset:
    name: str
    items: List[Tuple[int, int]]  # (value, count)
    edge: Callable[["Multiset"], bool]

    @property
    def n(self) -> int:
        return sum(c for _, c in self.items)

    @property
    def s(self) -> int:
        return sum(v * c for v, c in self.items)

    @property
    def m0(self) -> int:
        return self.s // self.n

    @property
    def s2(self) -> int:
        """S2 = sum (x - floor(mean))^2, exactly."""
        m0 = self.m0
        return sum(c * (v - m0) ** 2 for v, c in self.items)

    def values(self, seed: int = 0) -> np.ndarray:
        """Every row, shuffled (the device adds them in whatever order its threads arrive)."""
        x = np.repeat(np.array([v for v, _ in self.items], np.int64), [c for _, c in self.items])
        np.random.default_rng(seed).shuffle(x)
        return x


def exact_mean(m: Multiset) -> Fraction:
    return Fraction(m.s, m.n)


def exact_variance(m: Multiset) -> Fraction:
    return Fraction(m.n * sum(c * v * v for v, c in m.items) - m.s * m.s, m.n * m.n)


def exact_std(m: Multiset, bits: int = 80) -> Fraction:
    """sqrt(variance) within 2^-bits: an integer square root of the variance scaled by 4^bits, rounded down."""
    v = exact_variance(m)
    return Fraction(math.isqrt(v.numerator * 4 ** bits // v.denominator), 2 ** bits)


def close(got: float, exact: Fraction, ulps: float = 1.0, abs_tol: float = 2.0 ** -20) -> bool:
    """got within `ulps` ulps of the exact value, plus a small absolute term (for results near 0)."""
    return abs(Fraction(got) - exact) <= Fraction(ulps) * Fraction(math.ulp(float(exact))) + Fraction(abs_tol)


def close_mean(got: float, exact: Fraction) -> bool:
    """double(S) / double(n) rounds twice: half an ulp for the division, and |S| 2^-53 / n < one ulp of the mean for
    the conversion of S."""
    return close(got, exact, ulps=1.5)


def is_tie(v: int) -> bool:
    """|v| lies exactly halfway between two neighbouring doubles."""
    v = abs(v)
    k = v.bit_length() - 53
    return k > 0 and v % (1 << k) == 1 << (k - 1)


def s2_rows(target: int) -> List[Tuple[int, int]]:
    """Rows whose S2 is exactly `target`: a row of 1 when the target is odd, then pairs (u, -u).  The sum is 0 or 1
    over at least two rows, so floor(mean) = 0 and S2 = sum x^2."""
    items = [(1, 1)] if target & 1 else []
    r = target - (target & 1)
    while r:
        u = min(math.isqrt(r // 2), I64_MAX)
        items += [(u, 1), (-u, 1)]
        r -= 2 * u * u
    return items if len(items) > 1 else items + [(0, 1), (0, 1)]


def sum_tie(s: int) -> List[Tuple[int, int]]:
    """Four rows of MAX (MIN for a negative s) and one row that brings the sum to exactly s."""
    base = I64_MAX if s > 0 else I64_MIN
    return [(base, 4), (s - 4 * base, 1)]


def _beyond_int64(m: Multiset) -> bool:
    return not I64_MIN <= m.s <= I64_MAX


def _dev_ge_2_63(m: Multiset) -> bool:
    return max(abs(v - m.m0) for v, _ in m.items) >= 2 ** 63


def _s2_ge_2_128(m: Multiset) -> bool:
    return m.s2 >= 2 ** 128


def _negative_floor(mod_zero: bool):
    return lambda m: m.s < 0 and (m.s % m.n == 0) == mod_zero


def _zero_variance(m: Multiset) -> bool:
    return exact_variance(m) == 0 and len({v for v, _ in m.items}) == 1


def _smallest_positive_variance(m: Multiset) -> bool:
    # the least variance a key of n integers can have without being constant: (n - 1) / n^2
    return exact_variance(m) == Fraction(m.n - 1, m.n * m.n)


def _sum_tie(m: Multiset) -> bool:
    return abs(m.s) > 2 ** 64 and is_tie(m.s)


def _s2_tie(lo: int):
    return lambda m: m.s2 > lo and is_tie(m.s2)


T65, T116, T128 = 2 ** 65, 2 ** 116, 2 ** 128
SUM_ULP_65 = 2 ** 13  # the spacing of doubles in [2^65, 2^66)

CASES: List[Multiset] = [
    # sums beyond int64, both signs
    Multiset("2^20 rows of 3 h and one of 1 ns", [(H3, 2 ** 20), (1, 1)], _beyond_int64),
    Multiset("[MAX, MAX]", [(I64_MAX, 2)], _beyond_int64),
    Multiset("[MIN, -1]", [(I64_MIN, 1), (-1, 1)], _beyond_int64),
    Multiset("[MIN, MIN, MIN]", [(I64_MIN, 3)], _beyond_int64),
    Multiset("2^20 rows of -3 h", [(-H3, 2 ** 20)], _beyond_int64),
    # |x - floor(mean)| >= 2^63
    Multiset("[MAX, MIN, MIN]", [(I64_MAX, 1), (I64_MIN, 2)], _dev_ge_2_63),
    Multiset("[MIN, MAX, MAX]", [(I64_MIN, 1), (I64_MAX, 2)], _dev_ge_2_63),
    # S2 >= 2^128
    Multiset("[MIN, MAX] x 2", [(I64_MIN, 2), (I64_MAX, 2)],  # S2 = 2^128 - 2^65 + 2, one pair short of 2^128
             lambda m: _dev_ge_2_63(m) and 2 ** 127 < m.s2 < 2 ** 128),
    Multiset("[MIN, MAX] x 3", [(I64_MIN, 3), (I64_MAX, 3)], _s2_ge_2_128),
    Multiset("[MIN, MAX] x 4", [(I64_MIN, 4), (I64_MAX, 4)], _s2_ge_2_128),
    Multiset("[MIN, MAX] x 64", [(I64_MIN, 64), (I64_MAX, 64)], _s2_ge_2_128),
    Multiset("[MIN, MAX] x 2^16", [(I64_MIN, 2 ** 16), (I64_MAX, 2 ** 16)], _s2_ge_2_128),
    # floor(mean) of negative sums, n = 1 .. 5
    Multiset("[-1]", [(-1, 1)], _negative_floor(True)),
    Multiset("[-1, -2]", [(-1, 1), (-2, 1)], _negative_floor(False)),
    Multiset("[-1, -3]", [(-1, 1), (-3, 1)], _negative_floor(True)),
    Multiset("[-1, 0, 0]", [(-1, 1), (0, 2)], _negative_floor(False)),
    Multiset("[-3, 0, 0]", [(-3, 1), (0, 2)], _negative_floor(True)),
    Multiset("[-5, 0, 0, 0]", [(-5, 1), (0, 3)], _negative_floor(False)),
    Multiset("[-8, 0, 0, 0]", [(-8, 1), (0, 3)], _negative_floor(True)),
    Multiset("[-7, 0, 0, 0, 0]", [(-7, 1), (0, 4)], _negative_floor(False)),
    Multiset("[-10, -5, 0, 0, 0]", [(-10, 1), (-5, 1), (0, 3)], _negative_floor(True)),
    # variance that cancels: exactly 0, and the least positive variance of n rows
    Multiset("7 rows of 5", [(5, 7)], _zero_variance),
    Multiset("3 rows of MIN", [(I64_MIN, 3)], _zero_variance),
    Multiset("3 rows of MAX", [(I64_MAX, 3)], _zero_variance),
    Multiset("2^20 rows of MIN", [(I64_MIN, 2 ** 20)], _zero_variance),
    Multiset("[0, 1]", [(0, 1), (1, 1)], _smallest_positive_variance),
    Multiset("2^20 - 1 rows of 0 and one of -1", [(0, 2 ** 20 - 1), (-1, 1)], _smallest_positive_variance),
    Multiset("2^20 - 1 rows of MAX and one of MAX - 1", [(I64_MAX, 2 ** 20 - 1), (I64_MAX - 1, 1)],
             _smallest_positive_variance),
    Multiset("2^20 - 1 rows of MIN and one of MIN + 1", [(I64_MIN, 2 ** 20 - 1), (I64_MIN + 1, 1)],
             _smallest_positive_variance),
    # round-to-nearest-even: sums halfway between two doubles above 2^64 (even and odd significands, both signs), and
    # just above / below a tie, where only the bits under the leading 64 decide
    Multiset("sum 2^65 + 2^12: a tie, rounds down to even", sum_tie(T65 + SUM_ULP_65 // 2), _sum_tie),
    Multiset("sum 2^65 + 3 * 2^12: a tie, rounds up to even", sum_tie(T65 + 3 * SUM_ULP_65 // 2), _sum_tie),
    Multiset("sum -(2^65 + 3 * 2^12): a negative tie, rounds to even", sum_tie(-(T65 + 3 * SUM_ULP_65 // 2)), _sum_tie),
    Multiset("sum 2^65 + 2^12 + 1: just above a tie", sum_tie(T65 + SUM_ULP_65 // 2 + 1),
             lambda m: m.s - 1 > 2 ** 64 and is_tie(m.s - 1)),
    Multiset("sum 2^65 + 2^12 - 1: just below a tie", sum_tie(T65 + SUM_ULP_65 // 2 - 1),
             lambda m: m.s + 1 > 2 ** 64 and is_tie(m.s + 1)),
    # ... and S2 halfway above 2^128 and above 2^64 (where hi * 2^64 + lo rounded twice would go wrong)
    Multiset("S2 2^128 + 2^75: a tie, rounds down to even", s2_rows(T128 + 2 ** 75), _s2_tie(T128)),
    Multiset("S2 2^128 + 3 * 2^75: a tie, rounds up to even", s2_rows(T128 + 3 * 2 ** 75), _s2_tie(T128)),
    Multiset("S2 2^128 + 2^75 + 1: just above a tie", s2_rows(T128 + 2 ** 75 + 1),
             lambda m: m.s2 > T128 and is_tie(m.s2 - 1)),
    Multiset("S2 2^116 + 2^63: a tie above 2^64", s2_rows(T116 + 2 ** 63), _s2_tie(2 ** 64)),
    Multiset("S2 2^116 + 2^63 + 1: its low word alone rounds to the tie", s2_rows(T116 + 2 ** 63 + 1),
             lambda m: m.s2 > 2 ** 64 and is_tie(m.s2 - 1) and float(m.s2 & (2 ** 64 - 1)) == 2.0 ** 63),
]


def contention_case(seed: int = 7, n: int = 2 ** 24) -> Multiset:
    """One key of n rows over a palette of both signs and every magnitude: the shuffled rows make the carries of the
    128-bit sum and the 192-bit S2 fire from many threads at once."""
    rng = np.random.default_rng(seed)
    palette = [I64_MAX, I64_MIN, I64_MAX - 1, I64_MIN + 1, 2 ** 62 + 12345, -2 ** 62 - 54321, H3, -H3, 1, -1, 0,
               2 ** 32, -2 ** 32 - 1] + [int(v) for v in rng.integers(I64_MIN, I64_MAX, 19, dtype=np.int64, endpoint=True)]
    w = rng.random(len(palette))
    counts = np.floor(w / w.sum() * n).astype(np.int64)
    counts[0] += n - int(counts.sum())
    return Multiset(f"2^{n.bit_length() - 1} rows of mixed signs and magnitudes",
                    [(v, int(c)) for v, c in zip(palette, counts)],
                    lambda m: _beyond_int64(m) or _s2_ge_2_128(m))


def by_name(cases: Sequence[Multiset]) -> dict:
    return {c.name: c for c in cases}
