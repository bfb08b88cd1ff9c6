"""The expected-duration statistics on the device at int64 and 128-bit edges: every edge set of duration_edge_cases
through evg_expected_durations_batch, bit for bit against the canonical roundings of the oracle and within one ulp
of the exact Fraction / integer-square-root values, and then through evg_resolve_durations on a resident tick, where
the statistics become the planner's expected durations.  Also the $match window at its bounds, the saturating
truncation in k_dur_resolve, its TTL and clock edges, and the pair keys of an empty DisplayName."""
import struct

import numpy as np
import pytest

import duration_edge_cases as E
import oracle_durations as OD
from evergreen_b200 import model as M
from evergreen_b200 import soa as S
from evergreen_b200 import synth

pytestmark = pytest.mark.gpu

NOW = synth.NOW_NS
FIELDS = ("avg_ns", "std_ns", "value_ns", "pred_std_ns", "collected_ns", "source")
NEIGHBOUR = [7 * M.MINUTE, 9 * M.MINUTE, 9 * M.MINUTE]  # key 0 of every call: a plain key beside the edge case


def bits(x: float) -> int:
    return struct.unpack("<q", struct.pack("<d", float(x)))[0]


def rows_of(keys, values, n_keys, start=1, finish=2, flags=1, w0=0, w1=10):
    n = len(values)
    col = lambda v: np.broadcast_to(np.asarray(v, np.int64), (n,)).copy()  # noqa: E731
    return S.DurationRows(np.asarray(keys, np.int32), np.asarray(values, np.int64), col(start), col(finish),
                          np.broadcast_to(np.asarray(flags, np.uint8), (n,)).copy(), n_keys, w0, w1)


def case_rows(case, seed=0):
    """Key 0: NEIGHBOUR; key 1: the case's rows, shuffled among key 0's; key 2: no rows."""
    x = np.concatenate([np.array(NEIGHBOUR, np.int64), case.values(seed)])
    k = np.concatenate([np.zeros(len(NEIGHBOUR), np.int32), np.ones(case.n, np.int32)])
    p = np.random.default_rng(seed + 1).permutation(x.shape[0])
    return rows_of(k[p], x[p], 3)


def want_stats(case):
    return (case.n,) + OD.canonical_stats(case.n, case.s, case.s2)


NEIGHBOUR_CASE = E.Multiset("neighbour", [(v, NEIGHBOUR.count(v)) for v in sorted(set(NEIGHBOUR))], lambda m: True)


def assert_stat(st, want, case=None):
    n, mean, std = want
    assert int(st["count"]) == n
    assert (bits(st["mean_ns"]), bits(st["stddev_ns"])) == (bits(mean), bits(std)), \
        (float(st["mean_ns"]), float(st["stddev_ns"]), mean, std)
    if case is not None:
        assert E.close_mean(float(st["mean_ns"]), E.exact_mean(case))
        assert E.close(float(st["stddev_ns"]), E.exact_std(case))


def upload_tick(engine, n):
    tasks = [M.Task(id=f"t{i}", activated_time=NOW - M.HOUR) for i in range(n)]
    soa, table, _ = S.marshal_tasks([(M.Distro(id="d"), tasks)], NOW, resolve_durations=False)
    soa.expected_ns[:] = -12345
    engine.upload(soa, table)


def stale_cache(keys, **cols):
    """Listed rows 0 .. n-1 with no cached value (so the refresher runs) unless `cols` says otherwise."""
    n = len(keys)
    c = {f: np.zeros(n, np.int64) for f in ("value_ns", "std_ns", "ttl_ns", "expected_ns", "expected_std_ns")}
    c["collected_ns"] = np.full(n, M.ZERO_TIME, np.int64)
    for f, v in cols.items():
        c[f] = np.asarray(v, np.int64)
    return S.DurationCache(c["value_ns"], c["std_ns"], c["ttl_ns"], c["collected_ns"], c["expected_ns"],
                           c["expected_std_ns"], np.asarray(keys, np.int32)).normalize()


def refreshed(count, mean, std, now=NOW):
    """A stale row without a cached value against a key's statistics: FetchExpectedDuration's refresher with
    time.Duration(float64) saturating (DESIGN.md §3 (iv))."""
    if count == 0:
        avg, sd, src = M.DEFAULT_TASK_DURATION, 0, OD.DEFAULT
    else:
        a = M.duration_from_float(mean)
        avg, sd, src = (M.DEFAULT_TASK_DURATION, 0, OD.DEFAULT) if a == 0 else (a, M.duration_from_float(std), OD.HISTORY)
    return dict(avg_ns=avg, std_ns=sd, value_ns=avg, pred_std_ns=sd, collected_ns=now, source=src)


def resolve(engine, rows, cache, now=NOW, n_tasks=None):
    upload_tick(engine, n_tasks or cache.n_rows)
    hist = S.DurationHistory(rows, np.array([0, rows.n_keys], np.int64), [], {}, {})
    engine.resolve_durations(hist, now, cache)
    got, _ = engine.download_durations()
    return [{f: int(got[f][i]) for f in FIELDS} for i in range(cache.n_rows)]


def check_case(engine, case, seed=0):
    assert case.edge(case), "the case does not reach its edge"
    rows = case_rows(case, seed)
    st = engine.expected_durations_batch(rows).copy()
    want = want_stats(case)
    assert_stat(st[1], want, case)
    assert_stat(st[0], want_stats(NEIGHBOUR_CASE), NEIGHBOUR_CASE)
    assert_stat(st[2], (0, 0.0, 0.0))
    got = resolve(engine, rows, stale_cache([0, 1, 2]))
    assert got == [refreshed(*want_stats(NEIGHBOUR_CASE)), refreshed(*want), refreshed(0, 0.0, 0.0)]
    return st[1], got[1]


@pytest.mark.parametrize("case", E.CASES, ids=[c.name for c in E.CASES])
def test_edge_case(engine, case):
    check_case(engine, case)


def test_one_key_of_2_24_rows_under_contention(engine):
    case = E.contention_case()
    assert case.n == 2 ** 24
    check_case(engine, case, seed=11)


def test_2_22_keys_most_of_them_empty(engine):
    rng = np.random.default_rng(22)
    K = 2 ** 22
    used = rng.choice(K, 700, replace=False)
    palette = np.array([E.I64_MAX, E.I64_MIN, E.I64_MAX - 1, E.I64_MIN + 1, -E.H3, E.H3, -1, 0, 1], np.int64)
    n = 40_000
    keys = used[rng.integers(0, used.shape[0], n)].astype(np.int32)
    x = palette[rng.integers(0, palette.shape[0], n)]
    flags = rng.choice(np.array([1, 1, 1, 3, 0], np.uint8), n)
    rows = rows_of(keys, x, K, flags=flags)
    st = engine.expected_durations_batch(rows)
    ok = flags == 1
    groups = {}
    for k, v in zip(keys[ok].tolist(), x[ok].tolist()):
        groups.setdefault(k, []).append(v)
    cnt = np.zeros(K, np.int64)
    cnt[list(groups)] = [len(v) for v in groups.values()]
    assert np.array_equal(st["count"], cnt)
    empty = cnt == 0
    assert empty.sum() >= K - 700 and np.all(st["mean_ns"][empty] == 0.0) and np.all(st["stddev_ns"][empty] == 0.0)
    wraps = 0
    for k, xs in groups.items():
        m = E.Multiset(f"key {k}", [(v, xs.count(v)) for v in set(xs)], lambda m: True)
        wraps += not E.I64_MIN <= m.s <= E.I64_MAX
        assert_stat(st[k], want_stats(m), m)
    assert wraps > 50  # many keys sum beyond int64


# ---- the $match window ------------------------------------------------------------------------------------------------
def test_match_window_bounds(engine):
    w0, w1 = 1000, 2000
    # one row per key: (start, finish, flags, matched)
    spec = [(w0, 1500, 1, False), (w0 + 1, 1500, 1, True), (1500, w1, 1, True), (1500, w1 + 1, 1, False),
            (1500, 1500, 0xFD, True), (1500, 1500, 0xFF, False), (1500, 1500, 0xFC, False), (1500, 1500, 0x81, True)]
    x = [(k + 1) * M.MINUTE for k in range(len(spec))]
    rows = rows_of(range(len(spec)), x, len(spec), [s[0] for s in spec], [s[1] for s in spec], [s[2] for s in spec], w0, w1)
    st = engine.expected_durations_batch(rows).copy()
    assert st["count"].tolist() == [int(s[3]) for s in spec]
    assert st["mean_ns"].tolist() == [float(v) if s[3] else 0.0 for v, s in zip(x, spec)]
    got = resolve(engine, rows, stale_cache(range(len(spec))))
    assert got == [refreshed(int(s[3]), float(v), 0.0) for v, s in zip(x, spec)]
    # the widest window: StartTime > INT64_MIN excludes only INT64_MIN, FinishTime <= INT64_MAX admits everything
    lo, hi = E.I64_MIN, E.I64_MAX
    rows = rows_of([0, 1, 2], [M.MINUTE, 2 * M.MINUTE, 3 * M.MINUTE], 3, [lo, lo + 1, hi], [hi, hi, hi], 1, lo, hi)
    st = engine.expected_durations_batch(rows).copy()
    assert st["count"].tolist() == [0, 1, 1]


# ---- the truncation in k_dur_resolve ------------------------------------------------------------------------------------
TRUNCATIONS = [  # (case, avg_ns, std_ns, source)
    (E.Multiset("[MAX]: a mean of exactly 2^63 saturates", [(E.I64_MAX, 1)], lambda m: float(m.s) == 2.0 ** 63),
     E.I64_MAX, 0, OD.HISTORY),
    (E.Multiset("[MAX, MAX]: a mean of 2^63 from a sum beyond int64", [(E.I64_MAX, 2)], lambda m: m.s > E.I64_MAX),
     E.I64_MAX, 0, OD.HISTORY),
    (E.Multiset("[MIN, MAX - 500]: a deviation that rounds to 2^63 saturates, the mean -250.5 truncates to -250",
                [(E.I64_MIN, 1), (E.I64_MAX - 500, 1)], lambda m: OD.canonical_stats(m.n, m.s, m.s2)[1] == 2.0 ** 63),
     -250, E.I64_MAX, OD.HISTORY),
    (E.Multiset("[MIN, MIN]: a mean of exactly -2^63 fits", [(E.I64_MIN, 2)], lambda m: m.s < E.I64_MIN),
     E.I64_MIN, 0, OD.HISTORY),
    (E.Multiset("[MIN, MAX]: a mean of -0.5 truncates to 0", [(E.I64_MIN, 1), (E.I64_MAX, 1)], lambda m: 2 * m.s == -m.n),
     M.DEFAULT_TASK_DURATION, 0, OD.DEFAULT),
    (E.Multiset("[0, 1]: a mean of 0.5 truncates to 0", [(0, 1), (1, 1)], lambda m: 2 * m.s == m.n),
     M.DEFAULT_TASK_DURATION, 0, OD.DEFAULT),
    (E.Multiset("[-1, 0, 0]: a mean of -1/3 truncates to 0", [(-1, 1), (0, 2)], lambda m: 3 * m.s == -m.n),
     M.DEFAULT_TASK_DURATION, 0, OD.DEFAULT),
    (E.Multiset("[-1, -2]: a mean of -1.5 truncates to -1", [(-1, 1), (-2, 1)], lambda m: 2 * m.s == -3 * m.n),
     -1, 0, OD.HISTORY),
    (E.Multiset("[-5 min]: a negative average, as Go returns it", [(-5 * M.MINUTE, 1)], lambda m: m.s < 0),
     -5 * M.MINUTE, 0, OD.HISTORY),
]


@pytest.mark.parametrize("case,avg,std,src", TRUNCATIONS, ids=[t[0].name for t in TRUNCATIONS])
def test_truncation_in_resolve(engine, case, avg, std, src):
    _, got = check_case(engine, case)
    assert (got["avg_ns"], got["std_ns"], got["source"]) == (avg, std, src)


# ---- TTL and clock edges ------------------------------------------------------------------------------------------------
def finished_docs(project, bv, name, values, now=NOW, **kw):
    return [M.Task(id=f"{project}/{bv}/{name}/{i}", project=project, build_variant=bv, display_name=name,
                   status=kw.get("status", "success"), timed_out=kw.get("timed_out", False), time_taken=int(v),
                   start_time=now - M.HOUR, finish_time=now - M.MINUTE) for i, v in enumerate(values)]


def task(name, value=0, std=0, ttl=0, coll=M.ZERO_TIME, exp=0, project="p", bv="bv"):
    return M.Task(id=f"q-{name}-{value}-{ttl}-{coll}", project=project, build_variant=bv, display_name=name,
                  expected_duration=exp, duration_prediction=M.CachedDurationValue(value, std, ttl, coll))


def run_documents(engine, tasks, finished, now=NOW):
    """The tasks resolved on the device against the finished documents, and FetchExpectedDuration restated over the
    same documents (tests/oracle_durations.py)."""
    hist, codes = S.marshal_duration_history(finished, tasks, now)
    upload_tick(engine, len(tasks))
    engine.resolve_durations(hist, now, S.marshal_duration_cache(tasks, hist))
    got, _ = engine.download_durations()
    want = [OD.fetch_expected_duration(t, now, finished) for t in tasks]
    return [{f: int(got[f][i]) for f in FIELDS} for i in range(len(tasks))], \
        [dict(avg_ns=w["avg"], std_ns=w["std"], value_ns=w["value"], pred_std_ns=w["pred_std"],
              collected_ns=w["collected"], source=w["source"]) for w in want], codes


def test_ttl_and_clock_edges(engine):
    v, sd, H = 7 * M.MINUTE, M.MINUTE, M.HOUR
    for now, rows in (
            (NOW, [  # (ttl, collected, fresh?)
                (H, NOW - H, False),                  # since == ttl is stale
                (H, NOW - H + 1, True),
                (-5 * M.MINUTE, NOW, False),          # a negative TTL: only a collection in the future is fresh
                (-5 * M.MINUTE, NOW + 10 * M.MINUTE, True),
                (E.I64_MAX, M.ZERO_TIME, False),      # the zero time is infinitely old, even for the longest TTL
                (E.I64_MAX, E.I64_MIN + 1, False),    # now - collected beyond int64: since saturates at INT64_MAX
                (E.I64_MAX, NOW - 1, True),
                (0, NOW + H, True),                   # collected in the future
                (0, NOW - 8 * H, False),              # an unset TTL reads as 8 h
            ]),
            (-2 ** 62, [  # a clock before the epoch: since(now, INT64_MAX) saturates at INT64_MIN
                (E.I64_MIN + 1, E.I64_MAX, True),
                (E.I64_MIN, E.I64_MAX, False),
                (0, E.I64_MAX, True),
            ])):
        finished = finished_docs("p", "bv", "n", [20 * M.MINUTE, 21 * M.MINUTE], now)
        tasks = [task("n", v, sd, ttl, coll) for ttl, coll, _ in rows]
        got, want, _ = run_documents(engine, tasks, finished, now)
        assert got == want
        assert [g["source"] for g in got] == [OD.FRESH if f else OD.HISTORY for _, _, f in rows]


# ---- pair keys: DisplayName "" ------------------------------------------------------------------------------------------
def test_pair_keys(engine):
    finished = (finished_docs("one", "bv", "a", [10 * M.MINUTE, 12 * M.MINUTE]) +
                finished_docs("one", "bv", "b", [M.HOUR], timed_out=True) +
                finished_docs("zero", "bv", "a", [0, 1]) +
                finished_docs("zero", "bv", "b", [M.HOUR], status="started") +
                finished_docs("two", "bv", "a", [M.MINUTE]) + finished_docs("two", "bv", "b", [2 * M.MINUTE]) +
                finished_docs("wrap", "bv", "a", [E.I64_MAX, E.I64_MAX]))
    tasks = [task("", project="one"), task("", project="zero"), task("", project="two"),
             task("", value=3 * M.MINUTE, project="two"), task("", project="wrap")]
    got, want, codes = run_documents(engine, tasks, finished)
    assert all(c <= -2 for c in codes)
    assert got == want
    assert [g["source"] for g in got] == [OD.HISTORY, OD.DEFAULT, OD.DEFAULT, OD.PREVIOUS, OD.HISTORY]
    assert got[0]["avg_ns"] == 11 * M.MINUTE and got[4]["avg_ns"] == E.I64_MAX
