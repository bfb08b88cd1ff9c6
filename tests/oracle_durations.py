"""Restatement of Task.FetchExpectedDuration (model/task/task.go:3519-3590) with CachedDurationValue.Get
(util/cached_value.go:125-145) and the window query getExpectedDurationsForWindow (model/task/expected_duration.go:36-96)
over Task documents, with the clock frozen at `now`.

The window query is restated with its name filter: DisplayName "" drops it (expected_duration.go:54-56), and the
$group by name then returns one document per matched name of the (project, build variant); the refresher uses the
statistics only when exactly one document comes back (task.go:3556).  $avg / $stdDevPop use the canonical roundings of
include/evg_sched.h (double(sum) / double(n); the population variance accumulated exactly around floor(mean)).  The
TTL jitter is not drawn: an unset TTL reads as predictionTTL.  Only test code uses this module.
"""
import math
from typing import Dict, List, Sequence

from evergreen_b200 import model as M

WINDOW = 7 * 24 * M.HOUR  # taskCompletionEstimateWindow, task.go:60
FRESH, BACKFILL, HISTORY, PREVIOUS, DEFAULT = 0, 1, 2, 3, 4
I64_MAX = 2 ** 63 - 1


def since(now: int, t: int) -> int:
    """time.Since with a frozen clock: time.Time.Sub saturates, and the zero time is infinitely long ago."""
    if t == M.ZERO_TIME:
        return I64_MAX
    return max(min(now - t, I64_MAX), -I64_MAX - 1)


def window_documents(finished: Sequence[M.Task], name: str, project: str, build_variant: str, start: int, end: int):
    """getExpectedDurationsForWindow: [(display name, $avg, $stdDevPop)], one per matched name, in first-match order."""
    groups: Dict[str, List[int]] = {}
    for t in finished:
        if t.build_variant != build_variant or t.project != project:
            continue
        if t.status not in M.TASK_COMPLETED_STATUSES or t.timed_out:
            continue
        if not (t.start_time > start and t.finish_time <= end):
            continue
        if name != "" and t.display_name != name:
            continue
        groups.setdefault(t.display_name, []).append(t.time_taken)
    out = []
    for n, xs in groups.items():
        k, s = len(xs), sum(xs)
        m0 = s // k
        s2 = sum((x - m0) ** 2 for x in xs)
        out.append((n,) + canonical_stats(k, s, s2))
    return out


def canonical_stats(n: int, s: int, s2: int):
    """($avg, $stdDevPop) of a key from its exact count n, sum s and S2 = sum (x - floor(s/n))^2, with the roundings
    of include/evg_sched.h: float(s) and float(s2) are each one round-to-nearest-even of the exact integer."""
    rem = s - n * (s // n)
    fr = float(rem) / float(n)
    return float(s) / float(n), math.sqrt(max(float(s2) / float(n) - fr * fr, 0.0))


def fetch_expected_duration(t: M.Task, now: int, finished: Sequence[M.Task]) -> dict:
    """-> dict(avg, std, value, pred_std, collected, ttl, source, persisted); `t` is not modified."""
    p = t.duration_prediction
    ttl = p.ttl if p.ttl != 0 else M.PREDICTION_TTL  # task.go:3520-3522
    value, pstd, coll = p.value, p.std_dev, p.collected_at
    if value == 0 and t.expected_duration != 0:  # backfill, task.go:3524-3538
        avg, std, source = t.expected_duration, t.expected_duration_std_dev, BACKFILL
        value, coll = t.expected_duration, now - M.MINUTE
    elif since(now, coll) < ttl:  # cached_value.go:127-129
        avg, std, source = value, pstd, FRESH
    else:  # the refresher, task.go:3540-3574; ok is always true without a DB error
        docs = window_documents(finished, t.display_name, t.project, t.build_variant, now - WINDOW, now)
        if len(docs) != 1:
            source = DEFAULT if value == 0 else PREVIOUS
            avg, std = (M.DEFAULT_TASK_DURATION, 0) if value == 0 else (value, pstd)
        else:
            a = M.duration_from_float(docs[0][1])  # time.Duration(float64): truncation toward zero, saturated
            source = DEFAULT if a == 0 else HISTORY
            avg, std = (M.DEFAULT_TASK_DURATION, 0) if a == 0 else (a, M.duration_from_float(docs[0][2]))
        value, pstd, coll = avg, std, now  # cached_value.go:139-142
    return dict(avg=avg, std=std, value=value, pred_std=pstd, collected=coll, ttl=ttl, source=source,
                persisted=source != FRESH)


# ---- tests/golden/duration_cache.json -> model objects
def golden_task(d: dict, tid: str = "t") -> M.Task:
    p = d["prediction"]
    return M.Task(id=tid, project=d["project"], build_variant=d["build_variant"], display_name=d["display_name"],
                  expected_duration=d["expected_duration"], expected_duration_std_dev=d["expected_duration_std_dev"],
                  duration_prediction=M.CachedDurationValue(
                      value=p["value"], std_dev=p["std_dev"], ttl=p["ttl"],
                      collected_at=M.ZERO_TIME if p["collected_at"] is None else p["collected_at"]))


def golden_finished(rows: Sequence[dict], prefix: str = "f") -> List[M.Task]:
    return [M.Task(id=f"{prefix}{i}", **r) for i, r in enumerate(rows)]


# ---- numpy restatement of evg_resolve_durations over marshalled columns (scale tests)
def key_stats_np(rows):
    """Per key of a DurationRows: (count, mean_ns, stddev_ns) with the roundings of k_dur_final.  Exact as long as
    every matched TimeTaken lies within 2^20 ns of its key's floor(mean) times a few (synth.make_duration_cache)."""
    import numpy as np
    K = int(rows.n_keys)
    f = rows.flags
    m = ((f & 1) != 0) & ((f & 2) == 0) & (rows.start_ns > rows.window_start_ns) & (rows.finish_ns <= rows.window_end_ns)
    k, x = rows.key[m].astype(np.int64), rows.time_taken_ns[m].astype(np.int64)
    order = np.argsort(k, kind="stable")
    k, x = k[order], x[order]
    cnt = np.bincount(k, minlength=K).astype(np.int64)
    starts = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    has = cnt > 0
    s = np.zeros(K, np.int64)
    if x.shape[0]:
        s[has] = np.add.reduceat(x, starts[has])
    n1 = np.maximum(cnt, 1)
    m0 = np.floor_divide(s, n1)
    rem = s - m0 * n1
    dv = x - np.repeat(m0, cnt)
    assert np.all(np.abs(dv) < 2 ** 21)  # dv * dv summed over 2^20 rows stays below 2^63
    s2 = np.zeros(K, np.int64)
    if x.shape[0]:
        s2[has] = np.add.reduceat(dv * dv, starts[has])
    mean = s.astype(np.float64) / n1.astype(np.float64)
    fr = rem.astype(np.float64) / n1.astype(np.float64)
    var = np.maximum(s2.astype(np.float64) / n1.astype(np.float64) - fr * fr, 0.0)
    std = np.sqrt(var)
    return cnt, np.where(has, mean, 0.0), np.where(has, std, 0.0)


def duration_from_float_np(x):
    """model.duration_from_float over an array (numpy's astype of a value beyond the int64 range is undefined)."""
    import numpy as np
    x = np.asarray(x, np.float64)
    out = np.zeros(x.shape, np.int64)
    inside = (x >= -2.0 ** 63) & (x < 2.0 ** 63)
    out[inside] = np.trunc(x[inside]).astype(np.int64)
    out[x >= 2.0 ** 63] = I64_MAX
    out[x < -2.0 ** 63] = -I64_MAX - 1
    return out


def resolve_np(rows, pair_key_off, cache, now: int):
    """evg_resolve_durations' per-row results for a DurationCache -> dict of avg_ns, std_ns, value_ns, pred_std_ns,
    collected_ns, source (listed-row order)."""
    import numpy as np
    cnt, mean, std = key_stats_np(rows)
    P = int(pair_key_off.shape[0]) - 1
    single = np.full(max(P, 1), -1, np.int64)
    if P > 0 and cnt.shape[0]:
        pair_of = np.searchsorted(pair_key_off, np.arange(cnt.shape[0]), side="right") - 1
        matched = cnt > 0
        n_match = np.bincount(pair_of[matched], minlength=P)
        last = np.full(P, -1, np.int64)
        last[pair_of[matched]] = np.nonzero(matched)[0]
        single[:P] = np.where(n_match == 1, last, -1)
    key = cache.key.astype(np.int64)
    doc = np.full(key.shape[0], -1, np.int64)
    pos = key >= 0
    doc[pos] = np.where(cnt[key[pos]] > 0, key[pos], -1)
    pr = key <= -2
    doc[pr] = single[-2 - key[pr]]
    value, pstd, coll = cache.value_ns, cache.std_ns, cache.collected_ns
    e, es = cache.expected_ns, cache.expected_std_ns
    ttl = np.where(cache.ttl_ns == 0, M.PREDICTION_TTL, cache.ttl_ns)
    with np.errstate(over="ignore"):
        age = np.where(coll == M.ZERO_TIME, I64_MAX, now - coll)  # no other saturation within synth's ranges
    backfill = (value == 0) & (e != 0)
    fresh = ~backfill & (age < ttl)
    stale = ~backfill & ~fresh
    a = np.where(doc >= 0, duration_from_float_np(mean[np.maximum(doc, 0)]), 0) if mean.shape[0] else np.zeros_like(key)
    sd = np.where(doc >= 0, duration_from_float_np(std[np.maximum(doc, 0)]), 0) if std.shape[0] else np.zeros_like(key)
    src = np.where(backfill, BACKFILL, FRESH)
    src = np.where(stale & (doc < 0), np.where(value == 0, DEFAULT, PREVIOUS), src)
    src = np.where(stale & (doc >= 0), np.where(a == 0, DEFAULT, HISTORY), src)
    d = M.DEFAULT_TASK_DURATION
    avg = np.select([backfill, fresh, src == DEFAULT, src == PREVIOUS], [e, value, d, value], a)
    sdv = np.select([backfill, fresh, src == DEFAULT, src == PREVIOUS], [es, pstd, 0, pstd], sd)
    return dict(avg_ns=avg, std_ns=sdv, value_ns=np.where(backfill, e, np.where(fresh, value, avg)),
                pred_std_ns=np.where(backfill | fresh, pstd, sdv),
                collected_ns=np.where(backfill, now - M.MINUTE, np.where(fresh, coll, now)), source=src.astype(np.uint8))
