#!/usr/bin/env python3
"""Write tests/golden/duration_cache.json: what Task.FetchExpectedDuration (model/task/task.go:3519-3590) with
CachedDurationValue.Get (util/cached_value.go:125-145) and getExpectedDurationsForWindow
(model/task/expected_duration.go:36-96) leave on one task, with the clock frozen at NOW.  Transcribed by hand: the Go
code reads MongoDB and cannot run here.

`derived` cases are not asserted by any Go test: each follows from the lines given in `ref`.  `asserted` cases restate
TestCachedDurationValue (util/cached_value_test.go:61-114) where FetchExpectedDuration can reach it: the fresh branch
and the refresher that returns ok (the refresher of task.go:3540-3574 never returns false without a DB error).

A task's `prediction` is its DurationPrediction; `collected_at` null is Go's zero time.  `expect` is what the task
holds afterwards: avg / std = the returned DurationStats (= ExpectedDuration / ExpectedDurationStdDev), value /
pred_std / collected = the DurationPrediction, source = the EVG_DS_* branch (include/evg_sched.h).  A row is persisted
(cacheExpectedDuration, task.go:893-905) exactly when source != fresh; the document then gets ExpectedDuration = value
and ExpectedDurationStdDev = pred_std.  `finished` are the task documents of the window query; the window is
(NOW - 1 week, NOW] (taskCompletionEstimateWindow, task.go:60,3543-3544).
"""
import json
import os

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "duration_cache.json")
SEC = 10 ** 9
MIN = 60 * SEC
HOUR = 60 * MIN
WEEK = 7 * 24 * HOUR
NOW = 1_800_000_000 * SEC
T = "model/task/task.go"
CV = "util/cached_value.go"
ED = "model/task/expected_duration.go"
FRESH, BACKFILL, HISTORY, PREVIOUS, DEFAULT = 0, 1, 2, 3, 4


def task(name="compile", value=0, std_dev=0, ttl=0, collected_at=None, expected=0, expected_std=0):
    return dict(project="proj", build_variant="bv", display_name=name, expected_duration=expected,
                expected_duration_std_dev=expected_std,
                prediction=dict(value=value, std_dev=std_dev, ttl=ttl, collected_at=collected_at))


def done(name, taken, finish=NOW, status="success", timed_out=False, project="proj", bv="bv"):
    """A finished task of the window query: started `taken` before it finished."""
    return dict(project=project, build_variant=bv, display_name=name, status=status, timed_out=timed_out,
                start_time=finish - taken, finish_time=finish, time_taken=taken)


def expect(avg, std, value, pred_std, collected, source):
    return dict(avg=avg, std=std, value=value, pred_std=pred_std, collected=collected, source=source)


# rows that never match the $match of expected_duration.go:37-52: timed out, not completed, outside the window, another
# variant.  A case that needs "no document" for "compile" carries them so the query has something to reject.
decoys = [done("compile", 30 * MIN, timed_out=True), done("compile", 30 * MIN, status="started"),
          done("compile", 30 * MIN, finish=NOW + 1), done("compile", 30 * MIN, finish=NOW - WEEK + 30 * MIN),
          done("compile", 30 * MIN, bv="other")]
cases = []
# 1. fresh
cases.append(dict(name="fresh", kind="derived", ref=f"{CV}:127-129, {T}:3577-3588",
                  task=task(value=20 * MIN, std_dev=2 * MIN, collected_at=NOW - HOUR, expected=5 * MIN),
                  finished=[done("compile", 40 * MIN)],
                  expect=expect(20 * MIN, 2 * MIN, 20 * MIN, 2 * MIN, NOW - HOUR, FRESH)))
# 2. since == ttl: `<` is strict, so the value is stale; no document and a previous value
cases.append(dict(name="since_equals_ttl", kind="derived", ref=f"{CV}:127 (time.Since(c) < TTL), {T}:3556-3562",
                  task=task(value=20 * MIN, std_dev=2 * MIN, ttl=HOUR, collected_at=NOW - HOUR),
                  finished=decoys, expect=expect(20 * MIN, 2 * MIN, 20 * MIN, 2 * MIN, NOW, PREVIOUS)))
# 3. zero CollectedAt: time.Since(time.Time{}) saturates at MaxInt64, always stale
cases.append(dict(name="zero_collected_at", kind="derived", ref=f"{CV}:127, time.Time.Sub saturation; {T}:3564-3569",
                  task=task(value=20 * MIN, std_dev=2 * MIN, collected_at=None),
                  finished=[done("compile", 30 * MIN), done("compile", 30 * MIN)],
                  expect=expect(30 * MIN, 0, 30 * MIN, 0, NOW, HISTORY)))
# 4. CollectedAt in the future: a negative age is below any positive TTL
cases.append(dict(name="collected_in_future", kind="derived", ref=f"{CV}:127",
                  task=task(value=20 * MIN, std_dev=2 * MIN, ttl=HOUR, collected_at=NOW + HOUR),
                  finished=[done("compile", 30 * MIN)],
                  expect=expect(20 * MIN, 2 * MIN, 20 * MIN, 2 * MIN, NOW + HOUR, FRESH)))
# 5. ttl == 0 reads as predictionTTL (8 h, unjittered): fresh one nanosecond before, stale at 8 h
cases.append(dict(name="ttl_zero_fresh", kind="derived", ref=f"{T}:67,3520-3522",
                  task=task(value=20 * MIN, std_dev=2 * MIN, ttl=0, collected_at=NOW - 8 * HOUR + 1),
                  finished=[done("compile", 30 * MIN)],
                  expect=expect(20 * MIN, 2 * MIN, 20 * MIN, 2 * MIN, NOW - 8 * HOUR + 1, FRESH)))
cases.append(dict(name="ttl_zero_stale", kind="derived", ref=f"{T}:67,3520-3522, {CV}:127",
                  task=task(value=20 * MIN, std_dev=2 * MIN, ttl=0, collected_at=NOW - 8 * HOUR),
                  finished=[done("compile", 30 * MIN)],
                  expect=expect(30 * MIN, 0, 30 * MIN, 0, NOW, HISTORY)))
# 6. backfill: (E, Es) returned; Value = E, CollectedAt = now - 1 min, StdDev untouched -- and persisted as
#    ExpectedDurationStdDev (task.go:900-902), not Es
cases.append(dict(name="backfill", kind="derived", ref=f"{T}:3524-3538, {T}:893-905",
                  task=task(value=0, std_dev=3 * MIN, collected_at=None, expected=12 * MIN, expected_std=1 * MIN),
                  finished=[done("compile", 30 * MIN)],
                  expect=expect(12 * MIN, 1 * MIN, 12 * MIN, 3 * MIN, NOW - MIN, BACKFILL)))
# 7. one document, fractional mean, truncated deviation: TimeTaken B+1, B+2, B+4 -> $avg B + 7/3, $stdDevPop sqrt(14/9)
B = 10 * MIN
cases.append(dict(name="history_truncates", kind="derived", ref=f"{T}:3564-3569 (time.Duration(float64) truncates), {ED}:66-76",
                  task=task(value=20 * MIN, std_dev=2 * MIN, collected_at=NOW - 9 * HOUR),
                  finished=[done("compile", B + 1), done("compile", B + 2), done("compile", B + 4)] + decoys,
                  expect=expect(B + 2, 1, B + 2, 1, NOW, HISTORY)))
# 8. no document: previous 0 -> default; previous != 0 -> previous
cases.append(dict(name="no_document_previous_zero", kind="derived", ref=f"{T}:3556-3560",
                  task=task(value=0, std_dev=5 * MIN, collected_at=NOW - 9 * HOUR), finished=decoys,
                  expect=expect(10 * MIN, 0, 10 * MIN, 0, NOW, DEFAULT)))
cases.append(dict(name="no_document_previous", kind="derived", ref=f"{T}:3556-3562",
                  task=task(value=7 * MIN, std_dev=5 * MIN, collected_at=NOW - 9 * HOUR), finished=decoys,
                  expect=expect(7 * MIN, 5 * MIN, 7 * MIN, 5 * MIN, NOW, PREVIOUS)))
# 9. a mean that truncates to 0: TimeTaken 0 and 1 ns -> $avg 0.5 -> avg 0 -> default
cases.append(dict(name="mean_truncates_to_zero", kind="derived", ref=f"{T}:3564-3567",
                  task=task(value=7 * MIN, std_dev=5 * MIN, collected_at=NOW - 9 * HOUR),
                  finished=[done("compile", 0), done("compile", 1)],
                  expect=expect(10 * MIN, 0, 10 * MIN, 0, NOW, DEFAULT)))
# 10. DisplayName "": no name filter, grouped by name -- one document only when exactly one name matched
cases.append(dict(name="empty_name_one_match", kind="derived", ref=f"{ED}:54-56,66-76, {T}:3556,3564-3569",
                  task=task(name="", value=7 * MIN, std_dev=5 * MIN, collected_at=NOW - 9 * HOUR),
                  finished=[done("a", 20 * MIN), done("a", 40 * MIN), done("b", 5 * MIN, timed_out=True),
                            done("c", 5 * MIN, bv="other")],
                  expect=expect(30 * MIN, 10 * MIN, 30 * MIN, 10 * MIN, NOW, HISTORY)))
cases.append(dict(name="empty_name_two_matches", kind="derived", ref=f"{ED}:54-56,66-76, {T}:3556-3560",
                  task=task(name="", value=0, std_dev=5 * MIN, collected_at=NOW - 9 * HOUR),
                  finished=[done("a", 20 * MIN), done("b", 40 * MIN)],
                  expect=expect(10 * MIN, 0, 10 * MIN, 0, NOW, DEFAULT)))
# TestCachedDurationValue, where FetchExpectedDuration reaches it
C = "util/cached_value_test.go"
cases.append(dict(name="TestCachedDurationValue/fresh", kind="asserted", ref=f"{C}:69-81",
                  task=task(value=21 * SEC, ttl=MIN, collected_at=NOW), finished=[done("compile", 42 * SEC)],
                  expect=expect(21 * SEC, 0, 21 * SEC, 0, NOW, FRESH)))
cases.append(dict(name="TestCachedDurationValue/true_refresher", kind="asserted", ref=f"{C}:83-105 (a 42 s document)",
                  task=task(value=21 * SEC, ttl=SEC, collected_at=NOW - MIN), finished=[done("compile", 42 * SEC)],
                  expect=expect(42 * SEC, 0, 42 * SEC, 0, NOW, HISTORY)))
json.dump(dict(source="model/task/task.go FetchExpectedDuration", now=NOW, cases=cases), open(OUT, "w"), indent=1)
print("wrote", OUT)
