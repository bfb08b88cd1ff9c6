"""Compare one synthetic tick run through the CUDA path (C-ABI) with the oracle."""
import numpy as np

from evergreen_b200 import _lib as L
from oracle import oracle as O

INFO_FIELDS = ("length", "length_with_dependencies_met", "count_dep_filled_merge_queue_tasks", "expected_duration",
               "max_duration_threshold", "count_duration_over_threshold", "duration_over_threshold",
               "count_wait_over_threshold", "secondary_queue")
GROUP_FIELDS = ("count", "max_hosts", "expected_duration", "count_duration_over_threshold",
                "count_wait_over_threshold", "count_dep_filled_merge_queue_tasks", "duration_over_threshold")


def first_diff(a, b):
    idx = np.nonzero(np.asarray(a) != np.asarray(b))[0]
    return int(idx[0]) if idx.size else -1


def check_against_oracle(w, po, ao, distros=None, threads=8, check_groups=True):
    """Bit-exact: ranked order, TotalValue per rank, every DistroQueueInfo /
    TaskGroupInfo scalar, (new_hosts, free_hosts, status) and deficit_ns."""
    job = O.SoAJob(w.tasks, w.distros, w.hosts, distros)
    ref = job.run(w.now, threads)
    toff = w.distros.task_off
    goff = w.distros.group_off
    sel_gid = w.tasks.group_id if distros is None else _sel_gid(w, job)
    for j, d in enumerate(job.sel):
        a, b = int(toff[d]), int(toff[d + 1])
        ra, rb = int(ref["task_off"][j]), int(ref["task_off"][j + 1])
        k = first_diff(po.total_value[a:b], ref["total_value"][ra:rb])
        assert k < 0, (f"distro {d}: TotalValue differs at rank {k}: gpu {po.total_value[a + k]} vs oracle "
                       f"{ref['total_value'][ra + k]} (gpu task {po.order[a + k]}, oracle task {ref['order'][ra + k]})")
        k = first_diff(po.order[a:b], ref["order"][ra:rb])
        assert k < 0, (f"distro {d}: order differs at rank {k}: gpu task {po.order[a + k]} vs oracle "
                       f"{ref['order'][ra + k]} (value {po.total_value[a + k]})")
        for f in INFO_FIELDS:
            assert int(po.info[d][f]) == int(ref["info"][j][f]), (d, f, int(po.info[d][f]), int(ref["info"][j][f]))
        if check_groups:
            og = job.groups_by_id(ref, j, sel_gid)
            n_named = int(goff[d + 1] - goff[d])
            assert int(po.info[d]["has_ungrouped"]) == int(-1 in og), d
            assert len(og) == n_named + int(-1 in og), (d, len(og), n_named)
            for g, row in og.items():
                mine = po.info[d]["ungrouped"] if g < 0 else po.group_info[int(goff[d]) + g]
                for f in GROUP_FIELDS:
                    if g < 0 and f == "max_hosts":
                        continue  # the "" bucket's MaxHosts is never read (allocator.go:80-82)
                    assert int(mine[f]) == int(row[f]), (d, g, f, int(mine[f]), int(row[f]))
                if ao is not None and g >= 0:  # an error status leaves them at 0 on both sides (evg_sched.h)
                    for f in ("count_free", "count_required"):
                        assert int(mine[f]) == int(row[f]), (d, g, f, int(mine[f]), int(row[f]))
        if ao is not None:
            got = (int(ao.result[d]["new_hosts"]), int(ao.result[d]["free_hosts"]), int(ao.status[d]))
            want = (int(ref["new_hosts"][j]), int(ref["free_hosts"][j]), int(ref["status"][j]))
            assert got == want, (d, got, want)
            # max(0, ExpectedDuration - free_hosts * MaxDurationThreshold), int64 with wrap (evg_sched.h)
            deficit = max(0, _wrap64(int(ref["info"][j]["expected_duration"]) -
                                     _wrap64(int(ref["free_hosts"][j]) * int(ref["info"][j]["max_duration_threshold"]))))
            assert int(ao.result[d]["deficit_ns"]) == deficit, (d, int(ao.result[d]["deficit_ns"]), deficit)
    return ref


def _wrap64(x: int) -> int:
    return (x + 2 ** 63) % 2 ** 64 - 2 ** 63


def _sel_gid(w, job):
    toff = w.distros.task_off
    return np.concatenate([w.tasks.group_id[int(toff[d]):int(toff[d + 1])] for d in job.sel])


def check_properties(w, po, ao=None):
    """Size-independent invariants, cheap enough for BASELINE's full sizes:
    each distro's order is a permutation, TotalValue is non-increasing along
    the rank, queue-info sums equal independent numpy reductions."""
    t, dt = w.tasks, w.distros
    toff = dt.task_off
    T, D = t.n_tasks, dt.n_distros
    sizes = np.diff(toff)
    distro_of = np.repeat(np.arange(D), sizes)
    # permutation: sorting (distro, order) must give 0..T_d-1 everywhere
    key = distro_of.astype(np.int64) * (1 << 22) + po.order.astype(np.int64)
    key.sort()
    local = np.arange(T, dtype=np.int64) - toff[distro_of]
    assert np.array_equal(key, distro_of.astype(np.int64) * (1 << 22) + local), "order is not a per-distro permutation"
    # sortedness
    if T > 1:
        same = distro_of[1:] == distro_of[:-1]
        assert np.all(po.total_value[1:][same] <= po.total_value[:-1][same]), "TotalValue increases along the rank"
    # queue-info reductions (scheduler.go:56-159)
    met = (t.flags & L.EVG_TF_DEPS_MET) != 0
    incl = dt.cfg["includes_dependencies"][distro_of] != 0
    counted = ~incl | met
    thr = dt.cfg["target_time_ns"][distro_of]
    over = counted & (t.expected_ns > thr)

    def seg(x):
        return np.bincount(distro_of, weights=None, minlength=D) if x is None else np.add.reduceat(
            np.concatenate([x.astype(np.int64), [0]]), np.minimum(toff[:-1], T))[:D] * (sizes > 0)
    assert np.array_equal(po.info["length"], sizes)
    assert np.array_equal(po.info["length_with_dependencies_met"], seg(met))
    assert np.array_equal(po.info["expected_duration"], seg(np.where(counted, t.expected_ns, 0)))
    assert np.array_equal(po.info["count_duration_over_threshold"], seg(over))
    assert np.array_equal(po.info["duration_over_threshold"], seg(np.where(over, t.expected_ns, 0)))
    assert np.array_equal(po.info["max_duration_threshold"], dt.cfg["target_time_ns"])
    if ao is not None:
        assert np.all(ao.result["new_hosts"] >= 0) and np.all(ao.result["free_hosts"] >= 0)
        ok = ao.status == 0
        # host_allocator_fuzzer_test.go:163-170: never more hosts than (dependency-met) tasks + minimum top-up
        cap = po.info["length_with_dependencies_met"] + w.hosts.cfg["minimum_hosts"]
        assert np.all(ao.result["new_hosts"][ok] <= cap[ok])
