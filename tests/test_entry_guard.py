"""The plumbing every entry point shares.  Without a GPU: every call that takes a context fails a NULL one with
EVG_ERR_INVALID and its own name.  On the GPU: evg_last_launch_count() agrees with the kernels torch.profiler sees
each call launch -- a call that resets the count reports exactly its own kernels, any other call adds them."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from evergreen_b200 import _lib as L
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S
from evergreen_b200 import synth
from test_gpu_tick_state import plan_aliases, resolve, update, upload, upload_with_deps, world  # noqa: F401 (world: fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "evg_sched.h")


def context_functions():
    """Every function of evg_sched.h whose first parameter is an evg_ctx*."""
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return sorted(set(re.findall(r"\b(evg_[a-z_0-9]+)\s*\(\s*evg_ctx\s*\*\s*\w*\s*[,)]", src)))


def test_every_context_call_fails_a_null_context_by_name():
    lib = L.load()
    names = context_functions()
    assert len(names) >= 35 and "evg_run_resident" in names and "evg_host_job" in names
    for name in sorted(set(names) - {"evg_shutdown", "evg_last_launch_count", "evg_device_result_ptr"}):
        restype, argtypes = L.SYMBOLS[name]
        assert restype is C.c_int, name
        args = [None if t is C.c_void_p or issubclass(t, C._Pointer) else 0 for t in argtypes]
        rc = getattr(lib, name)(*args)
        assert rc == L.EVG_ERR_INVALID, (name, rc, L.last_error())
        assert L.last_error() == f"{name}: null context"


def test_queries_and_shutdown_accept_a_null_context():
    lib = L.load()
    assert lib.evg_last_launch_count(None) == 0
    assert lib.evg_device_result_ptr(None) is None
    lib.evg_shutdown(None)


# ---------------------------------------------------------------- launch counts on the GPU
ADDS, RESETS, RESETS_AFTER_UPLOAD = "adds", "resets", "resets after its upload"


def launched_kernels(fn):
    """The names of the kernels fn launches, in start order, from torch.profiler's CUDA activity."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
    return [n for n in (re.sub(r"^void ", "", e.name) for e in ev) if n.startswith("k_")]


@pytest.fixture(scope="module")
def counts_world(world):  # noqa: F811
    return dict(world, general=synth.make(np.array([20_000, 300, 40]), 1320, tg_frac=0.1, n_hosts=10),
                edges=synth.make(np.array([100, 40, 700]), 1321, unmet_dep_frac=0.05, met_dep_frac=0.02,
                                 includes_dependencies=True, tg_frac=0.1, n_hosts=10))


def nothing(eng, W):
    return None


def upload_run(eng, W):
    upload(eng, W)
    eng.run(W["w"].now)


def upload_of(key):
    return lambda eng, W: eng.upload(W[key].tasks, W[key].distros, W[key].hosts)


def device_columns(eng, W):
    import torch
    t = W["edges"].tasks
    assert t.n_edges > 0
    cols = {name: torch.from_numpy(np.concatenate([getattr(t, name), np.zeros(8, dt)])).cuda() for name, dt in S.TaskSoA.COLUMNS}
    cols["dep_off"], cols["dep_idx"] = torch.from_numpy(t.dep_off).cuda(), torch.from_numpy(t.dep_idx).cuda()
    torch.cuda.synchronize()
    return cols  # the context borrows these until the case is done


def upload_device(eng, W, cols):
    w = W["edges"]
    eng.upload_device({k: v.data_ptr() for k, v in cols.items()}, w.n_tasks, w.distros, w.hosts, n_edges=w.tasks.n_edges)


def edit(eng, W, _):
    e = synth.next_tick(W["w"], 1310)
    eng.edit_tasks(e.edit, e.workload.distros, e.workload.hosts)


def alloc(eng, W, _):
    w = W["w"]
    po, _ = eng.download()
    eng.alloc_batch(w.hosts, po.info.copy(), po.group_info.copy(), w.distros.group_off, w.now)


def dag(eng, W, _):
    eng.dag_rebuild_batch(np.array([0, 3, 5], np.int64), np.array([0, 1, 1], np.int64), np.array([0, 0, 1, 1, 2, 2], np.int64),
                          np.array([0, 0], np.int32), np.array([0, -1, 0, -1, -1], np.int32), np.array([0, 0, 1, 0, 0], np.int32))


def call(fn):
    return lambda eng, W, _: fn(eng, W)


def run(opts):
    return lambda eng, W, _: eng.run(W["w"].now, opts)


def one_shot(key):
    return call(lambda eng, W: eng.plan_and_alloc_batch(W[key].tasks, W[key].distros, W[key].hosts, W[key].now))


CASES = {  # name: (set-up, measured call, how the call treats the count)
    "upload": (nothing, call(upload), ADDS),
    "upload_with_deps": (nothing, call(upload_with_deps), ADDS),
    "upload_device": (device_columns, upload_device, ADDS),
    "update_tasks": (upload, call(update), ADDS),
    "run_on_chip": (upload_of("plain"), run(0), RESETS),
    "run_on_chip_breakdown": (upload_of("plain"), run(L.EVG_OPT_BREAKDOWN), RESETS),
    "run_general": (upload_of("general"), run(0), RESETS),
    "run_general_breakdown": (upload_of("general"), run(L.EVG_OPT_BREAKDOWN), RESETS),
    "plan_and_alloc_batch": (nothing, one_shot("w"), RESETS_AFTER_UPLOAD),
    "plan_and_alloc_batch_pipelined": (nothing, one_shot("big"), RESETS),
    "download_queue": (upload_run, call(lambda eng, W: eng.download_queue(0, W["w"].distros.task_off)), ADDS),
    "resolve_durations": (upload, call(resolve), ADDS),
    "deps_met_batch": (nothing, call(lambda eng, W: eng.deps_met_batch(W["table"].deps)), RESETS),
    "find_runnable_batch": (nothing, call(lambda eng, W: eng.find_runnable_batch(W["table"])), RESETS),
    "plan_from_finder": (nothing, call(lambda eng, W: eng.plan_from_finder(W["table"], W["w"].tasks, W["w"].distros, W["w"].hosts,
                                                                             W["fin"], W["w"].now)), RESETS),
    "edit_tasks": (upload, edit, RESETS),
    "plan_aliases": (nothing, call(plan_aliases), RESETS),
    "rebuild_dispatchers": (upload_run, call(lambda eng, W: eng.rebuild_dispatchers(0)), RESETS),
    "host_job": (upload_run, call(lambda eng, W: eng.host_job(np.zeros(W["w"].distros.n_distros, L.HOST_JOB_CFG_DTYPE))), RESETS),
    "alloc_batch": (upload_run, alloc, RESETS),
    "expected_durations_batch": (nothing, call(lambda eng, W: eng.expected_durations_batch(W["dw"].history.rows)), RESETS),
    "prioritize_legacy_batch": (nothing, call(lambda eng, W: eng.prioritize_legacy_batch(W["legacy"])), RESETS),
    "dag_rebuild_batch": (nothing, dag, RESETS),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_launch_count_matches_the_profiler(counts_world, case):
    setup, measured, how = CASES[case]
    eng = scheduler.Engine(0)
    try:
        state = setup(eng, counts_world)
        before = eng.last_launch_count()
        names = launched_kernels(lambda: measured(eng, counts_world, state))
        after = eng.last_launch_count()
        del state
    finally:
        eng.close()
    assert names, "the call launched no kernel"
    if how == ADDS:
        assert after - before == len(names), names
    elif how == RESETS:
        assert after == len(names), names
    else:  # the upload's range check runs before evg_run_resident resets the count
        assert names[0].startswith("k_validate") and after == len(names) - 1, names
