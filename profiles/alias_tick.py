"""Alias queues of one tick, two routes to the same planned queues:
  host    the shim's fan-out in Python (every task to each distro whose applicable set names it), marshal_tasks over
          every alias queue (a task in k queues is marshalled k times), evg_upload_with_deps
  device  marshal_aliases over the tick's tasks once, evg_plan_aliases (fan-out, compaction, ids and edges on the GPU)
each followed by evg_run_resident + evg_download.  Prints per-stage medians and the device memory in use after the
first evg_plan_aliases.  usage: python profiles/alias_tick.py [n_distros] [n_tasks] [reps]"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from evergreen_b200 import model as M  # noqa: E402
from evergreen_b200 import scheduler, soa as S, synth  # noqa: E402

D = int(sys.argv[1]) if len(sys.argv) > 1 else 2000
T = int(sys.argv[2]) if len(sys.argv) > 2 else 10000
REPS = int(sys.argv[3]) if len(sys.argv) > 3 else 5
NOW = synth.NOW_NS
rng = np.random.default_rng(7)
distros = [M.Distro(id=f"d{e}", aliases=[f"a{int(x)}" for x in rng.integers(0, D // 4 + 1, rng.integers(0, 3))]) for e in range(D)]
tasks = []
for i in range(T):
    names = []
    if rng.random() < 0.2:  # ~20 % of tasks carry 1-3 names: distro ids or alias names
        names = [f"d{int(rng.integers(D))}" if rng.random() < 0.5 else f"a{int(rng.integers(D // 4 + 1))}"
                 for _ in range(int(rng.integers(1, 4)))]
    tg = f"g{i // 8}" if rng.random() < 0.1 else ""
    tasks.append(M.Task(id=f"t{i}", project="p", version=f"v{i % 50}", build_variant="bv", distro_id=f"d{int(rng.integers(D))}",
                        secondary_distros=names, task_group=tg, task_group_max_hosts=2 if tg else 0,
                        priority=int(rng.integers(0, 5)), expected_duration=int(rng.integers(1, 60)) * M.MINUTE,
                        activated_time=NOW - int(rng.integers(1, 600)) * M.MINUTE, scheduled_time=NOW - M.HOUR,
                        depends_on=[M.Dependency(f"t{int(rng.integers(T))}")] if rng.random() < 0.05 else []))
db = {t.id: t for t in tasks}


def host_route(eng):
    t0 = time.perf_counter()
    index, dest_off, dest_idx = S.alias_name_table(distros)
    queues = [[] for _ in range(D)]
    for t in tasks:  # every task here passes the base query; single-host groups stay out
        if t.task_group_max_hosts == 1:
            continue
        seen = set()
        for n in t.secondary_distros:
            k = index.get(n)
            if k is not None:
                for e in dest_idx[dest_off[k]:dest_off[k + 1]]:
                    if int(e) not in seen:
                        seen.add(int(e))
                        queues[int(e)].append(t)
    batch = list(zip(distros, queues))
    t1 = time.perf_counter()
    soa, table, _ = S.marshal_tasks(batch, NOW, db)
    deps, fin = S.marshal_deps(batch, db), S.marshal_dep_finished(batch)
    t2 = time.perf_counter()
    eng.upload_with_deps(soa, table, None, deps, fin, NOW)
    eng.run(NOW)
    po, _ = eng.download(want_alloc=False)
    t3 = time.perf_counter()
    return (t1 - t0, t2 - t1, t3 - t2), soa.n_tasks, po.total_value.copy()


def device_route(eng):
    t0 = time.perf_counter()
    at, cfg, _ = S.marshal_aliases(distros, tasks, NOW, db)
    t1 = time.perf_counter()
    task_off, _, _ = eng.plan_aliases(at, cfg, NOW)
    eng.run(NOW)
    po, _ = eng.download(want_alloc=False)
    t2 = time.perf_counter()
    return (0.0, t1 - t0, t2 - t1), int(task_off[-1]), po.total_value.copy()


def main():
    torch.cuda.init()
    print(torch.cuda.get_device_name(0), "power limit:", os.popen("nvidia-smi --query-gpu=power.limit --format=csv,noheader").read().strip())
    eng_h, eng_d = scheduler.Engine(0), scheduler.Engine(0)
    free0, _ = torch.cuda.mem_get_info()
    device_route(eng_d)
    free1, _ = torch.cuda.mem_get_info()
    host_route(eng_h)
    res = {"host": [], "device": []}
    for _ in range(REPS):
        for name, fn, eng in (("host", host_route, eng_h), ("device", device_route, eng_d)):
            stages, n, tv = fn(eng)
            res[name].append(stages)
    _, nh, tvh = host_route(eng_h)
    _, nd, tvd = device_route(eng_d)
    print(f"{D} distros x {T} tasks: {nd} alias queue rows (host route {nh}); TotalValue per rank identical: {np.array_equal(tvh, tvd)}")
    for name in ("host", "device"):
        a = np.array(res[name]) * 1e3
        med = np.median(a, axis=0)
        print(f"  {name:6s} fan-out {med[0]:8.1f} ms  marshal {med[1]:8.1f} ms  upload/plan + run + download {med[2]:7.2f} ms"
              f"  total {np.median(a.sum(axis=1)):8.1f} ms  (median of {REPS})")
    print(f"  device memory taken by a fresh context after its first evg_plan_aliases + run: {(free0 - free1) / 2**20:.1f} MiB")
    eng_h.close()
    eng_d.close()


if __name__ == "__main__":
    main()
