#!/usr/bin/env python3
"""evg_queue_index_batch against a host group-by over the same strings:
`python profiles/queue_index.py [steps] [out.json]`.

Workload: Q queues of 10 000 saved items (Q = 200, 2 000) with ids shaped like Evergreen task ids (60 bytes), about a
tenth of the tasks placed in 2-4 queues the way distro aliases place them, each queue in random order.  Per shape:
  device  one evg_queue_index_batch, timed with CUDA events on the engine's stream (H2D of the strings, kernels, D2H of
          the outputs) and with the host clock around the call, which ends in a stream synchronise; a warm-up call,
          then `steps` calls, medians;
  kernels the call's kernel and copy time from torch.profiler, in a pass of its own;
  host    the same two views from NumPy on one core: np.unique over the fixed-width ids (a sort-based group-by,
          byte-exact), then per id the smallest index and the lowest and highest queue; one call.
The outputs of both are compared.  Prints one JSON line (and writes it to out.json when given) with the card's name and
power limit, read in the same process, and the host's core count."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from evergreen_b200 import scheduler  # noqa: E402
from evergreen_b200 import synth  # noqa: E402

PER_QUEUE = 10_000
ID_BYTES = 60
PREFIX = b"evergreen_ubuntu2204_compile_patch_"  # 35 bytes, then 16 hex digits, "_" and 8 decimal digits


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in q.split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def make(Q, seed):
    """-> (ids uint8 [N, 60], item_off [Q + 1]): N = Q x 10 000 items."""
    rng = np.random.default_rng(seed)
    N = Q * PER_QUEUE
    U = int(N / 1.2)                     # 0.9 U single-queue tasks + 0.1 U tasks in 3 queues on average = 1.2 U items
    n_alias = U // 10
    k = rng.integers(2, 5, n_alias)      # each aliased task sits in 2-4 distinct queues
    q0 = rng.integers(0, Q, n_alias)
    step = rng.integers(1, max(Q // 4, 2), n_alias)
    a_task = np.repeat(np.arange(n_alias, dtype=np.int64), k)
    j = np.arange(a_task.shape[0]) - np.repeat(np.cumsum(k) - k, k)
    a_queue = (q0[a_task] + j * step[a_task]) % Q
    per_q = np.bincount(a_queue, minlength=Q)
    assert per_q.max() <= PER_QUEUE
    own = PER_QUEUE - per_q              # each queue filled up with tasks of its own
    o_queue = np.repeat(np.arange(Q, dtype=np.int64), own)
    o_task = n_alias + np.arange(o_queue.shape[0], dtype=np.int64)
    task = np.concatenate([a_task, o_task])
    queue = np.concatenate([a_queue, o_queue])
    order = np.lexsort((rng.random(task.shape[0]), queue))  # queue by queue, each in random order
    task = task[order]
    ids = np.empty((N, ID_BYTES), np.uint8)
    ids[:, :len(PREFIX)] = np.frombuffer(PREFIX, np.uint8)
    h = synth.mix64(task.astype(np.uint64))
    hexd = np.frombuffer(b"0123456789abcdef", np.uint8)
    for d in range(16):
        ids[:, len(PREFIX) + d] = hexd[((h >> np.uint64(60 - 4 * d)) & np.uint64(15)).astype(np.int64)]
    ids[:, len(PREFIX) + 16] = ord("_")
    for d in range(8):
        ids[:, len(PREFIX) + 17 + d] = ord("0") + (task // 10 ** (7 - d)) % 10
    return ids, np.arange(Q + 1, dtype=np.int64) * PER_QUEUE


def host_views(ids, item_off):
    """The group-by on one core: per item 1 + its id's smallest index; the ids in two or more queues."""
    N, Q = ids.shape[0], item_off.shape[0] - 1
    keys = np.ascontiguousarray(ids).view(np.dtype((np.void, ID_BYTES))).ravel()
    _, first, inv = np.unique(keys, return_index=True, return_inverse=True)
    queue = np.repeat(np.arange(Q, dtype=np.int64), np.diff(item_off))
    index = np.arange(N, dtype=np.int64) - item_off[queue]
    order = np.argsort(inv, kind="stable")
    starts = np.concatenate([[0], np.nonzero(np.diff(inv[order]))[0] + 1])
    pos = np.minimum.reduceat(index[order], starts)
    lo = np.minimum.reduceat(queue[order], starts)
    hi = np.maximum.reduceat(queue[order], starts)
    dup_first = np.sort(first[lo != hi])
    return (pos[inv] + 1).astype(np.int32), dup_first


def kernel_ms(eng, data, off, item_off):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.queue_index((data, off), item_off)
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    k = sum(e.device_time for e in ev if e.name.startswith("k_") or e.name.startswith("void k_")) / 1e3
    copy = sum(e.device_time for e in ev if "Memcpy" in e.name) / 1e3
    return k, copy


def shape(Q, steps):
    import torch
    ids, item_off = make(Q, 7 + Q)
    N = ids.shape[0]
    data, off = ids.ravel(), np.arange(N + 1, dtype=np.int64) * ID_BYTES
    stream = torch.cuda.Stream()
    eng = scheduler.Engine(0, stream=stream.cuda_stream)
    ev_ms, wall = [], []
    for step in range(steps + 1):  # step 0 warms up and is not kept
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        a.record(stream)
        got = eng.queue_index((data, off), item_off)
        b.record(stream)
        b.synchronize()
        t1 = time.perf_counter()
        if step:
            ev_ms.append(a.elapsed_time(b))
            wall.append((t1 - t0) * 1e3)
    launches = eng.last_launch_count()
    got = {k: v.copy() for k, v in got.items()}
    k_ms, copy_ms = kernel_ms(eng, data, off, item_off)
    eng.close()
    t0 = time.perf_counter()
    pos, dup_first = host_views(ids, item_off)
    host_ms = (time.perf_counter() - t0) * 1e3
    assert np.array_equal(pos, got["min_position"])
    assert np.array_equal(dup_first, got["dup_item"])
    return {"queues": Q, "items": N, "id_bytes": int(data.nbytes), "duplicated_ids": int(got["dup_item"].shape[0]),
            "dup_pairs": int(got["dup_off"][-1]), "steps": steps, "device_event_ms": float(np.median(ev_ms)),
            "device_wall_ms": float(np.median(wall)), "launches": int(launches), "kernel_ms": k_ms, "copy_ms": copy_ms,
            "host_groupby_ms": host_ms, "outputs_equal": True}


if __name__ == "__main__":
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    res = {"card": card(), "host_cores": os.cpu_count(), "host_groupby_cores": 1,
           "shapes": [shape(Q, steps) for Q in (200, 2000)]}
    line = json.dumps(res)
    print(line)
    if len(sys.argv) > 2:
        with open(sys.argv[2], "w") as f:
            f.write(line + "\n")
