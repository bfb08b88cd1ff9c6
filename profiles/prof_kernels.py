#!/usr/bin/env python3
"""Per-kernel split of one resident tick, from a torch.profiler trace with CUDA activities.
  python profiles/prof_kernels.py headline|c3 [ticks] [library.so]
headline: bench.py's workload (2000 distros x 100 000 tasks of configs[2]'s mix, tiled on the device as bench.py tiles it);
c3: 48 distros x 100 000 tasks of the same mix (prof_general.py's c3).  Prints the card and its power limit, the tick
time with the profiler off, then every kernel's device time per tick, largest first (template arguments folded)."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ctypes as C  # noqa: E402

import numpy as np  # noqa: E402

from evergreen_b200 import _lib as L  # noqa: E402

if len(sys.argv) > 3:  # another build of the library, e.g. another commit's, to compare the two
    lib = C.CDLL(sys.argv[3])
    for name, (res, args) in L.SYMBOLS.items():
        if hasattr(lib, name):
            fn = getattr(lib, name); fn.restype = res; fn.argtypes = args
    L._lib = lib
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import bench  # noqa: E402
from evergreen_b200 import scheduler, synth  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip() or r.stderr.strip()


def short(name):
    name = re.sub(r"^void ", "", name)
    name = name.split("(")[0]
    return re.sub(r"<.*>", "<>", name)


def main():
    which = sys.argv[1] if len(sys.argv) > 1 else "headline"
    ticks = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    eng = scheduler.Engine(0, stream.cuda_stream)
    keep = None
    if which == "headline":
        blk = bench.headline_block(0, 40, 100_000)
        distros, hosts = bench.tile_tables(blk, 50)
        cols, keep, T, E = bench.tile_device(torch, dev, blk, 50)
        eng.upload_device(cols, T, distros, hosts, n_edges=E)
        now = blk.now
    else:
        w = synth.config(3, 0.0048, each=True)
        eng.upload(w.tasks, w.distros, w.hosts)
        T, now = w.n_tasks, w.now
    for _ in range(3):
        eng.run(now)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(ticks):
        eng.run(now)
    e1.record(stream)
    torch.cuda.synchronize()
    tick_ms = e0.elapsed_time(e1) / ticks
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(ticks):
            eng.run(now)
        torch.cuda.synchronize()
    tot = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            k = short(ev.name)
            n, us = tot.get(k, (0, 0.0))
            tot[k] = (n + 1, us + ev.device_time)
    po, ao = eng.download()
    checksum = int(ao.result["new_hosts"].astype(np.int64).sum()) + int(po.order[::997].sum())
    print(f"card: {card()}")
    print(f"shape {which}: {T} tasks, tick {tick_ms:.3f} ms (profiler off, {ticks} ticks), checksum {checksum}, "
          f"device memory in use {(torch.cuda.mem_get_info(dev)[1] - torch.cuda.mem_get_info(dev)[0]) / 1e9:.1f} GB")
    print("| kernel | launches / tick | ms / tick |\n|---|---:|---:|")
    s = 0.0
    for k, (n, us) in sorted(tot.items(), key=lambda kv: -kv[1][1]):
        s += us
        print(f"| `{k}` | {n / ticks:g} | {us / ticks / 1e3:.3f} |")
    print(f"| sum of kernel times | | {s / ticks / 1e3:.3f} |")
    eng.close()
    del keep


if __name__ == "__main__":
    main()
