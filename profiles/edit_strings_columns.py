"""The device and PCIe side of a tick whose strings stay resident, at the size of DESIGN.md §8.6 (200 distros x 100 000
tasks), with the columns marshalled ahead of time so that no Go-level Task loop is in the way: (b) evg_upload_strings of
the whole composed string table against (c) evg_edit_strings of the edit, on two contexts that hold the same tick.
Every step 5 % of each queue leaves and 5 % arrives; 10 % of the tasks are in task groups and about 13 % name a
dependency (an earlier or a later task of their queue, or an id no task has).  Strings are fixed-width ASCII (ids 29
bytes, versions 9, group keys 11).  After each step both contexts run and their download_queue rows must be equal.
Reports per arm the median and range of the call time (host clock around the synchronised call, the copies from
pageable memory included), the H2D bytes per step, the device memory each context holds (cudaMemGetInfo deltas), and
the card's name and power limit.

    python profiles/edit_strings_columns.py --distros 200 --tasks-per-distro 100000 --steps 4 --warmup 1
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

NOW = 1_700_000_000 * 10 ** 9


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip()


def digits(x, k):
    """Decimal digits of the int64 array x, k of them, as an (n, k) uint8 ASCII matrix."""
    x = np.array(x, dtype=np.int64)
    out = np.empty((x.shape[0], k), np.uint8)
    for j in range(k - 1, -1, -1):
        out[:, j] = (x % 10 + 48).astype(np.uint8)
        x //= 10
    return out


def lit(s, n):
    return np.broadcast_to(np.frombuffer(s.encode(), np.uint8), (n, len(s)))


def col(mat, mask=None):
    """An (n, W) matrix as an evg_str_col; rows where mask is False are empty strings."""
    n, w = mat.shape
    lens = np.full(n, w, np.int64) if mask is None else np.where(mask, w, 0).astype(np.int64)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    data = np.ascontiguousarray(mat if mask is None else mat[mask]).ravel()
    return np.ascontiguousarray(data), off


def id_mat(d, num):
    n = d.shape[0]
    return np.hstack([lit("task_", n), digits(d, 3), lit("_", n), digits(num, 9), lit("_bv_linux_x", n)])


class Table:
    """A tick in state arrays: per row its distro, task number, version, group (-1: none), numeric columns, and a CSR
    of DependsOn ids, each a (distro, number)."""
    NUMERIC = ("priority", "expected_ns", "queue_basis_ns", "wait_basis_ns", "num_dependents", "task_group_order", "flags")

    def __init__(self, **kw):
        self.__dict__.update(kw)

    @property
    def n(self):
        return self.dist.shape[0]

    def strings(self, D):
        from evergreen_b200 import soa as S
        n = self.n
        task_off = np.concatenate([[0], np.cumsum(np.bincount(self.dist, minlength=D))]).astype(np.int64)
        ver = np.hstack([lit("ver_", n), digits(self.ver, 5)])
        gk = np.hstack([lit("tg", n), digits(np.maximum(self.grp, 0), 3), lit("_", n), digits(self.ver, 5)])
        return S.StringCols(task_off, col(id_mat(self.dist, self.num)), col(ver), col(gk, self.grp >= 0),
                            np.ascontiguousarray(self.gmh, np.int32), self.dep_off.astype(np.int64), col(id_mat(self.dep_d, self.dep_n)))

    def numeric(self):
        from evergreen_b200 import soa as S
        z = np.zeros(self.n, np.int32)
        return S.TaskSoA(**{k: getattr(self, k) for k in self.NUMERIC}, group_id=z, version_id=z)

    def rows(self, r):
        """The rows r (in that order) as a Table."""
        cnt = np.diff(self.dep_off)[r]
        off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
        e = np.repeat(self.dep_off[:-1][r] - off[:-1], cnt) + np.arange(int(off[-1]))
        kw = {k: getattr(self, k)[r] for k in ("dist", "num", "ver", "grp", "gmh") + self.NUMERIC}
        return Table(**kw, dep_off=off, dep_d=self.dep_d[e], dep_n=self.dep_n[e])

    @staticmethod
    def cat(a, b):
        kw = {k: np.concatenate([getattr(a, k), getattr(b, k)]) for k in ("dist", "num", "ver", "grp", "gmh", "dep_d", "dep_n") + Table.NUMERIC}
        return Table(**kw, dep_off=np.concatenate([a.dep_off, b.dep_off[1:] + a.dep_off[-1]]))


def new_tasks(rng, dist, first, counter, tick):
    """Tasks of the given distros, numbered from first (per row); DependsOn: 10 % an earlier or later task of the
    queue, 3 % an id no task has."""
    n = dist.shape[0]
    ver = rng.integers(tick, tick + 20, n)
    grp = np.where(rng.random(n) < 0.1, rng.integers(0, 50, n), -1)
    has_q, has_x = rng.random(n) < 0.10, rng.random(n) < 0.03
    cnt = has_q.astype(np.int64) + has_x
    dep_off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    own = np.repeat(np.arange(n), cnt)
    is_q = np.ones(own.shape[0], bool)
    is_q[dep_off[1:][has_x] - 1] = False
    dep_d = np.where(is_q, dist[own], 999)
    dep_n = np.where(is_q, (rng.random(own.shape[0]) * (counter[dist[own]] * 1.05 + 10)).astype(np.int64), rng.integers(0, 10 ** 9, own.shape[0]))
    return Table(dist=dist, num=first, ver=ver, grp=grp, gmh=((grp * 7 + ver) % 4 + 1).astype(np.int32) * (grp >= 0),
                 priority=rng.integers(0, 100, n).astype(np.int32), expected_ns=rng.integers(1, 10 ** 12, n),
                 queue_basis_ns=NOW - rng.integers(0, 10 ** 13, n), wait_basis_ns=NOW - rng.integers(0, 10 ** 12, n),
                 num_dependents=rng.integers(0, 4, n).astype(np.int32), task_group_order=rng.integers(0, 5, n).astype(np.int32),
                 flags=rng.integers(0, 8, n).astype(np.uint32), dep_off=dep_off, dep_d=dep_d, dep_n=dep_n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--distros", type=int, default=200)
    ap.add_argument("--tasks-per-distro", type=int, default=100000)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--frac", type=float, default=0.05)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    from evergreen_b200 import _lib as L, scheduler, soa as S

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this profile measures on the GPU only")
    rng = np.random.default_rng(7)
    D, N = args.distros, args.tasks_per_distro
    cfg = np.zeros(D, L.DISTRO_CFG_DTYPE)
    cfg["patch_factor"], cfg["expected_runtime_factor"], cfg["target_time_ns"] = 1, 1, 60 * 10 ** 9
    counter = np.full(D, N, np.int64)
    dist0 = np.repeat(np.arange(D), N)
    tab = new_tasks(rng, dist0, np.tile(np.arange(N), D), counter, 0)
    engines, mem, call, h2d = {}, {}, {}, {}
    keys = ("b_upload_strings", "c_edit_strings")
    sc = tab.strings(D)
    for a in keys:
        free0 = torch.cuda.mem_get_info()[0]
        engines[a] = scheduler.Engine(0)
        engines[a].upload_strings(tab.numeric(), sc, cfg)
        torch.cuda.synchronize()
        mem[a] = free0 - torch.cuda.mem_get_info()[0]
        call[a], h2d[a] = [], []

    def strings_bytes(s):
        return sum(c[0].nbytes + c[1].nbytes for c in (s.id, s.version, s.group_key, s.dep_id)) + s.group_max_hosts.nbytes + s.dep_off.nbytes

    for k in range(args.warmup + args.steps):
        T0 = tab.n
        keep = rng.random(T0) >= args.frac
        n_new = rng.binomial(np.bincount(tab.dist, minlength=D), args.frac)
        dist_new = np.repeat(np.arange(D), n_new)
        first = counter[dist_new] + (np.arange(dist_new.shape[0]) - np.repeat(np.concatenate([[0], np.cumsum(n_new)[:-1]]), n_new))
        arr = new_tasks(rng, dist_new, first, counter, k + 1)
        counter += n_new
        surv = np.nonzero(keep)[0]
        both = Table.cat(tab.rows(surv), arr)
        composed = both.rows(np.argsort(both.dist, kind="stable"))  # survivors in order, then arrivals, per distro
        edit = S.StringEdit(np.nonzero(~keep)[0].astype(np.int64), arr.numeric(), arr.strings(D))
        comp_sc, comp_num = composed.strings(D), composed.numeric()
        ins_bytes = edit.nbytes()
        res = {}

        def arm_b():
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            t0 = time.perf_counter()
            engines["b_upload_strings"].upload_strings(comp_num, comp_sc, cfg)
            torch.cuda.synchronize()
            res["b_upload_strings"] = ((time.perf_counter() - t0) * 1e3, sum(getattr(comp_num, c).nbytes for c in Table.NUMERIC) + strings_bytes(comp_sc))
            mem["b_upload_strings"] += free0 - torch.cuda.mem_get_info()[0]

        def arm_c():
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            t0 = time.perf_counter()
            engines["c_edit_strings"].edit_strings(edit, cfg)
            torch.cuda.synchronize()
            res["c_edit_strings"] = ((time.perf_counter() - t0) * 1e3, ins_bytes)
            mem["c_edit_strings"] += free0 - torch.cuda.mem_get_info()[0]

        for f in ((arm_b, arm_c) if k % 2 == 0 else (arm_c, arm_b)):
            f()
        q = []
        for a in keys:
            engines[a].run(NOW, 0)
            off, items = engines[a].download_queue(0, comp_sc.task_off)
            q.append((off.copy(), items.copy()))
        assert np.array_equal(q[0][0], q[1][0]) and np.array_equal(q[0][1], q[1][1]), f"step {k}: download_queue"
        print(json.dumps({"step": k, "tasks": composed.n, "call_ms": {a: round(res[a][0], 2) for a in keys}}), flush=True)
        if k >= args.warmup:
            for a in keys:
                call[a].append(res[a][0])
                h2d[a].append(res[a][1])
        tab = composed
    rng_of = lambda v: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}  # noqa: E731
    out = {"gpu": gpu_info(), "distros": D, "tasks": tab.n, "steps": args.steps, "frac": args.frac,
           "call_ms_per_step": {a: rng_of(v) for a, v in call.items()},
           "h2d_bytes_per_step": {a: int(np.mean(v)) for a, v in h2d.items()},
           "device_bytes_per_context": {a: int(v) for a, v in mem.items()},
           "outputs_equal_every_step": True}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    for eng in engines.values():
        eng.close()


if __name__ == "__main__":
    main()
