"""Seeded multi-tick Go-level batches for evg_edit_strings: every tick some tasks leave and others arrive, task groups
and versions appear and vanish, survivors name arrivals in DependsOn before they exist and keep naming departed ones,
and some DependsOn lists repeat an id."""
import random

import numpy as np

from evergreen_b200 import model as M
from evergreen_b200 import soa as S

NOW = 1_700_000_000 * 10 ** 9


class Script:
    """One distro list and its batches, tick by tick; next_batch() returns the batch in ResidentTick's canonical
    order (survivors in their previous order, then arrivals)."""

    def __init__(self, seed: int, sizes=(0, 1, 40, 700, 0, 300, 13), n_ext: int = 5):
        self.rng = random.Random(seed)
        self.distros = [M.Distro(id=f"d{d}") for d in range(len(sizes))]
        self.counter = [0] * len(sizes)
        self.tick = 0
        self.n_ext = n_ext
        self.batch = [(d, [self.task(k) for _ in range(n)]) for k, (d, n) in enumerate(zip(self.distros, sizes))]

    def task(self, d: int) -> M.Task:
        rng, i = self.rng, self.counter[d]
        self.counter[d] += 1
        ver = f"v{rng.randrange(self.tick, self.tick + 3)}"
        t = M.Task(id=f"d{d}-t{i}", version=ver, project="p", build_variant=f"bv{rng.randrange(2)}",
                   priority=rng.choice([0, 0, 1, 50, -1]), requester=rng.choice(["gitter_request", "patch_request", "ad_hoc"]),
                   num_dependents=rng.randrange(4), distro_id=f"d{d}", ingest_time=NOW - rng.randrange(10 ** 13),
                   scheduled_time=rng.choice([M.ZERO_TIME, NOW - rng.randrange(10 ** 12)]),
                   activated_by=rng.choice(["", "stepback"]), generate_task=rng.random() < 0.1)
        if rng.random() < 0.4:
            g = rng.randrange(self.tick // 2, self.tick // 2 + 3)  # groups appear over the ticks, old ones run dry
            t.task_group, t.task_group_order = f"tg{g}", rng.randrange(5)
            t.task_group_max_hosts = 1 + (g + int(t.version[1:]) + int(t.build_variant[2:])) % 3
        for _ in range(rng.choice([0, 0, 1, 2, 3])):
            # an earlier task (maybe departed), a task that arrives later, another distro's, an external or a missing one
            target = rng.choice([f"d{d}-t{rng.randrange(i + 40)}", f"d{d}-t{rng.randrange(i + 40)}",
                                 f"d{(d + 1) % len(self.counter)}-t0", f"ext{rng.randrange(self.n_ext)}", "missing"])
            t.depends_on.append(M.Dependency(target, status=rng.choice(["", "success", "failed"])))
        if t.depends_on and rng.random() < 0.2:
            t.depends_on.append(M.Dependency(t.depends_on[0].task_id))  # a repeated DependsOn id
        return t

    def next_batch(self, leave: float = 0.1, arrive: float = 0.1, empty=(), replace_all=()):
        """The next tick: each task leaves with probability `leave`, about `arrive` times the queue arrives; distros in
        `empty` lose every task, those in `replace_all` every task and get new ones."""
        self.tick += 1
        out = []
        for d, (dist, ts) in enumerate(self.batch):
            if d in empty:
                out.append((dist, []))
                continue
            kept = [] if d in replace_all else [t for t in ts if self.rng.random() >= leave]
            n_new = max(len(ts), 5) if d in replace_all else int(round(len(ts) * arrive)) + (self.rng.randrange(2) if arrive > 0 else 0)
            out.append((dist, kept + [self.task(d) for _ in range(n_new)]))
        self.batch = out
        return out


def string_edit(prev, batch, prev_soa_off, soa=None):
    """The evg_edit_strings edit from `prev` to `batch` (both in canonical order, same distro list): the rows of the
    departed tasks, the arrivals' numeric columns (from `soa`, the marshalled `batch`, when given) and strings."""
    remove, arrivals, ins_rows = [], [], []
    toff = np.concatenate([[0], np.cumsum([len(ts) for _, ts in batch])])
    for d, ((dist, ts), (_, old)) in enumerate(zip(batch, prev)):
        ids = {t.id for t in ts}
        n = sum(1 for t in old if t.id in ids)
        remove.extend(int(prev_soa_off[d]) + k for k, t in enumerate(old) if t.id not in ids)
        arrivals.append((dist, ts[n:]))
        ins_rows.extend(range(int(toff[d]) + n, int(toff[d + 1])))
    rows = np.array(ins_rows, dtype=np.int64)
    if soa is None:
        soa = S.marshal_tasks(batch, NOW, intern=False)[0]
    insert = S.TaskSoA(**{name: getattr(soa, name)[rows] for name, _ in S.TaskSoA.COLUMNS})
    return S.StringEdit(np.array(remove, dtype=np.int64), insert, S.string_cols(arrivals))
