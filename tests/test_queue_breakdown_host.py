"""The host side of evg_download_queue_breakdown without a GPU: the binding and its null-context guard, and what the
persist_* mirrors ask of the engine -- with breakdown=False exactly what they asked before (a plain run, TotalValue
only), with breakdown=True the option and the downloaded rows on every item."""
import numpy as np

from evergreen_b200 import _lib as L
from evergreen_b200 import model as M
from evergreen_b200 import scheduler
from evergreen_b200 import soa as S


def test_binding_and_null_context():
    assert L.EVG_OPT_QUEUE_BREAKDOWN == 0x2 and L.EVG_OPT_QUEUE_BREAKDOWN & L.EVG_OPT_BREAKDOWN == 0
    assert L.EVG_ERR_INTERNAL == -5
    lib = L.load()
    off, bd = np.zeros(2, np.int64), np.zeros((1, L.EVG_BD_N), np.int64)
    assert lib.evg_download_queue_breakdown(None, 0, L.ptr(off), L.ptr(bd), 1) == L.EVG_ERR_INVALID
    assert "evg_download_queue_breakdown: null context" in L.last_error()


class FakeEngine:
    """Answers the calls persist_task_queues / persist_alias_task_queues make; every queue ranks its tasks in input
    order, rank r of the tick scored 1000 + r."""

    def __init__(self):
        self.opts, self.bd_calls = [], 0

    def _tick(self, task_off, group_off):
        self.task_off, self.group_off = np.asarray(task_off, np.int64), np.asarray(group_off, np.int64)

    def upload_with_deps(self, soa, table, hosts, deps, fin, now):
        self._tick(table.task_off, table.group_off)

    def download_deps(self):
        T = int(self.task_off[-1])
        return np.ones(T, np.uint8), np.full(T, M.ZERO_TIME, np.int64)

    def plan_aliases(self, table, cfg, now):
        D = cfg.shape[0]
        self._tick(np.zeros(D + 1, np.int64), np.zeros(D + 1, np.int64))
        return self.task_off, self.group_off, np.zeros(D, np.int32)

    def download_alias_map(self):
        return np.zeros(0, np.int32), np.zeros(0, np.int32)

    def run(self, now, opts=0):
        self.opts.append(opts)

    def download(self, want_breakdown=False, want_alloc=None):
        D, G = self.task_off.shape[0] - 1, int(self.group_off[-1])
        po = S.PlanOutput(np.zeros(int(self.task_off[-1]), np.int32), np.zeros(int(self.task_off[-1]), np.int64),
                          np.zeros(D, L.QUEUE_INFO_DTYPE), np.zeros(G, L.GROUP_INFO_DTYPE), None)
        return po, None

    def _rows(self, cap):
        cap = cap or L.EVG_PERSISTED_QUEUE_CAP
        n = np.minimum(np.diff(self.task_off), cap)
        off = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
        ranks = np.concatenate([np.arange(int(k)) for k in n] + [np.zeros(0, np.int64)]).astype(np.int64)
        return off, ranks

    def download_queue(self, cap=0, task_off=None):
        off, ranks = self._rows(cap)
        items = np.zeros(ranks.shape[0], L.QUEUE_ITEM_DTYPE)
        items["task"] = ranks
        items["total_value"] = 1000 + np.arange(ranks.shape[0])
        return off, items

    def download_queue_breakdown(self, cap=0, task_off=None):
        self.bd_calls += 1
        off, ranks = self._rows(cap)
        bd = np.arange(ranks.shape[0] * L.EVG_BD_N, dtype=np.int64).reshape(-1, L.EVG_BD_N)
        bd[:, L.EVG_BD_TOTAL_VALUE] = 1000 + np.arange(ranks.shape[0])
        return off, bd


def batch():
    out = []
    for d, n in enumerate([3, 0, 5]):
        tasks = [M.Task(id=f"d{d}t{i}", distro_id=f"d{d}", version="v", priority=i) for i in range(n)]
        out.append((M.Distro(id=f"d{d}"), tasks))
    return out


def test_persist_default_is_unchanged_and_breakdown_fills_every_field():
    eng = FakeEngine()
    qs = scheduler.persist_task_queues(batch(), 10 ** 18, engine=eng, cap=4)
    assert eng.opts == [0] and eng.bd_calls == 0
    tv = [[it.sorting_value_breakdown for it in q.queue] for q in qs]
    assert tv == [[M.SortingValueBreakdown(total_value=1000 + k) for k in ks] for ks in ([0, 1, 2], [], [3, 4, 5, 6])]
    eng = FakeEngine()
    b = batch()
    qs = scheduler.persist_task_queues(b, 10 ** 18, engine=eng, cap=4, breakdown=True)
    assert eng.opts == [L.EVG_OPT_QUEUE_BREAKDOWN] and eng.bd_calls == 1
    rows = [it.sorting_value_breakdown.row() for q in qs for it in q.queue]
    want = np.arange(7 * L.EVG_BD_N).reshape(-1, L.EVG_BD_N)
    want[:, L.EVG_BD_TOTAL_VALUE] = 1000 + np.arange(7)
    assert rows == want.tolist()
    assert [t.sorting_value_breakdown.row() for t in b[0][1]] == want[:3].tolist()  # the task carries it too
    eng = FakeEngine()
    q = scheduler.PersistTaskQueue(*batch()[2], now=10 ** 18, engine=eng, breakdown=True)
    assert eng.opts == [L.EVG_OPT_QUEUE_BREAKDOWN] and len(q.queue) == 5


def test_persist_alias_default_asks_for_no_breakdown():
    for breakdown, opts, calls in ((False, 0, 0), (True, L.EVG_OPT_QUEUE_BREAKDOWN, 1)):
        eng = FakeEngine()
        kw = {"breakdown": True} if breakdown else {}
        qs = scheduler.persist_alias_task_queues([M.Distro(id="a"), M.Distro(id="b")], [], 10 ** 18, engine=eng, **kw)
        assert eng.opts == [opts] and eng.bd_calls == calls and [q.queue for q in qs] == [[], []]
