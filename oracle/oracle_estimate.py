"""CPU restatement of the task start-time estimator (model/task_start_estimation.go), statement by statement.

Simulator is the reference's estimatedTimeSimulator OBJECT: simulate(pos) sorts the pool on every call and keeps
currentPos, timeElapsed and the dequeued tasks between calls, which is how the reference's own tests drive it
(model/task_start_estimation_test.go).  GetEstimatedStartTime builds a fresh simulator per request (:121), so in
production the pool is sorted once: fresh_estimates() is that, for every position of a queue at once.  The two differ
as soon as an insertion leaves the pool unsorted and a later call sorts it again.

All values are int64 nanoseconds with Go's wrapping arithmetic.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

MINUTE = 60 * 10 ** 9
HOST_INITIALIZING_DELAY = 4 * MINUTE   # :19
HOST_STARTING_DELAY = 3 * MINUTE       # :20
HOST_PROVISIONING_DELAY = 1 * MINUTE   # :21

HOST_UNINITIALIZED, HOST_STARTING, HOST_PROVISIONING, HOST_RUNNING = "initializing", "starting", "provisioning", "running"  # globals.go:24-36
ZERO_TIME = -(2 ** 63)
I64_MAX, I64_MIN = 2 ** 63 - 1, -(2 ** 63)

LOOKUP_ERROR = object()  # running_tasks value: task.FindOneIdAndExecution returned an error (:142-147)


def wrap(x: int) -> int:
    """int64 two's-complement wrap."""
    return (x + 2 ** 63) % 2 ** 64 - 2 ** 63


def since(now: int, t: int) -> int:
    """time.Since(t) at a frozen clock; saturates like time.Time.Sub."""
    if t == ZERO_TIME:
        return I64_MAX
    return max(I64_MIN, min(I64_MAX, now - t))


class Simulator:
    """estimatedTimeSimulator (:34-39)."""

    def __init__(self, durations: Sequence[int] = (), hosts: Sequence[int] = ()):
        self.tasks: List[int] = list(durations)   # estimatedTaskQueue.Items
        self.hosts: List[int] = list(hosts)       # estimatedHostPool: timeToCompletion of each host
        self.time_elapsed = 0
        self.current_pos = 0

    def simulate(self, pos: int) -> int:  # :53-67
        if len(self.hosts) == 0:
            return -1
        if len(self.tasks) == 0:
            return -1
        self.hosts.sort()
        while self.current_pos <= pos:
            self.dispatch_next_task()
            self.current_pos += 1
        return self.time_elapsed

    def dispatch_next_task(self) -> None:  # :69-96
        count = len(self.hosts)
        fast_forward = self.hosts[0]
        self.time_elapsed = wrap(self.time_elapsed + fast_forward)
        self.hosts = self.hosts[1:]
        for i in range(len(self.hosts)):
            self.hosts[i] = wrap(self.hosts[i] - fast_forward)
        duration = self.tasks.pop(0)  # Dequeue
        for i in range(count):
            if i < count - 2:
                if self.hosts[i] <= duration and self.hosts[i + 1] >= duration:
                    self.hosts = self.hosts[:i] + [duration] + self.hosts[i:]
                    return
            else:
                self.hosts.append(duration)
                return


def create_simulator_model(durations: Sequence[int], hosts: Sequence, running_tasks: dict, now: int) -> Simulator:
    """createSimulatorModel (:124-163).  `hosts`: objects with status and running_task, in query order;
    running_tasks[id]: an object with expected_duration and dispatch_time, None / absent for "no document" (the host
    is skipped, :148-154), LOOKUP_ERROR for a failed lookup (the pool built so far is returned, :142-147)."""
    est = Simulator(durations)
    for h in hosts:
        if h.status == HOST_UNINITIALIZED:
            est.hosts.append(HOST_INITIALIZING_DELAY)
        elif h.status == HOST_STARTING:
            est.hosts.append(HOST_STARTING_DELAY)
        elif h.status == HOST_PROVISIONING:
            est.hosts.append(HOST_PROVISIONING_DELAY)
        elif h.status == HOST_RUNNING:
            if h.running_task == "":
                est.hosts.append(0)
            else:
                t = running_tasks.get(h.running_task)
                if t is LOOKUP_ERROR:
                    return est
                if t is None:
                    continue
                est.hosts.append(wrap(t.expected_duration - since(now, t.dispatch_time)))
    return est


def fresh_estimates(durations: Sequence[int], pool: Sequence[int]) -> List[int]:
    """What a FRESH simulator's simulate(p) returns for every p: one sort, one run, every prefix."""
    if len(pool) == 0 or len(durations) == 0:
        return [-1] * len(durations)
    s = Simulator(durations, pool)
    s.hosts.sort()
    out = []
    for _ in range(len(durations)):
        s.dispatch_next_task()
        out.append(s.time_elapsed)
    return out


def get_estimated_start_time(task_id: str, queue_ids: Optional[Sequence[str]], durations: Sequence[int], hosts: Sequence,
                             running_tasks: dict, now: int) -> int:
    """GetEstimatedStartTime (:99-122): queue_ids None = no queue document."""
    if queue_ids is None:
        return -1
    if task_id not in queue_ids:
        return -1
    return create_simulator_model(durations, hosts, running_tasks, now).simulate(list(queue_ids).index(task_id))
