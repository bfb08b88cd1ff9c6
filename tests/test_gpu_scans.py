"""The general path's per-distro tile scan (k_gscan) across its 1024-entry chunks.  One block scans a distro's tile sums
1024 at a time and carries the running total into the next chunk; only a distro of multi-member units spanning more
than 1024 tiles takes that carry."""
import numpy as np
import pytest

import parity
from evergreen_b200 import _lib as L
from evergreen_b200 import synth

pytestmark = pytest.mark.gpu

GTILE = 2048  # kGTile: tasks per general-path tile; tiles start at multiples of 4 tasks


def test_tile_scan_carries_past_1024_tiles(engine):
    """Distro 0 has 3 mod 4 tasks, so distro 1 (MAX_TASKS_PER_DISTRO tasks, with task groups) starts at residue 3 and
    its tiles span 1025: the last tile's run positions come from the carry.  Bit-exact against the oracle."""
    w = synth.make(np.array([4003, L.MAX_TASKS_PER_DISTRO]), 97, zipf_priority=True, tg_frac=0.1, n_hosts=20)
    a, b = (int(x) for x in w.distros.task_off[1:3])
    assert a % 4 == 3 and -(-(b - (a & ~3)) // GTILE) == 1025
    assert int(w.distros.group_off[2] - w.distros.group_off[1]) > 0
    assert (w.tasks.group_id[b - 2:b] < 0).all()  # the last tile's two tasks are placed from the carried offset
    engine.upload(w.tasks, w.distros, w.hosts)
    engine.run(w.now, 0)
    po, ao = engine.download()
    parity.check_against_oracle(w, po, ao)
    parity.check_properties(w, po, ao)
