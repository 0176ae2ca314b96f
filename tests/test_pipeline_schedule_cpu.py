"""Host-side schedule of ``PipelinedParser.run`` (no GPU): stages are stubbed with sleeps that record what overlaps.

Invariants (the second one was violated by a shared caption thread pool: batch i+2 could start on lane 0 while batch i
was still decoding there, corrupting the lane's plan state):
  * results come back in order, one per batch;
  * two batches of the same caption lane are never in flight together, while different lanes do overlap;
  * a batch's io slot is not handed to a later detection before the batch's caption stage has finished.
"""
import contextlib
import random
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import pytest

from omniparser_b200.utils import PipelinedParser


class _Sched(PipelinedParser):
    def __init__(self, lanes, seed, group=1):   # no CUDA objects: only what run() itself touches
        self.lanes, self.group = lanes, group
        self._pool = ThreadPoolExecutor(max_workers=1)
        self._cap_pools = [ThreadPoolExecutor(max_workers=1) for _ in range(lanes)]
        self._job = 0
        self.rng = random.Random(seed)
        self.lock = threading.Lock()
        self.active_lanes, self.busy_slots = {}, {}
        self.max_parallel, self.errors = 0, []

    def _device_ctx(self):
        return contextlib.nullcontext()

    def _ensure_plan(self, g, pending, fut):
        pass

    def _ensure_io(self, slot, images, pending):
        return slot

    def _submit(self, slot, images, resident_src=None, ocr=None):
        with self.lock:
            if slot in self.busy_slots:
                self.errors.append(f"slot {slot} reused while batch {self.busy_slots[slot]} still owns it")
            self.busy_slots[slot] = images
        time.sleep(self.rng.uniform(0.0, 0.004))
        return dict(slot=slot, batch=images)

    def _glue(self, h, ocr):
        time.sleep(self.rng.uniform(0.0, 0.003))
        lane = (self._job // self.group) % self.lanes
        self._job += 1
        return dict(h=h, lane=lane, crop_boxes=[0], n_crops=1)

    def _caption_group(self, gs):
        lane, batches = gs[0]["lane"], [g["h"]["batch"] for g in gs]
        assert all(g["lane"] == lane for g in gs) and len(gs) <= self.group
        with self.lock:
            if lane in self.active_lanes:
                self.errors.append(f"lane {lane}: group {batches} started while {self.active_lanes[lane]} was in flight")
            self.active_lanes[lane] = batches
            self.max_parallel = max(self.max_parallel, len(self.active_lanes))
        time.sleep(self.rng.choice([0.001, 0.004, 0.012]))
        with self.lock:
            del self.active_lanes[lane]
            for g in gs:
                del self.busy_slots[g["h"]["slot"]]
        return batches


@pytest.mark.parametrize("group", [1, 2, 3])
@pytest.mark.parametrize("lanes", [1, 2, 3])
@pytest.mark.parametrize("seed", [0, 1])
def test_schedule_invariants_through_caption_group(lanes, seed, group):
    s = _Sched(lanes, seed, group)
    n = 41
    out = list(s.run((i, None) for i in range(n)))
    assert out == list(range(n))
    assert not s.errors, s.errors[:3]
    if lanes > 1:
        assert s.max_parallel > 1, "caption lanes never overlapped"
    assert list(s.run(iter(()))) == []
    assert list(s.run([(7, None)])) == [7]


def test_group_trim_matches_per_batch_stop():
    """Grouped captioning generates until EVERY row of the group has finished; a batch captioned alone would have stopped
    at the first step where all of ITS rows had finished (HF semantics), so its slice is trimmed there."""
    import torch
    from omniparser_b200.caption import B200Florence2Model
    m = object.__new__(B200Florence2Model)
    m.gen = dict(eos_token_id=2, pad_token_id=1)
    g = torch.Generator().manual_seed(0)
    for _ in range(50):
        T = 9
        rows = []
        for _r in range(7):
            L = int(torch.randint(2, T + 3, (1,), generator=g))          # eos position (may be beyond T: unfinished)
            body = torch.randint(5, 100, (T,), generator=g)
            row = torch.cat([torch.tensor([2]), body])                    # decoder start, then tokens
            if L <= T:
                row[L] = 2
                row[L + 1:] = 1
            rows.append(row)
        seq = torch.stack(rows)
        # what the group pass returns: truncated where ALL rows are done
        d_all = m._first_all_finished(seq)
        grp = seq[:, :d_all + 1] if d_all is not None else seq
        for sl in (slice(0, 3), slice(3, 7)):
            alone = seq[sl]
            d = m._first_all_finished(alone)
            alone = alone[:, :d + 1] if d is not None else alone
            part = grp[sl]
            dp = m._first_all_finished(part)
            part = part[:, :dp + 1] if dp is not None else part
            assert torch.equal(part, alone)
