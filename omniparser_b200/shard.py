"""Multi-GPU sharding of the parse path: screenshots are independent (ref:util/utils.py:417-496 is a pure function of
its inputs), so rank r of R takes screenshots i = r (mod R), weights are replicated, and the only exchange is ONE
gather of fixed-size padded result records to rank 0 per batch (SURVEY.md §8e).  NCCL over NVLink on the GPUs, gloo in
the CPU tests.  The payload (~10 KB per screenshot) is latency-bound; no fused compute+collective kernel is warranted.
"""
from __future__ import annotations

import queue
import threading
from typing import List, Sequence, Tuple

import numpy as np
import torch

from . import ops

# record capacity per screenshot: every detected icon can be captioned (max_det = 300, ref:util/yolov9.py:131 `[:max_det]`;
# the reference captions ALL of them, in chunks of batch_size, ref:util/utils.py:116) and the element list holds the icons
# plus the OCR boxes that survive the overlap filter.  Exceeding a capacity raises: a truncated record would make rank 0
# report something the single-GPU path does not.
REC_TOK = 300
OCR_CAP = 724
REC_BOXES = REC_TOK + OCR_CAP


def shard_indices(n: int, rank: int, world: int) -> List[int]:
    return list(range(rank, n, world))


def record_width(max_new_tokens: int) -> int:
    return 2 + REC_BOXES * 4 + REC_TOK * (max_new_tokens + 1)


def pack_records(results: Sequence[Tuple[list, torch.Tensor]], max_new_tokens: int, out: np.ndarray | None = None) -> torch.Tensor:
    """[(filtered_boxes_elem, caption ids)] -> float32 [B, record_width]: n_elem, n_cap, bboxes[REC_BOXES x 4],
    ids[REC_TOK x (T+1)] (ids padded with the pad token 1; token ids < 2^24 are exact in float32; only the first n_elem /
    n_cap entries are meaningful).  ``out``: write into this (pinned) array instead of allocating."""
    T1 = max_new_tokens + 1
    host = out if out is not None else np.zeros((len(results), record_width(max_new_tokens)), np.float32)
    if out is not None:
        host[:len(results), :2] = 0
    for b, (elems, ids) in enumerate(results):
        nb, nt = len(elems), int(ids.shape[0])
        if nb > REC_BOXES or nt > REC_TOK or ids.shape[1] > T1:
            raise ValueError(f"screenshot {b}: {nb} elements / {nt} captions x {ids.shape[1]} ids exceed the gather record "
                             f"capacity ({REC_BOXES} / {REC_TOK} x {T1})")
        host[b, 0], host[b, 1] = nb, nt
        if nb:
            host[b, 2:2 + nb * 4] = np.asarray([e["bbox"] for e in elems[:nb]], np.float32).ravel()
        if nt:
            tk = np.ones((nt, T1), np.float32)
            tk[:, :ids.shape[1]] = ids[:nt].numpy()
            host[b, 2 + REC_BOXES * 4:2 + REC_BOXES * 4 + tk.size] = tk.ravel()
    return torch.from_numpy(host) if out is None else None


def unpack_records(rec: torch.Tensor, max_new_tokens: int):
    T1 = max_new_tokens + 1
    out = []
    r = rec.cpu().numpy()
    for row in r:
        nb, nt = int(row[0]), int(row[1])
        boxes = row[2:2 + nb * 4].reshape(nb, 4)
        ids = row[2 + REC_BOXES * 4:2 + REC_BOXES * 4 + nt * T1].reshape(nt, T1).astype(np.int64)
        out.append((boxes, ids))
    return out


def gather_records(rec: torch.Tensor, rank: int, world: int, bufs=None):
    """One collective per batch.  Returns the list of per-rank record tensors on rank 0, None elsewhere."""
    import torch.distributed as dist
    if world == 1:
        return [rec]
    if rank == 0 and bufs is None:
        bufs = [torch.zeros_like(rec) for _ in range(world)]
    dist.gather(rec, bufs if rank == 0 else None, dst=0)
    return bufs if rank == 0 else None


class GatherPipe:
    """The per-batch gather, off the submit path: ``submit(results)`` packs the records into a page-locked buffer and
    returns; a worker thread copies them to the device and issues the collective on its OWN stream, so a rank never waits
    for the slowest rank inside its parse loop (gathering synchronously on the default stream and ran the ranks in
    lockstep).  ``drain()`` returns once every submitted gather has completed; rank 0 then holds ``received`` =
    [per-step list of per-rank record tensors].  All collectives of a run are issued by the worker thread, in submit
    order, which is the same on every rank.  CPU tensors + gloo work too (tests/test_shard_cpu.py)."""

    def __init__(self, rank: int, world: int, device, batch: int, max_new_tokens: int, keep: bool = True):
        self.rank, self.world, self.dev, self.T, self.keep = rank, world, torch.device(device), max_new_tokens, keep
        self.shape = (batch, record_width(max_new_tokens))
        self.cuda = self.dev.type == "cuda"
        self.stream = ops.role_stream("gather", self.dev) if self.cuda else None
        self.free: "queue.Queue" = queue.Queue()
        self.work: "queue.Queue" = queue.Queue()
        self.received: list = []
        self.error = None
        self._pending = 0
        self._cv = threading.Condition()
        self._thread = threading.Thread(target=self._run, name="b2p-gather", daemon=True)
        self._thread.start()

    def _slot(self):
        try:
            return self.free.get_nowait()
        except queue.Empty:
            host = torch.zeros(self.shape, dtype=torch.float32)
            if self.cuda:
                host = host.pin_memory()
            dev = torch.zeros(self.shape, dtype=torch.float32, device=self.dev) if self.cuda else host
            bufs = [torch.zeros(self.shape, dtype=torch.float32, device=self.dev) for _ in range(self.world)] if self.rank == 0 else None
            return dict(host=host, dev=dev, bufs=bufs)

    def submit(self, results) -> None:
        if self.error is not None:
            raise self.error
        if self.world == 1:
            return
        sl = self._slot()
        pack_records(results, self.T, out=sl["host"].numpy())
        with self._cv:
            self._pending += 1
        self.work.put(sl)

    def _run(self):
        import torch.distributed as dist
        if self.cuda:
            torch.cuda.set_device(self.dev)
        while True:
            sl = self.work.get()
            if sl is None:
                return
            try:
                if self.cuda:
                    with torch.cuda.stream(self.stream):
                        sl["dev"].copy_(sl["host"], non_blocking=True)
                        dist.gather(sl["dev"], sl["bufs"] if self.rank == 0 else None, dst=0)
                    self.stream.synchronize()
                else:
                    dist.gather(sl["dev"], sl["bufs"] if self.rank == 0 else None, dst=0)
                if self.rank == 0 and self.keep:
                    self.received.append([b.clone() for b in sl["bufs"]])
            except Exception as exc:   # noqa: BLE001  (surfaced by the next submit / drain)
                self.error = exc
            self.free.put(sl)
            with self._cv:
                self._pending -= 1
                self._cv.notify_all()

    def drain(self) -> None:
        with self._cv:
            self._cv.wait_for(lambda: self._pending == 0)
        if self.error is not None:
            raise self.error

    def close(self) -> None:
        self.drain()
        self.work.put(None)
        self._thread.join(timeout=30)


def interleave(per_rank: Sequence[Sequence], n: int, world: int) -> list:
    """Inverse of shard_indices: per-rank result lists back to global screenshot order."""
    out = [None] * n
    for r, items in enumerate(per_rank):
        for k, i in enumerate(shard_indices(n, r, world)):
            out[i] = items[k]
    return out
