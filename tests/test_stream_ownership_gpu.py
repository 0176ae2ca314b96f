"""GPU: split-K workspace ownership at the benchmark's workload.

Split-K GEMM/conv launches park partial tiles in a workspace slot of the launching stream (the capture stream, for a graph)
and meet on per-tile arrival counters that the last CTA of a tile resets.  Checked here: every stream of the pipelined parser
and every capture stream owns its own slot; the pipelined parser at the benchmark's workload returns bit for bit what the
one-batch-at-a-time path returns; every counter is back at zero after the run and after one launch of each split-K path
class; and a stream that finds every slot taken runs without split-K and still within the fp64 bound."""
import ctypes as C
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
DEV = torch.device("cuda", 0)
N_SLOTS = 24


def _lib():
    from omniparser_b200 import _lib
    return _lib.lib()


def _audit():
    """{slot: non-zero counter words} of every owned slot (synchronises the device)"""
    got = (C.c_int * N_SLOTS)()
    assert _lib().b2p_ws_audit(got, N_SLOTS) == N_SLOTS
    return {i: n for i, n in enumerate(got) if n >= 0}


def _slot(stream):
    return _lib().b2p_ws_slot(stream.cuda_stream)


def _split_k_classes():
    """the first production case of each split-K path class (park-only plans run through b2p_gemm_ln: not here)"""
    import test_gemm_paths_gpu as G
    from gemm_plan_util import FLAG_PARK
    seen, out = set(), []
    for i, c in enumerate(G.PRODUCTION):
        cls = G.cpu_class(c)
        if cls[3] and not c.flags & FLAG_PARK and cls not in seen:
            seen.add(cls)
            out.append(i)
    return out


@pytest.fixture(scope="module")
def models():
    """a detector and captioner of their own (no plan or graph built by another test), as __graft_entry__.standin_models"""
    from omniparser_b200.caption import B200Florence2Model, B200Florence2Processor
    from omniparser_b200.detector import B200YOLOv9Detector
    from standin import florence as FS
    from standin.yolo_weights import yolo_standin
    torch.cuda.set_device(DEV)
    det = B200YOLOv9Detector(state_dict=yolo_standin(0).state_dict(), device=DEV)
    fl = FS.florence_standin(0)
    cap = B200Florence2Model(fl.state_dict(), DEV, FS.GEN, "fp16x3", name_or_path="seeded/florence2-standin")
    return det, {"model": cap, "processor": B200Florence2Processor(None, FS.PROMPT_IDS)}


def test_benchmark_workload_owns_distinct_slots_and_equals_sequential(models):
    """8 x 1920x1080 screenshots per batch (about 60 boxes each), 2 caption lanes, caption group 2, 20 tokens, 6 batches:
    the pipelined parser builds its plans and graphs on its own streams, every role stream and capture stream owns a slot
    of its own, the results equal parse_screenshots batch by batch at the same batch size, and no counter is left dirty."""
    from omniparser_b200 import ops, synth
    from omniparser_b200.utils import PipelinedParser, parse_screenshots
    det, cmp_ = models
    T, lanes, group = 20, 2, 2
    batches = []
    for b in range(6):
        seeds = [100 + 8 * b + i for i in range(8)]
        batches.append(([synth.screenshot(s) for s in seeds], [synth.ocr_boxes(s) for s in seeds]))
    pp = PipelinedParser(det, cmp_, BOX_TRESHOLD=0.05, iou_threshold=0.7, max_new_tokens=T, caption_lanes=lanes, caption_group=group)
    got = list(pp.run(iter(batches)))
    torch.cuda.synchronize()
    roles = ["det", "yolo"] + [f"{r}{lane}" for lane in range(lanes) for r in ("cap", "florence")] + \
            [f"florence{lane}_dec0" for lane in range(lanes)]
    slots = {r: _slot(ops.role_stream(r, DEV)) for r in roles}
    print("[stream slots]", slots, flush=True)
    assert all(s >= 0 for s in slots.values()), slots
    assert len(set(slots.values())) == len(slots), slots
    assert pp.s_det is ops.role_stream("det", DEV) and all(s is ops.role_stream(f"cap{i}", DEV) for i, s in enumerate(pp.s_caps))
    dirty = {i: n for i, n in _audit().items() if n}
    assert not dirty, f"split-K arrival counters left non-zero: {dirty}"
    ref = [parse_screenshots(imgs, det, cmp_, ocr, BOX_TRESHOLD=0.05, iou_threshold=0.7, max_new_tokens=T) for imgs, ocr in batches]
    assert len(got) == len(ref)
    n_caps = 0
    for bi, (gb, rb) in enumerate(zip(got, ref)):
        assert len(gb) == len(rb) == 8
        for si, ((ge_, gi), (re_, ri)) in enumerate(zip(gb, rb)):
            assert [e["bbox"] for e in ge_] == [e["bbox"] for e in re_], f"batch {bi} shot {si}: element boxes differ"
            assert gi.shape == ri.shape and torch.equal(gi, ri), (
                f"batch {bi} (lane {(bi // group) % lanes}) shot {si}: caption ids differ in "
                f"{int((gi != ri).any(1).sum()) if gi.shape == ri.shape else -1} of {ri.shape[0]} rows")
            assert ge_ == re_
            n_caps += ri.shape[0]
    assert n_caps >= 6 * 8 * 10, n_caps         # the benchmark's load: dozens of captioned boxes per screenshot
    dirty = {i: n for i, n in _audit().items() if n}
    assert not dirty, f"split-K arrival counters left non-zero: {dirty}"


def test_counters_reset_after_each_split_k_class():
    """one launch (two: run_case repeats split-K launches) of each split-K path class of the production plans on the
    default stream, each within its fp64 bound; afterwards every owned slot's counters are zero"""
    import test_gemm_paths_gpu as G
    idx = _split_k_classes()
    assert len(idx) >= 4, idx
    for i in idx:
        ratio, p = G.run_case(G.PRODUCTION[i], 3000 + i)
        assert p["ksplit"] > 1
        print(f"[split-K class] case {i}: ksplit {p['ksplit']}, max error / bound {ratio:.3g}", flush=True)
    assert _slot(torch.cuda.current_stream()) >= 0
    dirty = {i: n for i, n in _audit().items() if n}
    assert not dirty, f"split-K arrival counters left non-zero: {dirty}"


_CHILD = r"""
import ctypes as C, sys
sys.path[:0] = [{root!r}, {tests!r}]
import torch
from omniparser_b200 import _lib, ops
import test_gemm_paths_gpu as G

torch.cuda.set_device(0)
lib = _lib.lib()
case = G.PRODUCTION[{case}]


def new_stream():
    h = C.c_void_p(0)
    _lib.check(lib.b2p_stream_create(C.byref(h)))
    return h.value


x = torch.randn(128, 64, device="cuda").half()
w = torch.randn(64, 64, device="cuda").half()
owned = []
for i in range({n_slots}):       # a fresh process: every slot is free; one GEMM per stream claims one
    h = new_stream()
    with torch.cuda.stream(torch.cuda.ExternalStream(h)):
        ops.linear(x, w)
    owned.append((h, lib.b2p_ws_slot(h)))
torch.cuda.synchronize()
assert sorted(s for _, s in owned) == list(range({n_slots})), owned
extra = new_stream()
with torch.cuda.stream(torch.cuda.ExternalStream(extra)):
    ratio, p = G.run_case(case, 4000, slot_free=False)
assert p["ksplit"] > 1 and lib.b2p_ws_slot(extra) == -1
print("no slot left: ksplit 1, max error / bound", ratio, flush=True)
h0, s0 = owned.pop(0)
_lib.check(lib.b2p_stream_destroy(h0))
again = new_stream()
with torch.cuda.stream(torch.cuda.ExternalStream(again)):
    ratio, p = G.run_case(case, 4001)
assert p["ksplit"] > 1 and lib.b2p_ws_slot(again) == s0, (lib.b2p_ws_slot(again), s0)
print("slot", s0, "released and re-claimed: ksplit", p["ksplit"], "max error / bound", ratio, flush=True)
nz = (C.c_int * {n_slots})()
assert lib.b2p_ws_audit(nz, {n_slots}) == {n_slots}
assert all(v == 0 for v in nz), list(nz)
torch.cuda.synchronize()
for h in [extra, again] + [h for h, _ in owned]:
    _lib.check(lib.b2p_stream_destroy(h))
print("CHILD OK", flush=True)
"""


def test_slot_exhaustion_falls_back_to_no_split_k():
    """In a child process (this session's slots stay as they are): 24 streams claim every slot, a split-K production case
    on a 25th stream launches without split-K and stays within its fp64 bound; destroying one stream frees its slot for
    the next stream, which splits K again."""
    case = _split_k_classes()[0]
    code = _CHILD.format(root=str(ROOT), tests=str(ROOT / "tests"), case=case, n_slots=N_SLOTS)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, cwd=str(ROOT),
                       env=dict(os.environ))
    print(r.stdout[-3000:], r.stderr[-3000:], flush=True)
    assert r.returncode == 0 and "CHILD OK" in r.stdout, (r.returncode, r.stderr[-3000:])
