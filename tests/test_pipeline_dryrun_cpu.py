"""CPU dry run of ``PipelinedParser`` end to end (threads, lanes, io slots, caption grouping): the CUDA library is the
recorder of test_plan_dryrun_cpu.py (no arithmetic), the detector is a stub that "finds" fixed boxes, CUDA streams/events are
dummies.  What is checked is the host-side plumbing the GPU tests cannot reach without hardware time: every code path of
``_submit`` / ``_glue`` / ``_caption_group`` runs, results come back per batch in order with the right
shapes, crops of a group land in consecutive row blocks of ONE plan, and the opt-in grouping launches fewer Florence passes."""
import contextlib
import ctypes as C
import threading

import numpy as np
import pytest
import torch

from omniparser_b200 import _lib, ops
from standin import florence as FS
from test_plan_dryrun_cpu import _Recorder, _Stream

H, W, B = 270, 480, 2


class _Event:
    def record(self, *a):
        pass

    def synchronize(self):
        pass


class _FakeDetector:
    """B200YOLOv9Detector stand-in: same io dictionary keys, 'detects' 3 + (batch parity) boxes per screenshot."""

    def __init__(self):
        self.device = torch.device("cpu")
        self._io = {}
        self.lock = threading.Lock()
        self._lock = threading.RLock()          # the handle-level lock of the real detector
        self.n = 0

    @staticmethod
    def check_capacity(cand_count_host, cap):
        assert int(cand_count_host.max()) <= cap

    def io_slot(self, sizes, imgsz, max_det, slot=0, drain=None):
        (H_, W_), B_ = sizes[0], len(sizes)
        key = (B_, H_, W_, slot)
        if key not in self._io:
            self._io[key] = dict(src=torch.zeros((B_, H_, W_, 3), dtype=torch.uint8), B=B_,
                                 host_count=torch.zeros((B_,), dtype=torch.int32), host_box=torch.zeros((B_, max_det, 4)),
                                 out_count=torch.zeros((B_,), dtype=torch.int32), out_box=torch.zeros((B_, max_det, 4)),
                                 cand_count=torch.zeros((B_,), dtype=torch.int32), host_cand=torch.zeros((B_,), dtype=torch.int32), cap=8400,
                                 meta_hw=torch.tensor([[H_, W_]] * B_, dtype=torch.int32),
                                 meta_off=torch.tensor([i * H_ * W_ * 3 for i in range(B_)], dtype=torch.int64))
        return self._io[key]

    @staticmethod
    def stage(io, images, resident=None):
        for i, im in enumerate(images):
            io["src"][i].copy_(torch.from_numpy(im))

    def filter_device(self, io, ocr_elems, iou_threshold, max_det=300):
        return False      # "more OCR boxes than the device filter takes": the pipeline runs the host list logic (host_glue)

    def detect(self, io, conf, iou, max_det):
        with self.lock:
            k = 3 + self.n % 2
            self.n += 1
        for i in range(io["B"]):
            for j in range(k):
                io["out_box"][i, j] = torch.tensor([20.0 + 60 * j, 30.0 + 10 * i, 60.0 + 60 * j, 80.0 + 10 * i])
            io["out_count"][i] = k


def _cap_model(florence):
    from omniparser_b200.caption import B200Florence2Model, DEFAULT_GEN
    from omniparser_b200.florence_engine import FlorenceWeights
    m = object.__new__(B200Florence2Model)
    m.device = torch.device("cpu")
    m.gen = dict(DEFAULT_GEN)
    m.weights = FlorenceWeights(florence.state_dict(), m.device, m.gen, "fp16x3")
    m.use_graph = False
    m._plans = {}
    m._plan_lock = threading.Lock()
    m._lock = threading.RLock()
    return m


@pytest.fixture()
def env(monkeypatch):
    rec = _Recorder()
    monkeypatch.setattr(_lib, "_lib", rec)
    monkeypatch.setattr(ops, "_stream", lambda: C.c_void_p(0))
    for name, val in [("device", lambda *a, **k: contextlib.nullcontext()), ("stream", lambda *a, **k: contextlib.nullcontext()),
                      ("Stream", _Stream), ("Event", _Event), ("current_stream", lambda *a, **k: _Stream()),
                      ("synchronize", lambda *a, **k: None), ("set_device", lambda *a, **k: None)]:
        monkeypatch.setattr(torch.cuda, name, val)
    return rec


@pytest.fixture(scope="module")
def florence():
    return FS.florence_standin(0)


def _batches(n):
    rng = np.random.default_rng(0)
    out = []
    for b in range(n):
        imgs = [rng.integers(0, 256, size=(H, W, 3), dtype=np.uint8) for _ in range(B)]
        ocr = [([f"t{b}"], [[5, 5, 45, 20]]) for _ in range(B)]
        out.append((imgs, ocr))
    return out


@pytest.mark.parametrize("lanes,group", [(1, 1), (2, 1), (2, 2), (1, 3)])
def test_pipelined_parser_stage_plumbing(env, florence, lanes, group):
    from omniparser_b200.caption import B200Florence2Processor
    from omniparser_b200.utils import PipelinedParser
    det = _FakeDetector()
    cmp_ = dict(model=_cap_model(florence), processor=B200Florence2Processor())
    pp = PipelinedParser(det, cmp_, BOX_TRESHOLD=0.05, iou_threshold=0.7, max_new_tokens=3, caption_lanes=lanes, caption_group=group)
    nb = 7
    got = list(pp.run(iter(_batches(nb))))
    assert len(got) == nb
    for out in got:
        assert len(out) == B
        for elems, ids in out:
            n_icon = sum(1 for e in elems if e["source"] == "box_yolo_content_yolo")
            assert n_icon in (3, 4) and ids.shape[0] == n_icon and ids.dtype == torch.long
            assert all(isinstance(e["content"], str) for e in elems)
    names = [c[0] for c in env.calls]
    n_crops_calls = names.count("b2p_crop_resize")
    n_passes = names.count("b2p_encoder_embed")                  # one per Florence-2 encode
    assert n_crops_calls == nb                                    # every batch cuts its own crops from its own slot
    assert n_passes == -(-nb // group)                            # grouped: one Florence pass per group of batches
    assert pp.timings["batches"] == nb and pp.timings["n_crops"] == sum(ids.shape[0] for out in got for _, ids in out)
    # crop blocks of a group are consecutive row blocks of the same plan buffer
    plans = list(cmp_["model"]._plans.values())
    base = {p.crops.data_ptr(): p for p in plans}
    crop_calls = [c[1] for c in env.calls if c[0] == "b2p_crop_resize"]
    for a in crop_calls:
        dst, n_box = a[7], a[5]
        owner = [p for ptr, p in base.items() if ptr <= dst < ptr + p.crops.numel()]
        assert len(owner) == 1 and (dst - owner[0].crops.data_ptr()) % (64 * 64 * 3) == 0 and n_box in (2 * 3, 2 * 4)


@pytest.mark.parametrize("caption_size", [64, 768])
def test_parse_screenshots_stage_plumbing(env, florence, monkeypatch, caption_size):
    """the one-batch-at-a-time entry point, both caption modes (768: device resize + chunked generate)"""
    from omniparser_b200 import caption
    from omniparser_b200.caption import B200Florence2Processor
    from omniparser_b200.utils import ParseTimings, parse_screenshots
    monkeypatch.setattr(caption, "BUCKET_768", 1)        # one crop per chunk keeps the CPU-side buffers small
    det = _FakeDetector()
    cmp_ = dict(model=_cap_model(florence), processor=B200Florence2Processor())
    (imgs, ocr), = _batches(1)
    boxes = [[[10.0, 10.0, 60.0, 70.0], [100.0, 40.0, 150.0, 90.0], [300.0, 100.0, 380.0, 180.0]], []]
    tm = ParseTimings()
    out = parse_screenshots(imgs, det, cmp_, ocr, BOX_TRESHOLD=0.05, iou_threshold=0.7, max_new_tokens=2, timings=tm,
                            _det_override=boxes, caption_size=caption_size)
    assert [ids.shape[0] for _, ids in out] == [3, 0] and tm["n_crops"] == 3
    names = [c[0] for c in env.calls]
    assert names.count("b2p_crop_resize") == 1
    if caption_size == 768:
        assert names.count("b2p_resize_u8") == 3 and names.count("b2p_encoder_embed") == 3      # three chunks of one crop
    else:
        assert "b2p_resize_u8" not in names and names.count("b2p_encoder_embed") == 1
