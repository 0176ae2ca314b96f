"""The reference's three-function API (``ref:util/utils.py``) on the GPU path.

``get_yolo_model`` / ``get_caption_model_processor`` / ``get_som_labeled_img`` keep the reference signatures,
argument meaning, return schema and error behaviour, so ``util/omniparser.py`` (ref:util/omniparser.py:1,12-13,30),
``gradio_demo.py`` and the eval harness can import them from here instead of ``util.utils`` (see INTEGRATION.md).

``parse_screenshots`` is the batched form the benchmark and the multi-GPU driver use: detector -> host list logic
-> device crop+resize -> caption, one H2D copy of the u8 screenshots and two small D2H reads per batch.
"""
from __future__ import annotations

import base64
import io
import os
import threading
import time
from pathlib import Path
from typing import List, Optional, Sequence, Union

import numpy as np
import torch
from PIL import Image

from . import host_glue, ops, som_overlay
from .caption import (CAPTION_PROMPT_IDS, B200Florence2Model, B200Florence2Processor, beam_settings, find_tokenizer_dir,
                      load_beam_defaults, load_florence_state, load_tokenizer)
from .detector import B200YOLOv9Detector


def get_yolo_model(model_path=None, device=None, precision=None):
    """ref:util/utils.py:72-85.  Only the YOLOv9-E ``icon_detect_v3`` branch exists here (no ultralytics fallback).
    ``precision`` (extension): "fp16" (default, the reference's CUDA autocast precision) or "fp16x3" (parity grade: the
    fp32 CPU path's boxes); default from B2P_DETECTOR_PRECISION."""
    if model_path is None:
        local = Path(__file__).resolve().parents[1] / "weights/icon_detect_v3/model.pt"
        if local.is_file():
            model_path = local
    if model_path is None:
        raise FileNotFoundError("weights/icon_detect_v3/model.pt not found and no network access: pass model_path")
    return B200YOLOv9Detector(model_path=model_path, device=device, precision=precision)


def get_caption_model_processor(model_name, model_name_or_path="microsoft/Florence-2-base", device=None,
                                precision: str = "fp16x3", tokenizer_path=None, allow_id_captions: Optional[bool] = None):
    """ref:util/utils.py:48-69 (florence2 branch).  ``model_name_or_path`` must be a local directory holding
    ``model.safetensors`` (+ ``generation_config.json``).  The detokeniser (the reference takes it from the hub id
    ``microsoft/Florence-2-base``, :64) is looked up offline by :func:`caption.find_tokenizer_dir`; if none is found
    this raises -- captions made of id tags (``<25924> <13>``) are only produced when the caller opts in with
    ``allow_id_captions=True`` / B2P_ALLOW_ID_CAPTIONS=1."""
    if model_name != "florence2":
        raise NotImplementedError(f"caption model {model_name!r}: only the florence2 branch is on the GPU hot path")
    if not device:
        device = "cuda"
    if allow_id_captions is None:
        allow_id_captions = bool(os.environ.get("B2P_ALLOW_ID_CAPTIONS"))
    tdir = find_tokenizer_dir(model_name_or_path, tokenizer_path)
    if tdir is None and not allow_id_captions:
        raise FileNotFoundError(
            "no Florence-2 tokenizer files (tokenizer.json or vocab.json + merges.txt) found for the caption processor: "
            "pass tokenizer_path=, set B2P_FLORENCE_PROCESSOR, or put them next to the weights "
            "(allow_id_captions=True returns token-id tags instead of strings)")
    sd, gen = load_florence_state(model_name_or_path)
    tok = load_tokenizer(tdir) if tdir is not None else None
    model = B200Florence2Model(sd, device, gen, precision, name_or_path=str(model_name_or_path),
                               beam_defaults=load_beam_defaults(model_name_or_path))
    if "florence" not in model.config.name_or_path.lower():
        model.config.name_or_path = "florence2:" + model.config.name_or_path   # ref:util/utils.py:109 looks for 'florence'
    return {"model": model, "processor": B200Florence2Processor(tok)}


# ------------------------------------------------------------------------------------------------ batched hot path
class ParseTimings(dict):
    pass


# B2P_HOST_GLUE=1: run the reference's list logic (overlap filter, ref:util/utils.py:241-319) on the host (host_glue.py) instead
# of the device kernel b2p_overlap_filter -- identical results (tests/test_pipeline_gpu.py), kept for A/B timing and as the path
# for screenshots with more OCR boxes than the kernel takes
_HOST_GLUE = bool(os.environ.get("B2P_HOST_GLUE"))


def _check_crop_status(status: torch.Tensor) -> None:
    """b2p_crop_resize flags crops whose truncated box is empty.  The reference silently skips such a crop
    (ref:util/utils.py:104-105) and then mis-assigns every later caption; int_box_area > 0 (:444-445) makes it impossible
    on this path, so a flagged crop is a bug and raises.  ``status`` is the host copy, made on the stream before the
    ids' D2H sync: checking it costs no kernel and no extra synchronisation."""
    bad = int(status.count_nonzero().item())
    if bad:
        raise RuntimeError(f"{bad} crop boxes were empty after truncation (status flags of b2p_crop_resize)")


def _detect(model: B200YOLOv9Detector, io_, sizes, ocr, conf, iou_threshold):
    """Stage 1, on the current stream, after ``model.stage``: detection, the overlap filter on the device (unless
    B2P_HOST_GLUE is set or a screenshot has more OCR boxes than the kernel takes), then async copies of the counts, boxes
    and candidate counts into the slot's pinned mirrors and an event behind them (no host sync) -> the batch's handle."""
    model.detect(io_, conf, 0.1, 300)
    ocr_elems, on_device = None, False
    if not _HOST_GLUE:
        ocr_elems = [host_glue.ocr_elements((torch.tensor(ob) / torch.Tensor([w, h, w, h])).tolist() if ob else None, tx, w, h)
                     for (h, w), (tx, ob) in zip(sizes, ocr)]   # :437-444
        on_device = model.filter_device(io_, ocr_elems, iou_threshold, 300)
    io_["host_count"].copy_(io_["out_count"], non_blocking=True)
    if not on_device:
        io_["host_box"].copy_(io_["out_box"], non_blocking=True)
    io_["host_cand"].copy_(io_["cand_count"], non_blocking=True)
    ev = torch.cuda.Event()
    ev.record()
    return dict(io=io_, ev=ev, sizes=sizes, ocr_elems=ocr_elems, on_device=on_device)


def _host_lists(model: B200YOLOv9Detector, h, ocr, iou_threshold, det_override=None):
    """Stage 2, after stage 1's event: the box counts and the crop list of a batch.  When the overlap filter ran on the
    device, the crop list stays there and the element lists are built later from its flags (:func:`_elements`); otherwise
    the reference's host list logic runs per screenshot.  ``det_override`` (tests) replaces the detector's boxes."""
    io_ = h["io"]
    if det_override is None:
        counts, boxes = io_["host_count"].tolist(), io_["host_box"]
        model.check_capacity(io_["host_cand"], io_["cap"])
    else:
        counts = [len(b) for b in det_override]
        boxes = [torch.as_tensor(b, dtype=torch.float32).reshape(-1, 4) for b in det_override]
    g = dict(h=h, counts=counts, all_elems=None, crop_boxes=[], crop_img=[])
    if h["on_device"]:
        g["n_crops"] = int(io_["host_crop_counts"][len(counts)])
        return g
    g["all_elems"] = []
    for i, (hi, wi) in enumerate(h["sizes"]):
        whwh = torch.Tensor([wi, hi, wi, hi])
        xyxy = (boxes[i][:counts[i]] / whwh).tolist()                         # ref:util/utils.py:432
        texts, obox = ocr[i]
        oratio = (torch.tensor(obox) / whwh).tolist() if obox else None       # :437-442
        elems, _ = host_glue.build_elements(xyxy, oratio, texts, wi, hi, iou_threshold)
        g["all_elems"].append(elems)
        for e in elems:
            if e["content"] is None:
                g["crop_boxes"].append(e["bbox"])
                g["crop_img"].append(i)
    g["n_crops"] = len(g["crop_boxes"])
    return g


def _elements(model: B200YOLOv9Detector, g):
    """A batch's element lists; built here from the device overlap filter's flags if stage 2 left them to later."""
    if g["all_elems"] is None:
        h = g["h"]
        g["all_elems"] = [model.elements_from_io(h["io"], i, n, h["ocr_elems"][i]) for i, n in enumerate(g["counts"])]
    return g["all_elems"]


def _cut_crops(gs, dst):
    """Stage 3, on the current stream: the 64x64 crops of each batch of ``gs``, cut from its slot's screenshots into
    consecutive row blocks of ``dst`` -> the status flags of b2p_crop_resize (see :func:`_check_crop_status`)."""
    status = torch.zeros((sum(g["n_crops"] for g in gs),), dtype=torch.int32, device=dst.device)
    off = 0
    for g in gs:
        n, io_ = g["n_crops"], g["h"]["io"]
        if not n:
            continue
        if g["h"]["on_device"]:
            boxes, img = io_["crop_box"], io_["crop_img"]
        else:
            boxes = torch.tensor(g["crop_boxes"], dtype=torch.float32).to(dst.device, non_blocking=True)
            img = torch.tensor(g["crop_img"], dtype=torch.int32).to(dst.device, non_blocking=True)
        ops.crop_resize(io_["src"], io_["meta_hw"], io_["meta_off"], boxes, img, n, 64, dst[off:], status[off:])
        off += n
    return status


def _results(processor, all_elems, ids):
    """Stage 4: captions into the element lists -> per screenshot ``(elements, caption ids)``, ids in crop order."""
    texts = [t.strip() for t in processor.batch_decode(ids, skip_special_tokens=True)] if ids is not None else []
    out, k = [], 0
    for elems in all_elems:
        m = sum(1 for e in elems if e["content"] is None)
        host_glue.fill_captions(elems, texts[k:k + m])
        out.append((elems, ids[k:k + m] if ids is not None else torch.zeros((0, 1), dtype=torch.long)))
        k += m
    return out


@torch.inference_mode()
def parse_screenshots(images: Sequence[np.ndarray], model: B200YOLOv9Detector, caption_model_processor: dict,
                      ocr: Sequence[tuple], BOX_TRESHOLD=0.01, iou_threshold=0.9, imgsz=640, max_new_tokens=20,
                      prompt_ids: Sequence[int] = CAPTION_PROMPT_IDS, timings: Optional[ParseTimings] = None,
                      _skip_h2d: bool = False, _det_override=None, caption_size: int = 64, num_beams: int = 1,
                      early_stopping=None, length_penalty=None):
    """``caption_size`` 64 = the reference's CUDA branch (crops captioned at 64x64, ref:util/utils.py:121); 768 = its
    CPU branch (CLIP processor bicubic-resizes every crop to 768x768 first, :123), done on the device, in chunks.
    u8 HWC screenshots (of one size, or of different sizes: those share one detector batch through the ragged letterbox)
    + per-image ``(ocr_text, ocr_bbox_xyxy_pixels)`` -> per-image
    ``(filtered_boxes_elem, caption_token_ids)``; the compute of ``get_som_labeled_img`` without the overlay drawing.
    NMS IoU is fixed at 0.1 as in ref:util/utils.py:431; ``iou_threshold`` feeds the overlap filter (:446).
    ``num_beams`` > 1 captions with HF beam search (one caption per crop; early_stopping / length_penalty default to the
    caption model's ``beam_defaults``)."""
    bs = beam_settings(num_beams, False, early_stopping, length_penalty, 1, caption_model_processor["model"].beam_defaults)
    bs.pop("num_return_sequences")
    sizes = [tuple(im.shape[:2]) for im in images]
    if _skip_h2d and len(set(sizes)) > 1:
        raise ValueError("_skip_h2d takes screenshots of one size: a batch of different sizes has no resident one-size buffer")
    cap_model: B200Florence2Model = caption_model_processor["model"]
    t0 = time.perf_counter()
    with model._lock, torch.cuda.device(model.device):   # io slot 0 / caption plan instance 0 are this handle's: one call at a time
        io_ = model.io_slot(sizes, imgsz, 300)
        if not _skip_h2d:   # bench "value" leg: the u8 screenshots are already resident in io_["src"]
            model.stage(io_, images)
        if _det_override is None:
            h = _detect(model, io_, sizes, ocr, BOX_TRESHOLD, iou_threshold)
            h["ev"].synchronize()
        else:   # tests: inject detector output (e.g. the golden boxes) to pin the stages after it exactly
            h = dict(io=io_, sizes=sizes, on_device=False)
        t1 = time.perf_counter()
        g = _host_lists(model, h, ocr, iou_threshold, _det_override)
        n = g["n_crops"]
        t2 = time.perf_counter()
        ids = None
        if n:
          with cap_model._lock:   # plan instance 0 of the caption handle (also what model.generate() uses)
            if caption_size == 64:
                plan = cap_model.plan_for(n, max_new_tokens, prompt_ids, **bs)
                crops = plan.crops
            else:
                crops = torch.empty((n, 64, 64, 3), dtype=torch.uint8, device=model.device)
            status = _cut_crops([g], crops)
            if caption_size == 64:
                ids = cap_model.generate_from_device_crops(plan, n)
            else:
                ids = cap_model.generate_chunked(crops, max_new_tokens, prompt_ids, from_resized=False, **bs)
            _elements(model, g)   # device overlap filter: element lists from its flags, while the GPU captions
            status = status.to("cpu", non_blocking=True)   # completed by the ids' D2H sync below
            ids = ids.cpu()
            _check_crop_status(status)
        all_elems = _elements(model, g)
        t3 = time.perf_counter()
    out = _results(caption_model_processor["processor"], all_elems, ids)
    if timings is not None:
        timings.update(detect_s=t1 - t0, glue_s=t2 - t1, caption_s=t3 - t2, n_boxes=sum(g["counts"]), n_crops=n)
    return out


class _Member:
    """Result handle of one batch inside a grouped caption job."""

    def __init__(self, fut, idx):
        self.fut, self.idx = fut, idx

    def result(self):
        return self.fut.result()[self.idx]


class PipelinedParser:
    """Three-stage software pipeline over batches of screenshots: detection of batch i+1 (stream A), the host
    list logic of batch i and the captioning of batch i-1 (stream B) run concurrently.  Same results as :func:`parse_screenshots`, batch by
    batch; only the scheduling differs.  Usage::

        pp = PipelinedParser(model, caption_model_processor, BOX_TRESHOLD=0.05, iou_threshold=0.7)
        for result in pp.run(iter_of_(images, ocr)):   # result = [(elems, ids), ...] per batch, in order
            ...
    """

    def __init__(self, model: B200YOLOv9Detector, caption_model_processor: dict, BOX_TRESHOLD=0.01, iou_threshold=0.9,
                 imgsz=640, max_new_tokens=20, prompt_ids: Sequence[int] = CAPTION_PROMPT_IDS, caption_lanes: int = 2,
                 caption_group: int = 1):
        """caption_group > 1 (opt-in): the crops of ``caption_group`` consecutive batches are captioned in ONE Florence-2
        pass (the decode steps are latency-bound at a few hundred rows, so their cost per screenshot falls with the row
        count); results are identical, a batch's result is delayed until its group has been captioned."""
        self.model, self.cmp = model, caption_model_processor
        self.conf, self.iou_thr, self.imgsz, self.T, self.prompt = BOX_TRESHOLD, iou_threshold, imgsz, max_new_tokens, list(prompt_ids)
        dev = model.device
        # role streams (ops.role_stream): one per stage and lane, shared by every parser of the device, never aliased
        self.s_det = ops.role_stream("det", dev)
        self.s_cap = ops.role_stream("cap0", dev)
        self.timings = ParseTimings(detect_wait_s=0.0, glue_s=0.0, caption_s=0.0, n_boxes=0, n_crops=0, batches=0)
        from concurrent.futures import ThreadPoolExecutor
        self._pool = ThreadPoolExecutor(max_workers=1, thread_name_prefix="b2p-submit")   # host staging copy off the main thread
        # caption stage: CAPTION_LANES batches in flight, each on its own stream with its own plan instance -- the
        # latency-bound decode steps of one batch fill the SMs the other batch's encoder leaves idle, and vice versa
        self.lanes = max(1, int(caption_lanes))
        self.s_caps = [self.s_cap] + [ops.role_stream(f"cap{i}", dev) for i in range(1, self.lanes)]
        # one single-worker executor PER LANE: two batches of the same lane share a plan and a stream, so they must
        # never be in flight together (a shared pool lets batch i+2 start on lane 0 while batch i still decodes there)
        self._cap_pools = [ThreadPoolExecutor(max_workers=1, thread_name_prefix=f"b2p-caption{i}") for i in range(self.lanes)]
        self._tm_lock = threading.Lock()
        self._job = 0
        self.group = max(1, int(caption_group))

    @torch.inference_mode()
    def _submit(self, io_, images, resident_src, ocr):
        """Stage 1 (submit thread, detection stream): the batch into its io slot, detection, the device overlap filter."""
        torch.cuda.set_device(self.model.device)   # runs on the worker thread: device and inference mode are thread-local
        with torch.cuda.stream(self.s_det):
            self.model.stage(io_, images, resident_src)
            return _detect(self.model, io_, [tuple(im.shape[:2]) for im in images], ocr, self.conf, self.iou_thr)

    def _glue(self, h, ocr):
        """Stage 2 (caller's thread): wait for the detector's boxes, run the reference's host list logic."""
        t0 = time.perf_counter()
        h["ev"].synchronize()
        t1 = time.perf_counter()
        g = _host_lists(self.model, h, ocr, self.iou_thr)
        t2 = time.perf_counter()
        tm = self.timings
        tm["detect_wait_s"] += t1 - t0; tm["glue_s"] += t2 - t1
        tm["n_boxes"] += sum(g["counts"]); tm["n_crops"] += g["n_crops"]; tm["batches"] += 1
        g["lane"] = (self._job // self.group) % self.lanes   # the batches of one caption group share a lane
        self._job += 1
        return g

    @torch.inference_mode()
    def _caption_group(self, gs):
        """Stage 3 (caption thread, the lane's stream): one Florence-2 pass over the crops of up to ``caption_group``
        batches, cut batch by batch into row blocks of ``plan.crops`` from each batch's resident screenshots; token ids back
        to the host, captions into the element lists -> the per-batch results, in order."""
        torch.cuda.set_device(self.model.device)
        model, cap_model = self.model, self.cmp["model"]
        lane = gs[0]["lane"]
        n = sum(g["n_crops"] for g in gs)
        t2 = time.perf_counter()
        ids = None
        if n:
            with torch.cuda.stream(self.s_caps[lane]):
                plan = cap_model.plan_for(n, self.T, self.prompt, instance=lane)
                status = _cut_crops(gs, plan.crops)
                ids = cap_model.generate_from_device_crops(plan, n)
                for g in gs:   # device overlap filter: element lists from its flags, while the GPU captions
                    _elements(model, g)
                status = status.to("cpu", non_blocking=True)   # completed by the ids' D2H sync below
                ids = ids.cpu()
                _check_crop_status(status)
        for g in gs:
            _elements(model, g)
        t3 = time.perf_counter()
        outs, off = [], 0
        for g in gs:
            ng, ids_b = g["n_crops"], None
            if ng:
                ids_b = ids[off:off + ng]
                # HF would have stopped this batch alone at the first step where all ITS rows had finished
                done_at = cap_model._first_all_finished(ids_b) if ids_b.shape[1] > 2 else None
                if done_at is not None:
                    ids_b = ids_b[:, :done_at + 1]
                off += ng
            outs.append(_results(self.cmp["processor"], g["all_elems"], ids_b))
        with self._tm_lock:
            self.timings["caption_s"] += t3 - t2
        return outs

    @torch.inference_mode()
    def run(self, batches, resident=None):
        """batches: iterable of (images, ocr), images a list of u8 HWC numpy arrays (of one size, or of different sizes: a
        ragged batch, batch by batch) or one page-locked u8 torch tensor [B,H,W,3]; resident: optional parallel iterable of device u8 tensors [B,H,W,3] (skips the H2D copy).
        Stages in flight: detect(i+1) on stream A (submit thread) | host list logic of batch i (this thread) |
        caption(i-1), caption(i-2) on their lane's stream (caption threads).  lanes + 2 io slots (more with caption_group) keep a batch's resident
        screenshots alive until its crops have been cut.  Results come out in order, ``lanes`` batches behind the glue."""
        from collections import deque
        self._job = 0   # lane assignment is a function of the position in THIS run (batch i -> lane i % lanes)
        with self._device_ctx():   # also takes the handle lock: the pipeline owns the io slots and caption lanes while it runs
            it = iter(batches)
            rit = iter(resident) if resident is not None else None
            cur = next(it, None)
            if cur is None:
                return
            pending = deque()
            slot = 0
            h = self._submit(self._ensure_io(slot, cur[0], pending), cur[0], next(rit) if rit is not None else None, cur[1])
            grp = []
            while cur is not None:
                nxt = next(it, None)
                fut = None
                if nxt is not None:
                    # slots alive at once: lanes*group in caption + up to group-1 glued batches waiting for their group
                    # + the batch in the host list logic + the batch in detection  (= lanes + 2 when group == 1)
                    slot = (slot + 1) % (self.lanes * self.group + self.group + 1)
                    io_ = self._ensure_io(slot, nxt[0], pending)
                    fut = self._pool.submit(self._submit, io_, nxt[0], next(rit) if rit is not None else None, nxt[1])
                grp.append(self._glue(h, cur[1]))
                if len(grp) == self.group or nxt is None:
                    self._ensure_plan(dict(n_crops=sum(x["n_crops"] for x in grp), lane=grp[0]["lane"]), pending, fut)
                    fc = self._cap_pools[grp[0]["lane"]].submit(self._caption_group, grp)
                    pending.extend(_Member(fc, j) for j in range(len(grp)))
                    grp = []
                while len(pending) > self.lanes * self.group:
                    yield pending.popleft().result()
                hn = fut.result() if fut is not None else None
                cur, h = nxt, hn
            while pending:
                yield pending.popleft().result()

    def _device_ctx(self):
        import contextlib

        @contextlib.contextmanager
        def ctx():
            with self.model._lock, torch.cuda.device(self.model.device):
                yield
        return ctx()

    @torch.inference_mode()
    def prewarm(self, crop_counts):
        """Build + capture the caption plans of every lane for the given per-batch crop counts up front (each distinct
        32-crop bucket costs a plan per lane), so that no batch of a later run() pays for it."""
        cap_model = self.cmp["model"]
        with self._device_ctx():
            torch.cuda.synchronize()
            for n in crop_counts:
                for lane in range(self.lanes):
                    if n and not cap_model.plan_ready(n, self.T, self.prompt, instance=lane):
                        cap_model.warm_plan(n, self.T, self.prompt, instance=lane, stream=self.s_caps[lane])
            torch.cuda.synchronize()

    def _ensure_io(self, slot, images, pending):
        """A batch's io slot (caller's thread).  When a batch of different sizes does not fit the buffers its slot already
        holds, every batch in flight is finished before the slot grows (see B200YOLOv9Detector.io_slot)."""
        def drain():
            for p in pending:
                p.result()
        return self.model.io_slot([tuple(im.shape[:2]) for im in images], self.imgsz, 300, slot, drain)

    def _ensure_plan(self, g, pending, fut):
        """First batch of a crop-count bucket on a lane: drain the pipeline and build + capture the caption plan with
        the GPU idle (buffers and graphs are created once; steady state never comes here)."""
        n = g["n_crops"]
        cap_model = self.cmp["model"]
        if not n or cap_model.plan_ready(n, self.T, self.prompt, instance=g["lane"]):
            return
        for p in pending:
            p.result()
        if fut is not None:
            fut.result()
        torch.cuda.synchronize()
        cap_model.warm_plan(n, self.T, self.prompt, instance=g["lane"], stream=self.s_caps[g["lane"]])
        torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ reference API
def _prompt_ids(prompt, caption_model_processor) -> Sequence[int]:
    """ref:util/utils.py:107-112: no prompt -> "<CAPTION>" for Florence-2, which the HF processor rewrites to "What does
    the image describe?" (hf:models/florence2/processing_florence2.py:81).  Any other prompt needs the tokenizer."""
    proc = caption_model_processor["processor"]
    if not prompt or prompt == "<CAPTION>":
        return list(getattr(proc, "prompt_ids", CAPTION_PROMPT_IDS))
    tok = getattr(proc, "tokenizer", None)
    enc = getattr(tok, "encode", None) or getattr(getattr(tok, "tk", None), "encode", None)
    if enc is None:
        raise NotImplementedError(f"prompt={prompt!r}: a custom prompt has to be tokenised, and this processor was built "
                                  "without tokenizer files (see get_caption_model_processor)")
    ids = enc(prompt)
    ids = list(getattr(ids, "ids", ids))
    return ids


def get_som_labeled_img(image_source: Union[str, Image.Image], model=None, BOX_TRESHOLD=0.01, output_coord_in_ratio=False,
                        ocr_bbox=None, text_scale=0.4, text_padding=5, draw_bbox_config=None,
                        caption_model_processor=None, ocr_text=[], use_local_semantics=True, iou_threshold=0.9,
                        prompt=None, scale_img=False, imgsz=None, batch_size=128):
    """ref:util/utils.py:417-496.  Returns ``(base64 PNG, {str(i): [x, y, w, h]}, filtered_boxes_elem)`` -- the element
    list, the label coordinates and the decoded overlay image equal the reference's (tests/golden, tests/test_overlay_cpu.py).
    ``batch_size`` only chunks the reference's generate calls (rows are independent under greedy decoding), so it has no
    effect on the result here; it is validated and otherwise unused."""
    if not (isinstance(batch_size, int) and batch_size > 0):
        raise ValueError(f"batch_size must be a positive int, got {batch_size!r}")
    if isinstance(image_source, str):
        image_source = Image.open(image_source)
    image_source = image_source.convert("RGB")
    w, h = image_source.size
    if not imgsz:
        imgsz = (h, w)
    img = np.asarray(image_source)
    use_imgsz = imgsz if scale_img else 640          # ref:util/utils.py:391-404: imgsz only reaches the detector if scale_img
    if not ocr_bbox:
        print("no ocr bbox!!!")                      # side effect kept (ref:util/utils.py:441)
    if use_local_semantics:
        res = parse_screenshots([img], model, caption_model_processor, [(list(ocr_text), ocr_bbox or None)], BOX_TRESHOLD,
                                iou_threshold, use_imgsz, prompt_ids=_prompt_ids(prompt, caption_model_processor))
        elems = res[0][0]
    else:
        r = model.predict(img, conf=BOX_TRESHOLD, imgsz=use_imgsz, iou=0.1)[0].boxes
        whwh = torch.Tensor([w, h, w, h])
        xyxy = (r.xyxy.cpu() / whwh).tolist()
        oratio = (torch.tensor(ocr_bbox) / whwh).tolist() if ocr_bbox else None
        elems, _ = host_glue.build_elements(xyxy, oratio, list(ocr_text), w, h, iou_threshold)
    print("len(filtered_boxes):", len(elems), next((i for i, e in enumerate(elems) if e["content"] is None), -1))
    boxes = [e["bbox"] for e in elems]
    cfg = draw_bbox_config if draw_bbox_config else dict(text_scale=text_scale, text_padding=text_padding)
    encoded, coords, _ = som_overlay.som_outputs(img, boxes, output_coord_in_ratio, **cfg,
                                                 device=getattr(model, "device", None))
    return encoded, coords, elems
