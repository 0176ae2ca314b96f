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
    on this path, so a flagged crop is a bug and raises (read after the ids' D2H sync: no extra synchronisation)."""
    bad = int(status.count_nonzero().item())
    if bad:
        raise RuntimeError(f"{bad} crop boxes were empty after truncation (status flags of b2p_crop_resize)")


def _crop_meta(model: B200YOLOv9Detector, io_, B, H, W, *key):
    """(img_hw, img_off) of b2p_crop_resize for a batch's screenshots in io_["src"]: a ragged batch's are filled per batch in
    its io slot; a one-size batch's are built once per (B, H, W, *key) and cached on the detector handle."""
    if io_.get("mixed"):
        return io_["meta_hw"], io_["meta_off"]
    key = ("crop_meta", B, H, W) + key
    meta = model._io.get(key)
    if meta is None:
        dev = model.device
        meta = dict(hw=torch.tensor([[H, W]] * B, dtype=torch.int32, device=dev),
                    off=torch.tensor([i * H * W * 3 for i in range(B)], dtype=torch.int64, device=dev))
        model._io[key] = meta
    return meta["hw"], meta["off"]


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
    B = len(images)
    mixed = B200YOLOv9Detector.is_mixed(images)
    if mixed and _skip_h2d:
        raise ValueError("_skip_h2d takes screenshots of one size: a batch of different sizes has no resident one-size buffer")
    H, W = (None, None) if mixed else images[0].shape[:2]
    sizes = [tuple(im.shape[:2]) for im in images] if mixed else [(H, W)] * B
    cap_model: B200Florence2Model = caption_model_processor["model"]
    processor = caption_model_processor["processor"]
    t0 = time.perf_counter()
    with model._lock, torch.cuda.device(model.device):   # io slot 0 / caption plan instance 0 are this handle's: one call at a time
        if mixed:
            mb = model.plan_mixed(sizes, imgsz)
            io_ = model._get_io_mixed(B, imgsz, 300)
            model.reserve_mixed(io_, mb)
            model.stage_mixed(io_, mb, images)
        else:
            io_ = model._get_io(B, H, W, imgsz, 300)
        if not mixed and not _skip_h2d:   # bench "value" leg: the u8 screenshots are already resident in io_["src"]
            for i, im in enumerate(images):
                io_["host"][i].copy_(torch.from_numpy(np.ascontiguousarray(im)))
            io_["src"].copy_(io_["host"], non_blocking=True)
        whwh = [torch.Tensor([w, h, w, h]) for h, w in sizes]
        ocr_elems = [host_glue.ocr_elements((torch.tensor(ob) / whwh[i]).tolist() if ob else None, tx, sizes[i][1], sizes[i][0])
                     for i, (tx, ob) in enumerate(ocr)]   # :437-444
        on_device = False
        if _det_override is None:
            if mixed:
                model.detect_device_mixed(io_, sizes, BOX_TRESHOLD, 0.1, 300)
            else:
                model.detect_device(io_, B, H, W, BOX_TRESHOLD, 0.1, 300)
            on_device = not _HOST_GLUE and model.filter_device(io_, B, H, W, ocr_elems, iou_threshold, 300)
            counts = io_["out_count"].cpu().tolist()                   # D2H #1 (sync; the filter's flags ride along)
            boxes = None if on_device else io_["out_box"].cpu()
            model.check_capacity(io_["cand_count"].cpu(), io_["cap"])
        else:   # tests: inject detector output (e.g. the golden boxes) to pin the stages after it exactly
            counts = [len(b) for b in _det_override]
            boxes = [torch.as_tensor(b, dtype=torch.float32).reshape(-1, 4) for b in _det_override]
        t1 = time.perf_counter()
        all_elems, crop_boxes, crop_img = [], [], []
        if on_device:
            # overlap filter ran on the GPU (b2p_overlap_filter): element lists from its flags, crop list already on the device
            for i in range(B):
                all_elems.append(model.elements_from_io(io_, i, counts[i], ocr_elems[i]))
            n = int(io_["host_crop_counts"][B])
        else:
            for i in range(B):
                xyxy = (boxes[i][:counts[i]] / whwh[i]).tolist()           # ref:util/utils.py:432
                texts, obox = ocr[i]
                oratio = (torch.tensor(obox) / whwh[i]).tolist() if obox else None   # :437-442
                elems, start = host_glue.build_elements(xyxy, oratio, texts, sizes[i][1], sizes[i][0], iou_threshold)
                all_elems.append(elems)
                for e in elems:
                    if e["content"] is None:
                        crop_boxes.append(e["bbox"])
                        crop_img.append(i)
            n = len(crop_boxes)
        t2 = time.perf_counter()
        ids = None
        if n:
          with cap_model._lock:   # plan instance 0 of the caption handle (also what model.generate() uses)
            dev = model.device
            if caption_size == 64:
                plan = cap_model.plan_for(n, max_new_tokens, prompt_ids, **bs)
                crops_dst = plan.crops
            else:
                crops_dst = torch.empty((n, 64, 64, 3), dtype=torch.uint8, device=dev)
            if on_device:
                d_boxes, d_bimg = io_["crop_box"], io_["crop_img"]
            else:
                d_boxes = torch.tensor(crop_boxes, dtype=torch.float32).to(dev, non_blocking=True)
                d_bimg = torch.tensor(crop_img, dtype=torch.int32).to(dev, non_blocking=True)
            hw, off = _crop_meta(model, io_, B, H, W)
            status = torch.zeros((n,), dtype=torch.int32, device=dev)
            ops.crop_resize(io_["src"], hw, off, d_boxes, d_bimg, n, 64, crops_dst, status)
            if caption_size == 64:
                ids = cap_model.generate_from_device_crops(plan, n).cpu()  # D2H #2 (sync)
            else:
                ids = cap_model.generate_chunked(crops_dst, max_new_tokens, prompt_ids, from_resized=False, **bs).cpu()
            _check_crop_status(status)
        t3 = time.perf_counter()
    out = []
    k = 0
    texts_all = processor.batch_decode(ids, skip_special_tokens=True) if ids is not None else []
    texts_all = [t.strip() for t in texts_all]
    for i in range(B):
        m = sum(1 for e in all_elems[i] if e["content"] is None)
        host_glue.fill_captions(all_elems[i], texts_all[k:k + m])
        out.append((all_elems[i], ids[k:k + m] if ids is not None else torch.zeros((0, 1), dtype=torch.long)))
        k += m
    if timings is not None:
        timings.update(detect_s=t1 - t0, glue_s=t2 - t1, caption_s=t3 - t2, n_boxes=sum(counts), n_crops=n)
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
    def _submit(self, slot: int, images, resident_src=None, ocr=None, mb=None):
        torch.cuda.set_device(self.model.device)   # runs on the worker thread: device and inference mode are thread-local
        B = len(images)
        m = self.model
        if mb is not None:   # screenshots of different sizes (run() has sized the slot: see _ensure_io)
            if resident_src is not None:
                raise ValueError("resident= batches have one size: a batch of different sizes has no one-size device tensor")
            sizes = [tuple(im.shape[:2]) for im in images]
            H = W = None
            io_ = m._get_io_mixed(B, self.imgsz, 300, slot)
            assert not m.mixed_grow_needed(io_, mb)
            m.reserve_mixed(io_, mb)
        else:
            H, W = images[0].shape[:2]
            sizes = [(H, W)] * B
            io_ = m._get_io(B, H, W, self.imgsz, 300, slot)
        with torch.cuda.stream(self.s_det):
            if mb is not None:
                m.stage_mixed(io_, mb, images)
                m.detect_device_mixed(io_, sizes, self.conf, 0.1, 300)
            else:
                if resident_src is not None:
                    io_["src"].copy_(resident_src, non_blocking=True)
                elif torch.is_tensor(images) and images.is_pinned():
                    # caller-owned page-locked [B,H,W,3] u8 batch: DMA straight from it (it must stay untouched until the
                    # batch's result has been yielded); pageable numpy screenshots go through the slot's pinned staging copy
                    io_["src"].copy_(images, non_blocking=True)
                else:
                    for i, im in enumerate(images):
                        io_["host"][i].copy_(torch.from_numpy(np.ascontiguousarray(im)))
                    io_["src"].copy_(io_["host"], non_blocking=True)
                m.detect_device(io_, B, H, W, self.conf, 0.1, 300)
            ocr_elems, on_device = None, False
            if ocr is not None and not _HOST_GLUE:
                # overlap filter on the device, right behind NMS on the detector's stream (no host round trip in between)
                whwh = [torch.Tensor([w, h, w, h]) for h, w in sizes]
                ocr_elems = [host_glue.ocr_elements((torch.tensor(ob) / whwh[i]).tolist() if ob else None, tx, sizes[i][1], sizes[i][0])
                             for i, (tx, ob) in enumerate(ocr)]
                on_device = m.filter_device(io_, B, H, W, ocr_elems, self.iou_thr, 300)
            io_["host_count"].copy_(io_["out_count"], non_blocking=True)
            if not on_device:
                io_["host_box"].copy_(io_["out_box"], non_blocking=True)
            io_["host_cand"].copy_(io_["cand_count"], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.s_det)
        return dict(io=io_, ev=ev, B=B, H=H, W=W, sizes=sizes, ocr_elems=ocr_elems, on_device=on_device)

    def _glue(self, h, ocr):
        """Stage 2 (caller's thread): wait for the detector's boxes, run the reference's host list logic."""
        io_, B, H, W = h["io"], h["B"], h["H"], h["W"]
        t0 = time.perf_counter()
        h["ev"].synchronize()
        t1 = time.perf_counter()
        counts = io_["host_count"].tolist()
        self.model.check_capacity(io_["host_cand"], io_["cap"])
        all_elems, crop_boxes, crop_img = [], [], []
        if h.get("on_device"):
            # the device filter's flags arrived with the counts: element lists are built later, on the caption thread (they are
            # only needed for the result); the crop list stays on the device
            n_crops = int(io_["host_crop_counts"][B])
            all_elems = None
        else:
            boxes = io_["host_box"]
            for i, (hi, wi) in enumerate(h["sizes"]):
                whwh = torch.Tensor([wi, hi, wi, hi])
                xyxy = (boxes[i][:counts[i]] / whwh).tolist()
                texts, obox = ocr[i]
                oratio = (torch.tensor(obox) / whwh).tolist() if obox else None
                elems, _ = host_glue.build_elements(xyxy, oratio, texts, wi, hi, self.iou_thr)
                all_elems.append(elems)
                for e in elems:
                    if e["content"] is None:
                        crop_boxes.append(e["bbox"])
                        crop_img.append(i)
            n_crops = len(crop_boxes)
        t2 = time.perf_counter()
        tm = self.timings
        tm["detect_wait_s"] += t1 - t0; tm["glue_s"] += t2 - t1
        tm["n_boxes"] += sum(counts); tm["n_crops"] += n_crops; tm["batches"] += 1
        lane = (self._job // self.group) % self.lanes   # the batches of one caption group share a lane
        self._job += 1
        return dict(h=h, all_elems=all_elems, crop_boxes=crop_boxes, crop_img=crop_img, lane=lane, n_crops=n_crops, counts=counts)

    @torch.inference_mode()
    def _caption(self, g):
        """Stage 3 (caption thread, stream B): crop+resize from the resident screenshots, Florence-2 greedy decode,
        token ids back to the host, captions into the element lists."""
        torch.cuda.set_device(self.model.device)
        h, all_elems, crop_boxes, crop_img = g["h"], g["all_elems"], g["crop_boxes"], g["crop_img"]
        io_, B, H, W = h["io"], h["B"], h["H"], h["W"]
        model, cap_model, processor = self.model, self.cmp["model"], self.cmp["processor"]
        n = g["n_crops"]
        t2 = time.perf_counter()
        ids = None
        if n:
            dev = model.device
            lane = g.get("lane", 0)
            with torch.cuda.stream(self.s_caps[lane]):
                plan = cap_model.plan_for(n, self.T, self.prompt, instance=lane)
                if h.get("on_device"):
                    d_boxes, d_bimg = io_["crop_box"], io_["crop_img"]
                else:
                    d_boxes = torch.tensor(crop_boxes, dtype=torch.float32).to(dev, non_blocking=True)
                    d_bimg = torch.tensor(crop_img, dtype=torch.int32).to(dev, non_blocking=True)
                hw, off = _crop_meta(model, io_, B, H, W, lane)
                status = torch.zeros((n,), dtype=torch.int32, device=dev)
                ops.crop_resize(io_["src"], hw, off, d_boxes, d_bimg, n, 64, plan.crops, status)
                ids = cap_model.generate_from_device_crops(plan, n)
                if all_elems is None:   # device overlap filter: element lists from its flags, while the GPU captions
                    all_elems = [model.elements_from_io(io_, i, g["counts"][i], h["ocr_elems"][i]) for i in range(B)]
                ids = ids.cpu()
                _check_crop_status(status)
        if all_elems is None:
            all_elems = [model.elements_from_io(io_, i, g["counts"][i], h["ocr_elems"][i]) for i in range(B)]
        t3 = time.perf_counter()
        texts_all = [t.strip() for t in processor.batch_decode(ids, skip_special_tokens=True)] if ids is not None else []
        out, k = [], 0
        for i in range(B):
            mcap = sum(1 for e in all_elems[i] if e["content"] is None)
            host_glue.fill_captions(all_elems[i], texts_all[k:k + mcap])
            out.append((all_elems[i], ids[k:k + mcap] if ids is not None else torch.zeros((0, 1), dtype=torch.long)))
            k += mcap
        with self._tm_lock:
            self.timings["caption_s"] += t3 - t2
        return out

    @torch.inference_mode()
    def _caption_group(self, gs):
        """caption_group > 1: one Florence-2 pass over the crops of several batches (same lane); returns the per-batch
        results in order.  Row blocks of ``plan.crops`` are filled batch by batch from each batch's resident screenshots."""
        torch.cuda.set_device(self.model.device)
        model, cap_model, processor = self.model, self.cmp["model"], self.cmp["processor"]
        lane = gs[0]["lane"]
        counts = [g["n_crops"] for g in gs]
        n = sum(counts)
        for g in gs:
            if g["all_elems"] is None:
                hh = g["h"]
                g["all_elems"] = [model.elements_from_io(hh["io"], i, g["counts"][i], hh["ocr_elems"][i]) for i in range(hh["B"])]
        t2 = time.perf_counter()
        ids = None
        if n:
            dev = model.device
            with torch.cuda.stream(self.s_caps[lane]):
                plan = cap_model.plan_for(n, self.T, self.prompt, instance=lane)
                off = 0
                for g, ng in zip(gs, counts):
                    if not ng:
                        continue
                    io_, B, H, W = g["h"]["io"], g["h"]["B"], g["h"]["H"], g["h"]["W"]
                    if g["h"].get("on_device"):
                        d_boxes, d_bimg = io_["crop_box"], io_["crop_img"]
                    else:
                        d_boxes = torch.tensor(g["crop_boxes"], dtype=torch.float32).to(dev, non_blocking=True)
                        d_bimg = torch.tensor(g["crop_img"], dtype=torch.int32).to(dev, non_blocking=True)
                    hw, moff = _crop_meta(model, io_, B, H, W, lane)
                    status = torch.zeros((ng,), dtype=torch.int32, device=dev)
                    ops.crop_resize(io_["src"], hw, moff, d_boxes, d_bimg, ng, 64, plan.crops[off:], status)
                    off += ng
                ids = cap_model.generate_from_device_crops(plan, n).cpu()
        t3 = time.perf_counter()
        outs, off = [], 0
        for g, ng in zip(gs, counts):
            all_elems, B = g["all_elems"], g["h"]["B"]
            ids_b = None
            if ng:
                ids_b = ids[off:off + ng]
                # HF would have stopped this batch alone at the first step where all ITS rows had finished
                done_at = cap_model._first_all_finished(ids_b) if ids_b.shape[1] > 2 else None
                if done_at is not None:
                    ids_b = ids_b[:, :done_at + 1]
                off += ng
            texts_all = [t.strip() for t in processor.batch_decode(ids_b, skip_special_tokens=True)] if ids_b is not None else []
            out, k = [], 0
            for i in range(B):
                mcap = sum(1 for e in all_elems[i] if e["content"] is None)
                host_glue.fill_captions(all_elems[i], texts_all[k:k + mcap])
                out.append((all_elems[i], ids_b[k:k + mcap] if ids_b is not None else torch.zeros((0, 1), dtype=torch.long)))
                k += mcap
            outs.append(out)
        with self._tm_lock:
            self.timings["caption_s"] += t3 - t2
        return outs

    def _finish(self, h, ocr):
        return self._caption(self._glue(h, ocr))

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
            slot = 0
            mb = self._ensure_io(slot, cur[0], ())
            h = self._submit(slot, cur[0], next(rit) if rit is not None else None, cur[1], **({} if mb is None else dict(mb=mb)))
            pending = deque()
            grp = []
            while cur is not None:
                nxt = next(it, None)
                fut = None
                if nxt is not None:
                    # slots alive at once: lanes*group in caption + up to group-1 glued batches waiting for their group
                    # + the batch in the host list logic + the batch in detection  (= lanes + 2 when group == 1)
                    slot = (slot + 1) % (self.lanes * self.group + self.group + 1)
                    mb = self._ensure_io(slot, nxt[0], pending)
                    fut = self._pool.submit(self._submit, slot, nxt[0], next(rit) if rit is not None else None, nxt[1],
                                            **({} if mb is None else dict(mb=mb)))
                g = self._glue(h, cur[1])
                if self.group == 1:
                    self._ensure_plan(g, pending, fut)
                    pending.append(self._cap_pools[g["lane"]].submit(self._caption, g))
                else:
                    grp.append(g)
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
        """A batch of screenshots of different sizes -> its letterbox plan (None for a one-size batch).  When the batch does
        not fit the buffers its io slot already holds, the pipeline is drained (every batch in flight finished, device
        synchronised) before the slot grows: the freed buffers may still be read by another stream until then."""
        if not B200YOLOv9Detector.is_mixed(images):
            return None
        m = self.model
        mb = m.plan_mixed([tuple(im.shape[:2]) for im in images], self.imgsz)
        io_ = m._get_io_mixed(len(images), self.imgsz, 300, slot)
        if m.mixed_grow_needed(io_, mb):
            for p in pending:
                p.result()
            torch.cuda.synchronize()
            m.reserve_mixed(io_, mb)
        return mb

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
