"""Drop-in for ``util.yolov9.YOLOv9Detector`` (ref:util/yolov9.py:27-136) running on the package's CUDA kernels.

Same constructor / ``predict`` signature and result objects (``[Result(Boxes(xyxy, conf))]`` with device
tensors), same letterbox geometry, strict ``>`` confidence filter, un-letterbox, ``batched_nms`` semantics,
``[:max_det]`` and clamp.  Everything between the u8 image and the final boxes runs on the GPU without a host
sync: LANCZOS letterbox -> YOLOv9-E forward (CUDA graph) -> decode/filter -> bitmask NMS.
"""
from __future__ import annotations

import threading
from pathlib import Path
from typing import Dict, List, Sequence, Union

import numpy as np
import torch

from . import ops
from .yolo_engine import YoloPlan, YoloWeights, rename_upstream


class Boxes:   # ref:util/yolov9.py:16-19
    def __init__(self, xyxy: torch.Tensor, confidence: torch.Tensor):
        self.xyxy = xyxy
        self.conf = confidence


class Result:  # ref:util/yolov9.py:22-24
    def __init__(self, boxes: Boxes):
        self.boxes = boxes


def _canvas(imgsz):
    """(tw, th) of the letterbox canvas, ref:util/yolov9.py:52-61."""
    if isinstance(imgsz, int):
        tw = th = imgsz
    elif len(imgsz) == 2:
        th, tw = imgsz
    else:
        raise ValueError(f"Expected one or two image dimensions, got {imgsz}")
    return ((int(tw) + 31) // 32) * 32, ((int(th) + 31) // 32) * 32


def _geometry(w: int, h: int, imgsz):
    """ref:util/yolov9.py:52-61,73-80."""
    tw, th = _canvas(imgsz)
    scale = min(tw / w, th / h)
    rw, rh = int(w * scale), int(h * scale)
    if rw < 1 or rh < 1:   # Pillow's resize raises the same (e.g. 641 x 1 at imgsz 640 resizes to 640 x 0)
        raise ValueError(f"height and width must be > 0: a {w} x {h} image resizes to {rw} x {rh} at imgsz {imgsz}")
    return tw, th, scale, rw, rh, (tw - rw) // 2, (th - rh) // 2


class B200YOLOv9Detector:
    strides = (8, 16, 32)
    CAND_CAP = 16384
    OCR_CAP = 256      # OCR boxes per screenshot the device overlap filter takes (host_glue.OCR_DEVICE_CAP); more -> host path

    def __init__(self, model_path: Union[str, Path, None] = None, device: Union[str, torch.device, None] = None,
                 state_dict: Dict[str, torch.Tensor] | None = None, use_graph: bool = True, precision: str | None = None):
        """precision: "fp16" (default; the reference's own CUDA path is fp16 autocast, ref:util/yolov9.py:110-113) or
        "fp16x3" (parity grade: reproduces the fp32 CPU path's kept boxes; ~3x the tensor work).  Default from the
        environment variable B2P_DETECTOR_PRECISION."""
        import os
        self.precision = precision or os.environ.get("B2P_DETECTOR_PRECISION", "fp16")
        self.device = torch.device(device or "cuda")
        if self.device.type != "cuda" or not torch.cuda.is_available():
            # ref:util/yolov9.py:40-41 raises when CUDA is requested but unavailable; this build has no CPU path.
            raise RuntimeError(f"the detector needs a CUDA device (requested {self.device}); there is no CPU fallback")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        if state_dict is None:
            if model_path is None:
                raise FileNotFoundError("model_path (TorchScript archive or state_dict file) is required: no network here")
            self.model_path = Path(model_path)
            try:
                state_dict = torch.jit.load(str(self.model_path), map_location="cpu").state_dict()
            except Exception:
                state_dict = torch.load(str(self.model_path), map_location="cpu")
        if any(k.startswith("model.") for k in state_dict):
            state_dict = rename_upstream(state_dict)
        with torch.cuda.device(self.device):
            self.weights = YoloWeights(state_dict, self.device, precision=self.precision)
        self.model = self.weights   # attribute the reference exposes (inspected in demo.ipynb)
        self.use_graph = use_graph
        self._plans: Dict[tuple, YoloPlan] = {}
        self._io: Dict[tuple, dict] = {}
        # One parse at a time per detector handle: the reference's callers share ONE module-level model between worker
        # threads (ref:gradio_demo.py:15-16,35-59) and its PyTorch modules are re-entrant; this object's launch plans and io
        # buffers are not, so every public entry point serialises on this lock (SURVEY.md §8b "self-serialising per device").
        self._lock = threading.RLock()

    def to(self, device):   # called at ref:eval/ss_pro_gpt4o_omniv2.py:30
        return self

    # ------------------------------------------------------------------------------------------
    @staticmethod
    def _load_image(source) -> np.ndarray:
        from PIL import Image
        if isinstance(source, np.ndarray):
            return np.asarray(Image.fromarray(source).convert("RGB"))
        if isinstance(source, Image.Image):
            return np.asarray(source.convert("RGB"))
        with Image.open(source) as im:
            return np.asarray(im.convert("RGB"))

    def _common_io(self, B, th, tw, max_det):
        """The buffers of an io slot that do not depend on the screenshots' size: detector plan of (B, th, tw), candidates,
        NMS outputs and the device overlap filter's buffers."""
        dev = self.device
        pk = (B, th, tw)
        if pk not in self._plans:
            self._plans[pk] = YoloPlan(self.weights, B, th, tw, self.use_graph)
        plan = self._plans[pk]
        A = sum(h * w for h, w in plan.hw)
        cap = min(self.CAND_CAP, A)
        f32 = dict(dtype=torch.float32, device=dev)
        io = dict(
            plan=plan, cap=cap, B=B,
            host_count=torch.zeros((B,), dtype=torch.int32).pin_memory(),
            host_box=torch.zeros((B, max_det, 4), dtype=torch.float32).pin_memory(),
            host_cand=torch.zeros((B,), dtype=torch.int32).pin_memory(),
            cand_box=torch.empty((B, cap, 4), **f32), cand_score=torch.empty((B, cap), **f32),
            cand_cls=torch.empty((B, cap), dtype=torch.int32, device=dev),
            cand_count=torch.zeros((B,), dtype=torch.int32, device=dev),
            keep=torch.empty((B, max_det), dtype=torch.int32, device=dev),
            out_box=torch.empty((B, max_det, 4), **f32), out_score=torch.empty((B, max_det), **f32),
            out_count=torch.zeros((B,), dtype=torch.int32, device=dev),
        )
        # device overlap filter (b2p_overlap_filter, ref:util/utils.py:241-319): OCR ratio boxes in, flags + crop list out
        mo = self.OCR_CAP
        i32 = dict(dtype=torch.int32, device=dev)
        io.update(
            max_ocr=mo,
            ocr_ratio=torch.zeros((B, mo, 4), **f32), ocr_count=torch.zeros((B,), **i32),
            host_ocr_ratio=torch.zeros((B, mo, 4), dtype=torch.float32).pin_memory(),
            host_ocr_count=torch.zeros((B,), dtype=torch.int32).pin_memory(),
            icon_state=torch.zeros((B, max_det), **i32), label_mask=torch.zeros((B, max_det, mo // 32), **i32),
            ocr_removed=torch.zeros((B, mo), **i32), icon_ratio=torch.zeros((B, max_det, 4), **f32),
            crop_box=torch.zeros((B * max_det, 4), **f32), crop_img=torch.zeros((B * max_det,), **i32),
            crop_counts=torch.zeros((B + 1,), **i32), arrive=torch.zeros((1,), **i32),
            host_state=torch.zeros((B, max_det), dtype=torch.int32).pin_memory(),
            host_mask=torch.zeros((B, max_det, mo // 32), dtype=torch.int32).pin_memory(),
            host_removed=torch.zeros((B, mo), dtype=torch.int32).pin_memory(),
            host_ratio=torch.zeros((B, max_det, 4), dtype=torch.float32).pin_memory(),
            host_crop_counts=torch.zeros((B + 1,), dtype=torch.int32).pin_memory(),
        )
        return io

    def io_slot(self, sizes, imgsz, max_det, slot=0, drain=None):
        """The io slot of a batch of screenshots of these (H, W) sizes, for :meth:`stage` and :meth:`detect`.  Screenshots of
        one size get the slot of their size (:meth:`_get_io`); screenshots of different sizes share the ragged slot of their
        canvas, which takes this batch's letterbox plan and grows when the batch does not fit its buffers.  Growing frees
        buffers another stream may still read, so ``drain()`` (the caller finishes every batch it has in flight) runs first.
        A slot is complete when this returns: what building or growing it launched on the caller's stream has finished, so
        any stream may use it.  One batch owns a slot index from here until its crops have been cut."""
        sizes = [tuple(s) for s in sizes]
        if len(set(sizes)) > 1:
            return self._ragged_io(sizes, imgsz, max_det, slot, drain)
        return self._get_io(len(sizes), *sizes[0], imgsz, max_det, slot)

    def _get_io(self, B, H, W, imgsz, max_det, slot=0):
        tw, th, scale, rw, rh, pl, pt = _geometry(W, H, imgsz)
        key = (B, H, W, tw, th, max_det, slot)
        io = self._io.get(key)
        if io is None:
            dev = self.device
            f32 = dict(dtype=torch.float32, device=dev)
            io = self._common_io(B, th, tw, max_det)
            io.update(
                geom=(tw, th, scale, rw, rh, pl, pt),
                host=torch.empty((B, H, W, 3), dtype=torch.uint8).pin_memory(),
                src=torch.empty((B, H, W, 3), dtype=torch.uint8, device=dev),
                tmp=torch.empty((B, H, max(rw, 1), 3), dtype=torch.uint8, device=dev),
                pad_l=torch.full((B,), float(pl), **f32), pad_t=torch.full((B,), float(pt), **f32),
                scale=torch.full((B,), float(np.float32(scale)), **f32),
                img_w=torch.full((B,), float(W), **f32), img_h=torch.full((B,), float(H), **f32),
                # crop metadata of b2p_crop_resize: (H, W) and byte offset of each screenshot in src
                meta_hw=torch.tensor([[H, W]] * B, dtype=torch.int32, device=dev),
                meta_off=torch.tensor([i * H * W * 3 for i in range(B)], dtype=torch.int64, device=dev),
            )
            torch.cuda.synchronize(dev)   # the fills above ran on the caller's stream; other streams read the slot
            self._io[key] = io
        return io

    # ---- screenshots of different sizes in one batch (one canvas, ragged source buffer) ----
    @staticmethod
    def plan_mixed(sizes, imgsz):
        """Host only: (H, W) per screenshot -> dict(canvas, geom, desc, tables, need) of one ragged batch; ``need`` = (src
        bytes, tmp bytes, table ints) the io slot must hold."""
        tw, th = _canvas(imgsz)
        geom = []
        for H, W in sizes:
            _, _, scale, rw, rh, pl, pt = _geometry(W, H, imgsz)
            geom.append((H, W, rw, rh, pl, pt, float(np.float32(scale))))
        desc, tables, tmp_b, src_b = ops.letterbox_batch_plan([g[:6] for g in geom], tw, th)
        return dict(canvas=(tw, th), geom=geom, desc=desc, tables=tables, need=(src_b, tmp_b, int(tables.size)))

    def _ragged_io(self, sizes, imgsz, max_det, slot, drain):
        """The ragged slot of (B, canvas, slot), sized for the batch: src / tmp are flat byte buffers addressed by per-image
        descriptors, and the per-image geometry and crop metadata (meta_hw / meta_off) are filled per batch by :meth:`stage`
        from ``io["batch"]``, the letterbox plan of the batch the slot was last given to."""
        mb = self.plan_mixed(sizes, imgsz)
        tw, th = mb["canvas"]
        key = ("mixed", len(sizes), tw, th, max_det, slot)
        io = self._io.get(key)
        if io is None:
            io = self._io[key] = dict(self._common_io(len(sizes), th, tw, max_det), mixed=True, canvas=(tw, th), src=None)
        if drain is not None and self.mixed_grow_needed(io, mb):
            drain()
        self.reserve_mixed(io, mb)
        io["batch"] = mb
        return io

    @staticmethod
    def mixed_grow_needed(io, mb) -> bool:
        """True when the slot already holds buffers and the batch does not fit them."""
        return io["src"] is not None and not B200YOLOv9Detector._mixed_fits(io, mb["need"])

    @staticmethod
    def _mixed_fits(io, need):
        return need[0] <= io["cap_src"] and need[1] <= io["cap_tmp"] and need[2] <= io["cap_tab"]

    def reserve_mixed(self, io, mb):
        """Size the slot's buffers for the batch.  A slot that already has buffers grows geometrically (x1.5) and only
        after a device synchronise; steady state allocates nothing."""
        need = mb["need"]
        if io["src"] is not None and self._mixed_fits(io, need):
            return
        if io["src"] is not None:
            torch.cuda.synchronize(self.device)
            grow = lambda n, c: max(n, c + c // 2)                     # noqa: E731
            need = (grow(need[0], io["cap_src"]), grow(need[1], io["cap_tmp"]), grow(need[2], io["cap_tab"]))
        B, dev = io["B"], self.device
        cap_src, cap_tmp, cap_tab = need
        # the batch's small data, one H2D copy: desc int64 [B,12] | meta_off int64 [B] | pad_l, pad_t, scale, img_w, img_h
        # f32 [B] | meta_hw int32 [B,2] | tables int32 [cap_tab]
        o_off, o_f32 = B * ops.LB_DESC * 8, B * (ops.LB_DESC + 1) * 8
        o_hw = o_f32 + 5 * B * 4
        o_tab = (o_hw + 8 * B + 15) // 16 * 16
        small_bytes = o_tab + 4 * max(cap_tab, 1)
        host_small = torch.zeros((small_bytes,), dtype=torch.uint8).pin_memory()
        small = torch.zeros((small_bytes,), dtype=torch.uint8, device=dev)

        def views(buf):
            f = buf[o_f32:o_hw].view(torch.float32)
            return dict(desc=buf[:o_off].view(torch.int64).view(B, ops.LB_DESC), meta_off=buf[o_off:o_f32].view(torch.int64),
                        pad_l=f[:B], pad_t=f[B:2 * B], scale=f[2 * B:3 * B], img_w=f[3 * B:4 * B], img_h=f[4 * B:],
                        meta_hw=buf[o_hw:o_hw + 8 * B].view(torch.int32).view(B, 2), tables=buf[o_tab:].view(torch.int32))
        io.update(views(small))
        io.update(small=small, host_small=host_small, host_views=views(host_small), small_layout=o_tab,
                  host=torch.empty((max(cap_src, 1),), dtype=torch.uint8).pin_memory(),
                  src=torch.empty((max(cap_src, 1),), dtype=torch.uint8, device=dev),
                  tmp=torch.empty((max(cap_tmp, 1),), dtype=torch.uint8, device=dev),
                  cap_src=cap_src, cap_tmp=cap_tmp, cap_tab=cap_tab)
        torch.cuda.synchronize(dev)   # as in _get_io

    def stage(self, io, images, resident=None):
        """Copy a batch's screenshots into its io slot on the current stream: a list of u8 HWC numpy arrays through the
        slot's pinned buffer, a page-locked [B,H,W,3] u8 tensor by DMA straight from it (the caller keeps it untouched until
        the batch's results are out), or ``resident``, a [B,H,W,3] u8 device tensor, device to device."""
        if io.get("mixed"):
            if resident is not None:
                raise ValueError("resident= batches have one size: a batch of different sizes has no one-size device tensor")
            self._stage_ragged(io, images)
        elif resident is not None:
            io["src"].copy_(resident, non_blocking=True)
        elif torch.is_tensor(images) and images.is_pinned():
            io["src"].copy_(images, non_blocking=True)
        else:
            for i, im in enumerate(images):
                io["host"][i].copy_(torch.from_numpy(np.ascontiguousarray(im)))
            io["src"].copy_(io["host"], non_blocking=True)

    @staticmethod
    def _stage_ragged(io, images):
        """Pack the screenshots and the batch's small data into the slot's pinned buffers and copy both to the device (two
        H2D copies)."""
        mb = io["batch"]
        assert len(images) == io["B"] == len(mb["geom"])
        hv, host = io["host_views"], io["host"]
        hv["desc"].numpy()[:] = mb["desc"]
        g = np.asarray(mb["geom"], dtype=np.float64)
        hv["meta_off"].numpy()[:] = mb["desc"][:, 0]
        for name, col in (("pad_l", 4), ("pad_t", 5), ("scale", 6), ("img_w", 1), ("img_h", 0)):
            hv[name].numpy()[:] = g[:, col].astype(np.float32)
        hv["meta_hw"].numpy()[:] = g[:, :2].astype(np.int32)
        n_tab = mb["need"][2]
        hv["tables"].numpy()[:n_tab] = mb["tables"]
        hn = host.numpy()
        for i, im in enumerate(images):
            H, W = mb["geom"][i][:2]
            assert im.shape == (H, W, 3) and im.dtype == np.uint8
            o = int(mb["desc"][i, 0])
            hn[o:o + 3 * H * W] = np.ascontiguousarray(im).reshape(-1)
        n_small = io["small_layout"] + 4 * n_tab
        io["small"][:n_small].copy_(io["host_small"][:n_small], non_blocking=True)
        n_src = mb["need"][0]
        io["src"][:n_src].copy_(host[:n_src], non_blocking=True)

    def detect(self, io, conf, iou, max_det):
        """After :meth:`stage`, on the same stream: letterbox (the ragged kernel for a batch of different sizes) -> YOLOv9-E
        forward -> decode -> NMS, outputs in the slot (no host sync)."""
        plan: YoloPlan = io["plan"]
        B = io["B"]
        if io.get("mixed"):
            tw, th = io["canvas"]
            ops.letterbox_batch(io["src"], B, io["host_views"]["desc"], io["desc"], io["tables"], tw, th, io["tmp"],
                                plan.canvas)
        else:
            H, W = io["src"].shape[1:3]
            tw, th, scale, rw, rh, pl, pt = io["geom"]
            ops.letterbox(io["src"], B, H, W, rw, rh, tw, th, pl, pt, io["tmp"], plan.canvas)
        plan.run()
        ops.yolo_decode(plan.cls_out, plan.box_out, plan.hw, self.weights.nc, B, float(conf), io["pad_l"], io["pad_t"],
                        io["scale"], io["cap"], io["cand_box"], io["cand_score"], io["cand_cls"], io["cand_count"])
        ops.batched_nms(io["cand_box"], io["cand_score"], io["cand_cls"], io["cand_count"], B, io["cap"], iou, max_det,
                        io["img_w"], io["img_h"], io["keep"], io["out_box"], io["out_score"], io["out_count"])

    def filter_device(self, io, ocr_elems, iou_threshold, max_det=300) -> bool:
        """After :meth:`detect`, on the same stream: the reference's overlap filter (ref:util/utils.py:241-319,
        :411-415, :444-451) on the device -> per-icon state, OCR label masks / removed flags and the batch's crop list, plus
        the async D2H of the flags into this io slot's pinned mirrors.  ``ocr_elems[i]`` = host_glue.ocr_elements(...) of
        screenshot i (the strings stay on the host).  Returns False -- nothing launched -- when a screenshot has more OCR boxes
        than the kernel takes; the caller then runs the host list logic (host_glue.build_elements) instead."""
        mo = io["max_ocr"]
        if any(len(e) > mo for e in ocr_elems):
            return False
        hr, hc = io["host_ocr_ratio"], io["host_ocr_count"]
        for i, e in enumerate(ocr_elems):
            hc[i] = len(e)
            if e:
                hr[i, :len(e)] = torch.tensor([x["bbox"] for x in e], dtype=torch.float32)
        io["ocr_ratio"].copy_(hr, non_blocking=True)
        io["ocr_count"].copy_(hc, non_blocking=True)
        ops.overlap_filter(io["out_box"], io["out_count"], len(ocr_elems), max_det, io["img_w"], io["img_h"], io["ocr_ratio"],
                           io["ocr_count"], mo, float(iou_threshold), io["icon_state"], io["label_mask"], io["ocr_removed"],
                           io["icon_ratio"], io["crop_box"], io["crop_img"], io["crop_counts"], io["arrive"])
        for h_, d_ in (("host_state", "icon_state"), ("host_mask", "label_mask"), ("host_removed", "ocr_removed"),
                       ("host_ratio", "icon_ratio"), ("host_crop_counts", "crop_counts")):
            io[h_].copy_(io[d_], non_blocking=True)
        return True

    @staticmethod
    def elements_from_io(io, i, n_det, ocr_elem):
        """Screenshot i of a filtered batch (after the D2H above has completed) -> the reference's sorted element list."""
        from . import host_glue
        return host_glue.elements_from_flags(io["host_ratio"][i, :n_det].tolist(), io["host_state"][i, :n_det].tolist(),
                                             (io["host_mask"][i, :n_det].numpy().view("uint32")), ocr_elem,
                                             io["host_removed"][i, :len(ocr_elem)].tolist())

    @staticmethod
    def check_capacity(cand_count_host: torch.Tensor, cap: int) -> None:
        """The decode kernel keeps the first ``cap`` candidates in anchor order; more than that (only reachable with
        full-resolution ``imgsz`` and a very low threshold) would silently drop the coarse-stride candidates."""
        m = int(cand_count_host.max()) if cand_count_host.numel() else 0
        if m > cap:
            raise RuntimeError(f"{m} candidates above the confidence threshold exceed the NMS capacity ({cap}): raise the "
                               "threshold or lower imgsz")

    @torch.inference_mode()
    def predict_batch(self, images: Sequence[np.ndarray], conf=0.25, imgsz=640, iou=0.7, max_det=300) -> List[Result]:
        """u8 HWC images -> one Result per image (one H2D copy of the screenshots, one D2H of the counts).  Screenshots of
        different sizes share one batch through the ragged letterbox."""
        for im in images:
            assert im.ndim == 3 and im.shape[2] == 3 and im.dtype == np.uint8
        with self._lock, torch.cuda.device(self.device):
            io = self.io_slot([im.shape[:2] for im in images], imgsz, max_det)
            self.stage(io, images)
            self.detect(io, conf, iou, max_det)
            return self._results(io)

    def _results(self, io):
        counts = io["out_count"].cpu().tolist()
        self.check_capacity(io["cand_count"].cpu(), io["cap"])
        return [Result(Boxes(io["out_box"][i, :n].clone(), io["out_score"][i, :n].clone())) for i, n in enumerate(counts)]

    @torch.inference_mode()
    def predict(self, source, conf=0.25, imgsz=640, iou=0.7, max_det=300):
        """ref:util/yolov9.py:115-136."""
        return self.predict_batch([self._load_image(source)], conf, imgsz, iou, max_det)
