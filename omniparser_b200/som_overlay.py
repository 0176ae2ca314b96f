"""Set-of-Marks overlay, label coordinates and PNG/base64 of ``get_som_labeled_img`` (ref:util/utils.py:478-494), the
post-caption part of the path (SURVEY.md §8a row G1, §8f-1).

Restated so that the outputs are IDENTICAL to the reference's:
* ``label_coordinates``: the reference pushes the float32 xyxy ratios through ``box_convert(xyxy->cxcywh)``, a multiply
  by (w, h, w, h), ``box_convert(cxcywh->xywh)`` (= cxcywh->xyxy->xywh) and an optional divide, all in float32
  (ref:util/utils.py:478, :352-355, :335-354 of ``annotate``); the same float32 operations in the same order are done
  here in numpy (checked bit for bit against torchvision in tests/test_overlay_cpu.py and against the goldens).
* label placement: ``get_optimal_label_pos`` (ref:util/box_annotator.py:189-262) is an O(N^2) Python loop over all
  detections per candidate position; here every candidate box is tested against all detections in one vectorised
  int64/float64 expression (same integer areas, same float64 divisions, same strict ``> 0.3``), candidates tried in the
  reference's order (top left, outer left, outer right, top right; last one kept if all overlap).
* drawing: the same ``cv2.rectangle`` / ``cv2.putText`` calls in the same order with the same arguments as
  ``BoxAnnotator.annotate`` (ref:util/box_annotator.py:45-167), including its quirk of drawing ``as_bgr()`` colours on
  an RGB frame.  ``supervision`` itself is not needed: its ``ColorPalette.DEFAULT`` (supervision 0.18.0, pinned at
  ref:requirements.txt) is restated below (recalled; the oracle shim uses the same table).
* PNG: the reference's ``PIL.Image.save(format="PNG")`` (zlib level 6) costs 80-550 ms per screenshot and dominates
  the call once the models are fast; ``encode_png`` writes the same pixels with the Up filter and a zlib level-1 stream
  deflated in parallel row bands.  The decoded image is identical; the byte stream is not (and need not be).
  ``DevicePngEncoder`` does the same encode on the GPU (csrc/png_encode.cu: LZ77 + dynamic Huffman per row band, with
  checksums combined across bands); ``som_outputs(device=cuda)`` uses it, every other device the host encoder.
"""
from __future__ import annotations

import base64
import threading
from typing import Dict, List, Sequence, Tuple

import numpy as np

# supervision 0.18.0 `ColorPalette.DEFAULT` (supervision/draw/color.py DEFAULT_COLOR_PALETTE), hex RGB
DEFAULT_PALETTE_HEX = ["A351FB", "FF4040", "FFA1A0", "FF7633", "FFB633", "D1D435", "4CFB12", "94CF1A", "40DE8A", "1B9640",
                       "00D6C1", "2E9CAA", "00C4FF", "364797", "6675FF", "0019EF", "863AFF", "530087", "CD3AFF", "FF97CA",
                       "FF39C9"]
PALETTE_RGB = [(int(h[0:2], 16), int(h[2:4], 16), int(h[4:6], 16)) for h in DEFAULT_PALETTE_HEX]


def boxes_cxcywh_f32(xyxy_ratio: Sequence[Sequence[float]]) -> np.ndarray:
    """``box_convert(torch.tensor(bboxes), "xyxy", "cxcywh")`` in float32 (ref:util/utils.py:478)."""
    b = np.asarray(xyxy_ratio, dtype=np.float32).reshape(-1, 4)
    x1, y1, x2, y2 = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
    two = np.float32(2)
    return np.stack([(x1 + x2) / two, (y1 + y2) / two, x2 - x1, y2 - y1], -1).astype(np.float32)


def pixel_boxes_f32(cxcywh_ratio: np.ndarray, w: int, h: int) -> Tuple[np.ndarray, np.ndarray]:
    """``annotate``'s first lines (ref:util/utils.py:352-355): scale to pixels, -> (xyxy, xywh), float32."""
    b = (cxcywh_ratio * np.asarray([w, h, w, h], dtype=np.float32)).astype(np.float32)
    cx, cy, bw, bh = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
    half = np.float32(0.5)
    x1, y1, x2, y2 = cx - half * bw, cy - half * bh, cx + half * bw, cy + half * bh
    xyxy = np.stack([x1, y1, x2, y2], -1).astype(np.float32)
    xywh = np.stack([x1, y1, x2 - x1, y2 - y1], -1).astype(np.float32)
    return xyxy, xywh


def label_coordinates(xywh_px: np.ndarray, w: int, h: int, output_coord_in_ratio: bool) -> Dict[str, list]:
    """ref:util/utils.py:363 (``{phrase: xywh}``) and :491-492 (optional ratio form); values are float32 numbers."""
    out = {}
    for i, v in enumerate(xywh_px):
        if output_coord_in_ratio:
            out[str(i)] = [v[0] / np.float32(w), v[1] / np.float32(h), v[2] / np.float32(w), v[3] / np.float32(h)]
        else:
            out[str(i)] = v
    return out


def _overlaps(bg: Sequence[int], det: np.ndarray, det_area: np.ndarray, image_size: Tuple[int, int]) -> bool:
    """``get_is_overlap`` (ref:util/box_annotator.py:195-206): IoU* of the label box with ANY detection > 0.3, or the
    label box leaves the image."""
    bx1, by1, bx2, by2 = (int(v) for v in bg)
    if bx1 < 0 or bx2 > image_size[0] or by1 < 0 or by2 > image_size[1]:
        return True
    if det.shape[0] == 0:
        return False
    iw = np.maximum(0, np.minimum(bx2, det[:, 2]) - np.maximum(bx1, det[:, 0]))
    ih = np.maximum(0, np.minimum(by2, det[:, 3]) - np.maximum(by1, det[:, 1]))
    inter = iw * ih                                               # int64
    a1 = (bx2 - bx1) * (by2 - by1)
    union = a1 + det_area - inter
    with np.errstate(divide="ignore", invalid="ignore"):
        iou = inter / union
        if a1 > 0:
            pos = det_area > 0
            r1 = np.where(pos, inter / a1, 0.0)
            r2 = np.where(pos, inter / np.where(pos, det_area, 1), 0.0)
            iou = np.maximum(np.maximum(iou, r1), r2)
    return bool((iou > 0.3).any())


def optimal_label_pos(pad: int, tw: int, th: int, x1: int, y1: int, x2: int, y2: int, det: np.ndarray, det_area: np.ndarray,
                      image_size: Tuple[int, int]):
    """ref:util/box_annotator.py:189-262 -> (text_x, text_y, bg_x1, bg_y1, bg_x2, bg_y2)."""
    cands = (
        (x1 + pad, y1 - pad, x1, y1 - 2 * pad - th, x1 + 2 * pad + tw, y1),                      # top left
        (x1 - pad - tw, y1 + pad + th, x1 - 2 * pad - tw, y1, x1, y1 + 2 * pad + th),            # outer left
        (x2 + pad, y1 + pad + th, x2, y1, x2 + 2 * pad + tw, y1 + 2 * pad + th),                 # outer right
        (x2 - pad - tw, y1 - pad, x2 - 2 * pad - tw, y1 - 2 * pad - th, x2, y1),                 # top right
    )
    for c in cands:
        if not _overlaps(c[2:], det, det_area, image_size):
            return c
    return cands[-1]


def annotate(image_rgb: np.ndarray, xyxy_px: np.ndarray, text_scale: float, text_padding: int = 5, text_thickness: int = 2,
             thickness: int = 3) -> np.ndarray:
    """``BoxAnnotator(...).annotate(scene=image.copy(), detections, labels=[str(i)], image_size=(w, h))``
    (ref:util/box_annotator.py:45-167 as called from ref:util/utils.py:359-361)."""
    import cv2
    h, w = image_rgb.shape[:2]
    scene = np.ascontiguousarray(image_rgb.copy())
    det = xyxy_px.astype(int).reshape(-1, 4)           # truncation toward zero, as `.astype(int)` at :95
    det_area = (det[:, 2] - det[:, 0]) * (det[:, 3] - det[:, 1])
    font = cv2.FONT_HERSHEY_SIMPLEX
    for i in range(det.shape[0]):
        x1, y1, x2, y2 = (int(v) for v in det[i])
        r, g, b = PALETTE_RGB[i % len(PALETTE_RGB)]
        bgr = (b, g, r)                                  # `color.as_bgr()` on an RGB frame: the reference's quirk, kept
        cv2.rectangle(img=scene, pt1=(x1, y1), pt2=(x2, y2), color=bgr, thickness=thickness)
        text = str(i)
        tw_, th_ = cv2.getTextSize(text=text, fontFace=font, fontScale=text_scale, thickness=text_thickness)[0]
        tx, ty, bx1, by1, bx2, by2 = optimal_label_pos(text_padding, tw_, th_, x1, y1, x2, y2, det, det_area, (w, h))
        cv2.rectangle(img=scene, pt1=(bx1, by1), pt2=(bx2, by2), color=bgr, thickness=cv2.FILLED)
        luminance = 0.299 * r + 0.587 * g + 0.114 * b
        text_color = (0, 0, 0) if luminance > 160 else (255, 255, 255)
        cv2.putText(img=scene, text=text, org=(tx, ty), fontFace=font, fontScale=text_scale, color=text_color,
                    thickness=text_thickness, lineType=cv2.LINE_AA)
    return scene


_POOL = None


def _pool():
    global _POOL
    if _POOL is None:
        import os
        from concurrent.futures import ThreadPoolExecutor
        n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 4)
        _POOL = ThreadPoolExecutor(max_workers=max(1, min(16, n)), thread_name_prefix="b2p-png")
    return _POOL


def encode_png(frame_rgb: np.ndarray, level: int = 1, stripes: int = 0) -> bytes:
    """Lossless 8-bit RGB PNG of the annotated frame.  The reference's ``PIL.Image.save(format="PNG")`` (one zlib stream at
    level 6, adaptive filters) is the largest remaining cost of the call; here every row gets the Up filter (one vectorised
    subtraction) and the IDAT stream is deflated in ``stripes`` row bands in parallel (zlib releases the GIL), each band
    ending on a sync-flush boundary so the concatenation is ONE valid zlib stream (the pigz construction).  Same pixels
    after decoding; not the same bytes."""
    import struct
    import zlib
    h, w, c = frame_rgb.shape
    assert c == 3 and frame_rgb.dtype == np.uint8
    rows = np.ascontiguousarray(frame_rgb).reshape(h, w * 3)
    filt = np.empty((h, 1 + w * 3), np.uint8)
    filt[:, 0] = 2                                  # filter type Up: Raw(x) - Prior(x) mod 256 (first row: prior = 0)
    filt[0, 1:] = rows[0]
    np.subtract(rows[1:], rows[:-1], out=filt[1:, 1:])
    pool = _pool()
    n = stripes or min(pool._max_workers, max(1, h // 64))
    edges = [h * i // n for i in range(n + 1)]
    raw = memoryview(filt).cast("B")
    pitch = 1 + w * 3

    def band(i):
        co = zlib.compressobj(level, zlib.DEFLATED, -15)
        data = co.compress(raw[edges[i] * pitch:edges[i + 1] * pitch])
        return data + co.flush(zlib.Z_FINISH if i == n - 1 else zlib.Z_SYNC_FLUSH)

    parts = list(pool.map(band, range(n))) if n > 1 else [band(0)]
    idat = b"\x78\x01" + b"".join(parts) + struct.pack(">I", zlib.adler32(raw) & 0xFFFFFFFF)

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)

    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0)) + chunk(b"IDAT", idat) +
            chunk(b"IEND", b""))


class DevicePngEncoder:
    """PNG encode of RGB frames on one CUDA device (b2p_png_encode), for callers on any thread.  One lock serialises the
    encodes; they run on the encoder's own role stream.  Pinned input / output staging and the device buffers grow to
    the largest frame seen and are kept."""

    def __init__(self, device):
        import torch
        from . import ops
        self.device = ops._stream_device(device)
        self.stream = ops.role_stream("png", self.device)
        self.lock = threading.Lock()
        self._pin_in = self._pin_out = self._dev_in = self._dev_out = self._ws = None
        self._dev_len = None
        self._pin_len = self._pinned(1, torch.int64)

    @staticmethod
    def _pinned(n, dtype=None):
        import torch
        return torch.empty(n, dtype=dtype or torch.uint8, pin_memory=True)

    def _device_buf(self, n, dtype=None):
        import torch
        return torch.empty(n, dtype=dtype or torch.uint8, device=self.device)

    @staticmethod
    def _grow(buf, n, alloc):
        return buf if buf is not None and buf.numel() >= n else alloc(n)

    def encode(self, frame_rgb: np.ndarray) -> bytes:
        import torch
        from . import ops
        h, w, c = frame_rgb.shape
        assert c == 3 and frame_rgb.dtype == np.uint8
        _, ws_bytes, out_cap = ops.png_plan(h, w)
        n_in = h * w * 3
        with self.lock:
            self._pin_in = self._grow(self._pin_in, n_in, self._pinned)
            self._dev_in = self._grow(self._dev_in, n_in, self._device_buf)
            self._ws = self._grow(self._ws, ws_bytes, self._device_buf)
            self._pin_out = self._grow(self._pin_out, out_cap, self._pinned)
            self._dev_out = self._grow(self._dev_out, out_cap, self._device_buf)
            if self._dev_len is None:
                self._dev_len = self._device_buf(1, torch.int64)
            self._pin_in[:n_in].numpy().reshape(h, w, 3)[...] = frame_rgb
            with torch.cuda.stream(self.stream):
                self._dev_in[:n_in].copy_(self._pin_in[:n_in], non_blocking=True)
                ops.png_encode(self._dev_in, h, w, self._ws, self._ws.numel(), self._dev_out, self._dev_out.numel(),
                               self._dev_len)
                self._pin_len.copy_(self._dev_len, non_blocking=True)
                self.stream.synchronize()
                n = int(self._pin_len[0])
                assert 0 < n <= out_cap, (n, out_cap)
                self._pin_out[:n].copy_(self._dev_out[:n], non_blocking=True)
                self.stream.synchronize()
            return self._pin_out[:n].numpy().tobytes()


_ENCODERS = {}
_ENCODERS_LOCK = threading.Lock()


def device_encoder(device) -> DevicePngEncoder:
    """the process's encoder for ``device`` (created on first use)"""
    from . import ops
    key = str(ops._stream_device(device))
    with _ENCODERS_LOCK:
        enc = _ENCODERS.get(key)
        if enc is None:
            enc = _ENCODERS[key] = DevicePngEncoder(device)
        return enc


def _is_cuda(device) -> bool:
    if device is None:
        return False
    try:
        import torch
        return torch.device(device).type == "cuda"
    except (TypeError, RuntimeError):
        return False


def som_outputs(image_rgb: np.ndarray, boxes_xyxy_ratio: List[List[float]], output_coord_in_ratio: bool, text_scale=0.4,
                text_padding=5, text_thickness=2, thickness=3, png_level: int = 1, device=None):
    """Everything after the captions: -> (base64 PNG, label_coordinates) (ref:util/utils.py:478-494).  With a CUDA
    ``device`` the PNG is encoded there (:class:`DevicePngEncoder`); otherwise on the host (:func:`encode_png`).  The
    decoded overlay is the same either way."""
    h, w = image_rgb.shape[:2]
    cxcywh = boxes_cxcywh_f32(boxes_xyxy_ratio)
    xyxy_px, xywh_px = pixel_boxes_f32(cxcywh, w, h)
    frame = annotate(image_rgb, xyxy_px, text_scale, text_padding, text_thickness, thickness)
    png = device_encoder(device).encode(frame) if _is_cuda(device) else encode_png(frame, png_level)
    encoded = base64.b64encode(png).decode("ascii")
    return encoded, label_coordinates(xywh_px, w, h, output_coord_in_ratio), frame
