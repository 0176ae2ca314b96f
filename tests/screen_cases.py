"""Case definitions of the screen kernels' tests (letterbox, overlap filter, crop + resize), shared by
tests/test_screen_kernels_gpu.py, which runs them on the device, and tests/test_screen_cases_cpu.py, which checks on the
CPU that the oracles agree with their libraries on exactly these cases and that the cases reach every branch of the
kernels.  Everything is seeded; the expensive reference evaluations are cached per case."""
from __future__ import annotations

import functools
from dataclasses import dataclass

import numpy as np
import torch

from omniparser_b200 import host_glue
from oracle import ref_restate as R

W, H = 1920, 1080
WHWH = torch.Tensor([W, H, W, H])
MAX_DET, MAX_OCR = 300, 256          # the detector's device overlap filter (detector.py: max_det 300, OCR_CAP 256)
KERNEL_LIMIT = 512                   # overlap_filter.cu: kOvlMaxIcons = kOvlMaxOcr = 512
CHUNK = 256                          # overlap_filter.cu: kOvlThreads, the compaction chunk


# ------------------------------------------------------------------------------------------------ overlap filter
# Engineered structures live right of x = 1420 px; random icons and free OCR boxes stay left of it, so the engineered
# icons are never suppressed by a random one and the label / drop indices below are exactly what the walk sees.
BIG = (1430, 20, 1900, 400)                   # labelled by OCR boxes in all 8 mask words (needs m = 256)
BIG_LABELS = (5, 40, 70, 100, 130, 170, 200, 250)
# (icon, OCR indices inside it, index of the OCR box that contains it = where the walk drops it)
DROPS = [((1430, 450, 1530, 520), (2, 17), 31),      # drop at k % 32 == 31
         ((1560, 450, 1660, 520), (6, 30), 32),      # drop at k % 32 == 0, first box of a mask word
         ((1690, 450, 1790, 520), (101, 224, 251), 255),
         ((1430, 560, 1530, 630), (41, 45), 47),     # drop inside a word, after labels in the same word
         ((1820, 450, 1910, 520), (), 3)]            # drop before any label
NESTED = [(1560, 560, 1700, 660), (1570, 570, 1690, 650), (1580, 580, 1680, 640), (1590, 590, 1670, 630)]
ZERO_AREA_AT = (250, 253, 255, 256, 259, 262)   # zero int_box_area icons: holes on both sides of the chunk boundary


def _label_box(icon, j):
    """a small OCR box strictly inside `icon` (pixel ints), shifted by j so that several labels of one icon differ"""
    x0, y0, x1, y1 = icon
    w, h = max(4, (x1 - x0) // 6), max(3, (y1 - y0) // 6)
    ox = x0 + 2 + (j * 7) % max(1, x1 - x0 - w - 4)
    oy = y0 + 2 + (j * 5) % max(1, y1 - y0 - h - 4)
    return [ox, oy, ox + w, oy + h]


def screenshot(seed, n, m):
    """-> (px fp32 [n, 4] detector boxes in pixels, OCR int pixel boxes [m], texts [m]).  n icons in NMS output format
    (fp32 pixels inside the image), m OCR boxes that all pass int_box_area, with the engineered structures above placed
    where n and m allow."""
    rng = np.random.default_rng(seed)
    x0 = rng.uniform(0, 1360, n); y0 = rng.uniform(0, 1040, n)
    bw = rng.uniform(6, 60, n); bh = rng.uniform(6, 40, n)
    px = np.stack([x0, y0, x0 + bw, y0 + bh], 1)
    for i in range(3, n, 17):                           # duplicates (equal areas: neither suppresses the other)
        px[i] = px[i - 1]
    for i in range(9, n - 3, 41):                       # nested chains of three
        px[i + 1] = px[i] + (2, 2, -2, -2)
        px[i + 2] = px[i] + (4, 3, -4, -3)
    for i in ZERO_AREA_AT:
        if i < n:
            px[i, 0] = np.floor(px[i, 0]) + 0.3; px[i, 2] = px[i, 0] + 0.2
    eng = [BIG] + [d[0] for d in DROPS] + NESTED
    slots = [n - 1, 1, 257, 120, 290, 7, 200, 201, 258, 12]   # spread over both compaction chunks
    placed = set()
    for s, box in zip(slots, eng):
        if 0 <= s < n:
            px[s] = box
            placed.add(box)
    ocr = [None] * m
    # engineered OCR boxes first (fixed indices), then free ones in the gaps
    if BIG_LABELS[-1] < m and BIG in placed:
        for j, k in enumerate(BIG_LABELS):
            ocr[k] = _label_box(BIG, j)
    for icon, labels, kd in DROPS:
        if kd < m and icon in placed:
            assert all(ocr[k] is None for k in labels + (kd,))
            for j, k in enumerate(labels):
                ocr[k] = _label_box(icon, j + 1)
            ocr[kd] = [icon[0] - 8, icon[1] - 7, icon[2] + 9, icon[3] + 8]
    for k in range(m):
        if ocr[k] is not None:
            continue
        r = rng.uniform()
        if n and r < 0.3:                                  # label of a random icon
            i = int(rng.integers(0, n))
            b = px[i]
            if b[2] - b[0] >= 8 and b[3] - b[1] >= 8 and b[0] < 1400:
                ocr[k] = _label_box([int(np.ceil(b[0])), int(np.ceil(b[1])), int(b[2]), int(b[3])], k)
                continue
        if n and r < 0.45:                                 # contains a random icon
            i = int(rng.integers(0, n))
            b = px[i]
            if b[0] < 1400:
                ocr[k] = [int(b[0]) - 6, int(b[1]) - 5, min(1419, int(b[2]) + 7), int(b[3]) + 6]
                if ocr[k][2] - ocr[k][0] >= 4 and ocr[k][3] - ocr[k][1] >= 4:
                    continue
        x, y = int(rng.integers(0, 1300)), int(rng.integers(0, 1050))
        ocr[k] = [x, y, x + int(rng.integers(8, 110)), y + int(rng.integers(6, 26))]
    ocr = [[min(max(0, v), lim) for v, lim in zip(b, (W, H, W, H))] for b in ocr]
    texts = [f"s{seed}k{k}" for k in range(m)]
    for k in range(60, m, 97):                             # equal OCR dicts: same box, same text
        ocr[k] = list(ocr[k - 1]); texts[k] = texts[k - 1]
    px = np.clip(px, 0, [W, H, W, H]).astype(np.float32)
    return torch.from_numpy(px), ocr, texts


@dataclass(frozen=True)
class OvlCase:
    name: str
    counts: tuple          # detector count per screenshot (may exceed max_det: the kernel clips)
    ocr: tuple             # OCR boxes per screenshot
    thrs: tuple
    max_det: int = MAX_DET
    max_ocr: int = MAX_OCR
    seed: int = 0

    @property
    def B(self):
        return len(self.counts)


OVL_CASES = [
    OvlCase("b8_bench", (300, 0, 257, 256, 1, 350, 255, 300), (256, 33, 0, 32, 1, 255, 31, 256), (0.7, 0.9), seed=100),
    OvlCase("b16", (0, 300, 1, 255, 256, 257, 300, 350, 300, 0, 257, 299, 256, 1, 300, 255),
            (256, 256, 0, 31, 32, 33, 255, 256, 1, 0, 256, 33, 31, 1, 255, 32), (0.7, 0.9), seed=200),
    OvlCase("b3_small_thr01", (40, 300, 12), (33, 256, 5), (0.1,), seed=300),
    OvlCase("b2_kernel_limits", (512, 512), (512, 512), (0.7,), max_det=KERNEL_LIMIT, max_ocr=KERNEL_LIMIT, seed=400),
]


@functools.lru_cache(maxsize=None)
def ovl_inputs(case: OvlCase):
    """per screenshot: (px [min(count, max_det), 4] fp32, ocr int boxes, texts, icon ratio list, OCR ratio list, OCR elements)"""
    out = []
    for b, (n, m) in enumerate(zip(case.counts, case.ocr)):
        px, ob, texts = screenshot(case.seed + b, min(n, case.max_det), m)
        ratio = (px / WHWH).tolist()                                        # ref:util/utils.py:432
        el = host_glue.ocr_elements((torch.tensor(ob) / WHWH).tolist() if ob else None, texts, W, H)
        assert len(el) == m, "every OCR box of the cases passes int_box_area"
        out.append((px, ob, texts, ratio, [e["bbox"] for e in el], el))
    return out


@functools.lru_cache(maxsize=None)
def ovl_flags(case: OvlCase, thr: float):
    """the reference loops' flags per screenshot: (state, mask [n][max_ocr/32], removed)"""
    out = []
    for px, ob, texts, ratio, oratio, el in ovl_inputs(case):
        st, mk, rm = R.overlap_flags_loops(ratio, oratio, W, H, thr)
        words = case.max_ocr // 32
        out.append((st, [row + [0] * (words - len(row)) for row in mk], rm))
    return out


@functools.lru_cache(maxsize=None)
def ovl_elements(case: OvlCase, thr: float):
    """per screenshot: host_glue.build_elements (pinned to the unmodified reference) -> (elements, crop boxes in order)"""
    out = []
    for px, ob, texts, ratio, oratio, el in ovl_inputs(case):
        elems, _ = host_glue.build_elements(ratio, oratio if oratio else None, texts, W, H, thr)
        out.append((elems, [e["bbox"] for e in elems if e["content"] is None]))
    return out


def ovl_crop_list(case: OvlCase, thr: float):
    """the batch crop list the kernel must emit: fp32 ratio boxes and screenshot ids, screenshot-major in element order"""
    boxes, img = [], []
    for b, (elems, crops) in enumerate(ovl_elements(case, thr)):
        boxes += crops
        img += [b] * len(crops)
    return np.asarray(boxes, np.float32).reshape(-1, 4), np.asarray(img, np.int32)


def drop_index(icon, oratio):
    """index of the OCR box where the reference walk drops `icon` (contains it without being inside it), else None"""
    for k, o in enumerate(oratio):
        if host_glue._inter(o, icon) / host_glue._area(o) > 0.80:
            continue
        if host_glue._inter(icon, o) / host_glue._area(icon) > 0.80:
            return k
    return None


# ------------------------------------------------------------------------------------------------ images
def image(seed, h, w, kind):
    """u8 HWC.  'noise': uniform bytes; 'edges': per channel, axis-aligned 0/255 bands 12..160 px wide in both directions
    (hard steps the Lanczos / bilinear lobes ring across, so clipping at 0 and 255 occurs) plus a noise patch; 'stripes':
    0/255 vertical and horizontal stripes 1..7 px wide (saturated content at crop scale)."""
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
    lo, hi = (12, 160) if kind == "edges" else (1, 8)

    def bands(n):
        cuts = np.cumsum(rng.integers(lo, hi, size=n // lo + 2))
        return (np.searchsorted(cuts, np.arange(n), side="right") & 1).astype(bool)

    img = np.empty((h, w, 3), np.uint8)
    for c in range(3):
        img[..., c] = np.where(bands(h)[:, None] ^ bands(w)[None, :], 255, 0)
    if kind == "edges":
        ph, pw = max(1, h // 5), max(1, w // 5)
        img[:ph, :pw] = rng.integers(0, 256, size=(ph, pw, 3), dtype=np.uint8)
    return img


# ------------------------------------------------------------------------------------------------ letterbox
@dataclass(frozen=True)
class LbCase:
    name: str
    w: int
    h: int
    B: int
    imgsz: object = 640
    kind: str = "edges"
    seed: int = 0


LB_CASES = [
    LbCase("1280x720", 1280, 720, 2, seed=1),
    LbCase("1366x768", 1366, 768, 2, seed=2),
    LbCase("2560x1440", 2560, 1440, 1, seed=3),
    LbCase("3840x2160_ksize37", 3840, 2160, 1, seed=4),
    LbCase("portrait_1170x2532", 1170, 2532, 1, seed=5),
    LbCase("2532x1170", 2532, 1170, 1, seed=6),
    LbCase("4000x60_to_640x9", 4000, 60, 2, seed=7),
    LbCase("60x4000_to_9x640", 60, 4000, 2, seed=8),
    LbCase("300x200_upscale", 300, 200, 2, seed=9),
    LbCase("636x50_h_only", 636, 50, 2, seed=14),        # scale 640/636: 50 rows stay 50, the vertical pass is skipped
    LbCase("50x636_v_only", 50, 636, 2, seed=15),
    # get_som_labeled_img's default imgsz is the image's own (h, w) (ref:util/utils.py:428-429): 1366 -> 1376 wide
    # canvas at scale 1, so both passes are skipped and the image is pasted with a 5 px pad
    LbCase("1366x768_imgsz_hw", 1366, 768, 2, imgsz=(768, 1366), seed=10),
    LbCase("1920x1080_tuple_upscale", 1920, 1080, 1, imgsz=(1440, 2560), seed=11),
    LbCase("b8_1920x1080_bench", 1920, 1080, 8, kind="noise", seed=12),
    LbCase("b8_1920x1080_edges", 1920, 1080, 8, seed=13),
]


def lb_images(c: LbCase):
    return np.stack([image(c.seed * 100 + b, c.h, c.w, c.kind) for b in range(c.B)])


@functools.lru_cache(maxsize=None)
def lb_expected(c: LbCase):
    """(canvas [B, th, tw, 3] through Pillow, geometry)"""
    imgs = lb_images(c)
    return np.stack([R.letterbox_pil(im, c.imgsz)[0] for im in imgs]), R.letterbox_geometry(c.w, c.h, c.imgsz)


def lanczos_extremes(img, rw, rh):
    """(min, max) over both passes of the unclipped 8-bit results (acc >> 22) of Pillow's two-pass LANCZOS, as
    oracle.ref_restate.resize_lanczos_numpy computes them before np.clip"""
    h, w, _ = img.shape
    lo, hi = 0, 255
    cur = img.astype(np.int64)
    if rw != w:
        bounds, kk = R.lanczos_coeffs(w, rw)
        acc = np.empty((h, rw, 3), np.int64)
        for xx in range(rw):
            x0, n = bounds[xx]
            acc[:, xx] = ((1 << 21) + (cur[:, x0:x0 + n] * kk[xx, :n, None].astype(np.int64)[None]).sum(1)) >> 22
        lo, hi = min(lo, int(acc.min())), max(hi, int(acc.max()))
        cur = np.clip(acc, 0, 255)
    if rh != h:
        bounds, kk = R.lanczos_coeffs(h, rh)
        for yy in range(rh):
            y0, n = bounds[yy]
            a = ((1 << 21) + (cur[y0:y0 + n] * kk[yy, :n, None, None].astype(np.int64)).sum(0)) >> 22
            lo, hi = min(lo, int(a.min())), max(hi, int(a.max()))
    return lo, hi


@functools.lru_cache(maxsize=None)
def lb_clipping(c: LbCase):
    """(clips at 0, clips at 255) somewhere in the batch"""
    _, _, _, rw, rh, _, _ = R.letterbox_geometry(c.w, c.h, c.imgsz)
    ext = [lanczos_extremes(im, rw, rh) for im in lb_images(c)]
    return any(e[0] < 0 for e in ext), any(e[1] > 255 for e in ext)


def lb_ksize(in_size, out_size):
    return int(np.ceil(3.0 * max(1.0, in_size / out_size))) * 2 + 1


# ------------------------------------------------------------------------------------------------ crop + resize
# Hand-placed boxes as pixel rectangles; ratios are (px + 0.5) / size in fp32, so int(ratio * size) is exactly px.
# Entries that are already ratios (clamped / empty / full-screen cases) are given as ("r", x0, y0, x1, y1).
CROP_BOXES = [
    ("sw1", (500, 300, 501, 340)), ("sh1", (500, 300, 540, 301)), ("1x1", (700, 700, 701, 701)),
    ("64x64", (10, 10, 74, 74)), ("128x128_area", (100, 100, 228, 228)), ("128x127", (300, 100, 428, 227)),
    ("127x128", (300, 400, 427, 528)), ("128x64", (600, 100, 728, 164)), ("64x128", (600, 300, 664, 428)),
    ("2x1", (20, 900, 22, 901)), ("up_x_down_y", (800, 100, 820, 400)), ("down_x_up_y", (800, 500, 1100, 517)),
    ("upscale_both", (1000, 700, 1031, 733)), ("63x65", (1200, 100, 1263, 165)), ("65x63", (1200, 300, 1265, 363)),
    ("odd_down", (1300, 500, 1491, 617)),
    ("full_screen", ("r", 0.0, 0.0, 1.0, 1.0)),
    ("xmax_ymax_at_edge", ("r", 0.9, 0.95, 1.0, 1.0)),
    ("right_edge_1px", ("r", 0.999, 0.5, 1.0, 0.55)),
    ("clamped_low", ("r", -0.1, -0.2, 0.05, 0.04)), ("clamped_high", ("r", 0.97, 0.96, 1.3, 1.2)),
    ("clamped_all", ("r", -0.5, -0.5, 1.5, 1.5)),
    ("empty_zero_w", ("r", 0.5, 0.5, 0.5, 0.6)), ("empty_reversed", ("r", 0.6, 0.5, 0.4, 0.6)),
    ("empty_outside", ("r", 1.2, 1.1, 1.5, 1.4)), ("empty_negative", ("r", -0.5, 0.2, -0.1, 0.4)),
]
EMPTY_SUB_PIXEL = ("empty_sub_pixel", 500.2, 500.8)   # both ends truncate to column 500


def crop_ratio(spec, w, h):
    if spec[0] == "r":
        return np.asarray(spec[1:], np.float32)
    x0, y0, x1, y1 = spec
    return np.asarray([(x0 + 0.5) / w, (y0 + 0.5) / h, (x1 + 0.5) / w, (y1 + 0.5) / h], np.float32)


@dataclass(frozen=True)
class CropCase:
    name: str
    sizes: tuple           # (h, w) per image, packed back to back through img_hw / img_off
    kinds: tuple


CROP_CASES = [
    CropCase("1920x1080", ((H, W), (H, W)), ("noise", "stripes")),
    CropCase("3840x2160", ((2160, 3840), (2160, 3840)), ("stripes", "noise")),
    CropCase("mixed_sizes", ((H, W), (2160, 3840), (768, 1366)), ("noise", "stripes", "noise")),
]


def crop_images(c: CropCase):
    return [image(7000 + i, h, w, k) for i, ((h, w), k) in enumerate(zip(c.sizes, c.kinds))]


def crop_boxes(c: CropCase):
    """every hand-placed box on every image of the case, then the sub-pixel empty box -> (ratios [n,4] fp32, image ids)"""
    boxes, img = [], []
    for i, (h, w) in enumerate(c.sizes):
        for _, spec in CROP_BOXES:
            boxes.append(crop_ratio(spec, w, h)); img.append(i)
        x = np.float32([EMPTY_SUB_PIXEL[1] / w, 0.3, EMPTY_SUB_PIXEL[2] / w, 0.4])
        boxes.append(x); img.append(i)
    return np.stack(boxes).astype(np.float32), np.asarray(img, np.int32)


def crop_geometry(ratio, w, h):
    """int(c * size) on fp32 (ref:util/utils.py:99-100), then numpy's slice clamping -> (raw ints, clamped ints)"""
    raw = R.crop_boxes_int(torch.from_numpy(np.ascontiguousarray(ratio[None])), w, h)[0]
    xa, ya, xb, yb = raw
    cl = (max(0, min(xa, w)), max(0, min(ya, h)), max(0, min(xb, w)), max(0, min(yb, h)))
    return raw, cl


def crop_branches(sw, sh, out=64):
    """the branches of crop_resize_kernel one crop of sw x sh takes"""
    if sw <= 0 or sh <= 0:
        return {"empty"}
    if sw == 2 * out and sh == 2 * out:
        return {"area"}
    br = set()
    d = np.arange(out, dtype=np.float64)
    fx = ((d + 0.5) * (1.0 / (out / sw)) - 0.5).astype(np.float32)
    sx = np.floor(fx).astype(np.int64)
    fy = ((d + 0.5) * (1.0 / (out / sh)) - 0.5).astype(np.float32)
    sy = np.floor(fy).astype(np.int64)
    if (sx < 0).any():
        br.add("x_snap_low")
    if (sx >= sw - 1).any():
        br.add("x_snap_high")
    if (sy < 0).any() or (sy + 1 > sh - 1).any():
        br.add("y_clamp")
    if sw == 1:
        br.add("sw1")
    if sh == 1:
        br.add("sh1")
    return br
