"""The byte and list kernels between the screenshot and the caption model, bit for bit, at full detector capacity and at
their geometric edges:

* `b2p_overlap_filter` (csrc/overlap_filter.cu) against the reference loops restated as flags
  (`oracle.ref_restate.overlap_flags_loops`) and, through `host_glue.elements_from_flags`, against the element lists of
  `host_glue.build_elements` (pinned to the unmodified reference), on batches of 8 and 16 screenshots with 0..350
  detections (past `max_det` = 300) and 0..256 OCR boxes, engineered labels / drops on mask-word boundaries, and one
  batch at the kernel's limits (512 icons, 512 OCR boxes).  Each batch runs twice on one arrival counter;
* `b2p_crop_resize` against `cv2.resize` on the overlap filter's own crop list (the production chain) and on
  hand-placed boxes that take every branch, on 1920x1080, 3840x2160 and mixed-size images;
* `b2p_letterbox` against Pillow on real screenshot sizes, extreme aspect ratios and hard-edged content that clips at 0
  and 255, and `b2p_resize_u8` at the 768 caption mode's one call (16 crops, 64 -> 768 BICUBIC);
* the host-side rejections of degenerate letterbox / resize geometries.

Every output buffer is poisoned and followed by a guard region that must come back unchanged; before every launch a
host-side check confirms that each address the kernel can touch lies inside its torch allocation.  The case lists
and their coverage live in tests/screen_cases.py (checked on the CPU by tests/test_screen_cases_cpu.py)."""
from __future__ import annotations

import numpy as np
import pytest
import torch

import screen_cases as S
from omniparser_b200 import host_glue, ops
from oracle import ref_restate as R
from test_parity_planes_gpu import _rejected

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
GUARD = 4096                 # elements after every output
POISON_U8 = 0xA5
SENT_I32 = -7
SENT_F32 = -60000.0


def guarded(n, dtype, fill):
    """n poisoned elements followed by GUARD poisoned ones -> (output view, whole buffer)"""
    big = torch.full((n + GUARD,), fill, dtype=dtype, device=DEV)
    return big[:n], big


def check_guard(big, n, fill, what):
    tail = big[n:].cpu()
    assert bool((tail == fill).all()), f"{what}: {int((tail != fill).sum())} guard elements after the output were written"


def covers(t, n_elems, what):
    """the kernel addresses elements [0, n_elems) of t (contiguous)"""
    assert t.is_contiguous() and n_elems <= t.numel(), (what, n_elems, t.numel())


def f32_bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


# ------------------------------------------------------------------------------------------------ overlap filter
def ovl_run(case: S.OvlCase, thr: float):
    """both launches of one case on one arrival counter -> host copies of every output (checked for identity, guards and
    arrive == 0 here) plus the device crop list in its production layout"""
    inputs = S.ovl_inputs(case)
    B, md, mo = case.B, case.max_det, case.max_ocr
    words = mo // 32
    f32, i32 = dict(dtype=torch.float32, device=DEV), dict(dtype=torch.int32, device=DEV)
    # inputs: rows past each screenshot's count / OCR count hold NaN, so a read there would show in the outputs
    box = torch.full((B, md, 4), float("nan"), **f32)
    oc = torch.full((B, mo, 4), float("nan"), **f32)
    for b, (px, ob, texts, ratio, oratio, el) in enumerate(inputs):
        box[b, :len(px)] = px.to(DEV)
        if oratio:
            oc[b, :len(oratio)] = torch.tensor(oratio, dtype=torch.float32).to(DEV)
    cnt = torch.tensor(case.counts, **i32)
    ocnt = torch.tensor(case.ocr, **i32)
    iw = torch.full((B,), float(S.W), **f32)
    ih = torch.full((B,), float(S.H), **f32)
    arrive = torch.zeros((1,), **i32)
    sizes = dict(state=(B * md, torch.int32, SENT_I32), mask=(B * md * words, torch.int32, SENT_I32),
                 removed=(B * mo, torch.int32, SENT_I32), ratio=(B * md * 4, torch.float32, SENT_F32),
                 cbox=(B * md * 4, torch.float32, SENT_F32), cimg=(B * md, torch.int32, SENT_I32),
                 ccnt=(B + 1, torch.int32, SENT_I32))
    bufs = {k: guarded(n, dt, fill) for k, (n, dt, fill) in sizes.items()}
    # host-side extent check: every index the kernel forms from (B, max_det, max_ocr)
    for t, n, what in ((box, B * md * 4, "box_px"), (cnt, B, "count"), (iw, B, "img_w"), (ih, B, "img_h"),
                       (oc, B * mo * 4, "ocr_ratio"), (ocnt, B, "ocr_count"), (arrive, 1, "arrive")):
        covers(t, n, what)
    for k, (n, _, _) in sizes.items():
        covers(bufs[k][0], n, k)
    runs = []
    for _ in range(2):
        for k, (n, dt, fill) in sizes.items():
            bufs[k][0].fill_(fill)
        v = {k: bufs[k][0] for k in sizes}
        ops.overlap_filter(box, cnt, B, md, iw, ih, oc, ocnt, mo, thr, v["state"], v["mask"], v["removed"], v["ratio"],
                           v["cbox"], v["cimg"], v["ccnt"], arrive)
        torch.cuda.synchronize()
        assert int(arrive.item()) == 0, "the arrival counter did not reset"
        runs.append({k: t.cpu().clone() for k, t in v.items()})
    for k in sizes:
        assert torch.equal(runs[0][k].view(torch.int32), runs[1][k].view(torch.int32)), f"{k}: the second run differs"
        check_guard(bufs[k][1], sizes[k][0], sizes[k][2], k)
    out = runs[1]
    host = dict(state=out["state"].view(B, md).numpy(), mask=out["mask"].view(B, md, words).numpy().view(np.uint32),
                removed=out["removed"].view(B, mo).numpy(), ratio=out["ratio"].view(B, md, 4).numpy(),
                cbox=out["cbox"].view(B * md, 4).numpy(), cimg=out["cimg"].numpy(), ccnt=out["ccnt"].numpy())
    return host, bufs["cbox"][0].view(B * md, 4), bufs["cimg"][0]


OVL_PARAMS = [(c, thr) for c in S.OVL_CASES for thr in c.thrs]


@pytest.mark.parametrize("case,thr", OVL_PARAMS, ids=[f"{c.name}-thr{t}" for c, t in OVL_PARAMS])
def test_overlap_filter_bit_exact(case, thr):
    got, _, _ = ovl_run(case, thr)
    flags = S.ovl_flags(case, thr)
    elems = S.ovl_elements(case, thr)
    md, mo = case.max_det, case.max_ocr
    for b, ((px, ob, texts, ratio, oratio, el), (st, mk, rm), (ref_el, _)) in enumerate(zip(S.ovl_inputs(case), flags, elems)):
        n, m = len(px), len(oratio)
        assert n == min(case.counts[b], md)
        tag = f"screenshot {b} ({case.counts[b]} icons, {m} OCR)"
        assert got["state"][b, :n].tolist() == st, f"{tag}: icon_state"
        assert not got["state"][b, n:].any(), f"{tag}: icon_state past the count"
        assert np.array_equal(got["mask"][b, :n], np.asarray(mk, np.uint32).reshape(n, mo // 32)), f"{tag}: label_mask"
        assert not got["mask"][b, n:].any(), f"{tag}: label_mask past the count"
        assert got["removed"][b, :m].tolist() == rm, f"{tag}: ocr_removed"
        assert not got["removed"][b, m:].any(), f"{tag}: ocr_removed past the OCR count"
        assert np.array_equal(f32_bits(got["ratio"][b, :n]), f32_bits((px / S.WHWH).numpy())), f"{tag}: icon_ratio != fp32 px / W"
        assert (got["ratio"][b, n:] == SENT_F32).all(), f"{tag}: icon_ratio written past the count"
        el_dev = host_glue.elements_from_flags(got["ratio"][b, :n].tolist(), got["state"][b, :n].tolist(), got["mask"][b, :n],
                                               el, got["removed"][b, :m].tolist())
        assert el_dev == ref_el, f"{tag}: element list differs from host_glue.build_elements"
    exp_box, exp_img = S.ovl_crop_list(case, thr)
    tot = len(exp_img)
    assert got["ccnt"].tolist() == [int((exp_img == b).sum()) for b in range(case.B)] + [tot]
    assert np.array_equal(f32_bits(got["cbox"][:tot]), f32_bits(exp_box)), "crop_box differs from the element order"
    assert np.array_equal(got["cimg"][:tot], exp_img), "crop_img differs from the element order"
    assert (got["cbox"][tot:] == SENT_F32).all() and (got["cimg"][tot:] == SENT_I32).all(), "crop list written past its end"


# ------------------------------------------------------------------------------------------------ crop + resize
def crop_run(imgs, boxes, bimg, n=None):
    """b2p_crop_resize over images packed back to back (img_hw / img_off) -> (out [n,64,64,3] u8, status [n]) on the host.
    boxes / bimg: host arrays or device tensors (the overlap filter's crop list)."""
    n = len(bimg) if n is None else n
    hw_l = [im.shape[:2] for im in imgs]
    off_l = np.concatenate([[0], np.cumsum([h * w * 3 for h, w in hw_l])]).astype(np.int64)
    flat = torch.from_numpy(np.concatenate([im.reshape(-1) for im in imgs])).to(DEV)
    hw = torch.tensor(hw_l, dtype=torch.int32, device=DEV)
    off = torch.from_numpy(off_l[:-1].copy()).to(DEV)
    d_box = boxes if torch.is_tensor(boxes) else torch.from_numpy(boxes).to(DEV)
    d_img = bimg if torch.is_tensor(bimg) else torch.from_numpy(bimg).to(DEV)
    hb, hi = d_box.cpu().numpy(), d_img.cpu().numpy()
    # host-side extent check: each box's clamped source rows inside its image's img_off span, inside the allocation
    covers(d_box, n * 4, "boxes"); covers(d_img, n, "box_img")
    assert off_l[-1] == flat.numel()
    for i in range(n):
        q = int(hi[i])
        assert 0 <= q < len(imgs)
        h, w = hw_l[q]
        _, (xa, ya, xb, yb) = S.crop_geometry(hb[i], w, h)
        if xb > xa and yb > ya:
            assert off_l[q] <= off_l[q] + (ya * w + xa) * 3 and off_l[q] + ((yb - 1) * w + xb) * 3 <= off_l[q + 1]
    out, out_big = guarded(n * 64 * 64 * 3, torch.uint8, POISON_U8)
    status, st_big = guarded(n, torch.int32, SENT_I32)
    ops.crop_resize(flat, hw, off, d_box, d_img, n, 64, out, status)
    torch.cuda.synchronize()
    check_guard(out_big, n * 64 * 64 * 3, POISON_U8, "crops")
    check_guard(st_big, n, SENT_I32, "status")
    return out.view(n, 64, 64, 3).cpu().numpy(), status.cpu().numpy(), hb[:n], hi[:n]


def check_crops(imgs, out, status, boxes, bimg):
    """the reference loop (ref:util/utils.py:97-103): int(c * size) truncation, slicing, cv2.resize to 64x64; empty crops
    (cv2.resize raises, the reference skips them) -> status 1 and a zeroed slot.  Boxes outside the image are clamped to
    it: the detector clamps its boxes to the image, so a negative ratio (where Python slicing would wrap) never arrives."""
    import cv2
    n_empty = 0
    for i in range(len(bimg)):
        img = imgs[bimg[i]]
        h, w = img.shape[:2]
        _, (xa, ya, xb, yb) = S.crop_geometry(boxes[i], w, h)
        if xb <= xa or yb <= ya:
            assert status[i] == 1, (i, boxes[i])
            assert not out[i].any(), f"crop {i}: the slot of an empty crop is not zeroed"
            n_empty += 1
            continue
        assert status[i] == 0, (i, boxes[i])
        ref = cv2.resize(np.ascontiguousarray(img[ya:yb, xa:xb]), (64, 64))
        if not np.array_equal(ref, out[i]):
            bad = np.argwhere(ref != out[i])
            raise AssertionError(f"crop {i} ({xb - xa}x{yb - ya} of image {bimg[i]}): {len(bad)} bytes differ, first at "
                                 f"{tuple(bad[0])}: got {out[i][tuple(bad[0])]}, expected {ref[tuple(bad[0])]}")
    return n_empty


def test_crop_resize_on_the_overlap_filter_crop_list():
    """production chain: the B = 8 overlap case's crop list, straight from the device buffers (crop_box [B*max_det, 4],
    crop_img), over the batch's screenshots laid out as parse_screenshots lays them out (hw [B, 2], off = i*H*W*3)"""
    case = S.OVL_CASES[0]
    got, d_box, d_img = ovl_run(case, 0.7)
    n = int(got["ccnt"][case.B])
    assert n > 1000
    imgs = [S.image(9000 + b, S.H, S.W, "noise" if b % 2 else "stripes") for b in range(case.B)]
    out, status, boxes, bimg = crop_run(imgs, d_box, d_img, n)
    assert check_crops(imgs, out, status, boxes, bimg) == 0


@pytest.mark.parametrize("case", S.CROP_CASES, ids=[c.name for c in S.CROP_CASES])
def test_crop_resize_branches(case):
    imgs = S.crop_images(case)
    boxes, bimg = S.crop_boxes(case)
    out, status, _, _ = crop_run(imgs, boxes, bimg)
    n_empty = check_crops(imgs, out, status, boxes, bimg)
    assert n_empty >= 5 * len(imgs)


# ------------------------------------------------------------------------------------------------ letterbox
@pytest.mark.parametrize("c", S.LB_CASES, ids=[c.name for c in S.LB_CASES])
def test_letterbox_bit_exact(c):
    imgs = S.lb_images(c)
    exp, (tw, th, scale, rw, rh, pl, pt) = S.lb_expected(c)
    B = c.B
    src = torch.from_numpy(imgs).to(DEV)
    tmp, tmp_big = guarded(B * c.h * rw * 3, torch.uint8, POISON_U8)
    canvas, cv_big = guarded(B * th * tw * 3, torch.uint8, POISON_U8)
    covers(src, B * c.h * c.w * 3, "src")
    assert 0 <= pl and pl + rw <= tw and 0 <= pt and pt + rh <= th
    ops.letterbox(src, B, c.h, c.w, rw, rh, tw, th, pl, pt, tmp, canvas)
    torch.cuda.synchronize()
    check_guard(cv_big, B * th * tw * 3, POISON_U8, "canvas")
    check_guard(tmp_big, B * c.h * rw * 3, POISON_U8, "tmp")
    got = canvas.view(B, th, tw, 3).cpu().numpy()
    pad = np.ones((th, tw), bool)
    pad[pt:pt + rh, pl:pl + rw] = False
    for b in range(B):
        assert (got[b][pad] == 114).all(), f"image {b}: pad bytes are not 114"
        if not np.array_equal(got[b], exp[b]):
            bad = np.argwhere(got[b] != exp[b])
            raise AssertionError(f"image {b}: {len(bad)} bytes differ from Pillow, first at {tuple(bad[0])}")
    if c.kind == "edges" and (rw, rh) != (c.w, c.h):
        assert S.lb_clipping(c) == (True, True), "the hard-edged content no longer clips at both 0 and 255"


def test_resize_u8_768_caption_mode():
    """the 768 caption mode's only resize: its crop batch (caption.BUCKET_768 = 16) of 64x64 crops -> 768x768 BICUBIC,
    saturated stripes (the bicubic lobes overshoot both ends)"""
    from PIL import Image
    from omniparser_b200.caption import BUCKET_768
    K, S_ = BUCKET_768, 768
    crops = np.stack([S.image(500 + k, 64, 64, "stripes" if k % 4 else "noise") for k in range(K)])
    src = torch.from_numpy(crops).to(DEV)
    tmp, tmp_big = guarded(K * 64 * S_ * 3, torch.uint8, POISON_U8)
    out, out_big = guarded(K * S_ * S_ * 3, torch.uint8, POISON_U8)
    covers(src, K * 64 * 64 * 3, "src")
    ops.resize_u8(src, K, 64, 64, S_, S_, 1, tmp, out)
    torch.cuda.synchronize()
    check_guard(out_big, K * S_ * S_ * 3, POISON_U8, "out")
    check_guard(tmp_big, K * 64 * S_ * 3, POISON_U8, "tmp")
    got = out.view(K, S_, S_, 3).cpu().numpy()
    for k in range(K):
        ref = np.asarray(Image.fromarray(crops[k]).resize((S_, S_), Image.Resampling.BICUBIC))
        assert np.array_equal(ref, got[k]), f"crop {k}"


def test_degenerate_resize_geometry_is_rejected_before_launch():
    """Pillow raises for an empty resize (641 x 1 at imgsz 640 -> 640 x 0); so do _geometry and the C entry points, and the
    C side refuses a resized image that does not lie inside the canvas.  Every buffer is large enough for the call as
    written, so nothing could run out of bounds even if a check were missing."""
    from omniparser_b200.detector import _geometry
    with pytest.raises(ValueError, match="height and width must be > 0"):
        _geometry(641, 1, 640)
    u8 = dict(dtype=torch.uint8, device=DEV)
    src = torch.zeros((1, 4, 641, 3), **u8)
    tmp = torch.zeros((1, 4, 641, 3), **u8)
    canvas = torch.zeros((1, 640, 641, 3), **u8)
    lb = lambda H, W, Wr, Hr, Tw, Th, pl, pt: ops.letterbox(src, 1, H, W, Wr, Hr, Tw, Th, pl, pt, tmp, canvas)  # noqa: E731
    _rejected(lambda: lb(1, 641, 640, 0, 640, 640, 0, 320), "sizes must be >= 1")
    _rejected(lambda: lb(4, 1, 0, 4, 640, 640, 320, 0), "sizes must be >= 1")
    _rejected(lambda: lb(4, 4, 8, 8, 16, 16, -1, 0), "inside the canvas")
    _rejected(lambda: lb(4, 4, 8, 8, 16, 16, 0, -1), "inside the canvas")
    _rejected(lambda: lb(4, 4, 8, 8, 16, 16, 9, 0), "inside the canvas")
    _rejected(lambda: lb(4, 4, 8, 8, 16, 16, 0, 9), "inside the canvas")
    rs = lambda H, W, Wr, Hr: ops.resize_u8(src, 1, H, W, Wr, Hr, 1, tmp, canvas)  # noqa: E731
    _rejected(lambda: rs(4, 4, 0, 8), "sizes must be >= 1")
    _rejected(lambda: rs(4, 4, 8, 0), "sizes must be >= 1")
    _rejected(lambda: rs(0, 4, 8, 8), "sizes must be >= 1")
    # the same calls at the edge of what is allowed still run and are exact
    lb(4, 4, 8, 8, 16, 16, 8, 8)
    torch.cuda.synchronize()
    exp = np.full((16, 16, 3), 114, np.uint8)
    exp[8:, 8:] = R.resize_lanczos_numpy(np.zeros((4, 4, 3), np.uint8), 8, 8)
    assert np.array_equal(canvas.view(-1)[:16 * 16 * 3].view(16, 16, 3).cpu().numpy(), exp)
