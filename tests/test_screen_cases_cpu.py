"""CPU half of tests/test_screen_kernels_gpu.py: on exactly the GPU module's cases,

* the restatements used as oracles agree with their libraries (`resize_bilinear_cv2_numpy` with `cv2.resize`,
  `letterbox_numpy` with Pillow, `overlap_flags_loops` + `elements_from_flags` with `host_glue.build_elements`), so a
  GPU mismatch there is a kernel bug;
* the cases reach every branch of the three kernels (coverage computed from the case definitions: removing a case that
  is the only one to reach a branch fails here);
* a resize to an empty image is rejected on the host, as Pillow rejects it, and the device overlap filter hands
  screenshots with more OCR boxes than it takes to the host list logic."""
from __future__ import annotations

import numpy as np
import pytest

import screen_cases as S
from omniparser_b200 import host_glue
from oracle import ref_restate as R

OVL_PARAMS = [(c, thr) for c in S.OVL_CASES for thr in c.thrs]


# ------------------------------------------------------------------------------------------------ oracles
@pytest.mark.parametrize("case,thr", OVL_PARAMS, ids=[f"{c.name}-thr{t}" for c, t in OVL_PARAMS])
def test_overlap_flags_oracle_equals_build_elements(case, thr):
    for b, (inp, (st, mk, rm), (elems, _)) in enumerate(zip(S.ovl_inputs(case), S.ovl_flags(case, thr),
                                                            S.ovl_elements(case, thr))):
        assert host_glue.elements_from_flags(inp[3], st, mk, inp[5], rm) == elems, f"screenshot {b}"


def _chain_crops():
    case = S.OVL_CASES[0]
    boxes, bimg = S.ovl_crop_list(case, 0.7)
    return [S.image(9000 + b, S.H, S.W, "noise" if b % 2 else "stripes") for b in range(case.B)], boxes, bimg


@pytest.mark.parametrize("which", [c.name for c in S.CROP_CASES] + ["overlap_chain"])
def test_bilinear_oracle_equals_cv2(which):
    import cv2
    if which == "overlap_chain":
        imgs, boxes, bimg = _chain_crops()
    else:
        case = next(c for c in S.CROP_CASES if c.name == which)
        imgs = S.crop_images(case)
        boxes, bimg = S.crop_boxes(case)
    for i, (box, q) in enumerate(zip(boxes, bimg)):
        h, w = imgs[q].shape[:2]
        _, (xa, ya, xb, yb) = S.crop_geometry(box, w, h)
        crop = np.ascontiguousarray(imgs[q][ya:yb, xa:xb])
        if xb <= xa or yb <= ya:
            with pytest.raises(cv2.error):
                cv2.resize(crop, (64, 64))
            continue
        assert np.array_equal(R.resize_bilinear_cv2_numpy(crop), cv2.resize(crop, (64, 64))), (i, crop.shape)


@pytest.mark.parametrize("c", S.LB_CASES, ids=[c.name for c in S.LB_CASES])
def test_letterbox_oracle_equals_pillow(c):
    exp, _ = S.lb_expected(c)
    imgs = S.lb_images(c)
    for b in range(c.B):
        assert np.array_equal(R.letterbox_numpy(imgs[b], c.imgsz)[0], exp[b]), f"image {b}"


# ------------------------------------------------------------------------------------------------ coverage
def test_overlap_cases_reach_every_branch():
    seen = set()
    for case in S.OVL_CASES:
        if case.max_det == S.KERNEL_LIMIT and case.max_ocr == S.KERNEL_LIMIT and max(case.counts) >= S.KERNEL_LIMIT \
                and max(case.ocr) >= S.KERNEL_LIMIT:
            seen.add("limits_512")
        if any(n > case.max_det for n in case.counts):
            seen.add("count_gt_max_det")
        if case.max_det == S.MAX_DET and 0 in case.counts and S.MAX_DET in case.counts:
            seen.add("0_and_300_icons")
        if S.MAX_DET == case.max_det and case.B >= 8 and {0.7, 0.9} <= set(case.thrs):
            seen.add("large_batch_thr_0.7_0.9_b%d" % case.B)
        for thr in case.thrs:
            crops = sum(len(e[1]) for e in S.ovl_elements(case, thr))
            if crops > S.CHUNK * (case.B - 1):
                seen.add("batch_compaction_second_chunk")
            for inp, (st, mk, rm) in zip(S.ovl_inputs(case), S.ovl_flags(case, thr)):
                n, m = len(inp[3]), len(inp[4])
                live = [(int(b[2] * S.W) - int(b[0] * S.W)) * (int(b[3] * S.H) - int(b[1] * S.H)) > 0 for b in inp[3]]
                if n > S.CHUNK:
                    seen.add("nraw_gt_256")
                    if sum(st[S.CHUNK:]) and any(st[i] == 1 for i in range(S.CHUNK, n)):
                        seen.add("second_chunk_icons_need_captions")
                    if not all(live[S.CHUNK - 8:S.CHUNK]) and not all(live[S.CHUNK:S.CHUNK + 8]):
                        seen.add("zero_area_both_sides_of_256")
                if m > 32:
                    seen.add("m_gt_32")
                if m == S.MAX_OCR:
                    seen.add("m_eq_256")
                if any(all(w != 0 for w in row[:8]) for row in mk):
                    seen.add("label_mask_8_words")
                if any(sum(w != 0 for w in row) >= 3 for row in mk):
                    seen.add("label_mask_3plus_words")
                if len({tuple(b) for b in inp[3]}) < n:
                    seen.add("duplicate_icons")
                if len({(tuple(e["bbox"]), e["content"]) for e in inp[5]}) < m and any(rm):
                    seen.add("equal_ocr_dicts")
                if thr == 0.1:
                    seen.add("thr_0.1")
                for i in range(n):
                    if st[i] == 0 and any(mk[i]):          # valid, labelled, then dropped
                        k = S.drop_index(inp[3][i], inp[4])
                        seen.add(f"drop_after_labels_k%32=={k % 32}")
                        if k == 255:
                            seen.add("drop_at_255")
    need = {"limits_512", "count_gt_max_det", "0_and_300_icons", "large_batch_thr_0.7_0.9_b8", "large_batch_thr_0.7_0.9_b16",
            "batch_compaction_second_chunk", "nraw_gt_256", "second_chunk_icons_need_captions", "zero_area_both_sides_of_256",
            "m_gt_32", "m_eq_256", "label_mask_8_words", "label_mask_3plus_words", "duplicate_icons", "equal_ocr_dicts",
            "thr_0.1", "drop_after_labels_k%32==31", "drop_after_labels_k%32==0", "drop_at_255"}
    assert need <= seen, sorted(need - seen)


def test_overlap_cases_have_nested_chains():
    """nested chains: only the innermost box of a chain survives the icon-vs-icon test at thr 0.7"""
    case = S.OVL_CASES[0]
    px = S.ovl_inputs(case)[0][0]
    st = S.ovl_flags(case, 0.7)[0][0]
    idx = [int(np.flatnonzero((px.numpy() == np.float32(b)).all(1))[0]) for b in S.NESTED]
    assert [st[i] for i in idx[:-1]] == [0] * (len(idx) - 1) and st[idx[-1]] != 0


def test_crop_cases_reach_every_branch():
    seen = set()
    for case in S.CROP_CASES:
        boxes, bimg = S.crop_boxes(case)
        for box, q in zip(boxes, bimg):
            h, w = case.sizes[q]
            raw, (xa, ya, xb, yb) = S.crop_geometry(box, w, h)
            seen |= S.crop_branches(xb - xa, yb - ya)
            if tuple(raw) != (xa, ya, xb, yb) and xb > xa and yb > ya:
                seen.add("edge_clamped")
            if (xa, ya, xb, yb) == (0, 0, w, h):
                seen.add(f"full_screen_{w}x{h}")
            if xb == w and yb == h and q == len(case.sizes) - 1 and xb > xa and yb > ya:
                seen.add("last_row_of_last_image")
        if len(set(case.sizes)) > 1:
            seen.add("mixed_image_sizes")
    imgs, boxes, bimg = _chain_crops()
    assert len(bimg) > 1000
    need = {"empty", "area", "x_snap_low", "x_snap_high", "y_clamp", "sw1", "sh1", "edge_clamped", "full_screen_1920x1080",
            "full_screen_3840x2160", "last_row_of_last_image", "mixed_image_sizes"}
    assert need <= seen, sorted(need - seen)


def test_letterbox_cases_reach_every_branch():
    seen = set()
    for c in S.LB_CASES:
        tw, th, scale, rw, rh, pl, pt = R.letterbox_geometry(c.w, c.h, c.imgsz)
        h_pass, v_pass = rw != c.w, rh != c.h
        seen.add({(True, False): "h_only", (False, True): "v_only", (True, True): "both", (False, False): "none"}[(h_pass, v_pass)])
        if rw > c.w or rh > c.h:
            seen.add("upscale")
        if (h_pass and S.lb_ksize(c.w, rw) > 31) or (v_pass and S.lb_ksize(c.h, rh) > 31):
            seen.add("ksize_gt_31")
        if not isinstance(c.imgsz, int):
            seen.add("tuple_imgsz")
        if c.B == 8 and (c.w, c.h) == (1920, 1080):
            seen.add("bench_batch")
        if c.kind == "edges" and (h_pass or v_pass):
            lo, hi = S.lb_clipping(c)
            seen |= {"clip_0"} if lo else set()
            seen |= {"clip_255"} if hi else set()
    need = {"h_only", "v_only", "both", "none", "upscale", "ksize_gt_31", "tuple_imgsz", "bench_batch", "clip_0", "clip_255"}
    assert need <= seen, sorted(need - seen)


# ------------------------------------------------------------------------------------------------ host-side rejections
@pytest.mark.parametrize("w,h,imgsz", [(641, 1, 640), (1, 641, 640), (4000, 3, 640), (2, 5000, (640, 640))])
def test_geometry_rejects_an_empty_resize_like_pillow(w, h, imgsz):
    from PIL import Image
    from omniparser_b200.detector import _geometry
    _, _, _, rw, rh, _, _ = R.letterbox_geometry(w, h, imgsz)
    assert rw < 1 or rh < 1
    with pytest.raises(ValueError, match="height and width must be > 0"):
        Image.new("RGB", (w, h)).resize((rw, rh), Image.Resampling.LANCZOS)
    with pytest.raises(ValueError, match="height and width must be > 0"):
        _geometry(w, h, imgsz)


def test_detector_io_rejects_an_empty_resize_before_allocating():
    from omniparser_b200.detector import B200YOLOv9Detector
    det = object.__new__(B200YOLOv9Detector)   # no device or weights: nothing past the geometry check may run
    det._io, det._plans = {}, {}
    with pytest.raises(ValueError, match="height and width must be > 0"):
        det._get_io(1, 1, 641, 640, 300)
    assert det._io == {} and det._plans == {}


def test_geometry_accepts_one_pixel_results():
    from omniparser_b200.detector import _geometry
    for w, h in [(640, 1), (1, 640), (1280, 2), (4000, 60)]:
        assert _geometry(w, h, 640) == R.letterbox_geometry(w, h, 640)


def test_filter_device_leaves_more_ocr_boxes_than_it_takes_to_the_host():
    """the device filter takes up to 256 OCR boxes per screenshot (detector.OCR_CAP = host_glue.OCR_DEVICE_CAP);
    filter_device returns False, launching nothing, as soon as one screenshot of the batch has more"""
    from omniparser_b200.detector import B200YOLOv9Detector
    assert B200YOLOv9Detector.OCR_CAP == host_glue.OCR_DEVICE_CAP == S.MAX_OCR
    io = {"max_ocr": S.MAX_OCR}   # nothing else: any use of a device buffer would raise
    assert B200YOLOv9Detector.filter_device(None, io, [[{}] * 3, [{}] * (S.MAX_OCR + 1)], 0.7) is False
