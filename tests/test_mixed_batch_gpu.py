"""GPU: screenshots of different sizes in one batch.

* `b2p_letterbox_batch` byte for byte against Pillow and against `b2p_letterbox` run image by image, on every imgsz=640
  letterbox case of tests/screen_cases.py in one ragged batch (plus a 640x480 image that skips both passes), on a tuple
  canvas, and on hard-edged content that clips at 0 and 255;
* the detector and the parse path at a FIXED batch size: row i of a mixed batch equals row i of a batch of B copies of image
  i (every GEMM row and every decode / NMS CTA depends only on its own image, so this is exact; a different B changes the
  GEMM plans and the last bits);
* the reference goldens in one mixed batch, and the pipelined parser over interleaved mixed / same-size batches."""
import gc
import json
from pathlib import Path

import numpy as np
import pytest
import torch

import screen_cases as S
import __graft_entry__ as ge
from omniparser_b200 import ops, synth
from omniparser_b200.detector import B200YOLOv9Detector
from omniparser_b200.utils import PipelinedParser, _prompt_ids, parse_screenshots
from oracle import ref_restate as R
from test_boundary_gpu import _same_elements as _tie_class_same, artefacts, loaded  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
GOLD = Path(__file__).resolve().parent / "golden"
POISON = 0xA5
GUARD = 4096


@pytest.fixture(scope="module", autouse=True)
def _release_what_this_module_added():
    """The stand-in models are shared by the whole session, and later tests run the benchmark workload near the card's
    memory: drop the io slots, detector plans and caption plans this module added to them, and the handles it made."""
    det, cmp_ = ge.standin_models(DEV)
    before = [(d, set(d)) for d in (det._io, det._plans, cmp_["model"]._plans)]
    yield
    torch.cuda.synchronize()
    for d, keys in before:
        for k in [k for k in d if k not in keys]:
            del d[k]
    gc.collect()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ letterbox
def _lb_batch(imgs, imgsz):
    """ragged letterbox of imgs -> (canvases [B, th, tw, 3], plan); guard bytes after tmp and canvas must stay untouched"""
    geom = [R.letterbox_geometry(im.shape[1], im.shape[0], imgsz) for im in imgs]
    tw, th = geom[0][:2]
    desc, tables, tmp_b, src_b = ops.letterbox_batch_plan([(im.shape[0], im.shape[1], g[3], g[4], g[5], g[6])
                                                           for im, g in zip(imgs, geom)], tw, th)
    B = len(imgs)
    src = torch.from_numpy(np.concatenate([im.reshape(-1) for im in imgs])).to(DEV)
    assert src.numel() == src_b
    tmp = torch.full((tmp_b + GUARD,), POISON, dtype=torch.uint8, device=DEV)
    canvas = torch.full((B * th * tw * 3 + GUARD,), POISON, dtype=torch.uint8, device=DEV)
    d_desc = torch.from_numpy(desc).to(DEV)
    d_tab = torch.from_numpy(tables if tables.size else np.zeros(1, np.int32)).to(DEV)
    ops.letterbox_batch(src, B, desc, d_desc, d_tab, tw, th, tmp, canvas)
    torch.cuda.synchronize()
    assert bool((tmp[tmp_b:] == POISON).all()) and bool((canvas[B * th * tw * 3:] == POISON).all()), "guard bytes written"
    return canvas[:B * th * tw * 3].view(B, th, tw, 3).cpu().numpy(), desc


def _per_image_letterbox(im, imgsz):
    tw, th, _, rw, rh, pl, pt = R.letterbox_geometry(im.shape[1], im.shape[0], imgsz)
    src = torch.from_numpy(np.ascontiguousarray(im)).to(DEV)
    tmp = torch.empty((im.shape[0] * rw * 3,), dtype=torch.uint8, device=DEV)
    canvas = torch.empty((th, tw, 3), dtype=torch.uint8, device=DEV)
    ops.letterbox(src, 1, im.shape[0], im.shape[1], rw, rh, tw, th, pl, pt, tmp, canvas)
    return canvas.cpu().numpy()


def _check_letterbox(imgs, imgsz, pil=None):
    got, desc = _lb_batch(imgs, imgsz)
    for b, im in enumerate(imgs):
        exp = pil[b] if pil is not None else R.letterbox_pil(im, imgsz)[0]
        assert np.array_equal(got[b], exp), f"image {b} ({im.shape[1]}x{im.shape[0]}): {int((got[b] != exp).sum())} bytes differ from Pillow"
        assert np.array_equal(got[b], _per_image_letterbox(im, imgsz)), f"image {b}: differs from b2p_letterbox"
    return desc


def test_letterbox_batch_every_640_case():
    cases = [c for c in S.LB_CASES if c.imgsz == 640]
    imgs, pil = [], []
    for c in cases:
        imgs += list(S.lb_images(c))
        pil += list(S.lb_expected(c)[0])
    imgs.append(S.image(99, 480, 640, "edges"))          # 640x480: both passes skipped, pasted at pad_t 80
    pil.append(R.letterbox_pil(imgs[-1], 640)[0])
    desc = _check_letterbox(imgs, 640, pil)
    assert desc[-1, 8] == -1 and desc[-1, 10] == -1
    clipping = [S.lb_clipping(c) for c in cases if c.kind == "edges" and (c.w, c.h) != (640, 640)]
    assert any(lo for lo, _ in clipping) and any(hi for _, hi in clipping), "no image of the batch clips at 0 and at 255"


def test_letterbox_batch_tuple_canvas():
    """imgsz=(768, 1366): 1366x768 skips both passes (1376-wide canvas), 1920x1080 and 1280x720 resample"""
    imgs = [S.image(31, 768, 1366, "edges"), S.image(32, 1080, 1920, "edges"), S.image(33, 720, 1280, "noise")]
    desc = _check_letterbox(imgs, (768, 1366))
    assert desc[0, 8] == -1 and desc[0, 10] == -1 and desc[1, 8] >= 0 and desc[2, 10] >= 0


def test_letterbox_batch_refuses_a_descriptor_that_disagrees():
    imgs = [S.image(1, 100, 200, "noise"), S.image(2, 300, 100, "noise")]
    desc, tables, tmp_b, _ = ops.letterbox_batch_plan([(100, 200, 640, 320, 0, 160), (300, 100, 213, 640, 213, 0)], 640, 640)
    bad = desc.copy()
    bad[0, 8] = -1                                       # horizontal table missing although Wr != W
    src = torch.from_numpy(np.concatenate([im.reshape(-1) for im in imgs])).to(DEV)
    canvas = torch.empty((2, 640, 640, 3), dtype=torch.uint8, device=DEV)
    n0 = ops._lib.launch_count()
    with pytest.raises(ops._lib.B2PError, match="disagree"):
        ops.letterbox_batch(src, 2, bad, torch.from_numpy(bad).to(DEV), torch.from_numpy(tables).to(DEV), 640, 640,
                            torch.empty((tmp_b,), dtype=torch.uint8, device=DEV), canvas)
    assert ops._lib.launch_count() == n0


# ------------------------------------------------------------------------------------------------ detector
MIXED6 = [(1920, 1080), (1280, 800), (1170, 2532), (1366, 768), (2560, 1440), (640, 480)]


@pytest.mark.parametrize("precision", ["fp16", "fp16x3"])
def test_predict_batch_mixed_equals_replicas(precision):
    from standin.yolo_weights import yolo_standin
    det = B200YOLOv9Detector(state_dict=yolo_standin(0).state_dict(), device=DEV, precision=precision)
    imgs = [synth.screenshot(40 + i, w, h) for i, (w, h) in enumerate(MIXED6)]
    got = det.predict_batch(imgs, conf=0.05)
    total = 0
    for i, im in enumerate(imgs):
        ref = det.predict_batch([im] * len(imgs), conf=0.05)[i].boxes
        g = got[i].boxes
        assert g.xyxy.shape == ref.xyxy.shape, (i, g.xyxy.shape, ref.xyxy.shape)
        assert torch.equal(g.xyxy, ref.xyxy) and torch.equal(g.conf, ref.conf), f"image {i}: boxes / scores differ"
        total += g.xyxy.shape[0]
    assert total > 0
    del det, got, ref, g
    gc.collect()


# ------------------------------------------------------------------------------------------------ parse
def _same(a, b):
    (ea, ia), (eb, ib) = a, b
    assert ea == eb
    assert torch.equal(ia, ib)


def test_parse_screenshots_mixed_equals_replicas():
    det, cmp_ = ge.standin_models(DEV)
    shots = [(50, 1920, 1080), (51, 1280, 800), (52, 1366, 768), (53, 1170, 2532)]
    imgs = [synth.screenshot(s, w, h) for s, w, h in shots]
    ocr = [synth.ocr_boxes(s, w, h) for s, w, h in shots]
    kw = dict(BOX_TRESHOLD=0.05, iou_threshold=0.7, max_new_tokens=8)
    got = parse_screenshots(imgs, det, cmp_, ocr, **kw)
    assert sum(ids.shape[0] for _, ids in got) > 0
    for i in range(len(imgs)):
        _same(got[i], parse_screenshots([imgs[i]] * len(imgs), det, cmp_, [ocr[i]] * len(imgs), **kw)[i])


def test_parse_screenshots_mixed_768_captions_and_host_glue(monkeypatch):
    """caption_size=768 and the host list logic (B2P_HOST_GLUE) on a mixed batch, detector output injected"""
    import omniparser_b200.utils as U
    det, cmp_ = ge.standin_models(DEV)
    shots = [(60, 1280, 800), (61, 900, 1600)]
    imgs = [synth.screenshot(s, w, h) for s, w, h in shots]
    ocr = [synth.ocr_boxes(s, w, h) for s, w, h in shots]
    boxes = [[[10.0, 10.0, 90.0, 70.0], [300.0, 200.0, 420.0, 330.0]], [[50.0, 900.0, 200.0, 1000.0]]]
    kw = dict(BOX_TRESHOLD=0.05, iou_threshold=0.7, max_new_tokens=6, caption_size=768)
    got = parse_screenshots(imgs, det, cmp_, ocr, _det_override=boxes, **kw)
    for i in range(2):
        _same(got[i], parse_screenshots([imgs[i]] * 2, det, cmp_, [ocr[i]] * 2, _det_override=[boxes[i]] * 2, **kw)[i])
    monkeypatch.setattr(U, "_HOST_GLUE", True)
    kw.pop("caption_size")
    got = parse_screenshots(imgs, det, cmp_, ocr, **kw)
    for i in range(2):
        _same(got[i], parse_screenshots([imgs[i]] * 2, det, cmp_, [ocr[i]] * 2, **kw)[i])


def test_skip_h2d_refuses_a_mixed_batch():
    det, cmp_ = ge.standin_models(DEV)
    imgs = [synth.screenshot(0, 640, 480), synth.screenshot(1, 800, 600)]
    with pytest.raises(ValueError, match="one size"):
        parse_screenshots(imgs, det, cmp_, [([], [])] * 2, _skip_h2d=True)


def test_synthetic_goldens_in_one_mixed_batch():
    det, cmp_ = ge.standin_models(DEV)
    gs = [json.loads((GOLD / f"{n}.json").read_text()) for n in ("synth_seed0", "synth_seed3_odd", "synth_seed5_3240x2160")]
    assert len({tuple(g["case"]["size"]) for g in gs}) == 3
    assert len({(g["box_threshold"], g["iou_threshold"], g["max_new_tokens"]) for g in gs}) == 1
    imgs = [synth.screenshot(g["case"]["seed"], *g["case"]["size"]) for g in gs]
    ocr = [synth.ocr_boxes(g["case"]["seed"], *g["case"]["size"]) for g in gs]
    g0 = gs[0]
    out = parse_screenshots(imgs, det, cmp_, ocr, BOX_TRESHOLD=g0["box_threshold"], iou_threshold=g0["iou_threshold"],
                            max_new_tokens=g0["max_new_tokens"], _det_override=[g["det_xyxy"] for g in gs])
    for (elems, ids), g in zip(out, gs):
        assert len(elems) == len(g["parsed_content_list"])
        for a, b in zip(elems, g["parsed_content_list"]):
            assert a["type"] == b["type"] and a["source"] == b["source"] and a["bbox"] == b["bbox"]
            assert a["content"].strip() == b["content"].strip()
        assert ids.tolist() == g["caption_ids"]


def test_real_goldens_in_one_mixed_batch(loaded):
    """the reference repo's four screenshots (3240x2160, 1919x1079 RGBA, 1280x90, 1024x768) in ONE batch through the
    parity-grade detector with the eval call site's parameters: each reproduces its golden under the tie-class rules of
    tests/parity_util.py (the batch size differs from the golden's B = 1, which moves the last bits)"""
    from PIL import Image
    det, cmp_ = loaded
    gs = [json.loads((GOLD / f"{n}.json").read_text()) for n in ("real_demo_image", "real_omni3", "real_excel_rgba", "real_header_bar_thin")]
    assert len({(g["box_threshold"], g["iou_threshold"]) for g in gs}) == 1
    imgs = [np.asarray(Image.open(GOLD / "imgs" / g["case"]["file"]).convert("RGB")) for g in gs]
    assert len({im.shape for im in imgs}) == 4
    ocr = [(list(g["ocr_text"]), g["ocr_bbox"] or None) for g in gs]
    out = parse_screenshots(imgs, det, cmp_, ocr, gs[0]["box_threshold"], gs[0]["iou_threshold"], 640,
                            prompt_ids=_prompt_ids(None, cmp_))
    for (elems, _), g, im in zip(out, gs, imgs):
        ev = _tie_class_same(elems, g["parsed_content_list"], (im.shape[1], im.shape[0]), golden=g)
        print(f"{g['case']['file']}: {len(elems)} elements, {ev} integer-boundary / order events")


# ------------------------------------------------------------------------------------------------ pipeline
def _stream_of_batches():
    """mixed and same-size batches interleaved.  Batches 0-5 are mixed, so whichever io slot batch 8 lands in (the parser
    rotates through lanes * group + group + 1 slots: 3, 4, 5 or 7 here) already holds a smaller mixed batch, and batch 8
    (a 4K screenshot among others) has to grow it."""
    sizes = [
        [(1920, 1080), (1280, 800), (1366, 768), (1170, 2532)],
        [(1280, 800), (800, 600), (1280, 800), (1024, 768)],
        [(1366, 768), (1920, 1080), (1280, 800), (800, 600)],
        [(1024, 768), (1280, 800), (1920, 1080), (1366, 768)],
        [(800, 600), (640, 480), (1280, 720), (1024, 768)],
        [(1280, 720), (1366, 768), (640, 480), (1920, 1080)],
        [(1280, 800)] * 4,
        [(1920, 1080)] * 4,
        [(3840, 2160), (2560, 1440), (1170, 2532), (1920, 1080)],
        [(1366, 768)] * 4,
        [(800, 600), (1920, 1080), (1280, 720), (1024, 768)],
    ]
    out = []
    for b, group in enumerate(sizes):
        seeds = [100 + 10 * b + i for i in range(len(group))]
        out.append(([synth.screenshot(s, w, h) for s, (w, h) in zip(seeds, group)],
                    [synth.ocr_boxes(s, w, h) for s, (w, h) in zip(seeds, group)]))
    return out


@pytest.mark.parametrize("lanes,group", [(1, 1), (2, 1), (1, 2), (2, 2)])
def test_pipelined_parser_mixed_stream_equals_parse_screenshots(lanes, group, monkeypatch):
    """run twice; the first run grows an io slot (with the pipeline drained), the reference runs between the two"""
    from standin.yolo_weights import yolo_standin
    _, cmp_ = ge.standin_models(DEV)
    det = B200YOLOv9Detector(state_dict=yolo_standin(0).state_dict(), device=DEV)   # fresh io slots
    grown, reserve = [], B200YOLOv9Detector.reserve_mixed

    def spy(self, io_, mb):
        if self.mixed_grow_needed(io_, mb):
            grown.append(mb["need"])
        reserve(self, io_, mb)
    monkeypatch.setattr(B200YOLOv9Detector, "reserve_mixed", spy)
    batches = _stream_of_batches()
    kw = dict(BOX_TRESHOLD=0.05, iou_threshold=0.7, max_new_tokens=8)
    pp = PipelinedParser(det, cmp_, caption_lanes=lanes, caption_group=group, **kw)
    runs = [list(pp.run(iter(batches)))]
    assert grown, "no io slot grew"
    ref = [parse_screenshots(imgs, det, cmp_, ocr, **kw) for imgs, ocr in batches]
    runs.append(list(pp.run(iter(batches))))
    for got in runs:
        assert len(got) == len(ref)
        for out, exp in zip(got, ref):
            assert len(out) == len(exp)
            for a, b in zip(out, exp):
                _same(a, b)
    del pp, det, runs, ref
    gc.collect()
