"""GPU: the device PNG encoder (csrc/png_encode.cu via som_overlay.DevicePngEncoder).  Every PNG is taken apart chunk by
chunk (signature, IHDR fields, one IDAT, IEND last, every CRC by zlib.crc32, the zlib header check bits), inflated by zlib
(which checks the Adler-32), un-filtered and compared with the frame byte for byte; PIL must decode the same pixels.  Frames:
the overlays of the golden images at their draw configs, synth screenshots up to 3240 x 2160, and edge frames (1 x 1, one
row, one column, one band, many bands, uniform, noise, period 3, rows repeating only beyond the 32 KiB window).  Also: the
size against the host encoder, determinism, concurrent callers, and the device path of get_som_labeled_img and the server."""
import base64
import io
import json
import struct
import threading
import zlib
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu

import __graft_entry__ as ge  # noqa: E402
from omniparser_b200 import ops, som_overlay as SO, synth  # noqa: E402

GOLD = Path(__file__).resolve().parent / "golden"
DEV = torch.device("cuda", 0)
SIZE_BOUND = 1.25     # device PNG bytes / host encode_png bytes on the overlays


def check_png(png: bytes, frame: np.ndarray):
    h, w, _ = frame.shape
    assert png[:8] == b"\x89PNG\r\n\x1a\n"
    pos, chunks = 8, []
    while pos < len(png):
        n, = struct.unpack(">I", png[pos:pos + 4])
        tag, data = png[pos + 4:pos + 8], png[pos + 8:pos + 8 + n]
        crc, = struct.unpack(">I", png[pos + 8 + n:pos + 12 + n])
        assert len(data) == n and zlib.crc32(tag + data) & 0xFFFFFFFF == crc, tag
        chunks.append((tag, data))
        pos += 12 + n
    assert pos == len(png)                                           # no trailing bytes
    assert [t for t, _ in chunks] == [b"IHDR", b"IDAT", b"IEND"] and chunks[2][1] == b""
    assert struct.unpack(">IIBBBBB", chunks[0][1]) == (w, h, 8, 2, 0, 0, 0)
    idat = chunks[1][1]
    assert idat[0] & 15 == 8 and (idat[0] << 8 | idat[1]) % 31 == 0   # deflate, check bits
    raw = np.frombuffer(zlib.decompress(idat), np.uint8)             # checks the Adler-32
    rows = raw.reshape(h, 1 + 3 * w)
    assert (rows[:, 0] == 2).all()                                  # Up on every row
    back = np.cumsum(rows[:, 1:], axis=0, dtype=np.uint8).reshape(h, w, 3)
    assert np.array_equal(back, frame)
    pil = Image.open(io.BytesIO(png))
    pil.load()
    assert pil.mode == "RGB" and np.array_equal(np.asarray(pil), frame)


def _enc():
    return SO.device_encoder(DEV)


def _golden_frames():
    out = []
    for name in ["real_demo_image", "real_excel_rgba", "real_omni3", "real_header_bar_thin"]:
        g = json.loads((GOLD / f"{name}.json").read_text())
        img = np.asarray(Image.open(GOLD / "imgs" / g["case"]["file"]).convert("RGB"))
        _, _, frame = SO.som_outputs(img, [e["bbox"] for e in g["parsed_content_list"]], True, **g["draw_bbox_config"])
        out.append((name, frame))
    for name in ["synth_seed0", "synth_seed3_odd", "synth_seed5_3240x2160"]:
        g = json.loads((GOLD / f"{name}.json").read_text())
        w, h = g["case"]["size"]
        img = synth.screenshot(g["case"]["seed"], w, h)
        _, _, frame = SO.som_outputs(img, [e["bbox"] for e in g["parsed_content_list"]], True)
        out.append((name, frame))
    return out


@pytest.fixture(scope="module")
def golden_frames():
    return _golden_frames()


def test_overlays_round_trip_and_size(golden_frames):
    sizes = {(f.shape[1], f.shape[0]) for _, f in golden_frames}
    assert {(1920, 1080), (1919, 1079), (3240, 2160)} <= sizes
    for name, frame in golden_frames:
        png = _enc().encode(frame)
        check_png(png, frame)
        host = SO.encode_png(frame)
        ratio = len(png) / len(host)
        print(f"{name} {frame.shape[1]}x{frame.shape[0]}: device {len(png)} B, host {len(host)} B, ratio {ratio:.3f}")
        assert ratio <= SIZE_BOUND, (name, ratio)
        assert len(png) <= ops.png_plan(*frame.shape[:2])[2]


def _edge_frames():
    rng = np.random.default_rng(11)
    y, x = np.mgrid[0:300, 0:700]
    period3 = (((x + y) % 3) * 80).astype(np.uint8)[..., None].repeat(3, 2)
    far_rows = rng.integers(0, 256, (2, 12000, 3), dtype=np.uint8)[np.arange(6) % 2]   # pitch 36001 > 32 KiB window
    return {
        "1x1": np.array([[[7, 200, 13]]], np.uint8),
        "1xW": rng.integers(0, 256, (1, 1920, 3), dtype=np.uint8),
        "Hx1": rng.integers(0, 4, (1080, 1, 3), dtype=np.uint8),
        "one_band": (rng.integers(0, 3, (5, 1920, 3)) * 100).astype(np.uint8),
        "many_bands": (rng.integers(0, 2, (6000, 64, 3)) * 255).astype(np.uint8),
        "uniform": np.full((1080, 1920, 3), 37, np.uint8),
        "noise": rng.integers(0, 256, (1080, 1920, 3), dtype=np.uint8),
        "period3": period3,
        "far_rows": far_rows,
    }


@pytest.mark.parametrize("name", list(_edge_frames()))
def test_edge_frames(name):
    frame = _edge_frames()[name]
    png = _enc().encode(frame)
    check_png(png, frame)
    bands, _, worst = ops.png_plan(*frame.shape[:2])
    assert len(png) <= worst
    if name == "one_band":
        assert bands == 1
    if name == "many_bands":
        assert bands > 20
    if name == "uniform":   # maximal matches: far below one byte per 258 filtered bytes, plus per-band headers
        assert len(png) < frame.size // 100
    print(f"{name}: {len(png)} B, {bands} bands, worst case {worst} B")


def test_deterministic_and_concurrent(golden_frames):
    frames = [f for _, f in golden_frames[:4]]
    first = [_enc().encode(f) for f in frames]
    assert [_enc().encode(f) for f in frames] == first
    got = [None] * len(frames)

    def run(i):
        got[i] = _enc().encode(frames[i])

    th = [threading.Thread(target=run, args=(i,)) for i in range(len(frames))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for png, frame, ref in zip(got, frames, first):
        check_png(png, frame)
        assert png == ref


def test_get_som_labeled_img_and_server_use_device_encoder():
    from omniparser_b200.server import BatchingOmniparser
    from omniparser_b200.utils import get_som_labeled_img
    det, cmp_ = ge.standin_models(DEV)
    img = synth.screenshot(0)
    texts, boxes = synth.ocr_boxes(0)
    enc, _, elems = get_som_labeled_img(Image.fromarray(img), det, BOX_TRESHOLD=0.05, output_coord_in_ratio=True,
                                        ocr_bbox=boxes, caption_model_processor=cmp_, ocr_text=texts, iou_threshold=0.7)
    host_b64, _, frame = SO.som_outputs(img, [e["bbox"] for e in elems], True)
    png = base64.b64decode(enc)
    assert png == _enc().encode(frame)
    check_png(png, frame)
    assert np.array_equal(np.asarray(Image.open(io.BytesIO(base64.b64decode(host_b64))).convert("RGB")), frame)

    def ocr_fn(image, **k):
        return (list(texts), list(boxes)), None

    srv = BatchingOmniparser({"BOX_TRESHOLD": 0.05, "ocr_fn": ocr_fn, "max_batch": 2, "max_wait_ms": 1.0}, models=(det, cmp_))
    try:
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format="PNG")
        enc2, elems2 = srv.parse(base64.b64encode(buf.getvalue()).decode("ascii"))
    finally:
        srv.close()
    r = max(img.shape[1], img.shape[0]) / 3200
    cfg = {"text_scale": 0.8 * r, "text_thickness": max(int(2 * r), 1), "text_padding": max(int(3 * r), 1),
           "thickness": max(int(3 * r), 1)}
    _, _, frame2 = SO.som_outputs(img, [e["bbox"] for e in elems2], True, **cfg)
    png2 = base64.b64decode(enc2)
    assert png2 == _enc().encode(frame2)
    check_png(png2, frame2)
