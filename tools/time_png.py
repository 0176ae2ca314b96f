"""Times the PNG encode of the Set-of-Marks overlay: the device encoder (csrc/png_encode.cu) against the host encoder
(som_overlay.encode_png), at 1920x1080, 2560x1440 and 3240x2160 overlays with 60 boxes each.

  * kernel time: CUDA events around many back-to-back b2p_png_encode launches on device-resident frames, after a warm-up;
  * wall time of one encode as a caller sees it: device path (pinned staging, H2D, launches, D2H of length and bytes)
    against encode_png, alternated, median of the repeats;
  * p50 of get_som_labeled_img on the seeded stand-in models at 1920x1080 with the two encoders alternated.

Prints one JSON object (card name and power limit included) and writes it to --out.

    python tools/time_png.py --out out/time_png.json
"""
import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import __graft_entry__ as ge  # noqa: E402
from omniparser_b200 import ops, som_overlay as SO, synth  # noqa: E402

SIZES = [(1920, 1080), (2560, 1440), (3240, 2160)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.stdout else q.stderr.strip()}


def overlay(w, h, seed, n=60):
    img = synth.screenshot(seed, w, h)
    rng = np.random.default_rng(seed)
    x1 = rng.uniform(0, 0.9, n)
    y1 = rng.uniform(0, 0.95, n)
    boxes = np.stack([x1, y1, x1 + rng.uniform(0.01, 0.1, n), y1 + rng.uniform(0.01, 0.05, n)], 1).clip(0, 1).tolist()
    r = max(w, h) / 3200
    cfg = {"text_scale": 0.8 * r, "text_thickness": max(int(2 * r), 1), "text_padding": max(int(3 * r), 1), "thickness": max(int(3 * r), 1)}
    return SO.som_outputs(img, boxes, True, **cfg)[2]


def kernel_ms(frame, iters):
    h, w, _ = frame.shape
    _, ws_bytes, cap = ops.png_plan(h, w)
    dev = torch.device("cuda", 0)
    src = torch.from_numpy(frame).to(dev)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    out = torch.empty(cap, dtype=torch.uint8, device=dev)
    n = torch.zeros(1, dtype=torch.int64, device=dev)
    for _ in range(5):
        ops.png_encode(src, h, w, ws, ws_bytes, out, cap, n)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ops.png_encode(src, h, w, ws, ws_bytes, out, cap, n)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, int(n.item())


def wall_ms(frames_fn, reps):
    """alternate the two encoders; median wall time of each"""
    dev_t, host_t = [], []
    enc = SO.device_encoder(torch.device("cuda", 0))
    for _ in range(reps):
        t0 = time.perf_counter()
        a = enc.encode(frames_fn)
        t1 = time.perf_counter()
        b = SO.encode_png(frames_fn)
        t2 = time.perf_counter()
        dev_t.append((t1 - t0) * 1e3)
        host_t.append((t2 - t1) * 1e3)
    return float(np.median(dev_t)), float(np.median(host_t)), len(a), len(b)


def labeled_p50(reps):
    from omniparser_b200.utils import get_som_labeled_img
    from PIL import Image
    dev = torch.device("cuda", 0)
    det, cmp_ = ge.standin_models(dev)
    img = Image.fromarray(synth.screenshot(0))
    texts, boxes = synth.ocr_boxes(0)
    is_cuda = SO._is_cuda

    def call():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        get_som_labeled_img(img, det, BOX_TRESHOLD=0.05, output_coord_in_ratio=True, ocr_bbox=boxes, caption_model_processor=cmp_,
                            ocr_text=texts, iou_threshold=0.7)
        return (time.perf_counter() - t0) * 1e3

    times = {"device": [], "host": []}
    try:
        for i in range(reps + 2):
            for mode in ("device", "host"):
                SO._is_cuda = is_cuda if mode == "device" else (lambda d: False)
                t = call()
                if i >= 2:       # warm-up: graphs, encoder buffers
                    times[mode].append(t)
    finally:
        SO._is_cuda = is_cuda
    return {m: float(np.median(v)) for m, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="out/time_png.json")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--labeled-reps", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_png.py measures on a GPU; there is no CPU fallback"
    ge.build()
    res = {"card": card(), "host_threads": len(os.sched_getaffinity(0)), "sizes": []}
    for k, (w, h) in enumerate(SIZES):
        frame = overlay(w, h, 100 + k)
        kms, nbytes = kernel_ms(frame, a.iters)
        dms, hms, dlen, hlen = wall_ms(frame, a.reps)
        res["sizes"].append({"w": w, "h": h, "kernel_ms": round(kms, 3), "device_wall_ms": round(dms, 3),
                             "host_wall_ms": round(hms, 3), "device_bytes": dlen, "host_bytes": hlen,
                             "size_ratio": round(dlen / hlen, 3), "device_faster": dms < hms})
        print(json.dumps(res["sizes"][-1]), flush=True)
    res["get_som_labeled_img_p50_ms"] = labeled_p50(a.labeled_reps)
    out = Path(a.out)
    out.parent.mkdir(parents=True, exist_ok=True)
    out.write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
