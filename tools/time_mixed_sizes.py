"""Time screenshots of different sizes in one batch against one batch per size (what a server keyed by image size does).

Per mix (two screenshots of each of four common sizes, 8 per step; the five mixes leave out one of the five sizes in turn):
  (a) one parse_screenshots call over the 8 mixed screenshots (ragged letterbox, one B = 8 detector forward, one caption pass)
  (b) one parse_screenshots call per size group (four calls at B = 2)
Steps of (a) and (b) alternate; every shape is warmed up first; each figure is the median of the repeats, in screenshots/s.
Then the letterbox alone: b2p_letterbox_batch over all ten screenshots against one b2p_letterbox call per size, kernel time
from CUDA events over many launches.  Seeded stand-in models and synth screenshots (no checkpoints needed).

    python tools/time_mixed_sizes.py [--steps 5] [--repeats 3] [--json out/mixed_sizes.json]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

SIZES = [(1920, 1080), (2560, 1440), (1366, 768), (1280, 800), (1170, 2532)]


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip().splitlines()[0] if q.stdout else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="steps per repeat and mode")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--lb-iters", type=int, default=200)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_mixed_sizes: no CUDA device (this script measures the GPU and has no CPU fall-back)")
    import __graft_entry__ as ge
    from omniparser_b200 import ops, synth
    from omniparser_b200.detector import _geometry
    from omniparser_b200.utils import parse_screenshots
    ge.build()
    dev = torch.device("cuda", 0)
    info = card()
    print("card:", info, flush=True)
    det, cmp_ = ge.standin_models(dev)
    kw = dict(BOX_TRESHOLD=0.05, iou_threshold=0.7, max_new_tokens=8)
    shots = {s: [(synth.screenshot(10 * k + j, *s), synth.ocr_boxes(10 * k + j, *s)) for j in range(2)] for k, s in enumerate(SIZES)}

    def step_mixed(mix):
        imgs = [im for s in mix for im, _ in shots[s]]
        ocr = [o for s in mix for _, o in shots[s]]
        parse_screenshots(imgs, det, cmp_, ocr, **kw)

    def step_grouped(mix):
        for s in mix:
            parse_screenshots([im for im, _ in shots[s]], det, cmp_, [o for _, o in shots[s]], **kw)

    def timed(fn, mix):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            fn(mix)
        torch.cuda.synchronize()
        return 8 * args.steps / (time.perf_counter() - t0)

    results = dict(card=info, steps=args.steps, repeats=args.repeats, mixes=[])
    for left_out in SIZES:
        mix = [s for s in SIZES if s != left_out]
        for _ in range(2):                                   # warm-up: plans, graphs, io slots, caption buckets
            step_mixed(mix)
            step_grouped(mix)
        a, b = [], []
        for _ in range(args.repeats):
            a.append(timed(step_mixed, mix))
            b.append(timed(step_grouped, mix))
        row = dict(mix=[f"{w}x{h}" for w, h in mix], mixed_sps=statistics.median(a), grouped_sps=statistics.median(b),
                   mixed_all=a, grouped_all=b)
        row["ratio"] = row["mixed_sps"] / row["grouped_sps"]
        results["mixes"].append(row)
        print(f"mix {' '.join(row['mix'])}: (a) one mixed call {row['mixed_sps']:.1f} screenshots/s, "
              f"(b) one call per size {row['grouped_sps']:.1f} screenshots/s, a/b {row['ratio']:.3f}", flush=True)

    # letterbox alone: all ten screenshots
    imgs = [im for s in SIZES for im, _ in shots[s]]
    geo = [_geometry(im.shape[1], im.shape[0], 640) for im in imgs]
    desc, tables, tmp_b, src_b = ops.letterbox_batch_plan([(im.shape[0], im.shape[1], g[3], g[4], g[5], g[6])
                                                           for im, g in zip(imgs, geo)], 640, 640)
    src = torch.from_numpy(np.concatenate([im.reshape(-1) for im in imgs])).to(dev)
    tmp = torch.empty((tmp_b,), dtype=torch.uint8, device=dev)
    B = len(imgs)
    canvas = torch.empty((B, 640, 640, 3), dtype=torch.uint8, device=dev)
    d_desc, d_tab = torch.from_numpy(desc).to(dev), torch.from_numpy(tables).to(dev)
    groups = []
    for k, s in enumerate(SIZES):
        g = _geometry(s[0], s[1], 640)
        gs = torch.from_numpy(np.stack([im for im, _ in shots[s]])).to(dev)
        groups.append((gs, g, torch.empty((2 * s[1] * g[3] * 3,), dtype=torch.uint8, device=dev), canvas[2 * k:2 * k + 2]))

    def lb_batch():
        ops.letterbox_batch(src, B, desc, d_desc, d_tab, 640, 640, tmp, canvas)

    def lb_per_size():
        for gs, (tw, th, _, rw, rh, pl, pt), t, cv in groups:
            ops.letterbox(gs, 2, gs.shape[1], gs.shape[2], rw, rh, tw, th, pl, pt, t, cv)

    def kernel_ms(fn):
        for _ in range(10):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.lb_iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.lb_iters

    lb = dict(batch_ms=[], per_size_ms=[])
    for _ in range(args.repeats):
        lb["batch_ms"].append(kernel_ms(lb_batch))
        lb["per_size_ms"].append(kernel_ms(lb_per_size))
    lb["batch_ms_median"], lb["per_size_ms_median"] = statistics.median(lb["batch_ms"]), statistics.median(lb["per_size_ms"])
    results["letterbox_10"] = lb
    print(f"letterbox of the 10 screenshots: b2p_letterbox_batch {lb['batch_ms_median'] * 1e3:.1f} us, "
          f"five b2p_letterbox calls {lb['per_size_ms_median'] * 1e3:.1f} us", flush=True)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
