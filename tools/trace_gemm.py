"""Where do a GEMM launch's microseconds go?  Runs with B2P_TRACE=1 (stamped launches of the wgmma kernel that
stamps %globaltimer per CTA at the phase boundaries) and prints, per launch, the median CTA's time in each phase.

  B2P_TRACE=1 B2P_NO_GRAPH=1 python tools/trace_gemm.py step      # one parse step (8 screenshots), every GEMM launch
  B2P_TRACE=1 python tools/trace_gemm.py shapes                     # the representative shapes of tools/prof_gemm.py

Phases: prologue (barrier init, descriptor prefetch) | dep-wait (griddepcontrol.wait: the previous kernel's
tail under PDL) | first TMA issued | first stage landed (TMA latency) | first tile's MMAs issued | accumulator ready ->
epilogue starts | epilogue + remaining tiles | teardown.  `span` = first CTA entry -> last CTA exit; `gap` = this launch's
first entry minus the previous launch's last exit (negative = overlapped through PDL).  `main` / `epi`: one consumer
thread's time per CTA summed over all of its items, item start -> accumulators ready (MMA main loop with its TMA waits) and
accumulators ready -> item end (epilogue, split-K reduction); `epi%` = epi / (main + epi) over all CTAs of the launches.
"""
import ctypes as C
import os
import sys

sys.path.insert(0, ".")
assert os.environ.get("B2P_TRACE"), "run with B2P_TRACE=1"
import numpy as np
import torch

from omniparser_b200 import _lib

CTAS, SLOTS, CAP = 160, 16, 1024
NAMES = ["prologue", "dep-wait", "->1st TMA", "TMA lat", "issue", "acc->epi", "epi+rest", "teardown"]


def read():
    stamps = np.zeros((CAP, CTAS, SLOTS), np.uint64)
    meta = np.zeros((CAP, 8), np.int32)
    n = _lib.lib().b2p_trace_read(C.c_void_p(stamps.ctypes.data), C.c_void_p(meta.ctypes.data), CAP)
    _lib.check(0 if n >= 0 else n)
    return stamps[:n].astype(np.int64), meta[:n]


def report(stamps, meta, limit=400):
    prev_exit = None
    agg = {}
    print("mode       M     N      K  bn ks x3 grid |  span    gap | " + " ".join(f"{x:>9s}" for x in NAMES) + "   (us, median CTA)")
    for i, (s, m) in enumerate(zip(stamps, meta)):
        grid = int(m[7])
        s = s[:grid]
        ok = s[:, 0] > 0
        if not ok.any():
            continue
        t0 = s[ok, 0].min()
        span = (s[ok, 8].max() - t0) / 1e3
        gap = (t0 - prev_exit) / 1e3 if prev_exit is not None else float("nan")
        prev_exit = s[ok, 8].max()
        ph = []
        for a, b in zip(range(0, 8), range(1, 9)):
            v = s[ok][:, [a, b]]
            v = v[(v[:, 0] > 0) & (v[:, 1] > 0)]
            ph.append(float(np.median(v[:, 1] - v[:, 0])) / 1e3 if len(v) else float("nan"))
        key = tuple(int(x) for x in m)
        a = agg.setdefault(key, [0, 0.0, np.zeros(8), 0.0, 0.0, 0.0])
        a[0] += 1; a[1] += span; a[2] += np.nan_to_num(np.array(ph)); a[3] += 0.0 if gap != gap else gap
        a[4] += s[ok, 9].sum() / 1e3; a[5] += s[ok, 10].sum() / 1e3
        if i < limit:
            print("%4d %7d %5d %6d %3d %2d %2d %4d | %5.1f %6.1f | " % (*key, span, gap) + " ".join(f"{x:9.2f}" for x in ph))
    print("\nper shape (mean over launches), sorted by total span:")
    top = sorted(agg.items(), key=lambda kv: -kv[1][1])
    for key, (n, sp, ph, gp, mn, ep) in top[:40]:
        print("%4d %7d %5d %6d %3d %2d %2d %4d | n=%3d span %6.1f gap %6.1f | " % (*key, n, sp / n, gp / n) + " ".join(f"{x:9.2f}" for x in ph / n)
              + "   epi%% %5.1f" % (100.0 * ep / max(mn + ep, 1e-9)))
    for k in (20, len(top)):
        mn = sum(v[4] for _, v in top[:k]); ep = sum(v[5] for _, v in top[:k]); sp = sum(v[1] for _, v in top[:k])
        print("top %3d shapes: total span %8.1f us, CTA-time main %10.1f us, epi %10.1f us, epi%% %5.1f"
              % (k, sp, mn, ep, 100.0 * ep / max(mn + ep, 1e-9)))


what = sys.argv[1] if len(sys.argv) > 1 else "shapes"
if what == "step":
    import __graft_entry__ as ge
    from omniparser_b200 import synth
    from omniparser_b200.utils import parse_screenshots
    dev = torch.device("cuda", 0)
    det, cmp_ = ge.standin_models(dev)
    imgs = [synth.screenshot(s) for s in range(8)]
    ocr = [synth.ocr_boxes(s) for s in range(8)]
    for _ in range(2):
        parse_screenshots(imgs, det, cmp_, ocr, BOX_TRESHOLD=0.05, iou_threshold=0.7, max_new_tokens=8)
    read()
    parse_screenshots(imgs, det, cmp_, ocr, BOX_TRESHOLD=0.05, iou_threshold=0.7, max_new_tokens=8)
    report(*read(), limit=0)
else:
    os.environ["PROF_ONCE"] = "1"
    import runpy
    try:
        runpy.run_path("tools/prof_gemm.py", run_name="__main__")   # one warm pass of every case
    except SystemExit:
        pass
    read()
    try:
        runpy.run_path("tools/prof_gemm.py", run_name="__main__")
    except SystemExit:
        pass
    report(*read())
