"""CPU: screenshots of different sizes in one batch, host side.

* `b2p_letterbox_batch_plan_host` on a batch made of every imgsz=640 letterbox case of tests/screen_cases.py plus a 640x480
  image: tables equal Pillow's (b2p_lanczos_coeffs_host and the oracle), skipped passes are flagged, offsets tile the
  reported buffer sizes, and degenerate geometry / a short table buffer are refused before anything is written;
* a dry run of `PipelinedParser` over mixed-size batches (the recording C library of test_plan_dryrun_cpu.py and a fake
  detector with the ragged-batch methods): order, the crop metadata each `b2p_crop_resize` call gets, io slot growth only
  with the pipeline drained, a bounded number of io slots, and the same results as `parse_screenshots`;
* `BatchingOmniparser`: requests of three sizes share one batch."""
import ctypes
import threading

import numpy as np
import pytest
import torch

import screen_cases as S
from omniparser_b200 import _lib, ops
from oracle import ref_restate as R
from test_pipeline_dryrun_cpu import _cap_model, env, florence  # noqa: F401  (fixtures)

SKIP = -1


def _batch_640():
    sizes = [(c.h, c.w) for c in S.LB_CASES if c.imgsz == 640 for _ in range(c.B)] + [(480, 640)]
    geom = []
    for h, w in sizes:
        tw, th, _, rw, rh, pl, pt = R.letterbox_geometry(w, h, 640)
        geom.append((h, w, rw, rh, pl, pt))
    return geom


def _plan(geom, Tw=640, Th=640, capacity=None):
    lib = _lib.lib()
    g = np.ascontiguousarray(np.asarray(geom, np.int32))
    sizes = np.full(3, -5, np.int64)
    rc = lib.b2p_letterbox_batch_plan_host(len(geom), g.ctypes.data, Tw, Th, None, None, 0, sizes.ctypes.data)
    assert rc == 0, lib.b2p_last_error()
    cap = int(sizes[0]) if capacity is None else capacity
    desc = np.full((len(geom), ops.LB_DESC), -7, np.int64)
    tables = np.full(max(cap, 1), -7, np.int32)
    sizes2 = np.full(3, -5, np.int64)
    rc = lib.b2p_letterbox_batch_plan_host(len(geom), g.ctypes.data, Tw, Th, desc.ctypes.data, tables.ctypes.data, cap,
                                           sizes2.ctypes.data)
    return rc, desc, tables, sizes, sizes2


def _host_coeffs(n_in, n_out):
    ks = ctypes.c_int(0)
    cap = n_out * 256
    bounds = np.zeros((n_out, 2), np.int32)
    kk = np.zeros(cap, np.int32)
    assert _lib.lib().b2p_lanczos_coeffs_host(n_in, n_out, ctypes.byref(ks), bounds.ctypes.data, kk.ctypes.data, cap) == 0
    return bounds, kk[:n_out * ks.value].reshape(n_out, ks.value)


def _tiles(intervals, total):
    """half-open intervals, sorted, cover [0, total) without gap or overlap"""
    pos = 0
    for a, b in sorted(intervals):
        assert a == pos, (a, pos)
        pos = b
    assert pos == total


def test_plan_tables_flags_and_offsets():
    geom = _batch_640()
    rc, desc, tables, sizes, sizes2 = _plan(geom)
    assert rc == 0 and np.array_equal(sizes, sizes2)
    n_tab, tmp_b, src_b = (int(x) for x in sizes)
    assert tables.size == n_tab
    src_iv, tmp_iv, tab_iv = [], [], set()
    for i, (h, w, rw, rh, pl, pt) in enumerate(geom):
        d = desc[i]
        assert list(d[2:8]) == [h, w, rw, rh, pl, pt]
        src_iv.append((d[0], d[0] + 3 * h * w))
        for (tab, ks), n_in, n_out, tmp_flag in (((d[8], d[9]), w, rw, True), ((d[10], d[11]), h, rh, False)):
            if n_in == n_out:                                   # Pillow skips the pass
                assert tab == SKIP and ks == SKIP
                if tmp_flag:
                    assert d[1] == SKIP
                continue
            assert tab >= 0 and ks == S.lb_ksize(n_in, n_out)
            bounds = tables[tab:tab + 2 * n_out].reshape(n_out, 2)
            kk = tables[tab + 2 * n_out:tab + 2 * n_out + n_out * ks].reshape(n_out, ks)
            hb, hk = _host_coeffs(n_in, n_out)
            rb, rk = R.lanczos_coeffs(n_in, n_out)
            assert np.array_equal(bounds, hb) and np.array_equal(kk, hk)
            assert np.array_equal(bounds, rb) and np.array_equal(kk, rk)
            tab_iv.add((int(tab), int(tab + n_out * (2 + ks))))
            if tmp_flag:
                assert d[1] >= 0
                tmp_iv.append((d[1], d[1] + 3 * h * rw))
    _tiles(src_iv, src_b)
    _tiles(tmp_iv, tmp_b)
    _tiles(tab_iv, n_tab)                                        # one table per distinct (in, out) pair, packed
    assert desc[-1, 8] == SKIP and desc[-1, 10] == SKIP          # the 640x480 image: both passes skipped
    assert any(g[0] == g[3] and g[1] != g[2] for g in geom) and any(g[1] == g[2] and g[0] != g[3] for g in geom)


def test_plan_is_stable_across_calls_and_cache_evictions():
    geom = _batch_640()
    _, d0, t0, _, _ = _plan(geom)
    for n in range(300):                                         # more distinct pairs than the host cache keeps
        _plan([(100 + n, 900, 640, 71, 0, 284)])
    _, d1, t1, _, _ = _plan(geom)
    assert np.array_equal(d0, d1) and np.array_equal(t0, t1)


@pytest.mark.parametrize("bad,why", [
    ((1, 641, 640, 0, 0, 320), "641x1: resizes to 640x0"),
    ((100, 100, 641, 100, 0, 0), "wider than the canvas"),
    ((100, 100, 100, 100, 600, 0), "pasted past the right edge"),
    ((100, 100, 100, 100, 0, -1), "negative pad"),
])
def test_plan_refuses_degenerate_geometry_before_writing(bad, why):
    lib = _lib.lib()
    geom = _batch_640()[:3] + [bad]
    g = np.ascontiguousarray(np.asarray(geom, np.int32))
    desc = np.full((4, ops.LB_DESC), -7, np.int64)
    tables = np.full(1 << 20, -7, np.int32)
    sizes = np.full(3, -5, np.int64)
    rc = lib.b2p_letterbox_batch_plan_host(4, g.ctypes.data, 640, 640, desc.ctypes.data, tables.ctypes.data, tables.size,
                                           sizes.ctypes.data)
    assert rc != 0, why
    assert (desc == -7).all() and (tables == -7).all() and (sizes == -5).all()
    assert b"letterbox_batch_plan" in lib.b2p_last_error()


def test_plan_refuses_a_short_table_buffer():
    geom = _batch_640()
    rc, desc, tables, sizes, sizes2 = _plan(geom)
    rc, desc, tables, _, sizes2 = _plan(geom, capacity=int(sizes[0]) - 1)
    assert rc != 0 and b"too small" in _lib.lib().b2p_last_error()
    assert (desc == -7).all() and (tables == -7).all() and (sizes2 == -5).all()


def test_ops_plan_front_end():
    geom = _batch_640()
    desc, tables, tmp_b, src_b = ops.letterbox_batch_plan(geom, 640, 640)
    _, d, t, sizes, _ = _plan(geom)
    assert np.array_equal(desc, d) and np.array_equal(tables, t) and (tmp_b, src_b) == (int(sizes[1]), int(sizes[2]))


# ------------------------------------------------------------------------------------------------ pipeline dry run
class _MixedFakeDetector:
    """B200YOLOv9Detector stand-in with both io kinds: one-size slots keyed by (B, H, W, slot) and ragged slots keyed by
    (B, slot) whose capacity (src bytes) grows.  'Detects' 3 boxes per screenshot; records what the pipeline asks of it."""

    def __init__(self, in_flight):
        self.device = torch.device("cpu")
        self._io = {}
        self._lock = threading.RLock()
        self.in_flight = in_flight          # callable: batches the pipeline has in flight on other threads
        self.growths, self.bad_growths = 0, []

    @staticmethod
    def check_capacity(cand_count_host, cap):
        pass

    def filter_device(self, io, ocr_elems, iou_threshold, max_det=300):
        return False

    def _buffers(self, B_, max_det=300):
        return dict(host_count=torch.zeros((B_,), dtype=torch.int32), host_box=torch.zeros((B_, max_det, 4)),
                    out_count=torch.zeros((B_,), dtype=torch.int32), out_box=torch.zeros((B_, max_det, 4)),
                    cand_count=torch.zeros((B_,), dtype=torch.int32), host_cand=torch.zeros((B_,), dtype=torch.int32), cap=8400,
                    B=B_)

    def io_slot(self, sizes, imgsz, max_det, slot=0, drain=None):
        sizes = [tuple(s) for s in sizes]
        B_ = len(sizes)
        if len(set(sizes)) == 1:
            H_, W_ = sizes[0]
            key = (B_, H_, W_, slot)
            if key not in self._io:
                self._io[key] = dict(self._buffers(B_), src=torch.zeros((B_, H_, W_, 3), dtype=torch.uint8),
                                     meta_hw=torch.tensor([[H_, W_]] * B_, dtype=torch.int32),
                                     meta_off=torch.tensor([i * H_ * W_ * 3 for i in range(B_)], dtype=torch.int64))
            return self._io[key]
        off = np.cumsum([0] + [3 * h * w for h, w in sizes])
        io = self._io.setdefault(("mixed", B_, slot), dict(self._buffers(B_), mixed=True, src=None, cap_src=0))
        if io["src"] is None or off[-1] > io["cap_src"]:
            if io["src"] is not None:
                if drain is not None:
                    drain()
                self.growths += 1
                if self.in_flight():
                    self.bad_growths.append(self.in_flight())
            io["cap_src"] = max(int(off[-1]), io["cap_src"] * 3 // 2)
            io["src"] = torch.zeros((io["cap_src"],), dtype=torch.uint8)
        io["batch"] = dict(sizes=sizes, off=off[:-1])
        return io

    @staticmethod
    def stage(io, images, resident=None):
        if io.get("mixed"):
            mb = io["batch"]
            assert [tuple(im.shape[:2]) for im in images] == mb["sizes"]
            io["meta_hw"] = torch.tensor(mb["sizes"], dtype=torch.int32)
            io["meta_off"] = torch.tensor(mb["off"], dtype=torch.int64)

    @staticmethod
    def detect(io, conf, iou, max_det):
        for i in range(io["B"]):
            for j in range(3):      # boxes inside every screenshot (the smallest is 200 x 120)
                io["out_box"][i, j] = torch.tensor([10.0 + 50 * j, 10.0 + 5 * i, 50.0 + 50 * j, 60.0 + 5 * i])
            io["out_count"][i] = 3


def _mixed_batches(n, B_=3):
    """batches of varying composition: mixed ones of growing total size, and one-size ones in between"""
    rng = np.random.default_rng(1)
    pool = [(120, 200), (270, 480), (360, 640), (200, 320), (480, 270), (600, 800)]
    out = []
    for b in range(n):
        if b % 3 == 2:
            sizes = [(270, 480)] * B_
        else:
            k = min(len(pool), 2 + b // 2)
            sizes = [pool[int(rng.integers(0, k))] for _ in range(B_ - 1)] + [pool[(b // 2) % len(pool)]]
            if len(set(sizes)) == 1:
                sizes[0] = (120, 200) if sizes[0] != (120, 200) else (360, 640)
        imgs = [rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in sizes]
        out.append((imgs, [([f"t{b}"], [[2, 2, 30, 12]]) for _ in sizes]))
    return out


@pytest.mark.parametrize("lanes,group", [(1, 1), (2, 1), (1, 2), (2, 2)])
def test_pipelined_parser_io_slot_dry_run(env, florence, lanes, group):
    from omniparser_b200.caption import B200Florence2Processor
    from omniparser_b200.utils import PipelinedParser
    busy = [0]
    lock = threading.Lock()

    det = _MixedFakeDetector(lambda: busy[0])
    cmp_ = dict(model=_cap_model(florence), processor=B200Florence2Processor())
    pp = PipelinedParser(det, cmp_, BOX_TRESHOLD=0.05, iou_threshold=0.7, max_new_tokens=3, caption_lanes=lanes, caption_group=group)

    def tracked(fn):
        def w(*a, **k):
            with lock:
                busy[0] += 1
            try:
                return fn(*a, **k)
            finally:
                with lock:
                    busy[0] -= 1
        return w
    pp._caption_group = tracked(pp._caption_group)
    nb = 14
    batches = _mixed_batches(nb)
    got = list(pp.run(iter(batches)))
    assert len(got) == nb
    for (imgs, _), out in zip(batches, got):
        assert len(out) == len(imgs)
        for elems, ids in out:
            n_icon = sum(1 for e in elems if e["source"] == "box_yolo_content_yolo")
            assert n_icon == 3 and ids.shape[0] == 3
    # results in order: batch b's element boxes are the fake's pixel boxes over batch b's own screenshot sizes
    for (imgs, _), out in zip(batches, got):
        for i, (im, (elems, _)) in enumerate(zip(imgs, out)):
            h, w = im.shape[:2]
            icons = [e["bbox"] for e in elems if e["source"] == "box_yolo_content_yolo"]
            exp = (torch.tensor([[10.0 + 50 * j, 10.0 + 5 * i, 50.0 + 50 * j, 60.0 + 5 * i] for j in range(3)]) /
                   torch.Tensor([w, h, w, h])).tolist()
            assert sorted(icons) == sorted(exp)
    assert sum(1 for c in env.calls if c[0] == "b2p_crop_resize") == nb    # one per batch, from its own slot
    # growth happened, and only with nothing in flight; slots stay bounded
    assert det.growths > 0 and not det.bad_growths, det.bad_growths
    n_slots = lanes * group + group + 1
    assert len([k for k in det._io if k[0] == "mixed"]) <= n_slots


def test_pipelined_parser_slot_crop_meta_per_batch(env, florence):
    """each crop_resize call of a mixed batch reads that batch's (H, W) and offsets at call time"""
    from omniparser_b200 import utils as U
    from omniparser_b200.caption import B200Florence2Processor
    seen = []
    real = U.ops.crop_resize

    def spy(imgs, img_hw, img_off, *a):
        seen.append((img_hw.tolist(), img_off.tolist()))
        return real(imgs, img_hw, img_off, *a)
    U.ops.crop_resize = spy
    try:
        det = _MixedFakeDetector(lambda: 0)
        cmp_ = dict(model=_cap_model(florence), processor=B200Florence2Processor())
        pp = U.PipelinedParser(det, cmp_, BOX_TRESHOLD=0.05, iou_threshold=0.7, max_new_tokens=3, caption_lanes=1)
        batches = _mixed_batches(6)
        list(pp.run(iter(batches)))
    finally:
        U.ops.crop_resize = real
    assert len(seen) == 6
    for (imgs, _), (hw, off) in zip(batches, seen):
        sizes = [list(im.shape[:2]) for im in imgs]
        if len(set(map(tuple, sizes))) > 1:
            assert hw == sizes
            assert off == list(np.cumsum([0] + [3 * h * w for h, w in sizes])[:-1])
        else:
            h, w = sizes[0]
            assert hw == sizes and off == [i * 3 * h * w for i in range(len(imgs))]


@pytest.mark.parametrize("group", [1, 2])
def test_pipelined_parser_equals_parse_screenshots(env, florence, group):
    """the two batch entry points share their stages: on the same one-size and mixed batches, PipelinedParser.run (two
    lanes) returns what parse_screenshots returns batch by batch"""
    from omniparser_b200.caption import B200Florence2Processor
    from omniparser_b200.utils import PipelinedParser, parse_screenshots
    det = _MixedFakeDetector(lambda: 0)
    cmp_ = dict(model=_cap_model(florence), processor=B200Florence2Processor())
    kw = dict(BOX_TRESHOLD=0.05, iou_threshold=0.7, max_new_tokens=3)
    batches = _mixed_batches(6)
    assert {len({im.shape for im in imgs}) > 1 for imgs, _ in batches} == {False, True}
    ref = [parse_screenshots(imgs, det, cmp_, ocr, **kw) for imgs, ocr in batches]
    got = list(PipelinedParser(det, cmp_, caption_lanes=2, caption_group=group, **kw).run(iter(batches)))
    assert len(got) == len(ref)
    for out, exp in zip(got, ref):
        assert len(out) == len(exp)
        for (elems, ids), (elems_ref, ids_ref) in zip(out, exp):
            assert elems == elems_ref and torch.equal(ids, ids_ref) and ids.shape[0] == 3


# ------------------------------------------------------------------------------------------------ server
def test_batching_server_puts_three_sizes_in_one_batch(monkeypatch):
    import base64
    import io

    from PIL import Image

    from omniparser_b200 import utils as U
    from omniparser_b200.server import BatchingOmniparser
    calls = []

    def fake_parse(imgs, som, cmp_, ocr, *a, **k):
        calls.append([im.shape for im in imgs])
        return [([{"type": "icon", "bbox": [0.1, 0.1, 0.2, 0.2], "interactivity": True, "content": f"{im.shape[1]}x{im.shape[0]}",
                   "source": "box_yolo_content_yolo"}], None) for im in imgs]
    monkeypatch.setattr(U, "parse_screenshots", fake_parse)

    def ocr_fn(image, **k):
        return ([], []), None
    srv = BatchingOmniparser({"BOX_TRESHOLD": 0.05, "ocr_fn": ocr_fn, "max_batch": 8, "max_wait_ms": 500.0}, models=(object(), object()))
    sizes = [(320, 200), (200, 320), (256, 256), (320, 200), (200, 320), (256, 256)]
    b64 = []
    for k, (w, h) in enumerate(sizes):
        buf = io.BytesIO()
        Image.fromarray(np.full((h, w, 3), 40 * k, np.uint8)).save(buf, format="PNG")
        b64.append(base64.b64encode(buf.getvalue()).decode("ascii"))
    got = {}
    th = [threading.Thread(target=lambda k=k: got.__setitem__(k, srv.parse(b64[k]))) for k in range(len(sizes))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    srv.close()
    assert srv.stats["batches"] == 1 and srv.stats["items"] == 6, srv.stats
    assert len(calls) == 1 and len({s[:2] for s in calls[0]}) == 3
    for k, (w, h) in enumerate(sizes):        # per-request results keep their own request
        assert got[k][1][0]["content"] == f"{w}x{h}"
