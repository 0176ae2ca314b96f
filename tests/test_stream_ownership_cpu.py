"""CPU: which stream every role of the parse path runs on, and so which split-K workspace slot its GEMMs use.

The split-K workspace of the GEMM/conv kernel is keyed by the launching stream; under graph capture that is the capture
stream, and the graph bakes its slot in.  Two roles that may run concurrently (the detector's graph on the detection stream,
a caption lane's graphs on that lane's stream, ...) must therefore launch on different stream handles, or their partial
tiles and arrival counters mix.  torch.cuda.Stream hands out a round-robin pool of 32 streams per device, so streams drawn
from it alias once 32 draws separate two of them; the role streams (ops.role_stream) come from b2p_stream_create instead.

The library is the recorder of test_plan_dryrun_cpu.py (no arithmetic) with a b2p_stream_create that hands out distinct
handles; torch's stream state is a thread-local fake with stream / graph contexts that behave like torch's (a capture makes
the capture stream current).  The plans live on the CPU, so the role streams are those of a stand-in CUDA device."""
import ast
import contextlib
import ctypes as C
import threading
from pathlib import Path

import pytest
import torch

from gemm_plan_util import GEMM_CALLS
from omniparser_b200 import _lib, ops
from standin import florence as FS
from test_pipeline_dryrun_cpu import _batches, _cap_model, _Event, _FakeDetector
from test_plan_dryrun_cpu import _Graph, _Recorder, _Stream

ROOT = Path(__file__).resolve().parents[1]
T = 3


class _ExternalStream(_Stream):
    """torch.cuda.ExternalStream stand-in: wraps the handle b2p_stream_create handed out"""

    def __init__(self, stream_ptr, device=None):
        self.cuda_stream = stream_ptr


class _Pool:
    """torch.cuda.Stream as torch implements it: a round-robin pool of 32 streams per device (the 33rd draw returns the
    stream of the 1st)"""

    def __init__(self):
        self.n = 0

    def __call__(self, *a, **k):
        h = 0x90000 + 0x10 * (self.n % 32)
        self.n += 1
        return _ExternalStream(h)


class _TorchStreams:
    """the current stream of each thread, torch.cuda.stream / torch.cuda.graph contexts, and a log of every capture:
    (capture handle, working stream handle when the capture began, first and one-past-last index into rec.calls)"""

    def __init__(self, rec):
        self.rec, self.tls, self.captures = rec, threading.local(), []

    def cur(self):
        return getattr(self.tls, "cur", 0)

    def capturing(self):
        return getattr(self.tls, "cap", None)

    def current_stream(self, *a, **k):
        return _ExternalStream(self.cur())

    @contextlib.contextmanager
    def stream(self, s):
        prev = self.cur()
        if s is not None:
            self.tls.cur = s.cuda_stream
        try:
            yield
        finally:
            self.tls.cur = prev

    @contextlib.contextmanager
    def graph(self, g, stream=None, **k):
        assert stream is not None and stream.cuda_stream != 0, "a capture on the default stream"
        assert self.capturing() is None
        prev = self.cur()
        self.tls.cur = self.tls.cap = stream.cuda_stream
        i0 = len(self.rec.calls)
        try:
            yield
        finally:
            self.tls.cur, self.tls.cap = prev, None
            self.captures.append((stream.cuda_stream, prev, i0, len(self.rec.calls)))


class _CtxRecorder(_Recorder):
    """the recorder, plus the capture (handle or None) each recorded call was made in; b2p_stream_create hands out a distinct
    non-null handle per stream, as the library's does (kept out of ``calls``: it is not a launch)"""

    def __init__(self):
        super().__init__()
        self.in_capture = []
        self.streams = []
        self.ts = None

    def __getattr__(self, name):
        if name == "b2p_stream_create":
            def create(out):
                _lib.PROTOTYPES[name][1][0].from_param(out)
                out._obj.value = 0x5000 + 0x10 * (len(self.streams) + 1)
                self.streams.append(out._obj.value)
                return 0
            return create
        f = super().__getattr__(name)

        def g(*args):
            n = len(self.calls)
            r = f(*args)
            if len(self.calls) > n:
                self.in_capture.append(self.ts.capturing())
            return r
        return g


@pytest.fixture()
def env(monkeypatch):
    rec = _CtxRecorder()
    ts = _TorchStreams(rec)
    rec.ts = ts
    pool = _Pool()
    monkeypatch.setattr(_lib, "_lib", rec)
    monkeypatch.setattr(ops, "_ROLE_STREAMS", {})
    monkeypatch.setattr(ops, "_stream_device", lambda device: torch.device("cuda", 0))   # the CPU plans' stand-in device
    monkeypatch.setattr(ops, "_stream", lambda: C.c_void_p(ts.cur()))
    monkeypatch.delenv("B2P_NO_GRAPH", raising=False)
    monkeypatch.delenv("B2P_DECODE_PARTS", raising=False)
    for name, val in [("device", lambda *a, **k: contextlib.nullcontext()), ("stream", ts.stream), ("graph", ts.graph),
                      ("CUDAGraph", _Graph), ("Stream", pool), ("ExternalStream", _ExternalStream), ("Event", _Event),
                      ("current_stream", ts.current_stream), ("synchronize", lambda *a, **k: None),
                      ("set_device", lambda *a, **k: None)]:
        monkeypatch.setattr(torch.cuda, name, val)
    return rec, ts, pool


@pytest.fixture(scope="module")
def florence():
    return FS.florence_standin(0)


@pytest.fixture(scope="module")
def yolo_weights():
    from omniparser_b200.yolo_engine import YoloWeights
    from standin.yolo_weights import yolo_standin
    return YoloWeights(yolo_standin(0).state_dict(), torch.device("cpu"))


def _kind(rec, i0, i1):
    names = {c[0] for c in rec.calls[i0:i1]}
    if "b2p_encoder_embed" in names:
        return "enc"
    if "b2p_greedy_pick" in names:
        return "dec"
    assert "b2p_yolo_decode" not in names
    return "yolo"


def _parser(det, cap, lanes, group):
    from omniparser_b200.caption import B200Florence2Processor
    from omniparser_b200.utils import PipelinedParser
    return PipelinedParser(det, dict(model=cap, processor=B200Florence2Processor()), BOX_TRESHOLD=0.05, iou_threshold=0.7, max_new_tokens=T,
                           caption_lanes=lanes, caption_group=group)


def _role_handles(env, cap, yolo_weights, lanes, group, offset):
    """Build what a process builds (a parser, the detector's graph, caption plans of two crop-count buckets, a second parser),
    with ``offset`` pool draws by other code between the detector's first capture and the caption plans'.
    -> {role: set of stream handles it was given}"""
    from omniparser_b200.yolo_engine import YoloPlan
    rec, ts, pool = env
    cap._plans.clear()
    roles = {}

    def put(role, h):
        roles.setdefault(role, set()).add(h)

    pp = _parser(_FakeDetector(), cap, lanes, group)
    put("det", pp.s_det.cuda_stream)
    for lane, s in enumerate(pp.s_caps):
        put(f"cap{lane}", s.cuda_stream)
    n0 = len(ts.captures)
    with ts.stream(pp.s_det):
        YoloPlan(yolo_weights, 1, 64, 96, use_graph=True).run()
    for h, _, i0, i1 in ts.captures[n0:]:
        put("yolo", h)
    for _ in range(offset):
        pool()
    for n, lanes_n in ((20, range(lanes)), (40, [lanes - 1])):    # buckets of 32 (every lane) and 64 crops (last lane)
        for lane in lanes_n:
            n0 = len(ts.captures)
            cap.warm_plan(n, T, FS.PROMPT_IDS, instance=lane, stream=pp.s_caps[lane])
            p = cap.plan_for(n, T, FS.PROMPT_IDS, instance=lane)
            for pt in p.parts:
                put(f"florence{lane}_part{pt['idx']}", pt["stream"].cuda_stream)
            for h, _, i0, i1 in ts.captures[n0:]:
                put(f"florence{lane}" if _kind(rec, i0, i1) == "enc" else f"florence{lane}_dec0", h)
    pp2 = _parser(_FakeDetector(), cap, lanes, group)     # a second parser of the same device: the same role streams
    put("det", pp2.s_det.cuda_stream)
    for lane, s in enumerate(pp2.s_caps):
        put(f"cap{lane}", s.cuda_stream)
    return roles


@pytest.mark.parametrize("lanes,group", [(1, 2), (2, 2), (3, 1)])
def test_role_streams_never_alias(env, florence, yolo_weights, lanes, group):
    """Every role gets one handle, whatever the plans and parsers built, and no two roles share one -- at every position of
    torch's stream pool (a pool stream would alias the caption lanes' capture streams with the detector's streams at some
    offset)."""
    expect = {"det", "yolo"} | {f"{r}{lane}" for lane in range(lanes) for r in ("cap", "florence")} | \
             {f"florence{lane}_{s}0" for lane in range(lanes) for s in ("dec", "part")}
    cap = _cap_model(florence)
    cap.use_graph = True
    n_created = []
    for offset in range(32):
        env[0].streams.clear()
        ops._ROLE_STREAMS.clear()
        roles = _role_handles(env, cap, yolo_weights, lanes, group, offset)
        assert set(roles) == expect, set(roles) ^ expect
        for role, hs in roles.items():
            assert len(hs) == 1, (offset, role, sorted(hs))
        handles = {role: next(iter(hs)) for role, hs in roles.items()}
        by_handle = {}
        for role, h in handles.items():
            by_handle.setdefault(h, []).append(role)
        shared = [r for r in by_handle.values() if len(r) > 1]
        assert not shared, f"pool offset {offset}: roles sharing one stream (and split-K slot): {shared}"
        assert 0 not in by_handle
        n_created.append(len(env[0].streams))
    assert n_created == [len(expect)] * 32          # one b2p_stream_create per role, none per plan or parser


def test_no_pool_streams_in_the_package():
    """No module of the package draws a stream from torch's pool: every stream is an ops.role_stream."""
    for f in sorted((ROOT / "omniparser_b200").glob("*.py")):
        for node in ast.walk(ast.parse(f.read_text())):
            if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "Stream":
                assert ast.unparse(node.func) not in ("torch.cuda.Stream", "cuda.Stream", "Stream"), (f.name, node.lineno)


class _YoloDetector(_FakeDetector):
    """the fake detector, plus the detector's real launch plan run (eagerly once, then captured) on the detection stream"""

    def __init__(self, yolo_weights):
        super().__init__()
        from omniparser_b200.yolo_engine import YoloPlan
        self.plan = YoloPlan(yolo_weights, 1, 64, 96, use_graph=True)

    def detect(self, io, conf, iou, max_det):
        self.plan.run()
        super().detect(io, conf, iou, max_det)


@pytest.mark.parametrize("lanes,group,parts", [(2, 2, 1), (3, 1, 1), (2, 1, 2)])
def test_gemm_calls_of_each_stage_carry_their_role_stream(env, florence, yolo_weights, monkeypatch, lanes, group, parts):
    """Run the pipelined parser end to end with graphs on: every split-K-capable GEMM/conv call made inside a capture carries
    the capture stream of its engine and lane; every eager one carries the working stream of its stage, lane or decode
    chain -- never the default stream, never a capture stream."""
    from omniparser_b200 import caption
    rec, ts, pool = env
    if parts > 1:       # decode chains on their own streams: 128 crops per lane and batch
        monkeypatch.setenv("B2P_DECODE_PARTS", str(parts))
        monkeypatch.setattr(_FakeDetector, "detect", _many_boxes)
    monkeypatch.setattr(caption, "BUCKET", 32)
    cap = _cap_model(florence)
    cap.use_graph = True
    pp = _parser(_YoloDetector(yolo_weights), cap, lanes, group)
    got = list(pp.run(iter(_batches(2 * lanes * group + 1))))
    assert len(got) == 2 * lanes * group + 1
    R = ops.role_stream
    dev = torch.device("cpu")
    det = R("det", dev).cuda_stream
    work = {det: "det"}
    capt = {R("yolo", dev).cuda_stream: ("yolo", det)}
    for lane in range(lanes):
        c = R(f"cap{lane}", dev).cuda_stream
        work[c] = f"cap{lane}"
        capt[R(f"florence{lane}", dev).cuda_stream] = (f"florence{lane}", c)
        for p in range(parts):
            wp = R(f"florence{lane}_part{p}", dev).cuda_stream
            work[wp] = f"florence{lane}_part{p}"
            # a decode chain is captured from its own stream (several chains) or the lane's stream (one chain)
            capt[R(f"florence{lane}_dec{p}", dev).cuda_stream] = (f"florence{lane}_dec{p}", wp if parts > 1 else c)
    assert len(set(work) | set(capt)) == len(work) + len(capt)
    n_gemm = {"eager": 0, "capture": 0}
    for (name, vals), cap_h in zip(rec.calls, rec.in_capture):
        if name not in GEMM_CALLS:
            continue
        st = vals[-1]
        if cap_h is not None:
            assert st == cap_h and st in capt, (name, st, cap_h)
            n_gemm["capture"] += 1
        else:
            assert st in work, (name, st, "eager GEMM outside the role streams")
            n_gemm["eager"] += 1
    assert n_gemm["eager"] > 0 and n_gemm["capture"] > 0
    # every capture runs on the capture stream of its engine, entered from the working stream of the same lane / chain
    seen = set()
    for h, prev, i0, i1 in ts.captures:
        role, from_ = capt[h]
        want = "yolo" if role == "yolo" else ("dec" if "_dec" in role else "enc")
        assert _kind(rec, i0, i1) == want, (role, _kind(rec, i0, i1))
        assert prev == from_, (role, work.get(prev, prev))
        seen.add(role)
    assert seen == {v[0] for v in capt.values()}, sorted(seen)


def _many_boxes(self, io, conf, iou, max_det):
    """65 boxes per screenshot (130 crops per batch of 2): enough rows for two decode chains"""
    for i in range(io["B"]):
        for j in range(65):
            x, y = 4 + 7 * (j % 13), 4 + 40 * (j // 13)
            io["out_box"][i, j] = torch.tensor([float(x), float(y) + i, float(x + 5), float(y + 30 + i)])
        io["out_count"][i] = 65
