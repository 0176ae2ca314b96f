"""CPU: the device PNG encoder's host side -- b2p_png_plan_host against a restatement of its band / worst-case / workspace
formulas, b2p_png_encode's argument checks (made before any launch, so they hold without a device), and the plumbing of
``som_outputs(device=cuda)`` through :class:`som_overlay.DevicePngEncoder` with the C library replaced by the argument-checking
recorder of test_plan_dryrun_cpu.py (no arithmetic runs)."""
import base64
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

from omniparser_b200 import _lib, ops, som_overlay
from test_plan_dryrun_cpu import _Recorder, _Stream

IDAT_MAX = 2 ** 31 - 1
BAND_TARGET = 32768       # filtered bytes per band (whole rows, at least one)


def _stored(n):
    return n + 5 * -(-n // 65535)


def _align(v, a):
    return -(-v // a) * a


def plan_py(H, W):
    """(bands, workspace bytes, worst-case bytes) or None if refused"""
    if H < 1 or W < 1:
        return None
    pitch = 1 + 3 * W
    rows = min(H, 1 if pitch >= BAND_TARGET else BAND_TARGET // pitch)
    bands = -(-H // rows)
    last = (H - (bands - 1) * rows) * pitch
    stream = (bands - 1) * _stored(rows * pitch) + _stored(last)
    if 2 + stream + 4 > IDAT_MAX:
        return None
    out = 43 + stream + 20      # signature, IHDR, IDAT head, zlib header | Adler-32, IDAT CRC, IEND
    filt = H * pitch
    stage = _align(_stored(rows * pitch), 16)
    ws = _align(filt + 16, 256) + _align(4 * filt, 256) + _align(bands * stage, 256) + _align(bands * 32, 256)
    return bands, ws, out


def _lib_plan(H, W):
    sizes = np.zeros(3, np.int64)
    rc = _lib.lib().b2p_png_plan_host(H, W, sizes.ctypes.data)
    return None if rc else tuple(int(v) for v in sizes)


def _largest_h(W):
    lo, hi = 1, 1
    while plan_py(hi, W) is not None:
        lo, hi = hi, hi * 2
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if plan_py(mid, W) is not None else (lo, mid)
    return lo


@pytest.mark.parametrize("H,W", [(1, 1), (1, 1920), (1, 40000), (1080, 1), (100000, 1), (1079, 1919), (1080, 1920),
                                 (2160, 3240), (5, 5461), (7, 5462)])
def test_plan_matches_formula(H, W):
    got = _lib_plan(H, W)
    assert got == plan_py(H, W), (H, W, got)
    bands, ws, out = got
    assert bands >= 1 and out >= 63 + H * (1 + 3 * W)


@pytest.mark.parametrize("W", [1920, 1, 700000])
def test_plan_largest_frame(W):
    Hmax = _largest_h(W)
    got = _lib_plan(Hmax, W)
    assert got is not None and got == plan_py(Hmax, W)
    assert got[2] - 43 - 20 + 6 <= IDAT_MAX
    assert _lib_plan(Hmax + 1, W) is None
    assert b"2^31" in _lib.lib().b2p_last_error()


@pytest.mark.parametrize("H,W", [(0, 10), (10, 0), (-1, 5), (5, -3)])
def test_plan_rejects_empty(H, W):
    assert _lib_plan(H, W) is None


def test_plan_rejects_wide_row():
    assert _lib_plan(1, 2 ** 30) is None


def _encode_rc(H, W, ws_bytes, out_cap, ptr=0x1000):
    p = C.c_void_p(ptr)
    return _lib.lib().b2p_png_encode(p, H, W, p, ws_bytes, p, out_cap, p, C.c_void_p(0))


def test_encode_rejects_before_launch():
    """every refusal returns before the library touches a device (this machine may have none)"""
    _, ws, out = plan_py(1080, 1920)
    assert _encode_rc(1080, 1920, ws - 1, out) == -1
    assert b"workspace" in _lib.lib().b2p_last_error()
    assert _encode_rc(1080, 1920, ws, out - 1) == -1
    assert b"capacity" in _lib.lib().b2p_last_error()
    for H, W in [(0, 1920), (1080, 0), (-4, 4)]:
        assert _encode_rc(H, W, ws, out) == -1
    assert _encode_rc(1080, 1920, ws, out, ptr=0) == -1
    assert b"null" in _lib.lib().b2p_last_error()


class _PlanRecorder(_Recorder):
    """the recorder, with the host-only plan answered by the real library; the encode writes the host encoder's PNG of
    the frame it was handed into the output buffer (CPU tensors standing in for device memory)"""

    def __init__(self, real):
        super().__init__()
        self.real = real

    def __getattr__(self, name):
        f = super().__getattr__(name)
        if name == "b2p_png_plan_host":
            def plan(H, W, sizes):
                f(H, W, sizes)
                return self.real.b2p_png_plan_host(H, W, sizes)
            return plan
        if name == "b2p_png_encode":
            def enc(rgb, H, W, ws, ws_bytes, out, out_cap, out_len, st):
                f(rgb, H, W, ws, ws_bytes, out, out_cap, out_len, st)
                frame = np.ctypeslib.as_array((C.c_ubyte * (H * W * 3)).from_address(rgb.value)).reshape(H, W, 3)
                png = som_overlay.encode_png(frame)
                assert len(png) <= out_cap
                C.memmove(out.value, png, len(png))
                C.c_longlong.from_address(out_len.value).value = len(png)
                return 0
            return enc
        if name == "b2p_stream_create":
            def create(out):
                _lib.PROTOTYPES[name][1][0].from_param(out)
                out._obj.value = 0x5010
                return 0
            return create
        return f


class _ExternalStream(_Stream):
    def __init__(self, stream_ptr, device=None):
        self.cuda_stream = stream_ptr


@pytest.fixture()
def png_rec(monkeypatch):
    real = _lib.lib()
    r = _PlanRecorder(real)
    monkeypatch.setattr(_lib, "_lib", r)
    monkeypatch.setattr(ops, "_ROLE_STREAMS", {})
    monkeypatch.setattr(ops, "_stream_device", lambda device: torch.device("cuda", 0))
    monkeypatch.setattr(ops, "_stream", lambda: C.c_void_p(0x5010))
    monkeypatch.setattr(torch.cuda, "device", lambda *a, **k: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "stream", lambda *a, **k: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "ExternalStream", _ExternalStream)
    monkeypatch.setattr(som_overlay, "_ENCODERS", {})
    # host tensors stand in for pinned and device memory
    monkeypatch.setattr(som_overlay.DevicePngEncoder, "_pinned", staticmethod(lambda n, dtype=None: torch.empty(n, dtype=dtype or torch.uint8)))
    monkeypatch.setattr(som_overlay.DevicePngEncoder, "_device_buf", lambda self, n, dtype=None: torch.empty(n, dtype=dtype or torch.uint8))
    return r


def test_som_outputs_device_plumbing(png_rec):
    rng = np.random.default_rng(3)
    img = (rng.integers(0, 4, (90, 130, 3)) * 60).astype(np.uint8)
    boxes = [[0.1, 0.1, 0.4, 0.5], [0.5, 0.2, 0.9, 0.8]]
    enc_dev, coords_dev, frame_dev = som_overlay.som_outputs(img, boxes, True, device="cuda:0")
    enc_host, coords_host, frame_host = som_overlay.som_outputs(img, boxes, True)
    assert np.array_equal(frame_dev, frame_host) and str(coords_dev) == str(coords_host)
    assert base64.b64decode(enc_dev) == som_overlay.encode_png(frame_host)
    names = [c[0] for c in png_rec.calls]
    assert names == ["b2p_png_plan_host", "b2p_png_encode"]
    _, H, W, _ws, ws_bytes, _out, out_cap, _len, st = png_rec.calls[-1][1]
    bands, ws_plan, out_plan = plan_py(90, 130)
    assert (H, W) == (90, 130) and ws_bytes >= ws_plan and out_cap >= out_plan and st == 0x5010
    # a second, smaller frame reuses the grown buffers
    enc = som_overlay.device_encoder("cuda:0")
    bufs = (enc._ws.data_ptr(), enc._dev_out.data_ptr(), enc._pin_in.data_ptr())
    small = img[:40, :50].copy()
    assert enc.encode(small) == som_overlay.encode_png(small)
    assert (enc._ws.data_ptr(), enc._dev_out.data_ptr(), enc._pin_in.data_ptr()) == bufs


def test_som_outputs_host_without_cuda_device(png_rec):
    img = np.full((20, 30, 3), 200, np.uint8)
    for dev in (None, "cpu", torch.device("cpu")):
        som_overlay.som_outputs(img, [[0.1, 0.1, 0.5, 0.5]], False, device=dev)
    assert png_rec.calls == []
