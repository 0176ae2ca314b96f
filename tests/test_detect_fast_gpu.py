"""The fast (fp16) detector's own non-GEMM kernels, exactly, at the shapes the detector runs.

`precision="fp16"` is the detector mode every default caller and the benchmark run (batch 8, 640x640 canvas).  End to end
it is only held to fp16 drift bounds (taps <= 2 % RMS, head logits <= 0.25), which a subtly wrong pooling, fusion or
decode kernel fits inside.  This module pins each of them on its own:

* ADown pooling (`adown_avg_kernel` / `adown_max_kernel`), CBFuse (`cbfuse_batched_kernel<NS>`, NS = 1..5, and the
  generic kernel at NS = 0), the SPPELAN max-pool chain and nearest upsample, bit for bit against a CPU float32
  restatement in the kernel's association order, in the production layouts (channel slices of concat buffers, CBFuse
  sources at their CBLinear offsets, the three max-pools inside one buffer), with exact ties and zeros of both signs;
* `im2col_u8` for both stems (YOLO 3x3/s2 with the /255 table, DaViT 7x7/s4 with the CLIP table), plain and [hi | lo];
* `yolo_decode` against fp64 (dense outputs, within a bound derived from the operation count) and against the compaction
  of its own dense outputs (candidates, bit for bit), including the strict `> conf`, first-maximum-wins over classes, the
  production launch without dense outputs and more candidates than the list holds;
* `batched_nms` on one batch whose images take every path (empty, one box, coordinate trick, per-class, full, clamped),
  against the documented rule (`oracle.ref_restate.greedy_nms_numpy`) bit for bit and against torchvision up to the
  order inside runs of exactly tied scores;
* host-side rejections, and on the CPU: that every non-GEMM call of the fast plan at (8, 640, 640) and (1, 1088, 1920)
  has a case here (coverage).

Every output buffer is poisoned with a sentinel and followed by a guard image: nothing outside the written region may
change.  Every pointer a launch uses lies inside its torch allocation (checked before the call).  Everything runs on the
current stream of one process."""
from __future__ import annotations

import collections
import ctypes as C
import functools
from dataclasses import dataclass

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from omniparser_b200 import _lib, ops
from oracle import ref_restate as R
from test_parity_planes_gpu import _bits, _covers, _rejected
from test_plan_dryrun_cpu import rec  # noqa: F401  (fixture: the C library replaced by an argument-checking recorder)

DEV = "cuda:0"
SENTINEL = -60000.0         # exactly representable in fp16 and fp32; no output here reaches that magnitude
SENTINEL_I32 = -7
ZERO_SIGN = collections.Counter()   # per kernel: elements whose only difference from the restatement is the sign of a zero
f32 = np.float32


# ------------------------------------------------------------------------------------------------ buffers
def fp16_values(shape, seed):
    """fp16 activations: a N(0, 2) bulk, 20 % multiples of 1/4 (exact ties), 5 % of magnitude 2^12..2^13 and 5 % near
    2^-20 (so that fp32 sums of a few values round, and their association order shows), 10 % +0 and 10 % -0 (SiLU
    outputs underflow to -0 in fp16).  Generated on the device (the large cases hold ~50 M values)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    v = torch.randn(shape, generator=g, device=DEV) * 2
    r = torch.rand(shape, generator=g, device=DEV)
    v = torch.where(r < 0.2, torch.round(v) * 0.25, v)
    v = torch.where((r >= 0.6) & (r < 0.65), v.sign() * (4096 + 4096 * torch.rand(shape, generator=g, device=DEV)), v)
    v = torch.where((r >= 0.65) & (r < 0.7), v * 2 ** -20, v)
    v = torch.where(r >= 0.9, torch.zeros_like(v), v)
    v = torch.where((r >= 0.8) & (r < 0.9), torch.zeros_like(v).neg(), v)
    return v.half()


def in_map(B, H, W, ld, c0, C_, seed, dev):
    """[B, H, W, ld] buffer, the slice [c0, c0 + C) is the operand; the guard channels hold random values too.  On the
    CPU (recording only) the buffer is left uninitialised."""
    if dev == "cpu":
        return ops.Map(torch.empty(B, H, W, ld, dtype=torch.float16), c0, C_)
    return ops.Map(fp16_values((B, H, W, ld), seed), c0, C_)


def out_map(B, H, W, ld, c0, C_, dev):
    """poisoned output slice of a [B, H, W, ld] buffer, followed by a poisoned guard image -> (map, whole buffer)"""
    if dev == "cpu":
        big = torch.empty(B + 1, H, W, ld, dtype=torch.float16)
    else:
        big = torch.full((B + 1, H, W, ld), SENTINEL, dtype=torch.float16, device=dev)
    return ops.Map(big[:B], c0, C_), big


def check_out(m: ops.Map, big):
    """outside the slice still the sentinel (bit for bit), inside nothing is; the guard image untouched"""
    mask = torch.zeros(m.ld, dtype=torch.bool)
    mask[m.c0:m.c0 + m.C] = True
    b = _bits(m.buf.cpu())
    s = _bits(torch.tensor([SENTINEL], dtype=m.buf.dtype))[0]
    assert bool((b[..., ~mask] == s).all()), f"{int((b[..., ~mask] != s).sum())} elements outside the output slice were written"
    assert not bool((b[..., mask] == s).any()), f"{int((b[..., mask] == s).sum())} elements of the output slice were not written"
    assert bool((big[m.B:] == SENTINEL).all()), "the guard image after the output was written"


def extent(m: ops.Map):
    _covers(m.buf, m.ptr, (m.B * m.H * m.W - 1) * m.ld + m.C)


def sl(m: ops.Map):
    """the slice's values, on the CPU"""
    return m.buf[..., m.c0:m.c0 + m.C].cpu()


def assert_exact(kernel, got, ref, what=""):
    """fp16 `got` == `ref` as values (torch.equal: -0 == +0), and bit for bit except where both are zeros of different
    sign (fmaxf / __hmax2 may return either zero); those are counted per kernel, not failed."""
    assert got.shape == ref.shape, (got.shape, ref.shape)
    gf, rf = got.float(), ref.float()
    if not torch.equal(gf, rf):
        bad = (gf != rf).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError(f"{kernel}{what}: {len(bad)} of {got.numel()} values differ; first at {i}: "
                             f"got {gf[i].item()!r}, expected {rf[i].item()!r}")
    diff = _bits(got) != _bits(ref)
    assert bool((gf[diff] == 0).all())
    ZERO_SIGN[kernel] += int(diff.sum())
    print(f"{kernel}{what}: exact, {int(diff.sum())} sign-of-zero differences (running total {ZERO_SIGN[kernel]})")


# ------------------------------------------------------------------------------------------------ ADown pooling
@dataclass(frozen=True)
class AdownCase:
    """x: (ld, c0) slice of C channels; x1 / x2: (ld, c0) of their C/2-channel outputs"""
    name: str
    B: int
    H: int
    W: int
    C: int
    x: tuple
    x1: tuple = None
    x2: tuple = None

    def o1(self):
        return self.x1 or (self.C // 2, 0)

    def o2(self):
        return self.x2 or (self.C // 2, 0)


def _plan_adown(tag, B, H1, W1):
    """the seven ADown calls of the fast plan (canvas 2*H1 x 2*W1): input maps and concat slices"""
    H2, W2, H3, W3, H4, W4 = H1 // 2, W1 // 2, H1 // 4, W1 // 4, H1 // 8, W1 // 8
    return [AdownCase(f"{tag}_l4_{H2}x{W2}_c256", B, H2, W2, 256, (256, 0)),
            AdownCase(f"{tag}_l6_{H3}x{W3}_c512", B, H3, W3, 512, (512, 0)),
            AdownCase(f"{tag}_l8_{H4}x{W4}_c1024", B, H4, W4, 1024, (1024, 0)),
            AdownCase(f"{tag}_l36_{H3}x{W3}_c256", B, H3, W3, 256, (256, 0)),
            AdownCase(f"{tag}_l23_{H3}x{W3}_c512_slice_of_1024", B, H3, W3, 512, (1024, 512)),
            AdownCase(f"{tag}_l39_{H4}x{W4}_c512", B, H4, W4, 512, (512, 0)),
            AdownCase(f"{tag}_l26_{H4}x{W4}_c1024_slice_of_1536", B, H4, W4, 1024, (1536, 512))]


ADOWN_CASES = _plan_adown("b8_640", 8, 320, 320) + _plan_adown("b1_1088x1920", 1, 544, 960) + [
    AdownCase("b3_2x2_one_output_pixel", 3, 2, 2, 32, (64, 16), (48, 8), (24, 8)),
    AdownCase("b3_4x6_out_slices", 3, 4, 6, 64, (96, 32), (64, 16), (48, 8)),
]


def adown_launch(c: AdownCase, dev):
    x = in_map(c.B, c.H, c.W, *c.x, c.C, sum(map(ord, c.name)), dev)
    x1, b1 = out_map(c.B, c.H, c.W, *c.o1(), c.C // 2, dev)
    x2, b2 = out_map(c.B, c.H // 2, c.W // 2, *c.o2(), c.C // 2, dev)
    for m in (x, x1, x2):
        extent(m)
    ops.adown_pool(x, x1, x2)
    return x, (x1, b1), (x2, b2)


def adown_ref(x16):
    """ADown front half in the kernels' order: a = ((a + b) + (c + d)) * 0.25 over the (H-1)x(W-1) windows; x1 = a[:C/2]
    with an exactly zero last row and column; x2 = 3x3 / stride 2 / pad 1 max over a[C/2:]"""
    v = x16.float()
    avg = ((v[:, :-1, :-1] + v[:, :-1, 1:]) + (v[:, 1:, :-1] + v[:, 1:, 1:])) * 0.25
    B, H, W, C_ = v.shape
    r1 = torch.zeros(B, H, W, C_ // 2)
    r1[:, :-1, :-1] = avg[..., :C_ // 2]
    r2 = F.max_pool2d(avg[..., C_ // 2:].permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert r2.shape[1:3] == (H // 2, W // 2)
    return r1.half(), r2.half()


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c.name for c in ADOWN_CASES])
def test_adown_pool_fp16_exact(name):
    c = next(c for c in ADOWN_CASES if c.name == name)
    x, (x1, b1), (x2, b2) = adown_launch(c, DEV)
    torch.cuda.synchronize()
    check_out(x1, b1)
    check_out(x2, b2)
    r1, r2 = adown_ref(sl(x))
    got1 = sl(x1)
    assert bool((_bits(got1[:, -1]) == 0).all() and (_bits(got1[:, :, -1]) == 0).all()), "x1's last row / column is not +0"
    assert_exact("adown_avg", got1, r1)
    assert_exact("adown_max", sl(x2), r2)


# ------------------------------------------------------------------------------------------------ CBFuse
@dataclass(frozen=True)
class CbfuseCase:
    """srcs[i]: (ld, c0) of source i, 2^i times coarser than the target; last / out: (ld, c0)"""
    name: str
    B: int
    H: int
    W: int
    C: int
    srcs: tuple
    last: tuple
    out: tuple


def _plan_cbfuse(tag, B, H1, W1):
    """the five CBFuse calls of the fast plan: sources are slices of the CBLinear outputs r10..r14 (64 / 192 / 448 / 960 /
    1984 channels, each at its own scale), `last` is a map (NS = 5: the second half of the stem output)"""
    r_ld = (64, 192, 448, 960, 1984)
    offs = {5: 0, 4: 64, 3: 192, 2: 448, 1: 960}
    out = []
    for ns, C_, lvl in ((5, 64, 0), (4, 128, 1), (3, 256, 2), (2, 512, 3), (1, 1024, 4)):
        srcs = tuple((r_ld[lvl + i], offs[ns]) for i in range(ns))
        last = (128, 64) if ns == 5 else (C_, 0)
        out.append(CbfuseCase(f"{tag}_ns{ns}_{H1 >> lvl}x{W1 >> lvl}_c{C_}", B, H1 >> lvl, W1 >> lvl, C_, srcs, last, (C_, 0)))
    return out


CBFUSE_CASES = _plan_cbfuse("b8_640", 8, 320, 320) + _plan_cbfuse("b1_1088x1920", 1, 544, 960) + [
    CbfuseCase("b3_ns0_generic_kernel", 3, 8, 12, 64, (), (96, 16), (80, 8)),
    CbfuseCase("b3_ns3_out_slice", 3, 8, 12, 64, ((80, 8), (64, 0), (72, 8)), (64, 0), (96, 24)),
]


BIG = 30000.0


def cbfuse_launch(c: CbfuseCase, dev):
    seed = sum(map(ord, c.name))
    srcs = [in_map(c.B, c.H >> i, c.W >> i, ld, c0, c.C, seed + i, dev) for i, (ld, c0) in enumerate(c.srcs)]
    last = in_map(c.B, c.H, c.W, *c.last, c.C, seed + 7, dev)
    if dev != "cpu" and len(srcs) >= 2:
        # every 8th channel: +BIG, -BIG, then small terms.  The fp32 sum then depends on the order of the sources
        # (with two sources the first two terms commute, so the order is only observable from three on).
        ch = slice(None, None, 8)
        g = torch.Generator(device=DEV).manual_seed(seed)
        for i, s in enumerate(srcs):
            v = s.buf[..., s.c0:s.c0 + c.C][..., ch]
            if i < 2:
                v.fill_(BIG if i == 0 else -BIG)
            else:
                v.copy_((torch.randn(v.shape, generator=g, device=DEV) * 2 ** -12).half())
        lv = last.buf[..., last.c0:last.c0 + c.C][..., ch]
        lv.copy_((torch.randn(lv.shape, generator=g, device=DEV) * 2 ** -12).half())
    out, big = out_map(c.B, c.H, c.W, *c.out, c.C, dev)
    for m in srcs + [last, out]:
        extent(m)
    ops.cbfuse(srcs, last, out)
    return srcs, last, (out, big)


def cbfuse_ref(srcs, last):
    """fp32 sum of the nearest-upsampled sources in order, then `last`, rounded once"""
    acc = None
    for i, s in enumerate(srcs):
        t = sl(s).float()
        if i:
            t = t.repeat_interleave(1 << i, 1).repeat_interleave(1 << i, 2)
        acc = t if acc is None else acc + t
    lf = sl(last).float()
    return (lf if acc is None else acc + lf).half()


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c.name for c in CBFUSE_CASES])
def test_cbfuse_fp16_exact(name):
    c = next(c for c in CBFUSE_CASES if c.name == name)
    srcs, last, (out, big) = cbfuse_launch(c, DEV)
    torch.cuda.synchronize()
    check_out(out, big)
    assert_exact(f"cbfuse_ns{len(srcs)}", sl(out), cbfuse_ref(srcs, last))


# ------------------------------------------------------------------------------------------------ SPPELAN max-pool chain, upsample
@dataclass(frozen=True)
class MapCase:
    name: str
    B: int
    H: int       # input size
    W: int
    C: int
    x: tuple     # (ld, c0)
    y: tuple


# the fast plan: three 5x5 max-pools inside one 1024-channel buffer (slice i -> slice i + 1); the two upsamples read a
# slice of a concat and write a slice of the next one
MAXPOOL_CASES = [MapCase(f"{t}_sppelan_{H}x{W}", B, H, W, 256, (1024, 0), (1024, 256))
                 for t, B, H, W in (("b8_640", 8, 20, 20), ("b1_1088x1920", 1, 34, 60), ("b3_3x5", 3, 3, 5))]
UPSAMPLE_CASES = []
for _t, _B, _H5, _W5 in (("b8_640", 8, 20, 20), ("b1_1088x1920", 1, 34, 60)):
    UPSAMPLE_CASES += [MapCase(f"{_t}_x29_{_H5}x{_W5}_into_cat31", _B, _H5, _W5, 512, (1024, 512), (1536, 0)),
                       MapCase(f"{_t}_x32_{2 * _H5}x{2 * _W5}_into_cat34", _B, 2 * _H5, 2 * _W5, 512, (768, 256), (1024, 0))]
UPSAMPLE_CASES.append(MapCase("b3_3x5_plain_maps", 3, 3, 5, 24, (24, 0), (24, 0)))


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c.name for c in MAXPOOL_CASES])
def test_sppelan_maxpool_chain_exact(name):
    """slice 0 of the buffer holds the input; launch i reads slice i and writes slice i + 1.  After each launch the slices
    already written are unchanged, the next one equals max_pool2d(5, 1, 2) of the previous one, the rest is poison."""
    c = next(c for c in MAXPOOL_CASES if c.name == name)
    ld, C_ = c.x[0], c.C
    sp, big = out_map(c.B, c.H, c.W, ld, 0, ld, DEV)
    sp.buf[..., :C_] = fp16_values((c.B, c.H, c.W, C_), sum(map(ord, c.name)))
    x0 = sp.buf[..., :C_].cpu()
    prev = x0
    for i in range(3):
        a, b = ops.Map(sp.buf, C_ * i, C_), ops.Map(sp.buf, C_ * (i + 1), C_)
        extent(a); extent(b)
        before = sp.buf[..., :C_ * (i + 1)].cpu()
        ops.maxpool_s1(a, b, 5)
        torch.cuda.synchronize()
        assert torch.equal(_bits(sp.buf[..., :C_ * (i + 1)].cpu()), _bits(before)), f"launch {i} changed its input slices"
        assert bool((sp.buf[..., C_ * (i + 2):] == SENTINEL).all()) and bool((big[c.B:] == SENTINEL).all())
        ref = F.max_pool2d(prev.float().permute(0, 3, 1, 2), 5, 1, 2).permute(0, 2, 3, 1).half()
        got = sl(b)
        assert_exact("maxpool_s1", got, ref, f" (pool {i + 1})")
        prev = got   # the next pool reads the kernel's output, as in the plan


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c.name for c in UPSAMPLE_CASES])
def test_upsample2x_exact(name):
    c = next(c for c in UPSAMPLE_CASES if c.name == name)
    x = in_map(c.B, c.H, c.W, *c.x, c.C, sum(map(ord, c.name)), DEV)
    y, big = out_map(c.B, 2 * c.H, 2 * c.W, *c.y, c.C, DEV)
    extent(x); extent(y)
    ops.upsample2x(x, y)
    torch.cuda.synchronize()
    check_out(y, big)
    ref = sl(x).repeat_interleave(2, 1).repeat_interleave(2, 2)
    got = sl(y)
    assert torch.equal(_bits(got), _bits(ref))     # a copy: every bit, zeros' signs included


@pytest.mark.gpu
def test_elementwise_malformed_calls_are_rejected_before_launch():
    """every buffer is large enough for the call as written; the C side must still refuse each call before launching"""
    z = lambda B, H, W, C_: ops.Map(torch.zeros(B, H, W, C_, dtype=torch.float16, device=DEV), 0, C_)
    _rejected(lambda: ops.adown_pool(z(1, 5, 8, 32), z(1, 5, 8, 16), z(1, 3, 4, 16)), "H, W must be even")
    _rejected(lambda: ops.adown_pool(z(1, 8, 5, 32), z(1, 8, 5, 16), z(1, 4, 3, 16)), "H, W must be even")
    _rejected(lambda: ops.adown_pool(z(1, 8, 8, 24), z(1, 8, 8, 16), z(1, 4, 4, 16)), "C a multiple of 16")
    srcs = [z(1, 8 >> min(i, 3), 8 >> min(i, 3), 16) for i in range(6)]
    _rejected(lambda: ops.cbfuse(srcs, z(1, 8, 8, 16), z(1, 8, 8, 16)), "at most 5")
    _rejected(lambda: ops.cbfuse(srcs[1:2], ops.Map(z(1, 8, 8, 16).buf, 0, 12), z(1, 8, 8, 16)), "multiple of 8")
    _rejected(lambda: ops.maxpool_s1(ops.Map(z(1, 8, 8, 16).buf, 0, 12), z(1, 8, 8, 16), 5), "multiple of 8")
    _rejected(lambda: ops.upsample2x(ops.Map(z(1, 4, 4, 16).buf, 0, 12), z(1, 8, 8, 16)), "multiple of 8")


# ------------------------------------------------------------------------------------------------ stem im2col
def yolo_lut():
    return (np.arange(256, dtype=np.float32) / np.float32(255.0))[None].repeat(3, 0).copy()   # as YoloPlan builds it


def clip_lut():
    from omniparser_b200.florence_engine import IMAGENET_MEAN, IMAGENET_STD
    lut = np.empty((3, 256), np.float32)                                    # as FlorenceWeights builds it
    for c in range(3):
        lut[c] = (np.arange(256, dtype=np.float32) * np.float32(1.0 / 255.0) - np.float32(IMAGENET_MEAN[c])) / np.float32(IMAGENET_STD[c])
    return lut


@dataclass(frozen=True)
class Im2colCase:
    name: str
    B: int
    H: int
    W: int
    k: int
    s: int
    p: int
    Kpad: int
    lut: str      # "yolo" (/255) | "clip"
    split: int

    @property
    def Ho(self):
        return (self.H + 2 * self.p - self.k) // self.s + 1

    @property
    def Wo(self):
        return (self.W + 2 * self.p - self.k) // self.s + 1


IM2COL_CASES = [Im2colCase(f"{n}_split{sp}", B, H, W, k, s, p, Kp, lut, sp)
                for n, B, H, W, k, s, p, Kp, lut in (("yolo_b8_640", 8, 640, 640, 3, 2, 1, 32, "yolo"),
                                                     ("yolo_b1_1088x1920", 1, 1088, 1920, 3, 2, 1, 32, "yolo"),
                                                     ("davit_37_crops_64", 37, 64, 64, 7, 4, 3, 160, "clip"),
                                                     ("davit_b2_768", 2, 768, 768, 7, 4, 3, 160, "clip"))
                for sp in (0, 1)]


def im2col_launch(c: Im2colCase, dev):
    rows, width = c.B * c.Ho * c.Wo, c.Kpad * (2 if c.split else 1)
    if dev == "cpu":
        img, out = torch.empty(c.B, c.H, c.W, 3, dtype=torch.uint8), torch.empty(rows + 1, width, dtype=torch.float16)
    else:
        rng = np.random.default_rng(sum(map(ord, c.name)))
        img = torch.from_numpy(rng.integers(0, 256, size=(c.B, c.H, c.W, 3), dtype=np.uint8)).to(dev)
        out = torch.full((rows + 1, width), SENTINEL, dtype=torch.float16, device=dev)   # + one guard row
    lut = torch.from_numpy(yolo_lut() if c.lut == "yolo" else clip_lut()).to(dev)
    _covers(out, out.data_ptr(), rows * width)
    _covers(lut, lut.data_ptr(), 3 * 256)
    ops.im2col_u8(img, c.B, c.H, c.W, c.k, c.s, c.p, c.Kpad, lut, out, split=bool(c.split))
    return img, lut, out


def im2col_ref(c: Im2colCase, img, lut):
    """rows [tap-major (ky, kx), then channel]: hi = fp16(table value), lo = fp16(value - hi); 0 at padding taps and in
    the columns K..Kpad"""
    img, lut = img.cpu().long(), lut.cpu()
    v = torch.stack([lut[ch][img[..., ch]] for ch in range(3)], 1)            # [B, 3, H, W] fp32
    vp = F.pad(v, (c.p, c.p, c.p, c.p))
    taps = [vp[:, :, ky:ky + c.s * (c.Ho - 1) + 1:c.s, kx:kx + c.s * (c.Wo - 1) + 1:c.s] for ky in range(c.k) for kx in range(c.k)]
    cols = torch.stack(taps, -1).permute(0, 2, 3, 4, 1).reshape(c.B * c.Ho * c.Wo, c.k * c.k * 3)
    K = c.k * c.k * 3
    hi = torch.zeros(cols.shape[0], c.Kpad, dtype=torch.float16)
    lo = torch.zeros_like(hi)
    hi[:, :K] = cols.half()
    lo[:, :K] = (cols - hi[:, :K].float()).half()
    return hi, lo


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c.name for c in IM2COL_CASES])
def test_im2col_u8_exact(name):
    c = next(c for c in IM2COL_CASES if c.name == name)
    img, lut, out = im2col_launch(c, DEV)
    torch.cuda.synchronize()
    got = out.cpu()
    assert bool((got[-1] == SENTINEL).all()), "the guard row after the output was written"
    hi, lo = im2col_ref(c, img, lut)
    assert torch.equal(_bits(got[:-1, :c.Kpad]), _bits(hi)), f"hi: {int((_bits(got[:-1, :c.Kpad]) != _bits(hi)).sum())} differ"
    if c.split:
        assert bool((lo != 0).any())
        assert torch.equal(_bits(got[:-1, c.Kpad:]), _bits(lo)), f"lo: {int((_bits(got[:-1, c.Kpad:]) != _bits(lo)).sum())} differ"


# ------------------------------------------------------------------------------------------------ yolo_decode
BENCH_HW = ((80, 80), (40, 40), (20, 20))          # 640 x 640 canvas: A = 8400
FULL_HW = ((136, 240), (68, 120), (34, 60))        # 1088 x 1920 canvas: A = 42840
PLANT_LOGIT = -2.9444389                            # ~ logit(0.05); the planted anchors' kernel score becomes `conf`


@dataclass(frozen=True)
class DecodeCase:
    """conf None: conf := the kernel's own score of PLANT_LOGIT, planted at 1 % of the anchors (they must be dropped).
    shift[b]: per-image offset of the class logits (sets how many anchors pass)"""
    name: str
    B: int
    hw: tuple
    nc: int
    cap: int
    shift: tuple
    conf: float | None = None

    @property
    def A(self):
        return sum(h * w for h, w in self.hw)


DECODE_CASES = [
    DecodeCase("b8_640_nc1", 8, BENCH_HW, 1, 8400, (-4.0, -2.0, 0.0, 2.0, -6.0, -3.0, 1.0, -1.0)),
    # image 0: ~37000 candidates > cap; image 1: fewer than cap
    DecodeCase("b2_1088x1920_nc1_over_cap", 2, FULL_HW, 1, 16384, (1.5, -4.0), conf=0.25),
    DecodeCase("b3_640_nc3_class_ties", 3, BENCH_HW, 3, 8400, (-2.0, 0.0, -5.0)),
]

_PADS = ((0.0, 140.0, 0.33333334), (3.0, 0.0, 1.0062893), (295.0, 0.0, 2.1262460), (0.0, 108.0, 0.5),
         (17.0, 35.0, 0.75), (0.0, 0.0, 1.0), (64.0, 2.0, 0.2962963), (1.0, 295.0, 1.3333334))


@functools.lru_cache(maxsize=None)
def decode_inputs(name):
    c = next(c for c in DECODE_CASES if c.name == name)
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    cls, box, planted = [], [], []
    for h, w in c.hw:
        lg = torch.randn(c.B, h * w, c.nc, generator=g) * 2.5 + torch.tensor(c.shift).view(-1, 1, 1)
        r = torch.rand(c.B, h * w, generator=g)
        if c.nc > 1:   # exact class ties: 0 == 1, 1 == 2 (both the maximum), all three equal
            lg[r < 0.05, 1] = lg[r < 0.05, 0]
            m = (r >= 0.05) & (r < 0.1)
            lg[m, 1] = lg[m, 2] = lg[m].max(-1).values + 0.5
            m = (r >= 0.1) & (r < 0.13)
            lg[m, 1] = lg[m, 2] = lg[m, 0]
        pm = (r >= 0.5) & (r < 0.51) if c.conf is None else torch.zeros_like(r, dtype=torch.bool)
        lg[pm] = PLANT_LOGIT
        cls.append(lg.float().contiguous())
        box.append((torch.randn(c.B, h * w, 64, generator=g) * 3).contiguous())
        planted.append(pm)
    pads = torch.tensor([_PADS[b % len(_PADS)] for b in range(c.B)], dtype=torch.float32)
    return cls, box, torch.cat(planted, 1), pads


def decode_launch(c: DecodeCase, conf, dense, dev):
    """-> (candidate buffers, dense buffers); every buffer poisoned and followed by a guard image"""
    cls, box, _, pads = decode_inputs(c.name)
    mk = (lambda *s, dt=torch.float32: torch.empty(*s, dtype=dt)) if dev == "cpu" else \
        (lambda *s, dt=torch.float32: torch.full(s, SENTINEL if dt == torch.float32 else SENTINEL_I32, dtype=dt, device=dev))
    cls_d = [t.to(dev) for t in cls]
    box_d = [t.to(dev) for t in box]
    pl, pt, sc = (pads[:, i].contiguous().to(dev) for i in range(3))
    cand = dict(box=mk(c.B + 1, c.cap, 4), score=mk(c.B + 1, c.cap), cls=mk(c.B + 1, c.cap, dt=torch.int32),
                count=mk(c.B + 1, dt=torch.int32))
    dn = dict(ltrb=mk(c.B + 1, c.A, 4), score=mk(c.B + 1, c.A, c.nc)) if dense else dict(ltrb=None, score=None)
    for (h, w), t, u in zip(c.hw, cls_d, box_d):
        _covers(t, t.data_ptr(), c.B * h * w * c.nc)
        _covers(u, u.data_ptr(), c.B * h * w * 64)
    for t in (pl, pt, sc):
        _covers(t, t.data_ptr(), c.B)
    for k, n in (("box", 4 * c.cap), ("score", c.cap), ("cls", c.cap)):
        _covers(cand[k], cand[k].data_ptr(), c.B * n)
    _covers(cand["count"], cand["count"].data_ptr(), c.B)
    if dense:
        _covers(dn["ltrb"], dn["ltrb"].data_ptr(), c.B * c.A * 4)
        _covers(dn["score"], dn["score"].data_ptr(), c.B * c.A * c.nc)
    ops.yolo_decode(cls_d, box_d, list(c.hw), c.nc, c.B, float(conf), pl, pt, sc, c.cap, cand["box"], cand["score"],
                    cand["cls"], cand["count"], dn["ltrb"], dn["score"])
    return cand, dn


def _fp64_dense(c: DecodeCase):
    """fp64 sigmoid scores [B, A, nc], DFL expectations [B, A, 4] and each side's max |logit - max logit| [B, A, 4]"""
    cls, box, _, _ = decode_inputs(c.name)
    s = torch.sigmoid(torch.cat(cls, 1).double())
    bl = torch.cat(box, 1).double().view(c.B, c.A, 4, 16)
    d = bl - bl.max(-1, keepdim=True).values
    e = (torch.softmax(bl, -1) * torch.arange(16, dtype=torch.float64)).sum(-1)
    return s, e, d.abs().max(-1).values


U = 2.0 ** -24   # unit roundoff of fp32


def _restate_candidates(c: DecodeCase, ltrb, score, conf, pads):
    """the compaction ref:util/yolov9.py:123-129 applied to the kernel's own dense outputs (detect_post.cu:81-89 in
    numpy float32: no FMA, so this is exact) -> per image (boxes [n, 4], scores [n], classes [n])"""
    gx, gy, st = [], [], []
    for s, (h, w) in enumerate(c.hw):
        yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
        gx.append(xx.ravel()); gy.append(yy.ravel()); st.append(np.full(h * w, 8 << s))
    stride = np.concatenate(st).astype(f32)
    ax = (np.concatenate(gx).astype(f32) + f32(0.5)) * stride
    ay = (np.concatenate(gy).astype(f32) + f32(0.5)) * stride
    out = []
    for b in range(c.B):
        d = ltrb[b]
        sc = score[b]
        best, bc = sc.max(1), sc.argmax(1)              # argmax: the first maximum
        keep = best > f32(conf)
        x1, y1 = ax - d[:, 0] * stride, ay - d[:, 1] * stride
        x2, y2 = ax + d[:, 2] * stride, ay + d[:, 3] * stride
        pl, pt, s_ = (f32(v) for v in pads[b].tolist())
        bx = np.stack([(x1 - pl) / s_, (y1 - pt) / s_, (x2 - pl) / s_, (y2 - pt) / s_], 1).astype(f32)
        out.append((bx[keep], best[keep].astype(f32), bc[keep].astype(np.int32)))
    return out


def _i32(a):
    return np.ascontiguousarray(a).view(np.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c.name for c in DECODE_CASES])
def test_yolo_decode(name):
    c = next(c for c in DECODE_CASES if c.name == name)
    _, _, planted, pads = decode_inputs(name)
    conf = c.conf
    if conf is None:   # the kernel's own score of the planted logit becomes the threshold: those anchors sit exactly on it
        _, dn = decode_launch(c, 0.5, True, DEV)
        torch.cuda.synchronize()
        ps = dn["score"][:c.B].cpu()[planted]
        assert ps.numel() > 0 and bool((ps == ps[0]).all())
        conf = float(ps[0, 0])
    cand, dn = decode_launch(c, conf, True, DEV)
    torch.cuda.synchronize()
    ltrb, score = dn["ltrb"].cpu().numpy(), dn["score"].cpu().numpy()
    assert (ltrb[c.B] == SENTINEL).all() and (score[c.B] == SENTINEL).all(), "dense outputs: guard image written"
    ltrb, score = ltrb[:c.B], score[:c.B]

    # (a) dense outputs against fp64.  sigmoid: expf (<= 2 ulp), 1 + e, 1 / (.) -> relative 2^-22 + 2^-23.  DFL: each
    # exp has relative error <= |d| u + 2^-22 (d = logit - max, rounded once), the 16-term sum adds 15 u, the quotient
    # and the product u each, the expectation's 15 additions 15 u (all terms >= 0): relative 2 max_eps + 32 u.
    s64, e64, dmax = _fp64_dense(c)
    eps_s = (4 * U + 2 * U) * 1.001
    r_s = ((torch.from_numpy(score).double() - s64).abs() / (s64 * eps_s)).max().item()
    eps_e = (2 * (dmax * U + 4 * U) + 32 * U) * 1.001
    r_e = ((torch.from_numpy(ltrb).double() - e64).abs() / (e64 * eps_e).clamp_min(1e-300)).max().item()
    print(f"{name}: dense error / bound: sigmoid {r_s:.3f}, DFL {r_e:.3f}")
    assert r_s <= 1 and r_e <= 1, (r_s, r_e)

    # (b) + (c): candidates == the order-preserving compaction of the kernel's dense outputs under score > conf
    exp = _restate_candidates(c, ltrb, score, conf, pads)
    cb, cs, cc = cand["box"].cpu().numpy(), cand["score"].cpu().numpy(), cand["cls"].cpu().numpy()
    cn = cand["count"].cpu().numpy()
    assert cn[c.B] == SENTINEL_I32 and (cb[c.B] == SENTINEL).all() and (cs[c.B] == SENTINEL).all() and (cc[c.B] == SENTINEL_I32).all()
    for b, (eb, es, ec) in enumerate(exp):
        n, k = len(es), min(len(es), c.cap)
        assert cn[b] == n, (b, cn[b], n)                                       # (e) the true total, also above cap
        assert np.array_equal(_i32(cb[b, :k]), _i32(eb[:k])), f"image {b}: candidate boxes differ"
        assert np.array_equal(_i32(cs[b, :k]), _i32(es[:k])), f"image {b}: candidate scores differ"
        assert np.array_equal(cc[b, :k], ec[:k]), f"image {b}: candidate classes differ"
        assert (cb[b, k:] == SENTINEL).all() and (cs[b, k:] == SENTINEL).all() and (cc[b, k:] == SENTINEL_I32).all()
    if c.conf is None:
        on = score[planted.numpy()].max(-1)
        assert on.size and (on == f32(conf)).all()                              # planted anchors sit exactly on conf
    if c.nc > 1:   # the class ties are real: anchors whose maximum is shared, some of them candidates
        top = score.max(-1, keepdims=True)
        shared = ((score == top).sum(-1) > 1) & (top[..., 0] > f32(conf))
        assert shared.sum() > 100 and (score.argmax(-1)[shared] < c.nc - 1).all()
    if c.cap < c.A:
        assert cn[0] > c.cap and cn[1] < c.cap

    # (d) the production launch (no dense outputs) writes the same candidates, bit for bit
    cand2, _ = decode_launch(c, conf, False, DEV)
    torch.cuda.synchronize()
    for k in cand:
        assert torch.equal(_bits(cand2[k].cpu()), _bits(cand[k].cpu())), k


# ------------------------------------------------------------------------------------------------ batched_nms
NMS_THRS = (0.1, 0.5, 0.7)
NMS_MAX_DETS = (1, 300, 1024)
NMS_NC = 3
NMS_CAPS = (8400, 16384)       # the bench geometry's cap (= A) and the candidate capacity of larger canvases


def nms_counts(cap):
    """one image per path: empty, one box, coordinate trick (<= 1000 boxes, also exactly 1000), per-class (1001 and
    more), a full list, and a count above cap (the kernel clamps it)"""
    return (0, 1, 777, 1000, 1001, 5040, cap, cap + 500)


def _thr_float(thr):
    """T = the largest float <= thr (the kernel's threshold) and the next float above it"""
    t = f32(thr)
    if float(t) > thr:
        t = np.nextafter(t, f32(-np.inf))
    return t, np.nextafter(t, f32(np.inf))


def _ovr(p, q):
    """torchvision's IoU in fp32 (and the kernel's iou_gt), p one box, q [..., 4]"""
    w = np.maximum(f32(0), np.minimum(p[2], q[..., 2]) - np.maximum(p[0], q[..., 0]))
    h = np.maximum(f32(0), np.minimum(p[3], q[..., 3]) - np.maximum(p[1], q[..., 1]))
    inter = w * h
    pa = (p[2] - p[0]) * (p[3] - p[1])
    qa = (q[..., 2] - q[..., 0]) * (q[..., 3] - q[..., 1])
    with np.errstate(invalid="ignore", divide="ignore"):
        return inter / ((pa + qa) - inter)


@functools.lru_cache(maxsize=None)
def exact_iou_pair(target, slot):
    """two 4x4-ish boxes below the image (y < -250, where nothing else lies) whose fp32 IoU is exactly `target`"""
    target = f32(target)
    for j in range(64):
        x0, y0 = f32(-40 + 12 * ((slot * 64 + j) % 150)), f32(-300 - 10 * slot)
        p = np.array([x0, y0, x0 + 4, y0 + 4], f32)
        dx0 = 4 * (1 - float(target)) / (1 + float(target))
        u = np.spacing(f32(abs(x0) + 8))
        X = (x0 + f32(dx0)) + np.arange(-64, 64, dtype=f32)[:, None, None] * u
        Hh = f32(4) - np.arange(0, 48, dtype=f32)[None, :, None] * u
        E = f32(4) + np.arange(-24, 24, dtype=f32)[None, None, :] * u
        X, Hh, E = np.broadcast_arrays(X, Hh, E)
        q = np.stack([X, np.full_like(X, y0), X + E, y0 + Hh], -1).astype(f32)
        hit = np.argwhere(_ovr(p, q) == target)
        if len(hit):
            return p, q[tuple(hit[0])]
    raise AssertionError(f"no box pair with IoU exactly {target!r}")


@functools.lru_cache(maxsize=None)
def nms_image(n, seed):
    """n candidates (boxes [n, 4] fp32, scores [n] fp32, classes [n] int32) in candidate-index order:
    * random boxes over x in [-60, 2120], y in [-60, 1270] (negative and out-of-image coordinates), 3 % zero-area,
      3 classes, scores uniform in (0.05, 0.39);
    * up to 150 higher scores, 20 exact ties at 0.5 / 0.75, n/10 exact ties at 0.25 / 0.3, a run of 30 saturated 1.0;
    * n >= 1000: 400 non-overlapping boxes (x >= 2200) tied at 0.4 -- fewer than 300 boxes outrank them, so a
      max_det = 300 cut falls inside that run;
    * n >= 40: for each thr, a pair whose IoU is exactly T (kept) and one whose IoU is the next float (suppressed).
    All planted structures sit at random candidate indices."""
    rng = np.random.default_rng(seed)
    xy = np.stack([rng.uniform(-60, 1900, n), rng.uniform(-60, 1050, n)], 1).astype(f32)
    wh = rng.uniform(0, 220, (n, 2)).astype(f32)
    za = rng.random(n) < 0.03
    wh[za, rng.integers(0, 2, n)[za]] = 0
    boxes = np.concatenate([xy, xy + wh], 1).astype(f32)
    cls = rng.integers(0, NMS_NC, n).astype(np.int32)
    scores = rng.uniform(0.05, 0.39, n).astype(f32)
    order = rng.permutation(n)
    pos = [0]

    def take(k):
        s = order[pos[0]:pos[0] + k]
        pos[0] += len(s)
        return s
    s = take(min(150, n // 6)); scores[s] = rng.uniform(0.41, 0.98, len(s))
    s = take(min(20, n // 10)); scores[s] = rng.choice(f32([0.5, 0.75]), len(s))
    s = take(n // 10); scores[s] = rng.choice(f32([0.25, 0.3]), len(s))
    s = take(min(30, n // 10)); scores[s] = 1.0
    if n >= 1000:
        s = take(400)
        j = np.arange(400)
        gx, gy = f32(2200) + (j % 20).astype(f32) * 40, f32(-200) + (j // 20).astype(f32) * 40
        boxes[s] = np.stack([gx, gy, gx + 30, gy + 30], 1)
        scores[s] = 0.4
    pairs = {}
    if n >= 40:
        for ti, thr in enumerate(NMS_THRS):
            for kind, target in enumerate(_thr_float(thr)):
                slot = 2 * ti + kind
                p, q = exact_iou_pair(float(target), slot)
                s = take(2)
                boxes[s[0]], boxes[s[1]] = p, q
                scores[s[0]], scores[s[1]] = f32(0.99) - f32(0.002) * slot, f32(0.989) - f32(0.002) * slot
                cls[s] = 0
                pairs[(thr, kind)] = (int(s[0]), int(s[1]))
    return boxes, scores, cls, pairs


@functools.lru_cache(maxsize=None)
def nms_data(cap):
    counts = nms_counts(cap)
    imgs = [nms_image(min(n, cap), 1000 * b + n) for b, n in enumerate(counts)]
    wh = [(1920.0 - 37 * b, 1080.0 + 23 * b) for b in range(len(counts))]
    return counts, imgs, wh


@functools.lru_cache(maxsize=None)
def nms_reference(cap, thr):
    """per image: the documented rule over the first min(count, cap) candidates (max_det 1024; smaller max_det are its
    prefixes), and torchvision's full batched_nms"""
    from torchvision.ops import batched_nms
    counts, imgs, _ = nms_data(cap)
    out = []
    for (boxes, scores, cls, _) in imgs:
        ref = R.greedy_nms_numpy(boxes, scores, cls, thr, 1024)
        tv = batched_nms(torch.from_numpy(boxes), torch.from_numpy(scores), torch.from_numpy(cls).long(), thr).numpy()
        out.append((ref, tv))
    return out


NMS_CASES = [(cap, thr) for cap in NMS_CAPS for thr in NMS_THRS]


def nms_launch(cap, thr, max_det, dev):
    counts, imgs, wh = nms_data(cap)
    B = len(counts)
    box = np.zeros((B, cap, 4), f32)
    score = np.zeros((B, cap), f32)
    cls = np.zeros((B, cap), np.int32)
    for b, (bx, sc, cl, _) in enumerate(imgs):
        box[b, :len(sc)], score[b, :len(sc)], cls[b, :len(sc)] = bx, sc, cl
    d = lambda a: torch.from_numpy(a).to(dev)
    mk = (lambda *s, dt=torch.float32: torch.empty(*s, dtype=dt)) if dev == "cpu" else \
        (lambda *s, dt=torch.float32: torch.full(s, SENTINEL if dt == torch.float32 else SENTINEL_I32, dtype=dt, device=dev))
    ins = dict(box=d(box), score=d(score), cls=d(cls), count=d(np.asarray(counts, np.int32)),
               img_w=d(np.asarray([w for w, _ in wh], f32)), img_h=d(np.asarray([h for _, h in wh], f32)))
    outs = dict(keep=mk(B + 1, max_det, dt=torch.int32), box=mk(B + 1, max_det, 4), score=mk(B + 1, max_det),
                count=mk(B + 1, dt=torch.int32))
    for k, n in (("box", 4 * cap), ("score", cap), ("cls", cap)):
        _covers(ins[k], ins[k].data_ptr(), B * n)
    for k in ("count", "img_w", "img_h"):
        _covers(ins[k], ins[k].data_ptr(), B)
    for k, n in (("keep", max_det), ("box", 4 * max_det), ("score", max_det)):
        _covers(outs[k], outs[k].data_ptr(), B * n)
    ops.batched_nms(ins["box"], ins["score"], ins["cls"], ins["count"], B, cap, thr, max_det, ins["img_w"], ins["img_h"],
                    outs["keep"], outs["box"], outs["score"], outs["count"])
    return outs


def _runs(s):
    """[(start, end)) runs of equal values in a score sequence"""
    cut = [0] + [i for i in range(1, len(s)) if s[i] != s[i - 1]] + [len(s)]
    return list(zip(cut[:-1], cut[1:]))


@pytest.mark.gpu
@pytest.mark.parametrize("cap,thr", NMS_CASES)
def test_batched_nms(cap, thr):
    counts, imgs, wh = nms_data(cap)
    refs = nms_reference(cap, thr)
    T, T_next = _thr_float(thr)
    tv_reordered = 0
    for max_det in NMS_MAX_DETS:
        o = nms_launch(cap, thr, max_det, DEV)
        torch.cuda.synchronize()
        keep, ob, os_, oc = (o[k].cpu().numpy() for k in ("keep", "box", "score", "count"))
        B = len(counts)
        assert oc[B] == SENTINEL_I32 and (keep[B] == SENTINEL_I32).all() and (ob[B] == SENTINEL).all() and (os_[B] == SENTINEL).all()
        for b, ((boxes, scores, cls, pairs), (ref, tv)) in enumerate(zip(imgs, refs)):
            r = ref[:max_det]
            k = len(r)
            assert oc[b] == k, (b, max_det, oc[b], k)
            assert np.array_equal(keep[b, :k], r.astype(np.int32)), f"image {b} (count {counts[b]}), max_det {max_det}: kept order differs"
            W, H = wh[b]
            eb = boxes[r].copy()
            eb[:, [0, 2]] = np.minimum(np.maximum(eb[:, [0, 2]], f32(0)), f32(W))
            eb[:, [1, 3]] = np.minimum(np.maximum(eb[:, [1, 3]], f32(0)), f32(H))
            assert np.array_equal(_i32(ob[b, :k]), _i32(eb)) and np.array_equal(_i32(os_[b, :k]), _i32(scores[r]))
            assert (keep[b, k:] == SENTINEL_I32).all() and (ob[b, k:] == SENTINEL).all() and (os_[b, k:] == SENTINEL).all()
            # torchvision: the same scores position by position; the same indices inside every run of equal scores
            # (the last run may be cut by max_det: a subset of torchvision's run); identical where nothing is tied
            assert np.array_equal(scores[tv[:k]], scores[r])
            for s0, s1 in _runs(scores[r]):
                mine, theirs = set(r[s0:s1].tolist()), set(tv[s0:s1].tolist())
                if s1 < k or len(tv) == k:
                    assert mine == theirs, (b, s0, s1)
                else:
                    assert mine <= set(tv[scores[tv] == scores[r[s0]]].tolist())
            tv_reordered += int(not np.array_equal(tv[:k], r))
            # the planted structures are where the case says they are
            if max_det == 1024 and pairs:
                kept = set(r.tolist())
                p, q = pairs[(thr, 0)]
                assert p in kept and q in kept, "IoU == T must not suppress"
                p, q = pairs[(thr, 1)]
                assert p in kept and q not in kept, "IoU == nextafter(T) must suppress"
            if max_det == 300 and len(scores) >= 1000:
                full = ref
                assert len(full) > 300 and scores[full[299]] == scores[full[300]] == f32(0.4), "the cut is not inside the tied run"
    print(f"cap {cap}, thr {thr}: {tv_reordered} kept lists that torchvision orders differently inside tied runs")


@pytest.mark.gpu
def test_batched_nms_rejections():
    """max_det > 1024 and cap > 16384 are refused before anything launches (count 0, so even a launch would not read)"""
    z = lambda *s, dt=torch.float32: torch.zeros(s, dtype=dt, device=DEV)
    cap = 16385
    box, score, cls, cnt = z(cap, 4), z(cap), z(cap, dt=torch.int32), z(1, dt=torch.int32)
    wh = torch.ones(1, device=DEV)
    _rejected(lambda: ops.batched_nms(box, score, cls, cnt, 1, 1024, 0.5, 1025, wh, wh, z(1025, dt=torch.int32), z(1025, 4),
                                      z(1025), z(1, dt=torch.int32)), "max_det > 1024")
    _rejected(lambda: ops.batched_nms(box, score, cls, cnt, 1, cap, 0.5, 300, wh, wh, z(300, dt=torch.int32), z(300, 4), z(300),
                                      z(1, dt=torch.int32)), "capacity > 16384")


# ------------------------------------------------------------------------------------------------ CPU: plan coverage
def classify(name, a):
    """every argument of a recorded non-GEMM call except pointers and the stream: geometry, pitches, NS, flags"""
    if name == "b2p_cbfuse":
        ns = a[0]
        return (name, ns, tuple(a[2])[:ns], tuple(a[3])[:ns], *a[5:10], a[11])
    types = _lib.PROTOTYPES[name][1]
    return (name,) + tuple(v for v, t in zip(a, types) if t is not C.c_void_p)


def _record_cases(rec):  # noqa: F811
    for c in ADOWN_CASES:
        adown_launch(c, "cpu")
    for c in CBFUSE_CASES:
        cbfuse_launch(c, "cpu")
    for c in MAXPOOL_CASES:
        for i in range(3):
            buf = torch.empty(c.B, c.H, c.W, c.x[0], dtype=torch.float16)
            ops.maxpool_s1(ops.Map(buf, c.C * i, c.C), ops.Map(buf, c.C * (i + 1), c.C), 5)
    for c in UPSAMPLE_CASES:
        ops.upsample2x(in_map(c.B, c.H, c.W, *c.x, c.C, 0, "cpu"), out_map(c.B, 2 * c.H, 2 * c.W, *c.y, c.C, "cpu")[0])
    for c in IM2COL_CASES:
        im2col_launch(c, "cpu")


def test_cases_cover_every_non_gemm_call_of_the_fast_plan(rec):  # noqa: F811
    """Record the fast plan at the bench geometry and at a 1088x1920 canvas; every non-GEMM call (kernel, geometry,
    pitches, NS, shifts) must be launched by a case above.  Decode / NMS: the candidate count A, the capacity and the
    NMS sort size of both geometries must each appear in a case."""
    from omniparser_b200.detector import B200YOLOv9Detector
    from omniparser_b200.yolo_engine import YoloPlan, YoloWeights
    from standin.yolo_weights import yolo_standin
    w = YoloWeights(yolo_standin(0).state_dict(), torch.device("cpu"))
    plan_calls, geoms = set(), set()
    for B, Hc, Wc in ((8, 640, 640), (1, 1088, 1920)):
        plan = YoloPlan(w, B, Hc, Wc, use_graph=False)
        plan.run()
        plan_calls |= {classify(n, a) for n, a in rec.calls if n not in ("b2p_gemm", "b2p_conv3x3")}
        rec.calls.clear()
        A = sum(h * wd for h, wd in plan.hw)
        cap = min(B200YOLOv9Detector.CAND_CAP, A)
        geoms.add((tuple(plan.hw), A, cap, 1 << max(1, (cap - 1).bit_length())))
    kinds = {k[0] for k in plan_calls}
    assert kinds == {"b2p_im2col_u8", "b2p_adown_pool", "b2p_cbfuse", "b2p_maxpool_s1", "b2p_upsample2x"}, kinds
    assert {k[1] for k in plan_calls if k[0] == "b2p_cbfuse"} == {1, 2, 3, 4, 5}
    _record_cases(rec)
    have = {classify(n, a) for n, a in rec.calls}
    missing = sorted(plan_calls - have, key=str)
    assert not missing, "non-GEMM calls of the fast plan without a case in this module:\n" + "\n".join(map(str, missing))
    assert ("b2p_cbfuse", 0) in {k[:2] for k in have}
    for hw, A, cap, sort_cap in geoms:
        assert any(c.hw == hw and c.A == A and c.cap == cap for c in DECODE_CASES), (hw, A, cap)
        assert cap in NMS_CAPS and any(1 << max(1, (cp - 1).bit_length()) == sort_cap for cp in NMS_CAPS), (cap, sort_cap)
    assert any(c.cap < c.A for c in DECODE_CASES) and any(c.nc > 1 for c in DECODE_CASES)
