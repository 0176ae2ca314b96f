"""Parity-grade (fp16x3) detector kernels against fp64, at the precision they promise.

With precision="fp16x3" every detector feature map is an fp16 hi/lo pair (pixel layout [hi(Ctot) | lo(Ctot)], ~22
significant bits) and every conv issues hi*hi + hi*lo + lo*hi.  A kernel that loses a lo plane is off by up to 2^-12 of
each value, which the end-to-end parity tests (bounds at fp16 rounding level) cannot see.  This module pins the
`_planes` / `_x3` entry points one by one:

* GEMM / conv cases (the shapes the parity plan issues at a 384x640 canvas) against an fp64 reference within 2e-5
  relative, plus a poison/guard check of every output buffer and a canonical-pair check of every fp16 pair output;
* the elementwise x3 kernels (ADown pooling, SPPELAN max-pool, upsample, CBFuse) bit for bit, both planes, against a
  CPU float32 restatement in the kernel's association order;
* host-side rejections of malformed lo-plane arguments;
* on the CPU: that every tolerance would catch a dropped lo plane (sensitivity), and that every class of `_planes` /
  `_x3` call the parity plan issues has a case here (coverage).

Every launch covers its operands with torch allocations (checked before the call, see ``_check_extents``) and runs on
the current stream of one process."""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

from omniparser_b200 import _lib, ops
from test_plan_dryrun_cpu import rec  # noqa: F401  (fixture: the C library replaced by an argument-checking recorder)

DEV = "cuda:0"
SENTINEL = -1234.0          # finite, exactly representable in fp16 and fp32, never a legitimate output here
TOL = 2e-5                  # relative to max(1, |ref|.max()): the bound of the existing fp16x3 operand tests
SENSITIVITY = 4.0           # a dropped lo plane must move the result by more than this many tolerances


# ------------------------------------------------------------------------------------------------ shared helpers
def pair(v32):
    """fp32 values -> canonical fp16 pair (hi = fp16(v), lo = fp16(v - hi))."""
    hi = v32.half()
    return hi, (v32 - hi.float()).half()


def pair_value(hi, lo):
    return hi.double() + lo.double()


def pair_map(v32, Ctot, c0, gen):
    """[B, H, W, C] fp32 values as hi/lo pairs in channels [c0, c0 + C) of a [hi(Ctot) | lo(Ctot)] buffer.  The guard
    channels on both sides of the slice, in both planes, hold random values, so reading the wrong columns shows."""
    B, H, W, C_ = v32.shape
    assert 0 <= c0 and c0 + C_ <= Ctot and Ctot % 8 == 0
    buf = (torch.randn(B, H, W, 2 * Ctot, generator=gen) * 4).half()
    hi, lo = pair(v32)
    buf[..., c0:c0 + C_] = hi
    buf[..., Ctot + c0:Ctot + c0 + C_] = lo
    return ops.Map(buf, c0, C_, lo=Ctot)


def planes(m: ops.Map):
    """(hi, lo) of a pair map's slice; lo is None for a plain map"""
    hi = m.buf[..., m.c0:m.c0 + m.C]
    return hi, (m.buf[..., m.lo + m.c0:m.lo + m.c0 + m.C] if m.lo else None)


def poisoned_map(B, H, W, Ctot, c0, C_, dev, x3=True, dtype=torch.float16):
    buf = torch.full((B, H, W, (2 if x3 else 1) * Ctot), SENTINEL, dtype=dtype, device=dev)
    return ops.Map(buf, c0, C_, lo=Ctot if x3 else 0)


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def check_poison(m: ops.Map):
    """Everything outside the written slice still holds the sentinel (bit for bit, both planes) and nothing inside does:
    a lo plane written at the wrong offset, or not at all, fails here."""
    mask = torch.zeros(m.ld, dtype=torch.bool)
    mask[m.c0:m.c0 + m.C] = True
    if m.lo:
        mask[m.lo + m.c0:m.lo + m.c0 + m.C] = True
    b = _bits(m.buf.cpu())
    s = _bits(torch.tensor([SENTINEL], dtype=m.buf.dtype))[0]
    outside, inside = b[..., ~mask], b[..., mask]
    assert bool((outside == s).all()), f"{int((outside != s).sum())} elements outside the output slice were written"
    assert not bool((inside == s).any()), f"{int((inside == s).sum())} elements of the output slice were not written"


def check_canonical(hi, lo):
    """hi == fp16(hi + lo) and |lo| <= ulp(hi)/2.  The kernels round t to hi, then t - hi to lo; when t - hi lies just
    below ulp/2 its rounding can reach ulp/2 exactly, and hi + lo is then a tie that fp16 rounds to the even neighbour:
    such an exact tie is the one allowed exception to the first condition."""
    hd, ld_ = hi.double(), lo.double()
    assert bool(torch.isfinite(hd).all() and torch.isfinite(ld_).all())
    _, e = torch.frexp(hd)
    ulp = torch.where(hd == 0, torch.full_like(hd, 2.0 ** -24), torch.ldexp(torch.ones_like(hd), (e - 1).clamp(min=-14) - 10))
    half_ulp = ulp / 2
    assert bool((ld_.abs() <= half_ulp).all()), f"max |lo| / ulp(hi) = {float((ld_.abs() / ulp).max())}"
    rounds_back = (hd + ld_).half() == hi
    tie = ld_.abs() == half_ulp
    assert bool((rounds_back | tie).all()), f"{int((~(rounds_back | tie)).sum())} pairs do not round back to hi"


def _covers(t, ptr, n_elems):
    """the allocation of `t` covers n_elems elements (of t's dtype) from address ptr"""
    assert t.is_contiguous()
    es = t.element_size()
    lo_, hi_ = t.data_ptr(), t.data_ptr() + t.numel() * es
    assert lo_ <= ptr and ptr + n_elems * es <= hi_, ("tensor map would address outside the allocation", ptr - lo_,
                                                       n_elems * es, hi_ - lo_)


# ------------------------------------------------------------------------------------------------ GEMM / conv cases
@dataclass(frozen=True)
class Case:
    """one `_planes` launch: A (Ctot, c0) channel slice of a pair map; out (Ctot, c0) of a pair map, or None = a whole
    fp32 map; res (Ctot, c0) of a pair map or None"""
    name: str
    op: str                  # "gemm" (conv1x1) | "conv" (3x3 pad 1)
    stride: int
    B: int
    H: int
    W: int
    cin: int
    cout: int
    a: tuple
    out: tuple | None
    res: tuple | None = None
    act: int = ops.ACT_SILU
    adown_x1: bool = False   # input is an ADown x1 map: last row and column zero

    @property
    def Ho(self):
        return self.H // self.stride

    @property
    def Wo(self):
        return self.W // self.stride


CASES = [
    # conv1x1 (b2p_gemm_planes)
    Case("stem_k32_multiwave", "gemm", 1, 1, 192, 320, 32, 128, a=(32, 0), out=(128, 0)),
    Case("x1_slice_k64_multiwave", "gemm", 1, 1, 192, 320, 64, 64, a=(128, 0), out=(64, 0), act=ops.ACT_NONE),
    Case("elan_input_slice", "gemm", 1, 1, 48, 80, 128, 128, a=(512, 128), out=(384, 128)),
    Case("k1024_n512_splitk", "gemm", 1, 1, 12, 20, 1024, 512, a=(1024, 0), out=(1024, 512)),
    Case("head_box_f32_n64", "gemm", 1, 1, 48, 80, 64, 64, a=(64, 0), out=None, act=ops.ACT_NONE),
    Case("head_cls_f32_n1", "gemm", 1, 1, 24, 40, 256, 1, a=(256, 0), out=None, act=ops.ACT_NONE),
    # N % 16 != 0 and an output pointer that is only 8-byte aligned: the scalar epilogue, split store and residual pair
    Case("n24_scalar_split_res", "gemm", 1, 1, 24, 40, 64, 24, a=(96, 32), out=(40, 4), res=(32, 8)),
    # 3x3 stride 1 (b2p_conv3x3_planes, mode 1 per-tap TMA: the halo path is off for fp16x3 operands)
    Case("s1_cin32_res", "conv", 1, 1, 96, 160, 32, 32, a=(32, 0), out=(64, 32), res=(64, 0)),
    Case("s1_cin32_input_slice", "conv", 1, 1, 96, 160, 32, 32, a=(64, 0), out=(32, 0)),
    Case("s1_cin32_n64", "conv", 1, 2, 12, 20, 32, 64, a=(32, 0), out=(64, 0)),
    Case("s1_cin128", "conv", 1, 1, 24, 40, 128, 128, a=(128, 0), out=(128, 0)),
    Case("s1_cin64_slice_res", "conv", 1, 1, 48, 80, 64, 64, a=(192, 64), out=(160, 32), res=(128, 64)),
    Case("s1_cin256_res_splitk", "conv", 1, 1, 12, 20, 256, 256, a=(256, 0), out=(256, 0), res=(512, 256)),
    Case("s1_cin256_odd_slice", "conv", 1, 2, 13, 21, 256, 256, a=(320, 64), out=(256, 0)),
    # 3x3 stride 2 (parity view)
    Case("s2_adown_x1", "conv", 2, 1, 96, 160, 128, 128, a=(128, 0), out=(256, 0), adown_x1=True),
    Case("s2_cin512_slice_splitk", "conv", 2, 1, 24, 40, 512, 512, a=(640, 64), out=(1024, 0)),
]
CASE_IDS = [c.name for c in CASES]


@functools.lru_cache(maxsize=None)
def case_data(name):
    """seeded fp32 operands of a case, split into pairs and placed in their (CPU) buffers"""
    c = next(c for c in CASES if c.name == name)
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    k = 1 if c.op == "gemm" else 3
    a32 = torch.randn(c.B, c.H, c.W, c.cin, generator=g)
    if c.adown_x1:
        a32[:, -1] = 0
        a32[:, :, -1] = 0
    w32 = torch.randn(c.cout, c.cin, k, k, generator=g) / math.sqrt(k * k * c.cin)
    whi, wlo = pair(w32.permute(0, 2, 3, 1))                           # [Co, ky, kx, Ci]
    wpk = torch.cat([whi, wlo], 3).reshape(c.cout, -1).contiguous()   # [Co][tap][hi(Ci) | lo(Ci)]
    bias = torch.randn(c.cout, generator=g) * 0.5
    x = pair_map(a32, c.a[0], c.a[1], g)
    res = pair_map(torch.randn(c.B, c.Ho, c.Wo, c.cout, generator=g), c.res[0], c.res[1], g) if c.res else None
    return dict(x=x, w=(whi, wlo), wpk=wpk, bias=bias, res=res)


def reference(c: Case, a_lo=True, w_lo=True, res_lo=True):
    """fp64 [B, Ho, Wo, N]: act(A @ W^T + bias) + res, each operand the exact value of its pair (or its hi half only)"""
    d = case_data(c.name)
    ah, al = planes(d["x"])
    a = ah.double() + (al.double() if a_lo else 0)
    whi, wlo = d["w"]
    w = (whi.double() + (wlo.double() if w_lo else 0)).permute(0, 3, 1, 2)
    z = F.conv2d(a.permute(0, 3, 1, 2), w, d["bias"].double(), stride=c.stride, padding=1 if c.op == "conv" else 0)
    z = z.permute(0, 2, 3, 1)
    if c.act == ops.ACT_SILU:
        z = F.silu(z)
    if d["res"] is not None:
        rh, rl = planes(d["res"])
        z = z + rh.double() + (rl.double() if res_lo else 0)
    return z


@functools.lru_cache(maxsize=None)
def reference_full(name):
    return reference(next(c for c in CASES if c.name == name))


def tolerance(ref):
    return TOL * max(1.0, ref.abs().max().item())


def _check_extents(c: Case, x, wpk, out, bias, res):
    """every element the C side's tensor maps / epilogue can address lies inside the torch allocations"""
    Mo = c.B * c.Ho * c.Wo
    span = x.lo + c.cin                                   # columns of A the tensor map covers
    if c.op == "gemm" or c.stride == 1:
        _covers(x.buf, x.ptr, (c.B * c.H * c.W - 1) * x.ld + span)
    else:                                                 # parity view: (pixel pair, ld + span) boxes
        pairs = c.B * c.H * c.W // 2
        _covers(x.buf, x.ptr, (pairs - 1) * 2 * x.ld + x.ld + span)
    _covers(wpk, wpk.data_ptr(), c.cout * wpk.shape[1])
    assert wpk.shape[1] == 2 * c.cin * (1 if c.op == "gemm" else 9)
    _covers(bias, bias.data_ptr(), c.cout)
    _covers(out.buf, out.ptr, (Mo - 1) * out.ld + out.lo + c.cout)
    if res is not None:
        _covers(res.buf, res.ptr, (Mo - 1) * res.ld + res.lo + c.cout)


def launch(c: Case, dev):
    """build the case's device buffers (outputs poisoned), check their extents, launch through ops; -> output map"""
    d = case_data(c.name)
    x = ops.Map(d["x"].buf.to(dev), d["x"].c0, d["x"].C, d["x"].lo)
    res = ops.Map(d["res"].buf.to(dev), d["res"].c0, d["res"].C, d["res"].lo) if d["res"] is not None else None
    wpk, bias = d["wpk"].to(dev), d["bias"].to(dev)
    if c.out is None:
        out = poisoned_map(c.B, c.Ho, c.Wo, c.cout, 0, c.cout, dev, x3=False, dtype=torch.float32)
    else:
        out = poisoned_map(c.B, c.Ho, c.Wo, c.out[0], c.out[1], c.cout, dev)
    _check_extents(c, x, wpk, out, bias, res)
    if c.op == "gemm":
        ops.conv1x1(x, wpk, out, bias, res, c.act, out_f32=c.out is None)
    else:
        ops.conv3x3(x, wpk, out, c.stride, bias, res, c.act, out_f32=c.out is None)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_IDS)
def test_planes_vs_fp64(name):
    c = next(c for c in CASES if c.name == name)
    out = launch(c, DEV)
    torch.cuda.synchronize()
    check_poison(out)
    hi, lo = planes(out)
    hi, lo = hi.cpu(), (lo.cpu() if lo is not None else None)
    if lo is not None:
        check_canonical(hi, lo)
        got = pair_value(hi, lo)
    else:
        got = hi.double()
    ref = reference_full(name)
    err, tol = (got - ref).abs().max().item(), tolerance(ref)
    assert err < tol, f"{name}: max abs err {err:.3g} > {tol:.3g}"


# ------------------------------------------------------------------------------------------------ elementwise x3 kernels
def _resplit(v):
    """the kernels' stf8: fp32 value -> (fp16(v), fp16(v - hi))"""
    hi = v.half()
    return hi, (v - hi.float()).half()


def _fp32(m: ops.Map):
    """[B, H, W, C] fp32 hi + lo (the kernels' ldf8: exact for canonical pairs)"""
    hi, lo = planes(m)
    return hi.float() + lo.float()


def _to(m: ops.Map, dev):
    return ops.Map(m.buf.to(dev), m.c0, m.C, m.lo)


def _assert_planes_equal(m: ops.Map, hi_ref, lo_ref):
    check_poison(m)
    hi, lo = (t.cpu() for t in planes(m))
    assert torch.equal(_bits(hi), _bits(hi_ref)), f"hi plane: {int((_bits(hi) != _bits(hi_ref)).sum())} elements differ"
    assert torch.equal(_bits(lo), _bits(lo_ref)), f"lo plane: {int((_bits(lo) != _bits(lo_ref)).sum())} elements differ"


def _extent_map(m: ops.Map):
    _covers(m.buf, m.ptr, (m.B * m.H * m.W - 1) * m.ld + m.lo + m.C)


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(24, 40), (4, 6)])
def test_adown_pool_x3_bit_exact(H, W):
    g = torch.Generator().manual_seed(H * W)
    B, C_ = 2, 256
    x = pair_map(torch.randn(B, H, W, C_, generator=g), 384, 64, g)
    xd = _to(x, DEV)
    x1 = poisoned_map(B, H, W, 160, 16, C_ // 2, DEV)
    x2 = poisoned_map(B, H // 2, W // 2, 144, 8, C_ // 2, DEV)
    for m in (xd, x1, x2):
        _extent_map(m)
    ops.adown_pool(xd, x1, x2)
    torch.cuda.synchronize()
    v = _fp32(x)
    avg = ((v[:, :-1, :-1] + v[:, :-1, 1:]) + (v[:, 1:, :-1] + v[:, 1:, 1:])) * 0.25     # [B, H-1, W-1, C]
    r1 = torch.zeros(B, H, W, C_ // 2)
    r1[:, :-1, :-1] = avg[..., :C_ // 2]                                                 # last row and column zero
    r2 = F.max_pool2d(avg[..., C_ // 2:].permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert r2.shape[1:3] == (H // 2, W // 2)
    _assert_planes_equal(x1, *_resplit(r1))
    _assert_planes_equal(x2, *_resplit(r2))


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W", [(1, 12, 20), (2, 3, 5)])
def test_maxpool_s1_x3_bit_exact(B, H, W):
    g = torch.Generator().manual_seed(B * H * W)
    C_ = 256
    x = pair_map(torch.randn(B, H, W, C_, generator=g), 512, 256, g)
    xd, y = _to(x, DEV), poisoned_map(B, H, W, 320, 32, C_, DEV)
    _extent_map(xd); _extent_map(y)
    ops.maxpool_s1(xd, y, 5)
    torch.cuda.synchronize()
    ref = F.max_pool2d(_fp32(x).permute(0, 3, 1, 2), 5, 1, 2).permute(0, 2, 3, 1)
    _assert_planes_equal(y, *_resplit(ref))


@pytest.mark.gpu
def test_upsample2x_x3_bit_exact():
    g = torch.Generator().manual_seed(3)
    B, H, W, C_ = 2, 12, 20, 128
    x = pair_map(torch.randn(B, H, W, C_, generator=g), 192, 32, g)
    xd, y = _to(x, DEV), poisoned_map(B, 2 * H, 2 * W, 384, 128, C_, DEV)
    _extent_map(xd); _extent_map(y)
    ops.upsample2x(xd, y)
    torch.cuda.synchronize()
    up = lambda t: t.repeat_interleave(2, 1).repeat_interleave(2, 2)
    hi, lo = planes(x)
    _assert_planes_equal(y, up(hi), up(lo))


CBFUSE_NSRC = [1, 2, 3, 4, 5]


@pytest.mark.gpu
@pytest.mark.parametrize("nsrc,sliced", [(n, False) for n in CBFUSE_NSRC] + [(5, True), (2, True)])
def test_cbfuse_x3_bit_exact(nsrc, sliced):
    """out = sum_i nearest_upsample(src_i) + last in fp32, in that order; source i is 2^i times coarser (the shifts of
    yolo_engine's CBFuse calls), each a channel slice of its own buffer with its own lo offset"""
    g = torch.Generator().manual_seed(10 * nsrc + sliced)
    B, H, W, C_ = 2, 32, 48, 64
    srcs = [pair_map(torch.randn(B, H >> i, W >> i, C_, generator=g), C_ * (i + 1) + 16, C_ * i + 8, g) for i in range(nsrc)]
    if sliced:
        last = pair_map(torch.randn(B, H, W, C_, generator=g), C_ + 32, 16, g)
        out = poisoned_map(B, H, W, 2 * C_, C_, C_, DEV)
    else:
        last = pair_map(torch.randn(B, H, W, C_, generator=g), C_, 0, g)
        out = poisoned_map(B, H, W, C_, 0, C_, DEV)
    srcs_d, last_d = [_to(s, DEV) for s in srcs], _to(last, DEV)
    for m in srcs_d + [last_d, out]:
        _extent_map(m)
    ops.cbfuse(srcs_d, last_d, out)
    torch.cuda.synchronize()
    acc = None
    for i, s in enumerate(srcs):
        t = _fp32(s).repeat_interleave(1 << i, 1).repeat_interleave(1 << i, 2)
        acc = t if acc is None else acc + t
    acc = acc + _fp32(last)
    _assert_planes_equal(out, *_resplit(acc))


# ------------------------------------------------------------------------------------------------ host-side rejections
def _rejected(fn, match):
    n0 = _lib.launch_count()
    with pytest.raises(_lib.B2PError, match=match):
        fn()
    assert _lib.launch_count() == n0


@pytest.mark.gpu
def test_malformed_lo_planes_are_rejected_before_launch():
    """Every buffer is large enough for the call as written, so nothing could run out of bounds even if a check were
    missing; the C side must still refuse each call before it launches anything."""
    K, N, Hm, Wm = 64, 64, 8, 16
    w1 = torch.zeros(N, 2 * K, dtype=torch.float16, device=DEV)
    w3 = torch.zeros(N, 18 * K, dtype=torch.float16, device=DEV)
    buf = torch.zeros(1, Hm, Wm, 4 * K, dtype=torch.float16, device=DEV)
    out = ops.Map(torch.zeros(1, Hm, Wm, 4 * N, dtype=torch.float16, device=DEV), 0, N, 2 * N)
    # lo plane of A inside the hi plane (lo_a < K), or not 8-aligned
    _rejected(lambda: ops.conv1x1(ops.Map(buf, 0, K, K - 32), w1, out), "lo-plane offset of A")
    _rejected(lambda: ops.conv1x1(ops.Map(buf, 0, K, K + 4), w1, out), "lo-plane offset of A")
    _rejected(lambda: ops.conv3x3(ops.Map(buf, 0, K, K - 32), w3, out), "lo-plane offset of A")
    _rejected(lambda: ops.conv3x3(ops.Map(buf, 0, K, K + 4), w3, out), "lo-plane offset of A")
    # split output whose lo plane is not 8-aligned
    x = ops.Map(buf, 0, K, 2 * K)
    _rejected(lambda: ops.conv1x1(x, w1, ops.Map(out.buf, 0, N, N + 4)), "8-aligned lo-plane offset")
    _rejected(lambda: ops.conv3x3(x, w3, ops.Map(out.buf, 0, N, N + 4)), "8-aligned lo-plane offset")
    # pair maps mixed with plain maps in the elementwise kernels
    plain = ops.Map(torch.zeros(1, Hm, Wm, 2 * K, dtype=torch.float16, device=DEV), 0, K)
    _rejected(lambda: ops.maxpool_s1(x, plain, 5), "lo planes must be both set")
    _rejected(lambda: ops.upsample2x(x, ops.Map(torch.zeros(1, 2 * Hm, 2 * Wm, 2 * K, dtype=torch.float16, device=DEV), 0, K)),
              "lo planes must be both set")
    _rejected(lambda: ops.adown_pool(x, ops.Map(buf, 0, K // 2, 2 * K), plain), "lo planes must be all set")
    src = ops.Map(torch.zeros(1, Hm // 2, Wm // 2, 2 * K, dtype=torch.float16, device=DEV), 0, K)   # plain fp16 source
    _rejected(lambda: ops.cbfuse([src], x, out), "lo planes must be all set")
    _rejected(lambda: ops.cbfuse([], x, plain), "lo planes must be all set")


# ------------------------------------------------------------------------------------------------ CPU: sensitivity
@pytest.mark.parametrize("name", CASE_IDS)
def test_tolerance_catches_a_dropped_lo_plane(name):
    """Each degraded reference (A's, W's, the residual's or the output's lo plane dropped) must differ from the fp64
    reference by more than SENSITIVITY x the case's tolerance, so a kernel that quietly falls back to plain fp16 on any
    operand fails test_planes_vs_fp64.  (No residual: nothing to drop; fp32 output: it has no lo plane.)"""
    c = next(c for c in CASES if c.name == name)
    ref = reference_full(name)
    bar = SENSITIVITY * tolerance(ref)
    degraded = {"A lo": reference(c, a_lo=False), "W lo": reference(c, w_lo=False)}
    if c.res is not None:
        degraded["residual lo"] = reference(c, res_lo=False)
    if c.out is not None:
        degraded["output lo"] = ref.half().double()
    for what, d in degraded.items():
        diff = (d - ref).abs().max().item()
        assert diff > bar, f"{name}: dropping the {what} plane moves the result by {diff:.3g}, not more than {bar:.3g}"


# ------------------------------------------------------------------------------------------------ CPU: plan coverage
def _conv_m_tiles(B, Ho, Wo):
    """M tiles of a non-halo implicit-GEMM conv (gemm_launch's spatial tiling: tw x th <= 128 output pixels)"""
    btw, bth, bu = 1, 1, -1.0
    for tw in range(1, min(Wo, 128) + 1):
        th = min(128 // tw, Ho)
        tiles = ((Wo + tw - 1) // tw) * ((Ho + th - 1) // th)
        u = Ho * Wo / (tiles * 128.0)
        if u > bu + 1e-9 or (u > bu - 1e-9 and tw > btw):
            bu, btw, bth = u, tw, th
    tx, ty = (Wo + btw - 1) // btw, (Ho + bth - 1) // bth
    if tx == 1 and ty == 1 and btw * bth * 2 <= 128 and B > 1:
        nb = min(128 // (btw * bth), B)
        return (B + nb - 1) // nb
    return tx * ty * B


def classify(name, a):
    """the features of a recorded `_planes` / `_x3` call that select different kernel code"""
    if name == "b2p_gemm_planes":
        _A, _lda, _B, M, N, K, _o, _ldc, _b, res, _ldr, _act, flags, lo_a, _lo_out, lo_res, _st = a
        op, stride, m_tiles = "gemm", 1, (M + 127) // 128
    elif name == "b2p_conv3x3_planes":
        _i, _ld, batch, H, W, K, stride, _w, N, _o, _ldc, _b, res, _ldr, _act, flags, lo_a, _lo_out, lo_res, _st = a
        op, m_tiles = "conv3x3", _conv_m_tiles(batch, H // stride, W // stride)
    elif name == "b2p_cbfuse_x3":
        return ("cbfuse_x3", a[0])
    else:
        return (name[len("b2p_"):],)
    return (op, f"s{stride}", f"Cin%64={K % 64 == 0}", f"lo_a>K={lo_a > K}", f"res_pair={bool(res) and lo_res > 0}",
            "out=f32" if flags & ops.FLAG_OUT_F32 else "out=split", f"N%16!=0={N % 16 != 0}",
            f"single_wave={m_tiles * ((N + 255) // 256) < 132}")


def test_cases_cover_every_call_class_of_the_parity_plan(rec):  # noqa: F811
    from omniparser_b200.yolo_engine import YoloPlan, YoloWeights
    from standin.yolo_weights import yolo_standin
    w = YoloWeights(yolo_standin(0).state_dict(), torch.device("cpu"), precision="fp16x3")
    YoloPlan(w, 1, 384, 640, use_graph=False).run()
    plan = {classify(n, a) for n, a in rec.calls if n.endswith(("_planes", "_x3"))}
    rec.calls.clear()
    for c in CASES:                     # the case table's launches, recorded the same way
        launch(c, "cpu")
    have = {classify(n, a) for n, a in rec.calls}
    have |= {("adown_pool_x3",), ("maxpool_s1_x3",), ("upsample2x_x3",)} | {("cbfuse_x3", n) for n in CBFUSE_NSRC}
    missing = sorted(plan - have)
    assert not missing, "call classes of the parity plan without a case in this module:\n" + "\n".join(map(str, missing))
    assert len(plan) >= 15
