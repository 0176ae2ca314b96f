"""The caption vision encoder's (DaViT) kernels against fp64, at the shapes both caption modes run.

``FlorencePlan.encode`` runs four DaViT stages (dims 128 / 256 / 512 / 1024).  The 64 mode works on maps of 16 / 8 / 4 / 2
pixels, the 768 mode on maps of 192 / 96 / 48 / 24 (up to 36 864 tokens per crop), and the C-side selection rules send the
same entry point to different kernels in the two modes.  This module pins each of them:

* ``b2p_dwconv_ln`` (per-token, tile and strip kernels): ``y`` against fp64 ``conv2d(groups=C) + bias + x``, the fp16
  output against fp64 LayerNorm of the fp64 ``y``;
* ``b2p_window_attn`` (per-window and one-window kernels) against fp64 windowed attention whose padded tokens carry
  qkv = bias, on full, partial and non-square window grids;
* ``b2p_channel_attn`` (first-version, small, register-tiled and rows kernels) against fp64, on unit-normal inputs and on
  mean-shifted ones (the kernel's input is the output of a biased linear layer, so its partial sums grow with N);
* the patch embeds: ``b2p_conv3x3`` stride 2 and the 64 mode's ``b2p_im2col3x3`` + GEMM route against fp64 ``conv2d``.

Every case runs with [hi | lo] pair outputs (``split``) and plain fp16 outputs, on poisoned buffers with one guard row
that must come back unchanged, after a host-side check that the allocations span every address the kernel can reach.
One case per kernel runs at the largest crop batch a plan issues; there only the first and last crop are compared with
fp64.  The fp64 references are anchored to transformers' own Florence-2 modules by tests/test_davit_cases_cpu.py, which
also checks that every class of call the Florence plans issue has a case here."""
from __future__ import annotations

import re
from dataclasses import dataclass, replace

import pytest
import torch
import torch.nn.functional as F

from omniparser_b200 import ops
from omniparser_b200.caption import BUCKET_768
from test_decode_step_gpu import SENTINEL, TOL_F16, TOL_GEMM16, TOL_LN32, TOL_X3, _act_value, _tol
from test_parity_planes_gpu import _covers, check_canonical, pair

DEV = "cuda:0"
WIN = 12                                   # DaViT window size
DIMS = (128, 256, 512, 1024)               # channels per stage; heads = groups = C / 32
MAPS = {64: (16, 8, 4, 2), 768: (192, 96, 48, 24)}
BUCKET_64 = 416                            # the largest 64-mode crop batch the caption lanes run (DESIGN.md)
V3, TILE = 4, 2                            # variant bits of the split argument (bit 0 is the [hi | lo] output)


# ================================================================================================ fp64 references
def dwconv_ln_ref(x, w9c, bias, gamma, beta, eps=1e-5):
    """x [B, H, W, C] -> (y, LayerNorm(y)) in fp64, y = depthwise 3x3 (pad 1) + bias + x; w9c [9, C] (tap-major)"""
    C = x.shape[-1]
    xr = x.double().permute(0, 3, 1, 2)
    y = F.conv2d(xr, w9c.double().t().reshape(C, 1, 3, 3), bias.double(), padding=1, groups=C) + xr
    y = y.permute(0, 2, 3, 1).reshape(-1, C)
    return y, F.layer_norm(y, (C,), gamma.double(), beta.double(), eps)


def window_attn_ref(qkv, bias, B, H, W, C, heads, win=WIN):
    """fp64 window attention on qkv [B*H*W, 3C] (real tokens).  The map is zero-padded to whole windows BEFORE the qkv
    projection, so padded tokens have qkv = bias and take part as keys / values, unmasked."""
    d, nwy, nwx = C // heads, -(-H // win), -(-W // win)
    full = bias.double().reshape(1, 1, 1, 3 * C).repeat(B, nwy * win, nwx * win, 1)
    full[:, :H, :W] = qkv.double().reshape(B, H, W, 3 * C)
    t = full.reshape(B, nwy, win, nwx, win, 3, heads, d).permute(5, 0, 1, 3, 6, 2, 4, 7).reshape(3, B, nwy, nwx, heads, win * win, d)
    a = torch.softmax((t[0] * d ** -0.5) @ t[1].transpose(-1, -2), -1) @ t[2]         # [B, nwy, nwx, heads, win*win, d]
    a = a.reshape(B, nwy, nwx, heads, win, win, d).permute(0, 1, 4, 2, 5, 3, 6).reshape(B, nwy * win, nwx * win, C)
    return a[:, :H, :W].reshape(B * H * W, C)


def channel_attn_ref(qkv, B, N, C, groups):
    """fp64 channel attention: per (image, group) S = N^-0.5 q^T k over the tokens, out = v softmax(S)^T"""
    t = qkv.double().reshape(B, N, 3, groups, C // groups).permute(2, 0, 3, 1, 4)      # [3, B, g, N, d]
    p = torch.softmax((t[0].transpose(-1, -2) @ t[1]) * N ** -0.5, -1)                 # [B, g, d, d]
    return (t[2] @ p.transpose(-1, -2)).transpose(1, 2).reshape(B * N, C)


def conv_s2_ref(x, w, bias):
    """x [B, H, W, Ci], w [Co, Ci, 3, 3] -> [B, H/2, W/2, Co], fp64, stride 2 pad 1"""
    return F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), bias.double(), stride=2, padding=1).permute(0, 2, 3, 1)


# ================================================================================================ the C-side selection rules
def _dw_v3_fits(B, H, W, C):
    """dwconv_ln_v3_launch (florence_simt.cu) takes the shape"""
    C4 = C // 4
    if C % 128 or C4 > 256 or 256 % C4 or B <= 0 or W < 1 or W & (W - 1):
        return False
    G = 256 // C4
    if W > 8 * G:
        return False
    R = min((8 * G) // W, H)
    smem = ((2 * R + 2) * W + 1) * C * 4 + (2 * R * W * (C4 // 32) + 4) * 4
    return smem <= 100 * 1024


def _crop_fits(B, H, W, C, heads, win):
    """window_attn_crop_launch takes the shape"""
    if H > win or W > win or C != heads * 32 or B <= 0 or H * W > 64:
        return False
    nreal = H * W
    hpc = min(256 // nreal, heads)
    while hpc > 1 and heads % hpc:
        hpc -= 1
    qb = 2 if nreal % 2 == 0 else 1
    threads = hpc * (nreal // qb)
    return 1 <= threads <= 256 // qb and 2 * nreal * hpc * 32 * 4 + 16 <= 65 * 1024


def _rows_fits(N, groups):
    """channel_attn_rows_go finds a group chunk whose tokens fit its shared memory"""
    gpc = min(groups, 8)
    while gpc > 1 and (groups % gpc or N * 3 * gpc * 128 > 64 * 1024):
        gpc -= 1
    return groups % gpc == 0 and N * 3 * gpc * 128 + 16 <= 65 * 1024


def kernel_for(name, a):
    """the kernel b2p_dwconv_ln / b2p_window_attn / b2p_channel_attn launch for these arguments (florence_ops.cu entry
    points + florence_simt.cu launchers, restated); None for the other entry points"""
    if name == "b2p_dwconv_ln":
        _x, B, H, W, C, _w, _b, _y, _g, _bt, _eps, _o, split, _st = a
        if split & V3 and _dw_v3_fits(B, H, W, C):
            return "dwconv_ln_v3_kernel"
        if split & TILE and H * W * C * 4 <= 200 * 1024 and B > 0:
            return "dwconv_ln_tile_kernel"
        return "dwconv_ln_kernel"
    if name == "b2p_window_attn":
        _q, _b, B, H, W, C, heads, win, _o, split, _st = a
        return "window_attn_crop_kernel" if split & V3 and _crop_fits(B, H, W, C, heads, win) else "window_attn_kernel"
    if name == "b2p_channel_attn":
        _q, B, N, C, groups, _o, split, _st = a
        if split & V3 and C == groups * 32 and B > 0 and 0 < N <= 320:
            if N <= 32 and _rows_fits(N, groups):
                return "channel_attn_rows_kernel"
            return "channel_attn_v3_kernel"               # NW = 1 / 2 / 8: the shared memory fits up to N = 320
        if split & TILE and N <= 16 and B > 0:
            return "channel_attn_small_kernel"
        return "channel_attn_kernel"
    return None


# ================================================================================================ the case table
@dataclass(frozen=True)
class Case:
    """one launch.  H x W: the map (channel_attn: N = H*W tokens; conv / im2col: the input map).  hg: heads (window),
    groups (channel) or output channels (conv).  flags: the variant bits the call passes besides the split bit (patch
    embeds: none).  split: [hi | lo] pair outputs (patch embeds: fp16x3 operands, fp32 output).  bucket: the largest crop
    batch of its mode; only the first and last crop are compared with fp64."""
    op: str
    B: int
    H: int
    W: int
    C: int
    hg: int
    flags: int
    split: bool
    scale: str = "unit"         # channel_attn inputs: "unit" = randn, "shifted" = randn + 1
    bucket: bool = False

    @property
    def key(self):
        return (self.op, self.B, self.H * self.W if self.op == "channel_attn" else (self.H, self.W), self.C, self.hg,
                self.flags, self.split, self.scale)

    @property
    def id(self):
        f = {0: "plain", TILE: "tile", V3: "v3", V3 | TILE: "plan"}[self.flags]
        shape = f"N{self.H * self.W}" if self.op == "channel_attn" else f"{self.H}x{self.W}"
        extra = f"-{self.scale}" if self.op == "channel_attn" else ""
        return f"{self.op}-B{self.B}-{shape}-C{self.C}-{self.hg}-{f}{extra}-{'split' if self.split else 'f16'}"


def _both_splits(cases):
    return [replace(c, split=s) for c in cases for s in (True, False)]


def _table():
    out = []
    stage = {H: s for m in MAPS.values() for s, H in enumerate(m)}
    plan_dw, plan_win, plan_ch = V3 | TILE, V3, V3 | TILE          # what FlorencePlan passes (B2P_NO_* unset)
    for mode, maps in MAPS.items():
        for H in maps:
            C = DIMS[stage[H]]
            B = 3 if mode == 64 else 2
            # dwconv + LayerNorm: the plan's flags, and in the 64 mode forced fall-backs so each kernel is run where it serves
            for fl in ((plan_dw, TILE, 0) if mode == 64 else (plan_dw,)):
                out.append(Case("dwconv_ln", B, H, H, C, 0, fl, True))
            for fl in ((plan_win, 0) if mode == 64 and H <= WIN else (plan_win,)):
                out.append(Case("window_attn", B, H, H, C, C // 32, fl, True))
            for scale in ("unit", "shifted"):
                for fl in ((plan_ch, TILE, 0) if mode == 64 else (plan_ch,)):
                    if fl == TILE and H * H > 16:
                        continue                                   # the small kernel serves N <= 16 only
                    out.append(Case("channel_attn", B, H, H, C, C // 32, fl, True, scale))
    # non-square maps: a wx / wy or x / y swap cannot hide (3 x 2 windows, the right column partial)
    out.append(Case("window_attn", 2, 36, 20, 128, 4, plan_win, True))
    out.append(Case("dwconv_ln", 2, 20, 12, 256, 0, plan_dw, True))
    # patch embeds: conv3x3 s2 where the plans run it, im2col3x3 + GEMM for the 64 mode's 8 -> 4 and 4 -> 2
    out.append(Case("conv3x3", 3, 16, 16, 128, 256, 0, True))
    for H, Ci in ((192, 128), (96, 256), (48, 512)):
        out.append(Case("conv3x3", 2, H, H, Ci, 2 * Ci, 0, True))
    for H, Ci in ((8, 256), (4, 512)):
        out.append(Case("im2col_gemm", 3, H, H, Ci, 2 * Ci, 0, True))
    # the largest batch of each mode, once per kernel
    big = [Case("dwconv_ln", BUCKET_768, 192, 192, 128, 0, plan_dw, True, bucket=True),
           Case("dwconv_ln", BUCKET_64, 16, 16, 128, 0, plan_dw, True, bucket=True),
           Case("dwconv_ln", BUCKET_64, 16, 16, 128, 0, TILE, True, bucket=True),
           Case("window_attn", BUCKET_768, 192, 192, 128, 4, plan_win, True, bucket=True),
           Case("window_attn", BUCKET_64, 16, 16, 128, 4, plan_win, True, bucket=True),
           Case("window_attn", BUCKET_64, 8, 8, 256, 8, plan_win, True, bucket=True),
           Case("channel_attn", BUCKET_768, 192, 192, 128, 4, plan_ch, True, "shifted", bucket=True),
           Case("channel_attn", BUCKET_64, 16, 16, 128, 4, plan_ch, True, "shifted", bucket=True),
           Case("channel_attn", BUCKET_64, 4, 4, 512, 16, plan_ch, True, "shifted", bucket=True),
           Case("channel_attn", BUCKET_64, 4, 4, 512, 16, TILE, True, "shifted", bucket=True),
           Case("conv3x3", BUCKET_768, 192, 192, 128, 256, 0, True, bucket=True),
           Case("conv3x3", BUCKET_64, 16, 16, 128, 256, 0, True, bucket=True),
           Case("im2col_gemm", BUCKET_64, 8, 8, 256, 512, 0, True, bucket=True)]
    return _both_splits(out + big)


CASES = _table()
assert len({c.key for c in CASES}) == len(CASES)
BY_ID = {c.id: c for c in CASES}
assert len(BY_ID) == len(CASES)


# ================================================================================================ buffers and launches
def _randn(shape, g, dev):
    if dev == "meta":
        return torch.empty(shape, device="meta")
    return torch.randn(shape, generator=g, device=dev)


def _poisoned(rows, cols, dtype, dev):
    """output buffer with one guard row past the end"""
    return torch.full((rows + 1, cols), SENTINEL, dtype=dtype, device=dev)


def _seed(c: Case):
    return sum(map(ord, c.id.replace("-split", "").replace("-f16", "")))


def make(c: Case, dev):
    """the case's seeded inputs and poisoned outputs on `dev` ("meta": shapes only, for the CPU recorder)"""
    g = torch.Generator(device=dev).manual_seed(_seed(c)) if dev != "meta" else None
    B, H, W, C = c.B, c.H, c.W, c.C
    T = B * H * W
    kx = 2 if c.split else 1
    if c.op == "dwconv_ln":
        x = _randn((T, C), g, dev)
        d = dict(x=x, w9c=_randn((9, C), g, dev) * 0.3, bias=_randn((C,), g, dev) * 0.5, gamma=_randn((C,), g, dev),
                 beta=_randn((C,), g, dev), y=_poisoned(T, C, torch.float32, dev), o16=_poisoned(T, kx * C, torch.float16, dev))
    elif c.op in ("window_attn", "channel_attn"):
        qkv = _randn((T, 3 * C), g, dev)
        if c.scale == "shifted":
            qkv = qkv + 1.0
        d = dict(qkv=qkv, bias=_randn((3 * C,), g, dev), out=_poisoned(T, kx * C, torch.float16, dev))
    else:                                   # conv3x3 / im2col_gemm: [hi | lo] pixels (split) or fp16 pixels
        Ci, Co, Ho, Wo = C, c.hg, H // 2, W // 2
        x32 = _randn((B, H, W, Ci), g, dev)
        w = _randn((Co, Ci, 3, 3), g, dev) / (9 * Ci) ** 0.5
        if c.split:
            hi, lo = pair(x32)
            xm = ops.Map(torch.cat([hi, lo], 3).contiguous(), 0, 2 * Ci)
        else:
            xm = ops.Map(x32.half(), 0, Ci)
        t = w.permute(0, 2, 3, 1)                                       # [Co, ky, kx, Ci]
        whi, wlo = pair(t)
        if c.op == "conv3x3":                                           # [Co][tap][hi(Ci) | lo(Ci)]
            wpk = (torch.cat([whi, wlo], 3) if c.split else whi).reshape(Co, -1).contiguous()
        else:                                                           # [Co][hi: 9*Ci | lo: 9*Ci]
            wpk = (torch.cat([whi.reshape(Co, -1), wlo.reshape(Co, -1)], 1) if c.split else whi.reshape(Co, -1)).contiguous()
        d = dict(x=xm, w=w, wpk=wpk, bias=_randn((Co,), g, dev) * 0.5, out=_poisoned(B * Ho * Wo, Co, torch.float32, dev))
        if c.op == "im2col_gemm":
            d["col"] = torch.full((B * Ho * Wo, kx * 9 * Ci), SENTINEL, dtype=torch.float16, device=dev)
    return d


def issue(c: Case, d):
    """check the extents, then launch through the ops front ends"""
    B, H, W, C = c.B, c.H, c.W, c.C
    T, kx = B * H * W, 2 if c.split else 1
    fl = c.flags | int(c.split)
    if c.op == "dwconv_ln":
        for k in ("x", "y"):
            _covers(d[k], d[k].data_ptr(), T * C)
        for k in ("w9c",):
            _covers(d[k], d[k].data_ptr(), 9 * C)
        for k in ("bias", "gamma", "beta"):
            _covers(d[k], d[k].data_ptr(), C)
        _covers(d["o16"], d["o16"].data_ptr(), T * kx * C)
        ops.dwconv_ln(d["x"], B, H, W, C, d["w9c"], d["bias"], d["y"], d["gamma"], d["beta"], d["o16"], split=c.split,
                      tile=bool(fl & TILE), v3=bool(fl & V3))
    elif c.op == "window_attn":
        _covers(d["qkv"], d["qkv"].data_ptr(), T * 3 * C)
        _covers(d["bias"], d["bias"].data_ptr(), 3 * C)
        _covers(d["out"], d["out"].data_ptr(), T * kx * C)
        ops.window_attn(d["qkv"], d["bias"], B, H, W, C, c.hg, d["out"], win=WIN, split=c.split, v3=bool(fl & V3))
    elif c.op == "channel_attn":
        _covers(d["qkv"], d["qkv"].data_ptr(), T * 3 * C)
        _covers(d["out"], d["out"].data_ptr(), T * kx * C)
        ops.channel_attn(d["qkv"], B, H * W, C, c.hg, d["out"], split=c.split, small=bool(fl & TILE), v3=bool(fl & V3))
    else:
        x, Co, M = d["x"], c.hg, B * (H // 2) * (W // 2)
        _covers(x.buf, x.ptr, T * x.ld)
        _covers(d["bias"], d["bias"].data_ptr(), Co)
        _covers(d["out"], d["out"].data_ptr(), M * Co)
        _covers(d["wpk"], d["wpk"].data_ptr(), Co * kx * 9 * C)
        out = ops.Map(d["out"][:M].view(B, H // 2, W // 2, Co), 0, Co)
        if c.op == "conv3x3":
            ops.conv3x3(x, d["wpk"], out, 2, d["bias"], None, ops.ACT_NONE, out_f32=True, x3=c.split)
        else:
            _covers(d["col"], d["col"].data_ptr(), M * kx * 9 * C)
            ops.im2col3x3(x, 2, d["col"], halves=kx)
            ops.gemm(d["col"], d["col"].stride(0), d["wpk"], M, Co, 9 * C, d["out"], Co, d["bias"], None, 0, ops.ACT_NONE,
                     out_f32=True, x3=c.split)


# ================================================================================================ checks
def _crops(c: Case):
    return (0, c.B - 1) if c.bucket else tuple(range(c.B))


def _rows_of(t, c: Case, per):
    """the rows of the compared crops (per = rows per crop), on the host"""
    return torch.cat([t[b * per:(b + 1) * per].cpu() for b in _crops(c)])


def _check_written(buf, rows, what):
    """every element of rows [0, rows) written, the guard row untouched (checked on the device: buckets are large)"""
    assert not bool((buf[:rows] == SENTINEL).any()), f"{what}: {int((buf[:rows] == SENTINEL).sum())} elements not written"
    assert bool((buf[rows] == SENTINEL).all()), f"{what}: guard row written"


def _check_act(o, ref, C, split, what):
    """o: fp16 rows ([hi | lo] when split) of the compared crops; -> err / tol"""
    if split:
        check_canonical(o[:, :C], o[:, C:2 * C])
    err, tol = (_act_value(o, C, split) - ref).abs().max().item(), _tol(ref, TOL_X3 if split else TOL_F16)
    print(f"[davit] {what}: max abs err {err:.3g}, tol {tol:.3g} ({err / tol:.3f} of it)")
    assert err < tol, f"{what}: max abs err {err:.3g} > {tol:.3g}"
    return err / tol


def check(c: Case, d):
    B, H, W, C = c.B, c.H, c.W, c.C
    HW = H * W
    T = B * HW
    if c.op == "dwconv_ln":
        _check_written(d["y"], T, "y")
        _check_written(d["o16"], T, "out16")
        x = _rows_of(d["x"], c, HW).view(-1, H, W, C)
        yr, hr = dwconv_ln_ref(x, d["w9c"].cpu(), d["bias"].cpu(), d["gamma"].cpu(), d["beta"].cpu())
        y = _rows_of(d["y"], c, HW).double()
        err, tol = (y - yr).abs().max().item(), _tol(yr, TOL_LN32)
        print(f"[davit] {c.id} y: max abs err {err:.3g}, tol {tol:.3g} ({err / tol:.3f} of it)")
        assert err < tol, f"y: max abs err {err:.3g} > {tol:.3g}"
        _check_act(_rows_of(d["o16"], c, HW), hr, C, c.split, f"{c.id} out16")
    elif c.op in ("window_attn", "channel_attn"):
        _check_written(d["out"], T, "out")
        qkv = _rows_of(d["qkv"], c, HW)
        nb = len(_crops(c))
        if c.op == "window_attn":
            ref = window_attn_ref(qkv, d["bias"].cpu(), nb, H, W, C, c.hg)
        else:
            ref = channel_attn_ref(qkv, nb, HW, C, c.hg)
        _check_act(_rows_of(d["out"], c, HW), ref, C, c.split, c.id)
    else:
        Ho, Wo, Co = H // 2, W // 2, c.hg
        _check_written(d["out"], B * Ho * Wo, "out")
        xm = d["x"]
        xs = torch.cat([xm.buf[b:b + 1].cpu() for b in _crops(c)])
        xv = (xs[..., :C].double() + xs[..., C:].double()) if c.split else xs.double()
        whi, wlo = pair(d["w"].cpu())
        w = (whi.double() + wlo.double()) if c.split else whi.double()
        ref = conv_s2_ref(xv, w, d["bias"].cpu()).reshape(-1, Co)
        got = _rows_of(d["out"], c, Ho * Wo).double()
        err, tol = (got - ref).abs().max().item(), _tol(ref, TOL_X3 if c.split else TOL_GEMM16)
        print(f"[davit] {c.id}: max abs err {err:.3g}, tol {tol:.3g} ({err / tol:.3f} of it)")
        assert err < tol, f"max abs err {err:.3g} > {tol:.3g}"


@pytest.mark.gpu
@pytest.mark.parametrize("cid", list(BY_ID))
def test_davit_kernel_vs_fp64(cid):
    c = BY_ID[cid]
    d = make(c, DEV)
    issue(c, d)
    torch.cuda.synchronize()
    check(c, d)


# ================================================================================================ which kernel ran
def _profiled_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type.name == "CUDA"]


def _launched(names, kernel):
    return any(re.search(rf"(^|[\s:]){kernel}[<(]", n) for n in names)


def representative_cases():
    """one small case per (op, kernel) class of the table: the cheapest one"""
    from test_davit_cases_cpu import case_class
    seen = {}
    for c in sorted(CASES, key=lambda c: c.B * c.H * c.W * c.C):
        seen.setdefault(case_class(c), c)
    return list(seen.values())


@pytest.mark.gpu
def test_each_case_runs_the_kernel_its_rule_predicts():
    """Without this a case can silently test another kernel than intended (a fall-through flag, a changed rule)."""
    from test_davit_cases_cpu import recorded_calls
    ran = {}
    for c in representative_cases():
        calls = recorded_calls(c)
        want = [kernel_for(n, a) for n, a in calls if kernel_for(n, a)]
        if not want:
            continue                                  # patch embeds: the GEMM's dispatch is not this module's subject
        d = make(c, DEV)
        torch.cuda.synchronize()
        names = _profiled_kernels(lambda: issue(c, d))
        assert _launched(names, want[0]), f"{c.id}: the rule predicts {want[0]}, the profiler saw {names}"
        others = {"dwconv_ln_kernel", "dwconv_ln_tile_kernel", "dwconv_ln_v3_kernel", "window_attn_kernel", "window_attn_crop_kernel",
                  "channel_attn_kernel", "channel_attn_small_kernel", "channel_attn_v3_kernel", "channel_attn_rows_kernel"} - {want[0]}
        assert not any(_launched(names, k) for k in others), f"{c.id}: {names}"
        ran[want[0]] = ran.get(want[0], 0) + 1
    print(f"[davit] kernels checked: {sorted(ran.items())}")
    assert set(ran) == {"dwconv_ln_kernel", "dwconv_ln_tile_kernel", "dwconv_ln_v3_kernel", "window_attn_kernel",
                        "window_attn_crop_kernel", "channel_attn_kernel", "channel_attn_small_kernel", "channel_attn_v3_kernel",
                        "channel_attn_rows_kernel"}
