"""CPU companion of tests/test_davit_kernels_gpu.py.

* The fp64 reference cores the GPU tests compare against are anchored to transformers' own Florence-2 vision modules:
  wrapped in a module's qkv / proj linears (and its depthwise conv and norm), they reproduce the module's output in fp64.
* Every class of DaViT call (``b2p_dwconv_ln`` / ``b2p_window_attn`` / ``b2p_channel_attn`` / ``b2p_conv3x3`` /
  ``b2p_im2col3x3``) that ``FlorencePlan.encode`` issues in the 64 and 768 modes, in both precisions, has a case in the
  GPU table, the kernel the C-side rules pick included."""
from __future__ import annotations

import contextlib
import ctypes as C
from unittest import mock

import pytest
import torch

from omniparser_b200 import _lib, ops
from test_davit_kernels_gpu import (CASES, WIN, Case, channel_attn_ref, dwconv_ln_ref, issue, kernel_for, make,
                                    window_attn_ref)
from test_plan_dryrun_cpu import _Recorder, rec  # noqa: F401  (fixture: the C library replaced by an argument-checking recorder)

DAVIT = ("b2p_dwconv_ln", "b2p_window_attn", "b2p_channel_attn", "b2p_conv3x3", "b2p_im2col3x3")


def classify(name, a):
    """the features of a recorded DaViT call that select different kernel code or addressing (not the batch)"""
    if name == "b2p_dwconv_ln":
        _x, _B, H, W, Cc, _w, _b, _y, _g, _bt, _eps, _o, split, _st = a
        return ("dwconv_ln", H, W, Cc, split & 1, kernel_for(name, a))
    if name == "b2p_window_attn":
        _q, _b, _B, H, W, Cc, heads, win, _o, split, _st = a
        return ("window_attn", H, W, Cc, heads, win, split & 1, kernel_for(name, a))
    if name == "b2p_channel_attn":
        _q, _B, N, Cc, groups, _o, split, _st = a
        return ("channel_attn", N, Cc, groups, split & 1, kernel_for(name, a))
    if name == "b2p_conv3x3":
        _i, ld_in, _B, H, W, Cin, stride, _w, Cout, _o, ldc, _b, res, _ldr, act, flags, _st = a
        return ("conv3x3", H, W, Cin, Cout, stride, ld_in, ldc, res is not None, act, flags)
    if name == "b2p_im2col3x3":
        _x, ld, _B, H, W, Cc, stride, halves, _o, _st = a
        return ("im2col3x3", H, W, Cc, stride, halves, ld)
    return None


@contextlib.contextmanager
def _recording():
    r = _Recorder()
    with mock.patch.object(_lib, "_lib", r), mock.patch.object(ops, "_stream", lambda: C.c_void_p(0)):
        yield r


def recorded_calls(c: Case):
    """the C-ABI calls a case issues, recorded (shapes only: nothing runs)"""
    with _recording() as r:
        issue(c, make(c, "meta"))
    return r.calls


def case_class(c: Case):
    classes = [classify(n, a) for n, a in recorded_calls(c)]
    return next(k for k in classes if k is not None)


# ------------------------------------------------------------------------------------------------ plan coverage
def test_cases_cover_every_davit_call_class_of_the_florence_plans(rec):  # noqa: F811
    from omniparser_b200.florence_engine import FlorencePlan, FlorenceWeights
    from standin import florence as FS
    sd = FS.florence_standin(0).state_dict()
    plan = {}
    for size in (64, 768):
        for prec in ("fp16x3", "fp16"):
            w = FlorenceWeights(sd, torch.device("cpu"), FS.GEN, prec)
            p = FlorencePlan(w, 2, 2, FS.PROMPT_IDS, use_graph=False, size=size)
            rec.calls.clear()
            p.encode()
            for n, a in rec.calls:
                if n in DAVIT:
                    plan.setdefault(classify(n, a), (size, prec))
            del p, w
    rec.calls.clear()
    have = {case_class(c) for c in CASES}
    print("DaViT call classes of the Florence plans (mode, precision, class):")
    for k, (size, prec) in sorted(plan.items(), key=lambda kv: (kv[1], str(kv[0]))):
        print(f"  {size:3d} {prec:6s} {k}{'' if k in have else '   <- no case'}")
    missing = sorted(map(str, set(plan) - have))
    assert not missing, "DaViT call classes of the Florence plans without a case:\n" + "\n".join(missing)
    kernels = {k[-1] for k in plan if k[0] in ("dwconv_ln", "window_attn", "channel_attn")}
    assert kernels == {"dwconv_ln_kernel", "dwconv_ln_v3_kernel", "window_attn_kernel", "window_attn_crop_kernel",
                       "channel_attn_kernel", "channel_attn_v3_kernel", "channel_attn_rows_kernel"}, kernels
    # 8 (map, dim) stages x 3 ops x 2 precisions, and the patch embeds (4 conv3x3 + 2 im2col3x3 classes per precision)
    assert len(plan) == 8 * 3 * 2 + 6 * 2, len(plan)
    # the forced fall-backs of the table run the tile and small kernels too
    assert {k[-1] for k in have if k[0] in ("dwconv_ln", "channel_attn")} >= {"dwconv_ln_tile_kernel", "channel_attn_small_kernel"}


def test_case_table_shape():
    """every case exists with [hi | lo] and plain outputs, and each kernel has a case at the largest batch of a mode"""
    keys = {c.key for c in CASES}
    for c in CASES:
        other = c.key[:6] + (not c.split,) + c.key[7:]
        assert other in keys, c.id
    big = {case_class(c)[-1] if c.op in ("dwconv_ln", "window_attn", "channel_attn") else c.op for c in CASES if c.bucket}
    assert big == {"dwconv_ln_kernel", "dwconv_ln_v3_kernel", "dwconv_ln_tile_kernel", "window_attn_kernel", "window_attn_crop_kernel",
                   "channel_attn_kernel", "channel_attn_v3_kernel", "channel_attn_rows_kernel", "channel_attn_small_kernel",
                   "conv3x3", "im2col_gemm"}, big


# ------------------------------------------------------------------------------------------------ references anchored to HF
def _config():
    from transformers.models.florence2.configuration_florence2 import Florence2VisionConfig
    cfg = Florence2VisionConfig(drop_path_rate=0.0)
    cfg._attn_implementation = "eager"
    return cfg


def _seeded(module, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in module.parameters():
            p.copy_(torch.randn(p.shape, generator=g, dtype=torch.float64) * 0.3)
    return module.double().eval()


@pytest.mark.parametrize("H,W", [(16, 16), (24, 24), (20, 28)])
def test_window_attn_ref_matches_hf(H, W):
    """16 x 16: one full and three partial windows (padding); 24 x 24: four full windows; 20 x 28: non-square, partial"""
    from transformers.models.florence2.modeling_florence2 import Florence2VisionWindowAttention
    cfg = _config()
    m = _seeded(Florence2VisionWindowAttention(cfg, 0), H * W)
    B, Cc, heads = 2, cfg.embed_dim[0], cfg.num_heads[0]
    x = torch.randn(B, H, W, Cc, generator=torch.Generator().manual_seed(H + W), dtype=torch.float64)
    with torch.no_grad():
        want = m(x)                                                     # [B, H*W, C]
        qkv = m.qkv(x.reshape(B * H * W, Cc))
        got = m.proj(window_attn_ref(qkv, m.qkv.bias, B, H, W, Cc, heads, WIN)).reshape(B, H * W, Cc)
    assert (got - want).abs().max().item() < 1e-12 * max(1.0, want.abs().max().item())


@pytest.mark.parametrize("N,stage", [(64, 1), (576, 0)])
@pytest.mark.parametrize("shift", [0.0, 1.0])
def test_channel_attn_ref_matches_hf(N, stage, shift):
    from transformers.models.florence2.modeling_florence2 import Florence2VisionChannelAttention
    cfg = _config()
    m = _seeded(Florence2VisionChannelAttention(cfg, stage), N + stage)
    B, Cc, groups = 2, cfg.embed_dim[stage], cfg.num_groups[stage]
    x = torch.randn(B, N, Cc, generator=torch.Generator().manual_seed(N), dtype=torch.float64) + shift
    with torch.no_grad():
        want = m(x)
        qkv = m.qkv(x.reshape(B * N, Cc))
        got = m.proj(channel_attn_ref(qkv, B, N, Cc, groups)).reshape(B, N, Cc)
    assert (got - want).abs().max().item() < 1e-12 * max(1.0, want.abs().max().item())


@pytest.mark.parametrize("H,W", [(16, 16), (12, 20)])
def test_dwconv_ln_ref_matches_hf(H, W):
    """the spatial block's first half up to its norm: conv1(x) + x, then norm1"""
    from transformers.models.florence2.modeling_florence2 import Florence2VisionSpatialBlock
    cfg = _config()
    blk = _seeded(Florence2VisionSpatialBlock(cfg, 0, 0.0), H * W + 1)
    B, Cc = 2, cfg.embed_dim[0]
    x = torch.randn(B, Cc, H, W, generator=torch.Generator().manual_seed(W), dtype=torch.float64)
    with torch.no_grad():
        y_hf = (blk.conv1(x) + x).flatten(2).transpose(1, 2).reshape(-1, Cc)
        h_hf = blk.norm1(y_hf)
        y, h = dwconv_ln_ref(x.permute(0, 2, 3, 1), blk.conv1.weight.reshape(Cc, 9).t(), blk.conv1.bias, blk.norm1.weight,
                             blk.norm1.bias, blk.norm1.eps)
    assert (y - y_hf).abs().max().item() < 1e-12 * max(1.0, y_hf.abs().max().item())
    assert (h - h_hf).abs().max().item() < 1e-12 * max(1.0, h_hf.abs().max().item())
