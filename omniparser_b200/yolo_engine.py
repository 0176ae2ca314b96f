"""YOLOv9-E icon detector on the package's CUDA kernels (replaces the TorchScript forward at ref:util/yolov9.py:120-121).

Host side only plans: it folds BatchNorm into the convolutions, re-parameterises RepConvN (3x3 + 1x1 -> one 3x3),
packs weights K-major fp16, lays every feature map out as an NHWC fp16 channel slice so that ``torch.cat`` /
``chunk`` become pointer offsets, and records the launch sequence once; the sequence is then replayed as a CUDA
graph.  All arithmetic runs in ``libb200parse.so``: wgmma implicit-GEMM convs with fused bias+SiLU(+residual)
epilogues plus the HBM-bound pooling / upsample / CBFuse kernels.

Topology: WongKinYiu/yolov9 ``yolov9-e.yaml`` (restated in standin/yolov9e.py, SURVEY.md §8a row D2).
"""
from __future__ import annotations

import math
import os
from typing import Dict, List

import numpy as np
import torch

from . import ops
from .ops import ACT_NONE, ACT_SILU, Map

BN_EPS = 1e-3


# --------------------------------------------------------------------------------------------- weight folding
class _TrackedState(dict):
    """state_dict that remembers which keys were read, so a loader can prove it consumed the whole archive."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.used = set()

    def __getitem__(self, k):
        self.used.add(k)
        return super().__getitem__(k)

    def get(self, k, default=None):
        if k in self:
            return self[k]
        return default


# keys of an upstream archive that carry no learned arithmetic of the deployed graph
_IGNORED_SUFFIXES = ("num_batches_tracked", "anchors", "strides")
_DFL_SUFFIXES = ("dfl.conv.weight", "detect.proj")   # the DFL expectation weights: must be arange(reg_max), checked


def _fold_conv_bn(sd, prefix):
    """conv (no bias) + BatchNorm(eval) -> (weight fp32 [Co,Ci,k,k], bias fp32 [Co]).  An archive exported with
    conv+BN already fused (no ``.bn.*`` keys, ``.conv.bias`` present) is taken as is."""
    w = sd[prefix + ".conv.weight"].float()
    if prefix + ".bn.weight" not in sd:
        if prefix + ".conv.bias" not in sd:
            raise KeyError(f"{prefix}: neither BatchNorm parameters nor a fused conv bias in the archive")
        return w, sd[prefix + ".conv.bias"].float()
    g, b = sd[prefix + ".bn.weight"].float(), sd[prefix + ".bn.bias"].float()
    mu, var = sd[prefix + ".bn.running_mean"].float(), sd[prefix + ".bn.running_var"].float()
    s = g / torch.sqrt(var + BN_EPS)
    return w * s[:, None, None, None], b - mu * s


def _fold_repconv(sd, prefix):
    if prefix + ".conv1.conv.weight" not in sd and prefix + ".conv.weight" in sd:
        # archive exported after RepConvN.fuse_convs(): one re-parameterised 3x3 conv with bias
        return sd[prefix + ".conv.weight"].float(), sd[prefix + ".conv.bias"].float()
    w3, b3 = _fold_conv_bn(sd, prefix + ".conv1")
    w1, b1 = _fold_conv_bn(sd, prefix + ".conv2")
    w = w3.clone()
    w[:, :, 1:2, 1:2] += w1
    return w, b3 + b1


def _dense_from_grouped(w, groups):
    """[Co, Ci/g, k, k] grouped weight -> block-diagonal dense [Co, Ci, k, k] (zeros outside the group)."""
    co, cig, kh, kw = w.shape
    ci = cig * groups
    d = torch.zeros(co, ci, kh, kw, dtype=w.dtype)
    cog = co // groups
    for gi in range(groups):
        d[gi * cog:(gi + 1) * cog, gi * cig:(gi + 1) * cig] = w[gi * cog:(gi + 1) * cog]
    return d


def _pack(w, device, kpad=None, x3=False):
    """[Co,Ci,kh,kw] -> fp16 [Co, kh*kw*Ci] ordered (ky,kx,c), optionally zero-padded along K.
    x3 (parity-grade fp16x3 operands): every tap becomes [hi(Ci) | lo(Ci)], hi = fp16(w), lo = fp16(w - hi); with
    ``kpad`` (the im2col'ed stem) the whole row is [hi(kpad) | lo(kpad)]."""
    co = w.shape[0]
    t = w.permute(0, 2, 3, 1).float()
    if not x3:
        m = t.reshape(co, -1)
        if kpad is not None and kpad > m.shape[1]:
            m = torch.cat([m, torch.zeros(co, kpad - m.shape[1], dtype=m.dtype)], 1)
        return m.contiguous().to(device=device, dtype=torch.float16)
    hi = t.half()
    lo = (t - hi.float()).half()
    if kpad is not None:
        mh, ml = hi.reshape(co, -1), lo.reshape(co, -1)
        z = torch.zeros(co, kpad - mh.shape[1], dtype=torch.float16)
        return torch.cat([mh, z, ml, z], 1).contiguous().to(device)
    return torch.cat([hi, lo], 3).reshape(co, -1).contiguous().to(device)


class _W:
    """Packed weights of one fused conv: fp16 K-major matrix + fp32 bias."""

    def __init__(self, w, b, device, kpad=None, x3=False):
        self.k = w.shape[2]
        self.cout, self.cin = w.shape[0], w.shape[1]
        self.w = _pack(w, device, kpad, x3)
        self.b = b.contiguous().to(device=device, dtype=torch.float32)
        self.flops_per_pixel = 2 * w.shape[0] * w.shape[1] * w.shape[2] * w.shape[3]


class YoloWeights:
    """Folded + packed parameters, from a state_dict in standin/yolov9e.py naming (``l{N}.…``, ``detect.…``);
    upstream archives name the same tensors ``model.{N}.…`` / ``model.42.…`` (see :func:`rename_upstream`)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device, nc: int | None = None, precision: str = "fp16"):
        """precision "fp16": fp16 operands / fp16 feature maps, fp32 accumulate (what the reference's CUDA path does under
        autocast, ref:util/yolov9.py:110-113).  "fp16x3": parity grade -- every feature map is an fp16 hi/lo pair and every
        conv issues hi*hi + hi*lo + lo*hi into the fp32 accumulator (22-bit operands), to reproduce the fp32 CPU path
        (ref:util/yolov9.py:114 nullcontext branch) box for box."""
        assert precision in ("fp16", "fp16x3")
        sd = _TrackedState({k: v.detach().cpu() for k, v in state_dict.items()})
        self.device = device
        self.precision = precision
        self.x3 = x3 = precision == "fp16x3"

        def _Wx(w, b, device, kpad=None):   # packs in the operand mode of this weight set
            return _W(w, b, device, kpad, x3)
        self.nc = nc if nc is not None else sd["detect.cv3.0.2.weight"].shape[0]
        W = {}

        def conv(name):
            w, b = _fold_conv_bn(sd, name)
            W[name] = _Wx(w, b, device)

        def elan(name):
            conv(name + ".cv1")
            for br in ("cv2", "cv3"):
                p = f"{name}.{br}.0"   # RepNCSP
                w1, b1 = _fold_conv_bn(sd, p + ".cv1")
                w2, b2 = _fold_conv_bn(sd, p + ".cv2")
                W[p + ".cv12"] = _Wx(torch.cat([w1, w2], 0), torch.cat([b1, b2], 0), device)   # merged 1x1 pair
                i = 0
                while f"{p}.m.{i}.cv2.conv.weight" in sd:
                    w, b = _fold_repconv(sd, f"{p}.m.{i}.cv1")
                    W[f"{p}.m.{i}.cv1"] = _Wx(w, b, device)
                    conv(f"{p}.m.{i}.cv2")
                    i += 1
                W[p + ".n"] = i
                conv(p + ".cv3")
                conv(f"{name}.{br}.1")
            conv(name + ".cv4")

        def adown(name):
            conv(name + ".cv1")
            conv(name + ".cv2")

        def cbl(name):
            W[name] = _Wx(sd[name + ".conv.weight"].float(), sd[name + ".conv.bias"].float(), device)

        # stem: l1 and l15 both read the image -> one GEMM with N = 128, K = 27 padded to 32
        w1, b1 = _fold_conv_bn(sd, "l1")
        w15, b15 = _fold_conv_bn(sd, "l15")
        W["stem"] = _Wx(torch.cat([w1, w15], 0), torch.cat([b1, b15], 0), device, kpad=32)
        conv("l2"); conv("l17")
        for n in (3, 5, 7, 9, 19, 22, 25, 28, 32, 35, 38, 41):
            elan(f"l{n}")
        for n in (4, 6, 8, 20, 23, 26, 36, 39):
            adown(f"l{n}")
        for n in (10, 11, 12, 13, 14):
            cbl(f"l{n}")
        conv("l29.cv1"); conv("l29.cv5")
        for i in range(3):
            wb, bb = _fold_conv_bn(sd, f"detect.cv2.{i}.0")
            wc, bc = _fold_conv_bn(sd, f"detect.cv3.{i}.0")
            W[f"head{i}.first"] = _Wx(torch.cat([wb, wc], 0), torch.cat([bb, bc], 0), device)
            wg, bg = _fold_conv_bn(sd, f"detect.cv2.{i}.1")
            W[f"head{i}.box1"] = _Wx(_dense_from_grouped(wg, 4), bg, device)
            W[f"head{i}.box2"] = _Wx(_dense_from_grouped(sd[f"detect.cv2.{i}.2.weight"].float(), 4),
                                    sd[f"detect.cv2.{i}.2.bias"].float(), device)
            conv(f"detect.cv3.{i}.1")
            W[f"head{i}.cls2"] = _Wx(sd[f"detect.cv3.{i}.2.weight"].float(), sd[f"detect.cv3.{i}.2.bias"].float(), device)
            self.c_box = wb.shape[0]
            self.c_cls = wc.shape[0]
        self.W = W
        # every tensor of the archive must have been consumed (a mis-named or unexpected parameter is an error, not a
        # silently different network), and the shapes must chain (checked layer by layer in YoloPlan._c1/_c3)
        for k in sd:
            if k.endswith(_DFL_SUFFIXES):   # the decode kernel hard-codes softmax(16 bins) . arange(16) (ref:util/yolov9.py head)
                t = sd[k].float().flatten()
                if t.numel() != 16 or not torch.equal(t, torch.arange(16.0)):
                    raise ValueError(f"{k}: DFL projection is not arange(16); this build's decode kernel assumes reg_max = 16")
        left = sorted(k for k in sd if k not in sd.used and not k.endswith(_IGNORED_SUFFIXES))
        if left:
            raise KeyError(f"YOLOv9-E archive has {len(left)} parameters this loader does not know: {left[:8]} ...")


def rename_upstream(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Map WongKinYiu/yolov9 parameter names (``model.N.*``; the detect head is the LAST module, ``model.42`` in
    yolov9-e) to the ``l{N}.`` / ``detect.`` naming used here.  Keys outside ``model.*`` are an error."""
    idx = sorted({int(k.split(".")[1]) for k in sd if k.startswith("model.") and k.split(".")[1].isdigit()})
    if not idx:
        raise KeyError("no model.N.* parameters in the archive")
    head = idx[-1]
    out = {}
    for k, v in sd.items():
        if not k.startswith("model."):
            raise KeyError(f"unexpected parameter outside model.*: {k}")
        n, rest = k[len("model."):].split(".", 1)
        out[("detect." if int(n) == head else f"l{n}.") + rest] = v
    return out


# --------------------------------------------------------------------------------------------- the plan
class YoloPlan:
    """Launch sequence + preallocated NHWC buffers for one (batch, canvas H, canvas W)."""

    def __init__(self, weights: YoloWeights, B: int, Hc: int, Wc: int, use_graph: bool = True):
        assert Hc % 32 == 0 and Wc % 32 == 0
        self.wts, self.B, self.Hc, self.Wc = weights, B, Hc, Wc
        self.dev = weights.device
        self.ops: List = []
        self.flops = 0
        self.x3 = weights.x3
        self.taps: Dict[str, Map] = {}
        self.canvas = torch.empty((B, Hc, Wc, 3), dtype=torch.uint8, device=self.dev)
        lut = (np.arange(256, dtype=np.float32) / np.float32(255.0))[None].repeat(3, 0)   # ref:util/yolov9.py:85
        self.lut = torch.from_numpy(lut.copy()).to(self.dev)
        self._build()
        self.graph = None
        self.use_graph = use_graph and os.environ.get("B2P_NO_GRAPH") is None   # eager launches for profiling

    # -- helpers that append launches
    def _fm(self, C, H, W):
        return ops.new_map(self.B, H, W, C, self.dev, x3=self.x3)

    def _c1(self, x: Map, wname, out: Map, act=ACT_SILU, out_f32=False):
        w = self.wts.W[wname]
        assert w.k == 1 and w.cin == x.C and w.cout == out.C, (wname, w.cin, x.C, w.cout, out.C)
        self.flops += w.flops_per_pixel * x.B * x.H * x.W
        self.ops.append(lambda: ops.conv1x1(x, w.w, out, w.b, None, act, out_f32))

    def _c3(self, x: Map, wname, out: Map, stride=1, res: Map | None = None, act=ACT_SILU):
        w = self.wts.W[wname]
        assert w.k == 3 and w.cin == x.C and w.cout == out.C, (wname, w.cin, x.C, w.cout, out.C)
        self.flops += w.flops_per_pixel * out.B * out.H * out.W
        self.ops.append(lambda: ops.conv3x3(x, w.w, out, stride, w.b, res, act))

    def _elan(self, name, x: Map, out: Map, c3, c4):
        cat = self._fm(c3 + 2 * c4, x.H, x.W)
        self._c1(x, name + ".cv1", cat.slice(0, c3))
        src = cat.slice(c3 // 2, c3 // 2)
        for bi, br in enumerate(("cv2", "cv3")):
            p = f"{name}.{br}.0"
            c_ = c4 // 2
            U = self._fm(2 * c_, x.H, x.W)
            self._c1(src, p + ".cv12", U)
            t = U.slice(0, c_)
            n = self.wts.W[p + ".n"]
            for i in range(n):
                h = self._fm(c_, x.H, x.W)
                self._c3(t, f"{p}.m.{i}.cv1", h)
                dst = U.slice(0, c_) if i == n - 1 else self._fm(c_, x.H, x.W)
                self._c3(h, f"{p}.m.{i}.cv2", dst, res=t)
                t = dst
            V = self._fm(c4, x.H, x.W)
            self._c1(U, p + ".cv3", V)
            dst = cat.slice(c3 + bi * c4, c4)
            self._c3(V, f"{name}.{br}.1", dst)
            src = dst
        self._c1(cat, name + ".cv4", out)

    def _adown(self, name, x: Map, out: Map):
        x1 = self._fm(x.C // 2, x.H, x.W)
        x2 = self._fm(x.C // 2, x.H // 2, x.W // 2)
        f_ = lambda: ops.adown_pool(x, x1, x2)
        f_.n_kernels = 1 if self.x3 else 2      # plain fp16 maps: separate average / max kernels (csrc/detect_ops.cu)
        self.ops.append(f_)
        half = out.C // 2
        self._c3(x1, name + ".cv1", out.slice(0, half), stride=2)
        self._c1(x2, name + ".cv2", out.slice(half, half))

    def _cbfuse(self, srcs, last: Map, out: Map):
        self.ops.append(lambda: ops.cbfuse(srcs, last, out))

    def _build(self):
        B, H1, W1 = self.B, self.Hc // 2, self.Wc // 2
        wts = self.wts
        # stem
        KX = 2 if self.x3 else 1
        self.A0 = torch.empty((B * H1 * W1, KX * 32), dtype=torch.float16, device=self.dev)
        self.ops.append(lambda: ops.im2col_u8(self.canvas, B, self.Hc, self.Wc, 3, 2, 1, 32, self.lut, self.A0, split=self.x3))
        S = self._fm(128, H1, W1)
        ws = wts.W["stem"]
        self.flops += 2 * 128 * 27 * B * H1 * W1
        A0m = ops.Map(self.A0.view(B, H1, W1, KX * 32), 0, 32, 32 if self.x3 else 0)   # im2col rows as a 1x1 "map"
        self.ops.append(lambda: ops.conv1x1(A0m, ws.w, S, ws.b, None, ACT_SILU))
        x1, x15 = S.slice(0, 64), S.slice(64, 64)
        H2, W2, H3, W3, H4, W4, H5, W5 = H1 // 2, W1 // 2, H1 // 4, W1 // 4, H1 // 8, W1 // 8, H1 // 16, W1 // 16
        x2 = self._fm(128, H2, W2); self._c3(x1, "l2", x2, stride=2)
        x3 = self._fm(256, H2, W2); self._elan("l3", x2, x3, 128, 64)
        x4 = self._fm(256, H3, W3); self._adown("l4", x3, x4)
        x5 = self._fm(512, H3, W3); self._elan("l5", x4, x5, 256, 128)
        x6 = self._fm(512, H4, W4); self._adown("l6", x5, x6)
        x7 = self._fm(1024, H4, W4); self._elan("l7", x6, x7, 512, 256)
        x8 = self._fm(1024, H5, W5); self._adown("l8", x7, x8)
        x9 = self._fm(1024, H5, W5); self._elan("l9", x8, x9, 512, 256)
        r10 = self._fm(64, H1, W1); self._c1(x1, "l10", r10, ACT_NONE)
        r11 = self._fm(192, H2, W2); self._c1(x3, "l11", r11, ACT_NONE)
        r12 = self._fm(448, H3, W3); self._c1(x5, "l12", r12, ACT_NONE)
        r13 = self._fm(960, H4, W4); self._c1(x7, "l13", r13, ACT_NONE)
        r14 = self._fm(1984, H5, W5); self._c1(x9, "l14", r14, ACT_NONE)
        x16 = self._fm(64, H1, W1)
        self._cbfuse([r10.slice(0, 64), r11.slice(0, 64), r12.slice(0, 64), r13.slice(0, 64), r14.slice(0, 64)], x15, x16)
        x17 = self._fm(128, H2, W2); self._c3(x16, "l17", x17, stride=2)
        x18 = self._fm(128, H2, W2)
        self._cbfuse([r11.slice(64, 128), r12.slice(64, 128), r13.slice(64, 128), r14.slice(64, 128)], x17, x18)
        x19 = self._fm(256, H2, W2); self._elan("l19", x18, x19, 128, 64)
        x20 = self._fm(256, H3, W3); self._adown("l20", x19, x20)
        x21 = self._fm(256, H3, W3)
        self._cbfuse([r12.slice(192, 256), r13.slice(192, 256), r14.slice(192, 256)], x20, x21)
        cat34 = self._fm(1024, H3, W3)
        x22 = cat34.slice(512, 512); self._elan("l22", x21, x22, 256, 128)
        x23 = self._fm(512, H4, W4); self._adown("l23", x22, x23)
        x24 = self._fm(512, H4, W4); self._cbfuse([r13.slice(448, 512), r14.slice(448, 512)], x23, x24)
        cat31 = self._fm(1536, H4, W4)
        x25 = cat31.slice(512, 1024); self._elan("l25", x24, x25, 512, 256)
        x26 = self._fm(1024, H5, W5); self._adown("l26", x25, x26)
        x27 = self._fm(1024, H5, W5); self._cbfuse([r14.slice(960, 1024)], x26, x27)
        x28 = self._fm(1024, H5, W5); self._elan("l28", x27, x28, 512, 256)
        # head
        cat40 = self._fm(1024, H5, W5)
        x29 = cat40.slice(512, 512)
        sp = self._fm(1024, H5, W5)
        self._c1(x28, "l29.cv1", sp.slice(0, 256))
        for i in range(3):
            a, b = sp.slice(256 * i, 256), sp.slice(256 * (i + 1), 256)
            self.ops.append(lambda a=a, b=b: ops.maxpool_s1(a, b, 5))
        self._c1(sp, "l29.cv5", x29)
        up = cat31.slice(0, 512); self.ops.append(lambda: ops.upsample2x(x29, up))
        cat37 = self._fm(768, H4, W4)
        x32 = cat37.slice(256, 512); self._elan("l32", cat31, x32, 512, 256)
        up2 = cat34.slice(0, 512); self.ops.append(lambda: ops.upsample2x(x32, up2))
        x35 = self._fm(256, H3, W3); self._elan("l35", cat34, x35, 256, 128)
        self._adown("l36", x35, cat37.slice(0, 256))
        x38 = self._fm(512, H4, W4); self._elan("l38", cat37, x38, 512, 256)
        self._adown("l39", x38, cat40.slice(0, 512))
        x41 = self._fm(512, H5, W5); self._elan("l41", cat40, x41, 1024, 512)
        # detect head
        self.cls_out, self.box_out, self.hw = [], [], []
        nc = wts.nc
        for i, x in enumerate((x35, x38, x41)):
            cb, cc = wts.c_box, wts.c_cls
            F = self._fm(cb + cc, x.H, x.W)
            self._c3(x, f"head{i}.first", F)
            b1 = self._fm(cb, x.H, x.W); self._c3(F.slice(0, cb), f"head{i}.box1", b1)
            bo = ops.new_map(B, x.H, x.W, 64, self.dev, torch.float32)
            self._c1(b1, f"head{i}.box2", bo, ACT_NONE, out_f32=True)
            c1 = self._fm(cc, x.H, x.W); self._c3(F.slice(cb, cc), f"detect.cv3.{i}.1", c1)
            co = ops.new_map(B, x.H, x.W, nc, self.dev, torch.float32)
            self._c1(c1, f"head{i}.cls2", co, ACT_NONE, out_f32=True)
            self.cls_out.append(co.buf); self.box_out.append(bo.buf); self.hw.append((x.H, x.W))
        self.taps.update(x1=x1, x2=x2, x3=x3, x5=x5, x7=x7, x9=x9, x16=x16, x18=x18, x19=x19, x22=x22, x25=x25,
                         x28=x28, x29=x29, x32=x32, x35=x35, x38=x38, x41=x41)
        self.n_launches = sum(getattr(f, "n_kernels", 1) for f in self.ops)

    def run(self):
        """Run the recorded launches on the current stream (canvas -> head tensors)."""
        if not self.use_graph:
            for f in self.ops:
                f()
            return
        if self.graph is None:
            for f in self.ops:   # warm-up (also creates the cached LANCZOS tables etc. outside capture)
                f()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with ops.CAPTURE_LOCK, torch.cuda.graph(g, stream=ops.role_stream('yolo', self.dev), capture_error_mode="thread_local"):
                for f in self.ops:
                    f()
            self.graph = g
        self.graph.replay()
        ops.count_graph_launches(self.n_launches)
