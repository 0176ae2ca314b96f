"""The host-only launch planner of the wgmma GEMM/conv kernel (``b2p_gemm_plan``) seen from Python: one plan as a dict of
named fields, and the path class a plan reduces to.  Shared by the CPU plan checks and the GPU path tests; needs no GPU."""
from __future__ import annotations

import ctypes as C

from omniparser_b200 import _lib

# field order of b2p_gemm_plan (include/b200parse.h)
PLAN_FIELDS = ("mode", "bk", "bn", "ksplit", "kb_per", "kb_merge", "stages", "stagesA", "sep", "bres", "nb", "tw", "tw_valid",
               "th", "m_tiles", "n_tiles", "mt_fast", "grid", "smem", "vec_ok", "split", "res_lo", "park",
               "x3", "num_kb", "taps", "a_bytes", "a_slot", "b_bytes", "b_slot", "tiles_x", "tiles_y",
               "rank_a", "box_a0", "box_a1", "box_a2", "box_a3", "box_a4", "box_b0", "box_b1", "extent_a", "extent_b",
               "swizzle_a", "swizzle_b", "swizzle_desc")
FLAG_PARK = 32                     # b2p_gemm_plan only: the park-only GEMM of b2p_gemm_ln
H100_SXM = (132, 232448)           # SMs, opt-in shared memory per block (bytes): H100 SXM5 data sheet
H100_PCIE = (114, 232448)          # H100 PCIe
BN_INSTANTIATIONS = (256, 192, 128, 96, 64, 48, 32, 16)
GEMM_CALLS = ("b2p_gemm", "b2p_gemm_planes", "b2p_conv3x3", "b2p_conv3x3_planes", "b2p_gemm_ln")


def planner_args(name, a):
    """positional arguments of b2p_gemm_plan (without num_sms, max_smem, out) for one recorded GEMM/conv call"""
    if name in ("b2p_gemm", "b2p_gemm_planes"):
        A, lda, B, M, N, K, out, ldc, bias, res, ldr, act, flags = a[:13]
        lo = tuple(a[13:16]) if name == "b2p_gemm_planes" else (0, 0, 0)
        return (A, lda, M, 1, 1, K, 0, B, N, out, ldc, bias, res, ldr, act, flags) + lo
    if name in ("b2p_conv3x3", "b2p_conv3x3_planes"):
        lo = tuple(a[16:19]) if name == "b2p_conv3x3_planes" else (0, 0, 0)
        return tuple(a[:16]) + lo
    if name == "b2p_gemm_ln":      # what b2p_gemm_ln hands the launcher: fp32 partial tiles parked in the workspace
        A, lda, B, M, N, K = a[:6]
        flags = a[16]
        return (A, lda, M, 1, 1, K, 0, B, N, None, N, None, None, 0, 0, (flags & 0x1ff08) | 2 | FLAG_PARK, 0, 0, 0)
    raise KeyError(name)


def plan(args, num_sms=H100_SXM[0], max_smem=H100_SXM[1]):
    """-> dict of the plan fields, or raises B2PError with the planner's rejection"""
    out = (C.c_int * len(PLAN_FIELDS))()
    _lib.check(_lib.lib().b2p_gemm_plan(*args, num_sms, max_smem, out))
    return dict(zip(PLAN_FIELDS, out))


def last_plan():
    """the plan fields of this thread's most recent GEMM/conv launch: what was actually launched"""
    out = (C.c_int * len(PLAN_FIELDS))()
    _lib.check(_lib.lib().b2p_gemm_last_plan(out))
    return dict(zip(PLAN_FIELDS, out))


def path_class(p, args):
    """(mode, bk, bn, split-K, park, bres, nb>1, mt_fast, x3, kb_merge, vec_ok, split out, res_lo, out_f32, residual, act)"""
    flags = args[15]
    return (p["mode"], p["bk"], p["bn"], int(p["ksplit"] > 1), p["park"], p["bres"], int(p["nb"] > 1), p["mt_fast"], p["x3"],
            p["kb_merge"], p["vec_ok"], int(p["split"] > 0), int(p["res_lo"] > 0), (flags >> 1) & 1, int(bool(args[12])), args[14])
