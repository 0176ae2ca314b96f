"""GPU: every dispatch path of the wgmma GEMM/conv kernel against fp64, with a per-element error bound.

The case list has one case per path class the production plans reach (test_gemm_plan_cpu.py records the classes and checks
that this list covers them, every N-tile instantiation and both k-block widths) plus the tiling edges: M below and not a
multiple of 128, N not a multiple of the N tile / of 16 / below 16, conv maps that the spatial tile does not divide, whole-
image tiles over a batch that is not a multiple of the images per tile, split-K slices that do not divide the k-blocks or
the 128 reduction rows, unaligned outputs (scalar epilogue), channel slices with lo planes, bf16 operands.

Before each launch: the plan (``b2p_gemm_plan`` at this device's SM count and shared memory) must be the case's CPU path
class; every buffer is allocated from a computed extent that covers what the tensor maps can address and the epilogue can
write, and everything outside the operands / the written slice is NaN.  The plan line is printed, flushed, first.
After: the written slice is compared with fp64 (operands exactly as stored: fp16 / bf16 values, hi + lo for fp16x3) to
    c * K_eff * 2^-23 * sum|a||b|  (fp32 accumulation)  + output rounding (fp16 half ulp, 2^-22 for a [hi | lo] pair, fp32)
    + the SiLU / GELU approximation + for fp16x3 the omitted lo*lo term,
everything outside it must still be NaN, split outputs must be canonical pairs, and split-K launches must repeat bit for bit.
"""
from __future__ import annotations

import math
from collections import namedtuple

import pytest

from gemm_plan_util import FLAG_PARK, H100_SXM, last_plan, path_class, plan

Case = namedtuple("Case", "name B H W K N stride lda ldc ldr flags act bias res lo_a lo_out lo_res a_off out_off res_off expect",
                  defaults=(0, 0, 0, None))
F_BF16, F_F32, F_SPLIT, F_X3, F_NOSPLIT = 1, 2, 4, 8, 16


def P(B, H, W, K, N, stride, lda, ldc, ldr, flags, act, bias, res, lo_a, lo_out, lo_res, name="production"):
    return Case(name, B, H, W, K, N, stride, lda, ldc, ldr, flags, act, bias, res, lo_a, lo_out, lo_res)


# one production call per path class: the smallest call of the class in the plans test_gemm_plan_cpu.py records
# (GEMM: B = M, H = W = 1, K = reduction; conv: B, H, W, K = Cin).  Columns as Case.
PRODUCTION = [
    P(400, 1, 1, 256, 1, 0, 512, 1, 0, 10, 0, 1, 0, 256, 0, 0),  # yolo B1 fp16x3
    P(400, 1, 1, 64, 64, 0, 128, 64, 0, 10, 0, 1, 0, 64, 0, 0),  # yolo B1 fp16x3
    P(16, 1, 1, 768, 768, 0, 1536, 768, 768, 10, 0, 1, 1, 0, 0, 0),  # florence 768 K16 fp16x3
    P(800, 1, 1, 1024, 256, 0, 2048, 2048, 0, 12, 1, 1, 0, 1024, 1024, 0),  # yolo B2 fp16x3
    P(160, 1, 1, 1024, 768, 0, 2048, 768, 0, 10, 0, 0, 0, 0, 0, 0),  # florence 64 K32 fp16x3
    P(32, 1, 1, 768, 768, 0, 1536, 768, 0, 42, 0, 0, 0, 0, 0, 0),  # florence 64 K32 fp16x3 B2P_GEMM_LN=1
    P(800, 1, 1, 64, 64, 0, 128, 64, 0, 10, 0, 1, 0, 64, 0, 0),  # yolo B2 fp16x3
    P(512, 1, 1, 512, 512, 0, 1024, 512, 512, 10, 0, 1, 1, 0, 0, 0),  # florence 64 K32 fp16x3
    P(400, 1, 1, 256, 256, 0, 2048, 512, 0, 12, 1, 1, 0, 1024, 256, 0),  # yolo B1 fp16x3
    P(16, 1, 1, 768, 3072, 0, 1536, 6144, 0, 12, 2, 1, 0, 0, 0, 0),  # florence 768 K16 fp16x3
    P(512, 1, 1, 768, 768, 0, 1536, 768, 0, 10, 0, 1, 0, 0, 0, 0),  # florence 64 K512 fp16x3
    P(416, 1, 1, 768, 768, 0, 1536, 768, 768, 10, 0, 1, 1, 0, 0, 0),  # florence 64 K32 fp16x3
    P(400, 1, 1, 512, 512, 0, 1024, 2048, 0, 12, 1, 1, 0, 512, 1024, 0),  # yolo B1 fp16x3
    P(2048, 1, 1, 1024, 256, 0, 2048, 256, 256, 10, 0, 1, 1, 0, 0, 0),  # florence 64 K32 fp16x3
    P(128, 1, 1, 1024, 4096, 0, 2048, 8192, 0, 12, 2, 1, 0, 0, 0, 0),  # florence 64 K32 fp16x3
    P(400, 1, 1, 1024, 1024, 0, 2048, 2048, 0, 12, 1, 1, 0, 1024, 1024, 0),  # yolo B1 fp16x3
    P(16, 1, 1, 3072, 768, 0, 6144, 768, 768, 10, 0, 1, 1, 0, 0, 0),  # florence 768 K16 fp16x3
    P(400, 1, 1, 1024, 256, 0, 2048, 2048, 0, 12, 1, 1, 0, 1024, 1024, 0),  # yolo B1 fp16x3
    P(32, 1, 1, 3072, 768, 0, 6144, 768, 0, 42, 0, 0, 0, 0, 0, 0),  # florence 64 K32 fp16x3 B2P_GEMM_LN=1
    P(6400, 1, 1, 64, 64, 0, 128, 64, 0, 10, 0, 1, 0, 64, 0, 0),  # yolo B1 fp16x3
    P(2048, 1, 1, 256, 256, 0, 512, 256, 256, 10, 0, 1, 1, 0, 0, 0),  # florence 64 K32 fp16x3
    P(102400, 1, 1, 64, 64, 0, 256, 128, 0, 12, 0, 1, 0, 128, 64, 0),  # yolo B1 fp16x3
    P(3200, 1, 1, 128, 128, 0, 256, 1536, 0, 12, 1, 1, 0, 128, 768, 0),  # yolo B2 fp16x3
    P(512, 1, 1, 512, 1536, 0, 1024, 1536, 0, 10, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16x3
    P(400, 1, 1, 1024, 1984, 0, 2048, 3968, 0, 12, 0, 1, 0, 1024, 1984, 0),  # yolo B1 fp16x3
    P(800, 1, 1, 1024, 1024, 0, 2048, 2048, 0, 12, 1, 1, 0, 1024, 1024, 0),  # yolo B2 fp16x3
    P(512, 1, 1, 2304, 512, 0, 4608, 512, 0, 10, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16x3
    P(128, 1, 1, 4096, 1024, 0, 8192, 1024, 1024, 10, 0, 1, 1, 0, 0, 0),  # florence 64 K32 fp16x3
    P(416, 1, 1, 768, 2304, 0, 1536, 2304, 0, 10, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16x3
    P(512, 1, 1, 512, 2048, 0, 1024, 4096, 0, 12, 2, 1, 0, 0, 0, 0),  # florence 64 K32 fp16x3
    P(512, 1, 1, 2048, 512, 0, 4096, 512, 512, 10, 0, 1, 1, 0, 0, 0),  # florence 64 K32 fp16x3
    P(400, 1, 1, 2048, 512, 0, 4096, 1024, 0, 12, 1, 1, 0, 2048, 512, 0),  # yolo B1 fp16x3
    P(8192, 1, 1, 160, 128, 0, 160, 128, 0, 2, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16
    P(8192, 1, 1, 160, 128, 0, 320, 128, 0, 10, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16x3
    P(102400, 1, 1, 32, 128, 0, 64, 256, 0, 12, 1, 1, 0, 32, 128, 0),  # yolo B1 fp16x3
    P(2048, 1, 1, 256, 768, 0, 512, 768, 0, 10, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16x3
    P(8192, 1, 1, 128, 128, 0, 256, 128, 128, 10, 0, 1, 1, 0, 0, 0),  # florence 64 K32 fp16x3
    P(1600, 1, 1, 1024, 960, 0, 2048, 1920, 0, 12, 0, 1, 0, 1024, 960, 0),  # yolo B1 fp16x3
    P(12800, 1, 1, 128, 128, 0, 256, 1536, 0, 12, 1, 1, 0, 128, 768, 0),  # yolo B8 fp16x3
    P(800, 1, 1, 1024, 1984, 0, 2048, 3968, 0, 12, 0, 1, 0, 1024, 1984, 0),  # yolo B2 fp16x3
    P(416, 1, 1, 768, 3072, 0, 1536, 6144, 0, 12, 2, 1, 0, 0, 0, 0),  # florence 64 K32 fp16x3
    P(102400, 1, 1, 32, 128, 0, 32, 128, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(131072, 1, 1, 160, 128, 0, 160, 128, 0, 2, 0, 1, 0, 0, 0, 0),  # florence 64 K512 fp16
    P(800, 1, 1, 2048, 512, 0, 4096, 1024, 0, 12, 1, 1, 0, 2048, 512, 0),  # yolo B2 fp16x3
    P(416, 1, 1, 3072, 768, 0, 6144, 768, 768, 10, 0, 1, 1, 0, 0, 0),  # florence 64 K32 fp16x3
    P(8192, 1, 1, 128, 384, 0, 256, 384, 0, 10, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16x3
    P(2048, 1, 1, 1024, 1024, 0, 2048, 1024, 1024, 10, 0, 1, 1, 0, 0, 0),  # florence 64 K512 fp16x3
    P(25600, 1, 1, 256, 192, 0, 512, 384, 0, 12, 0, 1, 0, 256, 192, 0),  # yolo B1 fp16x3
    P(2048, 1, 1, 256, 1024, 0, 512, 2048, 0, 12, 2, 1, 0, 0, 0, 0),  # florence 64 K32 fp16x3
    P(2048, 1, 1, 1024, 3072, 0, 2048, 3072, 0, 10, 0, 1, 0, 0, 0, 0),  # florence 64 K512 fp16x3
    P(16, 1, 1, 768, 51290, 0, 1536, 51296, 0, 10, 0, 0, 0, 0, 0, 0),  # florence 768 K16 fp16x3
    P(32768, 1, 1, 256, 256, 0, 512, 256, 256, 10, 0, 1, 1, 0, 0, 0),  # florence 64 K512 fp16x3
    P(6400, 1, 1, 512, 448, 0, 1024, 896, 0, 12, 0, 1, 0, 512, 448, 0),  # yolo B1 fp16x3
    P(12800, 1, 1, 256, 256, 0, 512, 1024, 0, 12, 1, 1, 0, 256, 512, 0),  # yolo B8 fp16x3
    P(8192, 1, 1, 128, 512, 0, 256, 1024, 0, 12, 2, 1, 0, 0, 0, 0),  # florence 64 K32 fp16x3
    P(512, 1, 1, 768, 51290, 0, 1536, 51296, 0, 10, 0, 0, 0, 0, 0, 0),  # florence 64 K512 fp16x3
    P(2048, 1, 1, 1024, 4096, 0, 2048, 8192, 0, 12, 2, 1, 0, 0, 0, 0),  # florence 64 K512 fp16x3
    P(2048, 1, 1, 4608, 1024, 0, 9216, 1024, 0, 10, 0, 1, 0, 0, 0, 0),  # florence 64 K512 fp16x3
    P(2048, 1, 1, 4096, 1024, 0, 8192, 1024, 1024, 10, 0, 1, 1, 0, 0, 0),  # florence 64 K512 fp16x3
    P(400, 1, 1, 256, 1, 0, 256, 1, 0, 2, 0, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(400, 1, 1, 1024, 256, 0, 1024, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(400, 1, 1, 64, 64, 0, 64, 64, 0, 2, 0, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(16, 1, 1, 768, 768, 0, 768, 768, 768, 2, 0, 1, 1, 0, 0, 0),  # florence 768 K16 fp16
    P(51200, 1, 1, 256, 1, 0, 256, 1, 0, 2, 0, 1, 0, 0, 0, 0),  # yolo B8 fp16
    P(400, 1, 1, 256, 256, 0, 1024, 256, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(800, 1, 1, 64, 64, 0, 64, 64, 0, 2, 0, 1, 0, 0, 0, 0),  # yolo B2 fp16
    P(512, 1, 1, 512, 512, 0, 512, 512, 512, 2, 0, 1, 1, 0, 0, 0),  # florence 64 K32 fp16
    P(400, 1, 1, 512, 512, 0, 512, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(160, 1, 1, 1024, 768, 0, 1024, 768, 0, 2, 0, 0, 0, 0, 0, 0),  # florence 64 K32 fp16
    P(800, 1, 1, 512, 512, 0, 512, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B2 fp16
    P(16, 1, 1, 768, 3072, 0, 768, 3072, 0, 0, 2, 1, 0, 0, 0, 0),  # florence 768 K16 fp16
    P(2048, 1, 1, 1024, 256, 0, 1024, 256, 256, 2, 0, 1, 1, 0, 0, 0),  # florence 64 K32 fp16
    P(400, 1, 1, 1024, 1024, 0, 1024, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(512, 1, 1, 768, 768, 0, 768, 768, 0, 2, 0, 1, 0, 0, 0, 0),  # florence 64 K512 fp16
    P(416, 1, 1, 768, 768, 0, 768, 768, 768, 2, 0, 1, 1, 0, 0, 0),  # florence 64 K32 fp16
    P(16, 1, 1, 3072, 768, 0, 3072, 768, 768, 2, 0, 1, 1, 0, 0, 0),  # florence 768 K16 fp16
    P(3200, 1, 1, 128, 128, 0, 128, 768, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B2 fp16
    P(3200, 1, 1, 64, 64, 0, 64, 64, 0, 2, 0, 1, 0, 0, 0, 0),  # yolo B8 fp16
    P(2048, 1, 1, 256, 256, 0, 256, 256, 256, 2, 0, 1, 1, 0, 0, 0),  # florence 64 K32 fp16
    P(400, 1, 1, 1024, 1984, 0, 1024, 1984, 0, 0, 0, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(800, 1, 1, 1024, 1024, 0, 1024, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B2 fp16
    P(512, 1, 1, 512, 1536, 0, 512, 1536, 0, 2, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16
    P(102400, 1, 1, 64, 64, 0, 128, 64, 0, 0, 0, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(25600, 1, 1, 64, 64, 0, 256, 64, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(51200, 1, 1, 64, 64, 0, 64, 64, 0, 2, 0, 1, 0, 0, 0, 0),  # yolo B8 fp16
    P(512, 1, 1, 2304, 512, 0, 2304, 512, 0, 2, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16
    P(512, 1, 1, 512, 2048, 0, 512, 2048, 0, 0, 2, 1, 0, 0, 0, 0),  # florence 64 K32 fp16
    P(416, 1, 1, 768, 2304, 0, 768, 2304, 0, 2, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16
    P(416, 1, 1, 3072, 768, 0, 3072, 768, 768, 2, 0, 1, 1, 0, 0, 0),  # florence 64 K32 fp16
    P(1600, 1, 1, 1024, 960, 0, 1024, 960, 0, 0, 0, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(12800, 1, 1, 128, 128, 0, 128, 768, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B8 fp16
    P(2048, 1, 1, 256, 768, 0, 256, 768, 0, 2, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16
    P(8192, 1, 1, 128, 128, 0, 128, 128, 128, 2, 0, 1, 1, 0, 0, 0),  # florence 64 K32 fp16
    P(800, 1, 1, 1024, 1984, 0, 1024, 1984, 0, 0, 0, 1, 0, 0, 0, 0),  # yolo B2 fp16
    P(416, 1, 1, 768, 3072, 0, 768, 3072, 0, 0, 2, 1, 0, 0, 0, 0),  # florence 64 K32 fp16
    P(25600, 1, 1, 128, 128, 0, 128, 256, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(131072, 1, 1, 128, 128, 0, 128, 128, 128, 2, 0, 1, 1, 0, 0, 0),  # florence 64 K512 fp16
    P(3200, 1, 1, 1024, 960, 0, 1024, 960, 0, 0, 0, 1, 0, 0, 0, 0),  # yolo B2 fp16
    P(2048, 1, 1, 256, 1024, 0, 256, 1024, 0, 0, 2, 1, 0, 0, 0, 0),  # florence 64 K32 fp16
    P(8192, 1, 1, 128, 384, 0, 128, 384, 0, 2, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16
    P(2048, 1, 1, 1024, 1024, 0, 1024, 1024, 1024, 2, 0, 1, 1, 0, 0, 0),  # florence 64 K512 fp16
    P(2048, 1, 1, 1024, 3072, 0, 1024, 3072, 0, 2, 0, 1, 0, 0, 0, 0),  # florence 64 K512 fp16
    P(25600, 1, 1, 256, 192, 0, 256, 192, 0, 0, 0, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(6400, 1, 1, 512, 448, 0, 512, 448, 0, 0, 0, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(12800, 1, 1, 256, 256, 0, 256, 512, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B8 fp16
    P(8192, 1, 1, 128, 512, 0, 128, 512, 0, 0, 2, 1, 0, 0, 0, 0),  # florence 64 K32 fp16
    P(16, 1, 1, 768, 51290, 0, 768, 51296, 0, 2, 0, 0, 0, 0, 0, 0),  # florence 768 K16 fp16
    P(8192, 1, 1, 512, 512, 0, 512, 512, 512, 2, 0, 1, 1, 0, 0, 0),  # florence 64 K512 fp16
    P(2048, 1, 1, 1024, 4096, 0, 1024, 4096, 0, 0, 2, 1, 0, 0, 0, 0),  # florence 64 K512 fp16
    P(512, 1, 1, 768, 51290, 0, 768, 51296, 0, 2, 0, 0, 0, 0, 0, 0),  # florence 64 K512 fp16
    P(25600, 1, 1, 256, 256, 0, 256, 256, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(32768, 1, 1, 256, 256, 0, 256, 256, 256, 2, 0, 1, 1, 0, 0, 0),  # florence 64 K512 fp16
    P(1, 20, 20, 64, 64, 1, 640, 128, 0, 12, 1, 1, 0, 320, 64, 0),  # yolo B1 fp16x3
    P(1, 160, 160, 32, 32, 1, 128, 64, 0, 12, 1, 1, 0, 64, 32, 0),  # yolo B1 fp16x3
    P(1, 160, 160, 32, 32, 1, 64, 64, 128, 12, 1, 1, 1, 32, 32, 64),  # yolo B1 fp16x3
    P(8, 20, 20, 64, 64, 1, 640, 128, 0, 12, 1, 1, 0, 320, 64, 0),  # yolo B8 fp16x3
    P(1, 80, 80, 64, 64, 1, 128, 128, 256, 12, 1, 1, 1, 64, 64, 128),  # yolo B1 fp16x3
    P(1, 20, 20, 128, 128, 1, 512, 256, 0, 12, 1, 1, 0, 256, 128, 0),  # yolo B1 fp16x3
    P(1, 20, 20, 128, 128, 1, 256, 256, 512, 12, 1, 1, 1, 128, 128, 256),  # yolo B1 fp16x3
    P(8, 20, 20, 128, 128, 1, 512, 256, 0, 12, 1, 1, 0, 256, 128, 0),  # yolo B8 fp16x3
    P(8, 20, 20, 128, 128, 1, 256, 256, 512, 12, 1, 1, 1, 128, 128, 256),  # yolo B8 fp16x3
    P(1, 40, 40, 128, 128, 1, 512, 256, 0, 12, 1, 1, 0, 256, 128, 0),  # yolo B1 fp16x3
    P(1, 40, 40, 128, 128, 1, 256, 256, 512, 12, 1, 1, 1, 128, 128, 256),  # yolo B1 fp16x3
    P(8, 40, 40, 64, 64, 1, 640, 128, 0, 12, 1, 1, 0, 320, 64, 0),  # yolo B8 fp16x3
    P(2, 80, 80, 64, 64, 1, 128, 128, 256, 12, 1, 1, 1, 64, 64, 128),  # yolo B2 fp16x3
    P(1, 20, 20, 256, 256, 1, 512, 2048, 0, 12, 1, 1, 0, 256, 1024, 0),  # yolo B1 fp16x3
    P(1, 20, 20, 256, 256, 1, 512, 512, 1024, 12, 1, 1, 1, 256, 256, 512),  # yolo B1 fp16x3
    P(1, 20, 20, 512, 512, 1, 1024, 4096, 0, 12, 1, 1, 0, 512, 2048, 0),  # yolo B1 fp16x3
    P(8, 40, 40, 128, 128, 1, 512, 256, 0, 12, 1, 1, 0, 256, 128, 0),  # yolo B8 fp16x3
    P(8, 40, 40, 128, 128, 1, 256, 256, 512, 12, 1, 1, 1, 128, 128, 256),  # yolo B8 fp16x3
    P(1, 40, 40, 256, 256, 1, 512, 2048, 0, 12, 1, 1, 0, 256, 1024, 0),  # yolo B1 fp16x3
    P(1, 80, 80, 256, 320, 1, 512, 640, 0, 12, 1, 1, 0, 256, 320, 0),  # yolo B1 fp16x3
    P(2, 20, 20, 512, 512, 1, 1024, 4096, 0, 12, 1, 1, 0, 512, 2048, 0),  # yolo B2 fp16x3
    P(8, 40, 40, 256, 256, 1, 512, 2048, 0, 12, 1, 1, 0, 256, 1024, 0),  # yolo B8 fp16x3
    P(8, 20, 20, 256, 256, 1, 512, 2048, 0, 12, 1, 1, 0, 256, 1024, 0),  # yolo B8 fp16x3
    P(8, 20, 20, 256, 256, 1, 512, 512, 1024, 12, 1, 1, 1, 256, 256, 512),  # yolo B8 fp16x3
    P(2, 80, 80, 128, 128, 2, 256, 1536, 0, 12, 1, 1, 0, 128, 768, 0),  # yolo B2 fp16x3
    P(32, 16, 16, 128, 256, 2, 256, 256, 0, 10, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16x3
    P(1, 80, 80, 128, 128, 2, 256, 1536, 0, 12, 1, 1, 0, 128, 768, 0),  # yolo B1 fp16x3
    P(1, 160, 160, 128, 128, 2, 256, 512, 0, 12, 1, 1, 0, 128, 256, 0),  # yolo B1 fp16x3
    P(1, 40, 40, 256, 256, 2, 512, 2048, 0, 12, 1, 1, 0, 256, 1024, 0),  # yolo B1 fp16x3
    P(1, 40, 40, 512, 512, 2, 1024, 2048, 0, 12, 1, 1, 0, 512, 1024, 0),  # yolo B1 fp16x3
    P(8, 80, 80, 128, 128, 2, 256, 1536, 0, 12, 1, 1, 0, 128, 768, 0),  # yolo B8 fp16x3
    P(1, 80, 80, 256, 256, 2, 512, 1024, 0, 12, 1, 1, 0, 256, 512, 0),  # yolo B1 fp16x3
    P(2, 40, 40, 512, 512, 2, 1024, 2048, 0, 12, 1, 1, 0, 512, 1024, 0),  # yolo B2 fp16x3
    P(16, 192, 192, 128, 256, 2, 256, 256, 0, 10, 0, 1, 0, 0, 0, 0),  # florence 768 K16 fp16x3
    P(8, 80, 80, 256, 256, 2, 512, 1024, 0, 12, 1, 1, 0, 256, 512, 0),  # yolo B8 fp16x3
    P(512, 16, 16, 128, 256, 2, 256, 256, 0, 10, 0, 1, 0, 0, 0, 0),  # florence 64 K512 fp16x3
    P(8, 40, 40, 256, 256, 2, 512, 2048, 0, 12, 1, 1, 0, 256, 1024, 0),  # yolo B8 fp16x3
    P(1, 80, 80, 128, 128, 2, 128, 768, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(32, 16, 16, 128, 256, 2, 128, 256, 0, 2, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16
    P(1, 40, 40, 256, 256, 2, 256, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(1, 160, 160, 128, 128, 2, 128, 256, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(2, 40, 40, 256, 256, 2, 256, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B2 fp16
    P(8, 40, 40, 256, 256, 2, 256, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B8 fp16
    P(1, 40, 40, 512, 512, 2, 512, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(8, 80, 80, 128, 128, 2, 128, 768, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B8 fp16
    P(1, 320, 320, 64, 128, 2, 128, 128, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(2, 40, 40, 512, 512, 2, 512, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B2 fp16
    P(8, 40, 40, 512, 512, 2, 512, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B8 fp16
    P(8, 80, 80, 256, 256, 2, 256, 512, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B8 fp16
    P(16, 192, 192, 128, 256, 2, 128, 256, 0, 2, 0, 1, 0, 0, 0, 0),  # florence 768 K16 fp16
    P(512, 16, 16, 128, 256, 2, 128, 256, 0, 2, 0, 1, 0, 0, 0, 0),  # florence 64 K512 fp16
    P(1, 160, 160, 32, 32, 1, 64, 32, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(1, 160, 160, 32, 32, 1, 32, 32, 64, 0, 1, 1, 1, 0, 0, 0),  # yolo B1 fp16
    P(1, 20, 20, 64, 64, 1, 320, 64, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(1, 20, 20, 128, 128, 1, 128, 128, 256, 0, 1, 1, 1, 0, 0, 0),  # yolo B1 fp16
    P(1, 40, 40, 64, 64, 1, 320, 64, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(1, 40, 40, 128, 128, 1, 128, 128, 256, 0, 1, 1, 1, 0, 0, 0),  # yolo B1 fp16
    P(8, 20, 20, 128, 128, 1, 256, 128, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B8 fp16
    P(8, 20, 20, 128, 128, 1, 128, 128, 256, 0, 1, 1, 1, 0, 0, 0),  # yolo B8 fp16
    P(1, 80, 80, 64, 64, 1, 128, 64, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(1, 80, 80, 64, 64, 1, 64, 64, 128, 0, 1, 1, 1, 0, 0, 0),  # yolo B1 fp16
    P(1, 160, 160, 64, 64, 1, 64, 256, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(8, 80, 80, 64, 64, 1, 64, 64, 128, 0, 1, 1, 1, 0, 0, 0),  # yolo B8 fp16
    P(8, 20, 20, 256, 256, 1, 256, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B8 fp16
    P(8, 20, 20, 256, 256, 1, 256, 256, 512, 0, 1, 1, 1, 0, 0, 0),  # yolo B8 fp16
    P(8, 40, 40, 128, 128, 1, 256, 128, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B8 fp16
    P(8, 40, 40, 128, 128, 1, 128, 128, 256, 0, 1, 1, 1, 0, 0, 0),  # yolo B8 fp16
    P(1, 80, 80, 256, 320, 1, 256, 320, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
    P(8, 40, 40, 256, 256, 1, 256, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B8 fp16
]

EDGES = [
    Case("gemm M<128, N % bn", 100, 1, 1, 192, 200, 0, 192, 200, 0, 0, 1, 1, 0, 0, 0, 0,
         expect=dict(mode=0, m_tiles=1, n_tiles=13, bn=16, vec_ok=1)),
    Case("gemm N % 16 = 8 scalar tail + residual", 300, 1, 1, 64, 72, 0, 64, 72, 72, 0, 0, 1, 1, 0, 0, 0,
         expect=dict(mode=0, bn=16, n_tiles=5, vec_ok=1)),
    Case("gemm N < 16, bk 32, fp32 out", 257, 1, 1, 96, 10, 0, 96, 10, 10, F_F32, 0, 1, 1, 0, 0, 0, expect=dict(bk=32, bn=16, m_tiles=3)),
    Case("gemm unaligned out (scalar epilogue)", 200, 1, 1, 128, 64, 0, 136, 67, 0, 0, 1, 1, 0, 0, 0, 0, out_off=1,
         expect=dict(vec_ok=0)),
    Case("gemm bf16 operands", 256, 1, 1, 128, 96, 0, 128, 96, 0, F_BF16, 2, 1, 0, 0, 0, 0, expect=dict(bk=64, vec_ok=1)),
    Case("gemm fp16x3 K 32, vector split out + residual lo plane", 200, 1, 1, 32, 64, 0, 64, 128, 128, F_X3 | F_SPLIT, 0, 1, 1, 0,
         64, 64, expect=dict(x3=1, bk=32, kb_merge=1, vec_ok=1, split=64, res_lo=64, ksplit=1)),
    Case("gemm fp16x3 K 64, vector split + residual lo planes, slices", 300, 1, 1, 64, 48, 0, 160, 160, 160, F_X3 | F_SPLIT, 1, 1, 1,
         80, 80, 80, a_off=8, out_off=16, res_off=16, expect=dict(x3=1, kb_merge=2, vec_ok=1, split=80, res_lo=80)),
    Case("split-K 5 (128 % 5 != 0)", 64, 1, 1, 2560, 200, 0, 2560, 200, 0, 0, 0, 1, 0, 0, 0, 0, expect=dict(ksplit=5, kb_per=8)),
    Case("split-K 8, last slice short", 64, 1, 1, 5888, 200, 0, 5888, 200, 200, F_F32, 0, 1, 1, 0, 0, 0,
         expect=dict(ksplit=8, kb_per=12, num_kb=92)),
    Case("split-K 7 fp16x3, fp32 out", 64, 1, 1, 1280, 128, 0, 2560, 128, 0, F_X3 | F_F32, 0, 1, 0, 0, 0, 0,
         expect=dict(ksplit=7, kb_merge=2)),
    Case("split-K 14, a slice with no reduction rows", 32, 1, 1, 3584, 48, 0, 3584, 48, 0, 0, 1, 1, 0, 0, 0, 0, expect=dict(ksplit=14)),
    Case("split-K fp16x3 split out, unaligned lo slice", 70, 1, 1, 2048, 48, 0, 4096, 104, 104, F_X3 | F_SPLIT, 0, 1, 1, 0, 56, 56,
         out_off=4, res_off=4, expect=dict(vec_ok=0, split=56, res_lo=56)),
    Case("halo conv, Ho/Wo not tile multiples", 2, 37, 45, 64, 80, 1, 64, 80, 80, 0, 1, 1, 1, 0, 0, 0, expect=dict(mode=3, bk=64)),
    Case("halo conv bk 32, channel slices", 1, 21, 30, 96, 40, 1, 160, 120, 0, 0, 1, 1, 0, 0, 0, 0, a_off=32, out_off=40,
         expect=dict(mode=3, bk=32, vec_ok=1)),
    Case("conv s1 fp16x3 planes, slices", 1, 23, 29, 32, 48, 1, 192, 160, 160, F_X3 | F_SPLIT, 1, 1, 1, 96, 80, 80,
         a_off=64, out_off=16, res_off=16, expect=dict(mode=1, vec_ok=1, split=80, res_lo=80)),
    Case("conv s1 fp16x3, nb > 1 over batch 13", 13, 4, 4, 32, 48, 1, 64, 96, 0, F_X3 | F_SPLIT, 0, 1, 0, 0, 0, 0,
         expect=dict(mode=1, nb=8, m_tiles=2)),
    Case("conv s2 nb > 1 over batch 11", 11, 8, 8, 64, 48, 2, 64, 48, 0, 0, 1, 1, 0, 0, 0, 0, expect=dict(mode=2, nb=8, m_tiles=2)),
    Case("conv s2 fp16x3, odd tiles, unaligned out", 2, 30, 42, 64, 24, 2, 128, 27, 0, F_X3 | F_F32, 0, 0, 0, 0, 0, 0, out_off=1,
         expect=dict(mode=2, vec_ok=0)),
    Case("conv s2 bf16", 2, 16, 20, 64, 32, 2, 64, 32, 0, F_BF16, 1, 1, 0, 0, 0, 0, expect=dict(mode=2, bk=64)),
]
CASES = PRODUCTION + EDGES


def _x3(c):
    return bool(c.flags & F_X3)


def _geom(c):
    """(rows of A, reduction size, pixels/rows of the output, Ktot, lo offset of A, columns of A a row carries)"""
    kred = c.K
    lo_a = (c.lo_a or kred) if _x3(c) else 0
    span = lo_a + kred if _x3(c) else kred
    rows_a = c.B * c.H * c.W
    rows_o = c.B if c.stride == 0 else c.B * (c.H // c.stride) * (c.W // c.stride)
    ktot = kred if c.stride == 0 else 9 * kred
    return rows_a, kred, rows_o, ktot, lo_a, span


def _out_cols(c):
    split = bool(c.flags & F_SPLIT) and not (c.flags & F_F32)
    lo = (c.lo_out or c.N) if split else 0
    return split, lo


def extents(c):
    """elements each buffer needs: A from its offset (what the tensor map covers), B, out / residual (what the epilogue
    writes / reads) -- plus one guard row of NaN after out and residual"""
    rows_a, kred, rows_o, ktot, lo_a, span = _geom(c)
    split, lo_out = _out_cols(c)
    ext_a = c.a_off + (rows_a - 1) * c.lda + span
    if c.stride == 2:
        ext_a = c.a_off + (rows_a - 1) * c.lda + c.lda + span     # the parity view's dim 0 spans two pixels
    ext_b = c.N * ktot * (2 if _x3(c) else 1)
    ext_o = c.out_off + (rows_o + 1) * c.ldc + (lo_out + c.N if split else c.N)
    res_cols = (c.lo_res + c.N) if c.lo_res else c.N
    ext_r = c.res_off + (rows_o + 1) * max(c.ldr, 1) + res_cols if c.res else 0
    return ext_a, ext_b, ext_o, ext_r


def case_args(c, base=None, ptrs=None):
    """b2p_gemm_plan arguments of a case: device pointers, or fake ones (base: 16-byte aligned) for the CPU planner"""
    esz = 4 if c.flags & F_F32 else 2
    if ptrs is None:
        ptrs = {"a": base, "b": base + (1 << 30), "out": base + (2 << 30), "bias": base + (3 << 30), "res": base + (4 << 30)}
    flags = c.flags
    return (ptrs["a"] + 2 * c.a_off, c.lda, c.B, c.H, c.W, c.K, c.stride, ptrs["b"], c.N,
            None if flags & FLAG_PARK else ptrs["out"] + esz * c.out_off, c.N if flags & FLAG_PARK else c.ldc,
            ptrs["bias"] if c.bias and not flags & FLAG_PARK else None,
            ptrs["res"] + esz * c.res_off if c.res and not flags & FLAG_PARK else None, 0 if flags & FLAG_PARK else c.ldr,
            c.act, flags, c.lo_a, c.lo_out, c.lo_res)


def cpu_class(c):
    args = case_args(c, base=1 << 24)
    return path_class(plan(args, *H100_SXM), args)


# ----------------------------------------------------------------------------------------------------- GPU side
U32 = 2.0 ** -23
_NOTED = [False]


def _fill_nan(n, dtype, torch):
    return torch.full((max(n, 1),), float("nan"), dtype=dtype, device="cuda")


def _rows_to_check(n, torch, gen):
    """every output row of small cases; else the first and last 1024 and 2048 drawn at random"""
    if n <= 8192:
        return torch.arange(n, device="cuda")
    r = torch.randint(0, n, (2048,), device="cuda", generator=gen)
    return torch.unique(torch.cat([torch.arange(1024, device="cuda"), torch.arange(n - 1024, n, device="cuda"), r]))


def _patches(c, a_eff, rows, torch):
    """fp64 operand rows of the selected output rows: A rows (GEMM) or their 3x3 pad-1 neighbourhoods ordered (ky, kx, c)"""
    if c.stride == 0:
        return a_eff[rows]
    Ho, Wo = c.H // c.stride, c.W // c.stride
    ap = torch.nn.functional.pad(a_eff.view(c.B, c.H, c.W, -1), (0, 0, 1, 1, 1, 1))
    b, rem = rows // (Ho * Wo), rows % (Ho * Wo)
    oy, ox = rem // Wo, rem % Wo
    k3 = torch.arange(3, device="cuda")
    p = ap[b[:, None, None], (oy * c.stride)[:, None, None] + k3[None, :, None], (ox * c.stride)[:, None, None] + k3[None, None, :]]
    return p.reshape(len(rows), -1)


def _act64(x, act, torch):
    if act == 1:
        return x * torch.sigmoid(x)
    if act == 2:
        return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))
    return x


def _launch(c, bufs, torch):
    from omniparser_b200 import _lib, ops
    esz = 4 if c.flags & F_F32 else 2
    A, Bw, out, bias, res = bufs["a"], bufs["b"], bufs["out"], bufs["bias"], bufs["res"]
    pa = A.data_ptr() + 2 * c.a_off
    po = out.data_ptr() + esz * c.out_off
    pb = bias.data_ptr() if bias is not None else None
    pr = res.data_ptr() + esz * c.res_off if res is not None else None
    st = ops._stream()
    if c.stride == 0:
        rc = _lib.lib().b2p_gemm_planes(pa, c.lda, Bw.data_ptr(), c.B, c.N, c.K, po, c.ldc, pb, pr, c.ldr, c.act, c.flags,
                                        c.lo_a, c.lo_out, c.lo_res, st)
    else:
        rc = _lib.lib().b2p_conv3x3_planes(pa, c.lda, c.B, c.H, c.W, c.K, c.stride, Bw.data_ptr(), c.N, po, c.ldc, pb, pr, c.ldr,
                                           c.act, c.flags, c.lo_a, c.lo_out, c.lo_res, st)
    _lib.check(rc)


def run_case(c, seed, slot_free=True):
    """-> (largest error / bound over the checked rows, plan); asserts everything the module docstring lists.
    slot_free=False: the launching stream can get no split-K workspace slot (all taken), so the launch must be the plan
    without split-K, with the same bound."""
    import torch
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x3, f32, bf16 = _x3(c), bool(c.flags & F_F32), bool(c.flags & F_BF16)
    split, lo_out = _out_cols(c)
    rows_a, kred, rows_o, ktot, lo_a, span = _geom(c)
    ext_a, ext_b, ext_o, ext_r = extents(c)
    opdt = torch.bfloat16 if bf16 else torch.float16
    odt = torch.float32 if f32 else torch.float16
    # operands: NaN everywhere the kernel must not read
    A = _fill_nan(ext_a, opdt, torch)
    a32 = torch.randn(rows_a, kred, device="cuda", generator=gen)
    a_hi = a32.to(opdt)
    av = A.as_strided((rows_a, span), (c.lda, 1), c.a_off)
    av[:, :kred] = a_hi
    a_eff = a_hi.double()
    a_lo_abs = None
    if x3:
        a_lo = (a32 - a_hi.float()).half()
        av[:, lo_a:lo_a + kred] = a_lo
        a_eff = a_eff + a_lo.double()
        a_lo_abs = a_lo.double().abs()
    taps = 1 if c.stride == 0 else 9
    w32 = torch.randn(c.N, taps, kred, device="cuda", generator=gen) / math.sqrt(ktot)
    w_hi = w32.to(opdt)
    w_eff = w_hi.double()
    if x3:
        w_lo = (w32 - w_hi.float()).half()
        Bw = torch.cat([w_hi, w_lo], dim=2).reshape(-1).contiguous()
        w_eff = w_eff + w_lo.double()
        w_lo_abs = w_lo.double().abs().reshape(c.N, -1)
    else:
        Bw = w_hi.reshape(-1).contiguous()
    assert Bw.numel() == ext_b
    w_eff = w_eff.reshape(c.N, -1)
    bias = (torch.randn(c.N, device="cuda", generator=gen) * 0.5) if c.bias else None
    res = None
    if c.res:
        res = _fill_nan(ext_r, odt, torch)
        rv = res.as_strided((rows_o, c.N), (c.ldr, 1), c.res_off)
        rv.copy_(torch.randn(rows_o, c.N, device="cuda", generator=gen).to(odt))
        r_eff = rv.double()
        if c.lo_res:
            rl = res.as_strided((rows_o, c.N), (c.ldr, 1), c.res_off + c.lo_res)
            # the kernel adds hi and lo in fp32, so the lo plane need not be a canonical remainder: O(2^-6) values make a
            # dropped lo plane visible at every K
            rl.copy_((torch.randn(rows_o, c.N, device="cuda", generator=gen) * 2.0 ** -6).to(odt))
            r_eff = r_eff + rl.double()
    out = _fill_nan(ext_o, odt, torch)
    bufs = {"a": A, "b": Bw, "out": out, "bias": bias, "res": res}
    # the plan at this device's limits: its path class is the one the CPU table assigns to the case, and its tensor maps
    # stay inside the buffers
    props = torch.cuda.get_device_properties(0)
    sms, smem = props.multi_processor_count, props.shared_memory_per_block_optin
    esz = 4 if f32 else 2
    ptrs = {"a": A.data_ptr(), "b": Bw.data_ptr(), "out": out.data_ptr(), "bias": bias.data_ptr() if bias is not None else 0,
            "res": res.data_ptr() if res is not None else 0}
    args = case_args(c, ptrs=ptrs)
    p = plan(args, sms, smem)
    print(f"[gemm case] {c.name}: B={c.B} H={c.H} W={c.W} K={c.K} N={c.N} s={c.stride} flags={c.flags} act={c.act} | "
          + " ".join(f"{k}={p[k]}" for k in ("mode", "bk", "bn", "ksplit", "kb_per", "kb_merge", "stages", "stagesA", "bres", "nb",
                                             "tw", "th", "m_tiles", "n_tiles", "mt_fast", "grid", "smem", "vec_ok")),
          flush=True)
    fake = case_args(c, base=1 << 24)
    assert path_class(p, args) == path_class(plan(fake, sms, smem), fake)     # the device pointers do not change the path
    if (sms, smem) == H100_SXM:
        assert path_class(p, args) == cpu_class(c), (path_class(p, args), cpu_class(c))
    elif not _NOTED[0]:
        _NOTED[0] = True
        print(f"[gemm case] device limits {sms} SMs / {smem} B differ from H100 SXM: the paths are checked against plans at the "
              f"device's limits, not against the CPU table's classes", flush=True)
    assert p["extent_a"] <= ext_a - c.a_off and p["extent_b"] <= ext_b, (p["extent_a"], ext_a, p["extent_b"], ext_b)
    _launch(c, bufs, torch)
    torch.cuda.synchronize()
    launched = last_plan()     # what was launched (split-K needs the stream's workspace slot): the plan checked above
    if slot_free:
        assert launched == p, {k: (p[k], launched[k]) for k in p if p[k] != launched[k]}
    else:
        assert launched["ksplit"] == 1, launched
    if launched["ksplit"] > 1:     # split-K: a second launch on the same stream repeats every bit (and found its counters reset)
        first = out.clone()
        out.fill_(float("nan"))
        _launch(c, bufs, torch)
        torch.cuda.synchronize()
        assert torch.equal(first.view(torch.int16 if odt == torch.float16 else torch.int32),
                           out.view(torch.int16 if odt == torch.float16 else torch.int32)), "split-K result not reproducible"
    # nothing outside the written slice was touched
    mask = torch.zeros(ext_o, dtype=torch.bool, device="cuda")
    mask.as_strided((rows_o, c.N), (c.ldc, 1), c.out_off).fill_(True)
    if split:
        mask.as_strided((rows_o, c.N), (c.ldc, 1), c.out_off + lo_out).fill_(True)
    assert out[~mask].isnan().all(), "the epilogue wrote outside its slice"
    # fp64 reference and per-element bound on the checked rows
    rows = _rows_to_check(rows_o, torch, gen)
    pa = _patches(c, a_eff, rows, torch)
    acc = pa @ w_eff.T
    s_abs = pa.abs() @ w_eff.abs().T
    k_eff = ktot * (3 if x3 else 1)
    err_pre = k_eff * U32 * s_abs
    if x3:
        err_pre = err_pre + _patches(c, a_lo_abs, rows, torch) @ w_lo_abs.T
    pre = acc + (bias.double() if bias is not None else 0)
    err_pre = err_pre + 2.0 ** -24 * (pre.abs() + err_pre)
    y = _act64(pre, c.act, torch)
    if c.act == 1:
        err = 1.1 * err_pre + 2.0 ** -20 * y.abs() + 2.0 ** -126
    elif c.act == 2:
        err = 1.13 * err_pre + pre.abs() * (0.5 * 1.5e-7 + 2.0 ** -21) + 2.0 ** -22 * y.abs()
    else:
        err = err_pre
    if c.res:
        y = y + r_eff[rows]
        err = err + (2.0 ** -23 if c.lo_res else 2.0 ** -24) * (y.abs() + err)   # one fp32 add per residual plane
    ov = out.as_strided((rows_o, c.N), (c.ldc, 1), c.out_off)[rows]
    if split:
        lo = out.as_strided((rows_o, c.N), (c.ldc, 1), c.out_off + lo_out)[rows]
        got = ov.double() + lo.double()
        bound = err + 2.0 ** -22 * (y.abs() + err) + 2.0 ** -25
        # canonical pair: |lo| <= half an ulp of hi (ulp of a normal fp16 m * 2^e, m in [0.5, 1): 2^(e - 11))
        ulp = torch.ldexp(torch.ones_like(got), torch.frexp(ov.double())[1] - 11).clamp_min(2.0 ** -24)
        assert (lo.double().abs() <= 0.5 * ulp).all(), "[hi | lo] pair not canonical"
    elif f32:
        got = ov.double()
        bound = err + 2.0 ** -24 * (y.abs() + err)
    else:
        got = ov.double()
        bound = err + 2.0 ** -11 * (y.abs() + err) + 2.0 ** -25
    e = (got - y).abs()
    bad = ~(e <= bound)
    assert not bad.any(), (f"{int(bad.sum())} of {bad.numel()} elements beyond the bound; first at "
                           f"{[int(v) for v in bad.nonzero()[0]]}, got {got[bad][:4].tolist()} want {y[bad][:4].tolist()}")
    return float((e / bound).max()), p


@pytest.mark.gpu
@pytest.mark.parametrize("i", [i for i, c in enumerate(CASES) if not c.flags & FLAG_PARK],
                         ids=[f"{i}-{c.name}" for i, c in enumerate(CASES) if not c.flags & FLAG_PARK])
def test_gemm_path(i):
    """(park-only plans run through b2p_gemm_ln: test_gemm_ln_path)"""
    c = CASES[i]
    ratio, p = run_case(c, 1000 + i)
    print(f"[gemm case] {i} class {cpu_class(c)}: max error / bound = {ratio:.3g}", flush=True)


@pytest.mark.gpu
@pytest.mark.parametrize("i", [i for i, c in enumerate(CASES) if c.flags & FLAG_PARK])
def test_gemm_ln_path(i):
    """park-only split-K GEMM + the slice-summing LayerNorm kernel (b2p_gemm_ln) against fp64 LayerNorm(A B^T + bias + res)"""
    import torch
    from omniparser_b200 import ops
    c = CASES[i]
    gen = torch.Generator(device="cuda").manual_seed(2000 + i)
    M, N, K, x3 = c.B, c.N, c.K, _x3(c)
    a32 = torch.randn(M, K, device="cuda", generator=gen)
    w32 = torch.randn(N, K, device="cuda", generator=gen) / math.sqrt(K)
    parts = []
    for t in (a32, w32):
        hi = t.half()
        lo = (t - hi.float()).half() if x3 else None
        parts.append((hi, lo))
    A = torch.cat([parts[0][0], parts[0][1]], 1) if x3 else parts[0][0]
    W = torch.cat([parts[1][0], parts[1][1]], 1) if x3 else parts[1][0]
    a_eff = parts[0][0].double() + (parts[0][1].double() if x3 else 0)
    w_eff = parts[1][0].double() + (parts[1][1].double() if x3 else 0)
    bias = torch.randn(N, device="cuda", generator=gen) * 0.5
    res = torch.randn(M, N, device="cuda", generator=gen)
    gam = 1 + 0.1 * torch.randn(N, device="cuda", generator=gen)
    bet = 0.1 * torch.randn(N, device="cuda", generator=gen)
    o16 = torch.full((M + 1, 2 * N), float("nan"), device="cuda", dtype=torch.float16)
    o32 = torch.full((M + 1, N), float("nan"), device="cuda")
    args = case_args(c, base=A.data_ptr() & ~15)
    props = torch.cuda.get_device_properties(0)
    p = plan((A.data_ptr(), A.stride(0)) + args[2:7] + (W.data_ptr(),) + args[8:], props.multi_processor_count,
             props.shared_memory_per_block_optin)
    print(f"[gemm case] {c.name} (park): M={M} N={N} K={K} | " + " ".join(f"{k}={p[k]}" for k in ("bk", "bn", "ksplit", "grid")), flush=True)
    assert p["park"] == 1 and p["extent_a"] <= A.numel() and p["extent_b"] <= W.numel()
    outs = []
    for _ in range(2):
        ops.gemm_ln(A, A.stride(0), W, M, N, K, bias, res, N, gam, bet, o16, 2 * N, o32, N, split=True, x3=x3)
        torch.cuda.synchronize()
        assert last_plan() == p
        outs.append(o32.clone())
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), "park-only split-K not reproducible"
    assert o32[M].isnan().all() and o16[M].isnan().all()
    y = a_eff @ w_eff.T + bias.double() + res.double()
    err_y = (K * (3 if x3 else 1) * U32 * (a_eff.abs() @ w_eff.abs().T) + 2.0 ** -23 * y.abs()).amax(1, keepdim=True)
    mu, sd = y.mean(1, keepdim=True), y.var(1, unbiased=False, keepdim=True).add(1e-5).sqrt()
    yh = (y - mu) / sd
    ref = yh * gam.double() + bet.double()
    bound = gam.double().abs() * (3 * err_y / sd + N * 2.0 ** -24 * (yh.abs() + 1)) + 2.0 ** -24 * ref.abs()
    e = (o32[:M].double() - ref).abs()
    assert (e <= bound).all(), float((e / bound).max())
    hi, lo = o16[:M, :N], o16[:M, N:]
    assert (hi.double() + lo.double() - o32[:M].double()).abs().le(2.0 ** -22 * o32[:M].double().abs() + 2.0 ** -25).all()
    print(f"[gemm case] {i} class {cpu_class(c)}: max error / bound = {float((e / bound).max()):.3g}", flush=True)
