"""CPU: the epilogue of every production GEMM/conv plan (``b2p_gemm_epilogue_plan``) at H100 SXM and PCIe limits.  The TMA
epilogue (staging buffers stored by TMA, residual loaded by TMA) must fit in shared memory, leave the ring at least two
stages deep and never take an fp16x3 stage, use boxes TMA can encode, and leave the path class of the plan unchanged.
Which launches take it is pinned here as data: every direct (not split-K, not park-only) mode-0 launch with 16-byte aligned rows,
an N tile that is a multiple of the chunk width and N a multiple of 8 (fp16) / 4 (fp32)."""
from __future__ import annotations

import collections
import ctypes as C

from gemm_plan_util import H100_PCIE, H100_SXM, path_class, plan, planner_args
from omniparser_b200 import _lib
from test_gemm_plan_cpu import production_calls

EPI_FIELDS = ("tma", "cols", "chunks", "stage_bufs", "out_planes", "res_bufs", "res_planes", "epi_bytes", "stages", "stagesA",
              "smem", "c_rank", "c_box0", "c_box1", "c_box2", "c_stride1", "c_stride2",
              "r_rank", "r_box0", "r_box1", "r_box2", "r_stride1", "r_stride2", "swizzle")

# launches with the TMA epilogue per production plan at 132 SMs (of all GEMM/conv launches of the plan)
EXPECTED_TMA = {
    "yolo B8 fp16": 91, "yolo B2 fp16": 85, "yolo B1 fp16": 87, "yolo B8 fp16x3": 89, "yolo B2 fp16x3": 87, "yolo B1 fp16x3": 85,
    "florence 64 K32 fp16x3": 138, "florence 64 K512 fp16x3": 173, "florence 768 K16 fp16x3": 188, "florence beam3 K32 fp16x3": 138,
    "florence 64 K32 fp16": 166, "florence 64 K512 fp16": 190, "florence 768 K16 fp16": 176, "florence beam3 K32 fp16": 166,
    "florence 64 K32 fp16x3 B2P_GEMM_LN=1": 114,
}


def epi_plan(args, num_sms, max_smem):
    out = (C.c_int * len(EPI_FIELDS))()
    _lib.check(_lib.lib().b2p_gemm_epilogue_plan(*args, num_sms, max_smem, out))
    return dict(zip(EPI_FIELDS, out))


def test_production_epilogues():
    counts = collections.Counter()
    totals = collections.Counter()
    for name, cl in production_calls().items():
        for n, a in cl:
            args = planner_args(n, a)
            flags = args[15]
            f32 = bool(flags & 2)
            for sms, smem in (H100_SXM, H100_PCIE):
                p = plan(args, sms, smem)
                e = epi_plan(args, sms, smem)
                assert (e["stages"], e["stagesA"], e["smem"]) == (p["stages"], p["stagesA"], p["smem"])
                assert p["smem"] <= smem
                direct = p["mode"] == 0 and p["ksplit"] == 1 and not p["park"]
                esz = 4 if f32 else 2
                N = args[8]
                eligible = direct and p["vec_ok"] and N % (16 // esz) == 0 and p["bn"] % (64 // esz) == 0
                if not e["tma"]:
                    # only an fp16x3 ring (never shortened) or a ring already at 2 stages can leave an eligible launch out
                    assert not eligible or p["x3"] or (p["stagesA"] if p["bres"] else p["stages"]) <= 2, (name, n, p, e)
                    assert e["epi_bytes"] == 8 * 16 * 36 * 4
                    continue
                assert eligible, (name, n, p, e)
                assert p["bres"] or p["stages"] >= 2
                assert not p["sep"] or p["stagesA"] >= 2
                # boxes: <= 256 per dimension, inner box = one 64-byte swizzle span, 16-byte aligned global strides
                assert e["cols"] * esz == 64 == e["swizzle"] and e["c_box0"] == e["cols"] and e["c_box1"] == 128
                assert e["chunks"] * e["cols"] == p["bn"]
                assert e["c_rank"] == (3 if e["out_planes"] == 2 else 2) and e["out_planes"] == (2 if p["split"] else 1)
                assert e["c_stride1"] % 16 == 0 and e["c_stride2"] % 16 == 0
                if e["res_planes"]:
                    assert e["r_rank"] == (3 if e["res_planes"] == 2 else 2) and e["r_box0"] == e["cols"] and e["r_box1"] == 128
                    assert e["r_stride1"] % 16 == 0 and e["r_stride2"] % 16 == 0 and e["res_bufs"] == 2
                else:
                    assert e["r_rank"] == 0 and e["res_bufs"] == 0
                for b in ("c_box0", "c_box1", "c_box2", "r_box0", "r_box1", "r_box2"):
                    assert e[b] <= 256
                assert e["epi_bytes"] == 2 * 128 * 64 * (e["out_planes"] + e["res_planes"])
                if sms == H100_SXM[0]:
                    counts[name] += 1
            totals[name] += 1
    print("\nplan: GEMM/conv launches, of which TMA epilogue  [132 SMs]")
    for name in totals:
        print(f"  {name:40s} {totals[name]:4d} {counts[name]:4d}")
    assert dict(counts) == EXPECTED_TMA, dict(counts)
