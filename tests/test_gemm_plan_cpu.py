"""CPU: the launch plan of every wgmma GEMM/conv call the production plans make, computed by the host-only planner
(``b2p_gemm_plan``, the same code the launcher runs) at H100 SXM (132 SMs) and H100 PCIe (114 SMs) limits, against the
invariants whose violation would fault or corrupt memory on the GPU: shared-memory budget, resident-weight slots, split-K
residency / workspace / counters / slices, TMA boxes, the halo tile's shifted reads, conv tile sizes.  Each plan reduces
to a path class; the classes production reaches are recorded here as data, and the GPU case list of
test_gemm_paths_gpu.py must cover each of them, every N-tile instantiation and both k-block widths."""
from __future__ import annotations

import collections
import contextlib
import ctypes as C
from unittest import mock

import pytest
import torch

from gemm_plan_util import BN_INSTANTIATIONS, GEMM_CALLS, H100_PCIE, H100_SXM, PLAN_FIELDS, path_class, plan, planner_args
from omniparser_b200 import _lib, ops
from standin import florence as FS
from test_plan_dryrun_cpu import _Recorder, _Stream

K_MAX_STAGES = 8
K_WS_BYTES = 64 << 20              # split-K workspace per stream (gemm_wgmma.cu kWsBytes)
K_MAX_COUNTER_TILES = 1 << 12      # split-K counters per stream (kMaxCounterTiles)


@contextlib.contextmanager
def _recording():
    """the C library replaced by the argument-checking recorder of test_plan_dryrun_cpu, CUDA streams by stubs"""
    r = _Recorder()
    with contextlib.ExitStack() as st:
        st.enter_context(mock.patch.object(_lib, "_lib", r))
        st.enter_context(mock.patch.object(ops, "_stream", lambda: C.c_void_p(0)))
        st.enter_context(mock.patch.object(torch.cuda, "device", lambda *a, **k: contextlib.nullcontext()))
        st.enter_context(mock.patch.object(torch.cuda, "Stream", _Stream))
        st.enter_context(mock.patch.object(torch.cuda, "current_stream", lambda *a, **k: _Stream()))
        st.enter_context(mock.patch.object(torch.cuda, "synchronize", lambda *a, **k: None))
        yield r


def _florence_calls(r, w, K, size, **kw):
    from omniparser_b200.florence_engine import FlorencePlan
    p = FlorencePlan(w, K, 8, FS.PROMPT_IDS, use_graph=False, size=size, **kw)
    p.encode()
    p.reset_decode(K)
    p.decode_step()                   # with the LM head
    p.decode_step(forced=True)        # forced token: no LM head
    return p


_PRODUCTION = None


def production_calls():
    """{plan name: [(call name, recorded args)]} of every GEMM/conv call of the production plans: the detector at batch 8
    (the benchmark's), 2 and 1 in both precisions; the captioner's 64 mode (32 and 512 crops) and 768 mode (16 crops, its
    only bucket) in both precisions, greedy and 3-beam decode steps with and without the LM head; B2P_GEMM_LN=1."""
    global _PRODUCTION
    if _PRODUCTION is not None:
        return _PRODUCTION
    from omniparser_b200.florence_engine import FlorenceWeights
    from omniparser_b200.yolo_engine import YoloPlan, YoloWeights
    from standin.yolo_weights import yolo_standin
    out = {}
    ysd = yolo_standin(0).state_dict()
    fsd = FS.florence_standin(0).state_dict()
    for prec in ("fp16", "fp16x3"):
        yw = YoloWeights(ysd, torch.device("cpu"), precision=prec)
        for B in (8, 2, 1):
            with _recording() as r:
                YoloPlan(yw, B, 640, 640, use_graph=False).run()
            out[f"yolo B{B} {prec}"] = r.calls
    for prec in ("fp16x3", "fp16"):
        fw = FlorenceWeights(fsd, torch.device("cpu"), FS.GEN, prec)
        for size, K in ((64, 32), (64, 512), (768, 16)):
            with _recording() as r:
                _florence_calls(r, fw, K, size)
            out[f"florence {size} K{K} {prec}"] = r.calls
        with _recording() as r:
            _florence_calls(r, fw, 32, 64, num_beams=3)
        out[f"florence beam3 K32 {prec}"] = r.calls
    fw = FlorenceWeights(fsd, torch.device("cpu"), FS.GEN, "fp16x3")
    with mock.patch.dict("os.environ", {"B2P_GEMM_LN": "1"}), _recording() as r:
        _florence_calls(r, fw, 32, 64)
    out["florence 64 K32 fp16x3 B2P_GEMM_LN=1"] = r.calls
    _PRODUCTION = {k: [(n, a) for n, a in v if n in GEMM_CALLS] for k, v in out.items()}
    return _PRODUCTION


def check_invariants(p, args):
    """the plan facts whose violation would fault, hang or corrupt memory"""
    stride, x3 = args[6], bool(args[15] & 8)
    # shared memory (smem <= the device limit: checked by the caller, which knows the limit)
    # (resident weights: "stages" is the number of weight slots, one per k-block, see below)
    assert p["bres"] or 2 <= p["stages"] <= K_MAX_STAGES
    assert (not p["sep"] or p["stagesA"] >= 2) and (p["sep"] or p["stagesA"] == 0)
    assert p["bn"] in BN_INSTANTIATIONS and p["bk"] in (32, 64) and p["x3"] == int(x3)
    assert p["taps"] == (9 if p["mode"] == 3 else 1)
    assert p["num_kb"] % p["kb_merge"] == 0 and p["kb_per"] % p["kb_merge"] == 0
    # resident weights: one slot per (k-block, tap) the producer loads on a CTA's first item, whole K in one slice
    if p["bres"]:
        assert p["sep"] and p["ksplit"] == 1 and p["n_tiles"] == 1 and not p["park"] and not x3
        assert p["stages"] == p["kb_per"] * p["taps"] == p["num_kb"] * p["taps"]
        assert p["b_slot"] * p["stages"] + p["a_slot"] * p["stagesA"] <= p["smem"]
    tiles = p["m_tiles"] * p["n_tiles"]
    # split-K: one item per CTA (the distributed reduction waits only among CTAs of one launch), counters, workspace, slices
    if p["ksplit"] > 1:
        assert tiles * p["ksplit"] <= p["grid"], p
        assert tiles <= K_MAX_COUNTER_TILES
        assert p["kb_per"] * (p["ksplit"] - 1) < p["num_kb"], "an empty k slice"
    if p["ksplit"] > 1 or p["park"]:
        assert tiles * p["ksplit"] * 128 * p["bn"] * 4 <= K_WS_BYTES
    assert p["kb_per"] * p["ksplit"] >= p["num_kb"], "k-blocks no slice covers"
    assert 1 <= p["grid"] <= tiles * p["ksplit"]
    # TMA: boxes, swizzle span, bytes per stage
    box_a = [p[f"box_a{i}"] for i in range(p["rank_a"])]
    assert all(1 <= b <= 256 for b in box_a) and 1 <= p["box_b1"] <= 256
    assert p["box_a0"] == p["box_b0"] == p["bk"] and p["box_b1"] == p["bn"]
    # one inner box row is exactly the swizzle span the tensor maps are encoded with, and the wgmma descriptors read the
    # same swizzle
    assert 2 * p["box_a0"] == p["swizzle_a"] and 2 * p["box_b0"] == p["swizzle_b"]
    assert p["swizzle_a"] == p["swizzle_b"] == p["swizzle_desc"] and p["swizzle_desc"] in (64, 128)
    vol = 1
    for b in box_a:
        vol *= b
    assert p["a_bytes"] == 2 * vol and p["b_bytes"] == 2 * p["bk"] * p["bn"]
    assert p["a_bytes"] <= p["a_slot"] and p["b_bytes"] <= p["b_slot"] and p["a_slot"] % 1024 == 0 and p["b_slot"] % 1024 == 0
    # halo conv: MMA row r of tap (ky, kx) reads halo-tile position r + ky*tw + kx (tw = the row pitch the consumers use).
    # The TMA box must have that pitch; every read of a valid output row (ty < th, tx < tw_valid) must land in the loaded
    # box; and the furthest read of any of the 128 rows (ky = kx = 2) must stay inside the A slot
    if p["mode"] == 3:
        assert p["box_a1"] == p["tw"] == p["tw_valid"] + 2 and p["box_a2"] == p["th"] + 2 and p["box_a3"] == 1
        assert (p["th"] - 1) * p["tw"] + (p["tw_valid"] - 1) < 128
        assert (p["th"] - 1) * p["tw"] + (p["tw_valid"] - 1) + 2 * p["tw"] + 2 < p["box_a1"] * p["box_a2"]
        assert (127 + 2 * p["tw"] + 2 + 1) * 2 * p["bk"] <= p["a_slot"]
    # conv tiles
    if stride:
        assert p["th"] * p["tw"] <= 128 and p["nb"] * p["tw"] * p["th"] <= 128
        assert p["mt_fast"] == 0
    assert p["split"] == 0 or p["split"] % 8 == 0


def test_plan_field_count_matches_the_header():
    """b2p_gemm_plan writes as many ints as the header documents; PLAN_FIELDS sizes the caller's array"""
    import re
    from pathlib import Path
    text = (Path(__file__).resolve().parents[1] / "include" / "b200parse.h").read_text()
    assert int(re.search(r"plan_host receives (\d+) ints", text).group(1)) == len(PLAN_FIELDS)


def test_planner_rejects_what_the_launcher_rejects():
    A, B = 1 << 20, 1 << 21
    base = (A, 64, 256, 1, 1, 64, 0, B, 64, 1 << 22, 64, None, None, 0, 0, 0, 0, 0, 0)

    def bad(**kw):
        a = list(base)
        for i, v in kw.items():
            a[int(i[1:])] = v
        with pytest.raises(_lib.B2PError):
            plan(tuple(a))
    plan(base)
    bad(a5=60)                       # K % 8
    bad(a1=60)                       # lda % 8
    bad(a0=A + 8)                    # A not 16-byte aligned
    bad(a6=1, a5=48)                 # conv: Cin % 32
    bad(a6=2, a3=7, a4=8, a5=64)     # s2: odd H
    bad(a6=3)                        # stride
    bad(a15=8 | 1)                   # fp16x3 + bf16
    bad(a15=8, a5=48, a1=96)         # fp16x3: K % 32
    bad(a15=8, a1=64)                # fp16x3: lda < lo + K
    bad(a15=4, a8=60, a10=120)       # split output: N % 8
    bad(a15=4, a10=100)              # split output: ldc < lo + N
    bad(a15=0, a12=1 << 23, a18=4)   # residual lo plane % 8
    bad(a6=1, a15=32)                # park-only: GEMMs only
    with pytest.raises(_lib.B2PError):
        plan(base, 0, 232448)


def test_every_production_plan_keeps_the_invariants():
    calls = production_calls()
    counts = collections.Counter()
    split_per_plan = {}
    for name, cl in calls.items():
        n_split, max_ks = 0, 1
        for n, a in cl:
            args = planner_args(n, a)
            for sms, smem in (H100_SXM, H100_PCIE):
                p = plan(args, sms, smem)
                assert p["smem"] <= smem, (name, n, p)
                check_invariants(p, args)
                if sms == H100_SXM[0]:
                    counts[path_class(p, args)] += 1
                    if p["ksplit"] > 1:
                        n_split += 1
                        max_ks = max(max_ks, p["ksplit"])
        split_per_plan[name] = (len(cl), n_split, max_ks)
    # the distributed split-K wait needs every CTA of a tile resident at once: how many launches of each stream's plan rely on it
    print("\nplan: GEMM/conv launches, of which split-K (distributed reduction), largest ksplit  [132 SMs]")
    for name, (n, ns, mk) in split_per_plan.items():
        print(f"  {name:40s} {n:4d} {ns:4d} {mk:3d}")
    assert dict(counts) == PRODUCTION_CLASSES, _diff(counts)


def _diff(counts):
    new = {k: v for k, v in counts.items() if k not in PRODUCTION_CLASSES}
    gone = {k: v for k, v in PRODUCTION_CLASSES.items() if k not in counts}
    changed = {k: (PRODUCTION_CLASSES[k], v) for k, v in counts.items() if k in PRODUCTION_CLASSES and PRODUCTION_CLASSES[k] != v}
    return f"new classes (each needs a GPU case): {new}\nclasses gone: {gone}\ncounts changed: {changed}"


def test_gpu_cases_cover_every_production_class_every_bn_and_both_bk():
    from test_gemm_paths_gpu import CASES, case_args
    classes, bns, bks = set(), set(), set()
    for c in CASES:
        args = case_args(c, base=1 << 24)
        p = plan(args)
        check_invariants(p, args)
        classes.add(path_class(p, args))
        bns.add(p["bn"])
        bks.add(p["bk"])
        if c.expect:   # an edge case stays on the path its name claims
            assert {k: p[k] for k in c.expect} == c.expect, (c.name, {k: p[k] for k in c.expect})
    missing = set(PRODUCTION_CLASSES) - classes
    assert not missing, f"production path classes without a GPU case: {sorted(missing)}"
    assert bns == set(BN_INSTANTIATIONS), bns
    assert bks == {32, 64}


# (mode, bk, bn, split-K, park, bres, nb>1, mt_fast, x3, kb_merge, vec_ok, split out, res_lo, out_f32, residual, act) -> launches,
# over the plans of production_calls() at 132 SMs and 232448 bytes of shared memory
PRODUCTION_CLASSES = {
    (0, 32, 16, 0, 0, 0, 0, 0, 1, 2, 0, 0, 0, 1, 0, 0): 9,
    (0, 32, 16, 0, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 0, 0): 49,
    (0, 32, 16, 0, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 1, 0): 72,
    (0, 32, 16, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 1,
    (0, 32, 16, 0, 0, 0, 0, 1, 1, 2, 1, 0, 0, 1, 0, 0): 3,
    (0, 32, 16, 0, 1, 0, 0, 0, 1, 2, 1, 0, 0, 1, 0, 0): 24,
    (0, 32, 32, 0, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 0, 0): 58,
    (0, 32, 32, 0, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 1, 0): 54,
    (0, 32, 32, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 28,
    (0, 32, 32, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 2): 48,
    (0, 32, 32, 0, 0, 0, 0, 1, 1, 2, 1, 0, 0, 1, 0, 0): 12,
    (0, 32, 32, 0, 0, 0, 0, 1, 1, 2, 1, 0, 0, 1, 1, 0): 42,
    (0, 32, 32, 0, 0, 0, 0, 1, 1, 2, 1, 1, 0, 0, 0, 1): 9,
    (0, 32, 48, 0, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 1, 0): 6,
    (0, 32, 48, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 2): 6,
    (0, 32, 48, 0, 0, 0, 0, 1, 1, 2, 1, 1, 0, 0, 0, 1): 3,
    (0, 32, 48, 1, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 1, 0): 42,
    (0, 32, 48, 1, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 1,
    (0, 32, 48, 1, 1, 0, 0, 0, 1, 2, 1, 0, 0, 1, 0, 0): 12,
    (0, 32, 64, 0, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 0, 0): 4,
    (0, 32, 64, 0, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 1, 0): 6,
    (0, 32, 64, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 0): 3,
    (0, 32, 64, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 91,
    (0, 32, 64, 0, 0, 0, 0, 1, 1, 2, 1, 0, 0, 1, 0, 0): 72,
    (0, 32, 64, 0, 0, 0, 0, 1, 1, 2, 1, 1, 0, 0, 0, 0): 1,
    (0, 32, 64, 0, 0, 0, 0, 1, 1, 2, 1, 1, 0, 0, 0, 1): 3,
    (0, 32, 64, 1, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 0, 0): 6,
    (0, 32, 64, 1, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 1, 0): 6,
    (0, 32, 96, 0, 0, 0, 0, 1, 1, 2, 1, 0, 0, 1, 0, 0): 30,
    (0, 32, 96, 0, 0, 0, 0, 1, 1, 2, 1, 1, 0, 0, 0, 2): 54,
    (0, 32, 96, 1, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 1, 0): 54,
    (0, 32, 96, 1, 0, 0, 0, 1, 1, 2, 1, 1, 0, 0, 0, 1): 1,
    (0, 32, 128, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 0, 0): 2,
    (0, 32, 128, 0, 0, 0, 0, 0, 1, 1, 1, 0, 0, 1, 0, 0): 5,
    (0, 32, 128, 0, 0, 0, 0, 0, 1, 1, 1, 1, 0, 0, 0, 1): 3,
    (0, 32, 128, 0, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 0, 0): 7,
    (0, 32, 128, 0, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 1, 0): 20,
    (0, 32, 128, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 0): 1,
    (0, 32, 128, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 57,
    (0, 32, 128, 0, 0, 0, 0, 1, 1, 2, 1, 1, 0, 0, 0, 0): 1,
    (0, 32, 128, 0, 0, 0, 0, 1, 1, 2, 1, 1, 0, 0, 0, 2): 30,
    (0, 32, 128, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 3,
    (0, 32, 128, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 1, 0, 0): 2,
    (0, 32, 128, 1, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 1,
    (0, 32, 128, 1, 0, 0, 0, 1, 1, 2, 1, 0, 0, 1, 1, 0): 30,
    (0, 32, 192, 0, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 0, 0): 16,
    (0, 32, 192, 0, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 1, 0): 14,
    (0, 32, 192, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 0): 5,
    (0, 32, 192, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 2): 6,
    (0, 32, 192, 0, 0, 0, 0, 1, 1, 2, 1, 0, 0, 1, 0, 0): 2,
    (0, 32, 256, 0, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 0, 0): 66,
    (0, 32, 256, 0, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 1, 0): 96,
    (0, 32, 256, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 0): 4,
    (0, 32, 256, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 51,
    (0, 32, 256, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 2): 64,
    (0, 32, 256, 0, 0, 0, 0, 1, 1, 2, 1, 0, 0, 1, 0, 0): 1,
    (0, 32, 256, 0, 0, 0, 0, 1, 1, 2, 1, 1, 0, 0, 0, 2): 2,
    (0, 32, 256, 1, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 0, 0): 1,
    (0, 32, 256, 1, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 1, 0): 2,
    (0, 64, 16, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0): 8,
    (0, 64, 16, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 1,
    (0, 64, 16, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 0, 0): 37,
    (0, 64, 16, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 1, 0): 76,
    (0, 64, 16, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0): 1,
    (0, 64, 32, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 24,
    (0, 64, 32, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 0, 0): 42,
    (0, 64, 32, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 1, 0): 72,
    (0, 64, 32, 0, 0, 0, 0, 1, 0, 1, 1, 0, 0, 0, 0, 1): 10,
    (0, 64, 32, 0, 0, 0, 0, 1, 0, 1, 1, 0, 0, 1, 0, 0): 2,
    (0, 64, 48, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 6,
    (0, 64, 48, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 2): 40,
    (0, 64, 48, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 1, 0): 4,
    (0, 64, 48, 0, 0, 0, 0, 1, 0, 1, 1, 0, 0, 0, 0, 1): 3,
    (0, 64, 48, 0, 0, 0, 0, 1, 0, 1, 1, 0, 0, 1, 0, 0): 12,
    (0, 64, 48, 0, 0, 0, 0, 1, 0, 1, 1, 0, 0, 1, 1, 0): 36,
    (0, 64, 48, 1, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 1, 0): 40,
    (0, 64, 64, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 67,
    (0, 64, 64, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 0, 0): 5,
    (0, 64, 64, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 1, 0): 4,
    (0, 64, 64, 0, 0, 0, 0, 1, 0, 1, 1, 0, 0, 0, 0, 0): 1,
    (0, 64, 64, 0, 0, 0, 0, 1, 0, 1, 1, 0, 0, 0, 0, 1): 3,
    (0, 64, 64, 0, 0, 0, 0, 1, 0, 1, 1, 0, 0, 1, 0, 0): 48,
    (0, 64, 64, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 0, 0, 0): 3,
    (0, 64, 64, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 24,
    (0, 64, 64, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 1, 0, 0): 1,
    (0, 64, 64, 1, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 0, 0): 4,
    (0, 64, 96, 0, 0, 0, 0, 1, 0, 1, 1, 0, 0, 0, 0, 2): 36,
    (0, 64, 96, 0, 0, 0, 0, 1, 0, 1, 1, 0, 0, 1, 0, 0): 24,
    (0, 64, 96, 1, 0, 0, 0, 1, 0, 1, 1, 0, 0, 1, 1, 0): 24,
    (0, 64, 128, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 0): 1,
    (0, 64, 128, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 37,
    (0, 64, 128, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 0, 0): 5,
    (0, 64, 128, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 1, 0): 8,
    (0, 64, 128, 0, 0, 0, 0, 1, 0, 1, 1, 0, 0, 0, 0, 0): 1,
    (0, 64, 128, 0, 0, 0, 0, 1, 0, 1, 1, 0, 0, 0, 0, 2): 24,
    (0, 64, 128, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 20,
    (0, 64, 128, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 1, 1, 0): 8,
    (0, 64, 192, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 0): 2,
    (0, 64, 192, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 2): 4,
    (0, 64, 192, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 0, 0): 15,
    (0, 64, 192, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 1, 0): 16,
    (0, 64, 192, 0, 0, 0, 0, 1, 0, 1, 1, 0, 0, 1, 0, 0): 2,
    (0, 64, 192, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 0, 0, 0): 3,
    (0, 64, 256, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 0): 4,
    (0, 64, 256, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 43,
    (0, 64, 256, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 2): 62,
    (0, 64, 256, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 0, 0): 65,
    (0, 64, 256, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 1, 0): 92,
    (0, 64, 256, 0, 0, 0, 0, 1, 0, 1, 1, 0, 0, 0, 0, 2): 2,
    (0, 64, 256, 0, 0, 0, 0, 1, 0, 1, 1, 0, 0, 1, 0, 0): 1,
    (0, 64, 256, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 8,
    (0, 64, 256, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 1, 1, 0): 4,
    (1, 32, 16, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 3,
    (1, 32, 32, 0, 0, 0, 0, 0, 1, 1, 1, 1, 0, 0, 0, 1): 24,
    (1, 32, 32, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 0, 1, 1): 24,
    (1, 32, 32, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 31,
    (1, 32, 32, 0, 0, 0, 0, 0, 1, 2, 1, 1, 1, 0, 1, 1): 28,
    (1, 32, 32, 1, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 16,
    (1, 32, 32, 1, 0, 0, 0, 0, 1, 2, 1, 1, 1, 0, 1, 1): 16,
    (1, 32, 48, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 8,
    (1, 32, 48, 0, 0, 0, 0, 0, 1, 2, 1, 1, 1, 0, 1, 1): 8,
    (1, 32, 48, 1, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 16,
    (1, 32, 48, 1, 0, 0, 0, 0, 1, 2, 1, 1, 1, 0, 1, 1): 16,
    (1, 32, 64, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 45,
    (1, 32, 64, 0, 0, 0, 0, 0, 1, 2, 1, 1, 1, 0, 1, 1): 24,
    (1, 32, 64, 1, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 19,
    (1, 32, 64, 1, 0, 0, 0, 0, 1, 2, 1, 1, 1, 0, 1, 1): 8,
    (1, 32, 96, 1, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 2,
    (1, 32, 128, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 30,
    (1, 32, 128, 0, 0, 0, 0, 0, 1, 2, 1, 1, 1, 0, 1, 1): 16,
    (1, 32, 128, 1, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 20,
    (1, 32, 192, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 4,
    (1, 32, 192, 1, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 3,
    (1, 32, 256, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 11,
    (1, 32, 256, 1, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 11,
    (1, 32, 256, 1, 0, 0, 0, 0, 1, 2, 1, 1, 1, 0, 1, 1): 4,
    (2, 32, 32, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 1,
    (2, 32, 48, 0, 0, 0, 1, 0, 1, 2, 1, 0, 0, 1, 0, 0): 3,
    (2, 32, 48, 1, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 1,
    (2, 32, 64, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 2,
    (2, 32, 64, 1, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 2,
    (2, 32, 96, 1, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 2,
    (2, 32, 128, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 11,
    (2, 32, 128, 1, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 4,
    (2, 32, 192, 1, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 2,
    (2, 32, 256, 0, 0, 0, 0, 0, 1, 2, 1, 0, 0, 1, 0, 0): 3,
    (2, 32, 256, 0, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 2,
    (2, 32, 256, 0, 0, 0, 1, 0, 1, 2, 1, 0, 0, 1, 0, 0): 1,
    (2, 32, 256, 1, 0, 0, 0, 0, 1, 2, 1, 1, 0, 0, 0, 1): 3,
    (2, 64, 32, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 4,
    (2, 64, 48, 0, 0, 0, 1, 0, 0, 1, 1, 0, 0, 1, 0, 0): 2,
    (2, 64, 48, 1, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 1,
    (2, 64, 64, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 4,
    (2, 64, 64, 1, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 1,
    (2, 64, 96, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 1,
    (2, 64, 96, 1, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 2,
    (2, 64, 128, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 5,
    (2, 64, 128, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 6,
    (2, 64, 128, 1, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 2,
    (2, 64, 192, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 2,
    (2, 64, 256, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 2,
    (2, 64, 256, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 1, 0, 0): 3,
    (2, 64, 256, 0, 0, 0, 1, 0, 0, 1, 1, 0, 0, 1, 0, 0): 1,
    (3, 32, 32, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 24,
    (3, 32, 32, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 0, 1, 1): 24,
    (3, 64, 16, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 28,
    (3, 64, 16, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 1, 1): 20,
    (3, 64, 32, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 56,
    (3, 64, 32, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 1, 1): 36,
    (3, 64, 48, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 11,
    (3, 64, 48, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 1, 1): 8,
    (3, 64, 64, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 42,
    (3, 64, 64, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 1, 1): 24,
    (3, 64, 64, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 25,
    (3, 64, 64, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 0, 1, 1): 12,
    (3, 64, 96, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 10,
    (3, 64, 96, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 1, 1): 4,
    (3, 64, 128, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 33,
    (3, 64, 128, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 1, 1): 16,
    (3, 64, 192, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 4,
    (3, 64, 256, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0, 0, 0, 1): 10,
}
