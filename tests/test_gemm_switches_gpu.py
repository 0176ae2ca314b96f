"""GPU: the wgmma GEMM/conv kernel under its A/B switches, against fp64 and against the default process.

The planner reads its switches once per process (gemm_knobs), so every switch runs in its own subprocess, one at a time,
through test_gemm_paths_gpu.run_case (plan checked at the device's limits, NaN poison and guard rows, fp64 bound):

- B2P_SPLITK_LAST: every case whose plan splits K -- the production classes, the split-K edges (5, 7, 8 and 14 slices, the
  short last slice, a slice with no reduction rows, the unaligned fp16x3 split output) and conv tiles spanning nb > 1 whole
  images.  The last-arriver reduction and the default distributed one both start from 0 and add the parked slices in
  slice order, so the outputs must be byte-identical to the default process's.
- B2P_DENSE_GRIDS, B2P_NO_HALO, B2P_NO_SPLITK: one case per path class the switch adds to production (the smallest
  production call of the class, as test_gemm_paths_gpu.PRODUCTION was picked), plus every case of CASES whose plan the
  switch changes; each held to the fp64 bound.  Park-only plans are skipped under B2P_NO_SPLITK: the planner rejects them.
- B2P_NO_BRES, B2P_NO_HALO32: every case whose plan changes.  Where the k-blocks are still summed in the same order (always
  for B2P_NO_BRES; for the halo -> per-tap switch only with one channel block, since the halo tile runs the taps inside a
  channel block and the per-tap path the channel blocks inside a tap) the output must be byte-identical to the default's.
- End to end: the fp16 detector at B=1, 640x640 (head tensors) and the fp16x3 captioner at 32 crops (encoder states and
  the logits of two decode steps) under B2P_SPLITK_LAST and under B2P_PDL_SIMT must equal the default process bit for bit.

test_gemm_switches_cpu.py checks the same case lists on the CPU: every class each switch reaches in production is run here.
"""
from __future__ import annotations

import json
import os
import subprocess
import sys
from pathlib import Path

import pytest

from test_gemm_paths_gpu import CASES, Case, F_F32, F_SPLIT, F_X3, P

HERE = Path(__file__).resolve().parent
SWITCHES = ("B2P_SPLITK_LAST", "B2P_DENSE_GRIDS", "B2P_NO_HALO", "B2P_NO_SPLITK", "B2P_NO_BRES", "B2P_NO_HALO32")
# every process starts without these, then sets its own
ENV_SWITCHES = SWITCHES + ("B2P_PDL_SIMT", "B2P_GEMM_LN", "B2P_NO_TMA_EPI", "B2P_CTA_PENALTY", "B2P_MAX_GRID")

# conv tiles spanning nb > 1 whole images with split-K: the last arriver's own row -> (image, pixel) mapping
NB_SPLIT = [
    Case("conv s1 fp16x3 nb 8 over batch 13, split-K 12", 13, 4, 4, 256, 48, 1, 512, 96, 96, F_X3 | F_SPLIT, 1, 1, 1, 0, 0, 0,
         expect=dict(mode=1, nb=8, m_tiles=2, ksplit=12)),
    Case("conv s2 nb 8 over batch 11, split-K 9", 11, 8, 8, 256, 32, 2, 256, 32, 32, 0, 1, 1, 1, 0, 0, 0,
         expect=dict(mode=2, nb=8, m_tiles=2, ksplit=9)),
    Case("conv s2 nb 11 = batch, 44 of 128 rows, split-K 9", 11, 4, 4, 512, 16, 2, 512, 16, 0, F_F32, 0, 1, 0, 0, 0, 0,
         expect=dict(mode=2, nb=11, m_tiles=1, ksplit=9)),
]

# one production call per path class that the switch adds (classes no case of CASES has under the switch): the smallest
# call of the class in the plans test_gemm_plan_cpu.production_calls() records.  Columns as test_gemm_paths_gpu.Case.
SWITCH_CASES = {
    "B2P_DENSE_GRIDS": [
        P(16, 1, 1, 768, 768, 0, 1536, 768, 0, 10, 0, 1, 0, 0, 0, 0),  # florence 768 K16 fp16x3
        P(12800, 1, 1, 64, 64, 0, 128, 64, 0, 10, 0, 1, 0, 64, 0, 0),  # yolo B8 fp16x3
        P(25600, 1, 1, 64, 64, 0, 512, 128, 0, 12, 1, 1, 0, 256, 64, 0),  # yolo B1 fp16x3
        P(128, 1, 1, 1024, 3072, 0, 2048, 3072, 0, 10, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16x3
        P(131072, 1, 1, 160, 128, 0, 320, 128, 0, 10, 0, 1, 0, 0, 0, 0),  # florence 64 K512 fp16x3
        P(131072, 1, 1, 128, 128, 0, 256, 128, 128, 10, 0, 1, 1, 0, 0, 0),  # florence 64 K512 fp16x3
        P(6656, 1, 1, 768, 768, 0, 1536, 768, 768, 10, 0, 1, 1, 0, 0, 0),  # florence 64 K512 fp16x3
        P(1600, 1, 1, 768, 512, 0, 1536, 2048, 0, 12, 1, 1, 0, 768, 1024, 0),  # yolo B1 fp16x3
        P(416, 1, 1, 768, 1536, 0, 1536, 1536, 0, 10, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16x3
        P(6400, 1, 1, 64, 64, 0, 64, 64, 0, 2, 0, 1, 0, 0, 0, 0),  # yolo B1 fp16
        P(16, 1, 1, 768, 768, 0, 768, 768, 0, 2, 0, 1, 0, 0, 0, 0),  # florence 768 K16 fp16
        P(6400, 1, 1, 128, 128, 0, 128, 256, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
        P(12800, 1, 1, 64, 64, 0, 64, 64, 0, 2, 0, 1, 0, 0, 0, 0),  # yolo B8 fp16
        P(16, 1, 1, 768, 2304, 0, 768, 2304, 0, 2, 0, 1, 0, 0, 0, 0),  # florence 768 K16 fp16
        P(400, 1, 1, 1024, 512, 0, 1024, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
        P(128, 1, 1, 1024, 3072, 0, 1024, 3072, 0, 2, 0, 1, 0, 0, 0, 0),  # florence 64 K32 fp16
        P(2560, 1, 1, 1024, 768, 0, 1024, 768, 0, 2, 0, 0, 0, 0, 0, 0),  # florence 64 K512 fp16
        P(800, 1, 1, 1024, 512, 0, 1024, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B2 fp16
        P(128, 1, 1, 1024, 4096, 0, 1024, 4096, 0, 0, 2, 1, 0, 0, 0, 0),  # florence 64 K32 fp16
        P(6656, 1, 1, 768, 768, 0, 768, 768, 768, 2, 0, 1, 1, 0, 0, 0),  # florence 64 K512 fp16
        P(1600, 1, 1, 1536, 512, 0, 1536, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
        P(2048, 1, 1, 4608, 1024, 0, 4608, 1024, 0, 2, 0, 1, 0, 0, 0, 0),  # florence 64 K512 fp16
        P(2048, 1, 1, 4096, 1024, 0, 4096, 1024, 1024, 2, 0, 1, 1, 0, 0, 0),  # florence 64 K512 fp16
        P(1, 40, 40, 64, 64, 1, 640, 128, 0, 12, 1, 1, 0, 320, 64, 0),  # yolo B1 fp16x3
        P(2, 20, 20, 512, 320, 1, 1024, 640, 0, 12, 1, 1, 0, 512, 320, 0),  # yolo B2 fp16x3
        P(1, 40, 40, 512, 320, 1, 512, 320, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
        P(1, 20, 20, 512, 320, 1, 512, 320, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
        P(2, 20, 20, 512, 320, 1, 512, 320, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B2 fp16
        P(8, 20, 20, 512, 320, 1, 512, 320, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B8 fp16
    ],
    "B2P_NO_HALO": [
        P(1, 20, 20, 256, 256, 1, 256, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
        P(1, 20, 20, 256, 256, 1, 256, 256, 512, 0, 1, 1, 1, 0, 0, 0),  # yolo B1 fp16
        P(8, 40, 40, 64, 64, 1, 320, 64, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B8 fp16
        P(2, 80, 80, 64, 64, 1, 64, 64, 128, 0, 1, 1, 1, 0, 0, 0),  # yolo B2 fp16
        P(2, 20, 20, 256, 256, 1, 256, 1024, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B2 fp16
        P(2, 20, 20, 256, 256, 1, 256, 256, 512, 0, 1, 1, 1, 0, 0, 0),  # yolo B2 fp16
        P(1, 20, 20, 512, 512, 1, 512, 2048, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B1 fp16
        P(2, 20, 20, 512, 512, 1, 512, 2048, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B2 fp16
        P(2, 40, 40, 512, 320, 1, 512, 320, 0, 0, 1, 1, 0, 0, 0, 0),  # yolo B2 fp16
    ],
    "B2P_NO_SPLITK": [
        P(8, 40, 40, 512, 512, 2, 1024, 2048, 0, 12, 1, 1, 0, 512, 1024, 0),  # yolo B8 fp16x3
    ],
}

# every case any process may run, by a stable index (the seed of run_case is 1000 + index in every process, so the
# default and the switched process see the same operands)
ALL_CASES = list(CASES) + NB_SPLIT
N_CASES = len(CASES)
OWN = {}                           # switch -> indices of its own cases in ALL_CASES
for _s in SWITCHES:
    OWN[_s] = range(len(ALL_CASES), len(ALL_CASES) + len(SWITCH_CASES.get(_s, [])))
    ALL_CASES += SWITCH_CASES.get(_s, [])


def switch_env(*on):
    """this process's environment without any planner / kernel switch, then the given ones set to 1"""
    env = {k: v for k, v in os.environ.items() if k not in ENV_SWITCHES}
    env.update({k: "1" for k in on})
    return env


_PLAN_SCRIPT = r"""
import json, sys
sys.path[:0] = [{here!r}, {root!r}]
import test_gemm_switches_gpu as S
from test_gemm_paths_gpu import case_args
from gemm_plan_util import H100_SXM, path_class, plan
from omniparser_b200 import _lib
out = []
for c in S.ALL_CASES:
    args = case_args(c, base=1 << 24)
    try:
        p = plan(args, *H100_SXM)
        out.append({{"plan": p, "cls": list(path_class(p, args))}})
    except _lib.B2PError as e:
        out.append({{"error": str(e)}})
json.dump(out, open({path!r}, "w"))
"""


def case_plans(switch, path):
    """[{"plan", "cls"} or {"error"}] of every case of ALL_CASES at H100 SXM limits, planned in a process with `switch` set
    (None: the default process)"""
    code = _PLAN_SCRIPT.format(here=str(HERE), root=str(HERE.parent), path=str(path))
    r = subprocess.run([sys.executable, "-c", code], env=switch_env(*([switch] if switch else [])), capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return json.loads(Path(path).read_text())


def same_k_order(pd, ps):
    """the two plans add the same products in the same order into each output element: no split-K in either or the same
    split, and the same sequence of k-blocks (the halo tile loops taps inside a channel block, the per-tap path channel
    blocks inside a tap: the same order only with one channel block)"""
    if pd["ksplit"] != ps["ksplit"] or pd["bk"] != ps["bk"] or pd["kb_merge"] != ps["kb_merge"] or pd["x3"] != ps["x3"]:
        return False
    modes = {pd["mode"], ps["mode"]}
    if len(modes) == 1:
        return True
    if modes == {1, 3}:
        halo = pd if pd["mode"] == 3 else ps
        return halo["num_kb"] == 1          # a halo plan's k-blocks are its channel blocks
    return False


def selection(switch, default, switched):
    """-> (indices of ALL_CASES to run under the switch, indices whose output must equal the default's byte for byte).
    Park-only cases (all in CASES) run through b2p_gemm_ln, as in test_gemm_paths_gpu."""
    run, same = [], []
    for i, (d, s) in enumerate(zip(default, switched)):
        if "error" in s:
            continue                        # (park-only plans under B2P_NO_SPLITK)
        if switch == "B2P_SPLITK_LAST":
            if s["plan"]["ksplit"] > 1 and not s["plan"]["park"] and i < N_CASES + len(NB_SPLIT):
                run.append(i)
                same.append(i)
        elif i in OWN[switch] or (i < N_CASES and s["plan"] != d["plan"]):
            run.append(i)
            if switch in ("B2P_NO_BRES", "B2P_NO_HALO32") and not s["plan"]["park"] and same_k_order(d["plan"], s["plan"]):
                same.append(i)
    return run, same


_RUN_SCRIPT = r"""
import json, sys, torch
sys.path[:0] = [{here!r}, {root!r}]
import test_gemm_paths_gpu as T
import test_gemm_switches_gpu as S
from gemm_plan_util import FLAG_PARK
job = json.loads({job!r})
outs = {{}}
orig = T._launch
def launch(c, bufs, torch_):
    orig(c, bufs, torch_)
    torch.cuda.synchronize()
    outs["last"] = bufs["out"].clone().cpu()
T._launch = launch
res = {{}}
for i in job["run"]:
    c = S.ALL_CASES[i]
    if c.flags & FLAG_PARK:        # park-only GEMM + b2p_gemm_ln, against fp64 LayerNorm
        T.test_gemm_ln_path(i)
        continue
    ratio, p = T.run_case(c, 1000 + i)
    print(f"[switch case] {{i}} {{c.name}}: max error / bound = {{ratio:.3g}}", flush=True)
    if i in job["keep"]:
        res[i] = outs["last"]
if job["e2e"]:
    res.update(S.end_to_end())
torch.save(res, job["path"])
"""


def run_gpu(env, run, keep, e2e, path):
    job = json.dumps({"run": run, "keep": keep, "e2e": e2e, "path": str(path)})
    code = _RUN_SCRIPT.format(here=str(HERE), root=str(HERE.parent), job=job)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    import torch
    return torch.load(path)


def end_to_end():
    """{name: tensor on the CPU}: the fp16 detector at B=1, 640x640 (head tensors) and the fp16x3 captioner at 32 crops
    (encoder states, the logits of two decode steps), eager launches on seeded stand-in weights and inputs"""
    import torch
    from omniparser_b200.florence_engine import FlorencePlan, FlorenceWeights
    from omniparser_b200.yolo_engine import YoloPlan, YoloWeights
    from standin import florence as FS
    from standin.yolo_weights import yolo_standin
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(11)
    out = {}
    yp = YoloPlan(YoloWeights(yolo_standin(0).state_dict(), dev, precision="fp16"), 1, 640, 640, use_graph=False)
    yp.canvas.copy_(torch.randint(0, 256, yp.canvas.shape, dtype=torch.uint8, generator=g).to(dev))
    yp.run()
    torch.cuda.synchronize()
    for i, (c, b) in enumerate(zip(yp.cls_out, yp.box_out)):
        out[f"yolo cls {i}"], out[f"yolo box {i}"] = c.cpu(), b.cpu()
    fw = FlorenceWeights(FS.florence_standin(0).state_dict(), dev, FS.GEN, "fp16x3")
    fp = FlorencePlan(fw, 32, 8, FS.PROMPT_IDS, use_graph=False)
    fp.crops.copy_(torch.randint(0, 256, fp.crops.shape, dtype=torch.uint8, generator=g).to(dev))
    fp.encode()
    fp.reset_decode(32)
    torch.cuda.synchronize()
    out["florence encoder"] = fp.enc_out32.cpu()
    for t in range(2):
        fp.decode_step()
        torch.cuda.synchronize()
        out[f"florence logits {t}"] = fp.logits.cpu()
    return out


def _bits(t):
    import torch
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _differ(a, b, keys):
    import torch
    return [k for k in keys if not torch.equal(_bits(a[k]), _bits(b[k]))]


@pytest.fixture(scope="module")
def plans(tmp_path_factory):
    d = tmp_path_factory.mktemp("plans")
    return {s: case_plans(s, d / f"{s}.json") for s in (None,) + SWITCHES}


@pytest.fixture(scope="module")
def default_run(plans, tmp_path_factory):
    """the default process: every case some switch compares byte for byte, and the end-to-end run"""
    keep = sorted({i for s in SWITCHES for i in selection(s, plans[None], plans[s])[1]})
    return run_gpu(switch_env(), keep, keep, True, tmp_path_factory.mktemp("default") / "out.pt")


@pytest.mark.gpu
@pytest.mark.parametrize("switch", SWITCHES)
def test_switch_cases(switch, plans, default_run, tmp_path):
    run, same = selection(switch, plans[None], plans[switch])
    assert run, f"{switch}: no case to run"
    e2e = switch == "B2P_SPLITK_LAST"
    got = run_gpu(switch_env(switch), run, same, e2e, tmp_path / "out.pt")
    bad = _differ(default_run, got, same)
    assert not bad, f"{switch}: cases whose bytes differ from the default process: {[(i, ALL_CASES[i].name) for i in bad]}"
    if e2e:
        keys = [k for k in default_run if isinstance(k, str)]
        bad = _differ(default_run, got, keys)
        assert not bad, f"{switch}: end-to-end tensors that differ from the default process: {bad}"
    print(f"{switch}: {len(run)} cases within the fp64 bound, {len(same)} byte-identical to the default")


@pytest.mark.gpu
def test_pdl_simt_end_to_end(default_run, tmp_path):
    """B2P_PDL_SIMT: the small SIMT kernels launch with programmatic dependent launch; results must not change"""
    got = run_gpu(switch_env("B2P_PDL_SIMT"), [], [], True, tmp_path / "out.pt")
    keys = [k for k in default_run if isinstance(k, str)]
    assert sorted(keys) == sorted(got)
    bad = _differ(default_run, got, keys)
    assert not bad, f"B2P_PDL_SIMT: end-to-end tensors that differ from the default process: {bad}"
