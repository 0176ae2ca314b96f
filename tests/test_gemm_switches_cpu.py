"""CPU: the launch plans of the wgmma GEMM/conv kernel under each of its A/B switches (B2P_SPLITK_LAST, B2P_DENSE_GRIDS,
B2P_NO_HALO, B2P_NO_SPLITK, B2P_NO_BRES, B2P_NO_HALO32).

The planner reads the switches once per process, so each switch plans in its own subprocess.  The GEMM/conv calls of
test_gemm_plan_cpu.production_calls() are recorded once here (the recorder stands in for the library, so the calls do not
depend on the planner's switches) and handed to every subprocess, which plans each at H100 SXM and H100 PCIe limits.
Every plan must keep test_gemm_plan_cpu.check_invariants and fit in shared memory; what each switch does to production is
pinned as data; and the case lists of test_gemm_switches_gpu.py must run every path class each switch reaches.
Under B2P_SPLITK_LAST a split-K class is a class of its own: its reduction is different kernel code, and only a case run
in the switched process executes it."""
from __future__ import annotations

import json
import subprocess
import sys
from pathlib import Path

import pytest

from gemm_plan_util import planner_args
import test_gemm_switches_gpu as S

HERE = Path(__file__).resolve().parent

_SCRIPT = r"""
import json, sys
sys.path[:0] = [{here!r}, {root!r}]
from gemm_plan_util import H100_PCIE, H100_SXM, path_class, plan
from test_gemm_plan_cpu import check_invariants
from omniparser_b200 import _lib
calls = json.load(open({src!r}))
out = []
for name, call, args in calls:
    args = tuple(args)
    try:
        p = plan(args, *H100_SXM)
    except _lib.B2PError as e:
        out.append({{"error": str(e)}})
        continue
    for sms, smem in (H100_SXM, H100_PCIE):
        q = plan(args, sms, smem)
        assert q["smem"] <= smem, (name, call, q)
        check_invariants(q, args)
    out.append({{"plan": p, "cls": list(path_class(p, args))}})
json.dump(out, open({dst!r}, "w"))
"""

# switch -> (launches planned, split-K launches, launches in classes no case of CASES has under the switch, those classes,
#            launches the planner rejects, launches whose plan differs from the default), over the 3234 GEMM/conv launches
#            of production_calls() at 132 SMs and 232448 bytes of shared memory
TABLE = {
    "B2P_SPLITK_LAST": (3234, 375, 0, 0, 0, 0),
    "B2P_DENSE_GRIDS": (3234, 1243, 335, 29, 0, 1780),
    "B2P_NO_HALO": (3234, 409, 75, 9, 0, 387),
    "B2P_NO_SPLITK": (3198, 0, 2, 1, 36, 363),
    "B2P_NO_BRES": (3234, 375, 0, 0, 0, 168),
    "B2P_NO_HALO32": (3234, 375, 0, 0, 0, 48),
}
PARK_ONLY_REJECTION = "gemm (park-only): needs mode 0 and a split-K workspace slot for this stream"


@pytest.fixture(scope="module")
def switched(tmp_path_factory):
    """{switch or None: (plans of the production launches, plans of test_gemm_switches_gpu.ALL_CASES)}"""
    from test_gemm_plan_cpu import production_calls
    d = tmp_path_factory.mktemp("switches")
    calls = [(name, n, list(planner_args(n, a))) for name, cl in production_calls().items() for n, a in cl]
    src = d / "calls.json"
    src.write_text(json.dumps(calls))
    out = {"calls": calls}
    for s in (None,) + S.SWITCHES:
        dst = d / f"{s}.json"
        code = _SCRIPT.format(here=str(HERE), root=str(HERE.parent), src=str(src), dst=str(dst))
        r = subprocess.run([sys.executable, "-c", code], env=S.switch_env(*([s] if s else [])), capture_output=True, text=True,
                           timeout=900)
        assert r.returncode == 0, f"{s}: " + r.stdout[-3000:] + r.stderr[-3000:]
        out[s] = (json.loads(dst.read_text()), S.case_plans(s, d / f"cases-{s}.json"))
    return out


def _key(switch, e):
    """path class, plus whether the launch runs the last-arriver split-K reduction"""
    p = e["plan"]
    return tuple(e["cls"]) + (int(switch == "B2P_SPLITK_LAST" and p["ksplit"] > 1 and not p["park"]),)


def test_default_process_matches_the_production_table(switched):
    """the default subprocess plans what test_gemm_plan_cpu pins"""
    import collections
    from test_gemm_plan_cpu import PRODUCTION_CLASSES
    prod, _ = switched[None]
    assert all("plan" in e for e in prod)
    assert dict(collections.Counter(tuple(e["cls"]) for e in prod)) == PRODUCTION_CLASSES


@pytest.mark.parametrize("switch", S.SWITCHES)
def test_switch_table(switched, switch):
    prod, cases = switched[switch]
    default, _ = switched[None]
    planned = [e for e in prod if "plan" in e]
    case_cls = {tuple(e["cls"]) for e in cases[:S.N_CASES] if "plan" in e}
    outside = [tuple(e["cls"]) for e in planned if tuple(e["cls"]) not in case_cls]
    changed = sum(1 for d, e in zip(default, prod) if "plan" in e and d["plan"] != e["plan"])
    got = (len(planned), sum(e["plan"]["ksplit"] > 1 for e in planned), len(outside), len(set(outside)), len(prod) - len(planned),
           changed)
    print(f"\n{switch}: planned, split-K, outside CASES (launches, classes), rejected, changed = {got}")
    assert got == TABLE[switch]


def test_no_splitk_rejects_exactly_the_park_only_launches(switched):
    """B2P_NO_SPLITK: the park-only GEMMs of b2p_gemm_ln need a split-K workspace, so the planner refuses them (and
    FlorencePlan does not choose b2p_gemm_ln under the switch: test_plan_dryrun_cpu), and nothing else"""
    prod, _ = switched["B2P_NO_SPLITK"]
    rejected = [(c[0], c[1]) for c, e in zip(switched["calls"], prod) if "error" in e]
    assert rejected == [("florence 64 K32 fp16x3 B2P_GEMM_LN=1", "b2p_gemm_ln")] * 36
    assert {e["error"] for e in prod if "error" in e} == {PARK_ONLY_REJECTION}


@pytest.mark.parametrize("switch", S.SWITCHES)
def test_gpu_cases_cover_every_class_the_switch_reaches(switched, switch):
    """every class production reaches under the switch is run by a GPU case: in the switched process
    (test_gemm_switches_gpu) or, for a case whose plan the switch leaves as it is, in the default one (test_gemm_paths_gpu)"""
    prod, cases = switched[switch]
    _, default = switched[None]
    run, same = S.selection(switch, default, cases)
    covered = {_key(switch, cases[i]) for i in run}
    for i in range(S.N_CASES):
        e = cases[i]
        if "plan" in e and e["plan"] == default[i]["plan"] and not _key(switch, e)[-1]:
            covered.add(_key(switch, e))
    reached = {_key(switch, e) for e in prod if "plan" in e}
    missing = reached - covered
    assert not missing, f"{switch}: production classes without a GPU case: {sorted(missing)}"
    # each case of the switch's own list is needed: its class is one no case of CASES has under the switch
    case_cls = {tuple(e["cls"]) for e in cases[:S.N_CASES] if "plan" in e}
    own = [tuple(cases[i]["cls"]) for i in S.OWN[switch]]
    assert len(set(own)) == len(own) and not set(own) & case_cls and set(own) <= {k[:-1] for k in reached}
    assert set(same) <= set(run)
    if switch == "B2P_SPLITK_LAST":
        # every split-K case of CASES, the edges included, and the nb > 1 conv tiles run under the switch
        split = [i for i in range(S.N_CASES + len(S.NB_SPLIT)) if "plan" in cases[i] and cases[i]["plan"]["ksplit"] > 1
                 and not cases[i]["plan"]["park"]]
        assert run == same == split
        names = {S.ALL_CASES[i].name for i in run}
        assert {"split-K 5 (128 % 5 != 0)", "split-K 8, last slice short", "split-K 7 fp16x3, fp32 out",
                "split-K 14, a slice with no reduction rows", "split-K fp16x3 split out, unaligned lo slice"} <= names
    if switch == "B2P_NO_BRES":
        assert run == same and all(default[i]["plan"]["bres"] and not cases[i]["plan"]["bres"] for i in run)


def test_nb_split_cases_stay_on_their_paths(switched):
    """the planner does produce conv tiles of nb > 1 whole images with split-K, at both reductions"""
    for s in (None, "B2P_SPLITK_LAST"):
        _, cases = switched[s]
        for i, c in enumerate(S.NB_SPLIT):
            p = cases[S.N_CASES + i]["plan"]
            assert {k: p[k] for k in c.expect} == c.expect, (c.name, p)
