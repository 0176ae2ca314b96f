"""GPU: the TMA epilogue writes exactly the bytes the register epilogue writes.  Every case of test_gemm_paths_gpu.CASES
(plus cases where the TMA store has to clip: M not a multiple of 128 and N not a multiple of the N tile) runs here with
the default epilogue and again in one subprocess with B2P_NO_TMA_EPI=1 (the knob is read once per process); the written
slices must be byte-identical.  run_case itself checks that every byte outside the slice is still the NaN sentinel and
the result against fp64."""
from __future__ import annotations

import os
import subprocess
import sys
from pathlib import Path

import pytest

HERE = Path(__file__).resolve().parent

_SCRIPT = r"""
import sys, torch
sys.path[:0] = [{here!r}, {root!r}]
import test_gemm_paths_gpu as T
from gemm_plan_util import FLAG_PARK
cases = T.CASES + [
    T.Case("clip M", 300, 1, 1, 128, 96, 0, 128, 96, 96, 2, 0, 1, 1, 0, 0, 0),          # fp32 out + residual, 44 rows past M
    T.Case("clip N", 1000, 1, 1, 64, 120, 0, 64, 120, 120, 0, 1, 1, 1, 0, 0, 0),         # fp16 + residual, N tile past N
    T.Case("clip split", 777, 1, 1, 64, 72, 0, 64, 160, 160, 4, 0, 1, 1, 0, 80, 80),   # [hi | lo] out + residual pair
]
outs = {{}}
orig = T._launch
def launch(c, bufs, torch_):
    orig(c, bufs, torch_)
    torch.cuda.synchronize()
    outs[c.name, c.B, c.K, c.N, c.flags, c.ldc] = bufs["out"].clone().cpu()
T._launch = launch
res = {{}}
for i, c in enumerate(cases):
    if c.flags & FLAG_PARK:
        continue
    outs.clear()
    T.run_case(c, 1000 + i)
    (o,) = outs.values()
    res[i] = o
torch.save(res, {path!r})
"""


def _run(env_extra, path):
    env = dict(os.environ)
    env.update(env_extra)
    code = _SCRIPT.format(here=str(HERE), root=str(HERE.parent), path=str(path))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.gpu
def test_tma_epilogue_is_byte_identical(tmp_path):
    import torch
    os.environ.pop("B2P_NO_TMA_EPI", None)
    _run({}, tmp_path / "tma.pt")
    _run({"B2P_NO_TMA_EPI": "1"}, tmp_path / "reg.pt")
    a, b = torch.load(tmp_path / "tma.pt"), torch.load(tmp_path / "reg.pt")
    assert a.keys() == b.keys()
    bad = [i for i in a if not torch.equal(a[i].view(torch.int16 if a[i].dtype == torch.float16 else torch.int32),
                                           b[i].view(torch.int16 if b[i].dtype == torch.float16 else torch.int32))]
    assert not bad, f"cases whose bytes differ between the TMA and the register epilogue: {bad}"
