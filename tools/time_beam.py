"""Caption generate() time by beam count: 416 64x64 crops x 20 new tokens, fp16x3, seeded stand-in weights.

    python tools/time_beam.py [--beams 1 3 5] [--crops 416] [--tokens 20] [--reps 5]

Each setting is warmed up (plan build + CUDA-graph capture) and then timed with CUDA events around whole generate()
calls; prints the card name and power limit with the numbers."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--beams", type=int, nargs="+", default=[1, 3, 5])
    ap.add_argument("--crops", type=int, default=416)
    ap.add_argument("--tokens", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_beam.py needs a CUDA device")
    from __graft_entry__ import build
    from omniparser_b200.caption import B200Florence2Model
    from standin import florence as FS
    build()
    dev = torch.device("cuda", 0)
    model = B200Florence2Model(FS.florence_standin(0).state_dict(), dev, FS.GEN, precision="fp16x3")
    g = torch.Generator().manual_seed(0)
    crops = torch.randint(0, 256, (args.crops, 64, 64, 3), dtype=torch.uint8, generator=g).to(dev)
    ids = FS.input_ids_for(args.crops)
    res = {}
    for nb in args.beams:
        kw = dict(num_beams=nb, early_stopping=True) if nb > 1 else {}
        model.generate(input_ids=ids, pixel_values=crops, max_new_tokens=args.tokens, **kw)   # warm-up: plan + graphs
        torch.cuda.synchronize()
        times = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = model.generate(input_ids=ids, pixel_values=crops, max_new_tokens=args.tokens, **kw)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        res[nb] = dict(ms_min=min(times), ms_median=sorted(times)[len(times) // 2], out_shape=list(out.shape))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps(dict(gpu=q.stdout.strip(), crops=args.crops, tokens=args.tokens, precision="fp16x3", generate_ms=res)))


if __name__ == "__main__":
    main()
