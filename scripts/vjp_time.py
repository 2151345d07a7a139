"""Time mvs_forward_vjp (exec modes 0 and 1), forward + backward through the autograd Function, and -- as the baseline a
user runs today -- torch autograd through oracle.closure_oracle.smpl_forward on CUDA in float32 (vmapped over the batch),
with dense cotangents on vertices and joints, at B = 1, 16, 64, 256.  CUDA events around REPS calls after WARM calls; the
card's name, power limit and largest SM clock are printed in the same run.

    python scripts/vjp_time.py [--reps 50] [--out vjp_time.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mvsmplfitting_b200 import synthetic as S                       # noqa: E402
from mvsmplfitting_b200.autograd import smpl_apply                  # noqa: E402
from mvsmplfitting_b200.context import FittingContext               # noqa: E402
from oracle import closure_oracle as O                              # noqa: E402

SEGS = ((0, 10), (10, 13), (13, 82), (82, 85), (85, 86))


def timed(fn, warm, reps):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warm", type=int, default=5)
    ap.add_argument("--batches", default="1,16,64,256")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vjp_time.py needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print("card:", card)
    model = S.make_model(0)
    N = model["v_template"].shape[0]
    om = O.OracleModel.from_numpy(model, dtype=torch.float32)
    for f in ("v_template", "shapedirs", "posedirs", "J_regressor", "lbs_weights", "lsp_regressor"):
        setattr(om, f, getattr(om, f).cuda())

    def oracle_one(x):
        v, j, _ = O.smpl_forward(om, *[x[a:e].view(1, -1) for a, e in SEGS])
        return v, j
    oracle_batch = torch.vmap(oracle_one)
    rows = []
    for B in [int(b) for b in a.batches.split(",")]:
        ctx = FittingContext(0)
        ctx.set_model(model)
        ctx.set_batch(B)
        rng = np.random.RandomState(B)
        X = S.pack_params(S.make_frames(model, S.make_cameras(2), B, seed=5)["gt"])
        x = torch.tensor(X, device="cuda")
        gv = torch.tensor(rng.normal(0, 1, (B, N, 3)).astype(np.float32), device="cuda")
        gj = torch.tensor(rng.normal(0, 1, (B, ctx.K, 3)).astype(np.float32), device="cuda")
        row = dict(B=B)
        for mode in (0, 1):
            ctx.set_exec_mode(mode)
            row["vjp_mode%d_ms" % mode] = timed(lambda: ctx.forward_vjp(x, gj, gv), a.warm, a.reps)
        ctx.set_exec_mode(0)

        def fwd_bwd():
            xp = x.clone().requires_grad_(True)
            j, v = smpl_apply(ctx, xp)
            ((v * gv).sum() + (j * gj).sum()).backward()
        row["function_fwd_bwd_ms"] = timed(fwd_bwd, a.warm, a.reps)
        ctx.close()

        def baseline():
            xp = x.clone().requires_grad_(True)
            with torch.device("cuda"):                           # the oracle's own constants (eye, ones) on the device too
                v, j = oracle_batch(xp)
            ((v * gv).sum() + (j * gj).sum()).backward()
        row["torch_autograd_fp32_ms"] = timed(baseline, 2, max(3, a.reps // 5))
        print(json.dumps(row))
        rows.append(row)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(card=card, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
