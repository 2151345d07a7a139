#!/usr/bin/env python
"""Throughput of mvs_fit_stream against batches, on the benchmark workload (bench.py: synthetic frames, 8 views, GMM + angle +
shape priors, the four-stage schedule with the SDF term as written in stages 2-3, grid 128).

    python scripts/stream_throughput.py [--frames 2048] [--slots 256] [--reps 3] [--out FILE]

The same F frames are fitted three ways:
  (a) stream    one context with B slots, ONE mvs_fit_stream call over all F frames
  (b) inflight  F / B contexts of B frames each, driven concurrently by as many host threads on their own streams (what
                bench.py's lanes do)
  (c) serial    the F / B batches one after another through one context (mvs_fit)
For each: frame-iterations/s (wall time of the whole fit, inputs already on the device), dense rounds, and the card name and
power limit.  Arms alternate over the repetitions; the fitted parameters of the three must be byte-identical."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                      text=True, timeout=30).strip().splitlines()[0]
        name, limit = [c.strip() for c in out.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception as e:                                        # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "unknown (%r)" % e}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=2048)
    ap.add_argument("--slots", type=int, default=256)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from bench import stage_table
    from mvsmplfitting_b200 import synthetic as S
    from mvsmplfitting_b200.context import FittingContext

    F, B = args.frames, args.slots
    assert F % B == 0, "--frames must be a multiple of --slots"
    nb = F // B
    dev = torch.device("cuda", 0)
    model, gmm, cams = S.make_model(0), S.make_gmm(7), S.make_cameras(args.views)
    fr = S.make_frames(model, cams, F, seed=4242)
    X0 = torch.tensor(S.pack_params(fr["init"]), device=dev)
    gt, cf = torch.tensor(fr["gt_uv"], device=dev), torch.tensor(fr["conf"], device=dev)
    jw = torch.tensor(fr["joint_weights"], device=dev)

    def new_ctx():
        ctx = FittingContext(0)
        ctx.set_model(model)
        ctx.set_gmm_from_dict(gmm)
        ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
        ctx.set_batch(B)
        return ctx

    ctx_s = new_ctx()
    lanes = [new_ctx() for _ in range(nb)]
    streams = [torch.cuda.Stream(device=dev) for _ in range(nb)]
    cfgs = [ctx_s.make_loss_config(body_prior="gmm", interpenetration=True, sdf_grid=128, **st) for st in stage_table()]
    opt = ctx_s.make_lbfgs_config()
    chunk = lambda i: (gt[:, i * B:(i + 1) * B].contiguous(), cf[:, i * B:(i + 1) * B].contiguous())
    for i, ln in enumerate(lanes):
        ln.set_keypoints(*chunk(i), jw)

    def arm_stream():
        x = X0.clone()
        _, st = ctx_s.fit_stream(x, gt, cf, jw, cfgs, opt)
        return x, [st]

    def arm_inflight():
        xs = [X0[i * B:(i + 1) * B].clone() for i in range(nb)]
        torch.cuda.synchronize()                                  # the copies are on the default stream, the fits on their own
        sts, err = [None] * nb, []

        def work(i):
            try:
                with torch.cuda.stream(streams[i]):
                    sts[i] = lanes[i].fit(xs[i], cfgs, opt)[1]
                    streams[i].synchronize()
            except Exception as e:                                # noqa: BLE001 -- re-raised below
                err.append(e)
        th = [threading.Thread(target=work, args=(i,)) for i in range(nb)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        if err:
            raise err[0]
        return torch.cat(xs), sts

    def arm_serial():
        ctx = lanes[0]
        xs, sts = [], []
        for i in range(nb):
            ctx.set_keypoints(*chunk(i), jw)
            x = X0[i * B:(i + 1) * B].clone()
            sts.append(ctx.fit(x, cfgs, opt)[1])
            xs.append(x)
        ctx.set_keypoints(*chunk(0), jw)
        return torch.cat(xs), sts

    arms = {"stream": arm_stream, "inflight": arm_inflight, "serial": arm_serial}
    names = list(arms)
    for n in names:                                               # warm-up (allocations, first-use set-up)
        arms[n]()
    runs = {n: [] for n in names}
    for r in range(args.reps):
        order = names[r % 3:] + names[:r % 3]
        outs = {}
        for n in order:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            x, sts = arms[n]()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            outs[n] = x.cpu().numpy()
            it = sum(s["frame_iterations"] for s in sts)
            runs[n].append({"seconds": dt, "frame_iterations_per_s": it / dt, "frame_iterations": it,
                            "dense_rounds": [s["dense_rounds"] for s in sts]})
        same = all(outs[n].tobytes() == outs["stream"].tobytes() for n in names)
        print("rep %d order %s: %s; params byte-identical: %s" % (r, ",".join(order), ", ".join(
            "%s %.0f it/s" % (n, runs[n][-1]["frame_iterations_per_s"]) for n in names), same), file=sys.stderr)
        assert same, "the three arms fitted different parameters"
    info = card()
    res = {"workload": "%d frames x %d views, %d slots per context; 4-stage schedule, GMM + angle + shape priors, SDF as written "
                       "in stages 2-3 (grid 128)" % (F, args.views, B), **info,
           "arms": {"stream": "one context, one mvs_fit_stream call",
                    "inflight": "%d contexts x %d frames on %d host threads" % (nb, B, nb),
                    "serial": "%d batches of %d one after another on one context" % (nb, B)},
           "params_byte_identical": True,
           "median_frame_iterations_per_s": {n: float(np.median([q["frame_iterations_per_s"] for q in runs[n]])) for n in names},
           "dense_rounds": {n: runs[n][0]["dense_rounds"] for n in names},
           "runs": runs}
    for c in [ctx_s] + lanes:
        c.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
