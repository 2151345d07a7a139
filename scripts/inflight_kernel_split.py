"""device time per kernel in the headline configuration: the bench.py workload (256 frames x 8 views, SDF term on) with
--inflight batches in flight, a few steps under torch.profiler (CUDA activities).

    python scripts/inflight_kernel_split.py [--inflight 8] [--steps 4] [--warmup 2] [--out DIR]

Prints device milliseconds, share and launch count per kernel name over the profiled steps (all lanes together), and writes
the table as JSON to DIR/inflight_kernel_split.json when --out is given.  Kernels of different lanes overlap on the device,
so the shares are of summed kernel time, not of wall time."""
import argparse
import json
import os
import sys
import threading

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import bench  # noqa: E402
from mvsmplfitting_b200 import synthetic as S  # noqa: E402
from mvsmplfitting_b200.context import FittingContext  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--inflight", type=int, default=8)
    ap.add_argument("--steps", type=int, default=4, help="profiled steps per lane")
    ap.add_argument("--warmup", type=int, default=2, help="steps per lane before profiling")
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    model, gmm, cams = S.make_model(0), S.make_gmm(7), S.make_cameras(a.views)
    lanes = []
    for i in range(a.inflight):                      # the bench.py lanes: own context, frames (same seeds) and stream
        fr = S.make_frames(model, cams, a.frames, seed=1000 + 97 * i)
        ctx = FittingContext(0)
        ctx.set_model(model); ctx.set_gmm_from_dict(gmm); ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
        ctx.set_batch(a.frames)
        stages = [ctx.make_loss_config(body_prior="gmm", interpenetration=True, sdf_grid=128, **st) for st in bench.stage_table()]
        x0 = torch.tensor(S.pack_params(fr["init"]), device="cuda")
        ctx.set_keypoints(torch.tensor(fr["gt_uv"], device="cuda"), torch.tensor(fr["conf"], device="cuda"),
                          torch.tensor(fr["joint_weights"], device="cuda"))
        lanes.append(dict(ctx=ctx, stages=stages, opt=ctx.make_lbfgs_config(), x0=x0, x=x0.clone(), stream=torch.cuda.Stream()))

    def work(ln, n):
        with torch.cuda.stream(ln["stream"]):
            for _ in range(n):
                ln["x"].copy_(ln["x0"])
                ln["ctx"].fit(ln["x"], ln["stages"], ln["opt"])
            ln["stream"].synchronize()

    def run(n):
        th = [threading.Thread(target=work, args=(ln, n)) for ln in lanes]
        for t in th:
            t.start()
        for t in th:
            t.join()

    run(a.warmup)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(a.steps)
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time_total > 0:
            d = per.setdefault(e.name, [0.0, 0])
            d[0] += e.device_time_total / 1e3
            d[1] += 1
    total = sum(v[0] for v in per.values())
    rows = sorted(per.items(), key=lambda kv: -kv[1][0])
    table = [{"kernel": k, "device_ms": round(v[0], 3), "share": round(v[0] / total, 4), "launches": v[1],
              "avg_us": round(v[0] * 1e3 / v[1], 2)} for k, v in rows]
    dev = torch.cuda.get_device_properties(0)
    print("%s, %d lanes x %d steps, summed kernel time %.1f ms" % (dev.name, a.inflight, a.steps, total))
    for r in table[:20]:
        print("%-70s %10.3f ms  %6.2f %%  %7d launches  %8.2f us" % (r["kernel"][:70], r["device_ms"], 100 * r["share"], r["launches"], r["avg_us"]))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        json.dump({"gpu": dev.name, "inflight": a.inflight, "steps": a.steps, "kernels": table},
                  open(os.path.join(a.out, "inflight_kernel_split.json"), "w"), indent=1)
    for ln in lanes:
        ln["ctx"].close()


if __name__ == "__main__":
    main()
