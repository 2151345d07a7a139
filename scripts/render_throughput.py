"""Throughput of mvs_render on an 8-view 2048 x 1536 rig (the synthetic wide rig) at 16, 64 and 256 frames.

Reports per call: the device time of each stage (torch.profiler, CUDA activities, in a run of its own), frame-views/s of the whole
call (CUDA events, profiler off), the raster kernel's achieved bytes/s against the composite's bandwidth bound (~6 B per pixel read
and written, at 3.35 TB/s), host cv2.imencode time per image for context, and the card's name and power limit read in the same
run.  Prints one JSON line (and writes it to --out when given).

    python scripts/render_throughput.py [--frames 16 64 256] [--reps 5] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from mvsmplfitting_b200 import synthetic as S  # noqa: E402
from mvsmplfitting_b200.context import FittingContext  # noqa: E402

W, H, V = 2048, 1536, 8
HBM_BPS = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = "nvidia-smi failed: %s" % e
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[16, 64, 256])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "render_throughput needs a GPU"
    model = S.make_model(0)
    cams = S.make_wide_cameras(V)
    nmax = max(a.frames)
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_camera_rigs([cams])
    ctx.set_batch(nmax)
    fr = S.make_frames_wide(model, cams, nmax, seed=3)
    fwd = ctx.forward_only(torch.tensor(S.pack_params(fr["gt"]), device="cuda"), want_verts=True)
    res = dict(card=card(), width=W, height=H, views=V, runs=[])
    for n in a.frames:
        verts, joints = fwd["verts"][:n].contiguous(), fwd["joints"][:n].contiguous()
        bg = torch.randint(0, 256, (n, V, H, W, 3), dtype=torch.uint8, device="cuda")
        out = ctx.render(verts, joints, background=bg)      # warm-up (grows the scratch)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for _ in range(a.reps):
            e0.record()
            out = ctx.render(verts, joints, background=bg)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) / 1e3)
        t = float(np.median(times))
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ctx.render(verts, joints, background=bg)
            torch.cuda.synchronize()
        stages = {}
        for ev in prof.key_averages():
            m = re.search(r"render_\w+_kernel(<\w+>)?", ev.key)
            k = m.group(0) if m else ("memset" if "memset" in ev.key.lower() else None)
            if k is not None:
                stages[k] = stages.get(k, 0.0) + ev.device_time_total / 1e3
        raster_ms = sum(v for k, v in stages.items() if "raster" in k)
        bytes_ = n * V * H * W * 6
        img = out["image"][0, 0].cpu().numpy()
        import cv2
        t0 = time.perf_counter()
        for _ in range(5):
            cv2.imencode(".jpg", img)
        enc = (time.perf_counter() - t0) / 5
        res["runs"].append(dict(frames=n, call_s=t, call_s_all=times, frame_views_per_s=n * V / t, stage_ms=stages,
                                raster_ms=raster_ms, composite_bytes=bytes_,
                                raster_bytes_per_s=bytes_ / (raster_ms / 1e3) if raster_ms else None,
                                raster_share_of_bandwidth_bound=(bytes_ / HBM_BPS) / (raster_ms / 1e3) if raster_ms else None,
                                call_share_of_bandwidth_bound=(bytes_ / HBM_BPS) / t, imencode_s_per_image=enc))
        del bg, out
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
