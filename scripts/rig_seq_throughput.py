#!/usr/bin/env python
"""Throughput of fitting video sequences recorded by different camera rigs: one seqio.fit_sequences call per rig against one
call with rigs=.

    python scripts/rig_seq_throughput.py [--sequences 64] [--mean-length 16] [--slots 32] [--reps 3] [--out FILE]

S sequences of unequal length (make_frames(smooth_walk=True)) are spread over R rigs that differ in view count (4..8),
placement, focal length, principal point and data-weight scale, for R = S (one rig per sequence) and R = 4.  Two arms:
  (a) per_rig   what a context with one set of cameras allows: for every rig, set_cameras(rig) and one fit_sequences call over
                that rig's sequences, with every stage's data_weight scaled by the rig's factor
  (b) rigs      set_camera_rigs once and ONE fit_sequences(rigs=...) call over all sequences
Both arms use a context of --slots slots; with the defaults no call has exactly that many sequences, so every call runs the
sequence stream (mvs_fit_seq_stream, or its _rigs form).  Configurations:
'shipped' (VPoser latent pose with the shipped snapshot, L2 prior, SDF off) and 'bench' (bench.py's GMM schedule, SDF as
written in stages 2-3, grid 128).  Wall time covers the initial guesses and the fit, inputs on the host.  frame-iterations/s
counts the iterations of the fitted frames (the sum (b) reports).  Arms alternate; the median of --reps runs is reported; the
fitted parameters of the two arms must be byte-identical."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from scripts.stream_throughput import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sequences", type=int, default=64)
    ap.add_argument("--mean-length", type=int, default=16)
    ap.add_argument("--slots", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rigs", default="64,4", help="numbers of rigs (one rig per sequence when equal to --sequences)")
    ap.add_argument("--configs", default="shipped,bench")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from bench import stage_table
    from mvsmplfitting_b200 import seqio
    from mvsmplfitting_b200 import synthetic as S
    from mvsmplfitting_b200.context import FittingContext
    from tests import golden_util as G

    S_, T = args.sequences, args.mean_length
    rng = np.random.RandomState(78)
    lengths = [int(n) for n in rng.randint(T // 2, T + T // 2 + 1, size=S_)]
    model, gmm = S.make_model(0), S.make_gmm(7)
    vposer_w = G.snapshot_vposer_weights()

    def make_rigs(R, seed):
        g = np.random.RandomState(seed)
        rigs, scales = [], []
        for _ in range(R):
            V = int(g.randint(4, 9))
            rigs.append(S.make_cameras(V, radius=float(g.uniform(16.0, 24.0)), focal=float(g.uniform(1800.0, 3000.0)),
                                       center=(float(g.uniform(900.0, 1150.0)), float(g.uniform(500.0, 850.0)))))
            scales.append(np.float32(1536.0 / g.choice([1080.0, 1536.0, 2048.0])))        # 500 / H over the bench's 500 / 1536
        return rigs, np.array(scales, np.float32)

    def new_ctx(B, vposer):
        ctx = FittingContext(0)
        ctx.set_model(model)
        ctx.set_gmm_from_dict(gmm)
        ctx.set_batch(B)
        if vposer:
            ctx.set_vposer(vposer_w)
        return ctx

    info = card()
    out = {"workload": "%d sequences of %d..%d frames (%d frames), 4..8 views per rig; contexts of %d slots"
                       % (S_, min(lengths), max(lengths), sum(lengths), args.slots), **info, "cases": {}}
    for R in [int(r) for r in args.rigs.split(",")]:
        rigs, scales = make_rigs(R, 500 + R)
        seq_rig = np.arange(S_) % R
        seqs = []
        for s_, n in enumerate(lengths):
            cams = rigs[seq_rig[s_]]
            fr = S.make_frames(model, cams, n, seed=9100 + s_, smooth_walk=True)
            seqs.append(dict(gt_uv=fr["gt_uv"], conf=fr["conf"], present=np.ones(fr["conf"].shape[:2], bool),
                             frames=["%05d" % t for t in range(n)], serial="s%03d" % s_, rig=int(seq_rig[s_])))
        for name in args.configs.split(","):
            vposer = name == "shipped"
            ctx_a, ctx_b = new_ctx(args.slots, vposer), new_ctx(args.slots, vposer)

            def cfgs(ctx, scale=np.float32(1.0)):
                out_ = []
                for st in stage_table():
                    st = dict(st, data_weight=float(np.float32(np.float32(st["data_weight"]) * np.float32(scale))))
                    if vposer:
                        st.pop("coll_loss_weight")
                        out_.append(ctx.make_loss_config(body_prior="l2", use_vposer=2, **st))
                    else:
                        out_.append(ctx.make_loss_config(body_prior="gmm", interpenetration=True, sdf_grid=128, **st))
                return out_

            opt = ctx_a.make_lbfgs_config()

            def arm_per_rig(sub):
                x = [None] * len(sub)
                its = 0
                for r in range(R):
                    mine = [i for i, q in enumerate(sub) if q["rig"] == r]
                    if not mine:
                        continue
                    c = rigs[r]
                    ctx_a.set_cameras(c["R"], c["t"], c["f"], c["c"])
                    res, tot = seqio.fit_sequences(ctx_a, [sub[i] for i in mine], cfgs(ctx_a, scales[r]), opt,
                                                   estimate_scale=True, pose_format="lsp14")
                    its += tot["frame_iterations"]
                    for i, rr in zip(mine, res):
                        x[i] = rr[0]
                return np.concatenate(x), its

            def arm_rigs(sub):
                res, tot = seqio.fit_sequences(ctx_b, sub, cfgs(ctx_b), opt, estimate_scale=True, pose_format="lsp14",
                                               rigs=rigs, rig_data_weight_scale=scales)
                return np.concatenate([r[0] for r in res]), tot["frame_iterations"]

            arms = {"per_rig": arm_per_rig, "rigs": arm_rigs}
            names = list(arms)
            for n in names:                                       # warm-up (allocations, first-use set-up)
                arms[n](seqs[:4])
            runs = {n: [] for n in names}
            for r in range(args.reps):
                order = names if r % 2 == 0 else names[::-1]
                outs, its = {}, {}
                for n in order:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    outs[n], its[n] = arms[n](seqs)
                    torch.cuda.synchronize()
                    runs[n].append({"seconds": time.perf_counter() - t0})
                same = outs["per_rig"].tobytes() == outs["rigs"].tobytes()
                for n in names:
                    runs[n][-1]["frame_iterations_per_s"] = its["rigs"] / runs[n][-1]["seconds"]
                print("%d rigs, %s rep %d order %s: %s; params byte-identical: %s" % (R, name, r, ",".join(order), ", ".join(
                    "%s %.2f s" % (n, runs[n][-1]["seconds"]) for n in names), same), file=sys.stderr)
                assert same, "the arms fitted different parameters"
            med = {n: float(np.median([q["seconds"] for q in runs[n]])) for n in names}
            out["cases"]["%d_rigs_%s" % (R, name)] = {
                "stages": "VPoser latent pose (shipped snapshot), L2 prior, SDF off" if vposer else
                          "GMM + angle + shape priors, SDF as written in stages 2-3 (grid 128)",
                "frame_iterations": its["rigs"], "params_byte_identical": True, "median_seconds": med,
                "median_frame_iterations_per_s": {n: float(np.median([q["frame_iterations_per_s"] for q in runs[n]]))
                                                  for n in names},
                "speedup_rigs_over_per_rig": med["per_rig"] / med["rigs"], "runs": runs}
            ctx_a.close()
            ctx_b.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
