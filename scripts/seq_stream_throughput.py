#!/usr/bin/env python
"""Throughput of mvs_fit_seq_stream against the lock-step sequence driver, on warm-started video sequences (is_seq).

    python scripts/seq_stream_throughput.py [--sequences 64] [--mean-length 32] [--slots 16] [--reps 2] [--out FILE]

The same S sequences of unequal length (make_frames(smooth_walk=True), 8 views) are fitted three ways:
  (a) lockstep  seqio.fit_sequences on a context of B = S: one mvs_init_guess + mvs_fit_seq per time step over frame t of
                every sequence, the warm / cold decision on the host
  (b) stream_S  one context of B = S slots: the cold start points ctx.B frames at a time, then ONE mvs_fit_seq_stream call
  (c) stream_B  the same on a context of --slots slots
in two configurations: 'shipped' (VPoser latent pose with the shipped snapshot, L2 prior, SDF off: every stage frame-resident)
and 'bench' (bench.py's GMM schedule with the SDF term as written in stages 2-3, grid 128: dense rounds).  Each arm's wall time
covers the initial guesses and the fit, inputs on the host.  frame-iterations/s counts the iterations the results need (the
streams' per-frame sums; the lock-step also fits finished sequences' last frames again, which is not counted).  Arms alternate
over the repetitions; the fitted parameters of all arms must be byte-identical.  Also reported: how many frames after a
sequence's first started cold (their predecessor ended above reinit_loss = 5000)."""
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
    ap.add_argument("--mean-length", type=int, default=32)
    ap.add_argument("--slots", type=int, default=16)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--configs", default="shipped,bench")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from bench import stage_table
    from mvsmplfitting_b200 import seqio
    from mvsmplfitting_b200 import synthetic as S
    from mvsmplfitting_b200.context import FittingContext
    from tests import golden_util as G

    S_, T = args.sequences, args.mean_length
    rng = np.random.RandomState(77)
    lengths = [int(n) for n in rng.randint(T // 2, T + T // 2 + 1, size=S_)]
    model, gmm, cams = S.make_model(0), S.make_gmm(7), S.make_cameras(args.views)
    seqs = []
    for s_, n in enumerate(lengths):
        fr = S.make_frames(model, cams, n, seed=9000 + s_, smooth_walk=True)
        seqs.append(dict(gt_uv=fr["gt_uv"], conf=fr["conf"], present=np.ones(fr["conf"].shape[:2], bool),
                         frames=["%05d" % t for t in range(n)], serial="s%03d" % s_))
    gt_uv = np.concatenate([q["gt_uv"] for q in seqs], 1)
    conf = np.concatenate([q["conf"] for q in seqs], 1)
    jw = seqio.joint_weights("lsp14")
    guess = dict(estimate_scale=True, fixed_scale=1.0, use_torso=True, hip_seed=1.0, want_joints3d=False,
                 umeyama_as_written=False)
    vposer_w = G.snapshot_vposer_weights()

    def new_ctx(B, vposer):
        ctx = FittingContext(0)
        ctx.set_model(model)
        ctx.set_gmm_from_dict(gmm)
        ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
        ctx.set_batch(B)
        if vposer:
            ctx.set_vposer(vposer_w)
        return ctx

    info = card()
    out = {"workload": "%d sequences of %d..%d frames (%d frames) x %d views; %d slots for stream_B"
                       % (S_, min(lengths), max(lengths), sum(lengths), args.views, args.slots), **info, "configs": {}}
    for name in args.configs.split(","):
        vposer = name == "shipped"
        ctx_l, ctx_s, ctx_b = new_ctx(S_, vposer), new_ctx(S_, vposer), new_ctx(args.slots, vposer)
        if vposer:
            cfgs = [ctx_l.make_loss_config(body_prior="l2", use_vposer=2, **{k: v for k, v in st.items() if k != "coll_loss_weight"})
                    for st in stage_table()]
        else:
            cfgs = [ctx_l.make_loss_config(body_prior="gmm", interpenetration=True, sdf_grid=128, **st) for st in stage_table()]
        opt = ctx_l.make_lbfgs_config()

        def arm_lockstep():
            res, tot = seqio.fit_sequences(ctx_l, seqs, cfgs, opt, estimate_scale=True, pose_format="lsp14")
            return np.concatenate([r[0] for r in res]), dict(tot, dense_rounds=None)

        final_loss = {}

        def stream(ctx):
            x = seqio._cold_guesses(ctx, gt_uv, conf, jw, cfgs, guess)
            final, st = ctx.fit_seq_stream(x, gt_uv, conf, jw, lengths, cfgs, opt)
            final_loss["last"] = final.cpu().numpy()
            return x.cpu().numpy(), st

        arms = {"lockstep": arm_lockstep, "stream_S": lambda: stream(ctx_s), "stream_B": lambda: stream(ctx_b)}
        names = list(arms)
        for n in names:                                           # warm-up (allocations, first-use set-up)
            arms[n]()
        runs = {n: [] for n in names}
        for r in range(args.reps):
            order = names[r % 3:] + names[:r % 3]
            outs, sts = {}, {}
            for n in order:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                outs[n], sts[n] = arms[n]()
                torch.cuda.synchronize()
                runs[n].append({"seconds": time.perf_counter() - t0, "dense_rounds": sts[n]["dense_rounds"],
                                "rounds": sts[n]["rounds"]})
            it = sts["stream_B"]["frame_iterations"]
            assert sts["stream_S"]["frame_iterations"] == it
            for n in names:
                runs[n][-1]["frame_iterations_per_s"] = it / runs[n][-1]["seconds"]
            same = all(outs[n].tobytes() == outs["lockstep"].tobytes() for n in names)
            print("%s rep %d order %s: %s; params byte-identical: %s" % (name, r, ",".join(order), ", ".join(
                "%s %.2f s" % (n, runs[n][-1]["seconds"]) for n in names), same), file=sys.stderr)
            assert same, "the arms fitted different parameters"
        # frames after a sequence's first that start cold (predecessor's loss above 5000); where cold frames park, every
        # re-initialisation of a sequence costs the call one more pass of the runs before the chaining run
        reinit = [int((~(final_loss["last"][o:o + n - 1] <= np.float32(5000.0))).sum())
                  for o, n in zip(np.cumsum([0] + lengths[:-1]), lengths)]
        out["configs"][name] = {
            "reinitialised_frames": sum(reinit), "most_reinitialisations_in_one_sequence": max(reinit),
            "stages": "VPoser latent pose (shipped snapshot), L2 prior, SDF off" if vposer else
                      "GMM + angle + shape priors, SDF as written in stages 2-3 (grid 128)",
            "frame_iterations": it, "params_byte_identical": True,
            "median_seconds": {n: float(np.median([q["seconds"] for q in runs[n]])) for n in names},
            "median_frame_iterations_per_s": {n: float(np.median([q["frame_iterations_per_s"] for q in runs[n]])) for n in names},
            "runs": runs}
        for c in (ctx_l, ctx_s, ctx_b):
            c.close()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
