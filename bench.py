#!/usr/bin/env python
"""bench.py -- L-BFGS iterations/s of the multi-view SMPL fitting hot path.

    python bench.py --gpus N --steps K --warmup W            (our arm; torchrun for N > 1)
    python bench.py --impl reference --steps K --warmup W    (the UNMODIFIED reference on the host cores; --ref-device cuda: on torch-CUDA)

Workload (BASELINE.json configs[3], the config the metric is quoted on): per GPU 256 frames x 8
calibrated views of the synthetic SMPL-shaped model (6890 verts, 207 pose blend shapes), GMM(6) +
angle + shape priors, GMoF data term, the four-stage weight schedule of cfg_files/fit_smpl.yaml with
the SDF interpenetration term (reference semantics "as written") active in stages 2-3.
One STEP = one complete four-stage fit (4 x FittingMonitor.run_fitting, maxiters 30, L-BFGS max_iter
30 / strong Wolfe / history 100) of all frames from the same initial guess.

  value  = frame-iterations / s (iteration = one pass of lbfgs_ls.py:304-434 for one frame), device
           resident: keypoints + initial parameters already in HBM, reset by a device copy.  The K steps are
           shared out among --inflight lanes (context + stream + host thread each) that run concurrently:
           frames are independent problems, and the long tail of a batch (a few straggler frames) leaves
           most SMs idle, which the other batches fill.  single_batch = the K steps one after the other.
  e2e    = the same metric through mvs_fit_host: pinned HOST keypoints + parameters copied in, results
           copied out, every step.
Timed with CUDA events, max over ranks; L2 is flushed between steps (256 MiB write).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

METRIC = "lbfgs_frame_iterations_per_s"
UNIT = "frame-iterations/s"


def stage_table():
    from mvsmplfitting_b200 import synthetic as S
    sw = S.STAGE_WEIGHTS
    return [dict(data_weight=500.0 / 1536, body_pose_weight=sw["body_pose_prior_weights"][i],
                 shape_weight=sw["shape_weights"][i], bending_prior_weight=3.17 * sw["body_pose_prior_weights"][i],
                 coll_loss_weight=sw["coll_loss_weights"][i]) for i in range(4)]


def workload_config(frames, views, sdf):
    return {"workload": "cfg4: %d frames/GPU x %d views, 4-stage fit_smpl.yaml schedule, GMM(6)+angle+shape priors, "
                        "GMoF rho=100, SDF interpenetration %s" % (frames, views, "on in stages 2-3 (G=128, as-written "
                                                                   "semantics: kernel sees triangle 0)" if sdf else "off"),
            "frames_per_gpu": frames, "views": views, "model": "synthetic SMPL-shaped (6890 verts, 13776 faces)",
            "params_per_frame": 86, "l2": "flushed between steps (256 MiB write)",
            "step": "one full 4-stage fit of all frames from the same initial guess"}


# ----------------------------------------------------------------------------- clocks sampler
class ClockSampler:
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index=0):
        self.rows, self.proc, self.index = [], None, index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "200"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc:
            self.proc.terminate()
        sm = sorted(float(r[1]) for r in self.rows if len(r) > 8 and r[1].replace(".", "").isdigit())
        mx = [float(r[2]) for r in self.rows if len(r) > 8 and r[2].replace(".", "").isdigit()]
        reasons = set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            if len(r) > 8:
                for n, v in zip(names, r[5:9]):
                    if v.lower().startswith("active"):
                        reasons.add(n)
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


# ----------------------------------------------------------------------------- our arm
def run_ours(args):
    import torch
    import torch.distributed as dist
    from mvsmplfitting_b200 import synthetic as S
    from mvsmplfitting_b200.context import FittingContext

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if args.gpus != world and rank == 0 and world > 1:
        print("warning: --gpus %d but WORLD_SIZE %d" % (args.gpus, world), file=sys.stderr)
    torch.cuda.set_device(local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    dev = torch.device("cuda", local)

    B, V = args.frames, args.views
    model = S.make_model(0)
    gmm = S.make_gmm(7)
    cams = S.make_cameras(V)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)

    class Lane:
        """one batch in flight: its own context (workspace, optimiser state), frames, stream and pinned host buffers"""

        def __init__(self, i):
            self.fr = fr = S.make_frames(model, cams, B, seed=1000 + rank + 97 * i)
            self.ctx = ctx = FittingContext(local)
            ctx.set_model(model)
            ctx.set_gmm_from_dict(gmm)
            ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
            ctx.set_batch(B)
            if args.vposer:      # cfg 1 style: pose in VPoser's latent space, decoded on the device (use_vposer = 2), no SDF term
                ctx.set_vposer(S.make_vposer(11))
                self.stages = [ctx.make_loss_config(body_prior="l2", use_vposer=2, **{k: v for k, v in st.items() if k != "coll_loss_weight"})
                               for st in stage_table()]
            else:
                self.stages = [ctx.make_loss_config(body_prior="gmm", interpenetration=bool(args.sdf), sdf_grid=128,
                                                    sdf_all_faces=args.sdf_all_faces, **st) for st in stage_table()]
            self.opt = ctx.make_lbfgs_config()
            self.X0 = X0 = S.pack_params(fr["init"])
            if args.vposer:      # latent code (zeros = the decoder's mean pose) in the first 32 entries of the pose slot
                X0[:, 13:82] = 0.0
            self.x0_dev = torch.tensor(X0, device=dev)
            self.x = self.x0_dev.clone()
            ctx.set_keypoints(torch.tensor(fr["gt_uv"], device=dev), torch.tensor(fr["conf"], device=dev),
                              torch.tensor(fr["joint_weights"], device=dev))
            # pinned host buffers for the end-to-end leg
            self.X_pin = torch.from_numpy(X0.copy()).pin_memory()
            self.gt_pin, self.conf_pin = torch.from_numpy(fr["gt_uv"]).pin_memory(), torch.from_numpy(fr["conf"]).pin_memory()
            self.stream = torch.cuda.Stream(device=dev)

        def step_resident(self):
            # inputs already in HBM; mvs_fit runs the whole stage schedule (frames change stage on their own)
            self.x.copy_(self.x0_dev)
            self.loss, st = self.ctx.fit(self.x, self.stages, self.opt)
            return st

        def step_host(self):
            self.X_pin.copy_(torch.from_numpy(self.X0))
            return self.ctx.fit_host(self.X_pin.numpy(), self.gt_pin.numpy(), self.conf_pin.numpy(), self.fr["joint_weights"],
                                     self.stages, self.opt)[1]

    if args.vposer:
        args.sdf = 0
    n_lanes = max(1, args.inflight)
    lanes = [Lane(i) for i in range(n_lanes)]
    ctx, fr, X0 = lanes[0].ctx, lanes[0].fr, lanes[0].X0

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(kind, steps, warmup, profile_mask=0, use_lanes=None):
        """`steps` steps (one step = one batch through the whole fit) spread over the lanes, which run concurrently: every
        lane is a host thread driving its own context on its own stream.  One lane = batches strictly one after the other."""
        L = lanes[:use_lanes] if use_lanes else lanes
        share_of = lambda n: [n // len(L) + (1 if i < n % len(L) else 0) for i in range(len(L))]
        stats = [[] for _ in L]
        err = []
        for ln in L:
            ln.timed_steps = 0

        def work(i, n, record):
            try:
                torch.cuda.set_device(local)
                with torch.cuda.stream(L[i].stream):
                    for k in range(n):
                        flush.fill_(k & 0xFF)
                        st = getattr(L[i], kind)()
                        if record:
                            stats[i].append(st)
                            L[i].timed_steps += 1
                    L[i].stream.synchronize()
            except Exception as e:                                         # noqa: BLE001 -- re-raised below
                err.append(e)

        def run(counts, record):
            th = [threading.Thread(target=work, args=(i, n, record)) for i, n in enumerate(counts) if n > 0]
            for t in th:
                t.start()
            for t in th:
                t.join()
            if err:
                raise err[0]

        run([max(1, c) if warmup > 0 else 0 for c in share_of(warmup)], False)
        barrier()
        for ln in L:
            if profile_mask:
                ln.ctx.profile(profile_mask)
        l0 = sum(ln.ctx.launch_count() for ln in L)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        wall0 = time.time()
        e0.record()
        run(share_of(steps), True)
        torch.cuda.synchronize()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        barrier()
        wall = time.time() - wall0
        launches = sum(ln.ctx.launch_count() for ln in L) - l0
        prof = {}
        for ln in L:
            if profile_mask:
                for k, v in ln.ctx.profile_read().items():
                    a = prof.get(k, (0.0, 0))
                    prof[k] = (a[0] + v[0], a[1] + v[1])
                ln.ctx.profile(0)
        t = torch.tensor([ms], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t[0]), [s_ for lane_stats in stats for s_ in lane_stats], launches, prof, wall

    def step_resident():
        return lanes[0].step_resident()

    # one fully instrumented warm-up step decides which kernel dominates; that kernel alone is then
    # timed with events INSIDE the timed region (two event records per launch of one kernel)
    barrier()
    ctx.profile(0xFFFFFFFF)
    step_resident()
    share = ctx.profile_read()
    ctx.profile(0)
    dom = max(share, key=lambda k: share[k][0]) if share else "vertex_fwd"
    from mvsmplfitting_b200 import _lib as _L
    names = [ctx.lib.mvs_kernel_name(k).decode() for k in range(_L.NUM_KERNEL_IDS)]
    dom_mask = 1 << names.index(dom)

    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    # headline: `inflight` batches in flight (throughput of a stream of 256-frame batches); then the same workload with ONE
    # batch at a time (latency of a batch; the dominant kernel's roofline is taken here, undisturbed by concurrent lanes)
    ms_res, stats_res, launches, _, wall = timed("step_resident", args.steps, args.warmup)
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, lanes, rank)
    ms_e2e, stats_e2e, _, _, _ = timed("step_host", args.steps, max(1, min(args.warmup, n_lanes)))
    ms_one, stats_one, launches_one, prof, _ = timed("step_resident", args.steps, 1, dom_mask, use_lanes=1)
    ms_one_e2e, stats_one_e2e, _, _, _ = timed("step_host", args.steps, 1, use_lanes=1)
    clocks = sampler.stop() if rank == 0 else {}
    # auxiliary (not the headline): the same fit with the SDF term off = the reference's shipped default
    # (cfg_files/fit_smpl.yaml: interpenetration false) -> every stage runs frame-resident (regime A)
    aux = None
    if args.sdf:
        stages_main = lanes[0].stages
        lanes[0].stages = [ctx.make_loss_config(body_prior="gmm", interpenetration=False, **st) for st in stage_table()]
        ms_a, stats_a, launches_a, _, _ = timed("step_resident", 2, 1, use_lanes=1)
        it_a = sum(s_["frame_iterations"] for s_ in stats_a)
        aux = {"workload": "same frames, SDF term off (all four stages frame-resident), one batch at a time", "ms_per_step": ms_a / 2,
               "frame_iterations_per_s_per_gpu": it_a / (ms_a * 1e-3), "gpu_launches_per_step": launches_a / 2}
        lanes[0].stages = stages_main

    it = sum(s_["frame_iterations"] for s_ in stats_res)
    ev = sum(s_["frame_evals"] for s_ in stats_res)
    rounds = sum(s_["rounds"] for s_ in stats_res)
    it_e2e = sum(s_["frame_iterations"] for s_ in stats_e2e)
    it_one = sum(s_["frame_iterations"] for s_ in stats_one)
    it_one_e2e = sum(s_["frame_iterations"] for s_ in stats_one_e2e)
    cnt = torch.tensor([it, ev, launches, it_e2e, it_one, it_one_e2e], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(cnt, op=dist.ReduceOp.SUM)
    it_all, ev_all, launches_all, it_e2e_all, it_one_all, it_one_e2e_all = [float(v) for v in cnt]

    # ---- BASELINE configs[4]: the sequence as ONE jointly regularised problem (temporal smoothness), frames sharded over the
    #      ranks, per sweep a 344-byte halo exchange with each neighbour + ONE all-reduce (2 doubles) over NCCL.  Not the
    #      headline (the reference has no such term): reported under "cfg5" whenever more than one rank runs, or with --smooth.
    cfg5 = None
    if (world > 1 or args.smooth > 0) and not args.vposer:
        cfg5 = run_cfg5(args, model, gmm, cams, world, rank, local, dev)
    if rank == 0:
        peaks = {}
        try:
            peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        except Exception:
            pass
        hbm_peak = float(peaks.get("hbm_gbs", 3350.0))
        peak_src = "measured (MEASURED_PEAKS.json, sustained-copy figure)" if peaks else "H100 SXM data sheet: 3350 GB/s HBM3"
        # ---- roofline of the dominant kernel: algorithmic bytes per launch (DESIGN.md section 5) / event time
        dom_ms, dom_n = prof.get(dom, (0.0, 0))
        # average active frames per launch of the dense-round kernels (compaction shrinks launches towards the tail):
        # closure evaluations made by dense rounds / dense rounds, both counted by the library (mvs_lbfgs_stats), one-batch leg
        dense_ev = sum(s_["dense_frame_evals"] for s_ in stats_one)
        dense_rd = sum(s_["dense_rounds"] for s_ in stats_one)
        na_avg = (dense_ev / dense_rd) if dense_rd else (sum(s_["frame_evals"] for s_ in stats_one) / max(sum(s_["rounds"] for s_ in stats_one), 1))
        alg = algorithmic_bytes(dom, na_avg, V, dense=bool(args.sdf))
        ach = (alg * dom_n) / (dom_ms * 1e-3) / 1e9 if dom_ms > 0 else None
        roof = {"kernel": dom, "bound": "hbm", "achieved": ach, "peak": hbm_peak, "unit": "GB/s",
                "frac": (ach / hbm_peak) if ach else None,
                "algorithmic_bytes_per_launch": alg, "launches": dom_n, "avg_launch_us": (dom_ms * 1e3 / dom_n) if dom_n else None,
                "avg_active_frames_per_launch": na_avg, "peak_source": peak_src,
                "measured_in": "the one-batch-at-a-time timed leg (events around every launch of this kernel on its stream)",
                "note": "the path is latency / L2 bound, not HBM bound: constants (20 MB) live in the 50 MB L2 and one "
                        "launch moves a few MB; see DESIGN.md section 5",
                "kernel_time_share_of_step": {k: round(v[0] / max(sum(x_[0] for x_ in share.values()), 1e-9), 4)
                                              for k, v in share.items()},
                "kernel_avg_us_instrumented_step": {k: round(v[0] * 1e3 / max(v[1], 1), 2) for k, v in share.items()},
                "kernel_launches_instrumented_step": {k: int(v[1]) for k, v in share.items()}}
        # the tensor-core contraction, from the fully instrumented warm-up step (events around every launch)
        if "posedirs_gemm_tc" in share and share["posedirs_gemm_tc"][1] > 0:
            g_ms, g_n = share["posedirs_gemm_tc"]
            tf32_peak = float(peaks.get("bf16_tflops_sustained", 989.0)) / 2.0
            g_ach = gemm_flops(na_avg) * g_n / (g_ms * 1e-3) / 1e12
            roof["posedirs_gemm"] = {"bound": "tensor", "achieved": g_ach, "peak": tf32_peak, "unit": "TFLOP/s",
                                     "frac": g_ach / tf32_peak, "avg_launch_us": g_ms * 1e3 / g_n,
                                     "peak_source": "MEASURED_PEAKS.json bf16_tflops_sustained / 2 as the TF32 proxy" if peaks
                                                    else "H100 SXM data sheet: 989 TFLOP/s dense BF16 / 2 (495 TF32)",
                                     "note": "M = frames in flight (skinny GEMM): bound by streaming posedirs once per "
                                             "128-frame tile, not by tensor throughput"}
        cpu = {"note": "measured at N = 1 only"} if world > 1 else \
            cpu_baseline_sample(V, bool(args.sdf), max_seconds=args.cpu_seconds) if not args.vposer else \
            {"note": "CPU sample not run for the VPoser workload (oracle fit driver has no latent-space mode)"}
        sec = ms_res * 1e-3
        out = {
            "metric": METRIC, "value": it_all / sec, "unit": UNIT, "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms_res / args.steps, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": dict(workload_config(B, V, bool(args.sdf)),
                           **({"sdf_semantics": "ALL faces (intended field), %s" % ("candidate lists (mvs_sdf_bins.cuh)" if args.sdf_all_faces == 1
                                                                                  else "brute force")} if args.sdf_all_faces else {}),
                           parallelism="frames sharded, dp%d, no data-path collective" % world,
                           inflight=n_lanes,
                           pipelining="%d batches of %d frames in flight per GPU: one libmvsmpl context + CUDA stream + host thread "
                                      "each, the K steps are shared out among them; single_batch = the same K steps strictly one "
                                      "after the other" % (n_lanes, B),
                           **({"pose": "VPoser latent code (32-D), decoded on the device (use_vposer = 2), l2 prior |z|^2"} if args.vposer else {})),
            "frame_closure_evals_per_s": ev_all / sec, "evals_per_iteration": ev_all / max(it_all, 1),
            "iterations_per_frame_per_step": it_all / (B * world * args.steps),
            "rounds_per_step": rounds / args.steps,
            "e2e": {"value": it_e2e_all / (ms_e2e * 1e-3), "unit": UNIT,
                    "h2d_bytes_per_step": int(fr["gt_uv"].nbytes + fr["conf"].nbytes + fr["joint_weights"].nbytes + X0.nbytes),
                    "d2h_bytes_per_step": int(X0.nbytes + B * 4), "ms_per_step": ms_e2e / args.steps,
                    "api": "mvs_fit_host (C ABI, host buffers)"},
            "single_batch": {"value": it_one_all / (ms_one * 1e-3), "unit": UNIT, "ms_per_step": ms_one / args.steps,
                             "rounds_per_step": sum(s_["rounds"] for s_ in stats_one) / args.steps,
                             "gpu_launches_per_step": launches_one / args.steps,
                             "e2e": {"value": it_one_e2e_all / (ms_one_e2e * 1e-3), "ms_per_step": ms_one_e2e / args.steps}},
            "gpu_launches": int(launches_all), "roofline": roof, "cpu_baseline": cpu, "clocks": clocks,
            "wall_s_timed_region": wall, "aux_no_sdf": aux, "cfg5": cfg5,
        }
        print(json.dumps(out))
    for ln in lanes:
        ln.ctx.close()
    if world > 1:
        dist.destroy_process_group()


def dump_outputs(out_dir, lanes, rank):
    """What the headline path (mvs_fit) hands its caller after the last timed step of every lane that ran one: the fitted
    parameters [B][86] and final losses [B], float32.  A lane's inputs depend only on its seed (1000 + rank + 97 lane), so
    two builds run with the same arguments can be compared output for output."""
    import torch
    torch.cuda.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    for i, ln in enumerate(lanes):
        if ln.timed_steps == 0:
            continue
        tag = "rank%d_lane%d" % (rank, i)
        np.save(os.path.join(out_dir, "params_%s.npy" % tag), ln.x.detach().cpu().numpy().astype(np.float32))
        np.save(os.path.join(out_dir, "loss_%s.npy" % tag), ln.loss.detach().cpu().numpy().astype(np.float32))


def run_cfg5(args, model, gmm, cams, world, rank, local, dev):
    """jointly regularised sequence (SequenceFitter): world x --seq-frames frames, block-Jacobi sweeps; returns the rank-0
    summary (device time max over ranks; the collective's own time from CUDA events around halo exchange + all-reduce)"""
    import torch
    import torch.distributed as dist
    from mvsmplfitting_b200 import synthetic as S
    from mvsmplfitting_b200.sequence import SequenceFitter, shard_bounds
    lam = args.smooth if args.smooth > 0 else 50.0
    Bs = args.seq_frames
    T = Bs * world
    fitter = SequenceFitter(model, cams, T, gmm=gmm, device=local)
    a, b = shard_bounds(T, world, rank)
    seq = S.make_frames(model, cams, T, seed=77, smooth_walk=True)       # smooth random walk of poses, the same on every rank
    sl = slice(a, b)
    x0 = torch.tensor(S.pack_params({k: v[sl] for k, v in seq["init"].items()}), device=dev)
    gt, cf = torch.tensor(seq["gt_uv"][:, sl].copy(), device=dev), torch.tensor(seq["conf"][:, sl].copy(), device=dev)
    jw = torch.tensor(seq["joint_weights"], device=dev)
    stages = [fitter.ctx.make_loss_config(body_prior="gmm", **{k: v for k, v in st.items() if k != "coll_loss_weight"}) for st in stage_table()]
    res = None
    for rep in range(2):                                    # first pass = warm-up
        x = x0.clone()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        res = fitter.fit(x, gt, cf, jw, stages, smooth_weight=lam, sweeps=args.sweeps, time_comm=True)
        e1.record()
        torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
        cnt = torch.tensor([float(sum(r["frame_iterations"] for r in res))], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            dist.all_reduce(cnt, op=dist.ReduceOp.SUM)
    fitter.ctx.close()
    return {"workload": "cfg5: %d frames x %d views as one sequence, %d per rank, temporal smoothness lambda=%g on pose / orientation / "
                        "translation, %d block-Jacobi sweeps (4-stage fit, then last-stage re-fits), GMM+angle+shape priors, SDF off"
                        % (T, args.views, Bs, lam, args.sweeps),
            "collective": "per sweep: 2 x 344 B point-to-point halo (NCCL send/recv) + ONE all-reduce of 2 doubles (NCCL)" if world > 1
                          else "none (one rank)",
            "ms_total": float(t[0]), "frame_iterations_per_s": float(cnt[0]) / (float(t[0]) * 1e-3),
            "comm_ms_per_sweep": [round(r.get("comm_ms", 0.0), 4) for r in res],
            "joint_energy_per_sweep": [r.get("joint_energy") for r in res],
            "smooth_energy_per_sweep": [r.get("smooth_energy") for r in res]}


def algorithmic_bytes(kernel: str, na: float, V: int, dense: bool) -> float:
    """Algorithmic (must-move) bytes of ONE launch of `kernel` with `na` active frames; derivation in
    DESIGN.md section 5 (per-frame figures from SURVEY.md 8d: constants 19.7 MB shared, 82 680 B / frame of
    vertices, 344 B parameters, 204 B / view keypoints)."""
    N = 6890
    nv = N if dense else 86
    q_bytes = 3 * nv * 218 * 4                      # posedirs + shapedirs + template rows of the vertex list
    w_bytes = nv * 4 * 8                            # skinning weights (4 (joint, weight) pairs)
    if kernel == "vertex_fwd":
        return q_bytes + w_bytes + na * (218 * 4 + 288 * 4 + 2 * nv * 12)
    if kernel == "posedirs_gemm_tc":                # posedirs (hi + lo parts of the 3xTF32 split) once, pose features (hi + lo) in,
        return 2 * 3 * N * 207 * 4 + na * (2 * 207 * 4 + 3 * N * 4)     # pose offsets out
    if kernel == "skin":                            # offsets in, template/shapedirs/weights once, v_posed + verts out
        return N * 33 * 4 + N * 32 + na * (3 * N * 4 + 288 * 4 + 40 + 2 * N * 12)
    if kernel == "vertex_bwd":
        return 3 * N * 218 * 4 + N * 24 * 4 + na * (1152 + 2 * N * 12 + 2048)
    if kernel in ("sdf_sample", "sdf_finalize"):
        return na * (N * 12 + N * 12)
    if kernel == "sdf_fused":                       # vertices + chunk boxes in, per-block sums / flags out (adjoint partials are rare)
        return na * (N * 12 + 108 * 48 + 27 * 24)
    if kernel == "frame_step":
        # once: the 86-vertex slice of Qk (adjoint) and the GMM precisions; per frame: 9 optimiser vectors, detections,
        # support vertices, SDF block sums, and the curvature history the two-loop recursion reads (about 50 of the
        # 100 pairs are live on average, 2 x 344 B each, on the ~40 % of the calls that start an iteration)
        return 3 * 86 * 224 * 4 + 6 * 69 * 69 * 4 + na * (344 * 9 + 204 * V + 86 * 24 + 27 * 24 + 0.4 * 2 * 50 * 344)
    if kernel in ("frame_fwd", "frame_bwd", "keypoint_loss", "lbfgs_advance"):
        return na * (344 * 3 + 204 * V + 2048 + 86 * 24)
    if kernel == "lbfgs_resident":                  # per frame and evaluation: two passes over its 86-vertex Qk slice
        return na * (2 * 3 * 86 * 218 * 4 + 344 * 3 + 204 * V)
    return na * 344


def gemm_flops(na: float) -> float:
    """algorithmic flops of one posedirs contraction launch: [na x 207] x [207 x 20670]"""
    return 2.0 * na * 207 * 20670


# ----------------------------------------------------------------------------- the reference arm
# The reference itself (staged unmodified under oracle/_ref/reference by oracle/stage_reference.py, or /root/reference in the
# authoring container), driven through its own utils/non_linear_solver.non_linear_solver by oracle/ref_fit.py.
_REF_CACHE = {}


def _ref_scene(V, device):
    key = (V, device)
    if key not in _REF_CACHE:
        import torch
        if device == "cpu":
            torch.set_num_threads(1)
        from mvsmplfitting_b200 import synthetic as S
        from oracle import ref_fit as RF
        model, gmm, cams = S.make_model(0), S.make_gmm(7), S.make_cameras(V)
        _REF_CACHE[key] = (model, cams, RF.build_scene(model, gmm, cams, device=device))
    return _REF_CACHE[key]


def _ref_fit_one(args):
    """complete 4-stage fit of ONE frame by the unmodified reference; returns (iterations, closure evals, seconds)"""
    seed, V, sdf, device = args
    import warnings
    warnings.filterwarnings("ignore")
    from mvsmplfitting_b200 import synthetic as S
    from oracle import ref_fit as RF
    model, cams, sc = _ref_scene(V, device)
    fr = S.make_frames(model, cams, 1, seed=seed)
    t0 = time.time()
    r = RF.fit_frame(sc, fr, 0, S.STAGE_WEIGHTS, interpenetration=bool(sdf))
    return r["iterations"], r["evals"], time.time() - t0


def _ref_warm(args):
    V, device, do_fit = args
    import warnings
    warnings.filterwarnings("ignore")
    _ref_scene(V, device)
    dt = _ref_fit_one((999, V, 0, device))[2] if do_fit else 0.0
    time.sleep(0.5)          # keep this worker busy until every other worker has taken its own warm-up task
    return dt


def cpu_baseline_sample(V, sdf, max_seconds=30.0):
    """bounded sample on one host core: complete 4-stage fits of 2 frames by the unmodified reference, SDF term off (the
    reference's SDF term is a CUDA kernel: it has no CPU path), about 10-30 s of CPU work"""
    import warnings
    warnings.filterwarnings("ignore")
    try:
        from oracle import ref_harness as RH
        if not RH.available():
            return {"error": "reference tree not staged (python -m oracle.stage_reference)"}
        it = ev = 0
        t0 = time.time()
        n = 0
        for seed in (1000, 1001):
            r = _ref_fit_one((seed, V, 0, "cpu"))
            it += r[0]; ev += r[1]; n += 1
            if time.time() - t0 > max_seconds:
                break
        dt = time.time() - t0
    except Exception as e:  # the GPU arm must not die because the checker could not run
        return {"error": repr(e)}
    return {"value": it / dt, "unit": UNIT, "cores": 1, "kind": "reference",
            "sample": "%d frame(s) x %d views, complete 4-stage fits by the UNMODIFIED reference (utils/non_linear_solver.py driving "
                      "fitting.py / lbfgs_ls.py, torch CPU, 1 thread), SDF term off (CUDA-only in the reference); %d iterations, "
                      "%d closure evals in %.1f s" % (n, V, it, ev, dt),
            "frame_closure_evals_per_s": ev / dt}


def run_ref_worker(args):
    """one worker of the reference arm (see run_reference): READY <seconds of the warm-up fit>, then per GO line the fits"""
    import warnings
    warnings.filterwarnings("ignore")
    V, device = args.views, args.ref_device
    _ref_scene(V, device)
    dt = _ref_fit_one((999, V, 0, device))[2] if args.warmup > 0 else 0.0
    print("READY %.6f" % dt, flush=True)
    for line in sys.stdin:
        parts = line.split()
        if len(parts) != 3 or parts[0] != "GO":
            continue
        sdf = int(parts[1])
        out = [_ref_fit_one((int(q), V, sdf, device)) for q in parts[2].split(",")]
        print("DONE " + json.dumps(out), flush=True)


def run_reference(args):
    """--impl reference: the reference's own implementation of the path (code/utils/non_linear_solver.py -> fitting.py,
    lbfgs_ls.py, smplx/, camera.py, prior.py, unmodified) on the box's host cores, one process per physical core, one
    thread each (the reference is batch-1: frames are its only parallelism).  --ref-device cuda runs the same code on
    torch-CUDA (its shipped mode, cfg_files/fit_smpl.yaml:19) with its own SDF kernel: the secondary arm."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    import warnings
    warnings.filterwarnings("ignore")
    from oracle import ref_harness as RH
    if not RH.available():
        print(json.dumps({"impl": "reference", "unavailable": "reference tree not staged under oracle/_ref/reference "
                                                              "(python -m oracle.stage_reference in the authoring container)"}))
        return
    V = args.views
    on_cuda = args.ref_device == "cuda"
    for k in ("OMP_NUM_THREADS", "MKL_NUM_THREADS", "OPENBLAS_NUM_THREADS"):      # one thread per worker process, from their start
        os.environ[k] = "1" if not on_cuda else os.environ.get(k, "8")
    # the reference's SDF term is a CUDA kernel (sdf/sdf/csrc): on the CPU arm the term is off, on the CUDA arm it follows --sdf
    sdf = bool(args.sdf) and on_cuda
    cores = 1 if on_cuda else max(1, min((os.cpu_count() or 2) // 2, args.ref_workers))
    # One plain subprocess per worker (python bench.py --ref-worker): it imports torch + the reference, builds the scene, runs one
    # complete warm-up fit (W >= 1; its duration sizes the timed sample -- a fit is ~10 s, W fits per worker would not fit the
    # time budget), reports READY and waits for its list of frames on stdin.  Results come back as one JSON line per worker.
    env = dict(os.environ)
    cmd = [sys.executable, os.path.abspath(__file__), "--ref-worker", "--views", str(V), "--ref-device", args.ref_device,
           "--warmup", str(args.warmup)]
    procs = [subprocess.Popen(cmd, stdin=subprocess.PIPE, stdout=subprocess.PIPE, env=env, text=True)
             for _ in range(cores)]

    def read_tagged(p, tag):
        while True:
            line = p.stdout.readline()
            if not line:
                raise RuntimeError("reference worker exited early (rc %s)" % p.poll())
            if line.startswith(tag):
                return line[len(tag):].strip()

    try:
        t_fit = [float(read_tagged(p, "READY")) for p in procs]
        t_f = max(1e-3, float(np.mean(t_fit))) if args.warmup > 0 else 12.0
        # bounded sample: every worker gets the same number of complete frame fits, sized so that the run fills about
        # --ref-seconds; every fit runs to completion (no wall-time cut), there is no barrier between steps
        per_worker = int(max(1, min(np.ceil(args.frames * args.steps / cores), np.floor(args.ref_seconds / t_f))))
        F = per_worker * cores / max(1, args.steps)
        t0 = time.time()
        for w, p in enumerate(procs):
            seeds = [7000 + w * per_worker + i for i in range(per_worker)]
            p.stdin.write("GO %d %s\n" % (int(sdf), ",".join(str(q) for q in seeds)))
            p.stdin.flush()
        res = []
        for p in procs:
            res += [tuple(r) for r in json.loads(read_tagged(p, "DONE"))]
        dt = time.time() - t0
    finally:
        for p in procs:
            try:
                p.stdin.close()
            except Exception:                                   # noqa: BLE001
                pass
        for p in procs:
            try:
                p.wait(timeout=30)
            except Exception:                                   # noqa: BLE001
                p.kill()
    it, ev = sum(r[0] for r in res), sum(r[1] for r in res)
    val = it / dt
    cfg = dict(workload_config(args.frames, V, sdf),
               parallelism=("1 process, torch-CUDA (cuda:0)" if on_cuda else "%d host processes x 1 thread" % cores),
               reference_arm="UNMODIFIED reference (oracle/_ref/reference: utils/non_linear_solver.py, fitting.py, lbfgs_ls.py, smplx/, "
                             "camera.py, prior.py) on %s; %s; each step = %.4g complete frame fits (bounded sample of the %d-frame "
                             "workload: every worker runs the same number of fits to completion, no wall-time cut)" % (
                                 "torch-CUDA with its own SDF kernel (sdf_cuda_kernel.cu compiled unchanged)" if on_cuda else "torch CPU",
                                 "SDF term as configured" if on_cuda else "SDF term OFF: it is a CUDA-only kernel in the reference, "
                                 "this is the only mode the reference can run on host cores (compare with aux_no_sdf of the GPU arm)",
                                 F, args.frames))
    out = {"impl": "reference", "metric": METRIC, "value": val, "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps,
           "warmup": args.warmup, "ms_per_step": dt * 1e3 / args.steps, "higher_is_better": True, "scaling": "weak",
           "vs_baseline": None, "dtype": "f32", "data": "synthetic", "config": cfg,
           "cpu_baseline": {"value": val, "unit": UNIT, "cores": cores, "kind": "reference",
                            "sample": "%d steps x %.4g complete 4-stage frame fits x %d views by the unmodified reference, %s; "
                                      "mean fit %.1f s; %d iterations, %d closure evals in %.1f s" % (
                                          args.steps, F, V, cfg["parallelism"], float(np.mean([r[2] for r in res])), it, ev, dt)},
           "e2e": {"value": val, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
           "frame_closure_evals_per_s": ev / dt, "evals_per_iteration": ev / max(it, 1),
           "iterations_per_frame": it / max(len(res), 1), "gpu_launches": 0}
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--frames", type=int, default=256, help="frames per GPU")
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--sdf", type=int, default=1)
    ap.add_argument("--sdf-all-faces", type=int, default=0, help="0: the reference call as written (triangle 0; the benchmark), 1: the "
                    "intended all-faces field over candidate lists (SURVEY N3), 2: the same by brute force")
    ap.add_argument("--inflight", type=int, default=8, help="batches in flight per GPU (contexts + streams + host threads); 1 = serial")
    ap.add_argument("--vposer", type=int, default=0, help="1: fit VPoser's 32-D latent code (decoded on the device), no SDF")
    ap.add_argument("--smooth", type=float, default=0.0, help="cfg5: temporal-smoothness weight (> 0 runs the cfg5 leg on one rank too)")
    ap.add_argument("--sweeps", type=int, default=6, help="cfg5: block-Jacobi sweeps")
    ap.add_argument("--seq-frames", type=int, default=128, help="cfg5: frames per rank (1024 / 8)")
    ap.add_argument("--cpu-seconds", type=float, default=30.0)
    ap.add_argument("--ref-workers", type=int, default=32, help="host processes of the reference arm (capped at half the logical "
                    "cores)")
    ap.add_argument("--ref-seconds", type=float, default=200.0, help="target wall time of the --impl reference run (sizes the sample)")
    ap.add_argument("--ref-device", default="cpu", choices=["cpu", "cuda"], help="reference arm: host cores (default) or torch-CUDA")
    ap.add_argument("--ref-worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write each lane's final parameters and losses of its last timed step as DIR/*.npy")
    args = ap.parse_args()
    if args.ref_worker:
        run_ref_worker(args)
    elif args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
