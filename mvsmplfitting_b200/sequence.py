"""Sequences of frames across GPUs (SURVEY section 8e).

Frames are independent fitting problems in the reference (code/main.py:32 processes them one by one;
`is_seq` only warm-starts), so the path shards with NO data-path collective: rank r of W owns a
contiguous block of frames and a private libmvsmpl context.

Jointly regularised mode (BASELINE configs[4]; NOT in the reference -> parity unpinned, checked against
the autograd restatement in oracle/smooth_oracle.py): the temporal smoothness energy

    E_s = lam * sum_t  || (x_t - x_{t-1}) * mask ||^2          (mask selects pose / translation entries)

is minimised by block-Jacobi sweeps: within a sweep every frame sees its two neighbours frozen, which
turns E_s into a per-frame quadratic anchor  2 lam || x_t - mean(neighbours) ||^2 (+ const) that the
closure kernels evaluate (mvs_set_anchor), so frames stay independent inside a sweep.  Between sweeps
ranks exchange ONE boundary frame with each neighbour (344 B halo) and all-reduce two scalars in ONE call (the global
smoothness energy and the sum of the frames' own losses = the joint objective) -- the only collective on the path, as the
north-star asks.  Block-Jacobi is a fixed-point iteration of the joint problem's stationarity conditions; its convergence on
a 64-frame chain is measured by scripts/cfg5_convergence.py.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist

from . import synthetic as S


def shard_bounds(num_frames: int, world: int, rank: int):
    """contiguous, balanced blocks: the first (T mod W) ranks get one extra frame"""
    base, rem = divmod(num_frames, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def smooth_mask(pose=True, transl=True, orient=True) -> torch.Tensor:
    m = torch.zeros(S.NUM_PARAMS)
    if orient:
        m[10:13] = 1.0
    if pose:
        m[13:82] = 1.0
    if transl:
        m[82:85] = 1.0
    return m


def exchange_halo(x_local: torch.Tensor, group=None):
    """Send my first / last frame to the previous / next rank.  Returns (left, right): the last frame of the
    previous rank and the first frame of the next rank ([86] tensors on x_local's device) or None at the
    sequence ends.  Point-to-point only (2 x 344 B per rank)."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return None, None
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    left = torch.empty_like(x_local[0]) if rank > 0 else None
    right = torch.empty_like(x_local[0]) if rank < world - 1 else None
    ops = []
    first, last = x_local[0].contiguous(), x_local[-1].contiguous()
    if rank > 0:
        ops += [dist.P2POp(dist.isend, first, rank - 1, group), dist.P2POp(dist.irecv, left, rank - 1, group)]
    if rank < world - 1:
        ops += [dist.P2POp(dist.isend, last, rank + 1, group), dist.P2POp(dist.irecv, right, rank + 1, group)]
    for req in dist.batch_isend_irecv(ops):
        req.wait()
    return left, right


def neighbour_anchor(x_local: torch.Tensor, left, right, lam: float, mask: torch.Tensor):
    """(anchor [B,86], weight_per_frame [B]) of the block-Jacobi sweep: anchor_t = mean of the existing
    neighbours, energy lam * n_t * ||x_t - anchor_t||^2 with n_t in {1,2} neighbours (0 for a 1-frame sequence)."""
    B = x_local.shape[0]
    prev = torch.cat([left[None] if left is not None else x_local[:1], x_local[:-1]], dim=0)
    nxt = torch.cat([x_local[1:], right[None] if right is not None else x_local[-1:]], dim=0)
    has_prev = torch.ones(B, device=x_local.device)
    has_next = torch.ones(B, device=x_local.device)
    if left is None:
        has_prev[0] = 0
    if right is None:
        has_next[-1] = 0
    n = has_prev + has_next
    anchor = (prev * has_prev[:, None] + nxt * has_next[:, None]) / n.clamp(min=1)[:, None]
    return anchor, lam * n


def smoothness_energy(x_local: torch.Tensor, left, lam: float, mask: torch.Tensor, group=None) -> torch.Tensor:
    """global E_s = lam * sum_t ||(x_t - x_{t-1}) mask||^2 : local differences + the one across my left
    boundary, then ONE scalar all-reduce."""
    m = mask.to(x_local.device)
    e = ((x_local[1:] - x_local[:-1]) * m).pow(2).sum()
    if left is not None:
        e = e + ((x_local[0] - left) * m).pow(2).sum()
    e = lam * e.reshape(1).to(torch.float64)
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(e, op=dist.ReduceOp.SUM, group=group)
    return e[0]


class SequenceFitter:
    """Fits this rank's block of a T-frame sequence; see the module docstring for the jointly regularised mode."""

    def __init__(self, model: dict, cams: dict, num_frames: int, gmm: dict | None = None, device: int | None = None,
                 group=None, model_type: str = "smpllsp"):
        from .context import FittingContext
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.T = num_frames
        self.start, self.stop = shard_bounds(num_frames, self.world, self.rank)
        dev = device if device is not None else (torch.cuda.current_device() if torch.cuda.is_available() else 0)
        self.ctx = FittingContext(dev)
        self.ctx.set_model(model, model_type=model_type)
        if gmm is not None:
            self.ctx.set_gmm_from_dict(gmm)
        self.ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"], dist=cams.get("dist"))   # lens distortion, if any
        self.ctx.set_batch(self.stop - self.start)
        self.B = self.stop - self.start

    def fit(self, x0_local: torch.Tensor, gt_uv_local, conf_local, joint_weights, stage_cfgs, opt_cfg=None,
            smooth_weight: float = 0.0, sweeps: int = 1, mask: torch.Tensor | None = None, time_comm: bool = False):
        """x0_local [B,86] (CUDA, updated in place); detections of this rank's frames.  Returns per-sweep stats;
        with smooth_weight > 0 also the global smoothness energy after every sweep."""
        ctx = self.ctx
        ctx.set_keypoints(gt_uv_local, conf_local, joint_weights)
        mask = smooth_mask() if mask is None else mask
        out = []
        x = x0_local
        for sweep in range(max(1, sweeps)):
            left = right = None
            if smooth_weight > 0:
                left, right = exchange_halo(x, self.group)
                anchor, wf = neighbour_anchor(x, left, right, smooth_weight, mask)
                # lam*||x-p||^2 + lam*||x-n||^2 = (lam * n_t) * ||x - mean||^2 + const, n_t = existing neighbours
                ctx.set_anchor(anchor, wf[:, None] * mask.to(x.device)[None, :])
            else:
                ctx.set_anchor(None)
            tot = dict(frame_iterations=0, frame_evals=0, rounds=0, frames_nan=0)
            stages = stage_cfgs if sweep == 0 else stage_cfgs[-1:]
            for cfg in stages:
                ctx.set_loss(config=cfg)
                _, st = ctx.lbfgs_run(x, opt_cfg)
                for k in tot:
                    tot[k] += st[k]
            if smooth_weight > 0:
                # joint objective after this sweep: sum of the frames' own losses (anchor off, last stage's weights) + E_s.
                # ONE all-reduce of two doubles; its device time is reported per sweep (comm_ms).
                ctx.set_anchor(None)
                ctx.set_loss(config=stage_cfgs[-1])
                own = ctx.closure(x, want_grad=False)["loss"].double().sum()
                ev = None
                if time_comm and torch.cuda.is_available():
                    ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                    ev[0].record()
                left, _ = exchange_halo(x, self.group)
                m = mask.to(x.device)
                e = ((x[1:] - x[:-1]) * m).pow(2).sum()
                if left is not None:
                    e = e + ((x[0] - left) * m).pow(2).sum()
                red = torch.stack([smooth_weight * e.double(), own])
                if dist.is_initialized() and self.world > 1:
                    dist.all_reduce(red, op=dist.ReduceOp.SUM, group=self.group)
                if ev:
                    ev[1].record()
                    torch.cuda.synchronize()
                    tot["comm_ms"] = ev[0].elapsed_time(ev[1])
                tot["smooth_energy"] = float(red[0])
                tot["fit_energy"] = float(red[1])
                tot["joint_energy"] = float(red[0] + red[1])
            out.append(tot)
        ctx.set_anchor(None)
        return out
