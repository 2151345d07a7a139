"""GPU: complete 4-stage fits (mvs_fit) against complete fits by the UNMODIFIED reference.

* SDF off: tests/golden/fit_e2e_ref.npz (oracle/make_golden_fit.py: the reference's own non_linear_solver on 16 frames,
  torch CPU).  The benchmark metric counts L-BFGS iterations, so the counts themselves are pinned here.
* SDF on: tests/golden/fit_e2e_sdf_ref.npz (oracle/make_golden_refruns.py: the same solver on torch-CUDA with the
  reference's own SDF kernel, the only place it can run, on 16 frames).

L-BFGS with ftol = 1e-9 on an fp32 loss is chaotic in the last bits: closures that agree to 1e-7 stop after different
iteration counts (the reference against its own fp64 run does too).  So single trajectories are not comparable; what is
pinned is the distribution: mean iterations / evaluations per frame, and the final losses frame by frame.
"""
import json
import os

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from tests import golden_util as G

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def stage_cfgs(ctx, sdf):
    sw = S.STAGE_WEIGHTS
    return [ctx.make_loss_config(body_prior="gmm", interpenetration=sdf, sdf_grid=128, data_weight=500.0 / 1536,
                                 body_pose_weight=sw["body_pose_prior_weights"][i], shape_weight=sw["shape_weights"][i],
                                 bending_prior_weight=3.17 * sw["body_pose_prior_weights"][i],
                                 coll_loss_weight=sw["coll_loss_weights"][i]) for i in range(4)]


def device_fit(model, gmm, cams, fr, X0, sdf):
    from mvsmplfitting_b200.context import FittingContext
    B = X0.shape[0]
    ctx = FittingContext(0)
    ctx.set_model(model)
    ctx.set_gmm_from_dict(gmm)
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"])
    ctx.set_batch(B)
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    x = torch.tensor(X0, device="cuda")
    final, st = ctx.fit(x, stage_cfgs(ctx, sdf))
    torch.cuda.synchronize()
    out = final.cpu().numpy(), x.cpu().numpy(), st
    ctx.close()
    return out


def _record(name, rec):
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "fit_e2e_%s.json" % name), "w") as f:
        json.dump(rec, f, indent=1)


def test_four_stage_fit_matches_reference_fixture(syn_model, syn_gmm):
    z = np.load(os.path.join(G.GOLD, "fit_e2e_ref.npz"))
    B, V = int(z["B"]), int(z["V"])
    cams = S.make_cameras(V)
    fr = S.make_frames(syn_model, cams, B, seed=int(z["seed"]))
    X0 = S.pack_params(fr["init"])
    assert np.array_equal(X0, z["X0"]), "synthetic frame generator changed: regenerate the fixture"
    final, x, st = device_fit(syn_model, syn_gmm, cams, fr, X0, sdf=False)
    ref_it, ref_ev = z["iterations"].sum(1).mean(), z["evals"].sum(1).mean()
    it, ev = st["frame_iterations"] / B, st["frame_evals"] / B
    rel_final = np.abs(final - z["final_loss"]) / z["final_loss"]
    rec = dict(frames=B, iterations_per_frame=dict(device=it, reference=float(ref_it)),
               evals_per_frame=dict(device=ev, reference=float(ref_ev)), final_loss_device=final.tolist(),
               final_loss_reference=z["final_loss"].tolist(), rel_final=rel_final.tolist())
    _record("nosdf", rec)
    print(json.dumps({k: rec[k] for k in ("iterations_per_frame", "evals_per_frame")}), "final-loss rel: median %.3g max %.3g" % (
        np.median(rel_final), rel_final.max()))
    assert abs(it - ref_it) / ref_it < 0.10, (it, ref_it)
    assert abs(ev - ref_ev) / ref_ev < 0.10, (ev, ref_ev)
    assert np.median(rel_final) < 0.02 and rel_final.max() < 0.10
    assert abs(final.mean() - z["final_loss"].mean()) / z["final_loss"].mean() < 0.01


def test_four_stage_fit_with_sdf_matches_live_reference_run(syn_model, syn_gmm):
    z = np.load(os.path.join(G.GOLD, "fit_e2e_sdf_ref.npz"))
    B, V = int(z["B"]), int(z["V"])
    cams = S.make_cameras(V)
    fr = S.make_frames(syn_model, cams, B, seed=int(z["seed"]))
    X0 = S.pack_params(fr["init"])
    assert np.array_equal(X0, z["X0"]), "synthetic frame generator changed: regenerate the fixture"
    runs = [dict(iterations=int(z["iterations"][b]), evals=int(z["evals"][b]), final_loss=float(z["final_loss"][b]),
                 params=z["params"][b], per_stage=z["per_stage"][b].tolist()) for b in range(B)]
    ref_it = np.mean([r["iterations"] for r in runs]); ref_ev = np.mean([r["evals"] for r in runs])
    ref_final = np.array([r["final_loss"] for r in runs])
    final, x, st = device_fit(syn_model, syn_gmm, cams, fr, X0, sdf=True)
    # deterministic part: the two implementations agree on the OBJECTIVE where the reference ended (its reported loss is the
    # one at the entry of its last optimiser step, i.e. at its final parameters up to the last, tiny, step)
    from mvsmplfitting_b200.context import FittingContext
    ctx = FittingContext(0)
    ctx.set_model(syn_model); ctx.set_gmm_from_dict(syn_gmm); ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"]); ctx.set_batch(B)
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    ctx.set_loss(config=stage_cfgs(ctx, True)[3])
    at_ref = ctx.closure(torch.tensor(np.stack([r["params"] for r in runs]), device="cuda"), want_grad=False)["loss"].cpu().numpy()
    ctx.close()
    # (a frame whose last step still moved a lot -- e.g. out of a penetration -- ends BELOW its reported loss, never above)
    rel_at = (at_ref - ref_final) / ref_final
    assert (rel_at < 1e-3).all() and (np.abs(rel_at) < 1e-3).mean() >= 0.8, (at_ref, ref_final)
    it, ev = st["frame_iterations"] / B, st["frame_evals"] / B
    rel_final = np.abs(final - ref_final) / ref_final
    rec = dict(frames=B, iterations_per_frame=dict(device=it, reference=float(ref_it)),
               evals_per_frame=dict(device=ev, reference=float(ref_ev)), per_stage_reference=[r["per_stage"] for r in runs],
               final_loss_device=final.tolist(), final_loss_reference=ref_final.tolist(), rel_final=rel_final.tolist())
    _record("sdf", rec)
    print(json.dumps({k: rec[k] for k in ("iterations_per_frame", "evals_per_frame")}), "final-loss rel: median %.3g max %.3g" % (
        np.median(rel_final), rel_final.max()))
    # 16 frames: the means carry the sampling noise of a chaotic stopping rule (see the module docstring).  With the SDF term
    # the objective is also DISCONTINUOUS (phi jumps where a voxel's inside / outside parity changes), so single frames may
    # end in different basins (measured: 4-6 of 8 frames within 2 %, the others 10 % .. 84 % apart, some better and some
    # worse than the reference): the test pins the bulk and the absence of a bias, not the outliers.
    assert abs(it - ref_it) / ref_it < 0.20, (it, ref_it)
    assert abs(ev - ref_ev) / ref_ev < 0.35, (ev, ref_ev)       # heavy-tailed: single frames spend 200-300 evaluations in one stage
    assert np.median(rel_final) < 0.06 and (rel_final < 0.05).sum() >= B // 2
    assert abs(np.mean(np.log(final / ref_final))) < 0.15
