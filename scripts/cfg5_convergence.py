"""Convergence of the block-Jacobi sweeps of the jointly regularised sequence mode (cfg5) on a 64-frame chain: joint energy
(sum of the frames' own losses + lambda * smoothness) after every sweep, against the value after many sweeps (the fixed point of
the sweeps is a stationary point of the joint problem).  Prints the result as JSON.  One GPU:
    python scripts/cfg5_convergence.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import bench  # noqa: E402
from mvsmplfitting_b200 import synthetic as S  # noqa: E402
from mvsmplfitting_b200.sequence import SequenceFitter  # noqa: E402

T, V, SWEEPS = 64, 8, 30
model, gmm, cams = S.make_model(0), S.make_gmm(7), S.make_cameras(V)
seq = S.make_frames(model, cams, T, seed=77, smooth_walk=True)
out = {"frames": T, "views": V, "sweeps": SWEEPS, "runs": {}}
for lam in (5.0, 50.0, 500.0):
    fitter = SequenceFitter(model, cams, T, gmm=gmm, device=0)
    stages = [fitter.ctx.make_loss_config(body_prior="gmm", **{k: v for k, v in st.items() if k != "coll_loss_weight"}) for st in bench.stage_table()]
    x = torch.tensor(S.pack_params(seq["init"]), device="cuda")
    res = fitter.fit(x, torch.tensor(seq["gt_uv"], device="cuda"), torch.tensor(seq["conf"], device="cuda"),
                     torch.tensor(seq["joint_weights"], device="cuda"), stages, smooth_weight=lam, sweeps=SWEEPS)
    E = [r["joint_energy"] for r in res]
    Einf = min(E[-5:])
    gap = [(e - Einf) / abs(Einf) for e in E]
    need = next((i + 1 for i, g in enumerate(gap) if g < 1e-3), None)
    out["runs"][str(lam)] = {"joint_energy": E, "smooth_energy": [r["smooth_energy"] for r in res], "relative_gap_to_fixed_point": gap,
                             "sweeps_to_1e-3": need, "iterations": [r["frame_iterations"] for r in res]}
    print("lambda %g: E after sweeps 1..8 %s ... fixed point %.6g; sweeps to 1e-3: %s" % (lam, ["%.6g" % e for e in E[:8]], Einf, need))
    fitter.ctx.close()
print(json.dumps(out, indent=1))
