"""TEST INFRASTRUCTURE -- writes tests/golden/seq3d_*.npz by RUNNING THE UNMODIFIED REFERENCE's reader of the 3-D joint
annotations (use_3d).  Authoring container only (needs /root/reference):

    python -m oracle.make_golden_seq3d

* seq3d_reader.npz  seeded keypoint JSON files (stored as text) of one sequence of 3 views x 6 frames and of a second
                    sequence with an 18-row annotation, with what the reference returns for them:
                    - per file, utils/data_parser.read_joints (use_hands = use_face = False): None, or person 0's rows [N,4]
                    - per frame, FittingData.read_item's data['3d_joint'][0] (data_parser.py:366-411, the first view in
                      camera order whose file exists and parses), or None
                    Cases: the annotation only in view 1's file while view 0's file has none (pose_keypoints_3d missing),
                    view 0's file missing, view 0's annotation of a length that is not a multiple of 4, no annotation in any
                    view, annotations in every view (view 0's wins), and view 0's file listing a second person without one.
* seq3d_e2e.npz     the reference's own main loop (main.py:76-86: init_guess or load_init, fix_params, non_linear_solver) with
                    is_seq and use_3d, on the CPU with the SDF term off: 2 sequences x 3 frames x 4 views of
                    synthetic.make_frames(smooth_walk=True), GMM prior, axis-angle pose, the 4-stage fit_smpl.yaml schedule.
                    Targets: true keypoints + 2 cm noise, confidences in [0.5, 1]; frame 1 of sequence 1 has no annotation;
                    use_hip is not set, so the solver zeroes the hips' 3-D confidences and the 2-D joint weights drop the hips
                    (data_parser.py:340-358).  Per frame: its cold start point (init_guess + fix_params on that frame,
                    computed for every frame, warm or cold), whether the loop started it warm, the final parameters, the loss
                    run_fitting returned, L-BFGS iterations and closure evaluations, and the reference's SMPLifyLoss at the
                    final parameters with the last stage's weights.
"""
from __future__ import annotations

import json
import os
import sys
import tempfile
import types
import warnings

import numpy as np

warnings.filterwarnings("ignore")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mvsmplfitting_b200 import synthetic as S  # noqa: E402
from oracle import ref_harness as H  # noqa: E402
from oracle.make_golden import model_checksum  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
VIEWS = 3


def reader_cases(rng):
    """{(serial, camera, frame): people list or None (no file)}: the cases of the module docstring"""
    def person(k3d=17, bad=False, with3d=True):
        p = {"pose_keypoints_2d": np.round(rng.uniform(0, 2000, 17 * 3), 3).astype(np.float32).tolist()}
        if with3d:
            a = np.concatenate([rng.normal(0, 1, (k3d, 3)), rng.uniform(0, 1, (k3d, 1))], 1).astype(np.float32).reshape(-1)
            p["pose_keypoints_3d"] = (a[:-1] if bad else a).tolist()
        return p
    files = {}
    cams = ["Camera%02d" % v for v in range(VIEWS)]
    plan = {                      # frame -> per view: 'ok', 'no3d', 'bad', 'missing', 'second_no3d'
        "00001": ("no3d", "ok", "ok"),
        "00002": ("missing", "ok", "no3d"),
        "00003": ("bad", "no3d", "ok"),
        "00004": ("no3d", "no3d", "missing"),
        "00005": ("ok", "ok", "ok"),
        "00006": ("second_no3d", "ok", "ok"),
    }
    for fr, kinds in plan.items():
        for cam, kind in zip(cams, kinds):
            if kind == "missing":
                files[("0000", cam, fr)] = None
            elif kind == "second_no3d":
                files[("0000", cam, fr)] = [person(), person(with3d=False)]
            else:
                files[("0000", cam, fr)] = [person(with3d=kind != "no3d", bad=kind == "bad")]
    for cam in cams:                                               # a sequence whose annotation has 18 rows
        files[("0001", cam, "00001")] = [person(k3d=18)]
    return files, cams


def reader(out_dir):
    H.import_reference()
    with H.in_reference_dir():
        import cv2
        from utils import data_parser as DP
    rng = np.random.RandomState(5300)
    files, cams = reader_cases(rng)
    out = {}
    names, texts = [], []
    with tempfile.TemporaryDirectory() as tmp:
        kp_root, img_root = os.path.join(tmp, "keypoints"), os.path.join(tmp, "images")
        for (serial, cam, fr), people in files.items():
            os.makedirs(os.path.join(kp_root, serial, cam), exist_ok=True)
            os.makedirs(os.path.join(img_root, serial, cam), exist_ok=True)
            cv2.imwrite(os.path.join(img_root, serial, cam, fr + ".jpg"), np.zeros((4, 4, 3), np.uint8))
            if people is None:
                continue
            rel = "%s/%s/%s_keypoints.json" % (serial, cam, fr)
            txt = json.dumps({"version": 1.3, "people": people})
            with open(os.path.join(kp_root, rel), "w") as f:
                f.write(txt)
            names.append(rel)
            texts.append(txt)
        for i, rel in enumerate(names):                            # the reference's read_joints per file
            kp = DP.read_joints(os.path.join(kp_root, rel), use_hands=False, use_face=False).keypoints
            out["rj_none_%d" % i] = np.bool_(kp is None)
            if kp is not None:
                out["rj_%d" % i] = np.asarray(kp[0], np.float32)
        # FittingData.read_item on the frames of sequence 0000, views in camera order; only the attributes it reads are set
        item = types.SimpleNamespace(keyp_folder=kp_root, use_hands=False, use_face=False, use_face_contour=False, use_3d=True)
        frames = sorted({fr for (s, _, fr) in files if s == "0000"})
        has = np.zeros(len(frames), bool)
        j3d = np.zeros((len(frames), 17, 4), np.float32)
        for b, fr in enumerate(frames):
            d = DP.FittingData.read_item(item, [os.path.join(img_root, "0000", cam, fr + ".jpg") for cam in cams])
            if d["3d_joint"] is not None:
                has[b], j3d[b] = True, np.asarray(d["3d_joint"][0], np.float32)
    out.update(names=np.array(names), texts=np.array(texts), cameras=np.array(cams), frames=np.array(frames), has3d=has,
               joints3d=j3d)
    np.savez_compressed(os.path.join(out_dir, "seq3d_reader.npz"), **out)
    print("wrote seq3d_reader.npz: has3d", has.tolist())


def _params_row(rm):
    return np.concatenate([getattr(rm, k).detach().numpy().reshape(-1) for k in S.PARAM_ORDER]).astype(np.float32)


def _solve(sc, setting, data, args):
    """the reference's non_linear_solver on the model's current parameters; (result, iterations, evaluations), counted as
    oracle/ref_fit.fit_frame counts them (every optimiser the solver creates)"""
    import contextlib
    import io
    ns, nls = sc["ns"], sc["nls"]
    made = []
    factory = ns.optim_factory.create_optimizer

    def recording_factory(params, **kw):
        out = factory(params, **kw)
        made.append(out[0])
        return out
    ns.optim_factory.create_optimizer = recording_factory
    try:
        with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
            result = nls.non_linear_solver(setting, data, use_cuda=False, **args)
    finally:
        ns.optim_factory.create_optimizer = factory
    its = sum(int(o.state[o._params[0]].get("n_iter", 0)) for o in made)
    evs = sum(int(o.state[o._params[0]].get("func_evals", 0)) for o in made)
    return result, its, evs


def e2e(out_dir):
    import torch
    from mvsmplfitting_b200 import seqio
    from oracle import ref_fit as RF
    from oracle.make_golden import stage_weights
    from oracle.make_golden_3d import reference_closure_3d, targets
    torch.set_num_threads(1)
    H.import_reference()
    with H.in_reference_dir():
        from utils import init_guess as RIG
    model, gmm = S.make_model(0), S.make_gmm(7)
    V, T, seeds, no3d = 4, 3, (5400, 5410), {(1, 1)}
    cams = {k: v[:V] for k, v in S.make_cameras(4).items() if isinstance(v, np.ndarray)}
    ext = np.tile(np.eye(4), (V, 1, 1))
    ext[:, :3, :3], ext[:, :3, 3] = cams["R"], cams["t"]
    intr = np.tile(np.eye(3), (V, 1, 1))
    intr[:, 0, 0], intr[:, 1, 1], intr[:, 0, 2], intr[:, 1, 2] = cams["f"][:, 0], cams["f"][:, 1], cams["c"][:, 0], cams["c"][:, 1]
    jw = seqio.joint_weights("lsp14", use_hip=False)
    sc = RF.build_scene(model, gmm, cams)
    rm, dt = sc["model"], torch.float32
    args = dict(RF.stage_args(S.STAGE_WEIGHTS, False), is_seq=True, use_3d=True)     # use_hip not set: hips zeroed
    kw = dict(use_torso=True, model_type="smpllsp", use_vposer=False, use_3d=True)
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self            # init_guess.py:38 hard-codes .cuda(); a no-op here
    out = {}
    try:
        for s_, seed in enumerate(seeds):
            fr = S.make_frames(model, cams, T, seed=seed, smooth_walk=True)
            gt3d, conf3d = targets(fr, seed + 1)
            has = np.array([(s_, t) not in no3d for t in range(T)])
            cold, warm, par, fin, its, evs = [], [], [], [], [], []
            results = None
            for t in range(T):
                kp = np.concatenate([fr["gt_uv"][:, t:t + 1], fr["conf"][:, t:t + 1, :, None]], axis=-1).astype(np.float32)
                data = {"keypoints": kp, "3d_joint": [np.concatenate([gt3d[t], conf3d[t][:, None]], 1)] if has[t] else None,
                        "img": [np.zeros((1536, 2, 3), np.uint8)], "img_path": None}
                setting = dict(model=rm, dtype=dt, batch_size=1, device=torch.device("cpu"), fix_scale=False, fixed_scale=None,
                               fixed_shape=None, extris=ext, intris=intr, views=V, vposer=None, camera=sc["cams"],
                               pose_embedding=None, joints_weight=torch.tensor(jw, dtype=dt).unsqueeze(0),
                               body_pose_prior=sc["body_pose_prior"], shape_prior=sc["shape_prior"],
                               angle_prior=sc["angle_prior"], adjustment=False, seq_start=t == 0)
                RIG.init_guess(setting, data, **kw)                     # the frame's cold start point
                RIG.fix_params(setting, scale=None, shape=None)
                cold.append(_params_row(rm))
                if setting["seq_start"]:                                # main.py:76-82
                    RIG.init_guess(setting, data, **kw)
                else:
                    RIG.load_init(setting, data, results, **kw)
                warm.append(not setting["seq_start"])
                RIG.fix_params(setting, scale=setting["fixed_scale"], shape=setting["fixed_shape"])
                results, it, ev = _solve(sc, setting, data, args)
                par.append(_params_row(rm))
                fin.append(float(results["loss"]))
                its.append(it)
                evs.append(ev)
                print("seq %d frame %d warm %s 3d %s: loss %.4f, %d iterations" % (s_, t, warm[-1], has[t], fin[-1], it))
            # the reference's SMPLifyLoss at its final parameters, last stage's weights, use_3d as the solver had it
            c3 = conf3d.copy()
            c3[:, [11, 12]] = 0.0                                       # non_linear_solver.py:92-94
            P = np.stack(par)
            pd, o = {}, 0
            for k, n in zip(S.PARAM_ORDER, S.PARAM_SIZES):
                pd[k] = P[:, o:o + n]
                o += n
            crm, crc = H.build_reference_model(model, dtype=dt), H.build_reference_cameras(cams, dtype=dt)
            bp = H.build_reference_gmm(gmm, dtype=dt)
            frd = dict(fr, joint_weights=jw)
            w3 = stage_weights(3)
            at = [reference_closure_3d(crm, crc, frd, t, w3, bp, dt, pd, gt3d, c3, 100.0, False)[0] if has[t] else
                  H.reference_closure_eval(crm, crc, frd, t, w3, bp, dtype=dt, params=pd)["loss"] for t in range(T)]
            tag = "s%d_" % s_
            out.update({tag + "seed": np.int64(seed), tag + "gt_uv": fr["gt_uv"], tag + "conf": fr["conf"],
                        tag + "gt3d": gt3d, tag + "conf3d": conf3d, tag + "has3d": has, tag + "cold": np.stack(cold),
                        tag + "warm": np.array(warm), tag + "params": P, tag + "final_loss": np.array(fin),
                        tag + "iterations": np.array(its), tag + "evals": np.array(evs), tag + "loss_at_final": np.array(at)})
    finally:
        torch.Tensor.cuda = cuda
    out.update(n_seq=np.int64(len(seeds)), joint_weights=jw, model_checksum=np.array(model_checksum(model)),
               **{"cam_" + k: cams[k] for k in ("R", "t", "f", "c")})
    np.savez_compressed(os.path.join(out_dir, "seq3d_e2e.npz"), **out)
    print("wrote seq3d_e2e.npz")


def main():
    what = sys.argv[1:] or ["reader", "e2e"]
    if "reader" in what:
        reader(GOLD)
    if "e2e" in what:
        e2e(GOLD)


if __name__ == "__main__":
    main()
