"""CPU: host-side sequence I/O (SURVEY §8f N4): camera file, keypoint JSON, result pickle / obj, batch driver."""
import json
import os
import pickle

import numpy as np
import pytest

from mvsmplfitting_b200 import seqio

DEMO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "demo")       # data the original project ships


def write_demo(tmp, V=3, B=4, missing=((1, 2),), seed=0):
    rng = np.random.default_rng(seed)
    kp = rng.uniform(0, 2000, size=(V, B, 19, 3)).astype(np.float32)        # 19 > 17: the reader keeps the first 17
    kp[..., 2] = rng.uniform(0, 1, size=(V, B, 19))
    for v in range(V):
        d = os.path.join(tmp, "keypoints", "0007", "Camera%02d" % v)
        os.makedirs(d)
        for b in range(B):
            if (v, b) in missing:
                continue
            people = [{"pose_keypoints_2d": kp[v, b].reshape(-1).tolist()}]
            with open(os.path.join(d, "%05d_keypoints.json" % (b + 1)), "w") as f:
                json.dump({"version": 1.1, "people": people}, f)
    ext = np.tile(np.eye(4), (V, 1, 1))
    ext[:, :3, :] = rng.normal(size=(V, 3, 4))
    intr = np.tile(np.eye(3), (V, 1, 1))
    intr[:, 0, 0] = intr[:, 1, 1] = rng.uniform(2000, 2500, V)
    intr[:, :2, 2] = rng.uniform(700, 1100, (V, 2))
    with open(os.path.join(tmp, "cams.txt"), "w") as f:
        for v in range(V):
            f.write("%d\n" % v)
            for r in intr[v]:
                f.write(" ".join(repr(float(x)) for x in r) + " \n")
            f.write("0 0\n")
            for r in ext[v, :3]:
                f.write(" ".join(repr(float(x)) for x in r) + " \n")
            f.write("\n")
    return kp, ext, intr


def test_camera_file_and_keypoint_folders(tmp_path):
    kp, ext, intr = write_demo(str(tmp_path))
    e, i = seqio.load_camera_para(str(tmp_path / "cams.txt"))
    assert np.array_equal(e, ext) and np.array_equal(i, intr)
    cams = seqio.camera_arrays(e, i, views=[0, 2])
    assert cams["R"].shape == (2, 3, 3) and cams["R"].dtype == np.float32
    assert np.allclose(cams["t"][1], ext[2, :3, 3]) and np.allclose(cams["f"][1], intr[2, 0, 0]) and np.allclose(cams["c"][0], intr[0, :2, 2])
    seq = seqio.load_sequence(str(tmp_path / "keypoints"), "0007")
    assert seq["cameras"] == ["Camera00", "Camera01", "Camera02"] and seq["frames"] == ["00001", "00002", "00003", "00004"]
    assert seq["gt_uv"].shape == (3, 4, 17, 2) and seq["conf"].shape == (3, 4, 17)
    assert not seq["present"][1, 2] and seq["present"].sum() == 11
    assert (seq["conf"][1, 2] == 0).all() and (seq["gt_uv"][1, 2] == 0).all()
    assert np.array_equal(seq["gt_uv"][2, 3], kp[2, 3, :17, :2]) and np.array_equal(seq["conf"][0, 0], kp[0, 0, :17, 2])
    sub = seqio.load_sequence(str(tmp_path / "keypoints"), "0007", cameras=["Camera02"], frames=["00002", "00009"])
    assert sub["gt_uv"].shape == (1, 2, 17, 2) and sub["present"].tolist() == [[True, False]]
    assert seqio.read_keypoints(str(tmp_path / "keypoints" / "0007" / "Camera00" / "00001_keypoints.json"), person=1) is None


def test_joint_weights():
    w = seqio.joint_weights("coco17", True)
    assert w[11] == 0 and w[12] == 0 and w.sum() == 15
    assert seqio.joint_weights("lsp14", True).sum() == 17 and seqio.joint_weights("lsp14", False).sum() == 15


def test_result_pickle_and_obj(tmp_path):
    x = np.arange(86, dtype=np.float32) + 1
    r = seqio.result_from_params(x, 12.5)
    assert [r[k].shape for k in ("betas", "global_orient", "body_pose", "transl", "scale")] == [(1, 10), (1, 3), (1, 69), (1, 3), (1,)]
    verts = np.random.default_rng(0).normal(size=(5, 3))
    faces = np.array([[0, 1, 2], [2, 3, 4]])
    out = seqio.save_results(str(tmp_path / "res"), "0007", "00001", r, verts=verts, faces=faces, mesh_folder=str(tmp_path / "mesh"))
    assert out == str(tmp_path / "res" / "0007" / "00001" / "000.pkl")
    with open(out, "rb") as f:
        raw = f.read()
    assert raw[:2] == b"\x80\x02"                                    # protocol 2, utils.py:862
    got = pickle.loads(raw)
    bp = got["body_pose"][0]
    assert (bp[18:24] == 0).all() and (bp[27:33] == 0).all() and (bp[57:] == 0).all() and (bp[:18] == x[13:31]).all()
    assert got["pose"].shape == (1, 72) and (got["pose"][0, :3] == x[10:13]).all() and got["loss"] == 12.5
    lines = open(tmp_path / "mesh" / "0007" / "00001" / "000.obj").read().splitlines()
    assert len(lines) == 7 and lines[5] == "f 1 2 3" and lines[6] == "f 3 4 5"
    assert np.allclose([float(t) for t in lines[0].split()[1:]], verts[0], atol=1e-7)


class StubCtx:                                      # records what the drivers ask of a FittingContext
    def __init__(self, B):
        self.B, self.calls = B, []

    def set_keypoints(self, gt_uv, conf, jw):
        self.calls.append(("kp", gt_uv.shape, conf.shape, jw.sum()))
        self.kp0 = float(gt_uv[0, 0, 0, 0])

    def set_loss(self, config=None):
        self.calls.append(("loss", config.use_vposer))

    def init_guess(self, **kw):
        import torch
        self.calls.append(("init", kw["estimate_scale"], kw["use_torso"], kw["hip_seed"]))
        return torch.arange(self.B * 86, dtype=torch.float32).reshape(self.B, 86), None

    def fit(self, params, stage_cfgs, opt_cfg, warm=None):
        import torch
        self.calls.append(("fit", len(stage_cfgs), None if warm is None else list(map(bool, warm)), params.clone()))
        params += 1
        return torch.arange(1, self.B + 1, dtype=torch.float32), dict(frame_iterations=7, frame_evals=9, rounds=1, frames_nan=0)

    def vposer_decode(self, params):
        import torch
        self.calls.append(("decode",))
        return torch.full((self.B, 69), 0.25) + params[:, 13:14]

    def forward_only(self, params, want_verts=True):
        import torch
        self.calls.append(("fwd", float(params[0, 13 + 18]), float(params[0, 13 + 17])))
        return dict(verts=torch.zeros(self.B, 5, 3))


def _cfgs(n, use_vposer=0, use_joints_conf=1):
    from types import SimpleNamespace
    return [SimpleNamespace(use_vposer=use_vposer, use_joints_conf=use_joints_conf) for _ in range(n)]


def test_fit_sequence_drives_the_context_in_batch_order(tmp_path):
    write_demo(str(tmp_path))
    seq = seqio.load_sequence(str(tmp_path / "keypoints"), "0007")
    ctx = StubCtx(4)
    x, loss, st = seqio.fit_sequence(ctx, seq, stage_cfgs=_cfgs(4), result_folder=str(tmp_path / "res"),
                                     mesh_folder=str(tmp_path / "mesh"), faces=np.array([[0, 1, 2]]))
    assert [c[0] for c in ctx.calls] == ["kp", "loss", "init", "fit", "fwd"]
    assert ctx.calls[0][1:] == ((3, 4, 17, 2), (3, 4, 17), 15.0) and ctx.calls[2][1:] == (False, True, 1.0)
    assert ctx.calls[4][1] == 0.0 and ctx.calls[4][2] == 13 + 17 + 1          # mesh from the saved (zeroed) pose
    assert x.shape == (4, 86) and x[1, 0] == 87 and loss.tolist() == [1, 2, 3, 4] and st["frame_iterations"] == 7
    for b, fr in enumerate(seq["frames"]):
        got = pickle.load(open(tmp_path / "res" / "0007" / fr / "000.pkl", "rb"))
        assert got["loss"] == b + 1 and got["transl"][0, 0] == b * 86 + 82 + 1 and got["pose_embedding"] is None
        assert os.path.exists(tmp_path / "mesh" / "0007" / fr / "000.obj")
    # a (view, frame) without detections is only neutral when the loss uses the confidences (main.py:45-56 drops the view)
    with pytest.raises(ValueError):
        seqio.fit_sequence(StubCtx(4), seq, stage_cfgs=_cfgs(4, use_joints_conf=0))
    with pytest.raises(NotImplementedError):
        seqio.fit_sequence(StubCtx(4), seq, stage_cfgs=_cfgs(4, use_vposer=1))


def test_fit_sequence_with_latent_pose_saves_the_decoded_pose(tmp_path):
    """use_vposer = 2 (the reference's default configuration): the initial guess sees the stage configuration (latent code
    starts at 0), results hold decode(latent) with the extremities zeroed plus 'pose_embedding' (utils.py:741-759), the mesh
    is built from that pose"""
    write_demo(str(tmp_path))
    seq = seqio.load_sequence(str(tmp_path / "keypoints"), "0007")
    ctx = StubCtx(4)
    x, loss, st = seqio.fit_sequence(ctx, seq, stage_cfgs=_cfgs(4, use_vposer=2), result_folder=str(tmp_path / "res"),
                                     mesh_folder=str(tmp_path / "mesh"), faces=np.array([[0, 1, 2]]))
    assert [c[0] for c in ctx.calls] == ["kp", "loss", "init", "fit", "decode", "fwd"] and ctx.calls[1][1] == 2
    got = pickle.load(open(tmp_path / "res" / "0007" / seq["frames"][1] / "000.pkl", "rb"))
    dec = 0.25 + x[1, 13]
    assert np.allclose(got["body_pose"][0, :18], dec) and (got["body_pose"][0, 18:24] == 0).all() and (got["body_pose"][0, 57:] == 0).all()
    assert got["pose_embedding"].shape == (1, 32) and np.array_equal(got["pose_embedding"][0], x[1, 13:45])
    assert np.allclose(got["pose"][0, 3:21], dec) and np.array_equal(got["pose"][0, :3], x[1, 10:13])
    assert ctx.calls[5][1] == 0.0 and np.isclose(ctx.calls[5][2], 0.25 + x[0, 13])       # mesh: decoded pose, zeroed extremities


def test_fit_sequences_lockstep_warm_start(tmp_path):
    """is_seq = True (main.py:76-79, non_linear_solver.py:157-162) for two sequences of different length in lock-step"""
    write_demo(str(tmp_path))
    a = seqio.load_sequence(str(tmp_path / "keypoints"), "0007")
    b = seqio.load_sequence(str(tmp_path / "keypoints"), "0007", frames=a["frames"][:2])
    ctx = StubCtx(2)
    res, tot = seqio.fit_sequences(ctx, [a, b], stage_cfgs=_cfgs(4), result_folder=str(tmp_path / "res"), reinit_loss=1.5)
    fits = [c for c in ctx.calls if c[0] == "fit"]
    assert len(fits) == 4 and tot["frame_iterations"] == 28
    assert fits[0][2] is None                                  # first frames: every stage, cold
    # the stub's losses are (1, 2): sequence 0 stays below the re-initialisation threshold (warm), sequence 1 does not
    assert fits[1][2] == [True, False] and fits[2][2] == [True, False]
    p1 = fits[1][3]
    cold = np.arange(2 * 86, dtype=np.float32).reshape(2, 86)
    assert np.array_equal(p1[0, :13].numpy(), cold[0, :13] + 1) and np.array_equal(p1[0, 82:].numpy(), cold[0, 82:] + 1)   # carried
    assert np.array_equal(p1[0, 13:82].numpy(), cold[0, 13:82])                       # fix_params: pose back to the seed
    assert np.array_equal(p1[1].numpy(), cold[1])                                     # re-initialised
    assert res[0][0].shape == (4, 86) and res[1][0].shape == (2, 86) and res[1][1].tolist() == [2, 2]
    assert sorted(os.listdir(tmp_path / "res" / "0007")) == a["frames"]


def test_readers_equal_the_reference_on_its_demo_data():
    """against what the original project's own load_camera_para / read_keypoints return for the data it ships
    (tests/golden/demo_readers_ref.npz, oracle/make_golden_refruns.py)"""
    ref = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "demo_readers_ref.npz"))
    e, i = seqio.load_camera_para(os.path.join(DEMO, "3DOH50K_Parameters.txt"))
    assert e.shape == (6, 4, 4) and np.array_equal(e, ref["extrinsics"]) and np.array_equal(i, ref["intrinsics"])
    seq = seqio.load_sequence(os.path.join(DEMO, "keypoints"), "0000")
    assert len(seq["cameras"]) == 6 and seq["frames"] == ["00001"] and seq["present"].all()
    assert list(seq["cameras"]) == ref["cameras"].tolist()
    for v in range(len(seq["cameras"])):
        kp = ref["keypoints"][v]
        assert np.array_equal(seq["gt_uv"][v, 0], kp[:, :2]) and np.array_equal(seq["conf"][v, 0], kp[:, 2])
