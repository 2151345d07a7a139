"""CPU: the 3-D joint annotations (use_3d) of whole sequences: the reader against the reference's own (tests/golden/seq3d_reader.npz,
oracle/make_golden_seq3d.py), and what every sequence driver asks of a FittingContext with use_3d=True."""
import os

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import seqio
from tests.test_seqio import StubCtx, _cfgs, write_demo

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "seq3d_reader.npz")


def write_reader_fixture(tmp):
    ref = np.load(GOLD)
    root = os.path.join(tmp, "keypoints")
    for rel, txt in zip(ref["names"].tolist(), ref["texts"].tolist()):
        os.makedirs(os.path.dirname(os.path.join(root, rel)), exist_ok=True)
        with open(os.path.join(root, rel), "w") as f:
            f.write(txt)
    return ref, root


def test_read_joints_equals_the_reference(tmp_path):
    ref, root = write_reader_fixture(str(tmp_path))
    n_none = 0
    for i, rel in enumerate(ref["names"].tolist()):
        got = seqio.read_joints(os.path.join(root, rel))
        if bool(ref["rj_none_%d" % i]):
            assert got is None, rel
            n_none += 1
        else:
            assert got.dtype == np.float32 and np.array_equal(got, ref["rj_%d" % i]), rel
    assert n_none >= 5                                   # missing pose_keypoints_3d, a malformed length, a second person without
    assert any(ref["rj_%d" % i].shape[0] == 18 for i in range(len(ref["names"])) if not ref["rj_none_%d" % i])


def test_load_sequence_takes_the_first_view_that_parses(tmp_path):
    ref, root = write_reader_fixture(str(tmp_path))
    seq = seqio.load_sequence(root, "0000", use_3d=True)
    assert seq["cameras"] == ref["cameras"].tolist() and seq["frames"] == ref["frames"].tolist()
    assert seq["has3d"].dtype == bool and seq["has3d"].tolist() == ref["has3d"].tolist() and not seq["has3d"].all()
    assert seq["joints3d"].shape == (6, 17, 3) and seq["conf3d"].shape == (6, 17)
    assert np.array_equal(seq["joints3d"], ref["joints3d"][..., :3]) and np.array_equal(seq["conf3d"], ref["joints3d"][..., 3])
    assert (seq["joints3d"][~seq["has3d"]] == 0).all() and (seq["conf3d"][~seq["has3d"]] == 0).all()
    plain = seqio.load_sequence(root, "0000")
    assert not {"joints3d", "conf3d", "has3d"} & set(plain)
    for k in ("gt_uv", "conf", "present"):
        assert np.array_equal(plain[k], seq[k])
    # the first view in the order the sequence is loaded with: view 0 left out, frame 00005 takes view 1's rows
    sub = seqio.load_sequence(root, "0000", cameras=ref["cameras"].tolist()[1:], use_3d=True)
    direct = seqio.read_joints(os.path.join(root, "0000", ref["cameras"][1], "00005_keypoints.json"))
    assert np.array_equal(sub["joints3d"][4], direct[:, :3]) and not np.array_equal(sub["joints3d"][4], seq["joints3d"][4])
    with pytest.raises(ValueError, match="0001.*00001_keypoints.json"):          # 18 rows
        seqio.load_sequence(root, "0001", use_3d=True)


class Stub3d(StubCtx):
    """StubCtx with the 3-D entry points: init_guess adds 0.5 while 3-D targets are set (it aligns to them)"""
    device = "cpu"

    def __init__(self, B):
        super().__init__(B)
        self.j3d = None

    def set_joints3d(self, gt_xyz, conf=None):
        self.j3d = None if gt_xyz is None else (np.array(gt_xyz, np.float32), np.array(conf, np.float32))
        self.calls.append(("j3d", self.j3d))

    def init_guess(self, **kw):
        x, _ = super().init_guess(**kw)
        self.calls[-1] += (self.j3d is not None,)
        return (x + 0.5 if self.j3d is not None else x), None

    def fit(self, params, stage_cfgs, opt_cfg, warm=None):
        out = super().fit(params, stage_cfgs, opt_cfg, warm)
        self.calls[-1] += (self.j3d,)
        return out

    def fit_stream(self, params, gt_uv, conf, jw, stage_cfgs, opt_cfg=None, joints3d=None, conf3d=None):
        self.calls.append(("stream", params.clone(), joints3d, conf3d))
        self.j3d = None
        params += 1
        return torch.arange(params.shape[0], dtype=torch.float32), dict(frame_iterations=3)

    def fit_seq_stream(self, params, gt_uv, conf, jw, lengths, stage_cfgs, opt_cfg=None, reinit_loss=5000.0, joints3d=None,
                       conf3d=None):
        self.calls.append(("seq_stream", params.clone(), list(lengths), reinit_loss, joints3d, conf3d))
        self.j3d = None
        params += 1
        return torch.arange(params.shape[0], dtype=torch.float32), dict(frame_iterations=5)


def seq3d(tmp, frames, has, seed):
    """a write_demo sequence (every view present) with 3-D annotations on the frames `has` marks"""
    d = os.path.join(tmp, "s%d" % seed)
    os.makedirs(d)
    write_demo(d, B=4, missing=(), seed=seed)
    q = seqio.load_sequence(os.path.join(d, "keypoints"), "0007", frames=["%05d" % (t + 1) for t in range(frames)])
    rng = np.random.default_rng(seed)
    q["has3d"] = np.array(has, bool)
    q["joints3d"] = rng.normal(size=(frames, 17, 3)).astype(np.float32) * q["has3d"][:, None, None]
    q["conf3d"] = rng.uniform(0.2, 1, size=(frames, 17)).astype(np.float32) * q["has3d"][:, None]
    return q


def expect(q, t, use_hip=False):
    """targets and confidences a driver must upload for frame t of q"""
    if not q["has3d"][t]:
        return np.zeros((17, 3), np.float32), np.zeros(17, np.float32)
    c = q["conf3d"][t].copy()
    if not use_hip:
        c[11] = c[12] = 0.0
    return q["joints3d"][t], c


def test_lockstep_uploads_each_step_and_merges_the_two_guesses(tmp_path):
    a = seq3d(str(tmp_path), 4, [True, False, True, True], 1)
    b = seq3d(str(tmp_path), 2, [True, True], 2)
    ctx = Stub3d(2)
    res, tot = seqio.fit_sequences(ctx, [a, b], _cfgs(4), reinit_loss=1.5, use_hip=False, use_3d=True)
    fits = [c for c in ctx.calls if c[0] == "fit"]
    inits = [c for c in ctx.calls if c[0] == "init"]
    assert len(fits) == 4 and tot["frame_iterations"] == 28
    # one guess with the targets per step, plus one without where a frame of the step has no annotation (a at t = 1)
    assert [c[-1] for c in inits] == [True, True, False, True, True]
    cold = np.arange(2 * 86, dtype=np.float32).reshape(2, 86)
    for t, f in enumerate(fits):
        rows = [expect(a, t), expect(b, min(t, 1))]                  # b idles on its last frame
        j3, c3 = f[-1]
        for s_ in range(2):
            assert np.array_equal(j3[s_], rows[s_][0]) and np.array_equal(c3[s_], rows[s_][1]), (t, s_)
        assert (c3[:, 11:13] == 0).all()
    p0 = fits[0][3].numpy()
    assert np.array_equal(p0, cold + 0.5)                            # both first frames align to their annotation
    p1 = fits[1][3].numpy()                                          # a warm, b cold (stub losses 1, 2; reinit 1.5)
    assert fits[1][2] == [True, False]
    assert np.array_equal(p1[0, 13:82], cold[0, 13:82])             # a's own row from the pass without targets (no annotation)
    assert np.array_equal(p1[1], cold[1] + 0.5)                     # b re-initialised, aligned to its annotation
    assert ctx.calls[-1] == ("j3d", None) and ctx.j3d is None
    assert res[0][0].shape == (4, 86) and res[1][0].shape == (2, 86)


def test_use_hip_keeps_the_hip_confidences(tmp_path):
    a = seq3d(str(tmp_path), 2, [True, True], 3)
    ctx = Stub3d(1)
    seqio.fit_sequences(ctx, [a], _cfgs(4), use_hip=True, use_3d=True)
    f = [c for c in ctx.calls if c[0] == "fit"][0]
    assert np.array_equal(f[-1][1][0], a["conf3d"][0]) and (f[-1][1][0, 11:13] > 0).all()


def test_refusals(tmp_path):
    a = seq3d(str(tmp_path), 2, [True, False], 4)
    with pytest.raises(ValueError, match="use_joints_conf"):
        seqio.fit_sequences(Stub3d(1), [a], _cfgs(4, use_joints_conf=0), use_3d=True)
    with pytest.raises(ValueError, match="use_joints_conf"):
        seqio.fit_sequence(Stub3d(2), a, _cfgs(4, use_joints_conf=0), use_3d=True)
    plain = {k: v for k, v in a.items() if k not in ("joints3d", "conf3d", "has3d")}
    with pytest.raises(ValueError, match="use_3d"):
        seqio.fit_sequences(Stub3d(1), [plain], _cfgs(4), use_3d=True)
    with pytest.raises(ValueError, match="use_3d"):
        seqio.fit_sequence(Stub3d(2), plain, _cfgs(4), use_3d=True)


def test_fit_sequence_batch(tmp_path):
    q = seq3d(str(tmp_path), 4, [True, False, True, False], 5)
    ctx = Stub3d(4)
    x, loss, st = seqio.fit_sequence(ctx, q, _cfgs(4), use_hip=False, use_3d=True)
    assert [c[0] for c in ctx.calls] == ["kp", "loss", "j3d", "init", "j3d", "init", "j3d", "fit", "j3d"]
    fit = ctx.calls[7]
    cold = np.arange(4 * 86, dtype=np.float32).reshape(4, 86)
    assert np.array_equal(fit[3].numpy(), cold + np.array([0.5, 0, 0.5, 0], np.float32)[:, None])
    for t in range(4):
        assert np.array_equal(fit[-1][0][t], expect(q, t)[0]) and np.array_equal(fit[-1][1][t], expect(q, t)[1])
    assert ctx.calls[-1] == ("j3d", None)


def test_fit_sequence_stream_chunks(tmp_path):
    q = seq3d(str(tmp_path), 4, [True, False, True, True], 6)
    ctx = Stub3d(3)
    x, loss, st = seqio.fit_sequence(ctx, q, _cfgs(4), use_hip=False, use_3d=True)
    # chunk 0 (frames 0-2) mixes: two guesses; chunk 1 (frame 3 + padding) has annotations only: one
    assert [c[-1] for c in ctx.calls if c[0] == "init"] == [True, False, True]
    stream = [c for c in ctx.calls if c[0] == "stream"][0]
    cold = np.arange(3 * 86, dtype=np.float32).reshape(3, 86)
    want = np.concatenate([cold + np.array([0.5, 0, 0.5], np.float32)[:, None], cold[:1] + 0.5])
    assert np.array_equal(stream[1].numpy(), want)
    for t in range(4):
        assert np.array_equal(stream[2][t], expect(q, t)[0]) and np.array_equal(stream[3][t], expect(q, t)[1])
    assert ctx.calls[-1] == ("j3d", None)


def test_fit_sequences_stream_arguments(tmp_path):
    a = seq3d(str(tmp_path), 3, [False, True, True], 7)
    b = seq3d(str(tmp_path), 2, [True, False], 8)
    ctx = Stub3d(4)
    res, st = seqio.fit_sequences(ctx, [a, b], _cfgs(4), reinit_loss=123.0, use_hip=False, use_3d=True)
    call = [c for c in ctx.calls if c[0] == "seq_stream"][0]
    assert call[2] == [3, 2] and call[3] == 123.0
    for f, (q, t) in enumerate([(a, 0), (a, 1), (a, 2), (b, 0), (b, 1)]):
        assert np.array_equal(call[4][f], expect(q, t)[0]) and np.array_equal(call[5][f], expect(q, t)[1]), f
    cold = np.arange(4 * 86, dtype=np.float32).reshape(4, 86)
    want = np.concatenate([cold + np.array([0, 0.5, 0.5, 0.5], np.float32)[:, None], cold[:1]])
    assert np.array_equal(call[1].numpy(), want)
    assert [c[-1] for c in ctx.calls if c[0] == "init"] == [True, False, False]
    assert ctx.calls[-1] == ("j3d", None) and st["frame_iterations"] == 5


def test_read_joints_without_people_raises_as_the_reference(tmp_path):
    fn = tmp_path / "x_keypoints.json"
    fn.write_text('{"version": 1.3}')
    with pytest.raises(KeyError):
        seqio.read_joints(str(fn))
