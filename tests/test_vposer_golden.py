"""CPU: the VPoser restatement (oracle/vposer_oracle.py), the oracle closure with use_vposer, and the device math of the
rotation head (csrc/mvs_math.cuh: cont6d_to_aa_fwd / _bwd, compiled for the host) against fixtures written by running
the unmodified reference VPoser class and fitting closure (oracle/make_golden_vposer.py)."""
import os
import subprocess

import numpy as np
import torch

from mvsmplfitting_b200 import synthetic as S
from oracle import closure_oracle as O
from oracle import vposer_oracle as VO
from tests import golden_util as G

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vposer_s11.npz")


def test_decode_restatement_matches_reference():
    c = np.load(GOLD)
    w = S.make_vposer(11)
    for dt, tag, tol in ((torch.float64, "f64", 1e-10), (torch.float32, "f32", 2e-4)):
        aa = VO.decode_aa(w, torch.tensor(c["Z"], dtype=dt)).numpy()
        ref = c["aa_" + tag]
        assert np.abs(aa - ref).max() < tol * max(1.0, np.abs(ref).max()), tag
    # the fixture exercises every branch of rotation_matrix_to_quaternion
    R = VO.cont6d_to_matrot(VO.decode_6d(w, torch.tensor(c["Z"], dtype=torch.float64)))
    m = R.transpose(1, 2)
    d2 = m[:, 2, 2] < 1e-6
    br = np.where(d2 & (m[:, 0, 0] > m[:, 1, 1]), 0, np.where(d2, 1, np.where(m[:, 0, 0] < -m[:, 1, 1], 2, 3)))
    assert set(np.unique(br).tolist()) == {0, 1, 2, 3}


def test_closure_with_vposer_matches_reference(syn_model):
    c = np.load(GOLD)
    w = S.make_vposer(11)
    cams = dict(R=c["cam_R"], t=c["cam_t"], f=c["cam_f"], c=c["cam_c"])
    for stage in (3, 0):
        dw, bpw, sw, bend = [float(v) for v in c["w%d" % stage]]
        for dt, tag, tol in ((torch.float64, "f64", 1e-9), (torch.float32, "f32", 1e-4)):
            om = O.OracleModel.from_numpy(syn_model, dtype=dt)
            pri = O.OraclePriors(kind="l2")
            cfg = O.LossConfig(data_weight=dw, body_pose_weight=bpw, shape_weight=sw, bending_prior_weight=bend, use_vposer=True)
            for b in range(2):
                r = O.closure_eval_vposer(om, cfg, pri, O.cams_to_torch(cams, dt), c["X"][b], c["closure_Z"][b], w,
                                          c["gt_uv"][:, b], c["conf"][:, b], c["joint_weights"])
                pre = "s%d_b%d_%s_" % (stage, b, tag)
                assert abs(r["loss"] - float(c[pre + "loss"])) / abs(float(c[pre + "loss"])) < tol
                assert G.relmax(r["joints"], c[pre + "joints"]) < tol
                assert G.relmax(r["body_pose"], c[pre + "body_pose"]) < max(tol, 1e-9)
                for k in ("betas", "global_orient", "transl", "scale", "pose_embedding"):
                    assert G.relmax(r["g_" + k], c[pre + "g_" + k]) < tol, (stage, b, tag, k)


HOST_SRC = r"""
#include <cstdio>
#include "%s"
using namespace mvs;
int main() {
    double o[6], daa[3];
    while (scanf("%%lf %%lf %%lf %%lf %%lf %%lf %%lf %%lf %%lf", o, o+1, o+2, o+3, o+4, o+5, daa, daa+1, daa+2) == 9) {
        double aa[3], dob[6];
        Cont6dState<double> S;
        cont6d_to_aa_fwd(o, aa, S);
        cont6d_to_aa_bwd(S, daa, dob);
        printf("%%.17g %%.17g %%.17g %%.17g %%.17g %%.17g %%.17g %%.17g %%.17g %%d\n", aa[0], aa[1], aa[2], dob[0], dob[1], dob[2], dob[3], dob[4], dob[5], S.branch);
    }
    return 0;
}
"""


def test_device_math_of_the_rotation_head_matches_autograd(tmp_path):
    """the __host__ __device__ functions the kernel calls, compiled with g++ (fp64), against torch autograd through the
    restatement (which the first test pins to the reference): forward values and the hand-derived adjoint"""
    hdr = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mvsmplfitting_b200", "csrc", "mvs_math.cuh")
    src = tmp_path / "h.cpp"
    src.write_text(HOST_SRC % hdr)
    exe = tmp_path / "h"
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-o", str(exe), str(src)])
    c = np.load(GOLD)
    w = S.make_vposer(11)
    x6 = VO.decode_6d(w, torch.tensor(c["Z"], dtype=torch.float64)).reshape(-1, 6).clone().requires_grad_(True)
    rng = np.random.RandomState(1)
    daa = rng.normal(size=(x6.shape[0], 3))
    aa = VO.quaternion_to_angle_axis(VO.matrot_to_quaternion(VO.cont6d_to_matrot(x6)))
    (aa * torch.tensor(daa)).sum().backward()
    inp = "\n".join(" ".join("%.17g" % v for v in np.concatenate([x6.detach().numpy()[i], daa[i]])) for i in range(x6.shape[0]))
    out = subprocess.run([str(exe)], input=inp, capture_output=True, text=True, check=True).stdout
    res = np.array([[float(v) for v in line.split()] for line in out.strip().splitlines()])
    assert np.abs(res[:, :3] - aa.detach().numpy()).max() < 1e-11
    assert np.abs(res[:, 3:9] - x6.grad.numpy()).max() < 1e-9 * max(1.0, np.abs(x6.grad.numpy()).max())
    assert set(res[:, 9].astype(int).tolist()) == {0, 1, 2, 3}


REAL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vposer_real.npz")


def _real_weights():
    """decoder weights of the snapshot the original project ships (priors/snapshots/poser_epoch091.pkl)"""
    return G.snapshot_vposer_weights()


def test_shipped_snapshot_known_answer_and_restatement(syn_model):
    """SURVEY 8c: decode(0) of the shipped snapshot has max |axis-angle| = 0.8225; restatement + oracle closure with the real
    weights against the unmodified reference class / closure (fixture vposer_real.npz)."""
    c = np.load(REAL)
    assert (c["Z"][0] == 0).all() and abs(np.abs(c["aa_f32"][0]).max() - 0.8225) < 1e-4
    w = _real_weights()
    aa = VO.decode_aa(w, torch.tensor(c["Z"], dtype=torch.float64)).numpy()
    assert np.abs(aa - c["aa_f64"]).max() < 1e-10 * max(1.0, np.abs(c["aa_f64"]).max())
    assert abs(np.abs(aa[0]).max() - 0.8225) < 1e-4
    cams = dict(R=c["cam_R"], t=c["cam_t"], f=c["cam_f"], c=c["cam_c"])
    dw, bpw, sw, bend = [float(v) for v in c["w3"]]
    om = O.OracleModel.from_numpy(syn_model, dtype=torch.float64)
    cfg = O.LossConfig(data_weight=dw, body_pose_weight=bpw, shape_weight=sw, bending_prior_weight=bend, use_vposer=True)
    for b in range(2):
        r = O.closure_eval_vposer(om, cfg, O.OraclePriors(kind="l2"), O.cams_to_torch(cams, torch.float64), c["X"][b],
                                  c["closure_Z"][b], w, c["gt_uv"][:, b], c["conf"][:, b], c["joint_weights"])
        pre = "s3_b%d_f64_" % b
        assert abs(r["loss"] - float(c[pre + "loss"])) / abs(float(c[pre + "loss"])) < 1e-9
        for k in ("betas", "global_orient", "transl", "scale", "pose_embedding"):
            assert G.relmax(r["g_" + k], c[pre + "g_" + k]) < 1e-9, (b, k)
