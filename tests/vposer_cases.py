"""Frames and latent codes for the float64 checks of the VPoser latent pose (tests/test_gpu_vposer_parity.py).  Built
without a GPU, so that tests/test_vposer_parity_cases.py can check on the CPU what the GPU tests rely on.

Every frame of a case carries a latent code z in the first 32 entries of its pose slot (use_vposer = 2) and zeros in the
other 37.  The codes are drawn at scales 0.3, 1, 2 and 4 (by frame) and kept only where, for the decoder of the case, every
one of the 23 decoded joint rotations lies

* at least BRANCH_MARGIN from each surface where rotation_matrix_to_quaternion decides its formula (m22 = eps, and
  m00 = m11 or m00 = -m11 on the side of it the rotation is on): a float32 decode picks the same branch as the float64 one;
* at least PI_MARGIN from an angle of pi, where quaternion_to_angle_axis flips the axis;
* where the decode is well conditioned: the float32 decode (the oracle's, on the CPU) within DECODE32_MARGIN of the float64
  one.  Codes whose 6-D columns come out short or nearly parallel amplify float32 rounding (one such frame of the first
  draw decoded 1.6e-5 off in float32), and would measure float32 rather than the kernels;

and where the bending term bend * sum exp(+-pose)^2 of every stage-weight set lies at least GATE_MARGIN (relative) from the
1e4 cut-off that the axis-angle pose applies (fitting.py:349-350) and the latent pose must not.  With the synthetic decoder
the codes are steered to both sides of that cut-off at body_pose_weight 57.4, alternating every four frames.

The decoders: "synthetic" (synthetic.make_vposer(11), which reaches all four quaternion branches) and "snapshot" (the
decoder of the VPoser snapshot the original project ships, whose rotations nearly all fall in branch 3).  Both are float32
weights, which the float64 oracle widens exactly.
"""
import functools

import numpy as np
import torch

from mvsmplfitting_b200 import synthetic as S
from oracle import vposer_oracle as VO
from tests import golden_util as G

POOL = 257                         # frames of a case: the largest batch of test_gpu_dense_parity.BATCHES
SCALES = (0.3, 1.0, 2.0, 4.0)      # latent scale of frame i: SCALES[i % 4]
BRANCH_MARGIN = 1e-3
PI_MARGIN = 1e-2
ANGLE_CUT = 1e4                    # fitting.py:349-350
GATE_MARGIN = 1e-3                 # as test_gpu_dense_parity.GATE_MARGIN
ANGLE_IDX, ANGLE_SIGN = (52, 55, 9, 12), (1.0, -1.0, -1.0, -1.0)     # prior.py:62-66,87
DECODERS = ("synthetic", "snapshot")
DECODE32_MARGIN = 2e-6            # largest |float32 decode - float64 decode| of a kept code (axis-angle entries)
CANDIDATES = 256                   # codes drawn per frame; the first that meets the margins is kept


def stage_weights():
    """the stage weights of the VPoser fixtures (first and last stage of cfg_files/fit_smpl.yaml), and the stage-2
    weights (body_pose_weight 57.4, bending 182) at which the synthetic decoder's poses straddle the bending cut-off"""
    c = np.load(G.GOLD + "/vposer_s11.npz")
    as_dict = lambda w: dict(data_weight=float(w[0]), body_pose_weight=float(w[1]), shape_weight=float(w[2]),
                             bending_prior_weight=float(w[3]))
    return dict(w0=as_dict(c["w0"]), w3=as_dict(c["w3"]),
                s2=dict(data_weight=500.0 / 1536, body_pose_weight=57.4, shape_weight=10.0, bending_prior_weight=3.17 * 57.4))


@functools.lru_cache(maxsize=None)
def decoder_weights(name):
    w = S.make_vposer(11) if name == "synthetic" else G.snapshot_vposer_weights()
    return {k: np.asarray(v, np.float32) for k, v in w.items()}


def decode64(w, Z):
    """decode(z, 'aa') in float64 of the float32 codes Z [n, 32] -> [n, 69]"""
    with torch.no_grad():
        return VO.decode_aa(w, torch.tensor(np.asarray(Z, np.float32).astype(np.float64))).numpy()


def angle_sum(pose):
    """sum_j exp(sign_j pose_j)^2 over the bending entries (prior.py:87-89): the bending term over its weight"""
    pose = np.atleast_2d(pose)
    return sum(np.exp(pose[:, j] * s) ** 2 for j, s in zip(ANGLE_IDX, ANGLE_SIGN))


def _margins_ok(w, Z):
    """per code: every rotation clear of the branch surfaces and of pi, a well-conditioned decode, and every weight set's
    bending term clear of 1e4"""
    with torch.no_grad():
        r = VO.rotation_branches(w, Z.astype(np.float64))
    ok = (r["margin"].min(axis=1) > BRANCH_MARGIN) & ((np.pi - r["angle"]).min(axis=1) > PI_MARGIN)
    pose = decode64(w, Z)
    with torch.no_grad():
        pose32 = VO.decode_aa(w, torch.tensor(np.asarray(Z, np.float32))).numpy()
    ok &= np.abs(pose32 - pose).max(axis=1) < DECODE32_MARGIN
    a = angle_sum(pose)
    for sw in stage_weights().values():
        ok &= np.abs(sw["bending_prior_weight"] * a / ANGLE_CUT - 1.0) > GATE_MARGIN
    return ok, a


def _want_above(i):
    """synthetic decoder: frame i is steered above the bending cut-off at body_pose_weight 57.4 in alternate groups of four
    frames (its scale 0.3 frame cannot get there)"""
    return (i // 4) % 2 == 1 and SCALES[i % 4] >= 1.0


@functools.lru_cache(maxsize=None)
def latent_codes(decoder, n=POOL, seed=905):
    """Z [n, 32] float32"""
    w = decoder_weights(decoder)
    bend = stage_weights()["s2"]["bending_prior_weight"]
    rng = np.random.RandomState(seed + DECODERS.index(decoder))
    Z = np.zeros((n, 32), np.float32)
    for i in range(n):
        cand = (rng.normal(size=(CANDIDATES, 32)) * SCALES[i % 4]).astype(np.float32)
        ok, a = _margins_ok(w, cand)
        if decoder == "synthetic":
            side = (bend * a > ANGLE_CUT) == _want_above(i)
            ok = ok & side if (ok & side).any() else ok
        assert ok.any(), (decoder, i)
        Z[i] = cand[np.flatnonzero(ok)[0]]
    return Z


@functools.lru_cache(maxsize=None)
def _frames(V, n, seed):
    model = S.make_model(0)
    cams = S.make_cameras(V)
    fr = S.make_frames(model, cams, n, seed=seed)
    rng = np.random.RandomState(seed + 1)
    X = S.pack_params(fr["init"])
    X[:, 0:10] = 0.5 * fr["gt"]["betas"]
    X[:, 85] = rng.uniform(0.9, 1.1, n)
    X[:, 13:82] = 0.0
    return cams, fr, X.astype(np.float32)


def make_case(decoder, V=4, n=POOL, seed=930):
    """frames, cameras, parameters X [n, 86] (latent code in X[:, 13:45]), the codes Z, the float64 decoded pose and the
    decoder weights of one case.  Frame i is the same frame in every case of the same V."""
    cams, fr, X = _frames(V, n, seed)
    Z = latent_codes(decoder)[:n]
    X = X.copy()
    X[:, 13:45] = Z
    w = decoder_weights(decoder)
    return dict(decoder=decoder, V=V, cams=cams, fr=fr, X=X, Z=Z, w=w, pose=decode64(w, Z))
