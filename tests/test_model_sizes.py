"""CPU: the meshes of tests/model_variants.py make_sized_model sit on their intended side of every vertex-count-dependent
tiling constant of the dense kernels, with the constants read from the CUDA sources, so that a changed constant fails here
instead of quietly leaving tests/test_gpu_model_sizes.py short of the branch a size was chosen for.  Also: the builder's
mesh and rows are sound, and the preconditions the GPU assertions rely on hold in the float64 oracle."""
import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from oracle import sdf_oracle
from tests import model_variants as MV


@pytest.fixture(scope="module")
def lim():
    return MV.limits()


def test_tiling_constants_are_read_from_the_sources(lim):
    want = dict(kTcRows=128, kSkinV=64, kTbRows=32, kSdfFThreads=256, kTileV=32, kSdfSkipWords=8, kBinCapD=1 << 17,
                kBinCapR=1 << 18, kSetupCh=4, kFlagList=64)
    assert {k: lim.get(k) for k in want} == want


# N -> what it must reach; tails() keys
REACH = {
    431: dict(tc_tiles=11, nbox=7, sdf_blocks=2),
    1723: dict(nbox=27, sdf_blocks=7),
    6890: dict(tc_last_rows=62, tc_last_wg1_rows=0, nbox=108, sdf_blocks=27, tb_pad=2, setup_groups=1),
    6912: dict(tc_last_rows=128, chunk_tail=0, block_tail=0, simt_tail=0, tb_pad=0),
    6913: dict(tc_last_rows=3, chunk_tail=1, block_tail=1, simt_tail=1, sdf_blocks=28),
    6944: dict(tc_last_rows=96, tc_last_wg1_rows=32),
    10475: dict(nbox=164, setup_groups=2, cull=True),
    27554: dict(nbox=431, cull=False, sdf_blocks=108, tc_tiles=646),
}


@pytest.mark.parametrize("N", MV.SIZES)
def test_size_sits_on_its_side_of_each_constant(N, lim):
    t = MV.tails(N, lim)
    for k, v in REACH[N].items():
        assert t[k] == v, (N, k, t[k], v)
    sm_h100 = 132
    if N == 431:
        assert t["tc_tiles"] < sm_h100 and t["nbox"] < 32
    if N == 1723:
        assert t["sdf_blocks"] < 8                               # frame_step's serial_sum8: one partial group of 8
    if N == 10475:
        assert 4 * 32 < t["nbox"] <= 32 * lim["kSdfSkipWords"]   # cull words 4-7 hold chunks; the fold loop runs twice
    if N == 27554:
        assert t["sdf_blocks"] > lim["kFlagList"]                # more blocks than frame_step's list holds
        assert -(-t["tc_tiles"] // sm_h100) == 5
    if N == 6912:
        assert (3 * N) % lim["kTcRows"] == 0 and N % lim["kSkinV"] == 0 and (3 * N) % lim["kTbRows"] == 0


@pytest.mark.parametrize("N", MV.SIZES + (32772,))
def test_sized_model_is_sound(N, lim):
    m, extra = MV.make_sized_model(N)
    f = m["f"].astype(np.int64)
    assert m["v_template"].shape == (N, 3) and f.shape == (2 * N - 4, 3)
    assert f.min() >= 0 and f.max() < N
    # closed and consistently oriented: every directed edge appears once, its reverse once
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key = e[:, 0] * N + e[:, 1]
    assert len(np.unique(key)) == len(key)
    assert np.array_equal(np.sort(key), np.sort(e[:, 1] * N + e[:, 0]))
    vt = m["v_template"].astype(np.float64)
    a, b, c = vt[f[:, 0]], vt[f[:, 1]], vt[f[:, 2]]
    assert (np.einsum("ij,ij->i", np.cross(b - a, c - a), a + b + c) > 0).all()           # outward
    for k in ("J_regressor", "weights"):
        assert (m[k] >= 0).all()
    assert np.abs(m["J_regressor"].sum(1) - 1).max() < 1e-5 and np.abs(m["weights"].sum(1) - 1).max() < 1e-5
    assert (m["weights"] != 0).sum(1).max() <= 4
    reg = m["lsp_regressor"]
    assert (reg >= 0).all() and np.abs(reg[MV.LSP_ROWS].sum(1) - 1).max() < 1e-5
    assert len(extra) == 5 and all(0 <= v < N for v in extra)
    bk = MV.bookkeeping(m, extra_vertex_ids=extra)
    assert bk["nsup"] + lim["kResExtraSup"] <= lim["kResMaxSup"]
    assert MV.branches(bk, 4, 6, lim) == dict(resident=True, kp_on=True, sj_on=True, ell_smem=True)
    if N > 65535 // 2:
        assert f.shape[0] > 65535                               # past the accelerated all-faces SDF's face limit


def test_sized_model_at_6890_is_make_model_geometry(syn_model):
    m, extra = MV.make_sized_model(6890)
    for k in ("v_template", "f", "shapedirs", "posedirs", "J_regressor", "weights"):
        assert np.array_equal(m[k], syn_model[k]), k
    assert extra == tuple(int(v) for v in S.FACE_VERTEX_IDS)


def _pen_grad_rows(N, sc, frames):
    """per checked frame: the vertices with a non-zero float64 penetration gradient (the GPU test's frames)"""
    from tests import test_gpu_model_sizes as T
    cams = S.make_cameras(4)
    fr = T.sized_frames(N, cams, max(T.D_BATCHES), 820)
    X = T.closure_params(fr, max(T.D_BATCHES), 821)
    om = T.sized_oracle(N)
    out = {}
    for i in frames:
        v = torch.tensor(T.fwd64(om, X[i])[0], requires_grad=True)
        sdf_oracle.penetration_loss(v, om.faces, sc["coll_loss_weight"], sc["sdf_grid"], bool(sc["sdf_all_faces"])).backward()
        out[i] = np.flatnonzero((v.grad.numpy() != 0).any(1))
    return out


def test_all_faces_frame_at_27554_flags_more_blocks_than_frame_steps_list(lim):
    from tests import test_gpu_model_sizes as T
    rows = _pen_grad_rows(27554, T.SDF_CASES["all_faces"], (0, 1))
    nfl = {i: len(np.unique(r // lim["kSdfFThreads"])) for i, r in rows.items()}
    print("flagged blocks at 27554, all faces:", nfl)
    assert max(nfl.values()) > lim["kFlagList"], nfl


def test_as_written_frame_at_10475_samples_past_chunk_128(lim):
    from tests import test_gpu_model_sizes as T
    rows = _pen_grad_rows(10475, T.SDF_CASES["as_written"], T.D_CHECK)
    past = {i: int((r // lim["kSkinV"] >= 128).sum()) for i, r in rows.items()}
    print("vertices with a penetration gradient in chunks >= 128 at 10475:", past)
    assert max(past.values()) > 0, past


def _box_tris(N, X, frames):
    """each frame's triangles in the box coordinates sdf_fused samples in (centre of the vertex box, 0.6 x its largest side)"""
    from tests import test_gpu_model_sizes as T
    om = T.sized_oracle(N)
    f = T.sized(N)[0]["f"].astype(np.int64)
    out = {}
    for i in frames:
        v = T.fwd64(om, X[i])[0].astype(np.float32)
        lo, hi = v.min(0), v.max(0)
        out[i] = ((v - (lo + hi) / np.float32(2)) / (np.float32(0.6) * (hi - lo).max()))[f]
    return out


@pytest.mark.parametrize("N,seed,nf", [(6913, 830, 9), (27554, 830, 9), (27554, 850, 4)])
def test_all_faces_frames_overflow_the_candidate_lists(N, seed, nf, lim):
    """the start frames of the GPU all-faces lbfgs_run (seed 830) and four-stage fit (seed 850): on the host build of
    mvs_sdf_bins.cuh every frame at 27554 vertices overflows kBinCapD or kBinCapR, so sdf_fused<true> falls back to the
    brute force for it; at 6913 some frames overflow and some fit"""
    from tests import hostsim as HS
    from tests import test_gpu_model_sizes as T
    fr = T.sized_frames(N, S.make_cameras(4), nf, seed)
    X = T.closure_params(fr, nf, seed + 1)
    counts = {i: HS.sdf_bin_entries(t) for i, t in _box_tris(N, X, range(nf)).items()}
    print("cell entries, ray entries, overflow at N = %d:" % N, counts)
    for d, r, rc in counts.values():
        assert rc == (1 if d > lim["kBinCapD"] else 2 if r > lim["kBinCapR"] else 0)
    over = [rc != 0 for _, _, rc in counts.values()]
    if N == 27554:
        assert all(over)
    else:
        assert any(over) and not all(over)


def test_penetration_gradient_is_material_at_27554_all_faces():
    """the penetration term's float64 gradient on the compared frames of the GPU all-faces closure at 27554 vertices is many
    times the allowance the GPU comparison grants (bar x largest |entry| + FP32_NOISE x the float32 oracle's deviation), so
    a dropped or doubled block partial fails that comparison"""
    from oracle import closure_oracle as O
    from tests import test_gpu_model_sizes as T
    N, sc = 27554, T.SDF_CASES["all_faces"]
    cams, gmm = S.make_cameras(4), S.make_gmm(7)
    fr = T.sized_frames(N, cams, max(T.D_BATCHES), 820)
    X = T.closure_params(fr, max(T.D_BATCHES), 821)
    on = dict(interpenetration=True, coll_loss_weight=sc["coll_loss_weight"], sdf_grid=sc["sdf_grid"], sdf_all_faces=True, **T.W2)
    ratios = []
    for i in (0, 1):
        kp = (fr["gt_uv"][:, i], fr["conf"][:, i], fr["joint_weights"])
        ev = lambda dt, pri, cfg: O.closure_eval(T.sized_oracle(N, dtype=dt), O.LossConfig(**cfg), pri,
                                                 O.cams_to_torch(cams, dt), X[i], *kp)["grad"]
        g = ev(torch.float64, T.oracle_priors(gmm, "gmm"), on)
        g0 = ev(torch.float64, T.oracle_priors(gmm, "gmm"), T.W2)
        g32 = ev(torch.float32, O.OraclePriors.gmm_from_dict(gmm, torch.float32), on)
        a, e = T.SEGS["body_pose"]
        allow = T.BAR_SDF_GRAD * np.abs(g[a:e]).max() + T.FP32_NOISE * np.abs(g32[a:e] - g[a:e]).max()
        ratios.append(np.abs(g[a:e] - g0[a:e]).max() / allow)
    print("penetration part of the body_pose gradient / allowance at 27554, all faces:", ratios)
    assert min(ratios) > 5, ratios
