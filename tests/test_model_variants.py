"""CPU: the model, prior and keypoint-set variants of tests/model_variants.py sit on the intended side of every limit of the
frame-resident kernels, with the limits read from the CUDA headers -- so a changed limit makes these fixtures fail loudly
instead of quietly no longer reaching the branch they were built for.  Also: the oracle's keypoint-set options."""
import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import synthetic as S
from oracle import closure_oracle as O
from tests import model_variants as MV

# name -> (model variant, model_type, keypoint set, views, GMM components, expected branches)
IN, OUT = True, False
CASES = dict(
    base=(None, "smpllsp", None, 4, 6, dict(resident=IN, kp_on=IN, sj_on=IN, ell_smem=IN)),
    gmm1=(None, "smpllsp", None, 4, 1, dict(resident=IN)),
    gmm8=(None, "smpllsp", None, 4, 8, dict(resident=IN)),
    gmm9=(None, "smpllsp", None, 4, 9, dict(resident=OUT)),
    sup86=("sup86", "smpllsp", None, 4, 6, dict(resident=IN, kp_on=IN, sj_on=IN)),
    sup90=("sup90", "smpllsp", None, 4, 6, dict(resident=IN, kp_on=IN, sj_on=IN)),
    sup91=("sup91", "smpllsp", None, 4, 6, dict(resident=OUT)),
    kpe_wide=("kpe_wide", "smpllsp", None, 4, 6, dict(resident=IN, kp_on=OUT, sj_on=IN)),
    skin_dense=("skin_dense", "smpllsp", None, 4, 6, dict(resident=IN, kp_on=IN, sj_on=OUT, ell_smem=IN)),
    skin_kw9=("skin_kw9", "smpllsp", None, 4, 6, dict(resident=IN, kp_on=IN, sj_on=IN, ell_smem=OUT)),
    K18_V15=(None, "smpllsp", "K18", 15, 6, dict(resident=IN)),
    K18_V16=(None, "smpllsp", "K18", 16, 6, dict(resident=OUT)),
    K32_V8=(None, "smpllsp", "K32", 8, 6, dict(resident=IN)),
    K32_V9=(None, "smpllsp", "K32", 9, 6, dict(resident=OUT)),
    V16_smpl=(None, "smpl", None, 16, 6, dict(resident=IN)),
)


@pytest.fixture(scope="module")
def lim():
    return MV.limits()


def test_limits_are_read_from_the_headers(lim):
    for k in ("kResMaxSup", "kResMaxSupJ", "kResMaxVK", "kResMaxM", "kResMaxKpE", "kSkinEllMax", "kMaxKeypoints",
              "kMaxViews", "kResExtraSup"):
        assert k in lim and lim[k] > 0, k


@pytest.mark.parametrize("name", list(CASES))
def test_variant_sits_on_its_side_of_each_limit(name, lim, syn_model):
    variant, model_type, jmap, V, M, want = CASES[name]
    m = MV.make_variant(variant, syn_model)
    bk = MV.bookkeeping(m, model_type, **(MV.KEYPOINT_SETS[jmap] if jmap else {}))
    got = MV.branches(bk, V, M, lim)
    for k, v in want.items():
        assert got[k] == v, (name, k, bk["nsup"], bk["nkpe"], bk["nsupj"], bk["KW"], V * bk["K"], M)
    # each variant is AT its limit: one more (or one fewer) and it would be on the other side
    if name in ("sup90", "sup91"):
        assert bk["nsup"] + lim["kResExtraSup"] == lim["kResMaxSup"] + (name == "sup91")
    if name == "sup86":
        assert bk["nsup"] == 86
    if name.startswith("gmm"):
        assert abs(M - lim["kResMaxM"]) <= 1 or M == 1
    if jmap:
        assert V * bk["K"] in (lim["kResMaxVK"] - 2, lim["kResMaxVK"] - 16, lim["kResMaxVK"] + 16)
    if name == "V16_smpl":
        assert V * bk["K"] == lim["kResMaxVK"] and V == lim["kMaxViews"]
    if name == "kpe_wide":
        assert bk["nkpe"] > lim["kResMaxKpE"] and bk["nsup"] + lim["kResExtraSup"] <= lim["kResMaxSup"]
    if name == "skin_dense":
        assert bk["KW"] == lim["kSkinEllMax"]
    if name == "skin_kw9":
        assert bk["KW"] == lim["kSkinEllMax"] + 1


@pytest.mark.parametrize("variant", ["sup86", "sup90", "sup91", "kpe_wide", "skin_dense", "skin_kw9"])
def test_variant_rows_stay_normalised_and_local(variant, syn_model):
    m = MV.make_variant(variant, syn_model)
    reg, W = np.asarray(m["lsp_regressor"]), np.asarray(m["weights"])
    assert (reg >= 0).all() and (W >= 0).all()
    assert np.abs(reg[MV.LSP_ROWS].sum(1) - 1).max() < 1e-5
    assert np.abs(W.sum(1) - 1).max() < 1e-5
    # the replaced rows regress keypoints within a few centimetres (model units) of where the original rows put them
    vt = np.asarray(syn_model["v_template"], dtype=np.float64)
    moved = np.linalg.norm((reg[MV.LSP_ROWS] - syn_model["lsp_regressor"][MV.LSP_ROWS]) @ vt, axis=1)
    assert moved.max() < 0.03, moved
    # everything else is the base model
    for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "f"):
        assert m[k] is syn_model[k]


def test_oracle_keypoint_set_defaults_are_the_reference_maps(syn_model):
    x = S.pack_params(S.make_frames(syn_model, S.make_cameras(2), 1, seed=3)["gt"])[0]
    parts = [torch.tensor(x[a:a + n], dtype=torch.float64).view(1, n) for a, n in zip(np.cumsum((0,) + O.PARAM_SIZES[:-1]),
                                                                                      O.PARAM_SIZES)]
    for model_type, jmap in (("smpllsp", O.MAP_LSP14), ("smpl", O.MAP_COCO17)):
        d = O.OracleModel.from_numpy(syn_model, dtype=torch.float64, model_type=model_type)
        e = O.OracleModel.from_numpy(syn_model, dtype=torch.float64, model_type=model_type, joint_map=jmap,
                                     extra_vertex_ids=O.FACE_IDS)
        assert torch.equal(O.smpl_forward(d, *parts)[1], O.smpl_forward(e, *parts)[1])
    # a custom set: keypoint k is source joint_map[k] of [regressor rows | extra vertices]
    ks = MV.KEYPOINT_SETS["K32"]
    om = O.OracleModel.from_numpy(syn_model, dtype=torch.float64, **ks)
    v, j, _ = O.smpl_forward(om, *parts)
    reg = torch.tensor(np.asarray(syn_model["lsp_regressor"], dtype=np.float64))
    src = torch.cat([reg @ (v - parts[3]), v[list(ks["extra_vertex_ids"])] - parts[3]])
    assert j.shape == (32, 3)
    assert torch.allclose(j, src[list(ks["joint_map"])] + parts[3], rtol=0, atol=1e-12)
