"""GPU: bitwise pin of the two alternating solves -- mvs_fit_shared_shape on the 'gmm', 'vposer' and 'scale' cases of
tests/test_gpu_shared_shape.py through a 2-slot context (three sequences: the shape step runs in two chunks; 'gmm' with two
sweeps), mvs_refine_cameras on the 1/2/8/16-view rigs of tests/test_gpu_camera_refine.py with 16 slots (23 view problems: two
chunks) and one frame whose row is not finite, and the two debug closures at fixed rows.  The fixture
(golden/alternating_pin.npz) was written by scripts/make_alternating_pin.py on an H100; any change of a floating-point
operation or of its order in the shape or camera closure, their per-problem reductions, the optimiser or the body refit shows
up as a bit difference in the rows, losses, cameras or gradients, or as different counts."""
import os

import numpy as np
import pytest

from tests import test_gpu_camera_refine as CR
from tests import test_gpu_shared_shape as SS

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "alternating_pin.npz")
SHAPE_SLOTS = 2
SWEEPS = dict(gmm=2, vposer=1, scale=1)
STATS = ("frame_iterations", "frame_evals", "rounds", "frames_nan", "dense_frame_evals", "dense_rounds")
CASES = tuple("shape_" + k for k in SS.KINDS) + ("camera", "shape_closure", "camera_closure")


def stats(st):
    return np.array([st[k] for k in STATS], dtype=np.int64)


def shape_case(kind, model, gmm):
    d = SS.make_case(model, kind)
    x, final, seq_loss, sh, po = SS.run(model, gmm, d, Bc=SHAPE_SLOTS, sweeps=SWEEPS[kind])
    return dict(x=x, final=final, seq_loss=seq_loss, shape_stats=stats(sh), pose_stats=stats(po))


def camera_data(model):
    cams = CR.specs_cams()
    return CR.make_case(model, cams, [CR.perturb(c, 10 + i) for i, c in enumerate(cams)], CR.RIG12)


def camera_case(model, gmm):
    d = camera_data(model)
    d["x0"][5, 20] = np.nan                                      # a frame without a finite row takes no part
    x, final, rigs, ca, po = CR.refine(model, gmm, d, B=16, scales=CR.specs_scales())
    return dict(x=x, final=final, R=np.concatenate([r["R"] for r in rigs]), t=np.concatenate([r["t"] for r in rigs]),
                camera_stats=stats(ca), pose_stats=stats(po))


def shape_closure_case(model, gmm):
    out = {}
    for kind in SS.KINDS:
        d = SS.make_case(model, kind)
        rows = SS.consensus(d)
        rows[:, :10] += np.float32(0.05)
        out[kind + "_loss"], out[kind + "_grad"] = SS.debug_shape_closure(model, gmm, d, rows)
    return out


def camera_closure_case(model, gmm):
    keys = [(r, v) for r, (V, *_) in enumerate(CR.SPECS) for v in range(1, V)]
    probs, loss, grad = CR.debug_closure(model, gmm, camera_data(model), lambda P: CR.random_rows(P, 5, lambda p: keys[p][1] == 1),
                                         CR.specs_scales())
    assert probs == keys
    return dict(loss=loss, grad=grad)


def run_case(name, model, gmm):
    """-> dict of arrays pinned for case `name`"""
    if name.startswith("shape_") and name != "shape_closure":
        return shape_case(name[len("shape_"):], model, gmm)
    return dict(camera=camera_case, shape_closure=shape_closure_case, camera_closure=camera_closure_case)[name](model, gmm)


@pytest.mark.parametrize("name", CASES)
def test_alternating_solves_bitwise(name, syn_model, syn_gmm):
    g = np.load(GOLD)
    r = run_case(name, syn_model, syn_gmm)
    assert sorted(r) == sorted(k.split("/", 1)[1] for k in g.files if k.startswith(name + "/"))
    for k, v in r.items():
        assert np.array_equal(v, g[name + "/" + k], equal_nan=True), (k, v, g[name + "/" + k])
