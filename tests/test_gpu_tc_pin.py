"""GPU: bitwise pin of the two tensor-core contractions of mvs_tc.cu -- posedirs_gemm_tc_kernel through the vertices of
mvs_forward, and vertex_bwd_tc_kernel through the dparams of mvs_forward_vjp (vertex cotangents alone and with joint
cotangents, both model types), in exec mode 0.  The batch sizes cover every wgmma N instance of each kernel at both ends of
its range and several column tiles: 1 .. 256 frames forward (instances 8 .. 128, a second 128-frame tile), 1 .. 256 frames
through the VJP (instances 8 .. 64, several 64-frame tiles).  The fixture (golden/tc_pin.npz) was written by
scripts/make_tc_pin.py on an H100.  It holds one 16-byte BLAKE2b digest of each frame's output bits (a batch of vertices is
5.3 MB per 64 frames), so any change of a floating-point operation or of its order in either contraction, or in the ring
that feeds it, shows up as a differing frame."""
import hashlib
import os

import numpy as np
import pytest
import torch

from tests import test_gpu_forward_vjp as V

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tc_pin.npz")
CASES = ("forward", "vjp_smpllsp", "vjp_smpl")
FWD_BATCHES = (1, 9, 17, 33, 65, 129, 256)
VJP_BATCHES = (1, 8, 9, 16, 17, 32, 33, 64, 65, 256)
KINDS = ("verts", "both")


def digests(a):
    """[B, 16] uint8: one BLAKE2b digest per frame of a float32 array [B, ...], over its bits"""
    rows = np.ascontiguousarray(a, dtype=np.float32).reshape(len(a), -1).view(np.uint32)
    return np.stack([np.frombuffer(hashlib.blake2b(r.tobytes(), digest_size=16).digest(), np.uint8) for r in rows])


def run_case(name, model):
    """-> dict of per-frame digests pinned for case `name`"""
    X = V.make_params()
    out = {}
    if name == "forward":
        for B in FWD_BATCHES:
            ctx = V.make_ctx(model, B, "smpllsp")
            out["B%d" % B] = digests(ctx.forward_only(torch.tensor(X[:B], device="cuda"))["verts"].cpu().numpy())
            ctx.close()
        return out
    model_type = name.split("_", 1)[1]
    for B in VJP_BATCHES:
        ctx = V.make_ctx(model, B, model_type)
        gv, gj = V.cotangents(ctx.N, ctx.K)
        x = torch.tensor(X[:B], device="cuda")
        gv, gj = torch.tensor(gv[:B], device="cuda"), torch.tensor(gj[:B], device="cuda")
        for kind in KINDS:
            d = ctx.forward_vjp(x, djoints=gj if kind == "both" else None, dverts=gv)
            out["B%d_%s" % (B, kind)] = digests(d.cpu().numpy())
        ctx.close()
    return out


@pytest.mark.parametrize("name", CASES)
def test_tensor_core_contractions_bitwise(name, syn_model):
    g = np.load(GOLD)
    r = run_case(name, syn_model)
    assert sorted(r) == sorted(k.split("/", 1)[1] for k in g.files if k.startswith(name + "/"))
    for k, v in r.items():
        want = g[name + "/" + k]
        assert v.shape == want.shape and np.array_equal(v, want), (name, k, np.flatnonzero((v != want).any(1)))
