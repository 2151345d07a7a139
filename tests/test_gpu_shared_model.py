"""GPU: contexts that upload the same model constants share one device copy of them (mvs_set_model, mvs_set_gmm_prior,
mvs_set_vposer).  Sharing is seen through the device's free memory; a context given other constants gets its own copy; the
last context out frees the copy; concurrent uploads of one model make one copy; and a fit is bit for bit the same whether its
context shares the constants, owns them (MVS_SHARE_MODEL=0) or outlived the context that uploaded them.  The fits run the
benchmark's workload (4-stage schedule, GMM prior, SDF term in stages 2-3) at 16 frames."""
import importlib.util
import os
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu
B = 16
MB = 1 << 20
QK_BYTES = 6890 * 3 * 224 * 4          # the posedirs table of the synthetic model alone: 18.5 MB


def _stage_table():
    spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m.stage_table()


class Workload:
    def __init__(self, seed=1000):
        from mvsmplfitting_b200 import synthetic as S
        self.model = S.make_model(0)
        self.gmm = S.make_gmm(7)
        self.cams = S.make_cameras(8)
        self.fr = S.make_frames(self.model, self.cams, B, seed=seed)
        self.X0 = S.pack_params(self.fr["init"])
        self.stages = _stage_table()

    def context(self, model_bytes=None):
        """a context set up for the workload; model_bytes (a list): gets the device memory mvs_set_model took"""
        from mvsmplfitting_b200.context import FittingContext
        ctx = FittingContext(0)
        u0 = _used() if model_bytes is not None else 0
        ctx.set_model(self.model)
        if model_bytes is not None:
            model_bytes.append(_used() - u0)
        ctx.set_gmm_from_dict(self.gmm)
        ctx.set_cameras(self.cams["R"], self.cams["t"], self.cams["f"], self.cams["c"])
        ctx.set_batch(B)
        ctx.set_keypoints(self.fr["gt_uv"], self.fr["conf"], self.fr["joint_weights"])
        return ctx

    def fit(self, ctx):
        """-> the fitted rows and final losses as raw bytes, and the counts of mvs_fit"""
        import torch
        stages = [ctx.make_loss_config(body_prior="gmm", interpenetration=True, sdf_grid=128, **st) for st in self.stages]
        x = torch.tensor(self.X0, device="cuda")
        final, st = ctx.fit(x, stages, ctx.make_lbfgs_config())
        torch.cuda.synchronize()
        return dict(params=x.cpu().numpy().tobytes(), final=final.cpu().numpy().tobytes(),
                    frame_iterations=st["frame_iterations"], rounds=st["rounds"], dense_rounds=st["dense_rounds"])


def _used():
    import torch
    torch.cuda.synchronize()
    free, total = torch.cuda.mem_get_info()
    return total - free


def _perturbed(model):
    m = dict(model)
    pd = np.array(model["posedirs"], dtype=np.float32, copy=True)
    pd.reshape(-1)[12345] += 1e-3
    m["posedirs"] = pd
    return m


@pytest.fixture(scope="module")
def wl():
    import torch
    torch.cuda.init()
    return Workload()


@pytest.fixture(scope="module")
def reference(wl):
    ctx = wl.context()
    r = wl.fit(ctx)
    ctx.close()
    return r


def test_same_model_shares_one_copy(wl):
    from mvsmplfitting_b200.context import FittingContext
    keep = wl.context()                                    # holds the model's entry and warms the allocator
    other = _perturbed(wl.model)
    deltas = {}
    for name, model in (("perturbed", other), ("perturbed_again", other), ("same", wl.model)):
        u0 = _used()
        c = FittingContext(0)
        c.set_model(model)
        deltas[name] = _used() - u0
        deltas[name + "_ctx"] = c
    # a new model costs at least its posedirs table; a model already on the device costs only per-context state
    assert deltas["perturbed"] >= QK_BYTES, deltas
    assert deltas["perturbed_again"] < 4 * MB and deltas["same"] < 4 * MB, deltas
    u0 = _used()
    deltas["perturbed_ctx"].close()                        # one holder of the perturbed copy is left
    assert u0 - _used() < 4 * MB
    u0 = _used()
    deltas["perturbed_again_ctx"].close()                  # the last holder frees it
    assert u0 - _used() >= QK_BYTES
    deltas["same_ctx"].close()
    keep.close()


def test_fit_after_the_uploading_context_is_gone(wl, reference):
    first, second = wl.context(), wl.context()
    first.close()
    r = wl.fit(second)
    second.close()
    assert r == reference


def test_concurrent_set_model_makes_one_copy(wl, reference):
    n = 8
    u0 = _used()
    ctxs = [wl.context() for _ in range(n)]                 # one after the other: one copy of the constants
    sequential = _used() - u0
    for c in ctxs:
        c.close()
    ctxs, errs = [None] * n, []
    go = threading.Barrier(n)

    def make(i):
        try:
            go.wait()
            ctxs[i] = wl.context()
        except Exception as e:                             # noqa: BLE001 -- re-raised below
            errs.append(e)

    u0 = _used()
    th = [threading.Thread(target=make, args=(i,)) for i in range(n)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    concurrent = _used() - u0
    # a second copy would add at least another posedirs table
    assert abs(concurrent - sequential) < QK_BYTES // 2, (concurrent, sequential)
    for c in ctxs:
        assert wl.fit(c) == reference
        c.close()


def test_close_during_another_fit(wl, reference):
    a, b = wl.context(), wl.context()
    out = {}
    t = threading.Thread(target=lambda: out.update(r=wl.fit(b)))
    t.start()
    time.sleep(0.005)
    a.close()
    t.join()
    b.close()
    assert out["r"] == reference


def _worker(path):
    """two contexts of one model fit the workload one after the other; their results and the device memory the second
    context's mvs_set_model took go to path"""
    import torch
    torch.cuda.init()
    wl = Workload()
    second = []
    c1, c2 = wl.context(), wl.context(second)
    r1, r2 = wl.fit(c1), wl.fit(c2)
    c1.close()
    c2.close()
    np.savez(path, second=np.int64(second[0]), **{"%s_%d" % (k, i): np.frombuffer(v, np.uint8) if isinstance(v, bytes) else np.int64(v)
                                               for i, r in enumerate((r1, r2)) for k, v in r.items()})


@pytest.mark.parametrize("share", ["0", "1"])
def test_share_off_and_on_fit_the_same_bits(reference, share, tmp_path):
    path = str(tmp_path / "out.npz")
    env = dict(os.environ, MVS_SHARE_MODEL=share)
    subprocess.run([sys.executable, os.path.abspath(__file__), path], env=env, check=True, cwd=ROOT, timeout=600)
    z = np.load(path)
    second = int(z["second"])
    assert second >= QK_BYTES if share == "0" else second < 4 * MB, second
    for i in range(2):
        for k, v in reference.items():
            got = z["%s_%d" % (k, i)]
            assert (got.tobytes() if isinstance(v, bytes) else int(got)) == v, (share, i, k)


if __name__ == "__main__":
    _worker(sys.argv[1])
