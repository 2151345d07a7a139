"""CPU: the camera-file writer and camera_matrices, seqio.fit_sequences / fit_sequence with refine_cameras driving a context as
the camera-refinement contract says (recording stubs), and the ctypes signature of mvs_refine_cameras against include/mvsmpl.h."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import seqio
from mvsmplfitting_b200 import synthetic as S
from tests.test_rig_abi import _code
from tests.test_seqio import _cfgs
from tests.test_seqio_shape import ShapeStub
from tests.test_seqio_temporal import _seq

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEMO = os.path.join(ROOT, "tests", "golden", "demo", "3DOH50K_Parameters.txt")


def _rig(V, seed):
    rng = np.random.RandomState(seed)
    c = S.make_cameras(V)
    c["R"] = (c["R"] + rng.normal(0, 1e-3, c["R"].shape)).astype(np.float32)      # arbitrary float32 bits
    c["t"] = (c["t"] + rng.normal(0, 1e-3, c["t"].shape)).astype(np.float32)
    c["f"] = (c["f"] * rng.uniform(0.9, 1.1, c["f"].shape)).astype(np.float32)
    return {k: c[k] for k in ("R", "t", "f", "c")}


def test_write_then_load_is_bitwise_for_float32(tmp_path):
    cams = _rig(6, 1)
    p = str(tmp_path / "cams.txt")
    seqio.write_camera_para(p, *seqio.camera_matrices(cams))
    back = seqio.camera_arrays(*seqio.load_camera_para(p))
    for k in ("R", "t", "f", "c"):
        assert back[k].dtype == np.float32 and back[k].tobytes() == cams[k].tobytes(), k


def test_layout_is_the_demo_files():
    ext, intr = seqio.load_camera_para(DEMO)
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "cams.txt")
        seqio.write_camera_para(p, ext, intr)
        mine, theirs = open(p).read().splitlines(), open(DEMO).read().splitlines()
    assert len(mine) == len(theirs) == 9 * ext.shape[0]
    for a, b in zip(mine, theirs):                       # the same lines and words; the numbers read back the same
        wa, wb = a.split(), b.split()
        assert len(wa) == len(wb)
        assert [float(x) for x in wa] == [float(x) for x in wb]
    e2, i2 = seqio.load_camera_para(DEMO)
    assert np.array_equal(e2, ext) and np.array_equal(i2, intr)


def test_camera_matrices_inverts_camera_arrays():
    cams = _rig(4, 2)
    ext, intr = seqio.camera_matrices(cams)
    assert ext.shape == (4, 4, 4) and intr.shape == (4, 3, 3)
    assert (ext[:, 3] == [0, 0, 0, 1]).all() and (intr[:, 2] == [0, 0, 1]).all() and (intr[:, 0, 1] == 0).all()
    back = seqio.camera_arrays(ext, intr)
    for k in ("R", "t", "f", "c"):
        assert back[k].tobytes() == cams[k].tobytes(), k
    ext, intr = seqio.load_camera_para(DEMO)
    e2, i2 = seqio.camera_matrices(seqio.camera_arrays(ext, intr))
    assert np.allclose(e2, ext, rtol=1e-6, atol=1e-6) and np.allclose(i2, intr, rtol=1e-6)


RIGS = [_rig(2, 5)]


class CameraStub(ShapeStub):
    """ShapeStub that also records refine_cameras, which adds 100 to every row's transl and returns the table shifted"""

    def refine_cameras(self, params, gt_uv, conf, jw, stage_cfg, opt_cfg=None, sweeps=1, **kw):
        self.calls.append(("camera", params.shape[0], stage_cfg, sweeps, np.asarray(gt_uv).shape, kw))
        params[:, 82:85] += 100
        rigs = [dict(r, t=(r["t"] + 1).astype(np.float32)) for r in RIGS]
        return torch.full((params.shape[0],), 5.0), rigs, dict(frame_iterations=4), dict(frame_iterations=6)


def _names(calls):
    return [c[0] for c in calls]


@pytest.mark.parametrize("B", [2, 1])
def test_off_makes_exactly_todays_calls(B):
    seqs = [_seq(3, "a"), _seq(2, "b")]
    ref, got = CameraStub(B), CameraStub(B)
    r0 = seqio.fit_sequences(ref, seqs, _cfgs(4))
    r1 = seqio.fit_sequences(got, seqs, _cfgs(4), refine_cameras=0)
    assert _names(ref.calls) == _names(got.calls) and "camera" not in _names(got.calls)
    assert all(np.array_equal(a[0], b[0]) for a, b in zip(r0[0], r1[0]))
    assert "refine_cameras" not in r1[1]
    ctx = CameraStub(2)
    seqio.fit_sequence(ctx, _seq(5, "a"), _cfgs(4), refine_cameras=0)
    assert "camera" not in _names(ctx.calls)


@pytest.mark.parametrize("B", [2, 1])
def test_on_adds_one_call_over_all_frames_before_the_shared_shape(B):
    seqs = [_seq(3, "a"), _seq(2, "b")]
    cfgs = _cfgs(4)
    ref, got = CameraStub(B), CameraStub(B)
    seqio.fit_sequences(ref, seqs, cfgs)
    res, stats = seqio.fit_sequences(got, seqs, cfgs, refine_cameras=3, shared_shape=1)
    assert _names(got.calls) == _names(ref.calls) + ["camera", "shape"]
    _, F, cfg, sweeps, shape, kw = got.calls[-2]
    assert F == 5 and cfg is cfgs[-1] and sweeps == 3 and shape == (2, 5, 17, 2) and kw == {}
    for x, loss in res:                                   # the rows the refinement left, then the shared shape
        assert (x[:, 82:85] >= 100).all() and (loss == 7.0).all()
    assert stats["refine_cameras"]["camera"] == dict(frame_iterations=4)
    assert stats["refine_cameras"]["pose"] == dict(frame_iterations=6)
    assert np.array_equal(stats["refine_cameras"]["rigs"][0]["t"], RIGS[0]["t"] + 1)
    only = CameraStub(B)
    res, _ = seqio.fit_sequences(only, seqs, cfgs, refine_cameras=1)
    assert _names(only.calls) == _names(ref.calls) + ["camera"]
    assert all((loss == 5.0).all() for _, loss in res)


def test_fit_sequence_refines_before_the_shared_shape():
    ctx = CameraStub(2)
    x, loss, stats = seqio.fit_sequence(ctx, _seq(5, "a"), _cfgs(4), refine_cameras=2, shared_shape=1)
    names = _names(ctx.calls)
    assert names.count("camera") == 1 and names.index("camera") < names.index("shape")
    assert (x[:, 82:85] >= 100).all() and "refine_cameras" in stats


@pytest.mark.parametrize("bad", [-1, 1.5, True])
def test_bad_sweeps_and_the_temporal_term_are_refused(bad):
    with pytest.raises(ValueError):
        seqio.fit_sequences(CameraStub(2), [_seq(2, "a"), _seq(2, "b")], _cfgs(4), refine_cameras=bad)
    with pytest.raises(ValueError):
        seqio.fit_sequence(CameraStub(2), _seq(2, "a"), _cfgs(4), refine_cameras=bad)
    with pytest.raises(ValueError):
        seqio.fit_sequences(CameraStub(2), [_seq(2, "a"), _seq(2, "b")], _cfgs(4), refine_cameras=1, temporal_weight=1.0)


@pytest.mark.parametrize("B", [2, 1])
def test_result_folder_gets_the_refined_calibration(B, tmp_path):
    ctx = CameraStub(B)
    seqio.fit_sequences(ctx, [_seq(3, "a"), _seq(2, "b")], _cfgs(4), refine_cameras=1, result_folder=str(tmp_path))
    assert len(list(tmp_path.rglob("*.pkl"))) == 5
    back = seqio.camera_arrays(*seqio.load_camera_para(str(tmp_path / "cameras_rig0.txt")))
    assert back["t"].tobytes() == (RIGS[0]["t"] + 1).astype(np.float32).tobytes()
    assert back["R"].tobytes() == RIGS[0]["R"].tobytes()


def test_refine_cameras_entry_point_matches_the_header(tmp_path):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    from mvsmplfitting_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libmvsmpl.so is not built")
    lib = _lib.load()
    src = tmp_path / "probe.cpp"
    lines = ['#include <cstdio>', '#include <string>', '#include <type_traits>', '#include "mvsmpl.h"',
             "template <class T> char code() {",
             "    if (std::is_pointer<T>::value) return 'p';",
             "    if (std::is_same<T, int>::value) return 'i';",
             "    if (std::is_same<T, float>::value) return 'f';",
             "    return '?';", "}",
             "template <class R, class... A> std::string sig(R (*)(A...)) {",
             "    std::string s = std::is_same<R, int>::value ? \"i:\" : \"?:\";",
             "    ((s += code<A>()), ...);", "    return s;", "}", "int main() {",
             '    std::printf("%s\\n", sig(static_cast<decltype(&mvs_refine_cameras)>(nullptr)).c_str());', "    return 0;", "}"]
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "probe"
    subprocess.check_call([cxx, "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    want = subprocess.check_output([str(exe)], text=True).strip()
    f = lib.mvs_refine_cameras
    got = ("i:" if f.restype is ctypes.c_int else "?:") + "".join(_code(t) for t in f.argtypes)
    assert got == want and "mvs_refine_cameras" in _lib.EXPORTS
