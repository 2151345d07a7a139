"""CPU: lens distortion on the host side: seqio.load_camera_distortion on the shipped camera file and on 2- and 5-number lines,
write_camera_para -> load_camera_para + load_camera_distortion round trips, camera_arrays without "dist" unchanged, that
FittingContext and the drivers reach mvs_set_camera_rigs_dist only when a rig has coefficients (recording stubs), that the
refined calibration files carry the coefficients, that SequenceFitter passes a rig's "dist" on, and the ctypes signature of the new
entry point against include/mvsmpl.h."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import seqio
from mvsmplfitting_b200 import synthetic as S
from mvsmplfitting_b200.context import FittingContext
from tests.test_rig_abi import RigStub, _code, _seq as _rig_seq
from tests.test_seqio import _cfgs
from tests.test_seqio_camera import CameraStub, RIGS, _rig
from tests.test_seqio_temporal import _seq

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEMO = os.path.join(ROOT, "tests", "golden", "demo", "3DOH50K_Parameters.txt")


def _dist(V, seed, full=True):
    rng = np.random.RandomState(seed)
    d = np.zeros((V, 5), np.float32)
    d[:, 0] = rng.uniform(-0.3, -0.1, V)
    d[:, 1] = rng.uniform(0.0, 0.1, V)
    if full:
        d[:, 2:4] = rng.normal(0, 1e-3, (V, 2))
        d[:, 4] = rng.normal(0, 0.01, V)
    return d


def test_demo_file_has_no_distortion():
    d = seqio.load_camera_distortion(DEMO)
    assert d.shape == (6, 5) and d.dtype == np.float64 and (d == 0).all()


def test_two_and_five_number_lines(tmp_path):
    ext, intr = seqio.load_camera_para(DEMO)
    lines = open(DEMO).read().splitlines()
    lines[4] = "-0.21 0.07"                                  # view 0: the line after its three intrinsic rows
    lines[9 + 4] = "-0.15 0.02 0.001 -0.0005 -0.01"          # view 1
    p = tmp_path / "cams.txt"
    p.write_text("\n".join(lines) + "\n")
    d = seqio.load_camera_distortion(str(p))
    assert d.shape == (6, 5)
    assert d[0].tolist() == [-0.21, 0.07, 0.0, 0.0, 0.0]
    assert d[1].tolist() == [-0.15, 0.02, 0.001, -0.0005, -0.01]
    assert (d[2:] == 0).all()
    e2, i2 = seqio.load_camera_para(str(p))                   # the reference's reader skips both lines, as before
    assert np.array_equal(e2, ext) and np.array_equal(i2, intr)


@pytest.mark.parametrize("full", [False, True])
def test_write_then_load_round_trips_float32(tmp_path, full):
    cams = _rig(6, 3)
    dist = _dist(6, 4, full)
    dist[2] = 0.0
    p = str(tmp_path / "cams.txt")
    seqio.write_camera_para(p, *seqio.camera_matrices(cams), dist=dist)
    words = [len(line.split()) for line in open(p).read().splitlines()[4::9]]
    assert words == [5 if full and v != 2 else 2 for v in range(6)]
    back = seqio.camera_arrays(*seqio.load_camera_para(p), dist=seqio.load_camera_distortion(p))
    for k in ("R", "t", "f", "c"):
        assert back[k].tobytes() == cams[k].tobytes(), k
    assert back["dist"].dtype == np.float32 and back["dist"].tobytes() == dist.tobytes()
    # without dist the file is what it was: '0 0' lines
    seqio.write_camera_para(p, *seqio.camera_matrices(cams))
    assert open(p).read().splitlines()[4::9] == ["0 0"] * 6


def test_camera_arrays_without_dist_is_unchanged():
    ext, intr = seqio.load_camera_para(DEMO)
    a = seqio.camera_arrays(ext, intr, views=[0, 2, 3])
    assert sorted(a) == ["R", "c", "f", "t"]
    b = seqio.camera_arrays(ext, intr, views=[0, 2, 3], dist=_dist(6, 1))
    assert all(a[k].tobytes() == b[k].tobytes() for k in a)
    assert b["dist"].tobytes() == _dist(6, 1)[[0, 2, 3]].tobytes()


class _Lib:
    """records the camera entry points FittingContext calls"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def f(*args):
            self.calls.append((name, args))
            return 0
        return f


def _ctx():
    ctx = FittingContext.__new__(FittingContext)
    ctx.lib, ctx.h = _Lib(), None
    return ctx


def test_context_reaches_the_dist_entry_point_only_with_coefficients():
    cams = {k: v for k, v in S.make_wide_cameras(3).items() if k in ("R", "t", "f", "c", "dist")}
    plain = {k: cams[k] for k in ("R", "t", "f", "c")}
    ctx = _ctx()
    ctx.set_camera_rigs([plain, dict(plain)])
    assert [c[0] for c in ctx.lib.calls] == ["mvs_set_camera_rigs"] and "dist" not in ctx._rigs[0]
    ctx = _ctx()
    ctx.set_cameras(plain["R"], plain["t"], plain["f"], plain["c"])
    assert [c[0] for c in ctx.lib.calls] == ["mvs_set_cameras"]
    ctx = _ctx()
    ctx.set_camera_rigs([plain, cams])
    assert [c[0] for c in ctx.lib.calls] == ["mvs_set_camera_rigs_dist"]
    assert "dist" not in ctx._rigs[0] and ctx._rigs[1]["dist"].tobytes() == cams["dist"].tobytes()
    ctx = _ctx()
    ctx.set_cameras(cams["R"], cams["t"], cams["f"], cams["c"], dist=cams["dist"])
    assert [c[0] for c in ctx.lib.calls] == ["mvs_set_camera_rigs_dist"] and ctx.rig_views == [3]
    with pytest.raises(ValueError, match="dist"):
        _ctx().set_camera_rigs([dict(plain, dist=np.zeros((2, 5)))])


class DistRigStub(RigStub):
    def set_camera_rigs(self, rigs, scale=None):
        self.calls.append(("rigs", [r.get("dist") is not None for r in rigs]))


def test_fit_sequences_passes_the_coefficients_with_the_rigs():
    rigs = [dict(_rig(2, 1), dist=_dist(2, 2)), _rig(4, 3)]
    ctx = DistRigStub(2)
    seqio.fit_sequences(ctx, [_rig_seq(2, 2, 0, "a"), _rig_seq(4, 2, 1, "b")], _cfgs(4), rigs=rigs)
    assert ctx.calls[0] == ("rigs", [True, False])


def test_refined_calibration_files_carry_the_coefficients(tmp_path):
    dist = _dist(2, 7)

    class DistCameraStub(CameraStub):
        def refine_cameras(self, *a, **kw):
            final, rigs, ca, po = super().refine_cameras(*a, **kw)
            return final, [dict(r, dist=dist) for r in rigs], ca, po

    seqio.fit_sequences(DistCameraStub(2), [_seq(3, "a"), _seq(2, "b")], _cfgs(4), refine_cameras=1, result_folder=str(tmp_path))
    p = str(tmp_path / "cameras_rig0.txt")
    back = seqio.camera_arrays(*seqio.load_camera_para(p), dist=seqio.load_camera_distortion(p))
    assert back["dist"].tobytes() == dist.tobytes()
    assert back["t"].tobytes() == (RIGS[0]["t"] + 1).astype(np.float32).tobytes()


def test_dist_entry_point_matches_the_header(tmp_path):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    from mvsmplfitting_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libmvsmpl.so is not built")
    lib = _lib.load()
    src = tmp_path / "probe.cpp"
    src.write_text("\n".join([
        '#include <cstdio>', '#include <string>', '#include <type_traits>', '#include "mvsmpl.h"',
        "template <class T> char code() {", "    if (std::is_pointer<T>::value) return 'p';",
        "    if (std::is_same<T, int>::value) return 'i';", "    if (std::is_same<T, float>::value) return 'f';", "    return '?';", "}",
        "template <class R, class... A> std::string sig(R (*)(A...)) {",
        "    std::string s = std::is_same<R, int>::value ? \"i:\" : \"?:\";", "    ((s += code<A>()), ...);", "    return s;", "}",
        "int main() {", '    std::printf("%s\\n", sig(static_cast<decltype(&mvs_set_camera_rigs_dist)>(nullptr)).c_str());', "    return 0;", "}"]) + "\n")
    exe = tmp_path / "probe"
    subprocess.check_call([cxx, "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    want = subprocess.check_output([str(exe)], text=True).strip()
    f = lib.mvs_set_camera_rigs_dist
    got = ("i:" if f.restype is ctypes.c_int else "?:") + "".join(_code(t) for t in f.argtypes)
    assert got == want == "i:pippppppp" and "mvs_set_camera_rigs_dist" in _lib.EXPORTS


def test_sequence_fitter_passes_the_coefficients(monkeypatch):
    from mvsmplfitting_b200 import context, sequence

    class Ctx:
        def __init__(self, dev):
            self.calls = []

        def set_model(self, *a, **k):
            pass

        def set_cameras(self, R, t, f, c, dist=None):
            self.calls.append(None if dist is None else np.asarray(dist))

        def set_batch(self, B):
            pass

    monkeypatch.setattr(context, "FittingContext", Ctx)
    cams = S.make_wide_cameras(3)
    fit = sequence.SequenceFitter(S.make_model(0), cams, 4, device=0)
    assert fit.ctx.calls[0].tobytes() == cams["dist"].tobytes()
    fit = sequence.SequenceFitter(S.make_model(0), S.make_cameras(3), 4, device=0)
    assert fit.ctx.calls[0] is None
