"""CPU: seqio.fit_sequences / fit_sequence with shared_shape drive a context as the shared-shape contract says (recording stubs),
and the ctypes signature of mvs_fit_shared_shape matches include/mvsmpl.h as the host compiler reads it."""
import ctypes
import os
import pickle
import shutil
import subprocess

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import seqio
from tests.test_rig_abi import _code
from tests.test_seqio import _cfgs
from tests.test_seqio_temporal import TemporalStub, _seq

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPE = np.arange(10, dtype=np.float32) + 0.5          # the stub's shared betas


class ShapeStub(TemporalStub):
    """TemporalStub that also records fit_stream and fit_shared_shape; the latter writes SHAPE into every row's betas"""

    def fit_stream(self, params, gt_uv, conf, jw, stage_cfgs, opt_cfg=None, **kw):
        self.calls.append(("frames", params.shape[0]))
        return torch.zeros(params.shape[0]), dict(frame_iterations=1, frame_evals=1, rounds=1, frames_nan=0)

    def fit_shared_shape(self, params, gt_uv, conf, jw, lengths, stage_cfg, opt_cfg=None, sweeps=1, **kw):
        self.calls.append(("shape", params.shape[0], list(lengths), stage_cfg, sweeps, np.asarray(gt_uv).shape, kw))
        params[:, :10] = torch.as_tensor(SHAPE)
        return (torch.full((params.shape[0],), 7.0), torch.zeros(len(lengths)), dict(frame_iterations=2),
                dict(frame_iterations=3))

    def vposer_decode(self, params):
        return torch.zeros(params.shape[0], 69)


def _names(calls):
    return [c[0] for c in calls]


@pytest.mark.parametrize("B", [2, 1])
def test_off_makes_exactly_todays_calls(B):
    seqs = [_seq(3, "a"), _seq(2, "b")]
    ref, got = ShapeStub(B), ShapeStub(B)
    r0 = seqio.fit_sequences(ref, seqs, _cfgs(4))
    r1 = seqio.fit_sequences(got, seqs, _cfgs(4), shared_shape=0)
    assert _names(ref.calls) == _names(got.calls) and "shape" not in _names(got.calls)
    assert all(np.array_equal(a[0], b[0]) for a, b in zip(r0[0], r1[0]))
    assert "shared_shape" not in r1[1]


@pytest.mark.parametrize("B", [2, 1])
def test_on_adds_one_call_over_all_frames_with_the_last_stage(B):
    seqs = [_seq(3, "a"), _seq(2, "b")]
    cfgs = _cfgs(4)
    ref, got = ShapeStub(B), ShapeStub(B)
    seqio.fit_sequences(ref, seqs, cfgs)
    res, stats = seqio.fit_sequences(got, seqs, cfgs, shared_shape=2)
    assert _names(got.calls) == _names(ref.calls) + ["shape"]
    _, F, lengths, cfg, sweeps, shape, kw = got.calls[-1]
    assert F == 5 and lengths == [3, 2] and sweeps == 2 and shape == (2, 5, 17, 2) and kw == {}
    assert cfg is cfgs[-1]
    for x, loss in res:                                   # the results carry the shared shape and the pose step's losses
        assert (x[:, :10] == SHAPE).all() and (loss == 7.0).all()
    assert stats["shared_shape"] == dict(shape=dict(frame_iterations=2), pose=dict(frame_iterations=3))


def test_fit_sequence_is_one_subject():
    ctx = ShapeStub(2)
    x, loss, stats = seqio.fit_sequence(ctx, _seq(5, "a"), _cfgs(4), shared_shape=1)
    sh = [c for c in ctx.calls if c[0] == "shape"]
    assert len(sh) == 1 and sh[0][1] == 5 and sh[0][2] == [5] and sh[0][4] == 1
    assert (x[:, :10] == SHAPE).all() and (loss == 7.0).all()
    ctx = ShapeStub(2)
    seqio.fit_sequence(ctx, _seq(5, "a"), _cfgs(4))
    assert "shape" not in _names(ctx.calls)


@pytest.mark.parametrize("bad", [-1, 1.5, True])
def test_bad_sweeps_and_the_temporal_term_are_refused(bad):
    with pytest.raises(ValueError):
        seqio.fit_sequences(ShapeStub(2), [_seq(2, "a"), _seq(2, "b")], _cfgs(4), shared_shape=bad)
    with pytest.raises(ValueError):
        seqio.fit_sequence(ShapeStub(2), _seq(2, "a"), _cfgs(4), shared_shape=bad)
    with pytest.raises(ValueError):
        seqio.fit_sequences(ShapeStub(2), [_seq(2, "a"), _seq(2, "b")], _cfgs(4), shared_shape=1, temporal_weight=1.0)


@pytest.mark.parametrize("B", [2, 1])
def test_exported_results_carry_the_shared_betas(B, tmp_path):
    ctx = ShapeStub(B)
    seqio.fit_sequences(ctx, [_seq(3, "a"), _seq(2, "b")], _cfgs(4), shared_shape=1, result_folder=str(tmp_path))
    files = sorted(p for p in tmp_path.rglob("*.pkl"))
    assert len(files) == 5
    for p in files:
        with open(p, "rb") as fh:
            r = pickle.load(fh)
        assert np.allclose(np.ravel(r["betas"]), SHAPE)


def test_shared_shape_entry_point_matches_the_header(tmp_path):
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
             '    std::printf("%s\\n", sig(static_cast<decltype(&mvs_fit_shared_shape)>(nullptr)).c_str());', "    return 0;", "}"]
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "probe"
    subprocess.check_call([cxx, "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    want = subprocess.check_output([str(exe)], text=True).strip()
    f = lib.mvs_fit_shared_shape
    got = ("i:" if f.restype is ctypes.c_int else "?:") + "".join(_code(t) for t in f.argtypes)
    assert got == want and "mvs_fit_shared_shape" in _lib.EXPORTS
