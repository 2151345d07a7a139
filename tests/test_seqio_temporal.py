"""CPU: seqio.fit_sequences(temporal_weight=...) drives a context as the temporal contract says (recording stubs), and the ctypes
signatures of mvs_fit_seq_temporal / mvs_fit_seq_stream_temporal match include/mvsmpl.h as the host compiler reads it."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import seqio
from mvsmplfitting_b200.sequence import smooth_mask
from tests.test_rig_abi import _code
from tests.test_seqio import _cfgs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("mvs_fit_seq_temporal", "mvs_fit_seq_stream_temporal")


class TemporalStub:
    """records what the drivers ask of a FittingContext, including the temporal arguments"""

    def __init__(self, B):
        self.B, self.calls, self.device = B, [], "cpu"

    def set_keypoints(self, gt_uv, conf, jw):
        self.calls.append(("kp",))

    def set_loss(self, config=None):
        self.calls.append(("loss",))

    def init_guess(self, **kw):
        n = len([c for c in self.calls if c[0] == "init"])
        self.calls.append(("init",))
        return (torch.arange(self.B * 86, dtype=torch.float32).reshape(self.B, 86) + 1000 * n).contiguous(), None

    def fit(self, params, stage_cfgs, opt_cfg, warm=None, prev=None, temporal_weight=None):
        self.calls.append(("fit", None if warm is None else list(map(bool, warm)), None if prev is None else prev.clone(),
                           temporal_weight, params.clone()))
        params += 1
        return torch.ones(self.B), dict(frame_iterations=1, frame_evals=1, rounds=1, frames_nan=0)

    def fit_seq_stream(self, params, gt_uv, conf, jw, lengths, stage_cfgs, opt_cfg=None, reinit_loss=5000.0, **kw):
        self.calls.append(("stream", list(lengths), kw))
        return torch.zeros(params.shape[0]), dict(frame_iterations=1, frame_evals=1, rounds=1, frames_nan=0)


def _seq(T, serial):
    return dict(gt_uv=np.zeros((2, T, 17, 2), np.float32), conf=np.ones((2, T, 17), np.float32),
                present=np.ones((2, T), bool), frames=["%05d" % t for t in range(T)], serial=serial)


def test_scalar_expands_to_the_smoothness_mask():
    w = seqio.temporal_weight_vector(2.5)
    assert w.dtype == np.float32 and w.shape == (86,)
    assert np.array_equal(w, np.float32(2.5) * smooth_mask().numpy())
    assert (w[10:85] == 2.5).all() and (w[:10] == 0).all() and w[85] == 0
    full = np.arange(86, dtype=np.float64)
    assert np.array_equal(seqio.temporal_weight_vector(full), full.astype(np.float32))
    assert seqio.temporal_weight_vector(None) is None
    with pytest.raises(ValueError):
        seqio.temporal_weight_vector(np.ones(85))


@pytest.mark.parametrize("latent", [False, True])
def test_lockstep_passes_the_previous_fitted_rows_and_the_warm_mask(latent):
    ctx = TemporalStub(2)
    seqio.fit_sequences(ctx, [_seq(3, "a"), _seq(2, "b")], _cfgs(4, use_vposer=2 if latent else 0), reinit_loss=5.0,
                        temporal_weight=3.0)
    fits = [c for c in ctx.calls if c[0] == "fit"]
    assert len(fits) == 3
    assert fits[0][1] is None and fits[0][2] is None and fits[0][3] is None          # first frames: cold, no term
    for t in (1, 2):
        _, warm, prev, tw, start = fits[t]
        assert warm == [True, True] and np.array_equal(tw, seqio.temporal_weight_vector(3.0))
        fitted = fits[t - 1][4] + 1                                                   # what step t-1 returned (the stub adds 1)
        assert torch.equal(prev, fitted)
        # the start point is the warm start: without a latent pose the body pose restarts from the cold guess (hip seed),
        # while prev keeps the fitted pose
        if latent:
            assert torch.equal(start, fitted)
        else:
            assert torch.equal(start[:, :13], fitted[:, :13]) and not torch.equal(start[:, 13:82], fitted[:, 13:82])


def test_lockstep_without_a_warm_frame_or_a_weight_is_unchanged():
    ctx = TemporalStub(2)
    seqio.fit_sequences(ctx, [_seq(2, "a"), _seq(2, "b")], _cfgs(4), reinit_loss=0.5, temporal_weight=3.0)
    fits = [c for c in ctx.calls if c[0] == "fit"]
    assert all(f[1] is None and f[2] is None and f[3] is None for f in fits)           # every frame re-initialised
    ctx = TemporalStub(2)
    seqio.fit_sequences(ctx, [_seq(2, "a"), _seq(2, "b")], _cfgs(4))
    fits = [c for c in ctx.calls if c[0] == "fit"]
    assert fits[1][1] == [True, True] and fits[1][2] is None and fits[1][3] is None


def test_stream_passes_the_86_vector():
    w = np.linspace(0, 1, 86).astype(np.float32)
    ctx = TemporalStub(1)
    seqio.fit_sequences(ctx, [_seq(3, "a"), _seq(2, "b")], _cfgs(4), temporal_weight=w)
    st = [c for c in ctx.calls if c[0] == "stream"]
    assert len(st) == 1 and st[0][1] == [3, 2] and np.array_equal(st[0][2]["temporal_weight"], w)
    ctx = TemporalStub(1)
    seqio.fit_sequences(ctx, [_seq(3, "a"), _seq(2, "b")], _cfgs(4), temporal_weight=0.5)
    assert np.array_equal([c for c in ctx.calls if c[0] == "stream"][0][2]["temporal_weight"], seqio.temporal_weight_vector(0.5))
    ctx = TemporalStub(1)
    seqio.fit_sequences(ctx, [_seq(3, "a"), _seq(2, "b")], _cfgs(4))
    assert "temporal_weight" not in [c for c in ctx.calls if c[0] == "stream"][0][2]


def test_temporal_entry_points_match_the_header(tmp_path):
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
             "    if (std::is_same<T, unsigned>::value) return 'u';",
             "    return '?';", "}",
             "template <class R, class... A> std::string sig(R (*)(A...)) {",
             "    std::string s = std::is_same<R, int>::value ? \"i:\" : \"?:\";",
             "    ((s += code<A>()), ...);", "    return s;", "}", "int main() {"]
    lines += ['    std::printf("%s %%s\\n", sig(static_cast<decltype(&%s)>(nullptr)).c_str());' % (n, n) for n in NEW]
    lines += ["    return 0;", "}"]
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "probe"
    subprocess.check_call([cxx, "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    want = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    for n in NEW:
        f = getattr(lib, n)
        got = ("i:" if f.restype is ctypes.c_int else "?:") + "".join(_code(t) for t in f.argtypes)
        assert got == want[n], (n, got, want[n])
        assert n in _lib.EXPORTS
