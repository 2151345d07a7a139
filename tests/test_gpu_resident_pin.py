"""GPU: bitwise pin of the frame-resident optimiser -- lbfgs_resident_kernel through mvs_fit (history 100 and 1, warm frames
whose slice of a run is empty, the temporal term, VPoser stages) and through a resident frame stream (three rigs, 3-D targets),
and the sequence-chaining kernel through mvs_fit_seq_stream (re-initialised frames, the temporal term, VPoser stages, and
cold successors parked for the earlier runs).  Every stage runs frame-resident (no SDF term).  The fixture
(golden/resident_pin.npz) was written by scripts/make_resident_pin.py on an H100; any change of a floating-point operation or
of its order in the resident closure, the optimiser, the stage transitions or the sequence walk shows up as a bit difference
in the rows or losses (compared as uint32, so NaN rows compare too), or as different counts."""
import os

import numpy as np
import pytest
import torch

from mvsmplfitting_b200 import seqio
from mvsmplfitting_b200 import synthetic as S
from tests import test_gpu_rigs as R
from tests import test_gpu_seq_stream as SQ
from tests import test_gpu_seq_temporal as TP

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resident_pin.npz")
STATS = ("frame_iterations", "frame_evals", "rounds", "frames_nan", "dense_frame_evals", "dense_rounds")
CASES = ("batch", "batch_h1", "warm_split", "temporal", "vposer", "stream", "seq", "seq_vposer", "seq_parked")
B_BATCH = 37
SEQ_LENGTHS = (1, 4, 7, 2, 9)


def result(x, final, st):
    return dict(x=np.asarray(x).view(np.uint32), final=np.asarray(final).view(np.uint32),
                stats=np.array([st[k] for k in STATS], dtype=np.int64))


def batch_case(model, gmm, history=100, mode=0, vposer=False, warm=False, temporal=False):
    """ctx.fit of B_BATCH frames seen by 8 views, 4 stages; warm frames every third, the others cold"""
    cams = S.make_cameras(8)
    fr = S.make_frames(model, cams, B_BATCH, seed=3)
    ctx = SQ.make_ctx(model, gmm, cams, B_BATCH, mode=mode)
    if vposer:
        ctx.set_vposer(S.make_vposer(11))
    ctx.set_keypoints(fr["gt_uv"], fr["conf"], fr["joint_weights"])
    x0 = S.pack_params(fr["init"])
    if vposer:
        x0[:, 13:82] = 0.0
    x = torch.tensor(x0, device="cuda")
    kw = {}
    if warm:
        kw["warm"] = np.arange(B_BATCH) % 3 == 1
    if temporal:
        prev = x0 + np.random.RandomState(4).normal(0, 0.05, x0.shape).astype(np.float32)
        kw.update(prev=torch.tensor(prev, device="cuda"), temporal_weight=TP.tw_vec())
    final, st = ctx.fit(x, SQ.stages(ctx, vposer=vposer), ctx.make_lbfgs_config(history_size=history), **kw)
    out = result(x.cpu().numpy(), final.cpu().numpy(), st)
    ctx.close()
    return out


def stream_case(model, gmm):
    """fit_stream: 53 frames through 16 slots, three rigs, 3-D targets (some rows without confidence)"""
    cams, sc = R.rig_cams(), R.rig_scales()
    rig = np.random.RandomState(9).randint(0, len(cams), 53).astype(np.int32)
    d = R.make_data(model, cams, rig, 17)
    d["c3"][[2, 19, 40]] = 0.0
    ctx = R.new_ctx(model, gmm, 16, rigs=cams, scales=sc)
    x = torch.tensor(d["x0"], device="cuda")
    final, st = ctx.fit_stream(x, d["gt_uv"], d["conf"], d["jw"], R.stage_cfgs(ctx, "gmm"), ctx.make_lbfgs_config(**R.OPT),
                               joints3d=d["j3"], conf3d=d["c3"], rig=rig)
    out = result(x.cpu().numpy(), final.cpu().numpy(), st)
    ctx.close()
    return out


def seq_case(model, gmm, kind):
    """fit_seq_stream of five sequences through 3 slots with the temporal term and a re-initialisation threshold between the
    final losses, so that some later frames start cold"""
    cams = S.make_cameras(4)
    seqs = SQ.make_seqs(model, cams, SEQ_LENGTHS, 1900)
    reinit = SQ.reinit_between(TP.stream(model, gmm, cams, seqs, 3, kind, tw=TP.tw_vec())[1])
    x, final, st, _ = TP.stream(model, gmm, cams, seqs, 3, kind, reinit=reinit, tw=TP.tw_vec())
    assert SQ.cold_after_first(seqs, final, reinit) >= 1
    return result(x, final, st)


def seq_parked_case(model, gmm):
    """exec mode 2, 3 stages: the chaining run is stage 2 alone, frame-resident; cold successors park, and the runs of stages 0
    and 1 take them as a resident frame stream"""
    cams = S.make_cameras(4)
    seqs = SQ.make_seqs(model, cams, SEQ_LENGTHS, 1950)
    gt_uv = np.concatenate([q["gt_uv"] for q in seqs], 1)
    conf = np.concatenate([q["conf"] for q in seqs], 1)
    jw = seqio.joint_weights("lsp14")

    def run(reinit):
        ctx = SQ.make_ctx(model, gmm, cams, 3, mode=2)
        cfgs = SQ.stages(ctx, n=3)
        x = seqio._cold_guesses(ctx, gt_uv, conf, jw, cfgs, SQ.GUESS)
        final, st = ctx.fit_seq_stream(x, gt_uv, conf, jw, SEQ_LENGTHS, cfgs, ctx.make_lbfgs_config(**SQ.OPT), reinit_loss=reinit,
                                       temporal_weight=TP.tw_vec())
        out = x.cpu().numpy(), final.cpu().numpy(), st
        ctx.close()
        return out

    reinit = SQ.reinit_between(run(5000.0)[1])
    x, final, st = run(reinit)
    assert SQ.cold_after_first(seqs, final, reinit) >= 1
    return result(x, final, st)


def run_case(name, model, gmm):
    """-> dict of arrays pinned for case `name`"""
    if name.startswith("seq"):
        return seq_parked_case(model, gmm) if name == "seq_parked" else seq_case(model, gmm, "vposer" if name == "seq_vposer" else "gmm")
    if name == "stream":
        return stream_case(model, gmm)
    return batch_case(model, gmm, history=1 if name == "batch_h1" else 100, mode=2 if name == "warm_split" else 0,
                      vposer=name == "vposer", warm=name in ("warm_split", "temporal"), temporal=name == "temporal")


@pytest.mark.parametrize("name", CASES)
def test_frame_resident_paths_bitwise(name, syn_model, syn_gmm):
    g = np.load(GOLD)
    r = run_case(name, syn_model, syn_gmm)
    assert sorted(r) == sorted(k.split("/", 1)[1] for k in g.files if k.startswith(name + "/"))
    for k, v in r.items():
        want = g[name + "/" + k]
        assert v.dtype == want.dtype and np.array_equal(v, want), (name, k, np.flatnonzero((v != want).reshape(len(v), -1).any(1)))
