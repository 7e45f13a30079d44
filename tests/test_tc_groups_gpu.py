"""Tensor-core forward (forward_tc.cu) on CTA groups: one cooperative persistent grid of floor(SMs / (L/256)) groups of L/256
CTAs, synchronised by counters in global memory that only ever grow.  The group count changes which group runs a tile and
how many tiles each group walks, never the arithmetic: outputs must be bit-identical for every cap (MLB_TC_CLUSTERS), and
a launch must never pass a barrier on a counter value an earlier launch left behind."""
import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = pytest.mark.gpu

BATCHES = (64, 4096, 4224)   # one tile; 64 tiles (two rounds of 33 groups); 66 tiles (a ragged third round)


def _mods():
    from oracle import loco_oracle as O
    from monoloco_b200 import synthetic, engine, _lib
    return O, synthetic, engine, _lib


def _engine(monkeypatch, sd, cap):
    _, _, engine, _ = _mods()
    if cap is None:
        monkeypatch.delenv('MLB_TC_CLUSTERS', raising=False)
    else:
        monkeypatch.setenv('MLB_TC_CLUSTERS', str(cap))
    try:
        return engine.LocoEngine(sd)   # the cap is read when the engine is created
    finally:
        monkeypatch.delenv('MLB_TC_CLUSTERS', raising=False)


def _run(eng, kps):
    _, synthetic, _, L_ = _mods()
    out = eng.forward(torch.from_numpy(kps).cuda(), kk=synthetic.KITTI_K, kind=L_.IN_KPS, want_xyzc=True, want_x=True,
                      kernel='tc')
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize('L', [1024, 512, 2048])
def test_tc_groups_bit_identical_across_caps(monkeypatch, L):
    O, synthetic, engine, L_ = _mods()
    sd = synthetic.make_state_dict('loco', 34, 9, L, 3, 11)
    kps = {B: synthetic.make_keypoints(B, seed=500 + B) for B in BATCHES}
    eng = _engine(monkeypatch, sd, None)
    n_max = L_.lib().mlb_tc_resident_clusters(eng._h)
    assert n_max == eng.n_sms // (L // 256)
    ref = {}
    for B in BATCHES:
        ref[B] = _run(eng, kps[B])
        assert eng.last_kernel()[0] == 3   # MLB_KERNEL_TC
    eng.check_error()
    eng.close()
    # the uncapped run is right, not merely repeatable
    x = O.preprocess_monoloco(kps[4224], synthetic.KITTI_K)
    k = 2.0 if L == 2048 else 1.0   # 2048 wide with three stages: 2 x the parity rule (DESIGN.md §9)
    ok, worst = O.close(ref[4224]['raw'].cpu().numpy(), O.loco_model_forward(sd, x), rtol=k * 1e-5, atol=k * 1e-6)
    assert ok, worst
    for cap in (1, 7, n_max):
        eng = _engine(monkeypatch, sd, cap)
        assert L_.lib().mlb_tc_resident_clusters(eng._h) == cap
        for B in BATCHES:
            # two launches in a row: the second reuses every slot and counter the first one left
            for rep in range(2):
                out = _run(eng, kps[B])
                for k in ref[B]:
                    assert torch.equal(out[k], ref[B][k]), (L, cap, B, rep, k)
        eng.check_error()
        eng.close()


def test_tc_groups_reused_counters_across_group_counts(monkeypatch):
    """Launches with different group counts (1, 2, 33 groups ...) interleaved on one engine: every slot's counter is left at
    a different value, and each launch must still wait for its own arrivals."""
    O, synthetic, engine, L_ = _mods()
    sd = synthetic.make_state_dict('loco', 34, 9, 1024, 3, 12)
    eng = _engine(monkeypatch, sd, None)
    kps = {B: synthetic.make_keypoints(B, seed=700 + B) for B in (64, 130, 2048, 4224)}
    first = {B: _run(eng, kps[B])['raw'].clone() for B in kps}
    for B in (4224, 64, 130, 4224, 2048, 64, 4224):
        assert torch.equal(_run(eng, kps[B])['raw'], first[B]), B
    eng.check_error()
    eng.close()
