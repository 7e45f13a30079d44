"""CPU: the float64 reference (oracle/fp64_ref.py) and its comparison rule.

* It computes the same function as the real reference: every live-reference fixture deviates from it by no more than a
  small constant times what the fp32 numpy oracle deviates (per column, max and RMS).
* Its rule is sharper than the 1e-5 rule: single-weight perturbations that `loco_oracle.close` accepts are rejected.
* The tensor-core arithmetic (3xTF32, emulated by tools/tf32x3_study.py) lands where the emulation says it should."""
import glob
import os

import numpy as np
import pytest

from monoloco_b200 import synthetic
from oracle import fp64_ref as R
from oracle import loco_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
FIXTURE_BOUND = 4.0   # a fixture (torch fp32 on the CPU) may be this many times less accurate than the numpy oracle


def _assert_rule(got, ref64, honest32, bound, what):
    mx, rms = R.fp64_rule(got, ref64, honest32)
    assert (mx <= bound).all() and (rms <= bound).all(), (what, mx.round(2).tolist(), rms.round(2).tolist())


def _sd(f):
    isz, osz, L, st, seed = [int(v) for v in f['cfg'][:5]]
    return synthetic.make_state_dict(str(f['kind']), isz, osz, L, st, seed)


def test_kinv32_is_the_engines_inverse():
    from monoloco_b200.engine import kinv_from_kk
    for kk in (synthetic.KITTI_K, [[700.0, 3.5, 612.0], [0.0, 705.25, 170.0], [0.0, 0.0, 1.0]]):
        for k in (kk, np.asarray(kk, dtype=np.float32)):
            assert np.array_equal(R.kinv32(k), kinv_from_kk(k))


@pytest.mark.parametrize('path', sorted(glob.glob(os.path.join(GOLDEN, 'ref_fwd_*.npz')) +
                                        glob.glob(os.path.join(GOLDEN, 'ref_wide_*.npz'))))
def test_network_fixtures_within_fp32_error(path):
    f = np.load(path)
    sd = _sd(f)
    ref64 = R.model_forward(sd, f['x'])
    _assert_rule(f['out'], ref64, O.model_forward(sd, f['x']), FIXTURE_BOUND, path)
    if 'dec_xyzd' in f.files:   # decode of the fixture's own raw outputs: only the decode's rounding differs
        kind = R.DECODE_LOCO if str(f['kind']) == 'loco' else R.DECODE_MONO
        d64 = R.decode(f['out'], kind)
        d32 = O.extract_outputs(f['out']) if kind == R.DECODE_LOCO else O.extract_outputs_mono(f['out'])
        _assert_rule(f['dec_xyzd'], d64[:, 0:4], d32['xyzd'], FIXTURE_BOUND, (path, 'xyzd'))
        _assert_rule(f['dec_bi'], d64[:, 4:5], d32['bi'], FIXTURE_BOUND, (path, 'bi'))


@pytest.mark.parametrize('name', ['kat_mono_train', 'kat_mono_val', 'kat_stereo_train', 'kat_stereo_val'])
def test_preprocess_fixtures_within_fp32_error(name):
    """The reference's own stored X against pre-process in float64 from the fp32 K^-1, per camera matrix."""
    f = np.load(os.path.join(GOLDEN, name + '.npz'))
    for k in np.unique(f['K'].reshape(-1, 9), axis=0):
        rows = np.where((f['K'].reshape(-1, 9) == k).all(1))[0]
        kps, kk = f['kps'][rows], k.reshape(3, 3)
        if 'mono' in name:
            x64, bound = R.preprocess_mono(kps, R.kinv32(kk))
            x32 = O.preprocess_monoloco(kps, kk)
        else:
            le, ri = np.ascontiguousarray(kps[:, :, :17]), np.ascontiguousarray(kps[:, :, 17:])
            xl, bl = R.preprocess_mono(le, R.kinv32(kk))
            xr, br = R.preprocess_mono(ri, R.kinv32(kk))
            x64, bound = np.concatenate([xl, xl - xr], 1), np.concatenate([bl, bl + br], 1)
            a, b = O.preprocess_monoloco(le, kk), O.preprocess_monoloco(ri, kk)
            x32 = np.concatenate([a, a - b], 1)
        _assert_rule(f['X'][rows], x64, x32, FIXTURE_BOUND, (name, rows[0]))
        # componentwise: a handful of fp32 ulps of sum |terms| * z_met (the K^-1 of the fixture is a different fp32 rounding)
        assert (np.abs(f['X'][rows] - x64) <= 8 * 2.0 ** -24 * bound + 1e-30).all()


def test_loco_fixtures_within_fp32_error():
    """End to end (pre-process, network, decode, bbox-centre ray) against the live-reference Loco.forward fixtures."""
    f = np.load(os.path.join(GOLDEN, 'ref_loco_mono_pifpaf.npz'))
    sd = synthetic.make_state_dict('loco', 34, 9, 1024, 3, 1)
    kinv = R.kinv32(f['K'])
    raw64 = R.model_forward(sd, R.preprocess_mono(f['keypoints'], kinv)[0])
    d64 = R.decode(raw64, R.DECODE_LOCO)
    d32 = O.loco_forward(sd, f['keypoints'], f['K'], mode='mono')
    for k, c in (('xyzd', slice(0, 4)), ('bi', slice(4, 5))):
        _assert_rule(f['out_' + k], d64[:, c], d32[k], FIXTURE_BOUND, k)
    for k in ('h', 'w', 'l', 'ori'):
        c = {'h': slice(4, 5), 'w': slice(5, 6), 'l': slice(6, 7), 'ori': slice(7, 9)}[k]
        _assert_rule(f['out_' + k], raw64[:, c], d32[k], FIXTURE_BOUND, k)
    c64 = R.xyzc(f['keypoints'], kinv, d64[:, 3])
    c32 = O.xyz_from_distance(d32['d'], O.pixel_to_camera(O.get_keypoints(f['keypoints'], 'center'), f['K'], 1))
    _assert_rule(f['xyz_from_distance'], c64[:, :3], c32, FIXTURE_BOUND, 'xyz_from_distance')

    g = np.load(os.path.join(GOLDEN, 'ref_loco_stereo.npz'))
    sd = synthetic.make_state_dict('loco', 68, 10, 1024, 3, 2)
    x64, _ = R.preprocess_stereo(g['left'], g['right'], R.kinv32(g['K']))
    _assert_rule(g['pairs_x'], x64, O.preprocess_monstereo(g['left'], g['right'], g['K'])[0], FIXTURE_BOUND, 'pairs_x')
    _assert_rule(g['pairs_raw'], R.model_forward(sd, g['pairs_x']), O.model_forward(sd, g['pairs_x']), FIXTURE_BOUND,
                 'pairs_raw')

    h = np.load(os.path.join(GOLDEN, 'ref_loco_images.npz'))
    sd = synthetic.make_state_dict('loco', 34, 9, 1024, 3, 1)
    off = np.concatenate([[0], np.cumsum(h['mono_n'])])
    d64 = np.concatenate([R.decode(R.model_forward(sd, R.preprocess_mono(h['mono_kps'][a:b], R.kinv32(kk))[0]),
                                   R.DECODE_LOCO) for a, b, kk in zip(off[:-1], off[1:], h['mono_K']) if b > a])
    d32 = np.concatenate([O.loco_forward(sd, h['mono_kps'][a:b], kk, mode='mono')['xyzd']
                          for a, b, kk in zip(off[:-1], off[1:], h['mono_K']) if b > a])
    _assert_rule(h['mono_out_xyzd'], d64[:, 0:4], d32, FIXTURE_BOUND, 'images xyzd')


# ------------------------------------------------------------------------------------------------ sharpness
@pytest.fixture(scope='module')
def net1024():
    sd = synthetic.make_state_dict('loco', 34, 9, 1024, 3, 0)
    x = synthetic.make_inputs(1024, 34, seed=0)
    return sd, x, R.model_forward(sd, x), O.loco_model_forward(sd, x)


PERTURBATIONS = [('w_fin.weight', (2, 100), 1e-3, True), ('w1.weight', (3, 33), 1e-3, True),
                 ('linear_stages.2.w1.weight', (1000, 1023), 1e-2, False)]


@pytest.mark.parametrize('name,idx,rel,rejected', PERTURBATIONS)
def test_rule_rejects_perturbations_the_old_rule_accepts(net1024, name, idx, rel, rejected):
    """One weight element scaled by (1 + rel) in an otherwise honest fp32 forward: the 1e-5 rule (loco_oracle.close)
    passes it, the float64 rule at the FFMA thresholds does not (for the first two; the third is pinned as measured)."""
    sd, x, ref64, ref32 = net1024
    sd2 = dict(sd)
    w = sd[name].copy()
    w[idx] = np.float32(w[idx] * (1 + rel))
    sd2[name] = w
    got = O.loco_model_forward(sd2, x)
    ok, worst = O.close(got, ref32)
    assert ok and worst < 1.0, worst                       # the gap the float64 rule closes
    mx, rms = R.fp64_rule(got, ref64, ref32)
    fails = bool((mx > R.FFMA_RULE[0]).any() or (rms > R.FFMA_RULE[1]).any())
    if rejected:
        assert fails, (mx.round(2).tolist(), rms.round(2).tolist())
    # the honest fp32 forward is the unit of the rule
    mx0, rms0 = R.fp64_rule(ref32, ref64, ref32)
    assert (mx0 <= 1.0).all() and (rms0 <= 1.0).all() and np.isclose(mx0.max(), 1.0)


# ------------------------------------------------------------------------------------------------ tensor-core arithmetic
@pytest.fixture(scope='module')
def net128():
    sd = synthetic.make_state_dict('loco', 34, 9, 1024, 3, 0)
    x = O.preprocess_monoloco(synthetic.make_keypoints(128, seed=0), synthetic.KITTI_K)
    return sd, x, R.model_forward(sd, x), O.loco_model_forward(sd, x)


def _seq_fp32(a, w):
    """a [B,K] @ w[N,K]^T with one fp32 accumulator per output, one rounding per product-add (FFMA order)."""
    a64, w64 = a.astype(np.float64), w.astype(np.float64)
    acc = np.zeros((a.shape[0], w.shape[0]), dtype=np.float32)
    for k in range(a.shape[1]):
        acc = (acc.astype(np.float64) + np.outer(a64[:, k], w64[:, k])).astype(np.float32)
    return acc


@pytest.mark.parametrize('mode,lo,hi', [('rn', 0.8, 1.6), ('rz', 8.0, 18.0), ('seq', 0.5, 4.0)])
def test_tf32x3_emulation_ratios(net128, mode, lo, hi):
    """The tensor-core kernel's scheme emulated (tools/tf32x3_study.mm_tf32x3_split, one K part): a = a_hi + a_lo in TF32,
    a_hi.w_hi into a main fp32 accumulator, a_lo.w_hi + a_hi.w_lo into a second one, one rounding per MMA of k = 8, the two
    added once in fp32.  With round-to-nearest accumulators it is as accurate as the fp32 oracle; with the truncating adder
    (the pessimistic model of the wgmma accumulator) it is 12x less accurate here (128 rows, width 1024), the order the GPU measures
    (DESIGN.md §2a).  A sequential fp32 accumulation (the FFMA kernels' order) is within 4x."""
    from tools import tf32x3_study as S
    sd, x, ref64, ref32 = net128
    mm = _seq_fp32 if mode == 'seq' else (lambda a, w: S.mm_tf32x3_split(np.asarray(a, np.float32), w, mode, 1))
    out = S.forward(sd, x, mm)
    mx, rms = R.fp64_rule(out, ref64, ref32)
    worst = max(mx.max(), rms.max())
    assert lo <= worst <= hi, (mode, mx.round(2).tolist(), rms.round(2).tolist())
    if mode != 'rz':
        assert worst <= R.TC_RULE[0]
