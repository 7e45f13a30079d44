"""GPU: every forward kernel family against the float64 reference (oracle/fp64_ref.py), at every hidden width it serves.

The rule: per output column, a kernel's max and RMS error against float64 divided by those of the fp32 numpy oracle on
the same rows (`fp64_rule`) stays under one (max, RMS) pair for the FFMA families and one for the 3xTF32 tensor-core
kernel (oracle/fp64_ref.py FFMA_RULE / TC_RULE).  The 1e-5 rule of the other forward tests is kept beside it.

* which family serves which width, and that a forced family either runs or is refused -- never silently replaced;
* width x family x batch edges (ragged tails, one row more or less than a tile, more tiles than SMs or CTA groups);
* a feature slice (stereo pairs, zero-centred mono, explicit dropout masks, MonolocoModel 2 / 9 outputs, 1 / 3 stages);
* a perturbed checkpoint that the 1e-5 rule accepts and this rule rejects;
* weight refresh: one element at each packer's boundaries changed through update_weights, on every family;
* degenerate detections through every fused prologue and mlb_preprocess; decode against float64 and bit-identical to
  mlb_decode.

With MLB_FP64_RATIOS=<path> the measured ratios are written there as JSON (tools/fp64_ratios.py prints them)."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = pytest.mark.gpu

FAMILIES = ('tile', 'cluster', 'wide', 'wide2', 'tc')
KERNEL_ID = {'tile': 0, 'cluster': 1, 'wide': 2, 'tc': 3, 'wide2': 4}
WIDTHS = (128, 256, 384, 512, 640, 768, 896, 1024, 1280, 1536, 1792, 2048, 1, 100, 300, 1001, 1500)
ULP = 2.0 ** -24
RATIOS = {}   # (family, test, width) -> [worst max ratio per column, worst RMS ratio per column]


def _old_rtol(family, padded):
    """The 1e-5 rule, with the stated exception of DESIGN.md §9: above a width of 1024 (every width the tensor-core kernel
    serves alone) the tensor-core kernel is held to 2e-5.  Its 63-row batches at 1500 / 1536 measure 1.25x / 1.07x of
    1e-5 and stay in the matrix as the regression cases of that gap."""
    return 2e-5 if family == 'tc' and padded > 1024 else 1e-5


def _mods():
    from oracle import fp64_ref as R, loco_oracle as O
    from monoloco_b200 import synthetic, engine, packing, _lib
    return R, O, synthetic, engine, packing, _lib


@pytest.fixture(scope='module', autouse=True)
def _dump_ratios():
    yield
    path = os.environ.get('MLB_FP64_RATIOS')
    if path:
        with open(path, 'w') as f:
            json.dump({'|'.join(map(str, k)): v for k, v in sorted(RATIOS.items())}, f)


def _rule(R, family):
    return R.TC_RULE if family == 'tc' else R.FFMA_RULE


def _record(key, mx, rms):
    old = RATIOS.get(key)
    mx, rms = [float(v) for v in mx], [float(v) for v in rms]
    if old is not None:
        mx, rms = [max(a, b) for a, b in zip(old[0], mx)], [max(a, b) for a, b in zip(old[1], rms)]
    RATIOS[key] = [mx, rms]


def _check(R, family, key, got, ref64, honest32, what, pool=None):
    mx, rms = R.fp64_rule(got, ref64, honest32, pool=pool)
    _record(key, mx, rms)
    lim = _rule(R, family)
    assert (mx <= lim[0]).all() and (rms <= lim[1]).all(), (what, family, mx.round(2).tolist(), rms.round(2).tolist())


def served(L_real, stereo=False):
    """Families that serve a model of hidden width L_real (mono or stereo input), as mlb_create sets them up on an H100:
    FFMA row tiles and the whole-grid kernel up to 1024 (padded to a multiple of 128), the 8-CTA cluster at 1024 only,
    wide2 where a quarter of the width holds the padded input (K slices of L/4 >= Kpad of 34 or 68 inputs), and the
    tensor cores at multiples of 256 up to 2048."""
    from monoloco_b200.packing import padded_width
    P = padded_width(L_real)
    out = set()
    if P <= 1024:
        out |= {'tile', 'wide'}
        if P // 4 >= (72 if stereo else 40):
            out.add('wide2')
    if P == 1024:
        out.add('cluster')
    if P % 256 == 0:
        out.add('tc')
    return out


def _pick_tm(n_rows, n_ctas):
    """forward.cu pick_rows_per_group: minimise waves(tm) * tm, tm in 16, 14, ..., 8."""
    best, best_cost = 16, None
    for tm in range(16, 7, -2):
        tiles = (n_rows + 2 * tm - 1) // (2 * tm)
        cost = ((tiles + n_ctas - 1) // n_ctas) * tm
        if best_cost is None or cost < best_cost:
            best, best_cost = tm, cost
    return best


def _sample(B, tile, rng, cap=512):
    """Rows checked in float64: first and last row of every tile, the ragged tail, then random rows up to `cap`."""
    s = {0, B - 1}
    for t0 in range(0, B, tile):
        s |= {t0, min(B, t0 + tile) - 1}
    rest = np.setdiff1d(np.arange(B), np.fromiter(s, dtype=np.int64))
    if len(s) < cap and rest.size:
        s |= set(rng.choice(rest, min(cap - len(s), rest.size), replace=False).tolist())
    return np.array(sorted(s), dtype=np.int64)


def _pre32(kps, kinv, zero_center=False, z_met=10.0):
    """The fused prologue's fp32 arithmetic with the engine's K^-1 (the honest fp32 pre-process the rule divides by)."""
    k = np.asarray(kinv, dtype=np.float32)
    f = np.float32
    u, v = kps[:, 0, :], kps[:, 1, :]
    x = (u * k[0] + v * k[1] + k[2]) * f(z_met)
    y = (u * k[3] + v * k[4] + k[5]) * f(z_met)
    if zero_center:
        uc = (u.max(1) - u.min(1)) / f(2) + u.min(1)
        vc = (v.max(1) - v.min(1)) / f(2) + v.min(1)
        x = x - ((uc * k[0] + vc * k[1] + k[2]) * f(z_met))[:, None]
        y = y - ((uc * k[3] + vc * k[4] + k[5]) * f(z_met))[:, None]
    return np.stack([x, y], 2).reshape(len(kps), 34).astype(np.float32)


def _xyzc32(kps, kinv, d):
    k = np.asarray(kinv, dtype=np.float32)
    u, v = kps[:, 0, :], kps[:, 1, :]
    uc = (u.max(1) - u.min(1)) / np.float32(2) + u.min(1)
    vc = (v.max(1) - v.min(1)) / np.float32(2) + v.min(1)
    c = np.stack([uc * k[0] + vc * k[1] + k[2], uc * k[3] + vc * k[4] + k[5], uc * k[6] + vc * k[7] + k[8]], 1)
    den = np.sqrt(np.float32(1) + c[:, 0:1] * c[:, 0:1] + c[:, 1:2] * c[:, 1:2])
    xyz = (c * np.asarray(d, dtype=np.float32).reshape(-1, 1) / den).astype(np.float32)
    return np.concatenate([xyz, np.sqrt((xyz * xyz).sum(1, keepdims=True))], 1)


def _decode_dev(raw, kind):
    """mlb_decode of a raw CUDA tensor -> [m, 8] CUDA tensor."""
    from monoloco_b200 import _lib as L_
    raw = raw.contiguous()
    dec = torch.empty((raw.shape[0], 8), dtype=torch.float32, device=raw.device)
    if raw.shape[0]:
        L_.check(L_.lib().mlb_decode(raw.data_ptr(), raw.shape[0], raw.shape[1], kind, dec.data_ptr(),
                                     C.c_void_p(torch.cuda.current_stream().cuda_stream)), 'mlb_decode')
    return dec


def _run(eng, family, x, **kw):
    out = eng.forward(x, kernel=family, **kw)
    torch.cuda.synchronize()
    assert eng.last_kernel()[0] == KERNEL_ID[family], (family, eng.last_kernel())
    return out


def _dec_bit_identical(out, decode_kind):
    ref = _decode_dev(out['raw'], decode_kind)
    a, b = out['dec'].cpu().numpy(), ref.cpu().numpy()
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), np.argwhere(a.view(np.uint32) != b.view(np.uint32))[:5]


# ------------------------------------------------------------------------------------------------ served-kernel table
# forced family -> 'ran' or 'refused', at 16 mono rows; the table written out (see `served` for the rules)
EXPECTED_TABLE = {
    128: 'tile wide', 256: 'tile wide wide2 tc', 384: 'tile wide wide2', 512: 'tile wide wide2 tc', 640: 'tile wide wide2',
    768: 'tile wide wide2 tc', 896: 'tile wide wide2', 1024: 'tile cluster wide wide2 tc', 1280: 'tc', 1536: 'tc',
    1792: 'tc', 2048: 'tc', 1: 'tile wide', 100: 'tile wide', 300: 'tile wide wide2', 1001: 'tile cluster wide wide2 tc',
    1500: 'tc'}


def test_served_kernel_table():
    """Each width x forced family: the family ran (mlb_last_kernel says so) or mlb_forward refused with a message.  A
    forced family replaced by another (wide2 -> tc above 1024 used to be) is a failure, not a pass."""
    R, O, synthetic, engine, packing, L_ = _mods()
    x = torch.from_numpy(synthetic.make_inputs(16, 34, seed=1)).cuda()
    table, msgs = {}, {}
    for L in WIDTHS:
        assert EXPECTED_TABLE[L] == ' '.join(f for f in FAMILIES if f in served(L)), L
        eng = engine.LocoEngine(synthetic.make_state_dict('loco', 34, 9, L, 1, 3))
        ran = []
        for fam in FAMILIES:
            try:
                eng.forward(x, kernel=fam)
                torch.cuda.synchronize()
            except RuntimeError as e:
                msgs[(L, fam)] = str(e)
                assert 'mlb_forward' in str(e) and len(str(e)) > 20, e
                continue
            k = eng.last_kernel()[0]
            ran.append(fam if k == KERNEL_ID[fam] else '%s->%s' % (fam, [f for f, i in KERNEL_ID.items() if i == k][0]))
        table[L] = ' '.join(ran)
        eng.close()
    assert table == EXPECTED_TABLE, {L: (table[L], EXPECTED_TABLE[L]) for L in WIDTHS if table[L] != EXPECTED_TABLE[L]}
    # beyond 16 rows wide2 is refused at every width, including batches the cost model would give to the tensor cores
    eng = engine.LocoEngine(synthetic.make_state_dict('loco', 34, 9, 1024, 1, 3))
    for B in (17, 1000):
        with pytest.raises(RuntimeError, match='mlb_forward'):
            eng.forward(torch.from_numpy(synthetic.make_inputs(B, 34, seed=2)).cuda(), kernel='wide2')
    eng.close()


# ------------------------------------------------------------------------------------------------ width x family x batch
def _batches(family, eng):
    n_sms = eng.n_sms
    if family == 'tile':
        tm = _pick_tm(31, n_sms)
        many = 2 * 16 * n_sms + 1
        return [(B, 2 * _pick_tm(B, n_sms)) for B in (2 * tm - 1, 2 * tm, 2 * tm + 1, many)]
    if family == 'cluster':
        return [(B, 16) for B in (1, 16, 17, 289)]
    if family == 'wide':
        return [(B, 32) for B in (1, 16, 17, 32, 33, 65)]
    if family == 'wide2':
        return [(B, 16) for B in (1, 15, 16)]
    g = eng.kernel_times()['tc_resident_clusters']
    return [(B, 64) for B in (63, 64, 65, 64 * g - 1, 64 * g + 1)]


@pytest.mark.parametrize('L', WIDTHS)
def test_width_family_batch_matrix(L):
    """LocoModel, 3 stages, raw keypoints in (MLB_IN_KPS): raw, x and xyzc of every served family at its batch edges
    against float64 (at most ~512 rows per case: every tile's first and last row and the ragged tail included)."""
    R, O, synthetic, engine, packing, L_ = _mods()
    sd = synthetic.make_state_dict('loco', 34, 9, L, 3, 10 + L)
    eng = engine.LocoEngine(sd)
    kk = synthetic.KITTI_K
    kinv = R.kinv32(kk)
    cases = [(fam, B, tile) for fam in FAMILIES if fam in served(L) for B, tile in _batches(fam, eng)]
    pool = synthetic.make_keypoints(max(B for _, B, _ in cases), seed=L)
    rng = np.random.RandomState(L)
    samples = {(fam, B): _sample(B, tile, rng) for fam, B, tile in cases}
    idx = np.unique(np.concatenate(list(samples.values())))
    x64, xb = R.preprocess_mono(pool[idx], kinv)
    raw64 = R.model_forward(sd, x64)
    raw32 = O.loco_model_forward(sd, _pre32(pool[idx], kinv))
    c64 = R.xyzc(pool[idx], kinv, raw64[:, 2])
    c32 = _xyzc32(pool[idx], kinv, raw32[:, 2])
    pos = {int(r): i for i, r in enumerate(idx)}
    kps_dev = torch.from_numpy(pool).cuda()
    for fam, B, _ in cases:
        out = _run(eng, fam, kps_dev[:B], kk=kk, kind=L_.IN_KPS, want_x=True, want_xyzc=True)
        s = samples[(fam, B)]
        j = np.array([pos[int(r)] for r in s])
        raw = out['raw'].cpu().numpy()[s]
        what = (L, fam, B)
        _check(R, fam, (fam, 'matrix', L), raw, raw64[j], raw32[j], what + ('raw',), pool=(raw64, raw32))
        ok, worst = O.close(raw, raw32[j], rtol=_old_rtol(fam, packing.padded_width(L)))
        assert ok, what + (worst,)
        assert (np.abs(out['x'].cpu().numpy()[s] - x64[j]) <= 4.5 * ULP * xb[j]).all(), what + ('x',)
        _check(R, fam, (fam, 'xyzc', L), out['xyzc'].cpu().numpy()[s], c64[j], c32[j], what + ('xyzc',), pool=(c64, c32))
        _dec_bit_identical(out, L_.DECODE_LOCO)
    eng.close()


# ------------------------------------------------------------------------------------------------ feature slice
def _feature_cases(synthetic, L):
    """(label, state dict, input kind, forward kwargs builder)."""
    return [('stereo', synthetic.make_state_dict('loco', 68, 10, L, 3, 20)),
            ('loco_s1', synthetic.make_state_dict('loco', 34, 9, L, 1, 21)),
            ('monoloco_o9', synthetic.make_state_dict('monoloco', 34, 9, L, 3, 22)),
            ('monoloco_o2', synthetic.make_state_dict('monoloco', 34, 2, L, 1, 23))]


@pytest.mark.parametrize('L', [300, 1024, 2048])
def test_feature_slice(L):
    """Stereo all-vs-all pairs, zero-centred mono, explicit dropout keep-masks, MonolocoModel with 9 (DECODE_MONO) and
    2 (DECODE_DB) outputs, 1 and 3 stages -- on every family that serves the width."""
    R, O, synthetic, engine, packing, L_ = _mods()
    kk = [[712.5, 1.75, 598.25], [0.0, 709.0, 183.5], [0.0, 0.0, 1.0]]   # skewed: K^-1[0, 1] != 0
    kinv = R.kinv32(kk)
    P = packing.padded_width(L)
    for label, sd in _feature_cases(synthetic, L):
        eng = engine.LocoEngine(sd)
        stereo = label == 'stereo'
        kps = synthetic.make_keypoints(72, seed=7)
        zc = label == 'monoloco_o9'
        masks = m = None
        if label == 'loco_s1':
            masks = (np.random.RandomState(8).uniform(size=(2, 72, P)) >= 0.2).astype(np.uint8)
            m = (masks[0][:, :L], masks[1][:, :L])
        if not stereo:
            x64, xb = R.preprocess_mono(kps, kinv, zero_center=zc)
            ref64 = R.model_forward(sd, x64, drop_masks=m)
            ref32 = O.model_forward(sd, _pre32(kps, kinv, zero_center=zc), drop_masks=m)
        for fam in FAMILIES:
            if fam not in served(L, stereo):
                continue
            key = (fam, 'feature', L)
            if stereo:
                nl, nr = (4, 4) if fam == 'wide2' else (9, 8)
                kl = synthetic.make_keypoints(nl, seed=5)
                kr = synthetic.make_keypoints(nr, seed=6, right=True)[1]
                out = _run(eng, fam, torch.from_numpy(kl).cuda(), x_right=torch.from_numpy(kr).cuda(), kk=kk,
                           kind=L_.IN_KPS_STEREO, want_x=True)
                x64, xb = R.preprocess_stereo(kl, kr, kinv)
                a, b = _pre32(kl, kinv), _pre32(kr, kinv)
                x32 = np.concatenate([np.repeat(a, nr, 0), np.repeat(a, nr, 0) - np.tile(b, (nl, 1))], 1)
                assert (np.abs(out['x'].cpu().numpy() - x64) <= 4.5 * ULP * xb).all(), (L, fam, label)
                _check(R, fam, key, out['raw'].cpu().numpy(), R.model_forward(sd, x64), O.model_forward(sd, x32),
                       (L, fam, label))
                _dec_bit_identical(out, L_.DECODE_LOCO)
                continue
            B = 16 if fam == 'wide2' else 72
            kw = dict(kk=kk, kind=L_.IN_KPS, zero_center=zc, want_x=True)
            if masks is not None:
                kw.update(dropout=True, drop_mask=torch.from_numpy(np.ascontiguousarray(masks[:, :B])).cuda())
            out = _run(eng, fam, torch.from_numpy(kps[:B]).cuda(), **kw)
            assert (np.abs(out['x'].cpu().numpy() - x64[:B]) <= 4.5 * ULP * xb[:B]).all(), (L, fam, label)
            _check(R, fam, key, out['raw'].cpu().numpy(), ref64[:B], ref32[:B], (L, fam, label), pool=(ref64, ref32))
            ok, worst = O.close(out['raw'].cpu().numpy(), ref32[:B], rtol=_old_rtol(fam, P))
            assert ok, (L, fam, label, worst)
            _dec_bit_identical(out, eng.decode_kind)
        eng.close()


# ------------------------------------------------------------------------------------------------ negative control
def test_perturbed_checkpoint_is_rejected():
    """An engine built from w_fin.weight[2, 100] * (1 + 1e-3), compared with the float64 reference of the unperturbed
    checkpoint: the 1e-5 rule passes it, the float64 rule rejects it on every FFMA family.  For the tensor-core kernel the
    smallest rejected relative perturbation (of 1e-3 ... 1e-1) is recorded."""
    R, O, synthetic, engine, packing, L_ = _mods()
    sd = synthetic.make_state_dict('loco', 34, 9, 1024, 3, 0)
    x = synthetic.make_inputs(1024, 34, seed=0)
    ref64, ref32 = R.model_forward(sd, x), O.loco_model_forward(sd, x)
    rows = {'wide2': 16, 'wide': 64}
    report = {}
    for rel in (1e-3, 3e-3, 1e-2, 3e-2, 1e-1):
        sd2 = dict(sd)
        w = sd['w_fin.weight'].copy()
        w[2, 100] = np.float32(w[2, 100] * (1 + rel))
        sd2['w_fin.weight'] = w
        eng = engine.LocoEngine(sd2)
        for fam in FAMILIES if rel == 1e-3 else ('tc',):
            B = rows.get(fam, 1024)
            out = _run(eng, fam, torch.from_numpy(x[:B]).cuda())
            got = out['raw'].cpu().numpy()
            mx, rms = R.fp64_rule(got, ref64[:B], ref32[:B], pool=(ref64, ref32))
            lim = _rule(R, fam)
            rejected = bool((mx > lim[0]).any() or (rms > lim[1]).any())
            report[(fam, rel)] = (O.close(got, ref32[:B])[1], float(mx.max()), float(rms.max()), rejected)
            # [[old rule worst / tol], [new rule max ratio, RMS ratio]]
            RATIOS[(fam, 'negative_control', rel)] = [[report[(fam, rel)][0]], [float(mx.max()), float(rms.max())]]
            if fam != 'tc':
                assert O.close(got, ref32[:B])[0] and rejected, (fam, report[(fam, rel)])
        eng.close()
        if report[('tc', rel)][3]:
            break
    assert report[('tc', rel)][3], report


# ------------------------------------------------------------------------------------------------ weight refresh
def _edge_positions(sd, L):
    """(tensor, index) at the packers' boundaries: first / last real row and column, rows 7/8 and 31/32 (whole-grid CTA
    and wide2 cluster column groups), 255/256 (tensor-core CTA slices), K at the KC = 8 and TCKB = 16 block edges, each
    head row's last weight, BN parameters and running statistics of the last real column, a head bias, a plain bias."""
    last = L - 1
    cols = sorted({0, 7, 8, 15, 16, 31, 32, 255, 256, last} & set(range(L)))
    pos = []
    for r, k in ((0, 0), (last, 33), (7, 8), (8, 7), (31, 32), (32, 15), (255, 16), (256, 0), (last, 0)):
        pos.append(('w1.weight', (r, k)))
    for name in ('linear_stages.0.w1.weight', 'linear_stages.0.w2.weight'):
        for r in cols:
            pos.append((name, (r, cols[(cols.index(r) + 3) % len(cols)])))
    pos += [('w2.weight', (last, last)), ('w2.weight', (0, last)), ('w3.weight', (last, 255 if L > 256 else 0)),
            ('w3.weight', (256 if L > 256 else 1, last))]
    pos += [('w_fin.weight', (r, last)) for r in range(sd['w_fin.weight'].shape[0])] + [('w_aux.weight', (0, last))]
    for bn in ('batch_norm1', 'linear_stages.0.batch_norm2', 'batch_norm3'):
        pos += [(bn + '.' + p, (last,)) for p in ('weight', 'bias', 'running_mean', 'running_var')]
    pos += [('w_fin.bias', (2,)), ('w_aux.bias', (0,)), ('w2.bias', (last,)), ('linear_stages.0.w1.bias', (0,))]
    return [(n, i) for n, i in dict.fromkeys(pos) if all(a < s for a, s in zip(i, sd[n].shape))]


@pytest.mark.parametrize('L', [300, 1024, 2048])
def test_refresh_packing_edges(L):
    """Engine A runs once on every family; then, one position at a time, the base checkpoint with ONE element changed by
    half the tensor's max |value| is refreshed through update_weights (each state differs from the base in that element
    only, so an element left over from the previous refresh is an error too).  On every family the output must be
    bit-identical to that of a new engine built from the same checkpoint, follow float64 within the rule of the new
    state, and move with the float64 change wherever that change exceeds what the family's rule allows on either side.  A stale or mis-indexed packed copy (cluster slab, whole-grid slab, wide2 slab,
    tensor-core planes) fails here."""
    R, O, synthetic, engine, packing, L_ = _mods()
    base = {k: np.array(v) for k, v in synthetic.make_state_dict('loco', 34, 9, L, 1, 30).items()}
    eng = engine.LocoEngine(base)
    fams = [f for f in FAMILIES if f in served(L)]
    x = synthetic.make_inputs(48, 34, seed=31)
    xd = torch.from_numpy(x).cuda()
    rows = {f: 16 if f == 'wide2' else 48 for f in fams}
    out_a = {f: _run(eng, f, xd[:rows[f]])['raw'].cpu().numpy() for f in fams}
    ref64_a = R.model_forward(base, x)
    moved = dict.fromkeys(fams, 0)
    positions = _edge_positions(base, L)
    for name, i in positions:
        sd = dict(base)
        t = base[name].copy()
        t[i] = np.float32(t[i] + 0.5 * np.abs(t).max())
        sd[name] = t
        eng.update_weights(sd)
        ref64, ref32 = R.model_forward(sd, x), O.loco_model_forward(sd, x)
        noise = np.maximum(np.abs(ref32 - ref64).max(0), ULP * np.abs(ref64).max(0))
        d64 = ref64 - ref64_a
        fresh = engine.LocoEngine(sd)
        for f in fams:
            n = rows[f]
            got = _run(eng, f, xd[:n])['raw'].cpu().numpy()
            # exact: the refreshed packed copies are the ones a new engine packs from the same checkpoint
            new = _run(fresh, f, xd[:n])['raw'].cpu().numpy()
            assert np.array_equal(got.view(np.uint32), new.view(np.uint32)), (L, f, name, i)
            _check(R, f, (f, 'refresh', L), got, ref64[:n], ref32[:n], (L, f, name, i), pool=(ref64, ref32))
            # both states are within the rule: a change beyond twice the rule's max ratio (x 2 margin) must show, signed
            visible = np.abs(d64[:n]) > 4 * _rule(R, f)[0] * noise
            moved[f] += bool(visible.any())
            d = got - out_a[f]
            assert (np.sign(d[visible]) == np.sign(d64[:n][visible])).all(), (L, f, name, i)
        fresh.close()
    RATIOS[('all', 'refresh_positions', L)] = [[len(positions)], [moved[f] for f in fams]]
    for f in fams:
        assert moved[f] >= 0.5 * len(positions), (f, moved[f], len(positions))
    eng.close()


def test_refresh_user_path():
    """The training workflow: LocoModel in eval mode, one train_step + FusedClipAdam step, then the eval forward on every
    family follows the new weights.  A checkpoint of another width: LocoModel.load_state_dict refuses it (torch's shape
    check), so the model's engine meets one only through LocoEngine.update_weights, which re-creates it."""
    R, O, synthetic, engine, packing, L_ = _mods()
    from monoloco_b200.network.architectures import LocoModel
    from monoloco_b200.train import FusedClipAdam, train_step
    sd0 = synthetic.make_state_dict('loco', 34, 9, 1024, 1, 40)
    m = LocoModel(34, 9, 1024, num_stage=1)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd0.items()})
    m = m.cuda().eval()
    x = synthetic.make_inputs(48, 34, seed=41)
    xd = torch.from_numpy(x).cuda()
    n = lambda f: 16 if f == 'wide2' else 48  # noqa: E731
    with torch.no_grad():
        m(xd)
    m.train()
    opt = FusedClipAdam(m.parameters(), lr=1e-3, max_norm=3.0)
    opt.zero_grad()
    train_step(m, torch.from_numpy(synthetic.make_inputs(64, 34, seed=42)).cuda(),
               torch.from_numpy(synthetic.make_labels(64, seed=43)).cuda(), ('d', 'x', 'y', 'h', 'w', 'l', 'ori'))
    opt.step()
    m.eval()
    sd1 = {k: v.detach().cpu().numpy() for k, v in m.state_dict().items()}
    assert any(not np.array_equal(sd1[k], sd0[k]) for k in sd0 if k.endswith('weight'))
    ref64, ref32 = R.model_forward(sd1, x), O.loco_model_forward(sd1, x)
    with torch.no_grad():
        eng = m.engine()
        for f in FAMILIES:
            _check(R, f, (f, 'user_path', 1024), _run(eng, f, xd[:n(f)])['raw'].cpu().numpy(), ref64[:n(f)], ref32[:n(f)],
                   ('user', f), pool=(ref64, ref32))
    for L in (300, 2048):
        sd2 = synthetic.make_state_dict('loco', 34, 9, L, 1, 44)
        with pytest.raises(RuntimeError, match='size mismatch'):
            m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd2.items()})
        eng.update_weights(sd2)
        assert eng.linear_size == packing.padded_width(L)
        ref64, ref32 = R.model_forward(sd2, x), O.loco_model_forward(sd2, x)
        for f in FAMILIES:
            if f in served(L):
                _check(R, f, (f, 'user_path', L), _run(eng, f, xd[:n(f)])['raw'].cpu().numpy(), ref64[:n(f)],
                       ref32[:n(f)], ('reload', L, f), pool=(ref64, ref32))
    eng.close()


# ------------------------------------------------------------------------------------------------ degenerate detections
def _degenerate_keypoints():
    rng = np.random.RandomState(50)
    k = rng.uniform(100, 1100, size=(16, 3, 17)).astype(np.float32)
    k[0, 0, :], k[0, 1, :] = 640.5, 200.25                            # zero-size box
    k[1, :, 3:9] = 0.0                                                # PifPaf zero-confidence joints at (0, 0)
    k[2, 0, :] = rng.uniform(-500, -1, 17)                            # negative pixels
    k[3, 0, :], k[3, 1, :] = rng.uniform(1300, 2500, 17), rng.uniform(-300, 900, 17)   # off-image
    k[4, 0:2, :] = rng.uniform(9.0e3, 1.1e4, size=(2, 17))            # ~1e4 px
    k[5, 0:2, :] = -rng.uniform(9.0e3, 1.1e4, size=(2, 17))
    k[6, 0, :] = np.float32(1e4)                                      # zero-width box far out
    k[7, :, :] = 0.0                                                  # every joint missing
    return k


def test_degenerate_detections_preprocess():
    """Degenerate detections through mlb_preprocess and the fused prologue of every family (mono, zero-centred mono,
    stereo) with a skewed K: within 4.5 fp32 ulps of sum |terms| * z_met of float64, componentwise."""
    R, O, synthetic, engine, packing, L_ = _mods()
    kps = _degenerate_keypoints()
    for kk in ([[712.5, 1.75, 598.25], [0.0, 709.0, 183.5], [0.0, 0.0, 1.0]], synthetic.KITTI_K):
        kinv = R.kinv32(kk)
        assert kinv[1] != 0 or kk is synthetic.KITTI_K
        for zc in (False, True):
            x64, xb = R.preprocess_mono(kps, kinv, zero_center=zc)
            got = engine.preprocess_device(torch.from_numpy(kps).cuda(), kk, zero_center=zc).cpu().numpy()
            assert (np.abs(got - x64) <= 4.5 * ULP * xb).all(), ('mlb_preprocess', zc)
        eng = engine.LocoEngine(synthetic.make_state_dict('loco', 34, 9, 1024, 1, 51))
        for f in FAMILIES:
            for zc in (False, True):
                out = _run(eng, f, torch.from_numpy(kps).cuda(), kk=kk, kind=L_.IN_KPS, zero_center=zc, want_x=True)
                x64, xb = R.preprocess_mono(kps, kinv, zero_center=zc)
                assert (np.abs(out['x'].cpu().numpy() - x64) <= 4.5 * ULP * xb).all(), (f, zc)
                assert np.isfinite(out['raw'].cpu().numpy()).all(), (f, zc)
        eng.close()
        eng = engine.LocoEngine(synthetic.make_state_dict('loco', 68, 10, 1024, 1, 52))
        left, right = kps[:4], kps[4:8]
        x64, xb = R.preprocess_stereo(left, right, kinv)
        for f in FAMILIES:
            out = _run(eng, f, torch.from_numpy(left).cuda(), x_right=torch.from_numpy(right).cuda(), kk=kk,
                       kind=L_.IN_KPS_STEREO, want_x=True)
            assert (np.abs(out['x'].cpu().numpy() - x64) <= 4.5 * ULP * xb).all(), ('stereo', f)
        eng.close()


# ------------------------------------------------------------------------------------------------ decode edges
def _decode_edge_rows():
    d = [0.0, -1.0, 1e-40, 1e30]
    s = [-100.0, 0.0, 88.0, 89.0]
    ang = [0.0, math.pi / 2, -math.pi / 2, 1e4, 1.3]
    ori = [(0.0, 0.0), (-0.0, -0.0), (0.0, -1.0)]
    aux = [100.0, -100.0, 20.0, -20.0, 0.0]
    rows = []
    for a in d:
        for b in s:
            for th in ang:
                for ps in ang:
                    for o in ori:
                        for x in aux:
                            rows.append([th, ps, a, b, 1.7, 0.6, 0.8, o[0], o[1], x])
    return np.array(rows, dtype=np.float32)


@pytest.mark.parametrize('kind', ['loco10', 'loco9', 'mono', 'db'])
def test_decode_edge_table(kind):
    """mlb_decode on d in {0, -1, denormal, 1e30}, log-scale in {-100, 0, 88, 89}, theta / psi at 0, +-pi/2, 1e4,
    ori (0, 0), (-0, -0), (0, -1), aux in {+-100, +-20, 0}: NaN and +-inf exactly where the fp32 oracle has them; finite
    well-conditioned columns (x, y, d, bi, yaw_pred, aux) within 8 fp32 ulps of float64."""
    R, O, synthetic, engine, packing, L_ = _mods()
    raw = _decode_edge_rows()
    if kind == 'loco9':
        raw = raw[:, :9]
    if kind == 'db':
        raw = np.ascontiguousarray(raw[:, 2:4])
    code = {'loco10': L_.DECODE_LOCO, 'loco9': L_.DECODE_LOCO, 'mono': L_.DECODE_MONO, 'db': L_.DECODE_DB}[kind]
    got = _decode_dev(torch.from_numpy(raw).cuda(), code).cpu().numpy().astype(np.float64)
    ref64 = R.decode(raw, code)
    with np.errstate(all='ignore'):
        if code == L_.DECODE_LOCO:
            o = O.extract_outputs(raw)
            ref32 = np.concatenate([o['xyzd'], o['bi'], o['yaw'][0], o['yaw'][1],
                                    o['aux'] if raw.shape[1] == 10 else np.zeros((len(raw), 1), np.float32)], 1)
        elif code == L_.DECODE_MONO:
            o = O.extract_outputs_mono(raw)
            ref32 = np.concatenate([o['xyzd'], o['bi'], o['yaw'][0], o['yaw'][1], np.zeros((len(raw), 1), np.float32)], 1)
        else:
            ref32 = np.zeros((len(raw), 8), np.float32)
            ref32[:, 3:4], ref32[:, 4:5] = raw[:, 0:1], O.unnormalize_bi(raw)
    ref32 = ref32.astype(np.float64)
    # z = sqrt(d^2 - x^2 - y^2) (and yaw_orig through it) is NaN or not by the sign of a residual; where that residual is
    # within rounding of zero the sign belongs to the sin / cos implementation, not to the kernel: skipped there
    check = np.ones(got.shape, dtype=bool)
    if code == L_.DECODE_LOCO:
        d, x, y = ref64[:, 3], ref64[:, 0], ref64[:, 1]
        with np.errstate(all='ignore'):
            resid = d * d - x * x - y * y
            robust = (np.abs(resid) > 1e-5 * d * d) | (d == 0) | ~np.isfinite(np.float32(d) ** 2)
        check[~robust, 2] = check[~robust, 6] = False
    for what, f in (('nan', np.isnan), ('+inf', np.isposinf), ('-inf', np.isneginf)):
        bad = (f(got) != f(ref32)) & check
        assert not bad.any(), (kind, what, np.argwhere(bad)[:5].tolist(), raw[np.argwhere(bad)[0][0]].tolist())
    # well-conditioned columns; exp / sigmoid only where fp32 exp neither overflows nor goes subnormal
    s_col, a_col = (1, None) if code == L_.DECODE_DB else (3, 9 if raw.shape[1] == 10 else None)
    rows_ok = {4: np.abs(raw[:, s_col]) <= 88.0}
    if a_col is not None:
        rows_ok[7] = np.abs(raw[:, a_col]) <= 20.0
    cond = [3, 4] + ([0, 1, 5] if code != L_.DECODE_DB else []) + ([7] if a_col is not None else [])
    for c in cond:
        fin = np.isfinite(ref32[:, c]) & np.isfinite(ref64[:, c]) & (np.abs(ref64[:, c]) < 3.4e38)
        fin &= rows_ok.get(c, True) & ((np.abs(ref64[:, c]) > 1e-30) | (ref64[:, c] == 0) | (c != 3))
        ulp = np.maximum(np.spacing(np.abs(ref64[fin, c]).astype(np.float32)).astype(np.float64), 2.0 ** -149)
        err = np.abs(got[fin, c] - ref64[fin, c]) / ulp
        assert (err <= 8).all(), (kind, c, float(err.max()), raw[fin][np.argmax(err)].tolist())
