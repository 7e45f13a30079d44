"""GPU: many images in one forward launch (mlb_forward_images / LocoEngine.forward_images / Loco.forward_batch), each with
its own camera matrix.  A row of a multi-image launch must equal, bit for bit, the same row run alone with its image's K
on the same kernel; the automatic choice is checked against the oracle and Loco.forward_batch against the reference."""
import ctypes as C
import os

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
KERNELS = ('tile', 'cluster', 'wide', 'wide2', 'tc')


def _kks(n, seed):
    """n distinct camera matrices: focal length, skew and principal point all vary."""
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        f = rng.uniform(600., 1300.)
        out.append([[f, rng.uniform(-3., 3.), rng.uniform(400., 800.)], [0., f * rng.uniform(0.98, 1.02), rng.uniform(150., 400.)],
                    [0., 0., 1.]])
    return out


@pytest.fixture(scope='module')
def engines():
    from monoloco_b200 import synthetic, engine
    cache = {}

    def get(kind, isz, osz, L, st, seed):
        key = (kind, isz, osz, L, st, seed)
        if key not in cache:
            sd = synthetic.make_state_dict(kind, isz, osz, L, st, seed)
            cache[key] = (sd, engine.LocoEngine(sd))
        return cache[key]
    yield get
    for _, eng in cache.values():
        eng.close()


# rows per image for each forced kernel: inside its row limits, images straddling its tiles (wide: 32-row launches,
# cluster: 16-row clusters, tile: 2 * TM row tiles, tc: 64-row tiles), empty images at the start, middle and end.  The
# whole-grid kernel splits K by its row slots (16- or 32-row instantiation, picked by the rows left for the launch), so a
# row's sum order depends on that choice: its layouts keep every launch, batched or per image, above 16 rows.
MONO_LAYOUT = {'wide2': [0, 3, 0, 7, 5, 0], 'wide': [0, 20, 0, 30, 0], 'cluster': [0, 9, 14, 0, 25, 3, 40, 0],
               'tile': [0, 9, 14, 0, 25, 3, 40, 0, 31], 'tc': [0, 50, 30, 0, 70, 1, 100, 0]}
STEREO_LAYOUT = {'wide2': [(0, 0), (2, 3), (0, 0), (3, 2), (1, 4), (0, 0)], 'wide': [(0, 0), (3, 6), (0, 0), (4, 5), (2, 9), (0, 0)],
                 'cluster': [(0, 0), (3, 5), (0, 0), (6, 4), (2, 9), (0, 0)],
                 'tile': [(0, 0), (3, 5), (0, 0), (6, 4), (2, 9), (0, 0)], 'tc': [(0, 0), (8, 9), (5, 7), (0, 0), (10, 6), (0, 0)]}
OUT_KEYS = ('raw', 'dec', 'xyzc', 'x')


def _mono_case(eng, counts, kernel, zero_center=False, masks=None, seed=0):
    from monoloco_b200 import synthetic, engine, _lib as L_
    kps = synthetic.make_keypoints(sum(counts), seed=10 + seed)
    kks = _kks(len(counts), seed)
    off = engine.image_offsets(counts)
    kw = dict(want_xyzc=True, want_x=True, zero_center=zero_center, kernel=kernel)
    if masks is not None:
        kw.update(dropout=True)
    out = eng.forward_images(torch.from_numpy(kps).cuda(), off, kks, kind=L_.IN_KPS,
                             drop_mask=torch.from_numpy(masks).cuda() if masks is not None else None, **kw)
    ref = {k: [] for k in OUT_KEYS}
    for i in range(len(counts)):
        if counts[i] == 0:
            continue
        a, b = off[i], off[i + 1]
        m = torch.from_numpy(np.ascontiguousarray(masks[:, a:b])).cuda() if masks is not None else None
        o = eng.forward(torch.from_numpy(kps[a:b]).cuda(), kk=kks[i], kind=L_.IN_KPS, drop_mask=m, **kw)
        for k in OUT_KEYS:
            ref[k].append(o[k])
    torch.cuda.synchronize()
    return out, {k: torch.cat(v) for k, v in ref.items()}


def _assert_equal(out, ref, what):
    for k in OUT_KEYS:
        assert out[k].shape == ref[k].shape, (what, k)
        assert torch.equal(out[k], ref[k]), (what, k, (out[k] - ref[k]).abs().max().item())


@pytest.mark.parametrize('kernel', KERNELS)
def test_bit_identical_to_per_image_forward_mono(engines, kernel):
    from monoloco_b200 import _lib as L_
    lib = L_.lib()
    sd, eng = engines('loco', 34, 9, 1024, 3, 1)
    counts = MONO_LAYOUT[kernel]
    out, ref = _mono_case(eng, counts, kernel)
    assert lib.mlb_last_kernel(eng._h) == {'tile': 0, 'cluster': 1, 'wide': 2, 'tc': 3, 'wide2': 4}[kernel]
    _assert_equal(out, ref, kernel)
    # explicit MC-dropout keep masks [sites][B][L], sliced per image for the reference calls
    masks = (np.random.RandomState(5).uniform(size=(2, sum(counts), 1024)) >= 0.2).astype(np.uint8)
    out, ref = _mono_case(eng, counts, kernel, masks=masks, seed=1)
    _assert_equal(out, ref, kernel + ' masks')


@pytest.mark.parametrize('kernel', KERNELS)
def test_bit_identical_to_per_image_forward_zero_center(engines, kernel):
    """legacy monoloco: zero-centred pre-process (net.py:96) with every image's own K."""
    sd, eng = engines('monoloco', 34, 2, 1024, 3, 3)
    out, ref = _mono_case(eng, MONO_LAYOUT[kernel], kernel, zero_center=True, seed=2)
    _assert_equal(out, ref, kernel)


@pytest.mark.parametrize('kernel', KERNELS)
def test_bit_identical_to_per_image_forward_stereo(engines, kernel):
    from monoloco_b200 import synthetic, engine, _lib as L_
    sd, eng = engines('loco', 68, 10, 1024, 3, 2)
    lr = STEREO_LAYOUT[kernel]
    nl, nr = [a for a, _ in lr], [b for _, b in lr]
    left, right = synthetic.make_keypoints(sum(nl), seed=21), synthetic.make_keypoints(sum(nr), seed=22)
    kks = _kks(len(lr), 3)
    lo, ro = engine.image_offsets(nl), engine.image_offsets(nr)
    row_off = engine.image_offsets([a * b for a, b in lr])
    kw = dict(want_xyzc=True, want_x=True, kernel=kernel)
    out = eng.forward_images(torch.from_numpy(left).cuda(), row_off, kks, kind=L_.IN_KPS_STEREO,
                             x_right=torch.from_numpy(right).cuda(), left_off=lo, right_off=ro, **kw)
    ref = {k: [] for k in OUT_KEYS}
    for i in range(len(lr)):
        if nl[i] * nr[i] == 0:
            continue
        o = eng.forward(torch.from_numpy(left[lo[i]:lo[i + 1]]).cuda(), x_right=torch.from_numpy(right[ro[i]:ro[i + 1]]).cuda(),
                        kk=kks[i], kind=L_.IN_KPS_STEREO, **kw)
        for k in OUT_KEYS:
            ref[k].append(o[k])
    torch.cuda.synchronize()
    _assert_equal(out, {k: torch.cat(v) for k, v in ref.items()}, kernel)


@pytest.mark.parametrize('total', [10, 40, 130, 1000, 5000])
def test_automatic_kernel_choice_against_oracle(engines, total):
    from oracle import loco_oracle as O
    from monoloco_b200 import synthetic, engine, _lib as L_
    sd, eng = engines('loco', 34, 9, 1024, 3, 1)
    rng = np.random.RandomState(total)
    counts = []
    while sum(counts) < total:
        counts.append(int(min(rng.choice([0, 1, 3, 8, 16, 40]), total - sum(counts))))
    kks = _kks(len(counts), total)
    kps = synthetic.make_keypoints(total, seed=total)
    off = engine.image_offsets(counts)
    out = eng.forward_images(torch.from_numpy(kps).cuda(), off, kks, want_xyzc=True)
    torch.cuda.synchronize()
    kernel = eng.last_kernel()
    print('total %d rows, %d images: %s' % (total, len(counts), kernel[1]))
    live = [i for i in range(len(counts)) if counts[i]]
    raw_ref = np.concatenate([O.loco_model_forward(sd, O.preprocess_monoloco(kps[off[i]:off[i + 1]],
                                                                             np.asarray(kks[i], dtype=np.float32))) for i in live])
    refs = [O.loco_forward(sd, kps[off[i]:off[i + 1]], kks[i], mode='mono') for i in live]
    ref = {'xyzd': np.concatenate([r['xyzd'] for r in refs]), 'bi': np.concatenate([r['bi'] for r in refs]),
           'yaw': tuple(np.concatenate([r['yaw'][j] for r in refs]) for j in (0, 1))}
    ok, worst = O.close(out['raw'].cpu().numpy(), raw_ref)
    assert ok, (total, kernel, worst)
    _check_dec(O, out['dec'].cpu().numpy(), ref, raw_ref)


def _check_dec(O, dec, ref, raw_ref):
    """The decoded columns under the rule of test_forward_gpu.py: x, y, z, d against one scale max |d|, and the yaw
    tolerances conditioned by the reference raw outputs they are atan2 of."""
    ok, worst = O.close(dec[:, 0:4], ref['xyzd'], col_scale=False)
    assert ok, ('xyzd', worst)
    ok, worst = O.close(dec[:, 4:5], ref['bi'])
    assert ok, ('bi', worst)
    rad = np.hypot(raw_ref[:, 7:8], raw_ref[:, 8:9])
    lin = 1e-5 * float(np.abs(raw_ref[:, 7:9]).max()) + 1e-6
    xyzd = np.asarray(ref['xyzd'])
    rad2 = np.minimum(rad / lin, np.hypot(xyzd[:, 0:1], xyzd[:, 2:3]) / (1e-5 * float(np.abs(xyzd[:, 3]).max()) + 1e-6))
    ok, worst = O.angle_close(dec[:, 5:6], ref['yaw'][0], radius=rad, lin_tol=lin)
    assert ok, ('yaw_pred', worst)
    ok, worst = O.angle_close(dec[:, 6:7], ref['yaw'][1], rtol=3e-5, radius=rad2, lin_tol=2.0)
    assert ok, ('yaw_orig', worst)


def test_stereo_filter_images_equals_per_image_filter(engines):
    from monoloco_b200 import engine
    sd, eng = engines('loco', 68, 10, 1024, 3, 2)
    # (n_left, n_right): ties, a single right pose, an image without left poses and one without right poses
    lr = [(3, 4), (0, 0), (2, 1), (4, 5), (2, 0), (1, 3), (0, 2)]
    lo, ro = engine.image_offsets([a for a, _ in lr]), engine.image_offsets([b for _, b in lr])
    row_off = engine.image_offsets([a * b for a, b in lr])
    B = int(row_off[-1])
    rng = np.random.RandomState(7)
    raw = rng.standard_normal((B, 10)).astype(np.float32)
    raw[:, 9] = np.round(raw[:, 9] * 2) / 2   # many ties on the arg-max column
    raw[1:3, 9] = raw[9:12, 9] = 5.0          # certain ones: left poses 0 and 2 of image 0
    dec = rng.standard_normal((B, 8)).astype(np.float32)
    xyzc = rng.standard_normal((B, 4)).astype(np.float32)
    t = lambda a: torch.from_numpy(a).cuda()  # noqa: E731
    got = eng.stereo_filter_images(t(raw), t(dec), row_off, lo, ro, xyzc=t(xyzc))
    exp_raw, exp_dec, exp_xyzc, exp_idx, exp_off = [], [], [], [], [0]
    for i, (nl, nr) in enumerate(lr):
        if nl * nr:
            a, b = row_off[i], row_off[i + 1]
            r, d, idx, x = eng.stereo_filter(t(raw[a:b]), t(dec[a:b]), nl, nr, xyzc=t(xyzc[a:b]))
            exp_raw.append(r), exp_dec.append(d), exp_xyzc.append(x), exp_idx.append(idx + int(a))
            exp_off.append(exp_off[-1] + r.shape[0])
        else:
            exp_off.append(exp_off[-1])
    assert got['sel_img_off'] == exp_off
    assert torch.equal(got['sel_raw'], torch.cat(exp_raw)) and torch.equal(got['sel_dec'], torch.cat(exp_dec))
    assert torch.equal(got['sel_xyzc'], torch.cat(exp_xyzc)) and torch.equal(got['sel_idx'], torch.cat(exp_idx))
    assert exp_off[1] >= 6 and got['sel_idx'][:2].tolist() == [1, 2]   # tied rows are all kept, in order


def _load_module(kind, isz, osz, L, st, seed):
    from monoloco_b200 import synthetic
    from monoloco_b200.network.architectures import LocoModel, MonolocoModel
    sd = synthetic.make_state_dict(kind, isz, osz, L, st, seed)
    m = LocoModel(isz, osz, L, num_stage=st) if kind == 'loco' else MonolocoModel(isz, osz, L, num_stage=st)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    return m


def _cmp(O, dic, ref, keys):
    for k in keys:
        ok, worst = O.close(dic[k].numpy(), ref[k], col_scale=(k != 'xyzd'))
        assert ok, (k, worst)
    assert O.angle_close(dic['yaw'][0].numpy(), ref['yaw_pred'])[0]
    assert O.angle_close(dic['yaw'][1].numpy(), ref['yaw_orig'], rtol=3e-5)[0]


def _boxes(kps):
    """a detection box around every pose (x1, y1, x2, y2, confidence)"""
    k = np.asarray(kps, dtype=np.float64).reshape(-1, 3, 17)
    return [[k[i, 0].min() - 3, k[i, 1].min() - 5, k[i, 0].max() + 3, k[i, 1].max() + 5, 0.5 + 0.01 * i] for i in range(len(k))]


def test_forward_batch_matches_reference_fixture():
    from oracle import loco_oracle as O
    from monoloco_b200.network import Loco
    from monoloco_b200.network.post import post_process_batch
    f = np.load(os.path.join(GOLDEN, 'ref_loco_images.npz'))
    # mono
    n = f['mono_n']
    kps = [k.tolist() for k in np.split(f['mono_kps'], np.cumsum(n)[:-1])]
    kks = [k.tolist() for k in f['mono_K']]
    net = Loco(model=_load_module('loco', 34, 9, 1024, 3, 1), mode='mono', device=torch.device('cuda'))
    res = net.forward_batch(kps, kks)
    assert len(res) == len(n)
    o = np.concatenate([[0], np.cumsum(n)])
    for i in range(len(n)):
        if n[i] == 0:
            assert res[i] is None
            continue
        ref = {k[len('mono_out_'):]: f[k][o[i]:o[i + 1]] for k in f.files if k.startswith('mono_out_')}
        _cmp(O, res[i], ref, ('xyzd', 'bi', 'd', 'h', 'w', 'l', 'ori'))
        assert res[i]['epi'] == [0.] * int(n[i]) and all(not v.is_cuda for v in res[i].values() if isinstance(v, torch.Tensor))
    # post_process_batch on forward_batch's dictionaries = on the per-image Loco.forward dictionaries
    single = [net.forward(k, kk) for k, kk in zip(kps, kks)]
    items = lambda dics: [(d, _boxes(k) if len(k) else [], k, kk, None) for d, k, kk in zip(dics, kps, kks)]  # noqa: E731
    pa, pb = post_process_batch(items(res)), post_process_batch(items(single))
    for a, b in zip(pa, pb):
        assert sorted(a.keys()) == sorted(b.keys())
        for k in a:
            if k in ('boxes', 'uv_kps', 'uv_centers', 'uv_shoulders', 'uv_heads', 'gt'):
                assert a[k] == b[k], k
            else:
                assert np.allclose(np.array(a[k], dtype=np.float64), np.array(b[k], dtype=np.float64), rtol=3e-5, atol=2e-5), k
    # stereo, including an image without right poses (net.py:115-116)
    nl, nr = f['stereo_nl'], f['stereo_nr']
    lefts = [k.tolist() for k in np.split(f['stereo_left'], np.cumsum(nl)[:-1])]
    rs = np.split(f['stereo_right'], np.cumsum(np.maximum(nr, 0))[:-1])
    rights = [rs[i].tolist() if nr[i] >= 0 else None for i in range(len(nl))]
    net = Loco(model=_load_module('loco', 68, 10, 1024, 3, 2), mode='stereo', device=torch.device('cuda'))
    res = net.forward_batch(lefts, [k.tolist() for k in f['stereo_K']], rights)
    o = np.concatenate([[0], np.cumsum(nl)])
    for i in range(len(nl)):
        ref = {k[len('stereo_out_'):]: f[k][o[i]:o[i + 1]] for k in f.files if k.startswith('stereo_out_')}
        _cmp(O, res[i], ref, ('xyzd', 'bi', 'd', 'aux', 'ori', 'h', 'w', 'l'))
        assert res[i]['epi'] == [0.] * int(nl[i])


@pytest.mark.parametrize('net_name', ['monoloco_pp', 'monoloco_p', 'monoloco'])
def test_forward_batch_every_mono_net_equals_forward(net_name):
    """Same dictionary keys and values (to the parity rule: the kernel may differ with the batch size) as Loco.forward."""
    from oracle import loco_oracle as O
    from monoloco_b200 import synthetic
    from monoloco_b200.network import Loco
    kind, osz, L = {'monoloco_pp': ('loco', 9, 1024), 'monoloco_p': ('monoloco', 9, 256), 'monoloco': ('monoloco', 2, 1024)}[net_name]
    net = Loco(model=_load_module(kind, 34, osz, L, 3, 4), mode='mono', net=net_name, device=torch.device('cuda'))
    counts = [3, 0, 12, 1]
    kps = synthetic.make_keypoints(sum(counts), seed=8)
    off = np.concatenate([[0], np.cumsum(counts)])
    kl = [kps[off[i]:off[i + 1]].tolist() for i in range(len(counts))]
    kks = _kks(len(counts), 9)
    res = net.forward_batch(kl, kks)
    for i in range(len(counts)):
        one = net.forward(kl[i], kks[i])
        if one is None:
            assert res[i] is None
            continue
        assert sorted(res[i].keys()) == sorted(one.keys())
        for k, v in one.items():
            if k == 'yaw':
                for a, b in zip(res[i][k], v):
                    assert O.angle_close(a.numpy(), b.numpy(), rtol=3e-5)[0]
            elif k == 'epi':
                assert res[i][k] == v
            else:
                assert O.close(res[i][k].numpy(), v.numpy(), col_scale=(k not in ('xyzd', 'xyz_c')))[0], k


def test_forward_batch_epistemic_statistics():
    """MC dropout over all images in one launch: the same statistical check as test_epistemic_uncertainty_statistics, with
    the expectation from the engine's own passes (the counter RNG is keyed by the launch row, so no per-image equality)."""
    from monoloco_b200 import synthetic, engine, _lib as L_
    from monoloco_b200.network import Loco
    n_drop = 20
    net = Loco(model=_load_module('loco', 34, 9, 1024, 3, 1), mode='mono', device=torch.device('cuda'), n_dropout=n_drop)
    counts = [7, 0, 21, 12]
    kps = synthetic.make_keypoints(sum(counts), seed=3)
    off = engine.image_offsets(counts)
    kks = _kks(len(counts), 4)
    res = net.forward_batch([kps[off[i]:off[i + 1]].tolist() for i in range(len(counts))], kks)
    assert res[1] is None
    epi = np.concatenate([res[i]['epi'].numpy() for i in (0, 2, 3)])
    assert epi.shape == (40,) and np.isfinite(epi).all() and (epi > 0).all()
    assert net.model.dropout.training is False
    eng = net.model.engine()
    B = sum(counts)
    tiled = np.concatenate([[0]] + [off[1:] + p * B for p in range(n_drop)])
    out = eng.forward_images(torch.from_numpy(kps).cuda().repeat(n_drop, 1, 1), tiled, kks * n_drop, kind=L_.IN_KPS,
                             dropout=True, drop_seed=1)
    mus = out['raw'][:, 2].cpu().numpy().reshape(n_drop, -1)
    bis = np.abs(out['dec'][:, 4].cpu().numpy().reshape(n_drop, -1))
    assert np.abs(mus - mus[0]).max() > 1e-4
    expect = np.sqrt((2 * bis ** 2).mean(0) + mus.var(0))
    assert np.allclose(epi, expect, rtol=0.10), np.abs(epi / expect - 1).max()


def test_rejected_arguments_launch_nothing(engines):
    from monoloco_b200 import synthetic, engine, _lib as L_
    lib = L_.lib()
    sd, eng = engines('loco', 34, 9, 1024, 3, 1)
    x = torch.from_numpy(synthetic.make_keypoints(8, seed=1)).cuda()
    raw = torch.empty((8, 9), device='cuda')
    off = torch.from_numpy(engine.image_offsets([3, 5])).cuda()
    kinv = torch.from_numpy(engine.kinv_images(_kks(2, 1))).cuda()

    def call(kind=L_.IN_KPS, n_gather=0, n_img=2, row_off=True, kinv_p=True, images=True, left=False):
        a = L_.MlbForwardArgs()
        a.input_kind, a.n_rows, a.x, a.out_raw, a.z_met = kind, 8, x.data_ptr(), raw.data_ptr(), 10.0
        a.n_gather = n_gather
        if n_gather:
            a.gather[0] = raw.data_ptr()
        if kind == L_.IN_KPS_STEREO:
            a.n_left, a.n_right, a.x_right = 8, 1, x.data_ptr()
        ib = L_.MlbImageBatch()
        ib.n_img = n_img
        ib.row_off = off.data_ptr() if row_off else None
        ib.kinv = kinv.data_ptr() if kinv_p else None
        if left:
            ib.left_off = off.data_ptr()
        return lib.mlb_forward_images(eng._h, C.byref(a), C.byref(ib) if images else None, None)

    torch.cuda.synchronize()
    before = lib.mlb_launch_count()
    for kw in (dict(kind=L_.IN_X), dict(n_gather=1), dict(kinv_p=False), dict(row_off=False), dict(n_img=0),
               dict(images=False), dict(kind=L_.IN_KPS_STEREO, left=True)):
        assert call(**kw) != 0, kw
        assert lib.mlb_last_error().decode().startswith('mlb_forward_images'), kw
    assert lib.mlb_launch_count() == before
    with pytest.raises(ValueError):   # host-side checks of the Python layer
        eng.forward_images(x, [0, 3, 9], _kks(2, 1))
    with pytest.raises(ValueError):
        eng.forward_images(x, [0, 3, 8], _kks(3, 1))
    assert call() == 0 and lib.mlb_launch_count() == before + 1   # the same arguments, well-formed, do launch
    torch.cuda.synchronize()
