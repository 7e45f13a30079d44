"""GPU: the activity heuristics for many images in one launch (mlb_social_distance / mlb_raising_hand,
social_distance_device / raising_hand_device, Loco.social_distance_batch / raising_hand_batch).  Every flag must equal
the reference's (tests/golden/ref_activity_batch.npz) and the host mirror's (monoloco_b200.activity) exactly."""
import ctypes as C
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_activity_batch_cpu import images  # noqa: E402  (fixture reader)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CODES = (None, 'left', 'right', 'both')


@pytest.fixture(scope='module')
def fix():
    return np.load(os.path.join(GOLDEN, 'ref_activity_batch.npz'))


def _device_flags(imgs, cfg, **kw):
    """One launch over the images [(centers, angles, dds, stds), ...] -> list of per-image flag lists."""
    from monoloco_b200.network.post import social_distance_device
    counts = [len(c) for c, _, _, _ in imgs]
    n = sum(counts)
    cat = lambda i, w: np.concatenate([np.asarray(im[i], dtype=np.float64).reshape(-1, w) for im in imgs] or  # noqa: E731
                                      [np.zeros((0, w))]).reshape(n, w)
    xz = torch.from_numpy(cat(0, 2)).cuda()
    ang, dds, stds = (torch.from_numpy(cat(i, 1).reshape(n)).cuda() for i in (1, 2, 3))
    out = social_distance_device(xz, ang, dds.float(), stds.float(), np.cumsum([0] + counts), **cfg, **kw)
    assert out.dtype == torch.bool and out.is_cuda and out.shape == (n,)
    vals = out.cpu().tolist()
    off = np.cumsum([0] + counts)
    return [vals[off[i]:off[i + 1]] for i in range(len(imgs))]


def _mirror(centers, angles, dds, stds, cfg):
    from monoloco_b200.activity import social_interactions
    return [bool(social_interactions(i, centers, angles, dds, stds=stds, **cfg)) for i in range(len(centers))]


def test_device_flags_equal_reference_fixture(fix):
    """Every person, image and parameter set of the fixture: all images of one parameter set in one launch, and each
    image in a launch of its own."""
    by_cfg = {}
    for centers, angles, dds, stds, cfg, ref in images(fix):
        by_cfg.setdefault(tuple(sorted(cfg.items())), []).append(((centers, angles, dds, stds), ref))
    assert len(by_cfg) == 6
    for key, items in by_cfg.items():
        cfg = dict(key)
        got = _device_flags([im for im, _ in items], cfg)
        for (im, ref), g in zip(items, got):
            assert g == ref, (len(im[0]), cfg)
        for im, ref in items:
            if len(im[0]):
                assert _device_flags([im], cfg)[0] == ref, (len(im[0]), cfg)


def test_raising_hand_equals_reference_fixture(fix):
    from monoloco_b200.network.post import raising_hand_device
    got = raising_hand_device(torch.from_numpy(fix['kps']).cuda())
    assert got.dtype == torch.int8
    assert got.cpu().tolist() == fix['raising'].tolist()


def test_random_images_equal_host_mirror():
    """300 seeded images of up to 24 people, every parameter set family, against the host mirror, flag for flag."""
    from monoloco_b200 import synthetic
    rng = np.random.RandomState(2024)
    cfgs = [dict(radii=(0.3, 0.5), social_distance=False, threshold_dist=2.0, n_samples=100, threshold_prob=0.25),
            dict(radii=(0.3, 0.5, 1.0), social_distance=True, threshold_dist=2.5, n_samples=100, threshold_prob=0.25),
            dict(radii=(0.5, 0.3, 0.8, 1.2), social_distance=False, threshold_dist=3.0, n_samples=33, threshold_prob=0.1),
            dict(radii=(0.3, 0.5), social_distance=True, threshold_dist=2.0, n_samples=1, threshold_prob=0.25),
            dict(radii=(1.0,), social_distance=False, threshold_dist=2.0, n_samples=0, threshold_prob=0.25)]
    groups = {k: [] for k in range(len(cfgs))}
    for i in range(300):
        n = int(rng.randint(0, 25))
        spacing = (0.3, float(rng.choice([1.5, 3.0])))
        groups[i % len(cfgs)].append(synthetic.make_crowd(n, seed=10_000 + i, spacing=spacing))
    flagged = total = 0
    for k, imgs in groups.items():
        got = _device_flags(imgs, cfgs[k])
        for im, g in zip(imgs, got):
            ref = _mirror(*im, cfgs[k])
            assert g == ref, (k, len(im[0]))
            flagged, total = flagged + sum(ref), total + len(ref)
    assert 0.1 * total < flagged < 0.9 * total


def test_random_poses_equal_host_mirror(fix):
    from monoloco_b200.activity import is_raising_hand
    from monoloco_b200.network.post import raising_hand_device
    rng = np.random.RandomState(5)
    base = fix['kps'][rng.randint(0, 16, 10_000)].copy()
    base[:, :2, :11] += rng.normal(0, 60, (10_000, 2, 11))
    base[::7, :2, :] = rng.uniform(0, 400, (len(base[::7]), 2, 17))          # unrelated joints
    base[::50, :2, 9] = base[::50, :2, 7]                                     # zero-length left forearm
    base[1::50, 1, 10] = base[1::50, 1, 6]                                    # right hand at shoulder height
    got = raising_hand_device(torch.from_numpy(base).cuda()).cpu().tolist()
    with np.errstate(invalid='ignore', divide='ignore'):
        ref = [CODES.index(is_raising_hand(k.tolist())) for k in base]
    assert got == ref
    assert set(ref) == {0, 1, 2, 3}


def _loco(seed=1):
    from monoloco_b200 import synthetic
    from monoloco_b200.network import Loco
    from monoloco_b200.network.architectures import LocoModel
    sd = synthetic.make_state_dict('loco', 34, 9, 1024, 3, seed)
    m = LocoModel(34, 9, 1024, num_stage=3)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    return Loco(model=m, mode='mono', device=torch.device('cuda'))


def test_end_to_end_batch_equals_per_image_methods():
    """forward_batch -> post_process_batch -> social_distance_batch / raising_hand_batch equals Loco.social_distance /
    raising_hand on the same dictionaries, key by key; social_distance_device on forward_images outputs (detection order)
    equals the host mirror in that order."""
    import copy
    import json
    from monoloco_b200 import engine
    from monoloco_b200.network import Loco
    from monoloco_b200.network.post import post_process_batch, social_distance_device
    net = _loco()
    with open(os.path.join(GOLDEN, 'pifpaf_002282.json')) as f:
        from monoloco_b200.network.process import preprocess_pifpaf
        boxes, kps = preprocess_pifpaf(json.load(f), im_size=(1238, 374))
    kk = [[718.3351, 0., 600.3891], [0., 718.3351, 181.5122], [0., 0., 1.]]
    sel = [list(range(16)), [], list(range(5)), list(range(3, 12)), [7]]
    kl = [[kps[j] for j in s] for s in sel]
    bl = [[boxes[j] for j in s] for s in sel]
    kks = [kk, kk, [[700., 0., 620.], [0., 700., 190.], [0., 0., 1.]], kk, kk]
    dics = net.forward_batch(kl, kks)
    posts = post_process_batch([(d, b, k, K, None) for d, b, k, K in zip(dics, bl, kl, kks)])
    args = SimpleNamespace(threshold_prob=0.25, threshold_dist=2.0, radii=(0.3, 0.5, 1.0))
    single = [Loco.raising_hand(Loco.social_distance(copy.deepcopy(p), args), k) for p, k in zip(posts, kl)]
    batch = Loco.raising_hand_batch(Loco.social_distance_batch([copy.deepcopy(p) for p in posts], args), kl)
    for a, b in zip(batch, single):
        assert a['social_distance'] == b['social_distance']
        assert a['raising_hand'] == b['raising_hand']
        assert sorted(a.keys()) == sorted(b.keys())
    assert batch[1]['social_distance'] == [] and batch[1]['raising_hand'] == []
    nd = Loco.social_distance_batch([None, {}], args)
    assert nd[0]['social_distance'] == [] and nd[1]['social_distance'] == []
    # device chain straight after forward_images, detection order
    eng = net.model.engine()
    counts = [len(k) for k in kl]
    off = engine.image_offsets(counts)
    x = torch.tensor(np.concatenate([np.asarray(k, dtype=np.float32).reshape(-1, 3, 17) for k in kl if k])).cuda()
    out = eng.forward_images(x, off, kks, want_xyzc=True)
    xyzc, dec = out['xyzc'], out['dec']
    flags = social_distance_device(xyzc[:, (0, 2)], dec[:, 5], dec[:, 3], dec[:, 4], off, threshold_prob=0.25,
                                   threshold_dist=2.0, radii=(0.3, 0.5, 1.0)).cpu().tolist()
    xz, d, ang = xyzc[:, (0, 2)].double().cpu().numpy(), dec.cpu().numpy().astype(np.float64), dec[:, 5].double().cpu()
    for i in range(len(counts)):
        a, b = off[i], off[i + 1]
        ref = _mirror(xz[a:b].tolist(), ang[a:b].tolist(), d[a:b, 3].tolist(), d[a:b, 4].tolist(),
                      dict(threshold_prob=0.25, threshold_dist=2.0, radii=(0.3, 0.5, 1.0)))
        assert flags[a:b] == ref, i


def test_invalid_laplace_arguments_raise_before_launch():
    from monoloco_b200 import _lib as L_
    from monoloco_b200.network import Loco
    args = SimpleNamespace(threshold_prob=0.25, threshold_dist=2.0, radii=(0.3, 0.5))
    dic = {'xyz_pred': [[0., 0., 5.], [0.5, 0., 5.2]], 'angles': [0.1, 3.0], 'dds_pred': [5., 5.2], 'stds_ale': [0.4, 0.0]}
    torch.cuda.synchronize()
    before = L_.lib().mlb_launch_count()
    with pytest.raises(ValueError):
        Loco.social_distance_batch([dic], args)
    with pytest.raises(ValueError):   # the per-image method raises there too (torch.distributions.Laplace)
        Loco.social_distance(dict(dic), args)
    assert L_.lib().mlb_launch_count() == before


def test_zero_one_people_and_the_people_cap():
    from monoloco_b200 import synthetic, _lib as L_
    cfg = dict(radii=(0.3, 0.5), social_distance=False, threshold_dist=2.0, n_samples=100, threshold_prob=0.25)
    empty, one = synthetic.make_crowd(0, seed=1), synthetic.make_crowd(1, seed=2)
    assert _device_flags([empty, one, empty], cfg) == [[], [False], []]
    assert _device_flags([one], cfg) == [[False]]
    big = synthetic.make_crowd(L_.SOCIAL_MAX_PEOPLE, seed=3, spacing=(0.3, 2.5))
    for c in (dict(cfg, n_samples=7), dict(cfg, n_samples=1)):
        got = _device_flags([one, big], c)
        assert got[0] == [False]
        rng = np.random.RandomState(4)
        from monoloco_b200.activity import social_interactions
        for idx in rng.choice(len(big[0]), 6, replace=False):
            ref = bool(social_interactions(int(idx), big[0], big[1], big[2], stds=big[3], **c))
            assert got[1][idx] == ref, idx
    over = synthetic.make_crowd(L_.SOCIAL_MAX_PEOPLE + 1, seed=5, spacing=(0.3, 2.5))
    torch.cuda.synchronize()
    before = L_.lib().mlb_launch_count()
    with pytest.raises(RuntimeError, match='max_people'):
        _device_flags([over], cfg)
    assert L_.lib().mlb_launch_count() == before


def test_4096_images_of_16_people_sampled_against_mirror():
    from monoloco_b200 import synthetic
    cfg = dict(radii=(0.3, 0.5, 1.0), social_distance=False, threshold_dist=2.0, n_samples=100, threshold_prob=0.25)
    imgs = [synthetic.make_crowd(16, seed=50_000 + i) for i in range(4096)]
    got = _device_flags(imgs, cfg)
    for i in np.random.RandomState(9).choice(4096, 24, replace=False):
        assert got[i] == _mirror(*imgs[i], cfg), i


def test_rejected_arguments_launch_nothing():
    from monoloco_b200 import _lib as L_
    from monoloco_b200.network.post import laplace_draw_table
    lib = L_.lib()
    n = 8
    off = torch.tensor([0, 3, 8], dtype=torch.int32, device='cuda')
    xz = torch.rand((n, 2), dtype=torch.float64, device='cuda') * 3
    ang = torch.rand((n,), dtype=torch.float64, device='cuda')
    dd = torch.full((n,), 5.0, device='cuda')
    sd = torch.full((n,), 0.5, device='cuda')
    table = laplace_draw_table(100 * 5).cuda()
    out = torch.empty((n,), dtype=torch.uint8, device='cuda')

    def call(**kw):
        a = L_.MlbSocialArgs()
        a.n_img, a.n_people, a.max_people, a.n_samples, a.n_radii = 2, n, 5, 100, 2
        a.threshold_prob, a.threshold_dist, a.radii[0], a.radii[1] = 0.25, 2.0, 0.3, 0.5
        a.table_len = table.numel()
        a.img_off, a.xz, a.angles, a.dds, a.stds, a.table, a.out = (off.data_ptr(), xz.data_ptr(), ang.data_ptr(),
                                                                      dd.data_ptr(), sd.data_ptr(), table.data_ptr(),
                                                                      out.data_ptr())
        for k, v in kw.items():
            setattr(a, k, v)
        return lib.mlb_social_distance(C.byref(a), None)

    torch.cuda.synchronize()
    before = lib.mlb_launch_count()
    for kw in (dict(n_img=0), dict(n_radii=0), dict(n_radii=9), dict(max_people=L_.SOCIAL_MAX_PEOPLE + 1),
               dict(max_people=-1), dict(n_people=-1), dict(table_len=100 * 5 - 1), dict(img_off=None), dict(xz=None),
               dict(angles=None), dict(out=None), dict(dds=None), dict(stds=None), dict(table=None)):
        assert call(**kw) != 0, kw
        assert lib.mlb_last_error().decode().startswith('mlb_social_distance'), kw
    assert lib.mlb_social_distance(None, None) != 0
    kps = torch.zeros((4, 3, 17), dtype=torch.float64, device='cuda')
    codes = torch.empty((4,), dtype=torch.int8, device='cuda')
    assert lib.mlb_raising_hand(None, 4, codes.data_ptr(), None) != 0
    assert lib.mlb_raising_hand(kps.data_ptr(), -1, codes.data_ptr(), None) != 0
    assert lib.mlb_last_error().decode().startswith('mlb_raising_hand')
    assert lib.mlb_launch_count() == before
    # the deterministic test needs neither draws nor distances
    assert call(n_samples=1, dds=None, stds=None, table=None, table_len=0) == 0
    assert call() == 0 and lib.mlb_raising_hand(kps.data_ptr(), 4, codes.data_ptr(), None) == 0
    assert lib.mlb_launch_count() == before + 3
    torch.cuda.synchronize()
