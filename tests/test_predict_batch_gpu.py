"""GPU: the predict chain for many images (mlb_preprocess_pifpaf, Loco.predict_batch).  The pre-process must equal the
live reference exactly (tests/golden/ref_predict_batch.npz); predict_batch must equal the four-call chain (host
preprocess_pifpaf, forward_batch, post_process_batch, social_distance_batch, raising_hand_batch) exactly, and the
reference's per-image chain (tests/golden/ref_predict_batch.json) under the project's 1e-5 rule."""
import copy
import json
import os
import sys
from collections import defaultdict
from types import SimpleNamespace

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from test_predict_batch_cpu import annotations, case, N_CASES  # noqa: E402  (fixture reader)

GOLDEN = os.path.join(ROOT, 'tests', 'golden')
ARGS = SimpleNamespace(threshold_prob=0.25, threshold_dist=2.0, radii=(0.3, 0.5, 1.0))
ARGS_WIDE = SimpleNamespace(threshold_prob=0.25, threshold_dist=8.0, radii=(0.5, 2.0, 5.0))
CLOSE = ('confs', 'dds_pred', 'stds_ale', 'xyz_pred', 'aux', 'xyz_real')
ANGLES = ('angles', 'angles_egocentric')


@pytest.fixture(scope='module')
def fix():
    return np.load(os.path.join(GOLDEN, 'ref_predict_batch.npz'))


@pytest.fixture(scope='module')
def chain():
    with open(os.path.join(GOLDEN, 'ref_predict_batch.json')) as f:
        return json.load(f)


def _loco(mode='mono', n_dropout=0):
    from monoloco_b200 import synthetic
    from monoloco_b200.network import Loco
    from monoloco_b200.network.architectures import LocoModel
    stereo = mode == 'stereo'
    sd = synthetic.make_state_dict('loco', 68 if stereo else 34, 10 if stereo else 9, 1024, 3, 2 if stereo else 1)
    m = LocoModel(68 if stereo else 34, 10 if stereo else 9, 1024, num_stage=3)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    return Loco(model=m, mode=mode, device=torch.device('cuda'), n_dropout=n_dropout)


def _four_calls(net, ann_list, kks, sizes, ann_r_list=None, gts=None, enlarge_boxes=False, min_conf=0., activities=(),
                args=None, reorder=True):
    """The same chain through the per-stage batch calls."""
    from monoloco_b200.network import Loco
    from monoloco_b200.network.process import preprocess_pifpaf
    from monoloco_b200.network.post import post_process_batch
    pre = [preprocess_pifpaf(a, s, enlarge_boxes=enlarge_boxes, min_conf=min_conf) for a, s in zip(ann_list, sizes)]
    bl, kl = [b for b, _ in pre], [k for _, k in pre]
    krl = [preprocess_pifpaf(a, s)[1] for a, s in zip(ann_r_list, sizes)] if ann_r_list is not None else None
    dics = net.forward_batch(kl, kks, krl)
    posts = post_process_batch([(d, b, k, K, g) for d, b, k, K, g in
                                zip(dics, bl, kl, kks, gts if gts is not None else [None] * len(kl))], reorder=reorder)
    if 'social_distance' in activities:
        posts = Loco.social_distance_batch(posts, args)
    if 'raise_hand' in activities:
        posts = Loco.raising_hand_batch(posts, kl)
    return list(zip(bl, kl, posts))


def _same(got, ref, what):
    assert len(got) == len(ref), what
    for i, ((b, k, d), (rb, rk, rd)) in enumerate(zip(got, ref)):
        assert b == rb and k == rk, (what, i)
        assert isinstance(d, defaultdict), (what, i)
        assert list(d.keys()) == list(rd.keys()), (what, i, list(d.keys()), list(rd.keys()))
        for key in rd:
            assert d[key] == rd[key], (what, i, key)


def _chain_inputs(chain, mode):
    ims = chain[mode]['images']
    return ([im['ann'] for im in ims], [im['kk'] for im in ims], [tuple(im['im_size']) if im['im_size'] else None for im in ims],
            [im['ann_r'] for im in ims], [im['gt'] for im in ims])


def _crowd(n_img, per_img, seed):
    """n_img images of up to per_img annotations drawn from the pifpaf fixture, shifted, some with a score."""
    with open(os.path.join(GOLDEN, 'pifpaf_002282.json')) as f:
        base = json.load(f)
    rng = np.random.RandomState(seed)
    ann_list, kks, sizes = [], [], []
    for i in range(n_img):
        anns = []
        for j in rng.choice(len(base), size=int(rng.randint(0, per_img + 1)), replace=True):
            a = copy.deepcopy(base[int(j)])
            s = float(rng.uniform(-60, 60))
            a['keypoints'][0::3] = [x + s for x in a['keypoints'][0::3]]
            a['bbox'] = [a['bbox'][0] + s, a['bbox'][1], a['bbox'][2] + s, a['bbox'][3]]
            if rng.uniform() < 0.3:
                x1, y1, x2, y2 = a['bbox']
                a = {'keypoints': a['keypoints'], 'bbox': [x1, y1, x2 - x1, y2 - y1], 'score': float(rng.uniform(0, 1))}
            anns.append(a)
        ann_list.append(anns)
        kks.append([[700. + i % 50, 0., 610.], [0., 700. + i % 50, 180.], [0., 0., 1.]])
        sizes.append((1238., 374.) if i % 5 else None)
    return ann_list, kks, sizes


def test_preprocess_kernel_equals_reference(fix):
    from monoloco_b200.network.process import pack_pifpaf, preprocess_pifpaf_device
    ann_list, sizes = annotations(fix)
    p = pack_pifpaf(ann_list, sizes)
    arrays = {k: torch.from_numpy(v).cuda() for k, v in p.items()}
    for c in range(N_CASES):
        enlarge, min_conf = case(fix, c)
        out = preprocess_pifpaf_device(arrays, len(ann_list), len(p['kps']), 1 if enlarge else 2, min_conf)
        off = out['kept_off'].cpu().numpy()
        n = int(off[-1])
        assert int(out['error'].item()) == 0
        assert np.array_equal(off, fix['c%d_off' % c]), c
        assert np.array_equal(out['src'][:n].cpu().numpy(), fix['c%d_src' % c]), c
        assert np.array_equal(out['boxes'][:n].cpu().numpy(), fix['c%d_boxes' % c]), c
        assert np.array_equal(out['kps'][:n].cpu().numpy(), fix['c%d_kps' % c]), c
        assert np.array_equal(out['kps32'][:n].cpu().numpy(), fix['c%d_kps' % c].astype(np.float32)), c


@pytest.mark.parametrize('n_dropout', [0, 4])
def test_predict_batch_equals_four_calls_mono(chain, n_dropout):
    net = _loco('mono', n_dropout)
    ann_list, kks, sizes, _, gts = _chain_inputs(chain, 'mono')
    crowd = _crowd(40, 9, seed=3)
    for anns, k, s, g, kw in ((ann_list, kks, sizes, gts, dict(activities=('social_distance', 'raise_hand'), args=ARGS)),
                              (ann_list, kks, sizes, None, dict(activities=('raise_hand',), enlarge_boxes=True, min_conf=0.3)),
                              (crowd[0], crowd[1], crowd[2], None, dict(activities=('social_distance',), args=ARGS_WIDE)),
                              (ann_list, kks, sizes, gts, dict(reorder=False))):
        before = copy.deepcopy(anns)
        got = net.predict_batch(anns, k, s, dic_gt_list=g, **kw)
        assert anns == before
        _same(got, _four_calls(net, anns, k, s, gts=g, **kw), kw)


def test_predict_batch_equals_four_calls_stereo(chain):
    net = _loco('stereo')
    ann_list, kks, sizes, ann_r, gts = _chain_inputs(chain, 'stereo')
    got = net.predict_batch(ann_list, kks, sizes, annotations_r_list=ann_r, dic_gt_list=gts, activities=('raise_hand',))
    _same(got, _four_calls(net, ann_list, kks, sizes, ann_r_list=ann_r, gts=gts, activities=('raise_hand',)), 'stereo')
    got = net.predict_batch(ann_list, kks, sizes)   # no right annotations: every image pairs with its first left pose
    _same(got, _four_calls(net, ann_list, kks, sizes, ann_r_list=[[]] * len(ann_list)), 'stereo, no right')


@pytest.mark.parametrize('mode', ['mono', 'stereo'])
def test_predict_batch_against_reference(chain, mode):
    from oracle import loco_oracle as O
    net = _loco(mode)
    ann_list, kks, sizes, ann_r, gts = _chain_inputs(chain, mode)
    stereo = mode == 'stereo'
    got = net.predict_batch(ann_list, kks, sizes, annotations_r_list=ann_r if stereo else None, dic_gt_list=gts,
                            activities=() if stereo else ('social_distance', 'raise_hand'), args=ARGS)
    n_sd = 0
    for i, ((b, k, d), im) in enumerate(zip(got, chain[mode]['images'])):
        rb, rk, rd = im['out']
        assert b == rb and k == rk, i
        assert list(d.keys()) == list(rd.keys()), (i, list(d.keys()), list(rd.keys()))
        for key, ref in rd.items():
            if key in CLOSE:
                if len(ref):
                    ok, worst = O.close(np.asarray(d[key], dtype=np.float64), np.asarray(ref, dtype=np.float64))
                    assert ok, (i, key, worst)
                else:
                    assert d[key] == ref, (i, key)
            elif key in ANGLES:
                assert len(d[key]) == len(ref) and O.angle_close(np.asarray(d[key]), np.asarray(ref))[0], (i, key)
            elif key == 'social_distance':
                clear = im['sd_clear']
                assert len(d[key]) == len(ref)
                assert [g for g, c in zip(d[key], clear) if c] == [r for r, c in zip(ref, clear) if c], i
                n_sd += sum(clear)
            else:   # order, matches, boxes, key points, pixels, ground truth, raised hands, epistemic 0
                assert d[key] == ref, (i, key)
    assert stereo or n_sd > 20


def test_degenerate_box_raises_after_preprocess_only():
    from monoloco_b200 import _lib as L_
    from monoloco_b200.network.process import preprocess_pifpaf
    net = _loco('mono')
    with open(os.path.join(GOLDEN, 'pifpaf_002282.json')) as f:
        base = json.load(f)
    bad = copy.deepcopy(base[:3])
    bad[1]['bbox'] = [100.0, 300.0, 150.0, 100.0]   # (y2 - y1) / 14 = -14.3 <= -5
    kk = [[718.3351, 0., 600.3891], [0., 718.3351, 181.5122], [0., 0., 1.]]
    with pytest.raises(AssertionError):
        preprocess_pifpaf(bad, (1238., 374.), enlarge_boxes=False)
    net.predict_batch([base[:2]], [kk], [None])   # warm every lazy set-up
    torch.cuda.synchronize()
    before = L_.lib().mlb_launch_count()
    with pytest.raises(AssertionError):
        net.predict_batch([base[:4], bad], [kk, kk], [None, (1238., 374.)], activities=('raise_hand',))
    assert L_.lib().mlb_launch_count() == before + 1
    stereo = _loco('stereo')
    stereo.predict_batch([base[:2]], [kk], [None], annotations_r_list=[base[:2]])
    torch.cuda.synchronize()
    before = L_.lib().mlb_launch_count()
    with pytest.raises(AssertionError):   # the right annotations go through the same check (predict.py:244)
        stereo.predict_batch([base[:4]], [kk], [None], annotations_r_list=[bad])
    assert L_.lib().mlb_launch_count() == before + 2


def test_empty_lists_images_without_detections_and_rejected_arguments():
    net = _loco('mono')
    assert net.predict_batch([], [], []) == []
    kk = [[718.3351, 0., 600.3891], [0., 718.3351, 181.5122], [0., 0., 1.]]
    with open(os.path.join(GOLDEN, 'pifpaf_002282.json')) as f:
        base = json.load(f)
    low = [{'keypoints': base[0]['keypoints'], 'bbox': [1., 2., 30., 40.], 'score': 0.1}]
    for anns, kw in (([[], []], {}), ([[], low], dict(min_conf=0.3)),
                     ([[], base[:5], low, []], dict(min_conf=0.3)),
                     ([[], base[:5], []], dict(activities=('social_distance', 'raise_hand'), args=ARGS))):
        kw.setdefault('activities', ('social_distance', 'raise_hand'))
        kw.setdefault('args', ARGS)
        got = net.predict_batch(anns, [kk] * len(anns), [None] * len(anns), **kw)
        _same(got, _four_calls(net, anns, [kk] * len(anns), [None] * len(anns), **kw), (len(anns), kw.get('min_conf')))
    for bad in (dict(kk_list=[kk]), dict(im_size_list=[None]), dict(enlarge_boxes=1), dict(min_conf=float('nan')),
                dict(activities=('wave',)), dict(activities=('social_distance',)), dict(annotations_r_list=[[], []]),
                dict(dic_gt_list=[None])):
        kw = dict(kk_list=[kk, kk], im_size_list=[None, None])
        kw.update(bad)
        with pytest.raises(ValueError):
            net.predict_batch([base[:2], []], **kw)


def test_4096_images():
    net = _loco('mono')
    ann_list, kks, sizes = _crowd(4096, 6, seed=7)
    kw = dict(activities=('social_distance', 'raise_hand'), args=ARGS_WIDE, min_conf=0.2)
    got = net.predict_batch(ann_list, kks, sizes, **kw)
    _same(got, _four_calls(net, ann_list, kks, sizes, **kw), 4096)
    assert sum(len(b) for b, _, _ in got) > 4096 * 2
