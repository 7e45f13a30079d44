"""preprocess_pifpaf for many images without a GPU: the host mirror and a numpy restatement of mlb_preprocess_pifpaf's
arithmetic against the live reference (tests/golden/ref_predict_batch.npz, tools/gen_predict_golden.py) bit for bit, the
packing of the annotations, rejected arguments, and the C entry's declaration and export."""
import copy
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
N_CASES = 4


@pytest.fixture(scope='module')
def fix():
    return np.load(os.path.join(GOLDEN, 'ref_predict_batch.npz'))


def annotations(f):
    """The fixture's inputs as the caller passes them: (annotations_list, im_size_list)."""
    anns = []
    for k in range(len(f['ann_kps'])):
        d = {'keypoints': f['ann_kps'][k].tolist(), 'bbox': f['ann_bbox'][k].tolist()}
        if f['ann_has_score'][k]:
            d['score'] = float(f['ann_score'][k])
        anns.append(d)
    off = f['ann_off']
    ann_list = [anns[off[i]:off[i + 1]] for i in range(len(off) - 1)]
    sizes = [tuple(s.tolist()) if h else None for s, h in zip(f['im_size'], f['im_has_size'])]
    return ann_list, sizes


def case(f, c):
    return bool(f['c%d_enlarge' % c]), float(f['c%d_min_conf' % c])


def kernel_numpy(p, enlarge, min_conf):
    """mlb_preprocess_pifpaf restated with numpy fp64 element-wise operations in the kernel's order (pairwise mean of the
    17 confidences, Python's max(0, v) / min(v, size)): (boxes [n, 5], kps [n, 3, 17], src [n], kept_off)."""
    kps, (x1, y1, x2, y2) = p['kps'], p['bbox'].T.copy()
    c = kps[:, 2::3]
    r = c[:, :8] + c[:, 8:16]
    mean = ((((r[:, 0] + r[:, 1]) + (r[:, 2] + r[:, 3])) + ((r[:, 4] + r[:, 5]) + (r[:, 6] + r[:, 7]))) + c[:, 16]) / 17.0
    has = p['has_score'].astype(bool)
    conf = np.where(has, p['score'], mean)
    dh = np.where(has, y2 / (10.0 * enlarge), (y2 - y1) / (7.0 * enlarge))
    dw = np.where(has, x2 / (5.0 * enlarge), (x2 - x1) / (3.5 * enlarge))
    x2, y2 = np.where(has, x2 + x1, x2), np.where(has, y2 + y1, y2)
    x1, y1, x2, y2 = x1 - dw, y1 - dh, x2 + dw, y2 + dh
    img = np.repeat(np.arange(len(p['ann_off']) - 1), np.diff(p['ann_off']))
    sized = p['has_size'][img].astype(bool)
    w, h = p['im_size'][img, 0], p['im_size'][img, 1]
    x1, y1 = np.where(sized & ~(x1 > 0), 0.0, x1), np.where(sized & ~(y1 > 0), 0.0, y1)
    x2, y2 = np.where(sized & (w < x2), w, x2), np.where(sized & (h < y2), h, y2)
    keep = conf >= min_conf
    boxes = np.stack([x1, y1, x2, y2, conf], axis=1)[keep]
    kept_off = np.concatenate([[0], np.cumsum(np.bincount(img[keep], minlength=len(p['ann_off']) - 1))])
    return boxes, kps.reshape(-1, 17, 3).transpose(0, 2, 1)[keep], np.flatnonzero(keep), kept_off


def test_host_mirror_equals_reference(fix):
    from monoloco_b200.network.process import preprocess_pifpaf
    ann_list, sizes = annotations(fix)
    for c in range(N_CASES):
        enlarge, min_conf = case(fix, c)
        boxes, kps = [], []
        for anns, size in zip(ann_list, sizes):
            before = copy.deepcopy(anns)
            b, k = preprocess_pifpaf(anns, size, enlarge_boxes=enlarge, min_conf=min_conf)
            assert anns == before   # the caller's dictionaries are left alone
            boxes += b
            kps += k
        assert np.array_equal(np.asarray(boxes).reshape(-1, 5), fix['c%d_boxes' % c]), c
        assert np.array_equal(np.asarray(kps).reshape(-1, 3, 17), fix['c%d_kps' % c]), c


def test_kernel_order_restated_equals_reference(fix):
    from monoloco_b200.network.process import pack_pifpaf
    ann_list, sizes = annotations(fix)
    p = pack_pifpaf(ann_list, sizes)
    for c in range(N_CASES):
        enlarge, min_conf = case(fix, c)
        boxes, kps, src, off = kernel_numpy(p, 1 if enlarge else 2, min_conf)
        assert np.array_equal(boxes, fix['c%d_boxes' % c]), c
        assert np.array_equal(kps, fix['c%d_kps' % c]), c
        assert np.array_equal(src, fix['c%d_src' % c]), c
        assert np.array_equal(off, fix['c%d_off' % c]), c
    # the fixture reaches the edges it was built for: filtered annotations, an all-filtered image, clamped boxes
    assert len(fix['c2_src']) < len(fix['ann_kps']) and (np.diff(fix['c2_off']) == 0).sum() > (np.diff(fix['ann_off']) == 0).sum()
    assert (fix['c0_boxes'][:, :2] == 0).any() and (fix['c0_boxes'][:, 2] == 1238.0).any() and (fix['c0_boxes'][:, 3] == 374.0).any()


def test_other_summation_order_differs():
    """np.mean's order matters: the first value plus a pairwise sum of the other 16 is not it."""
    rng = np.random.RandomState(3)
    c = rng.uniform(0, 1, (20_000, 17))
    r = c[:, :8] + c[:, 8:16]
    ours = ((((r[:, 0] + r[:, 1]) + (r[:, 2] + r[:, 3])) + ((r[:, 4] + r[:, 5]) + (r[:, 6] + r[:, 7]))) + c[:, 16]) / 17.0
    assert all(float(np.mean(x)) == o for x, o in zip(c[:2000], ours[:2000]))
    q = c[:, 1:9] + c[:, 9:17]
    other = (c[:, 0] + (((q[:, 0] + q[:, 1]) + (q[:, 2] + q[:, 3])) + ((q[:, 4] + q[:, 5]) + (q[:, 6] + q[:, 7])))) / 17.0
    assert (other != ours).mean() > 0.1


def test_packing_and_layout():
    from monoloco_b200.network.process import pack_pifpaf, pifpaf_layout, PIFPAF_FIELDS
    kp = [float(v) for v in range(51)]
    ann = [[{'keypoints': kp, 'bbox': [1., 2., 3., 4.], 'score': 0.5}], [], [{'keypoints': kp, 'bbox': [5., 6., 7., 8.]}] * 2]
    before = copy.deepcopy(ann)
    p = pack_pifpaf(ann, [(640, 480.5), None, (10., 20.)])
    assert ann == before
    assert p['ann_off'].tolist() == [0, 1, 1, 3] and p['ann_off'].dtype == np.int32
    assert p['kps'].shape == (3, 51) and p['bbox'][2].tolist() == [5., 6., 7., 8.]
    assert p['has_score'].tolist() == [1, 0, 0] and p['score'][0] == 0.5
    assert p['has_size'].tolist() == [1, 0, 1] and p['im_size'][0].tolist() == [640., 480.5]
    empty = pack_pifpaf([[], []], [None, None])
    assert empty['kps'].shape == (0, 51) and empty['ann_off'].tolist() == [0, 0, 0]
    lays, total = pifpaf_layout([p, empty])
    spans = []
    for pk, lay in zip([p, empty], lays):
        assert set(lay) == {n for n, _ in PIFPAF_FIELDS}
        for name, (o, shape, dt) in lay.items():
            assert o % 8 == 0 and shape == pk[name].shape and dt == pk[name].dtype
            spans.append((o, o + int(np.prod(shape)) * dt.itemsize))
    spans.sort()
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:])) and spans[-1][1] <= total


def test_rejected_arguments():
    from monoloco_b200.network.process import pack_pifpaf, check_pifpaf_options
    kp = [0.] * 51
    with pytest.raises(ValueError):
        pack_pifpaf([[]], [None, None])
    with pytest.raises(ValueError):
        pack_pifpaf([[{'keypoints': kp[:48], 'bbox': [0., 0., 1., 1.]}]], [None])
    with pytest.raises(ValueError):
        pack_pifpaf([[{'keypoints': kp, 'bbox': [0., 0., 1.]}]], [None])
    with pytest.raises(ValueError):
        pack_pifpaf([[{'bbox': [0., 0., 1., 1.]}]], [None])
    with pytest.raises(ValueError):
        pack_pifpaf([[{'keypoints': kp, 'bbox': [0., 0., 1., 1.]}]], [(640,)])
    for bad in (1, 'yes', None):
        with pytest.raises(ValueError):
            check_pifpaf_options(bad, 0.)
    for bad in (float('nan'), float('inf'), -float('inf'), 'x', None):
        with pytest.raises(ValueError):
            check_pifpaf_options(True, bad)
    assert check_pifpaf_options(True, 0.3) == (1, 0.3) and check_pifpaf_options(False, 0) == (2, 0.0)


def test_export_declared_and_loaded(tmp_path):
    from monoloco_b200 import _lib as L_
    assert 'mlb_preprocess_pifpaf' in L_.EXPORTS
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "monoloco_b200.h"', 'int main(void) {',
             '  int (*fn)(const mlb_pifpaf_args*, void*) = mlb_preprocess_pifpaf; (void)fn;',
             '  printf("sizeof %zu\\n", sizeof(mlb_pifpaf_args));']
    for fname, _ in L_.MlbPifpafArgs._fields_:
        lines.append('  printf("%s %%zu\\n", offsetof(mlb_pifpaf_args, %s));' % (fname, fname))
    lines += ['  return 0;', '}']
    src = tmp_path / 'layout.c'
    src.write_text('\n'.join(lines))
    obj = tmp_path / 'layout'
    subprocess.run(['gcc', '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(obj),
                    '-Wl,--unresolved-symbols=ignore-all'], check=True)
    got = dict(line.split() for line in subprocess.run([str(obj)], check=True, stdout=subprocess.PIPE,
                                                       text=True).stdout.splitlines())
    assert int(got['sizeof']) == C.sizeof(L_.MlbPifpafArgs)
    for fname, _ in L_.MlbPifpafArgs._fields_:
        assert int(got[fname]) == getattr(L_.MlbPifpafArgs, fname).offset, fname
    lib = L_.lib()
    assert hasattr(lib, 'mlb_preprocess_pifpaf')
    # argument checks run before anything touches a device
    assert lib.mlb_preprocess_pifpaf(None, None) != 0
    a = L_.MlbPifpafArgs()
    a.n_img, a.enlarge = 1, 3
    assert lib.mlb_preprocess_pifpaf(C.byref(a), None) != 0
    assert lib.mlb_last_error().decode().startswith('mlb_preprocess_pifpaf: enlarge')
