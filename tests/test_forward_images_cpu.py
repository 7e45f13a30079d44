"""Multi-image inference without a GPU: the ctypes mirror of mlb_image_batch against the header, the numpy oracle pinned to
the per-image reference fixture, and the host-side CSR / K^-1 packing that Loco.forward_batch and forward_images use."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def test_image_batch_layout_matches_header(tmp_path):
    from monoloco_b200 import _lib as L_
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "monoloco_b200.h"', 'int main(void) {',
             '  printf("sizeof %zu\\n", sizeof(mlb_image_batch));']
    for fname, _ in L_.MlbImageBatch._fields_:
        lines.append('  printf("%s %%zu\\n", offsetof(mlb_image_batch, %s));' % (fname, fname))
    lines += ['  return 0;', '}']
    src = tmp_path / 'layout.c'
    src.write_text('\n'.join(lines))
    exe = tmp_path / 'layout'
    subprocess.run(['gcc', '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)],
                   check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], check=True, stdout=subprocess.PIPE,
                                                       text=True).stdout.splitlines())
    assert int(got['sizeof']) == C.sizeof(L_.MlbImageBatch)
    for fname, _ in L_.MlbImageBatch._fields_:
        assert int(got[fname]) == getattr(L_.MlbImageBatch, fname).offset, fname
    assert 'mlb_forward_images' in L_.EXPORTS and 'mlb_stereo_filter_images' in L_.EXPORTS


def _split(f, prefix, counts):
    off = np.concatenate([[0], np.cumsum(counts)])
    return [{k[len(prefix):]: f[k][off[i]:off[i + 1]] for k in f.files if k.startswith(prefix)} for i in range(len(counts))]


def test_oracle_matches_per_image_reference_fixture():
    """oracle.loco_oracle.loco_forward, image by image with each image's own K, reproduces the reference Loco.forward."""
    from oracle import loco_oracle as O
    from monoloco_b200 import synthetic
    f = np.load(os.path.join(GOLDEN, 'ref_loco_images.npz'))
    sd = synthetic.make_state_dict('loco', 34, 9, 1024, 3, 1)
    n = f['mono_n']
    kps = np.split(f['mono_kps'], np.cumsum(n)[:-1])
    refs = _split(f, 'mono_out_', n)
    assert 0 in n and 1 in n and 17 in n and len(np.unique(f['mono_K'].reshape(len(n), 9), axis=0)) == len(n)
    for i in range(len(n)):
        dic = O.loco_forward(sd, kps[i], f['mono_K'][i], mode='mono')
        if n[i] == 0:
            assert dic is None
            continue
        for k in ('xyzd', 'bi', 'd', 'h', 'w', 'l', 'ori'):
            ok, worst = O.close(dic[k], refs[i][k], col_scale=(k != 'xyzd'))
            assert ok, (i, k, worst)
        assert O.angle_close(dic['yaw'][0], refs[i]['yaw_pred'])[0]
    sd = synthetic.make_state_dict('loco', 68, 10, 1024, 3, 2)
    nl, nr = f['stereo_nl'], f['stereo_nr']
    lefts = np.split(f['stereo_left'], np.cumsum(nl)[:-1])
    rights = np.split(f['stereo_right'], np.cumsum(np.maximum(nr, 0))[:-1])
    refs = _split(f, 'stereo_out_', nl)
    for i in range(len(nl)):
        dic = O.loco_forward(sd, lefts[i], f['stereo_K'][i], rights[i] if nr[i] >= 0 else None, mode='stereo')
        for k in ('xyzd', 'bi', 'd', 'aux'):
            ok, worst = O.close(dic[k], refs[i][k], col_scale=(k != 'xyzd'))
            assert ok, (i, k, worst)


def test_host_csr_and_kinv_packing():
    from monoloco_b200.engine import image_offsets, check_image_batch, kinv_images
    assert image_offsets([]).tolist() == [0]
    assert image_offsets([0, 3, 0, 2, 0]).tolist() == [0, 0, 3, 3, 5, 5]
    assert image_offsets([4]).dtype == np.int32
    ro, lo, rr = check_image_batch([0, 0, 12, 12, 14], 14, [0, 0, 4, 4, 6], [0, 2, 5, 7, 8], 6, 8)
    assert ro.dtype == lo.dtype == rr.dtype == np.int32
    assert check_image_batch(image_offsets([0, 5, 0]), 5)[1] is None
    for bad in (([1, 5], 5), ([0, 4], 5), ([0, 3, 2, 5], 5), ([0], 0)):
        with pytest.raises(ValueError):
            check_image_batch(*bad)
    with pytest.raises(ValueError):  # stereo: image 0 owns 2 x 3 rows, not 5
        check_image_batch([0, 5], 5, [0, 2], [0, 3], 2, 3)
    with pytest.raises(ValueError):  # offsets of different lengths
        check_image_batch([0, 6], 6, [0, 2, 2], [0, 3, 3], 2, 3)
    kks = [np.array([[718.3351, 0., 600.3891], [0., 718.3351, 181.5122], [0., 0., 1.]]),
           [[707.0, 2.5, 604.1], [0., 707.0, 180.5], [0., 0., 1.]]]
    kinv = kinv_images(kks)
    assert kinv.shape == (2, 9) and kinv.dtype == np.float32
    for i, kk in enumerate(kks):
        assert np.array_equal(kinv[i], np.linalg.inv(np.asarray(kk, dtype=np.float64)).astype(np.float32).reshape(9))
