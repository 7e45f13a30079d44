"""Every output of forced tensor-core forwards over a matrix of served configurations -> one .npz, for bit-identity
checks of changes to loco_forward_tc_kernel: run it on two builds and compare the files with np.array_equal.

    python tools/tc_dump.py OUT.npz

Widths 256, 512, 1024, 1280, 2048; mono, zero-centred and stereo keypoints, MonolocoModel with 2 and 9 outputs; explicit
dropout masks and the counter RNG; forward_images; batches of 64, 4096 and 4224 rows.  The device error word must be 0
after every call."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from monoloco_b200 import synthetic, _lib as L_
from monoloco_b200.engine import LocoEngine

WIDTHS = (256, 512, 1024, 1280, 2048)
BATCHES = (64, 4096, 4224)
STEREO_SHAPES = {64: (8, 8), 4096: (64, 64), 4224: (66, 64)}   # left x right poses = rows


def main(path):
    res = {}
    K = synthetic.KITTI_K
    kw = dict(kernel='tc', want_dec=True, want_xyzc=True, want_x=True)

    def put(tag, eng, out):
        torch.cuda.synchronize()
        eng.check_error()
        assert eng.last_kernel()[0] == 3, (tag, eng.last_kernel())
        for k, v in out.items():
            res['%s/%s' % (tag, k)] = v.cpu().numpy()

    for L in WIDTHS:
        eng = LocoEngine(synthetic.make_state_dict('loco', 34, 9, L, 3, 40 + L % 97))
        for B in BATCHES:
            kps = torch.from_numpy(synthetic.make_keypoints(B, seed=B)).cuda()
            put('L%d/B%d/mono' % (L, B), eng, eng.forward(kps, kk=K, kind=L_.IN_KPS, **kw))
            put('L%d/B%d/zc' % (L, B), eng, eng.forward(kps, kk=K, kind=L_.IN_KPS, zero_center=True, **kw))
            masks = (np.random.RandomState(B).uniform(size=(2, B, L)) >= 0.2).astype(np.uint8)
            put('L%d/B%d/mask' % (L, B), eng, eng.forward(kps, kk=K, kind=L_.IN_KPS, dropout=True,
                                                           drop_mask=torch.from_numpy(masks).cuda(), **kw))
            put('L%d/B%d/rng' % (L, B), eng, eng.forward(kps, kk=K, kind=L_.IN_KPS, dropout=True, drop_seed=B + 7, **kw))
            off = [0, B // 3, B // 2, B]
            kks = [[[K[0][0] * s, 0., K[0][2] + 3 * s], [0., K[1][1] * s, K[1][2]], [0., 0., 1.]] for s in (0.9, 1.0, 1.1)]
            put('L%d/B%d/images' % (L, B), eng, eng.forward_images(kps, off, kks, kind=L_.IN_KPS, **kw))
        eng.close()
        eng = LocoEngine(synthetic.make_state_dict('loco', 68, 10, L, 3, 50 + L % 89))
        for B in BATCHES:
            nl, nr = STEREO_SHAPES[B]
            left = torch.from_numpy(synthetic.make_keypoints(nl, seed=B + 1)).cuda()
            right = torch.from_numpy(synthetic.make_keypoints(nr, seed=B + 2, right=True)[1]).cuda()
            put('L%d/B%d/stereo' % (L, B), eng, eng.forward(left, x_right=right, kk=K, kind=L_.IN_KPS_STEREO, **kw))
        eng.close()
        for n_out in (2, 9):
            eng = LocoEngine(synthetic.make_state_dict('monoloco', 34, n_out, L, 3, 60 + n_out))
            for B in BATCHES:
                x = torch.from_numpy(synthetic.make_inputs(B, 34, seed=B + 3)).cuda()
                put('L%d/B%d/monoloco%d' % (L, B, n_out), eng, eng.forward(x, kernel='tc', want_dec=False))
            eng.close()
    np.savez(path, **res)
    print('%d arrays from %d forwards -> %s (%s)' % (len(res), len({k.rsplit('/', 1)[0] for k in res}), path,
                                                       torch.cuda.get_device_name()))


def compare(a_path, b_path):
    """Exit status 1 unless both files hold the same arrays, bit for bit."""
    a, b = np.load(a_path), np.load(b_path)
    bad = sorted(set(a.files) ^ set(b.files))
    bad += [k for k in sorted(set(a.files) & set(b.files))
            if a[k].shape != b[k].shape or a[k].tobytes() != b[k].tobytes()]
    print('%d arrays compared, %d differ%s' % (len(a.files), len(bad), (': ' + ', '.join(bad[:20])) if bad else ''))
    return 1 if bad else 0


if __name__ == '__main__':
    if len(sys.argv) == 4 and sys.argv[1] == '--compare':
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    main(sys.argv[1] if len(sys.argv) > 1 else 'tc_dump.npz')
