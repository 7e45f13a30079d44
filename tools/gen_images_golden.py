"""
Multi-image fixture: the REAL reference `Loco.forward` (net.py:83-133), called image by image, on images that each have
their own camera matrix.  TEST INFRASTRUCTURE ONLY; needs the reference sources (oracle/gen_golden.py imports them).

    python tools/gen_images_golden.py

Writes tests/golden/ref_loco_images.npz:
  * mono (monoloco_pp, width 1024, 3 stages, seed 1): 6 images with 0, 1, 17, 40, 5 and 9 detections taken from the
    committed KAT keypoints (kat_mono_val.npz), with KITTI K, a longer focal length, an off-centre principal point and
    non-zero skew.  mono_kps / mono_K / mono_n per image, mono_out_<key> rows of all images concatenated.
  * stereo (monstereo, width 1024, 3 stages, seed 2): 3 images with (n_left, n_right) = (4, 3), (2, none) and (5, 6), left
    and right poses from kat_stereo_val.npz.  stereo_nr = -1 marks "no right poses" (net.py:115-116: the first left pose
    becomes the right pose).  The filtered outputs have one row per left pose.
Weights are regenerated from monoloco_b200.synthetic seeds; the state-dict checksums are stored.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gen_golden as G  # noqa: E402  (imports the reference)

torch = G.torch

KITTI = [[718.3351, 0., 600.3891], [0., 718.3351, 181.5122], [0., 0., 1.]]
K_MONO = [KITTI,
          [[1266.4, 0., 816.3], [0., 1266.4, 491.5], [0., 0., 1.]],        # longer focal length (nuScenes-like)
          [[721.5, 0., 420.0], [0., 721.5, 260.0], [0., 0., 1.]],          # principal point off the image centre
          [[707.0, 2.5, 604.1], [0., 707.0, 180.5], [0., 0., 1.]],         # non-zero skew
          [[960.0, 0., 640.0], [0., 955.0, 360.0], [0., 0., 1.]],
          [[700.0, -1.2, 590.0], [0., 712.0, 175.0], [0., 0., 1.]]]
N_MONO = (0, 1, 17, 40, 5, 9)
K_STEREO = [KITTI, [[721.5, 0., 609.6], [0., 721.5, 172.9], [0., 0., 1.]], [[707.0, 1.5, 604.1], [0., 707.0, 180.5], [0., 0., 1.]]]
LR_STEREO = ((4, 3), (2, None), (5, 6))


def main():
    save = {}
    kat = np.load(os.path.join(G.OUT, 'kat_mono_val.npz'))
    model, sd = G.build('loco', 34, 9, 1024, 3, 1)
    net = G.Loco(model=model, mode='mono', device=torch.device('cpu'))
    kps_all, outs, p = [], [], 0
    for n, kk in zip(N_MONO, K_MONO):
        kps = kat['kps'][p:p + n]
        p += n
        kps_all.append(kps)
        dic = net.forward(kps.tolist(), kk)
        assert (dic is None) == (n == 0)
        if dic is not None:
            outs.append(G.dic_to_np(dic))
    save['mono_kps'] = np.concatenate(kps_all).astype(np.float32)
    save['mono_n'] = np.asarray(N_MONO, dtype=np.int32)
    save['mono_K'] = np.asarray(K_MONO, dtype=np.float32)
    for k in outs[0]:
        save['mono_out_' + k] = np.concatenate([o[k] for o in outs])
    save['mono_checksum'] = G.sd_checksum(sd)

    kat = np.load(os.path.join(G.OUT, 'kat_stereo_val.npz'))
    model, sd = G.build('loco', 68, 10, 1024, 3, 2)
    net = G.Loco(model=model, mode='stereo', device=torch.device('cpu'))
    lefts, rights, outs, pl, pr = [], [], [], 0, 40
    for (nl, nr), kk in zip(LR_STEREO, K_STEREO):
        left = kat['kps'][pl:pl + nl, :, :17]
        pl += nl
        lefts.append(left)
        right = None
        if nr is not None:
            right = kat['kps'][pr:pr + nr, :, 17:]
            pr += nr
            rights.append(right)
        dic = net.forward(left.tolist(), kk, right.tolist() if right is not None else None)
        outs.append(G.dic_to_np(dic))
    save['stereo_left'] = np.concatenate(lefts).astype(np.float32)
    save['stereo_right'] = np.concatenate(rights).astype(np.float32)
    save['stereo_nl'] = np.asarray([a for a, _ in LR_STEREO], dtype=np.int32)
    save['stereo_nr'] = np.asarray([-1 if b is None else b for _, b in LR_STEREO], dtype=np.int32)
    save['stereo_K'] = np.asarray(K_STEREO, dtype=np.float32)
    for k in outs[0]:
        save['stereo_out_' + k] = np.concatenate([o[k] for o in outs])
    save['stereo_checksum'] = G.sd_checksum(sd)
    np.savez_compressed(os.path.join(G.OUT, 'ref_loco_images.npz'), **save)
    print('ref_loco_images.npz', {k: v.shape for k, v in save.items() if hasattr(v, 'shape')})


if __name__ == '__main__':
    main()
