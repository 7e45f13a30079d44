"""
Predict-chain fixture: the REAL reference `preprocess_pifpaf` (process.py:155-207) and its per-image predict chain
(predict.py:226-240 / 244: preprocess_pifpaf -> Loco.forward -> post_process -> social_distance -> raising_hand) on seeded
images.  TEST INFRASTRUCTURE ONLY; needs the reference sources (oracle/gen_golden.py imports them).

    python tools/gen_predict_golden.py

Writes tests/golden/ref_predict_batch.npz (pre-process) and tests/golden/ref_predict_batch.json (chain):
  * pre-process: 9 images of annotations derived from the pifpaf fixture (tests/golden/pifpaf_002282.json): the fixture as
    it is, an empty image, xywh boxes with a 'score', boxes crossing every image border, confidences exactly at and one ulp
    either side of 0.3 (with and without a score), an image whose annotations all fall below 0.3, a mixed image, and
    images without a size.  Inputs ann_* / im_*, then per case c (enlarge_boxes x min_conf in {0, 0.3}) the kept boxes,
    key points, source annotation index and kept offsets.
  * chain: mono (monoloco_pp, width 1024, 3 stages, seed 1) on 6 images, some with dic_gt, with social_distance (args
    threshold_prob 0.25, threshold_dist 2, radii (0.3, 0.5, 1); the seeded network places everybody at about 20 m facing
    one way, so nobody is flagged) and raising_hand (some poses get a raised hand); stereo (monstereo, seed 2) on 4 images
    with right annotations (one image without).  Per person `sd_clear` says whether the reference's flag survives
    relative perturbations of 3e-5 of the network outputs it reads (the fp32 network's noise is far below that).
Weights are regenerated from monoloco_b200.synthetic seeds; the state-dict checksums are stored.
"""
import copy
import json
import os
import sys
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gen_golden as G  # noqa: E402  (imports the reference)

torch = G.torch
KITTI = [[718.3351, 0., 600.3891], [0., 718.3351, 181.5122], [0., 0., 1.]]
IM_SIZE = (1238.0, 374.0)
ARGS = SimpleNamespace(threshold_prob=0.25, threshold_dist=2.0, radii=(0.3, 0.5, 1.0))
CASES = [(True, 0.0), (False, 0.0), (True, 0.3), (False, 0.3)]


def fixture():
    with open(os.path.join(G.OUT, 'pifpaf_002282.json')) as f:
        return json.load(f)


def with_score(ann, score):
    """The annotation as an xywh box with a score (the openpifpaf json format)."""
    x1, y1, x2, y2 = ann['bbox']
    return {'keypoints': list(ann['keypoints']), 'bbox': [x1, y1, x2 - x1, y2 - y1], 'score': score}


def mean_at(ann, target):
    """The annotation without a score, its last keypoint confidence moved until float(np.mean(confs)) == target."""
    kps = list(ann['keypoints'])
    confs = np.asarray(kps[2::3], dtype=np.float64)
    for attempt in range(64):   # not every sum is reachable through the last value alone: nudge the first one too
        confs[0] = kps[2] + attempt * 1e-7
        up = down = 17 * target - confs[:16].sum()
        for _ in range(256):
            for c in (up, down):
                confs[16] = c
                if float(np.mean(confs)) == target:
                    kps[2], kps[50] = float(confs[0]), float(c)
                    return {'keypoints': kps, 'bbox': list(ann['bbox'])}
            up, down = np.nextafter(up, np.inf), np.nextafter(down, -np.inf)
    raise RuntimeError('no keypoint confidences give the mean %r' % target)


def preprocess_images(rng):
    base = fixture()
    lo, hi = np.nextafter(0.3, 0.0), np.nextafter(0.3, 1.0)
    imgs = [(base, IM_SIZE), ([], IM_SIZE), ([with_score(a, float(rng.uniform(0.05, 0.9))) for a in base[:8]], IM_SIZE)]
    border = []
    for k, a in enumerate(base[:8]):   # boxes over the left, top, right and bottom borders, with and without a score
        b = copy.deepcopy(a)
        x1, y1, x2, y2 = b['bbox']
        dx = [-x1 - 5.0, 0.0, IM_SIZE[0] - x2 + 7.5, 0.0][k % 4]
        dy = [0.0, -y1 - 3.0, 0.0, IM_SIZE[1] - y2 + 4.25][k % 4]
        b['bbox'] = [x1 + dx, y1 + dy, x2 + dx, y2 + dy]
        border.append(with_score(b, 0.5) if k >= 4 else b)
    imgs.append((border, IM_SIZE))
    imgs.append(([with_score(base[0], 0.3), with_score(base[1], lo), with_score(base[2], hi), mean_at(base[3], 0.3),
                  mean_at(base[4], lo), mean_at(base[5], hi)], IM_SIZE))
    imgs.append(([with_score(base[6], 0.1), mean_at(base[7], 0.2), with_score(base[8], -0.5)], IM_SIZE))
    imgs.append(([with_score(a, float(rng.uniform(0.2, 0.9))) if k % 2 else a for k, a in enumerate(base[4:14])], None))
    imgs.append((base[::3], None))
    imgs.append(([], None))
    return imgs


def run_preprocess(imgs):
    save = {}
    anns = [a for im, _ in imgs for a in im]
    save['ann_kps'] = np.asarray([a['keypoints'] for a in anns], dtype=np.float64)
    save['ann_bbox'] = np.asarray([a['bbox'] for a in anns], dtype=np.float64)
    save['ann_has_score'] = np.asarray(['score' in a for a in anns])
    save['ann_score'] = np.asarray([a.get('score', np.nan) for a in anns], dtype=np.float64)
    save['ann_off'] = np.cumsum([0] + [len(im) for im, _ in imgs]).astype(np.int32)
    save['im_size'] = np.asarray([s if s else (np.nan, np.nan) for _, s in imgs], dtype=np.float64)
    save['im_has_size'] = np.asarray([s is not None for _, s in imgs])
    for c, (enlarge, min_conf) in enumerate(CASES):
        boxes, kps, src, off = [], [], [], [0]
        a0 = 0
        for im, size in imgs:
            b, k = G.preprocess_pifpaf(copy.deepcopy(im), size, enlarge_boxes=enlarge, min_conf=min_conf)
            kept = [j for j, a in enumerate(im)
                    if G.preprocess_pifpaf(copy.deepcopy([a]), size, enlarge_boxes=enlarge, min_conf=min_conf)[0]]
            assert len(kept) == len(b)
            boxes += b
            kps += k
            src += [a0 + j for j in kept]
            off.append(off[-1] + len(b))
            a0 += len(im)
        save['c%d_enlarge' % c], save['c%d_min_conf' % c] = enlarge, min_conf
        save['c%d_boxes' % c] = np.asarray(boxes, dtype=np.float64).reshape(-1, 5)
        save['c%d_kps' % c] = np.asarray(kps, dtype=np.float64).reshape(-1, 3, 17)
        save['c%d_src' % c] = np.asarray(src, dtype=np.int32)
        save['c%d_off' % c] = np.asarray(off, dtype=np.int32)
        print('case', c, enlarge, min_conf, 'kept', off[-1], 'of', a0)
    return save


def chain_images(rng, n_img, stereo):
    base = fixture()
    out = []
    for i in range(n_img):
        if i == 1:
            out.append({'ann': [], 'ann_r': [], 'kk': KITTI, 'im_size': list(IM_SIZE), 'gt': None})
            continue
        sel = rng.choice(len(base), size=int(rng.randint(3, 12)), replace=False)
        shift = float(rng.uniform(-40, 40))
        anns = []
        for j in sel:
            a = copy.deepcopy(base[int(j)])
            a['keypoints'][0::3] = [x + shift for x in a['keypoints'][0::3]]
            a['bbox'] = [a['bbox'][0] + shift, a['bbox'][1], a['bbox'][2] + shift, a['bbox'][3]]
            if len(anns) % 3 == 0:   # a raised hand (left, right or both) for is_raising_hand to find
                kp = a['keypoints']
                for side in {0: (0,), 1: (1,), 2: (0, 1)}[len(anns) % 9 // 3]:
                    sho, elb, hand = 5 + side, 7 + side, 9 + side
                    kp[3 * elb], kp[3 * elb + 1] = kp[3 * sho] + (-12 if side == 0 else 12), kp[3 * sho + 1] - 6
                    kp[3 * hand], kp[3 * hand + 1] = kp[3 * elb] + (-3 if side == 0 else 3), kp[3 * sho + 1] - 30
            anns.append(with_score(a, float(rng.uniform(0.3, 0.9))) if i % 3 == 2 else a)
        kk = [[700.0 + 20 * i, 0., 600.0 + 3 * i], [0., 700.0 + 20 * i, 180.0 - 2 * i], [0., 0., 1.]]
        im_size = list(IM_SIZE) if i % 4 != 3 else None
        ann_r = []
        if stereo and i != 2:
            for a in anns:
                r = copy.deepcopy(a)
                disp = float(rng.uniform(8, 30))
                r['keypoints'][0::3] = [x - disp for x in r['keypoints'][0::3]]
                r.pop('score', None)
                r['bbox'] = list(base[0]['bbox'])
                ann_r.append(r)
        gt = None
        if i % 2 == 0:
            boxes, _ = G.preprocess_pifpaf(copy.deepcopy(anns), im_size, enlarge_boxes=False)
            gtb, ys = [], []
            for b in boxes[::2]:
                jit = rng.uniform(-4, 4, 4)
                gtb.append([b[0] + jit[0], b[1] + jit[1], b[2] + jit[2], b[3] + jit[3]])
                ys.append([0., 0., 0., float(rng.uniform(5, 40))])
            gtb.append([5.0, 5.0, 30.0, 60.0])   # matches nothing
            ys.append([0., 0., 0., 12.0])
            gt = {'boxes': gtb, 'ys': ys}
        out.append({'ann': anns, 'ann_r': ann_r, 'kk': kk, 'im_size': im_size, 'gt': gt})
    return out


def jsonable(v):
    if isinstance(v, dict):
        return {k: jsonable(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return [jsonable(x) for x in v]
    if isinstance(v, (np.floating, np.integer, np.bool_)):
        return v.item()
    if isinstance(v, torch.Tensor):
        return v.tolist()
    return v


def sd_clear(dic_out, rng, args):
    """Per person: does the reference's social_distance flag survive relative perturbations of its network inputs?"""
    ref = dic_out['social_distance']
    clear = [True] * len(ref)
    for _ in range(6):
        d = {'angles': [a * (1 + rng.uniform(-3e-5, 3e-5)) for a in dic_out['angles']],
             'dds_pred': [a * (1 + rng.uniform(-3e-5, 3e-5)) for a in dic_out['dds_pred']],
             'stds_ale': [a * (1 + rng.uniform(-3e-5, 3e-5)) for a in dic_out['stds_ale']],
             'xyz_pred': [[c * (1 + rng.uniform(-3e-5, 3e-5)) for c in xyz] for xyz in dic_out['xyz_pred']]}
        got = G.Loco.social_distance(d, args)['social_distance']
        clear = [c and g == r for c, g, r in zip(clear, got, ref)]
    return clear


def run_chain(mode, seed, n_img, rng, args=ARGS):
    stereo = mode == 'stereo'
    model, sd = G.build('loco', 68 if stereo else 34, 10 if stereo else 9, 1024, 3, seed)
    net = G.Loco(model=model, mode=mode, device=torch.device('cpu'))
    images = chain_images(rng, n_img, stereo)
    for im in images:
        size = tuple(im['im_size']) if im['im_size'] else None
        boxes, keypoints = G.preprocess_pifpaf(copy.deepcopy(im['ann']), size, enlarge_boxes=False)
        if stereo:
            _, keypoints_r = G.preprocess_pifpaf(copy.deepcopy(im['ann_r']), size)
            dic_out = net.forward(keypoints, im['kk'], keypoints_r=keypoints_r)
        else:
            dic_out = net.forward(keypoints, im['kk'])
        dic_out = net.post_process(dic_out, boxes, keypoints, im['kk'], im['gt'])
        if not stereo:
            dic_out = net.social_distance(dic_out, args)
            dic_out = net.raising_hand(dic_out, keypoints)
        im['out'] = jsonable([boxes, keypoints, dict(dic_out)])
        if not stereo:
            im['sd_clear'] = sd_clear(dic_out, rng, args)
        print(mode, 'image', len(boxes), 'detections', sum(dic_out.get('social_distance', [])), 'flagged',
              sum(im.get('sd_clear', [])), 'clear', dic_out.get('raising_hand'))
    return {'images': jsonable(images), 'checksum': G.sd_checksum(sd), 'seed': seed,
            'args': {'threshold_prob': args.threshold_prob, 'threshold_dist': args.threshold_dist, 'radii': list(args.radii)}}


def main():
    rng = np.random.RandomState(11)
    save = run_preprocess(preprocess_images(rng))
    np.savez_compressed(os.path.join(G.OUT, 'ref_predict_batch.npz'), **save)
    chain = {'mono': run_chain('mono', 1, 6, rng), 'stereo': run_chain('stereo', 2, 4, rng)}
    with open(os.path.join(G.OUT, 'ref_predict_batch.json'), 'w') as f:
        json.dump(chain, f)
    print('ref_predict_batch.npz / .json written')


if __name__ == '__main__':
    main()
