"""
Activity fixture: the REAL reference `social_interactions` / `is_raising_hand` (monoloco/activity.py:17-117) on many
seeded images.  TEST INFRASTRUCTURE ONLY; needs the reference sources (oracle/gen_golden.py imports them).

    python tools/gen_activity_golden.py

Writes tests/golden/ref_activity_batch.npz:
  * 60 images (synthetic.make_crowd, seed = image index) with n in N_PEOPLE, people 0.3 to 3 m apart, plus one image
    whose people 1 and 4 stand on exactly the same spot.  Image i runs parameter set (i + i // 12) % len(CONFIGS): radii (0.3, 0.5)
    or (0.3, 0.5, 1), social_distance both ways, threshold_dist 2 or 2.5, n_samples 100, 7 or 1.
    n / cfg per image; xz, angles, dds, stds, flags per person (images concatenated); cfg_* per parameter set.
    np.argsort breaks ties between the coincident people in an order that depends on the CPU's sort kernel; the seed
    of that image is the first one for which it takes them in index order (a stable sort), the order the device uses.
  * is_raising_hand codes (0 None, 1 left, 2 right, 3 both) of the pifpaf fixture's 16 poses, 200 random poses and
    degenerate ones: a zero-length forearm or arm, a hand exactly at shoulder height, a hand tucked next to the head.
  * table: the first 100 * 64 values of T = sign(u) * log1p(-|u|), u = torch's seed-1 uniform_(eps - 1, 1) stream.
"""
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gen_golden as G  # noqa: E402  (imports the reference)
from monoloco.activity import social_interactions, is_raising_hand  # noqa: E402
from monoloco_b200 import synthetic  # noqa: E402

torch = G.torch
N_PEOPLE = (0, 1, 2, 3, 5, 8, 12, 16, 20, 30, 40, 64)
# radii, social_distance, threshold_dist, n_samples, threshold_prob (predict.py defaults: 0.25, 2, (0.3, 0.5))
CONFIGS = [((0.3, 0.5), False, 2.0, 100, 0.25), ((0.3, 0.5, 1.0), True, 2.5, 100, 0.25),
           ((0.3, 0.5), True, 2.0, 1, 0.25), ((0.3, 0.5, 1.0), False, 2.5, 7, 0.25),
           ((0.3, 0.5, 1.0), False, 2.0, 100, 0.4), ((0.3, 0.5), False, 2.5, 1, 0.25)]
CODES = {None: 0, 'left': 1, 'right': 2, 'both': 3}


def flags(centers, angles, dds, stds, cfg):
    radii, sd, td, ns, tp = cfg
    return [bool(social_interactions(i, centers, angles, dds, stds=stds, social_distance=sd, n_samples=ns,
                                     threshold_prob=tp, threshold_dist=td, radii=radii)) for i in range(len(centers))]


def coincident_image():
    for seed in range(1000, 2000):
        centers, angles, dds, stds = synthetic.make_crowd(6, seed=seed, spacing=(0.3, 1.5))
        centers[4] = list(centers[1])
        dds[4] = dds[1]
        ok = True
        for idx in (1, 4):   # the reference's distances and its argsort (activity.py:24-28)
            dist = [math.sqrt((centers[idx][0] - c[0]) ** 2 + (centers[idx][1] - c[1]) ** 2) for c in centers]
            ok &= int(np.argsort(dist)[0]) == 1 and sum(d <= 2.0 for d in dist) >= 3
        if ok:
            return seed, (centers, angles, dds, stds)
    raise RuntimeError('no seed with index-ordered ties')


def degenerate_poses(kps):
    """Poses at the edges of is_raising_hand, derived from a real pose: left / right hand raised high, zero-length forearm
    or upper arm (NaN angle), hand exactly at shoulder height, hand tucked next to the head, both arms up."""
    base = np.asarray(kps, dtype=np.float64)
    out = []
    for side in (0, 1):
        sho, elb, hand = 5 + side, 7 + side, 9 + side
        up = base.copy()
        up[0, elb] = up[0, sho] + (-30 if side == 0 else 30)
        up[1, elb] = up[1, sho] - 10
        up[0, hand], up[1, hand] = up[0, elb], up[1, sho] - 80
        out.append(up)
        zero_fore = up.copy()
        zero_fore[:, hand] = zero_fore[:, elb]
        out.append(zero_fore)
        zero_arm = up.copy()
        zero_arm[:2, elb] = zero_arm[:2, sho]
        out.append(zero_arm)
        level = up.copy()
        level[1, hand] = level[1, sho]
        out.append(level)
        tucked = up.copy()
        tucked[0, hand] = tucked[0, sho] + (-5 if side == 1 else 5)
        tucked[1, hand] = tucked[1, 0] - 0.5 * abs(tucked[0, 3] - tucked[0, 4])
        out.append(tucked)
    both = out[0].copy()
    both[:, 6::2][:, :3] = out[5][:, 6::2][:, :3]
    out.append(both)
    return out


def main():
    xs, angs, dds_all, stds_all, fl, ns, cfg_of = [], [], [], [], [], [], []
    images = []
    for i in range(60):
        n = N_PEOPLE[i % len(N_PEOPLE)]
        images.append((i, synthetic.make_crowd(n, seed=i)))
    seed, coinc = coincident_image()
    images.append((len(images), coinc))
    for i, (centers, angles, dds, stds) in images:
        k = (i + i // len(N_PEOPLE)) % len(CONFIGS)   # every size meets several parameter sets
        cfg = CONFIGS[k]
        f = flags(centers, angles, dds, stds, cfg)
        xs += centers
        angs += angles
        dds_all += dds
        stds_all += stds
        fl += f
        ns.append(len(centers))
        cfg_of.append(k)
        print('image', i, 'n', len(centers), 'cfg', k, 'flags', sum(f), flush=True)
    with open(os.path.join(G.OUT, 'pifpaf_002282.json')) as fh:
        _, keypoints = G.preprocess_pifpaf(json.load(fh), im_size=(1238, 374))
    poses = [np.asarray(k, dtype=np.float64) for k in keypoints]
    poses += degenerate_poses(keypoints[0])
    rng = np.random.RandomState(7)
    for _ in range(200):
        p = np.asarray(keypoints[rng.randint(len(keypoints))], dtype=np.float64).copy()
        p[:2, 5:11] += rng.normal(0, 40, (2, 6))
        poses.append(p)
    codes = [CODES[is_raising_hand(p.tolist())] for p in poses]
    torch.manual_seed(1)
    mu = torch.zeros(64)
    u_draws = torch.distributions.Laplace(mu, torch.ones(64)).sample((100,))   # T = -(draws of Laplace(0, 1))
    table = (-u_draws).reshape(-1).numpy().astype(np.float32)
    rad = np.full((len(CONFIGS), 3), np.nan)
    for k, c in enumerate(CONFIGS):
        rad[k, :len(c[0])] = c[0]
    np.savez_compressed(os.path.join(G.OUT, 'ref_activity_batch.npz'), n=np.asarray(ns, dtype=np.int32),
                        cfg=np.asarray(cfg_of, dtype=np.int32), xz=np.asarray(xs, dtype=np.float64),
                        angles=np.asarray(angs, dtype=np.float64), dds=np.asarray(dds_all, dtype=np.float64),
                        stds=np.asarray(stds_all, dtype=np.float64), flags=np.asarray(fl, dtype=bool),
                        cfg_radii=rad, cfg_social_distance=np.asarray([c[1] for c in CONFIGS]),
                        cfg_threshold_dist=np.asarray([c[2] for c in CONFIGS]),
                        cfg_n_samples=np.asarray([c[3] for c in CONFIGS], dtype=np.int32),
                        cfg_threshold_prob=np.asarray([c[4] for c in CONFIGS]), coincident_seed=seed,
                        kps=np.stack(poses), raising=np.asarray(codes, dtype=np.int8), table=table)
    print('ref_activity_batch.npz', len(ns), 'images', len(fl), 'people', int(np.sum(fl)), 'flagged;', len(poses), 'poses',
          np.bincount(codes, minlength=4).tolist())


if __name__ == '__main__':
    main()
