"""The predict chain over many images: Loco.predict_batch against the four-call chain on the same inputs (host
preprocess_pifpaf per image, forward_batch, post_process_batch, social_distance_batch, raising_hand_batch).

    python tools/bench_predict.py [--shapes 1024x4 64x16] [--reps 20]

Mono LocoModel (width 1024, 3 stages), annotations drawn from the pifpaf fixture, both activities (S = 100 samples,
radii (0.3, 0.5, 1), threshold_dist 2, threshold_prob 0.25).  Wall time: host clock around a call (each call ends in a
stream synchronisation), the two variants alternating in the same process, median over --reps.  Device time: the sum of
the CUDA kernel and copy times torch.profiler records for one call, in separate profiled calls after the timed ones.
Prints the card's name and power limit beside the numbers."""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from monoloco_b200 import synthetic  # noqa: E402
from monoloco_b200.network import Loco  # noqa: E402
from monoloco_b200.network.architectures import LocoModel  # noqa: E402
from monoloco_b200.network.post import post_process_batch  # noqa: E402
from monoloco_b200.network.process import preprocess_pifpaf  # noqa: E402

ARGS = SimpleNamespace(threshold_prob=0.25, threshold_dist=2.0, radii=(0.3, 0.5, 1.0))
ACTS = ('social_distance', 'raise_hand')


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = torch.cuda.get_device_name() + ', power limit unknown'
    return q


def images(n_img, per_img, seed=0):
    with open(os.path.join(ROOT, 'tests', 'golden', 'pifpaf_002282.json')) as f:
        base = json.load(f)
    rng = np.random.RandomState(seed)
    ann_list = []
    for _ in range(n_img):
        anns = []
        for j in rng.choice(len(base), size=per_img, replace=True):
            a = copy.deepcopy(base[int(j)])
            s = float(rng.uniform(-60, 60))
            a['keypoints'][0::3] = [x + s for x in a['keypoints'][0::3]]
            a['bbox'] = [a['bbox'][0] + s, a['bbox'][1], a['bbox'][2] + s, a['bbox'][3]]
            anns.append(a)
        ann_list.append(anns)
    kk = [[718.3351, 0., 600.3891], [0., 718.3351, 181.5122], [0., 0., 1.]]
    return ann_list, [kk] * n_img, [(1238., 374.)] * n_img


def four_calls(net, ann_list, kks, sizes):
    pre = [preprocess_pifpaf(a, s, enlarge_boxes=False) for a, s in zip(ann_list, sizes)]
    bl, kl = [b for b, _ in pre], [k for _, k in pre]
    posts = post_process_batch([(d, b, k, K, None) for d, b, k, K in zip(net.forward_batch(kl, kks), bl, kl, kks)])
    posts = Loco.raising_hand_batch(Loco.social_distance_batch(posts, ARGS), kl)
    return list(zip(bl, kl, posts))


def one_call(net, ann_list, kks, sizes):
    return net.predict_batch(ann_list, kks, sizes, activities=ACTS, args=ARGS)


def device_ms(fn, reps=3):
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    total_us = sum(e.device_time_total for e in prof.key_averages() if e.device_type.name == 'CUDA' and e.device_time_total)
    kernels = sum(e.count for e in prof.key_averages() if e.device_type.name == 'CUDA')
    return total_us / 1e3 / reps, kernels / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--shapes', nargs='+', default=['1024x4', '64x16'])
    ap.add_argument('--reps', type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_predict needs a CUDA device')
    print('card:', card())
    sd = synthetic.make_state_dict('loco', 34, 9, 1024, 3, 1)
    m = LocoModel(34, 9, 1024, num_stage=3)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    net = Loco(model=m, mode='mono', device=torch.device('cuda'))
    print('%10s | %-12s | %9s %9s | %9s %11s' % ('images', 'variant', 'wall ms', 'ms/image', 'device ms', 'dev ops/call'))
    for shape in a.shapes:
        n_img, per = (int(v) for v in shape.split('x'))
        inputs = images(n_img, per)
        variants = (('four calls', four_calls), ('predict_batch', one_call))
        ref, got = four_calls(net, *inputs), one_call(net, *inputs)
        assert [(b, k, dict(d)) for b, k, d in ref] == [(b, k, dict(d)) for b, k, d in got], 'results differ'
        for _ in range(3):
            for _, fn in variants:
                fn(net, *inputs)
        wall = {name: [] for name, _ in variants}
        for _ in range(a.reps):
            for name, fn in variants:
                t0 = time.perf_counter()
                fn(net, *inputs)
                wall[name].append((time.perf_counter() - t0) * 1e3)
        for name, fn in variants:
            dms, ops = device_ms(lambda: fn(net, *inputs))
            w = statistics.median(wall[name])
            print('%10s | %-12s | %9.2f %9.4f | %9.3f %11.0f' % (shape, name, w, w / n_img, dms, ops))
        print('%10s | speed-up of predict_batch (wall, median): %.2fx' %
              (shape, statistics.median(wall['four calls']) / statistics.median(wall['predict_batch'])))


if __name__ == '__main__':
    main()
