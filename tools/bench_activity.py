"""Activity heuristics over many images: a per-image host loop of Loco.social_distance, Loco.social_distance_batch (host
lists in, pinned staging, one synchronisation) and social_distance_device alone (device tensors in, CUDA events).

    python tools/bench_activity.py [--images 64 256] [--people 8 20 40] [--host-images 3] [--reps 20]

S = 100 samples, radii (0.3, 0.5, 1), threshold_dist 2, threshold_prob 0.25.  The host loop runs on --host-images images
only (40 people take seconds each) and is reported per image; the batched paths run on every image.  Prints the card's
name and power limit beside the numbers."""
import argparse
import copy
import os
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
from monoloco_b200.network.post import social_distance_device  # noqa: E402

ARGS = SimpleNamespace(threshold_prob=0.25, threshold_dist=2.0, radii=(0.3, 0.5, 1.0))


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = torch.cuda.get_device_name() + ', power limit unknown'
    return q


def dicts(n_img, n_people, seed):
    out = []
    for i in range(n_img):
        c, a, d, s = synthetic.make_crowd(n_people, seed=seed + i)
        out.append({'xyz_pred': [[x, 1.0, z] for x, z in c], 'angles': a, 'dds_pred': d, 'stds_ale': s})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, nargs='+', default=[64, 256])
    ap.add_argument('--people', type=int, nargs='+', default=[8, 20, 40])
    ap.add_argument('--host-images', type=int, default=3)
    ap.add_argument('--reps', type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_activity needs a CUDA device')
    print('card:', card())
    print('%7s %7s | %14s | %12s %10s | %12s %10s | %s' % ('images', 'people', 'host ms/image', 'batch ms', 'ms/image',
                                                          'device ms', 'ms/image', 'flagged'))
    for n_people in a.people:
        for n_img in a.images:
            ds = dicts(n_img, n_people, seed=1000 * n_people)
            # host loop, a few images
            t0 = time.perf_counter()
            ref = [Loco.social_distance(copy.deepcopy(d), ARGS)['social_distance'] for d in ds[:a.host_images]]
            host = (time.perf_counter() - t0) * 1e3 / a.host_images
            # batched API (host lists in, flags out), warm-up then timed
            got = Loco.social_distance_batch([copy.deepcopy(d) for d in ds], ARGS)
            assert [g['social_distance'] for g in got[:a.host_images]] == ref
            work = [copy.deepcopy(ds) for _ in range(a.reps)]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for w in work:
                Loco.social_distance_batch(w, ARGS)
            batch = (time.perf_counter() - t0) * 1e3 / a.reps
            # device path alone: tensors already on the device
            xz = torch.tensor([[p[0], p[2]] for d in ds for p in d['xyz_pred']], dtype=torch.float64, device='cuda')
            ang = torch.tensor([v for d in ds for v in d['angles']], dtype=torch.float64, device='cuda')
            dd = torch.tensor([v for d in ds for v in d['dds_pred']], dtype=torch.float32, device='cuda')
            sd = torch.tensor([v for d in ds for v in d['stds_ale']], dtype=torch.float32, device='cuda')
            off = np.arange(n_img + 1) * n_people
            d_off = torch.from_numpy(off.astype(np.int32)).cuda()
            kw = dict(threshold_prob=ARGS.threshold_prob, threshold_dist=ARGS.threshold_dist, radii=ARGS.radii,
                      max_people=n_people)
            flags = social_distance_device(xz, ang, dd, sd, d_off, **kw)
            assert flags.cpu().tolist() == [v for g in got for v in g['social_distance']]
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(a.reps):
                social_distance_device(xz, ang, dd, sd, d_off, **kw)
            end.record()
            torch.cuda.synchronize()
            dev = start.elapsed_time(end) / a.reps
            print('%7d %7d | %14.2f | %12.3f %10.4f | %12.3f %10.5f | %d/%d' % (
                n_img, n_people, host, batch, batch / n_img, dev, dev / n_img, int(flags.sum()), flags.numel()), flush=True)
    # one small image: the per-image host call against a one-image batch
    ds = dicts(1, 8, seed=7)
    t0 = time.perf_counter()
    for _ in range(a.reps):
        Loco.social_distance(copy.deepcopy(ds[0]), ARGS)
    host = (time.perf_counter() - t0) * 1e3 / a.reps
    Loco.social_distance_batch(copy.deepcopy(ds), ARGS)
    t0 = time.perf_counter()
    for _ in range(a.reps):
        Loco.social_distance_batch(copy.deepcopy(ds), ARGS)
    batch = (time.perf_counter() - t0) * 1e3 / a.reps
    print('one image of 8 people: host %.2f ms, social_distance_batch %.3f ms' % (host, batch))


if __name__ == '__main__':
    main()
