"""Many images per call: a Python loop of Loco.forward against Loco.forward_batch against the device-level
LocoEngine.forward_images, on the same detections (every image with its own camera matrix).

    python tools/bench_images.py [--reps 20]

Cases: 256 images x 16 detections, 1024 x 4, 64 x 64 (monoloco_pp, width 1024, 3 stages) and monstereo over 64 image
pairs of 8 left x 8 right poses.  Times are wall-clock per call, each call ending in a device synchronisation (Loco.forward
and forward_batch return host tensors; forward_images is followed by torch.cuda.synchronize()), median over --reps calls
after warm-up.  Then the time (CUDA events, medians) of the C calls mlb_forward_images at 4096 rows (256 images x 16)
against a plain single-K mlb_forward of the same 4096 rows, alternating in one process, every argument prepared once.
Prints one JSON line per case and the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from monoloco_b200 import synthetic, engine, _lib as L_  # noqa: E402
from monoloco_b200.network import Loco  # noqa: E402
from monoloco_b200.network.architectures import LocoModel  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader',
                            '-i', str(torch.cuda.current_device())], stdout=subprocess.PIPE, text=True, timeout=30)
        power = q.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = 'unknown'
    return name, power


def kks(n, seed):
    rng = np.random.RandomState(seed)
    return [[[f, 0., rng.uniform(500., 700.)], [0., f, rng.uniform(150., 250.)], [0., 0., 1.]]
            for f in rng.uniform(650., 1300., n)]


def model(isz, osz, seed):
    sd = synthetic.make_state_dict('loco', isz, osz, 1024, 3, seed)
    m = LocoModel(isz, osz, 1024, num_stage=3)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    return m


def median_time(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    name, power = card()
    print(json.dumps({'card': name, 'power_limit, max_sm_clock': power}))
    dev = torch.device('cuda')
    mono = Loco(model=model(34, 9, 1), mode='mono', device=dev)
    stereo = Loco(model=model(68, 10, 2), mode='stereo', device=dev)

    for n_img, n_det in ((256, 16), (1024, 4), (64, 64)):
        kps = synthetic.make_keypoints(n_img * n_det, seed=n_img)
        kl = [kps[i * n_det:(i + 1) * n_det].tolist() for i in range(n_img)]
        kk = kks(n_img, n_det)
        eng = mono.model.engine()
        x = torch.from_numpy(kps).to(dev)
        off = engine.image_offsets([n_det] * n_img)
        t_loop = median_time(lambda: [mono.forward(kl[i], kk[i]) for i in range(n_img)], max(3, args.reps // 4), 1)
        t_batch = median_time(lambda: mono.forward_batch(kl, kk), args.reps, args.warmup)
        t_dev = median_time(lambda: eng.forward_images(x, off, kk, want_xyzc=True), args.reps, args.warmup)
        n = n_img * n_det
        print(json.dumps({'case': 'mono %d images x %d' % (n_img, n_det), 'detections': n,
                          'kernel': eng.last_kernel()[1], 'loop_forward_det_per_s': n / t_loop,
                          'forward_batch_det_per_s': n / t_batch, 'forward_images_det_per_s': n / t_dev,
                          'loop_ms': t_loop * 1e3, 'forward_batch_ms': t_batch * 1e3, 'forward_images_ms': t_dev * 1e3,
                          'card': name, 'power_limit': power}))

    n_img, nl, nr = 64, 8, 8
    left = synthetic.make_keypoints(n_img * nl, seed=5)
    right = synthetic.make_keypoints(n_img * nr, seed=6)
    ll = [left[i * nl:(i + 1) * nl].tolist() for i in range(n_img)]
    rl = [right[i * nr:(i + 1) * nr].tolist() for i in range(n_img)]
    kk = kks(n_img, 7)
    eng = stereo.model.engine()
    xl, xr = torch.from_numpy(left).to(dev), torch.from_numpy(right).to(dev)
    lo, ro = engine.image_offsets([nl] * n_img), engine.image_offsets([nr] * n_img)
    row_off = engine.image_offsets([nl * nr] * n_img)
    t_loop = median_time(lambda: [stereo.forward(ll[i], kk[i], rl[i]) for i in range(n_img)], max(3, args.reps // 4), 1)
    t_batch = median_time(lambda: stereo.forward_batch(ll, kk, rl), args.reps, args.warmup)
    t_dev = median_time(lambda: eng.forward_images(xl, row_off, kk, kind=L_.IN_KPS_STEREO, x_right=xr, left_off=lo,
                                                   right_off=ro, want_xyzc=True), args.reps, args.warmup)
    n = n_img * nl   # detections = left poses (one kept row each after the filter, ties aside)
    print(json.dumps({'case': 'stereo %d image pairs x (%d left x %d right)' % (n_img, nl, nr), 'detections': n,
                      'network_rows': n_img * nl * nr, 'kernel': eng.last_kernel()[1],
                      'loop_forward_det_per_s': n / t_loop, 'forward_batch_det_per_s': n / t_batch,
                      'forward_images_det_per_s': n / t_dev, 'loop_ms': t_loop * 1e3, 'forward_batch_ms': t_batch * 1e3,
                      'forward_images_ms': t_dev * 1e3, 'card': name, 'power_limit': power}))

    # kernel time at 4096 rows: per-row K^-1 lookup against the single-K launch, alternating, CUDA events around the C
    # calls with every argument (offsets, K^-1, outputs) prepared once, so that host-side packing is not in the window
    import ctypes as C
    eng = mono.model.engine()
    lib = L_.lib()
    x = torch.from_numpy(synthetic.make_keypoints(4096, seed=11)).to(dev)
    kk = kks(256, 12)
    a = L_.MlbForwardArgs()
    a.input_kind, a.n_rows, a.z_met, a.x = L_.IN_KPS, 4096, 10.0, x.data_ptr()
    keep_out = eng._outputs(a, 4096, True, True, False, None, 0)
    ib, keep_ib = eng._image_batch(engine.image_offsets([16] * 256), kk, 4096)
    a1 = L_.MlbForwardArgs.from_buffer_copy(a)
    for i, v in enumerate(engine.kinv_from_kk(kk[0])):
        a1.kinv[i] = float(v)
    st = eng._stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(call):
        e0.record()
        L_.check(call(), 'forward')
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)
    run_img = lambda: lib.mlb_forward_images(eng._h, C.byref(a), C.byref(ib), st)  # noqa: E731
    run_one = lambda: lib.mlb_forward(eng._h, C.byref(a1), st)  # noqa: E731
    for _ in range(5):
        timed(run_img), timed(run_one)
    t_img, t_one = [], []
    for _ in range(max(50, args.reps)):
        t_img.append(timed(run_img))
        k_img = eng.last_kernel()[1]
        t_one.append(timed(run_one))
        k_one = eng.last_kernel()[1]
    del keep_out, keep_ib
    print(json.dumps({'case': 'kernel time, 4096 rows (256 images x 16 vs one K)', 'forward_images_ms': float(np.median(t_img)),
                      'forward_single_K_ms': float(np.median(t_one)), 'kernel_images': k_img, 'kernel_single_K': k_one,
                      'pairs': len(t_img), 'card': name, 'power_limit': power}))


if __name__ == '__main__':
    main()
