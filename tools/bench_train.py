"""Time the fused train step (single cooperative launch) vs torch-eager CUDA autograd of the same step on cuda:0.

    python tools/bench_train.py [B ...] [--width L] [--stages S]     (defaults: B = 4096 512, L = 1024, S = 3)"""
import argparse
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from monoloco_b200 import synthetic
from monoloco_b200.train import train_step, CompositeLoss, MultiTaskLoss
from monoloco_b200.network.architectures import LocoModel
from oracle import torch_port as T

tasks = ('d', 'x', 'y', 'h', 'w', 'l', 'ori')


def timeit(fn, n=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


ap = argparse.ArgumentParser()
ap.add_argument('batch', type=int, nargs='*', default=[4096, 512])
ap.add_argument('--width', type=int, default=1024, help='hidden width (linear_size), 1..2048')
ap.add_argument('--stages', type=int, default=3)
args = ap.parse_args()
Lw, st = args.width, args.stages
def _power_limit():
    import subprocess   # read-only query of the card the numbers belong to
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=20)
        return r.stdout.strip() or 'unknown'
    except Exception:
        return 'unknown'


print('%s, power limit %s, width %d, %d stages' % (torch.cuda.get_device_name(0), _power_limit(), Lw, st))
for B in args.batch:
    sd = synthetic.make_state_dict('loco', 34, 9, Lw, st, 7)
    PD = float(os.environ.get('MLB_BENCH_PDROP', '0.2'))
    m = LocoModel(34, 9, Lw, p_dropout=PD, num_stage=st)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    m.cuda().train()
    x = torch.from_numpy(synthetic.make_inputs(B, 34, seed=3)).cuda()
    y = torch.from_numpy(synthetic.make_labels(B, seed=4)).cuda()
    mt = MultiTaskLoss(*CompositeLoss(tasks)(), (1,) * len(tasks), tasks)
    t_fused = timeit(lambda: train_step(m, x, y, tasks))
    from monoloco_b200.train.fused import phase_times
    print('   phases (ms):', ' '.join('%s%d:%.3f' % (n, b, ms) for n, b, ms in phase_times(m)))
    if os.environ.get('MLB_SUBPHASES'):
        from monoloco_b200.train.fused import subphase_times
        for n, b, pts in subphase_times(m):
            if n in ('FWD', 'BWD', 'FWD_FINAL'):
                # CTA first | last: stats loaded, rows finished, act written, tile ready, GEMM done, epilogue done, barrier left
                print('   %-9s %d  ' % (n, b) + ' | '.join(' '.join('%.3f' % pts[c][k] for k in (4, 5, 6, 0, 1, 2, 3)) for c in (0, 2)))

    def dropin():
        m.zero_grad(set_to_none=True)
        loss, _ = mt(m(x), y, phase='train')
        loss.backward()
    t_dropin = timeit(dropin)
    # torch-eager CUDA (cuBLAS SGEMM, TF32 off) -- the only GPU implementation the reference has
    tsd = {k: (torch.as_tensor(v).cuda().requires_grad_(True) if ('running' not in k and torch.as_tensor(v).is_floating_point())
               else torch.as_tensor(v).cuda()) for k, v in sd.items()}

    def eager():
        for v in tsd.values():
            v.grad = None
        out = T.model_forward(tsd, x, training=True, p_dropout=PD)
        loss, _ = T.multi_task_loss(out, y, tasks)
        loss.backward()
    t_eager = timeit(eager)
    fl = 3 * 2 * (34 * Lw + (2 * st + 2) * Lw * Lw + 9 * Lw) * B   # forward + 2x backward multiply-adds of the Linears
    print("train step L=%d B=%5d: fused 1-launch %.3f ms (%.1f TFLOP/s) | drop-in autograd (2 launches) %.3f ms | torch-eager CUDA %.3f ms | x%.2f"
          % (Lw, B, t_fused, fl / t_fused / 1e9, t_dropin, t_eager, t_eager / t_fused))
