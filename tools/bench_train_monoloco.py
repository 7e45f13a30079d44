"""Time one MonolocoModel training step on cuda:0: forward + torch loss + backward on the fused kernels (the autograd
drop-in, one forward and one backward launch) against torch-eager CUDA autograd of the same step.

    python tools/bench_train_monoloco.py [B ...] [--width L] [--stages S] [--outputs O] [--pdrop P]
    (defaults: B = 4096, L = 1024, S = 3, O = 9, P = 0.2: the BASELINE configuration MonolocoModel(34, 9, 1024))

The loss is monoloco_p's: LaplacianLoss on 'zb' = out[:, 2:4] against label column 2 plus L1 on out[:, 4:9] (with 2
outputs, LaplacianLoss on out[:, 0:2] against column 3).  Timings are CUDA events over `--steps` steps after `--warmup`,
fused and eager alternating for `--rounds` rounds; the median round is printed with the spread."""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from monoloco_b200 import synthetic  # noqa: E402
from monoloco_b200.network.architectures import MonolocoModel  # noqa: E402
from monoloco_b200.train.fused import phase_times  # noqa: E402
from oracle import torch_port as T  # noqa: E402


def loss_of(out, y):
    def laplace(mu_si, xx):
        mu, si = mu_si[:, 0:1], mu_si[:, 1:2]
        return (torch.abs(1 - mu / xx) * torch.exp(-si) + 0.01 + si + 2).mean()
    if out.shape[1] == 2:
        return laplace(out[:, 0:2], y[:, 3:4])
    return laplace(out[:, 2:4], y[:, 2:3]) + torch.nn.functional.l1_loss(out[:, 4:9], y[:, 4:9])


def timeit(fn, n, warm):
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


def card():
    """Name, power limit and max SM clock of the card the numbers belong to (read-only query)."""
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=20)
        return r.stdout.strip() or torch.cuda.get_device_name(0)
    except Exception:
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('batch', type=int, nargs='*', default=[4096])
    ap.add_argument('--width', type=int, default=1024)
    ap.add_argument('--stages', type=int, default=3)
    ap.add_argument('--outputs', type=int, default=9)
    ap.add_argument('--pdrop', type=float, default=0.2)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_train_monoloco needs a CUDA device')
    L, st, osz, pd = args.width, args.stages, args.outputs, args.pdrop
    print('card: %s | MonolocoModel(34, %d, %d), %d stages, p_dropout %.2f, TF32 %s'
          % (card(), osz, L, st, pd, torch.backends.cuda.matmul.allow_tf32))
    for B in args.batch:
        sd = synthetic.make_state_dict('monoloco', 34, osz, L, st, 7)
        m = MonolocoModel(34, osz, L, p_dropout=pd, num_stage=st)
        m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
        m.cuda().train()
        x = torch.from_numpy(synthetic.make_inputs(B, 34, seed=3)).cuda()
        y = torch.from_numpy(synthetic.make_labels(B, seed=4)).cuda()

        def fused():
            m.zero_grad(set_to_none=True)
            loss_of(m(x), y).backward()

        tsd = {k: (torch.as_tensor(v).cuda().requires_grad_(True)
                   if ('running' not in k and torch.as_tensor(v).is_floating_point()) else torch.as_tensor(v).cuda())
               for k, v in sd.items()}

        def eager():
            for v in tsd.values():
                v.grad = None
            loss_of(T.model_forward(tsd, x, training=True, p_dropout=pd), y).backward()

        tf, te = [], []
        for _ in range(args.rounds):
            tf.append(timeit(fused, args.steps, args.warmup))
            te.append(timeit(eager, args.steps, args.warmup))
        # per-phase wall times of one forward launch and of one backward launch
        m.zero_grad(set_to_none=True)
        out = m(x)
        ph_f = phase_times(m)
        loss_of(out, y).backward()
        ph_b = phase_times(m)
        print('  forward phases (ms):', ' '.join('%s%d:%.3f' % (n, b, ms) for n, b, ms in ph_f))
        print('  backward phases (ms):', ' '.join('%s%d:%.3f' % (n, b, ms) for n, b, ms in ph_b))
        print('  forward launch %.3f ms, backward launch %.3f ms (sum of phases)'
              % (sum(ms for _, _, ms in ph_f), sum(ms for _, _, ms in ph_b)))
        mf, me = float(np.median(tf)), float(np.median(te))
        print('train step B=%d: fused drop-in %.3f ms [%.3f..%.3f] | torch-eager CUDA %.3f ms [%.3f..%.3f] | eager/fused x%.2f'
              % (B, mf, min(tf), max(tf), me, min(te), max(te), me / mf))


if __name__ == '__main__':
    main()
