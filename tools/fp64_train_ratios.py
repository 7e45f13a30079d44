"""Print the float64-rule ratios of one fused training step, tensor by tensor: the numbers oracle/fp64_train.LIMITS are
set from (tests/test_train_fp64_gpu.py holds every case to them).  Needs a CUDA device; there is no fallback.

    python tools/fp64_train_ratios.py --kind loco --input 34 --output 9 -L 1024 --stages 3 -B 4096 --entry step
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--kind', default='loco', choices=('loco', 'monoloco'))
    ap.add_argument('--input', type=int, default=34)
    ap.add_argument('--output', type=int, default=9)
    ap.add_argument('-L', type=int, default=1024)
    ap.add_argument('--stages', type=int, default=3)
    ap.add_argument('-B', type=int, default=4096)
    ap.add_argument('--entry', default='step', choices=('step', 'auto', 'dropin'))
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit('fp64_train_ratios: no CUDA device')
    import test_train_fp64_gpu as G
    from oracle import fp64_train as F64
    print(torch.cuda.get_device_name(0))
    pb = G._problem(a.kind, a.input, a.output, a.L, a.stages, a.B)
    tasks = G._tasks(a.input)
    got = G._run_kernel(a.entry, G._model(a.kind, a.input, a.output, a.L, a.stages, pb['sd']), pb, tasks)
    r64, r32 = G._oracles(a.entry, pb, tasks)
    print('keep bits cleared: %.2e' % pb['cleared'])
    print('%-40s %-12s %10s %10s %12s %12s' % ('tensor', 'family', 'L2 ratio', 'max ratio', 'rel-L2 fused', 'rel-L2 fp32'))
    rows = [(n, got['grads'][n], r64['grads'][n], r32['grads'][n], F64.family(n, pb['sd'])) for n in r64['grads']]
    rows += [(n, got['running'][n], r64['running'][n], r32['running'][n], 'running stats') for n in r64['running']]
    if 'loss' in got:
        rows.append(('loss, task values', got['loss'], np.r_[r64['loss'], r64['vals']], np.r_[r32['loss'], r32['vals']], 'loss'))
    if 'g_log_sigmas' in got:
        rows.append(('log_sigmas', got['g_log_sigmas'], r64['g_log_sigmas'], r32['g_log_sigmas'], 'log_sigmas'))
    for n, g, a64, a32, fam in rows:
        l2, mx = F64.grad_rule(g, a64, a32, zero=fam == 'zero')
        nrm = max(float(np.linalg.norm(a64)), 1e-300)
        print('%-40s %-12s %10.2f %10.2f %12.2e %12.2e' % (n, fam, l2, mx, np.linalg.norm(np.ravel(g) - np.ravel(a64)) / nrm,
                                                            np.linalg.norm(np.ravel(a32) - np.ravel(a64)) / nrm))
    bad = G._compare('tool', pb['sd'], got, r64, r32)
    print('over the limits:', bad or 'nothing')
    sys.exit(1 if bad else 0)


if __name__ == '__main__':
    main()
