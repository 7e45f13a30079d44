"""
Training-step fixtures at hidden widths the fused step runs padded or in two column parts, from the REAL reference
LocoModel + MultiTaskLoss / AutoTuneMultiTaskLoss on the CPU (dropout p = 0, like oracle/gen_golden.py::ref_losses).
TEST INFRASTRUCTURE ONLY; needs the reference sources (oracle/gen_golden.py imports them).

    python tools/gen_train_wide_golden.py

Writes tests/golden/ref_train_wide_<mode>_l<L>_s<stages>.npz: inputs, labels, outputs, loss, per-task values, every
parameter gradient and the buffers after the step.  To keep the fixtures small, a gradient with more than FULL_MAX
entries is stored as N_SAMPLE entries at fixed flat positions (gidx / gval) plus the L2 norm of the whole tensor.
Weights are regenerated from monoloco_b200.synthetic seeds; the state-dict checksum is stored.  B * L stays below 2^20
so the tight gradient rule of the tests applies.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gen_golden as G  # noqa: E402  (imports the reference)

torch = G.torch

# (mode, L, stages, B, AutoTune, seed): the hyp_tuning configuration (2048, 3 stages), a padded stereo width with
# AutoTune, a width with L % 4 != 0 (unaligned rows and masks) and a padded width above 1024 (1536 = two parts of 768)
CONFIGS = (('mono', 2048, 3, 64, False, 31), ('stereo', 300, 2, 70, True, 32), ('mono', 1001, 1, 50, False, 33),
           ('stereo', 1500, 1, 40, False, 34))


FULL_MAX = 16384   # gradients up to this size are stored whole
N_SAMPLE = 4096    # larger ones: this many entries at fixed positions, plus the L2 norm of the whole tensor


def grad_entries(k, g):
    if g.size <= FULL_MAX:
        return {'grad.' + k: g}
    idx = np.sort(np.random.RandomState(g.size % 100003).choice(g.size, N_SAMPLE, replace=False)).astype(np.int64)
    return {'gidx.' + k: idx, 'gval.' + k: g.reshape(-1)[idx], 'gnorm.' + k: float(np.linalg.norm(g.astype(np.float64))),
            'gshape.' + k: np.array(g.shape)}


def name_of(mode, L, st):
    return 'ref_train_wide_%s_l%d_s%d' % (mode, L, st)


def main():
    for mode, L, st, B, auto, seed in CONFIGS:
        isz, osz = (34, 9) if mode == 'mono' else (68, 10)
        tasks = ('d', 'x', 'y', 'h', 'w', 'l', 'ori') + (('aux',) if mode == 'stereo' else ())
        lambdas = (1,) * len(tasks)
        sd = G.synthetic.make_state_dict('loco', isz, osz, L, st, seed)
        model = G.LocoModel(isz, osz, L, 0.0, st, device='cpu')
        model.load_state_dict(G.sd_to_torch(sd))
        model.train()
        x = G.synthetic.make_inputs(B, isz, seed=200 + seed)
        y = G.synthetic.make_labels(B, stereo=(mode == 'stereo'), seed=300 + seed)
        losses_tr, losses_val = G.CompositeLoss(tasks)()
        if auto:
            mt = G.AutoTuneMultiTaskLoss(losses_tr, losses_val, lambdas, tasks)
            with torch.no_grad():
                mt.log_sigmas.copy_(torch.linspace(-0.3, 0.4, len(tasks)))
        else:
            mt = G.MultiTaskLoss(losses_tr, losses_val, lambdas, tasks)
        out = model(torch.from_numpy(x))
        loss, vals = mt(out, torch.from_numpy(y), phase='train')
        loss.backward()
        save = dict(x=x, y=y, out=out.detach().numpy(), loss=float(loss), vals=np.array([float(v) for v in vals]),
                    cfg=np.array([isz, osz, L, st, seed, B]), auto=int(auto), checksum=G.sd_checksum(sd))
        for k, p in model.named_parameters():
            save.update(grad_entries(k, p.grad.numpy()))
        for k, b in model.named_buffers():
            save['buf.' + k] = b.detach().numpy()
        if auto:
            save['grad.log_sigmas'] = mt.log_sigmas.grad.numpy()
            save['log_sigmas'] = mt.log_sigmas.detach().numpy()
        np.savez_compressed(os.path.join(G.OUT, name_of(mode, L, st) + '.npz'), **save)
        print(name_of(mode, L, st), float(loss))


if __name__ == '__main__':
    main()
