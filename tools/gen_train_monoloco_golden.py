"""
Training-step fixtures for MonolocoModel (the legacy `monoloco` / `monoloco_p` nets and the BASELINE configuration),
from the REAL reference MonolocoModel on the CPU with dropout p = 0.  TEST INFRASTRUCTURE ONLY; needs the reference
sources (oracle/gen_golden.py imports them).

    python tools/gen_train_monoloco_golden.py

The reference defines no multi-task loss on MonolocoModel's outputs, so each fixture uses the loss of the net it stands
for, built from the reference's own loss modules:
  * 2 outputs (legacy monoloco, out = (d, log b)): LaplacianLoss(out[:, 0:2], labels[:, 3:4]);
  * 9 outputs (monoloco_p): LaplacianLoss on 'zb' = out[:, 2:4] (process.py:340) against labels[:, 2:3], plus
    nn.L1Loss(out[:, 4:9], labels[:, 4:9]).

Writes tests/golden/ref_train_monoloco_o<out>_l<L>_s<stages>.npz: inputs, labels, outputs, loss, every parameter
gradient and the buffers after the step, in the format of tools/gen_train_wide_golden.py (a gradient with more than
FULL_MAX entries is stored as a fixed sample plus the L2 norm of the whole tensor).  B * L stays below 2^20 so the
tight gradient rule of the tests applies.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from oracle import gen_golden as G  # noqa: E402  (imports the reference)
from gen_train_wide_golden import grad_entries  # noqa: E402

torch = G.torch
from monoloco.train.losses import LaplacianLoss  # noqa: E402  (the reference's, on sys.path through gen_golden)

# (input, output, L, stages, B, seed): legacy monoloco, monoloco_p, the BASELINE configuration MonolocoModel(34, 9, 1024),
# a padded width and a width run in two column parts
CONFIGS = ((34, 2, 256, 3, 64, 41), (34, 9, 256, 3, 64, 42), (34, 9, 1024, 3, 64, 43), (34, 9, 300, 2, 70, 44),
           (34, 9, 2048, 2, 48, 45))


def name_of(osz, L, st):
    return 'ref_train_monoloco_o%d_l%d_s%d' % (osz, L, st)


def monoloco_loss(out, y):
    """The loss of the net a MonolocoModel of this output size stands for (module docstring)."""
    if out.shape[1] == 2:
        return LaplacianLoss()(out[:, 0:2], y[:, 3:4])
    return LaplacianLoss()(out[:, 2:4], y[:, 2:3]) + torch.nn.L1Loss()(out[:, 4:9], y[:, 4:9])


def main():
    for isz, osz, L, st, B, seed in CONFIGS:
        assert B * L < (1 << 20)
        sd = G.synthetic.make_state_dict('monoloco', isz, osz, L, st, seed)
        model = G.MonolocoModel(isz, osz, L, 0.0, st)
        model.load_state_dict(G.sd_to_torch(sd))
        model.train()
        x = G.synthetic.make_inputs(B, isz, seed=200 + seed)
        y = G.synthetic.make_labels(B, seed=300 + seed)
        out = model(torch.from_numpy(x))
        loss = monoloco_loss(out, torch.from_numpy(y))
        loss.backward()
        save = dict(x=x, y=y, out=out.detach().numpy(), loss=float(loss), cfg=np.array([isz, osz, L, st, seed, B]),
                    checksum=G.sd_checksum(sd))
        for k, p in model.named_parameters():
            save.update(grad_entries(k, p.grad.numpy()))
        for k, b in model.named_buffers():
            save['buf.' + k] = b.detach().numpy()
        np.savez_compressed(os.path.join(G.OUT, name_of(osz, L, st) + '.npz'), **save)
        print(name_of(osz, L, st), float(loss))


if __name__ == '__main__':
    main()
