"""
Trainer fixtures from the REAL reference `monoloco.train.Trainer` on the CPU (matplotlib stubbed, no_save=True, dropout
p = 0 so that the CPU dropout draws no numbers and the loaders' permutations are those of a CUDA run).  TEST
INFRASTRUCTURE ONLY; needs the reference sources (oracle/gen_golden.py imports them).

    python tools/gen_trainer_golden.py

Runs (hidden width 64, 2 stages, batch 128 over 600 train / 150 val rows: 4 full batches and a ragged one, 8 epochs):
mono plain, mono AutoTune (train() only: its evaluate() raises IndexError), stereo plain, stereo AutoTune.
Writes tests/golden/ref_trainer_<mode>_<mtl|auto>.npz with
  * init_sha: sha256 of the initial state_dict (tensors in key order, raw bytes) -- bit identity without the weights;
  * epoch_losses: [phase, el, epoch] for phase train / val and el all + tasks; best_epoch;
  * final_out: eval outputs of the returned (best) model on the val inputs -- the final weights, seen through eval;
  * order_<phase>: the dataset rows of every epoch's batches (mono plain only: the order depends on the seed alone);
  * val_<k>_{out,lab,res}: the first train batch's and the ragged val batch's (outputs, labels) given to
    mt_loss(..., phase='val') in epoch 0, with the reference's (loss, loss values);
  * stats_<k>_{out,lab}, dic_err: the (outputs, labels) given to compute_stats by evaluate(load=True, model=<checkpoint
    of synthetic.make_state_dict('loco', in, out, 64, 2, CKPT_SEED)>) and its dic_err (not for mono AutoTune).
"""
import argparse
import hashlib
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gen_golden as G  # noqa: E402  (imports the reference)

torch = G.torch
from monoloco.train.trainer import Trainer  # noqa: E402  (the reference's)

RUNS = (('mono', False), ('mono', True), ('stereo', False), ('stereo', True))
HIDDEN, STAGES, BS, EPOCHS, LR, R_SEED, CKPT_SEED = 64, 2, 128, 8, 0.002, 7, 77
JOINT_SEED = {'mono': 11, 'stereo': 12}
DIC_KEYS = ('d', 'x', 'y', 'h', 'w', 'l', 'ori', 'bi', 'bi%', 'std', 'aux')
CLUSTERS = ('all', '10', '20', '30', '40')


def name_of(mode, auto):
    return 'ref_trainer_%s_%s' % (mode, 'auto' if auto else 'mtl')


def args_for(mode, auto, joints):
    return argparse.Namespace(mode=mode, joints=joints, epochs=EPOCHS, no_save=True, print_loss=False, lr=LR,
                              sched_step=20, sched_gamma=0.9, hidden_size=HIDDEN, n_stage=STAGES, r_seed=R_SEED,
                              auto_tune_mtl=auto, out=None, bs=BS, dropout=0.0)


def state_sha(sd):
    h = hashlib.sha256()
    for k, v in sd.items():
        h.update(k.encode())
        h.update(np.ascontiguousarray(v.detach().cpu().numpy()).tobytes())
    return h.hexdigest()


def check_dropout_p0_draws_nothing():
    drop = torch.nn.Dropout(p=0.0).train()
    before = torch.get_rng_state()
    drop(torch.ones(64, 64))
    assert torch.equal(before, torch.get_rng_state()), "nn.Dropout(p=0) drew from the generator"


def run(mode, auto, tmp):
    joints = os.path.join(tmp, 'joints_%s.json' % mode)
    dic = G.synthetic.make_trainer_joints(joints, stereo=mode == 'stereo', seed=JOINT_SEED[mode])
    os.makedirs(os.path.join(tmp, 'data', 'outputs'), exist_ok=True)
    cwd = os.getcwd()
    os.chdir(tmp)   # the reference asserts data/outputs exists
    try:
        tr = Trainer(args_for(mode, auto, joints))
    finally:
        os.chdir(cwd)
    save = {'init_sha': np.array(state_sha(tr.model.state_dict()))}
    rows = {ph: {tuple(np.float32(r)): i for i, r in enumerate(np.asarray(dic[ph]['X'], dtype=np.float32))}
            for ph in ('train', 'val')}
    order = {'train': [], 'val': []}
    for ph in ('train', 'val'):
        loader = tr.dataloaders[ph]
        # the batch order: wrap the loader so every batch's dataset rows are recorded (no extra draws)
        class Rec:  # noqa: E306
            def __init__(self, inner, ph):
                self.inner, self.ph = inner, ph

            def __iter__(self):
                for b in self.inner:
                    order[self.ph].append([rows[self.ph][tuple(r)] for r in b[0].numpy()])
                    yield b
        tr.dataloaders[ph] = Rec(loader, ph)
    calls = []
    fwd = tr.mt_loss.forward

    def mt_forward(outputs, labels, phase='train'):
        res = fwd(outputs, labels, phase=phase)
        if phase == 'val':
            calls.append((outputs.detach().numpy().copy(), labels.numpy().copy(),
                          np.array([float(res[0])] + [float(v) for v in res[1]])))
        return res
    tr.mt_loss.forward = mt_forward
    captured = {}
    tr._print_losses = lambda el: captured.update(el=el)
    best = tr.train()
    el = captured['el']
    keys = ['all'] + list(tr.tasks)
    save['epoch_losses'] = np.array([[el[ph][k] for k in keys] for ph in ('train', 'val')])
    save['best_epoch'] = np.array(best)
    tr.model.eval()
    with torch.no_grad():
        save['final_out'] = tr.model(torch.tensor(dic['val']['X'], dtype=torch.float32)).numpy()
    if (mode, auto) == ('mono', False):
        for ph in ('train', 'val'):
            save['order_' + ph] = np.concatenate([np.asarray(b, dtype=np.int16) for b in order[ph]])
    n_tr, n_val = (-(-len(dic[ph]['X']) // BS) for ph in ('train', 'val'))
    for k, idx in enumerate((0, n_tr + n_val - 1)):   # epoch 0: the first train batch, the last (ragged) val batch
        o, lab, res = calls[idx]
        save['val_%d_out' % k], save['val_%d_lab' % k], save['val_%d_res' % k] = o, lab, res
    if not (mode == 'mono' and auto):
        isz, osz = (34, 9) if mode == 'mono' else (68, 10)
        sd = G.synthetic.make_state_dict('loco', isz, osz, HIDDEN, STAGES, CKPT_SEED)
        ckpt = os.path.join(tmp, 'ckpt_%s.pkl' % mode)
        torch.save(G.sd_to_torch(sd), ckpt)
        pairs = []
        cs = tr.compute_stats

        def compute_stats(outputs, labels, dic_err, size_eval, clst):
            pairs.append((outputs.numpy().copy(), labels.numpy().copy()))
            return cs(outputs, labels, dic_err, size_eval, clst)
        tr.compute_stats = compute_stats
        dic_err, _ = tr.evaluate(load=True, model=ckpt)
        for k, (o, lab) in enumerate(pairs):
            save['stats_%d_out' % k], save['stats_%d_lab' % k] = o, lab
        e = dic_err['val']
        save['dic_err'] = np.array([[float(e[c][k]) for k in DIC_KEYS] for c in CLUSTERS])
        save['dic_err_sigmas'] = np.array(e['sigmas'], dtype=np.float64)
    return save


def main():
    check_dropout_p0_draws_nothing()
    with tempfile.TemporaryDirectory() as tmp:
        for mode, auto in RUNS:
            save = run(mode, auto, tmp)
            np.savez_compressed(os.path.join(G.OUT, name_of(mode, auto) + '.npz'), **save)
            print(name_of(mode, auto), 'best_epoch', int(save['best_epoch']),
                  'val d', np.round(save['epoch_losses'][1, 1], 4).tolist())


if __name__ == '__main__':
    main()
