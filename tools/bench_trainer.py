"""Milliseconds per epoch of the training loop on cuda:0, three loops alternating in one process:
  * trainer:   monoloco_b200.train.Trainer (train_step + FusedClipAdam + StepLR + mlb_task_stats per batch, one copy
               of the statistics per epoch);
  * ref_loop:  the reference's loop body (trainer.py:150-167, 193-197) over the same fused LocoModel: torch
               MultiTaskLoss, backward, clip_grad_norm_, torch.optim.Adam, the val-form losses and `.item()` per batch;
  * eager:     the same loop in torch-eager CUDA autograd on the oracle's functional model (oracle/torch_port.py).
Each epoch = the train phase + the val phase. Also reports host synchronisations per epoch (counted with
torch.cuda.set_sync_debug_mode('warn')), library launches per epoch, and the share of the epoch spent in the eval
engine's host re-pack (model.eval() after training steps).

    python tools/bench_trainer.py [--epochs 5] [--rounds 3] [--out DIR]
Defaults: 20 000 train / 2 000 val synthetic rows, batch 512, width 1024, 3 stages, mono, p = 0.2."""
import argparse
import json
import os
import sys
import tempfile
import time
import warnings

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from monoloco_b200 import _lib as L_, synthetic  # noqa: E402
from monoloco_b200.train import Trainer, CompositeLoss, MultiTaskLoss  # noqa: E402
from monoloco_b200.train.stats import task_stats  # noqa: F401,E402
from oracle import torch_port as T  # noqa: E402
from tools.bench_train_monoloco import card  # noqa: E402

TASKS = ('d', 'x', 'y', 'h', 'w', 'l', 'ori')


def make_trainer(joints, tmp):
    args = argparse.Namespace(mode='mono', joints=joints, epochs=1, no_save=True, print_loss=False, lr=1e-3,
                              sched_step=20, sched_gamma=0.98, hidden_size=1024, n_stage=3, r_seed=1,
                              auto_tune_mtl=False, out=os.path.join(tmp, 'm.pkl'), bs=512, dropout=0.2)
    tr = Trainer(args)
    tr._print_losses = lambda el: None
    return tr


def trainer_epoch(tr):
    tr.train()


def ref_loop_epoch(state):
    """trainer.py:144-167 with epoch_logs, on the fused LocoModel."""
    model, mt, opt, sched, loaders = state
    running = {}
    for phase in ('train', 'val'):
        model.train(phase == 'train')
        for x, y, _, _ in loaders[phase]:
            with torch.set_grad_enabled(phase == 'train'):
                if phase == 'train':
                    opt.zero_grad()
                    out = model(x)
                    loss, _ = mt(out, y, phase=phase)
                    loss.backward()
                    torch.nn.utils.clip_grad_norm_(model.parameters(), 3)
                    opt.step()
                    sched.step()
                else:
                    out = model(x)
                with torch.no_grad():
                    le, vals = mt(out, y, phase='val')
                    running[phase] = running.get(phase, 0.0) + le.item() * x.shape[0]
                    for v in vals:
                        running[phase] += v.item() * x.shape[0]


def eager_epoch(state):
    sd, params, opt, sched, loaders = state
    running = 0.0
    for phase in ('train', 'val'):
        for x, y, _, _ in loaders[phase]:
            if phase == 'train':
                opt.zero_grad()
                out = T.model_forward(sd, x, training=True, p_dropout=0.2)
                loss, _ = T.multi_task_loss(out, y, TASKS)
                loss.backward()
                torch.nn.utils.clip_grad_norm_(params, 3)
                opt.step()
                sched.step()
            else:
                with torch.no_grad():
                    out = T.model_forward(sd, x, training=False)
            with torch.no_grad():
                le, vals = T.multi_task_loss(out.detach(), y, TASKS)
                running += le.item() * x.shape[0]
                for v in vals:
                    running += v.item() * x.shape[0]


def timed(fn, arg):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn(arg)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def count_syncs(fn, arg):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn(arg)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum(1 for x in w if 'synchroniz' in str(x.message))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--epochs', type=int, default=5, help='timed epochs per loop and round')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--n-train', type=int, default=20000)
    ap.add_argument('--n-val', type=int, default=2000)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_trainer.py measures on a CUDA device"
    tmp = tempfile.mkdtemp()
    joints = os.path.join(tmp, 'joints.json')
    synthetic.make_trainer_joints(joints, n_train=a.n_train, n_val=a.n_val, seed=3)
    import logging
    logging.disable(logging.INFO)

    tr = make_trainer(joints, tmp)
    # the reference loop on its own fused model, same data on the device
    torch.manual_seed(1)
    from monoloco_b200.network.architectures import LocoModel
    model = LocoModel(34, 9, linear_size=1024, p_dropout=0.2, num_stage=3).cuda()
    mt = MultiTaskLoss(*CompositeLoss(TASKS)(), (1,) * len(TASKS), TASKS)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    ref_state = (model, mt, opt, torch.optim.lr_scheduler.StepLR(opt, 20, 0.98), tr.dataloaders)
    sd = T.to_torch({k: v.detach() for k, v in model.state_dict().items()}, requires_grad=True)
    params = [v for v in sd.values() if v.requires_grad]
    opt_e = torch.optim.Adam(params, lr=1e-3)
    eager_state = (sd, params, opt_e, torch.optim.lr_scheduler.StepLR(opt_e, 20, 0.98), tr.dataloaders)

    loops = (('trainer', trainer_epoch, tr), ('ref_loop', ref_loop_epoch, ref_state), ('eager', eager_epoch, eager_state))
    for _, fn, st in loops:          # warm-up: workspaces, engines, optimizer state, cuBLAS
        fn(st)
    times = {name: [] for name, _, _ in loops}
    for _ in range(a.rounds):
        for name, fn, st in loops:
            times[name].append(np.median([timed(fn, st) for _ in range(a.epochs)]))
    res = {'card': card(), 'config': 'mono, %d train / %d val rows, bs 512, width 1024, 3 stages, p 0.2'
           % (a.n_train, a.n_val)}
    for name, _, _ in loops:
        t = np.array(times[name])
        res[name + '_ms_per_epoch'] = float(np.median(t))
        res[name + '_spread_ms'] = [float(t.min()), float(t.max())]
    for name, fn, st in loops:
        n0 = L_.lib().mlb_launch_count()
        res[name + '_syncs_per_epoch'] = count_syncs(fn, st)
        res[name + '_lib_launches_per_epoch'] = int(L_.lib().mlb_launch_count() - n0)
    # the eval engine's host re-pack: once per epoch, at the first val forward after training steps
    tr.model.train()
    tr._run_phase('train', torch.zeros((1, L_.STATS_NACC), dtype=torch.float64, device='cuda'))
    tr.model.eval()
    x = tr.dataloaders['val'].inputs[:2]
    rep = []
    for _ in range(5):
        tr.optimizer.step()          # bumps the parameter versions: the next eval forward re-packs
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.no_grad():
            tr.model(x)
        torch.cuda.synchronize()
        rep.append((time.perf_counter() - t0) * 1e3)
    res['eval_repack_ms'] = float(np.median(rep))
    res['eval_repack_share_of_trainer_epoch'] = res['eval_repack_ms'] / res['trainer_ms_per_epoch']
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'bench_trainer.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
