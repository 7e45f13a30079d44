"""Trainer without a GPU: the mlb_task_stats_args layout, the initial weights and batch order of the reference Trainer
(fixtures of tools/gen_trainer_golden.py), the float64 statement of mlb_task_stats against the reference's
compute_stats / mt_loss(..., 'val') results, and the rejections that need no device."""
import ctypes as C
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

torch = pytest.importorskip('torch')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
RUNS = ('mono_mtl', 'mono_auto', 'stereo_mtl', 'stereo_auto')
HIDDEN, STAGES, BS, R_SEED = 64, 2, 128, 7
JOINT_SEED = {'mono': 11, 'stereo': 12}
CLUSTERS = ('all', '10', '20', '30', '40')


def _fx(run):
    return np.load(os.path.join(GOLDEN, 'ref_trainer_%s.npz' % run))


def _tasks(mode):
    return ('d', 'x', 'y', 'h', 'w', 'l', 'ori') + (('aux',) if mode == 'stereo' else ())


def test_task_stats_args_layout_matches_header(tmp_path):
    from monoloco_b200 import _lib as L_
    cls = L_.MlbTaskStatsArgs
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "monoloco_b200.h"', 'int main(void) {',
             '  printf("sizeof %zu\\n", sizeof(mlb_task_stats_args));']
    lines += ['  printf("%s %%zu\\n", offsetof(mlb_task_stats_args, %s));' % (f, f) for f, _ in cls._fields_]
    lines += ['  printf("max_seg %d nacc %d\\n", MLB_STATS_MAX_SEG, MLB_STATS_NACC);',
              '  printf("idx %d %d %d %d %d %d %d %d %d %d\\n", MLB_STAT_N, MLB_STAT_TOTAL, MLB_STAT_VAL, MLB_STAT_BI,',
              '         MLB_STAT_BI_HIT, MLB_STAT_ERR, MLB_STAT_ERR2, MLB_STAT_AUX_MISS, MLB_STAT_LAPLACE, MLB_STAT_ORI_L1);',
              '  return 0;', '}']
    src = tmp_path / 'layout.c'
    src.write_text('\n'.join(lines))
    exe = tmp_path / 'layout'
    subprocess.run(['gcc', '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)],
                   check=True)
    out = dict(l.split(' ', 1) for l in subprocess.run([str(exe)], check=True, stdout=subprocess.PIPE,
                                                       text=True).stdout.splitlines())
    assert int(out['sizeof']) == C.sizeof(cls)
    for f, _ in cls._fields_:
        assert int(out[f]) == getattr(cls, f).offset, f
    assert out['max_seg'] == '%d nacc %d' % (L_.STATS_MAX_SEG, L_.STATS_NACC)
    assert [int(v) for v in out['idx'].split()] == [L_.STAT_N, L_.STAT_TOTAL, L_.STAT_VAL, L_.STAT_BI, L_.STAT_BI_HIT,
                                                    L_.STAT_ERR, L_.STAT_ERR2, L_.STAT_AUX_MISS, L_.STAT_LAPLACE,
                                                    L_.STAT_ORI_L1]


def _sha(sd):
    h = hashlib.sha256()
    for k, v in sd.items():
        h.update(k.encode())
        h.update(np.ascontiguousarray(v.detach().cpu().numpy()).tobytes())
    return h.hexdigest()


@pytest.mark.parametrize('run', RUNS)
def test_initial_weights_bit_identical(run):
    """Trainer seeds the CPU generator and builds LocoModel on the CPU, as the reference does (trainer.py:84-123)."""
    from monoloco_b200.network.architectures import LocoModel
    mode = run.split('_')[0]
    torch.manual_seed(R_SEED)
    model = LocoModel(34 if mode == 'mono' else 68, 9 if mode == 'mono' else 10, linear_size=HIDDEN, p_dropout=0.0,
                      num_stage=STAGES)
    assert _sha(model.state_dict()) == str(_fx(run)['init_sha'])


def test_batch_order_matches_reference_loaders(tmp_path):
    """Per epoch: the train loader's permutation, then the val loader's, after the model's initial draws."""
    from monoloco_b200 import synthetic
    from monoloco_b200.network.architectures import LocoModel
    from monoloco_b200.train import DeviceLoader, KeypointsDataset
    f = _fx('mono_mtl')
    path = str(tmp_path / 'joints.json')
    synthetic.make_trainer_joints(path, seed=JOINT_SEED['mono'])
    loaders = {ph: DeviceLoader(KeypointsDataset(path, ph), BS, shuffle=True, device='cpu') for ph in ('train', 'val')}
    ids = {ph: {tuple(r): i for i, r in enumerate(loaders[ph].inputs.numpy())} for ph in loaders}
    torch.manual_seed(R_SEED)
    LocoModel(34, 9, linear_size=HIDDEN, p_dropout=0.0, num_stage=STAGES)
    got = {'train': [], 'val': []}
    n_epochs = f['epoch_losses'].shape[2]
    for _ in range(n_epochs):
        for ph in ('train', 'val'):
            for x, _, _, _ in loaders[ph]:
                got[ph] += [ids[ph][tuple(r)] for r in x.numpy()]
    for ph in ('train', 'val'):
        np.testing.assert_array_equal(np.array(got[ph]), f['order_' + ph])


def _val_pairs(f):
    k = 0
    while 'val_%d_out' % k in f:
        yield f['val_%d_out' % k], f['val_%d_lab' % k], f['val_%d_res' % k]
        k += 1


@pytest.mark.parametrize('run', RUNS)
def test_host_mirror_matches_reference_val_losses(run):
    """mt_loss(outputs, labels, 'val'): the val-form value per task and the train-form total (for AutoTune with the
    log_sigmas recovered from the exp(log_sigma) values the same call returns)."""
    from monoloco_b200 import _lib as L_
    from monoloco_b200.train.stats import task_stats_host, val_values
    mode, kind = run.split('_')
    tasks = _tasks(mode)
    for out, lab, res in _val_pairs(_fx(run)):
        acc = task_stats_host(out, lab, [0, out.shape[0]], tasks)[0]
        np.testing.assert_allclose(val_values(acc, tasks), res[1:1 + len(tasks)], rtol=2e-6, atol=1e-6)
        if kind == 'mtl':
            np.testing.assert_allclose(acc[L_.STAT_TOTAL] / out.shape[0], res[0], rtol=2e-6)
        else:   # AutoTune: the val call also returns exp(log_sigma); the total with those sigmas must match
            ls = np.log(res[1 + len(tasks):]).astype(np.float32)
            acc = task_stats_host(out, lab, [0, out.shape[0]], tasks, log_sigmas=ls)[0]
            np.testing.assert_allclose(acc[L_.STAT_TOTAL] / out.shape[0], res[0], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize('run', ('mono_mtl', 'stereo_mtl', 'stereo_auto'))
def test_host_mirror_matches_reference_compute_stats(run):
    from monoloco_b200 import _lib as L_
    from monoloco_b200.train.stats import err_std, task_stats_host, val_values
    f = _fx(run)
    mode = run.split('_')[0]
    tasks = _tasks(mode)
    for s, clst in enumerate(CLUSTERS):
        out, lab = f['stats_%d_out' % s], f['stats_%d_lab' % s]
        n = out.shape[0]
        acc = task_stats_host(out, lab, [0, n], tasks)[0]
        ref = dict(zip(('d', 'x', 'y', 'h', 'w', 'l', 'ori', 'bi', 'bi%', 'std', 'aux'), f['dic_err'][s]))
        got = dict(zip(tasks, val_values(acc, tasks)))
        got.update(bi=acc[L_.STAT_BI] / n, std=err_std(acc))
        for k in ('d', 'x', 'y', 'h', 'w', 'l', 'ori', 'bi', 'std'):
            np.testing.assert_allclose(got[k], ref[k], rtol=1e-5, err_msg='%s %s' % (clst, k))
        assert abs(acc[L_.STAT_BI_HIT] - ref['bi%'] * n) < 0.5
        if mode == 'stereo':
            assert abs(n - acc[L_.STAT_AUX_MISS] - ref['aux'] * n) < 0.5 + 1e-6 * n


def test_task_stats_rejections_without_gpu():
    from monoloco_b200.train.stats import _mask, _seg_off
    with pytest.raises(ValueError, match='unknown tasks'):
        _mask(('d', 'z'))
    with pytest.raises(ValueError, match='in the order'):
        _mask(('x', 'd'))
    with pytest.raises(ValueError, match='seg_off'):
        _seg_off([0])
    with pytest.raises(ValueError, match='seg_off'):
        _seg_off(list(range(19)))


def test_trainer_refuses_without_cuda_and_keeps_reference_asserts(tmp_path, monkeypatch):
    import argparse
    from monoloco_b200.train import Trainer
    args = argparse.Namespace(mode='mono', joints=str(tmp_path / 'missing.json'), epochs=1, no_save=True,
                              print_loss=False, lr=1e-3, sched_step=20, sched_gamma=1, hidden_size=64, n_stage=1,
                              r_seed=1, auto_tune_mtl=False, out=None, bs=16, dropout=0.0)
    with pytest.raises(AssertionError, match='Input file not found'):
        Trainer(args)
    from monoloco_b200 import synthetic
    args.joints = str(tmp_path / 'j.json')
    synthetic.make_trainer_joints(args.joints, n_train=20, n_val=10)
    args.out = str(tmp_path / 'nodir' / 'm.pkl')
    with pytest.raises(AssertionError, match='Directory to save the model not found'):
        Trainer(args)
    args.out = str(tmp_path / 'm.pkl')
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: False)
    with pytest.raises(RuntimeError, match='CUDA only'):
        Trainer(args)
