"""GPU: `Trainer` on the fused kernels against the reference Trainer (fixtures of tools/gen_trainer_golden.py) and
`mlb_task_stats` against its float64 statement."""
import argparse
import json
import os

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
HIDDEN, STAGES, BS, EPOCHS, LR, R_SEED, CKPT_SEED = 64, 2, 128, 8, 0.002, 7, 77
JOINT_SEED = {'mono': 11, 'stereo': 12}
CLUSTERS = ('all', '10', '20', '30', '40')
DIC_KEYS = ('d', 'x', 'y', 'h', 'w', 'l', 'ori', 'bi', 'bi%', 'std', 'aux')
# DESIGN §5c: measured deviations of the fused Trainer from the reference trajectory and the rules derived from them
FIRST_EPOCH_RTOL = 1e-5     # epoch 0 train phase: measured <= 4e-7 (five steps from bit-identical weights)
TRAIN_LOSS_RTOL = 0.1       # any epoch, train phase: measured <= 3.7e-2 (stereo AutoTune, epoch 7)
VAL_RTOL = 0.15             # any epoch, val phase: measured <= 7.2e-2
FINAL_OUT_DEV = 0.5         # eval outputs of the returned model / column max: measured <= 0.20


def _fx(mode, auto):
    return np.load(os.path.join(GOLDEN, 'ref_trainer_%s_%s.npz' % (mode, 'auto' if auto else 'mtl')))


def _tasks(mode):
    return ('d', 'x', 'y', 'h', 'w', 'l', 'ori') + (('aux',) if mode == 'stereo' else ())


def _trainer(tmp_path, mode, auto, epochs=EPOCHS, hidden=HIDDEN, stages=STAGES, dropout=0.0, n_train=600, n_val=150,
             bs=BS, no_save=True):
    from monoloco_b200 import synthetic
    from monoloco_b200.train import Trainer
    joints = str(tmp_path / ('joints_%s.json' % mode))
    synthetic.make_trainer_joints(joints, n_train=n_train, n_val=n_val, stereo=mode == 'stereo', seed=JOINT_SEED[mode])
    args = argparse.Namespace(mode=mode, joints=joints, epochs=epochs, no_save=no_save, print_loss=False, lr=LR,
                              sched_step=20, sched_gamma=0.9, hidden_size=hidden, n_stage=stages, r_seed=R_SEED,
                              auto_tune_mtl=auto, out=str(tmp_path / ('%s-test.pkl' % ('monoloco_pp' if mode == 'mono' else 'monstereo'))), bs=bs, dropout=dropout)
    return Trainer(args)


def _train(tr):
    got = {}
    tr._print_losses = lambda el: got.update(el=el)
    best = tr.train()
    return best, got['el']


# ---------------------------------------------------------------------------------------------------- 1. the kernel
def _random_rows(n, stereo, seed):
    rng = np.random.RandomState(seed)
    out = rng.normal(0, 1, (n, 10 if stereo else 9)).astype(np.float32)
    out[:, 2] = rng.uniform(1, 50, n)
    lab = rng.normal(0, 1, (n, 11 if stereo else 10)).astype(np.float32)
    lab[:, 3] = rng.uniform(1, 50, n)
    if stereo:
        lab[:, 10] = rng.randint(0, 2, n)
        out[:50, 9] = 0.0                          # sigmoid(0) = 0.5 counts as a positive
    # ties err == bi: log b = 0 (bi = d exactly) and d_gt = 2 d (err = d exactly)
    out[50:100, 3] = 0.0
    lab[50:100, 3] = 2 * out[50:100, 2]
    return out, lab


@pytest.mark.parametrize('stereo', (False, True))
@pytest.mark.parametrize('auto', (False, True))
def test_task_stats_kernel_matches_host_mirror(stereo, auto):
    from monoloco_b200 import _lib as L_
    from monoloco_b200.train import task_stats
    from monoloco_b200.train.stats import task_stats_host
    mode = 'stereo' if stereo else 'mono'
    tasks = _tasks(mode)
    f = _fx(mode, False)
    pieces = [_random_rows(100000, stereo, 5)] + [(f['stats_%d_out' % s], f['stats_%d_lab' % s]) for s in range(5)]
    pieces += [(f['val_%d_out' % k], f['val_%d_lab' % k]) for k in range(2)] + [_random_rows(1, stereo, 6)]
    out = np.concatenate([p[0] for p in pieces])
    lab = np.concatenate([p[1] for p in pieces])
    sizes = [p[0].shape[0] for p in pieces]
    sizes = sizes[:3] + [0] + sizes[3:] + [0]    # segments of length 0, a 1-row segment (std NaN)
    off = np.concatenate(([0], np.cumsum(sizes))).tolist()
    lam = tuple(1.0 + 0.25 * i for i in range(len(tasks)))
    ls = torch.linspace(-0.5, 0.7, len(tasks), device='cuda') if auto else None
    o, y = torch.from_numpy(out).cuda(), torch.from_numpy(lab).cuda()
    a1 = task_stats(o, y, off, tasks, lam, ls).cpu().numpy()
    a2 = task_stats(o, y, off, tasks, lam, ls).cpu().numpy()
    assert a1.tobytes() == a2.tobytes(), "two launches on the same inputs differ"
    ref = task_stats_host(out, lab, off, tasks, lam, None if ls is None else ls.cpu().numpy())
    count_cols = [L_.STAT_N, L_.STAT_BI_HIT, L_.STAT_AUX_MISS]
    # fp32 expf in the bi and sigmoid comparisons may differ from numpy's by one ulp: a row may change sides
    assert np.abs(a1[:, count_cols] - ref[:, count_cols]).max() <= 1
    np.testing.assert_array_equal(a1[:, L_.STAT_N], ref[:, L_.STAT_N])
    sums = [c for c in range(L_.STATS_NACC) if c not in count_cols + [L_.STAT_BI]]
    np.testing.assert_allclose(a1[:, sums], ref[:, sums], rtol=1e-10, atol=1e-9)
    # bi = expf(log b) * d in fp32: at most one ulp per (positive) row from numpy's exp
    np.testing.assert_allclose(a1[:, L_.STAT_BI], ref[:, L_.STAT_BI], rtol=2.4e-7)
    tie = ref[0]
    assert tie[L_.STAT_BI_HIT] == a1[0, L_.STAT_BI_HIT]
    assert (a1[3] == 0).all() and (a1[-1] == 0).all()        # empty segments add nothing
    from monoloco_b200.train.stats import err_std
    assert np.isnan(err_std(a1[-2])) and a1[-2, L_.STAT_N] == 1
    # accumulation: a second launch into the same buffer adds
    acc = task_stats(o, y, off, tasks, lam, ls)
    task_stats(o, y, off, tasks, lam, ls, acc=acc)
    np.testing.assert_allclose(acc.cpu().numpy(), 2 * a1, rtol=1e-14)


def test_task_stats_rejections():
    from monoloco_b200 import _lib as L_
    import ctypes as C
    from monoloco_b200.train import task_stats
    o = torch.zeros((4, 9), device='cuda')
    y = torch.ones((4, 10), device='cuda')
    n0 = L_.lib().mlb_launch_count()
    with pytest.raises(RuntimeError, match='non-decreasing'):
        task_stats(o, y, [0, 3, 2], ('d',))
    with pytest.raises(RuntimeError, match='aux task needs'):
        task_stats(o, y, [0, 4], ('d', 'aux'))
    with pytest.raises(RuntimeError, match='out_cols'):
        task_stats(torch.zeros((4, 8), device='cuda'), y, [0, 4], ('d',))
    a = L_.MlbTaskStatsArgs()
    a.n_seg, a.out_cols, a.label_ld, a.task_mask = 1, 9, 10, 1 << 9
    assert L_.lib().mlb_task_stats(C.byref(a), None) != 0 and b'task_mask' in L_.lib().mlb_last_error()
    a.task_mask = 1
    assert L_.lib().mlb_task_stats(C.byref(a), None) != 0 and b'acc is NULL' in L_.lib().mlb_last_error()
    assert L_.lib().mlb_task_stats(None, None) != 0
    assert L_.lib().mlb_launch_count() == n0


# ---------------------------------------------------------------------------------------------------- 2. evaluate
def _ckpt(tmp_path, mode):
    from monoloco_b200 import synthetic
    isz, osz = (34, 9) if mode == 'mono' else (68, 10)
    sd = synthetic.make_state_dict('loco', isz, osz, HIDDEN, STAGES, CKPT_SEED)
    path = str(tmp_path / ('ckpt_%s.pkl' % mode))
    torch.save({k: torch.from_numpy(np.array(v)) for k, v in sd.items()}, path)
    return path


@pytest.mark.parametrize('run', (('mono', False), ('stereo', False), ('stereo', True)))
def test_evaluate_against_reference_dic_err(tmp_path, run):
    mode, auto = run
    f = _fx(mode, auto)
    tr = _trainer(tmp_path, mode, auto, epochs=0)
    if auto:
        # the fixture evaluated after train(): its sigmas are 5 (segments) * exp(trained log_sigma)
        sig = torch.from_numpy(f['dic_err_sigmas'] / len(CLUSTERS)).float()
        tr.mt_loss.log_sigmas.data.copy_(torch.log(sig).cuda())
    dic_err, model = tr.evaluate(load=True, model=_ckpt(tmp_path, mode))
    assert model is tr.model
    e = dic_err['val']
    worst = 0.0
    for s, clst in enumerate(CLUSTERS):
        n = len(tr.datasets['val']) if clst == 'all' else tr.datasets['val'].get_cluster_annotations(clst)[2]
        for k, key in enumerate(DIC_KEYS):
            ref, got = float(f['dic_err'][s, k]), float(e[clst][key])
            if key in ('bi%', 'aux') and not (mode == 'mono' and key == 'aux'):
                assert abs(got - ref) * n <= 1 + 1e-6, (clst, key, got, ref)
            else:
                rel = abs(got - ref) / max(abs(ref), 1e-30)
                worst = max(worst, rel)
                assert rel <= 1e-5, (clst, key, got, ref)
        assert isinstance(e[clst]['std'], torch.Tensor)
    print('evaluate %s auto=%s worst rel %.3g' % (mode, auto, worst))
    np.testing.assert_allclose(np.array(e['sigmas'], dtype=np.float64), f['dic_err_sigmas'], rtol=1e-6)


def test_evaluate_mono_autotune_raises_like_reference(tmp_path):
    tr = _trainer(tmp_path, 'mono', True, epochs=0)
    with pytest.raises(IndexError):
        tr.evaluate(load=True, model=_ckpt(tmp_path, 'mono'))


def test_evaluate_refuses_split_over_val_bs_before_launch(tmp_path):
    from monoloco_b200 import _lib as L_
    tr = _trainer(tmp_path, 'mono', False, epochs=0, n_train=200, n_val=60)
    tr.VAL_BS = 50
    n0 = L_.lib().mlb_launch_count()
    with pytest.raises(AssertionError, match='partial evaluation'):
        tr.evaluate()
    assert L_.lib().mlb_launch_count() == n0
    with pytest.raises(NotImplementedError):
        tr.evaluate(debug=True)


# ---------------------------------------------------------------------------------------------------- 3. train()
@pytest.mark.parametrize('mode', ('mono', 'stereo'))
@pytest.mark.parametrize('auto', (False, True))
def test_train_against_reference_trajectory(tmp_path, mode, auto):
    f = _fx(mode, auto)
    tr = _trainer(tmp_path, mode, auto)
    best, el = _train(tr)
    keys = ['all'] + list(tr.tasks)
    got = np.array([[el[ph][k] for k in keys] for ph in ('train', 'val')])
    ref = f['epoch_losses']
    rel = np.abs(got - ref) / np.maximum(np.abs(ref), 1e-3)
    print('train %s auto=%s  train-phase worst rel %.3g (per epoch %s)  val worst rel %.3g' % (
        mode, auto, rel[0].max(), np.round(rel[0].max(0), 7).tolist(), rel[1].max()))
    assert rel[0, :, 0].max() <= FIRST_EPOCH_RTOL
    assert rel[0].max() <= TRAIN_LOSS_RTOL
    assert rel[1].max() <= VAL_RTOL
    # best_epoch: wherever the reference's val-d margin between the best epoch and the runner-up exceeds twice the
    # val-d deviation measured in this very run
    val_d = ref[1, 1]
    order = np.argsort(val_d)
    margin = (val_d[order[1]] - val_d[order[0]]) / val_d[order[0]]
    print('val d: worst rel deviation %.3g, best-epoch margin %.3g' % (rel[1, 1].max(), margin))
    if margin > 2 * rel[1, 1].max():
        assert best == int(f['best_epoch'])
    # final (best) weights, seen through eval outputs on the val inputs
    tr.model.eval()
    with torch.no_grad():
        out = tr.model(tr.dataloaders['val'].inputs).cpu().numpy()
    scale = np.abs(f['final_out']).max(0)
    dev = (np.abs(out - f['final_out']) / np.maximum(scale, 1e-6)).max()
    print('final eval outputs worst deviation / column max %.3g' % dev)
    assert dev <= FINAL_OUT_DEV


# ---------------------------------------------------------------------------------------------------- 4. no sync
def test_train_phase_has_no_host_sync_and_four_launches_per_batch(tmp_path):
    from monoloco_b200 import _lib as L_
    tr = _trainer(tmp_path, 'stereo', True, epochs=1)
    _train(tr)                                   # warm: workspaces, optimizer state, cached task weights
    acc = torch.zeros((1, L_.STATS_NACC), dtype=torch.float64, device='cuda')
    n_batches = len(tr.dataloaders['train'])
    tr.model.train()
    torch.cuda.synchronize()
    n0 = L_.lib().mlb_launch_count()
    torch.cuda.set_sync_debug_mode('error')
    try:
        tr._run_phase('train', acc)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert L_.lib().mlb_launch_count() - n0 == 4 * n_batches
    tr.model.eval()
    with torch.no_grad():
        tr.model(tr.dataloaders['val'].inputs[:2])   # the once-per-epoch host re-pack of the eval engine
    n0 = L_.lib().mlb_launch_count()
    tr._run_phase('val', acc)
    assert L_.lib().mlb_launch_count() - n0 == 2 * len(tr.dataloaders['val'])
    torch.cuda.synchronize()
    assert torch.isfinite(acc).all()


# ---------------------------------------------------------------------------------------------------- 5. end to end
@pytest.mark.parametrize('mode', ('mono', 'stereo'))
def test_end_to_end_width_1024_then_predict(tmp_path, mode):
    from monoloco_b200.network import Loco
    tr = _trainer(tmp_path, mode, False, epochs=6, hidden=1024, stages=3, dropout=0.2, n_train=2000, n_val=300, bs=512,
                  no_save=False)
    best, el = _train(tr)
    tr_all, va_all = el['train']['all'], el['val']['all']
    assert np.isfinite(tr_all).all() and np.isfinite(va_all).all()
    assert tr_all[-1] < tr_all[0]
    dic_err, _ = tr.evaluate()
    assert np.isfinite(dic_err['val']['all']['d'])
    assert os.path.exists(tr.path_model)
    if mode == 'mono':
        with open(os.path.join(GOLDEN, 'pifpaf_002282.json')) as fh:
            from monoloco_b200.network import preprocess_pifpaf, load_calibration
            boxes, keypoints = preprocess_pifpaf(json.load(fh), im_size=(1238, 374))
        kk = load_calibration('kitti', (1238, 374))
        net = Loco(model=tr.path_model, mode='mono', device=torch.device('cuda'), n_dropout=0)
        out = Loco.post_process(net.forward(keypoints, kk), boxes, keypoints, kk)
        assert len(out['xyz_pred']) == 16 and np.isfinite(np.array(out['dds_pred'])).all()
    else:
        v = np.load(os.path.join(GOLDEN, 'kat_stereo_val.npz'))
        left, right = v['kps'][:10, :, :17].tolist(), v['kps'][:7, :, 17:].tolist()
        net = Loco(model=tr.path_model, mode='stereo', device=torch.device('cuda'))
        dic = net.forward(left, v['K'][0].tolist(), right)
        assert dic['xyzd'].shape[0] >= 10 and np.isfinite(dic['d'].numpy()).all()
