"""GPU: the fused training step at hidden widths that are not a multiple of 128 (run zero-padded) and above 1024 (run in
two column parts): against the live-reference fixtures tests/golden/ref_train_wide_*.npz and against torch autograd
(oracle/torch_port.py) with explicit dropout masks.  Same gradient rules as test_train_gpu.py."""
import os

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
WIDE_FIXTURES = ['ref_train_wide_mono_l2048_s3', 'ref_train_wide_stereo_l300_s2', 'ref_train_wide_mono_l1001_s1',
                 'ref_train_wide_stereo_l1500_s1']
TASKS = {'mono': ('d', 'x', 'y', 'h', 'w', 'l', 'ori'), 'stereo': ('d', 'x', 'y', 'h', 'w', 'l', 'ori', 'aux')}


def _model(isz, osz, L, st, seed, p_dropout=0.0):
    from monoloco_b200 import synthetic
    from monoloco_b200.network.architectures import LocoModel
    sd = synthetic.make_state_dict('loco', isz, osz, L, st, seed)
    m = LocoModel(isz, osz, L, p_dropout=p_dropout, num_stage=st)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    return m.cuda(), sd


def _tight(name, got, ref, scale):
    """|a-b| <= 1e-4|b| + 2e-5 max|b| + 2e-7 elementwise (test_train_gpu.py::_cmp_grad)."""
    err = np.abs(got - ref)
    assert (err <= 1e-4 * np.abs(ref) + 2e-5 * scale + 2e-7).all(), (name, float(err.max()), scale)


def _cmp_grad(name, got, ref, rel_l2=1e-5):
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape, name
    _tight(name, got, ref, max(float(np.abs(ref).max()), 1e-12))
    nrm = float(np.linalg.norm(ref))
    if nrm > 1e-5 * np.sqrt(ref.size):
        assert float(np.linalg.norm(got - ref)) / nrm <= rel_l2, (name, float(np.linalg.norm(got - ref)) / nrm)


def _cmp_grad_statistical(name, got, ref, rel_l2=3e-3):
    """Full-size rule of test_train_gpu.py (justified in DESIGN.md §2): rel-L2 <= 3e-3, cosine >= 1 - 1e-5."""
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    scale = max(float(np.abs(ref).max()), 1e-12)
    nrm = float(np.linalg.norm(ref))
    if nrm > 1e-5 * np.sqrt(ref.size):
        assert float(np.linalg.norm(got - ref)) / nrm <= rel_l2, (name, float(np.linalg.norm(got - ref)) / nrm)
        cos = float((got * ref).sum() / (np.linalg.norm(got) * nrm))
        assert cos >= 1.0 - 1e-5, (name, cos)
    else:
        assert np.abs(got - ref).max() <= 2e-5 * scale + 2e-7, name


# w2.bias (LocoModel.w2 has no BatchNorm behind it) gets sum_rows dL/dA with heavy cancellation: the fp32 reference itself
# sits ~1.1e-5 rel-L2 from the fp64 gradient there (measured, DESIGN.md §9), so that one tensor is held to 3e-5
RELL2_FIXTURE = {'w2.bias': 3e-5}


def cmp_fixture_grad(f, name, got):
    """A gradient against a fixture: whole tensors with _cmp_grad; large ones (stored as a fixed sample plus the norm
    of the whole tensor) elementwise on the sample, scaled by the sample's max, and by the whole tensor's norm."""
    got = np.asarray(got, dtype=np.float64)
    if 'grad.' + name in f.files:
        _cmp_grad(name, got, f['grad.' + name], RELL2_FIXTURE.get(name, 1e-5))
        return
    assert tuple(got.shape) == tuple(f['gshape.' + name]), name
    ref = f['gval.' + name].astype(np.float64)
    _tight(name, got.reshape(-1)[f['gidx.' + name]], ref, max(float(np.abs(ref).max()), 1e-12))
    nrm = float(f['gnorm.' + name])
    assert abs(float(np.linalg.norm(got)) - nrm) <= 1e-5 * nrm, (name, float(np.linalg.norm(got)), nrm)


def _load(name):
    f = np.load(os.path.join(GOLDEN, name + '.npz'))
    isz, osz, L, st, seed, B = [int(v) for v in f['cfg']]
    return f, isz, osz, L, st, seed, bool(int(f['auto'])), ('stereo' if isz == 68 else 'mono')


def _check_buffers(model, f):
    for n, b in model.named_buffers():
        if 'num_batches' in n:
            assert int(b) == int(f['buf.' + n]), n
        else:
            assert np.allclose(b.cpu().numpy(), f['buf.' + n], rtol=1e-5, atol=1e-6), n


@pytest.mark.parametrize('name', WIDE_FIXTURES)
def test_train_wide_dropin_vs_reference(name):
    """out = model(x); mt(out, y).backward() at a padded / two-part width against the reference."""
    from monoloco_b200.train import CompositeLoss, MultiTaskLoss, AutoTuneMultiTaskLoss
    f, isz, osz, L, st, seed, auto, mode = _load(name)
    model, _ = _model(isz, osz, L, st, seed)
    tasks = TASKS[mode]
    losses_tr, losses_val = CompositeLoss(tasks)()
    if auto:
        mt = AutoTuneMultiTaskLoss(losses_tr, losses_val, (1,) * len(tasks), tasks).cuda()
        with torch.no_grad():
            mt.log_sigmas.copy_(torch.from_numpy(f['log_sigmas']))
    else:
        mt = MultiTaskLoss(losses_tr, losses_val, (1,) * len(tasks), tasks)
    model.train()
    x, y = torch.from_numpy(f['x']).cuda(), torch.from_numpy(f['y']).cuda()
    out = model(x)
    assert np.allclose(out.detach().cpu().numpy(), f['out'], rtol=1e-5, atol=1e-5)
    loss, vals = mt(out, y, phase='train')
    assert abs(float(loss) - float(f['loss'])) <= 3e-6 * abs(float(f['loss']))
    assert np.allclose(np.array([float(v) for v in vals]), f['vals'], rtol=1e-5)
    loss.backward()
    for n, p in model.named_parameters():
        cmp_fixture_grad(f, n, p.grad.cpu().numpy())
    _check_buffers(model, f)
    if auto:
        assert np.allclose(mt.log_sigmas.grad.cpu().numpy(), f['grad.log_sigmas'], rtol=1e-5)


@pytest.mark.parametrize('name', WIDE_FIXTURES)
def test_train_wide_step_single_launch_vs_reference(name):
    """train_step(): forward + loss + backward in ONE launch at a padded / two-part width."""
    from monoloco_b200.train import train_step
    from monoloco_b200 import _lib as L_
    f, isz, osz, L, st, seed, auto, mode = _load(name)
    model, _ = _model(isz, osz, L, st, seed)
    model.train()
    ls = torch.nn.Parameter(torch.from_numpy(f['log_sigmas']).cuda()) if auto else None
    n0 = L_.lib().mlb_launch_count()
    loss, vals, out = train_step(model, torch.from_numpy(f['x']).cuda(), torch.from_numpy(f['y']).cuda(), TASKS[mode],
                                 log_sigmas=ls)
    assert L_.lib().mlb_launch_count() - n0 == 1
    assert np.allclose(out.cpu().numpy(), f['out'], rtol=1e-5, atol=1e-5)
    assert abs(float(loss) - float(f['loss'])) <= 3e-6 * abs(float(f['loss']))
    assert np.allclose(np.array([float(v) for v in vals]), f['vals'], rtol=1e-5)
    for n, p in model.named_parameters():
        cmp_fixture_grad(f, n, p.grad.cpu().numpy())
    _check_buffers(model, f)
    if auto:
        assert np.allclose(ls.grad.cpu().numpy(), f['grad.log_sigmas'], rtol=1e-5)


def _oracle_step(sd, x, y, masks, p, tasks, dt):
    from oracle import torch_port as T
    tsd = {k: (v.to(dt).detach().requires_grad_(v.requires_grad) if v.is_floating_point() else v)
           for k, v in T.to_torch(sd, requires_grad=True).items()}
    out = T.model_forward(tsd, torch.from_numpy(x).to(dt), training=True, p_dropout=p,
                          masks=[torch.from_numpy(m) for m in masks])
    loss, _ = T.multi_task_loss(out, torch.from_numpy(y).to(dt), tasks)
    loss.backward()
    return tsd, out, loss


def _failures(cmp, model, tsd):
    bad = []
    for n, prm in model.named_parameters():
        try:
            cmp(n, prm.grad.cpu().numpy(), tsd[n].grad.numpy())
        except AssertionError as e:
            bad.append(str(e)[:200])
    return bad


@pytest.mark.parametrize('L,st,B,p', [(200, 2, 301, 0.2), (1001, 1, 257, 0.2), (1500, 1, 300, 0.2), (2048, 3, 500, 0.2),
                                      (2048, 3, 4096, 0.2)])
def test_train_wide_vs_torch_autograd(L, st, B, p):
    """Training step with explicit dropout keep-masks [sites][B][L] vs torch autograd (oracle/torch_port.py).
    Below B*L = 2^20: the tight rule on every gradient against the oracle run in float32 OR in float64.  With up to 10^7
    ReLU / BatchNorm decisions any two summation orders may resolve one borderline unit differently (measured on the
    H100: at L=1500, B=300 the fp32 oracle flips one unit and sits 1e-3 from the fp64 gradient, which the fused step
    matches to 1.4e-6; at L=2048, B=500 the fp64 oracle is the odd one out), so the step has to agree tightly with one of
    the two independent evaluations (DESIGN.md §9).  Full size: the statistical rule against the fp32 oracle, 4e-3 at
    L=2048 (measured, DESIGN.md §9)."""
    from monoloco_b200 import synthetic
    from monoloco_b200.train import train_step
    model, sd = _model(34, 9, L, st, 7, p_dropout=p)
    model.train()
    x = synthetic.make_inputs(B, 34, seed=3)
    y = synthetic.make_labels(B, seed=4)
    n_bn = 2 * st + 2
    rng = np.random.RandomState(5)
    masks = (rng.uniform(size=(n_bn, B, L)) >= p).astype(np.uint8)
    tasks = TASKS['mono']
    loss, vals, out = train_step(model, torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), tasks,
                                 drop_mask=torch.from_numpy(masks).cuda())
    tsd, ref_out, ref_loss = _oracle_step(sd, x, y, masks, p, tasks, torch.float32)
    assert np.allclose(out.cpu().numpy(), ref_out.detach().numpy(), rtol=2e-5, atol=2e-5)
    assert abs(float(loss) - float(ref_loss)) <= 1e-5 * abs(float(ref_loss))
    if B * L >= (1 << 20):
        bad = _failures(lambda n, a, b: _cmp_grad_statistical(n, a, b, 4e-3 if L > 1024 else 3e-3), model, tsd)
        assert not bad, bad
    else:
        bad32 = _failures(_cmp_grad, model, tsd)
        if bad32:
            tsd64, _, _ = _oracle_step(sd, x, y, masks, p, tasks, torch.float64)
            bad64 = _failures(_cmp_grad, model, tsd64)
            assert not bad64, (bad32, bad64)
    for n, b in model.named_buffers():
        if 'num_batches' not in n:
            assert np.allclose(b.cpu().numpy(), tsd[n].detach().numpy(), rtol=2e-5, atol=2e-6), n


@pytest.mark.parametrize('L', [300, 2048])
def test_train_wide_dropout_rng_consistency(L):
    """In-kernel counter RNG at a padded width and at 2048: a seed is reproducible, another seed differs, and forward
    and backward draw the same masks (d sum(out) / d w_fin.bias is exactly B)."""
    from monoloco_b200.train.fused import fused_train_forward
    from monoloco_b200 import synthetic
    model, _ = _model(34, 9, L, 2, 8, p_dropout=0.3)
    model.train()
    x = torch.from_numpy(synthetic.make_inputs(500, 34, seed=1)).cuda()
    a = fused_train_forward(model, x, seed=11)
    b = fused_train_forward(model, x, seed=11)
    c = fused_train_forward(model, x, seed=12)
    assert torch.equal(a, b) and not torch.equal(a, c)
    d = fused_train_forward(model, x, seed=11)
    assert torch.equal(a, d)
    d.sum().backward()
    assert torch.allclose(model.w_fin.bias.grad, torch.full((8,), 500.0, device='cuda'))
    assert float(model.w1.weight.grad.abs().sum()) > 0


@pytest.mark.parametrize('tm', [8, 16])
def test_train_wide_ragged_tiles(tm, monkeypatch):
    """Rows-per-group 8 and 16 at 2048 with a ragged last row tile (padded DW tail), tight rule."""
    monkeypatch.setenv('MLB_TRAIN_ROWS_PER_GROUP', str(tm))
    test_train_wide_vs_torch_autograd(2048, 1, 301, 0.2)


def test_train_wide_more_tiles_than_sms():
    """Batch 6000 at 2048: more row tiles than SMs, so CTAs walk several tiles per phase."""
    test_train_wide_vs_torch_autograd(2048, 1, 6000, 0.2)


def test_train_wide_widths_rejected_above_2048():
    from monoloco_b200.network.architectures import LocoModel
    m = LocoModel(34, 9, 2049, p_dropout=0.0, num_stage=1).cuda().train()
    with pytest.raises(RuntimeError, match='linear_size'):
        m(torch.zeros(8, 34, device='cuda'))


def test_hyp_tuning_2048_end_to_end(tmp_path):
    """The hyp_tuning configuration (hyp_tuning.py:52): LocoModel(34, 9, 2048, 3 stages) trains 10 FusedClipAdam steps
    on the KITTI-format fixture with a decreasing loss; its saved state_dict then runs the inference path
    (Loco.forward + post_process on the pifpaf fixture, tensor-core kernel) with finite outputs.  lr = 1e-4: at the
    trainer's default 1e-3 the loss of this 2048-wide network jumps 5.6 -> 35 after one step and oscillates, with torch
    eager autograd + torch.optim.Adam exactly as with the fused step (measured on the H100)."""
    import json
    from monoloco_b200 import synthetic
    from monoloco_b200.network import Loco, preprocess_pifpaf
    from monoloco_b200.network.architectures import LocoModel
    from monoloco_b200.train import train_step, FusedClipAdam
    torch.manual_seed(0)
    sd = synthetic.make_state_dict('loco', 34, 9, 2048, 3, 5)
    model = LocoModel(34, 9, 2048, p_dropout=0.2, num_stage=3)
    model.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    model = model.cuda().train()
    kat = np.load(os.path.join(GOLDEN, 'kat_mono_train.npz'))
    x = torch.from_numpy(kat['X'].astype(np.float32)).cuda()
    y = torch.from_numpy(kat['Y'].astype(np.float32)).cuda()
    opt = FusedClipAdam(model.parameters(), lr=1e-4, max_norm=3.0)
    losses = []
    for _ in range(10):
        opt.zero_grad()
        loss, _, _ = train_step(model, x, y, TASKS['mono'])
        opt.step()
        losses.append(float(loss))
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
    path = str(tmp_path / 'monoloco_pp-2048.pkl')
    torch.save(model.state_dict(), path)  # trainer.py:242
    net = Loco(model=path, mode='mono', device=torch.device('cuda'), linear_size=2048)
    with open(os.path.join(GOLDEN, 'pifpaf_002282.json')) as fh:
        boxes, keypoints = preprocess_pifpaf(json.load(fh), im_size=(1238, 374))
    kk = synthetic.KITTI_K
    dic = net.forward(keypoints, kk)
    assert net.model.linear_size == 2048 and len(dic['d']) == len(keypoints)
    for k, v in dic.items():
        if isinstance(v, torch.Tensor):
            assert torch.isfinite(v).all(), k
    post = Loco.post_process(dic, boxes, keypoints, kk)
    assert len(post['xyz_pred']) == len(boxes) and np.isfinite(np.asarray(post['xyz_pred'], dtype=np.float64)).all()
