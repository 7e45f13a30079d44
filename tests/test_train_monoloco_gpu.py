"""GPU: MonolocoModel (legacy monoloco / monoloco_p, and the BASELINE configuration MonolocoModel(34, 9, 1024)) trained
through the fused kernels' autograd drop-in: `model.train(); out = model(x); loss(out).backward()` is one forward and
one backward launch.  Against the live-reference fixtures tests/golden/ref_train_monoloco_*.npz and against torch
autograd (oracle/torch_port.py) with explicit dropout masks, with the rules of test_train_wide_gpu.py."""
import json
import os

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')

from test_train_monoloco_golden_cpu import FIXTURES, load_fixture, monoloco_loss  # noqa: E402
from test_train_wide_gpu import _cmp_grad, _cmp_grad_statistical, _failures, cmp_fixture_grad  # noqa: E402


def _model(isz, osz, L, st, seed, p_dropout=0.0):
    from monoloco_b200 import synthetic
    from monoloco_b200.network.architectures import MonolocoModel
    sd = synthetic.make_state_dict('monoloco', isz, osz, L, st, seed)
    m = MonolocoModel(isz, osz, L, p_dropout=p_dropout, num_stage=st)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    return m.cuda(), sd


def _launches():
    from monoloco_b200 import _lib as L_
    return int(L_.lib().mlb_launch_count())


@pytest.mark.parametrize('name', FIXTURES)
def test_monoloco_dropin_vs_reference(name):
    """out = model(x); loss(out, y).backward() against the reference MonolocoModel: outputs, loss, every gradient, the
    running statistics and num_batches_tracked, in one forward and one backward launch."""
    f, isz, osz, L, st, seed, B = load_fixture(name)
    model, _ = _model(isz, osz, L, st, seed)
    model.train()
    x, y = torch.from_numpy(f['x']).cuda(), torch.from_numpy(f['y']).cuda()
    n0 = _launches()
    out = model(x)
    assert out.shape == (B, osz)
    assert np.allclose(out.detach().cpu().numpy(), f['out'], rtol=1e-5, atol=1e-5)
    loss = monoloco_loss(out, y)
    assert abs(float(loss) - float(f['loss'])) <= 3e-6 * abs(float(f['loss']))
    loss.backward()
    assert _launches() - n0 == 2
    for n, p in model.named_parameters():
        cmp_fixture_grad(f, n, p.grad.cpu().numpy())
    for n, b in model.named_buffers():
        if 'num_batches' in n:
            assert int(b) == int(f['buf.' + n]), n
        else:
            assert np.allclose(b.cpu().numpy(), f['buf.' + n], rtol=1e-5, atol=1e-6), n


def _oracle_step(sd, x, y, masks, p, dt):
    from oracle import torch_port as T
    tsd = {k: (v.to(dt).detach().requires_grad_(v.requires_grad) if v.is_floating_point() else v)
           for k, v in T.to_torch(sd, requires_grad=True).items()}
    out = T.model_forward(tsd, torch.from_numpy(x).to(dt), training=True, p_dropout=p,
                          masks=[torch.from_numpy(m) for m in masks])
    loss = monoloco_loss(out, torch.from_numpy(y).to(dt))
    loss.backward()
    return tsd, out, loss


def _vs_autograd(L, st, B, p, osz=9, seed=7):
    """Drop-in step with explicit keep masks [1 + 2 st][B][L] against torch autograd.  Below B*L = 2^20 the tight rule
    against the oracle run in fp32 or in fp64 (test_train_wide_vs_torch_autograd); above, the full-size statistical rule
    (rel-L2 <= 3e-3, cosine >= 1 - 1e-5; 4e-3 above 1024 as for LocoModel, DESIGN.md §9)."""
    from monoloco_b200 import synthetic
    from monoloco_b200.train.fused import fused_train_forward
    model, sd = _model(34, osz, L, st, seed, p_dropout=p)
    model.train()
    x = synthetic.make_inputs(B, 34, seed=3)
    y = synthetic.make_labels(B, seed=4)
    rng = np.random.RandomState(5)
    masks = (rng.uniform(size=(1 + 2 * st, B, L)) >= p).astype(np.uint8)
    out = fused_train_forward(model, torch.from_numpy(x).cuda(), drop_mask=torch.from_numpy(masks).cuda())
    loss = monoloco_loss(out, torch.from_numpy(y).cuda())
    loss.backward()
    tsd, ref_out, ref_loss = _oracle_step(sd, x, y, masks, p, torch.float32)
    assert np.allclose(out.detach().cpu().numpy(), ref_out.detach().numpy(), rtol=2e-5, atol=2e-5)
    assert abs(float(loss) - float(ref_loss)) <= 1e-5 * abs(float(ref_loss))
    if B * L >= (1 << 20):
        bad = _failures(lambda n, a, b: _cmp_grad_statistical(n, a, b, 4e-3 if L > 1024 else 3e-3), model, tsd)
        assert not bad, bad
    else:
        bad32 = _failures(_cmp_grad, model, tsd)
        if bad32:
            tsd64, _, _ = _oracle_step(sd, x, y, masks, p, torch.float64)
            bad64 = _failures(_cmp_grad, model, tsd64)
            if bad64:
                _as_accurate_as_fp32(model, tsd, tsd64, bad32, bad64, 4e-3 if L > 1024 else 3e-3)
    for n, b in model.named_buffers():
        if 'num_batches' not in n:
            assert np.allclose(b.cpu().numpy(), tsd[n].detach().numpy(), rtol=2e-5, atol=2e-6), n


def _as_accurate_as_fp32(model, tsd32, tsd64, bad32, bad64, rel_l2):
    """When borderline ReLU units make the step ill-conditioned, fp32 evaluations in different summation orders flip
    different units, and each may sit outside the tight rule of the fp64 evaluation (DESIGN.md §9).  The fused step must
    then be as accurate as the fp32 oracle over the whole step: its worst rel-L2 from fp64 over all gradients is at most
    the fp32 oracle's, and every gradient holds the full-size statistical rule against fp64."""
    import warnings
    seen = []
    worst_f = worst_o = 0.0
    for n, prm in model.named_parameters():
        got = prm.grad.cpu().numpy().astype(np.float64)
        r64 = tsd64[n].grad.numpy().astype(np.float64)
        r32 = tsd32[n].grad.numpy().astype(np.float64)
        _cmp_grad_statistical(n, got, r64, rel_l2)
        nrm = float(np.linalg.norm(r64))
        if nrm <= 1e-5 * np.sqrt(r64.size):   # exactly-zero true gradients (biases before a BatchNorm): noise only
            continue
        l_f, l_o = float(np.linalg.norm(got - r64)) / nrm, float(np.linalg.norm(r32 - r64)) / nrm
        worst_f, worst_o = max(worst_f, l_f), max(worst_o, l_o)
        # share of the squared error in the worst output unit (row of a weight): one flipped unit puts most of it there
        err2 = (got - r64) ** 2
        row = float(err2.reshape(err2.shape[0], -1).sum(axis=1).max() / max(err2.sum(), 1e-300))
        seen.append((n, '%.2e' % l_f, '%.2e' % l_o, '%.2f' % row))
    # reported: (tensor, fused rel-L2, fp32 oracle rel-L2, worst unit's share of the fused error), against fp64
    warnings.warn('step outside the tight rule of both oracles; fused worst rel-L2 %.2e, fp32 oracle worst %.2e: %s'
                  % (worst_f, worst_o, seen))
    assert worst_f <= max(worst_o, 1e-5), (worst_f, worst_o, bad32, bad64)


@pytest.mark.parametrize('p', [0.0, 0.2])
@pytest.mark.parametrize('L,st,B', [(256, 3, 257), (300, 2, 301), (1024, 3, 257), (2048, 2, 500)])
def test_monoloco_vs_torch_autograd(L, st, B, p):
    _vs_autograd(L, st, B, p)


def test_monoloco_legacy_two_outputs_vs_torch_autograd():
    """The legacy monoloco net: 2 outputs (d, log b), one stage (the smallest block list, 3 blocks)."""
    _vs_autograd(256, 1, 301, 0.2, osz=2)


def test_monoloco_baseline_batch_4096():
    """The BASELINE configuration MonolocoModel(34, 9, 1024) at batch 4096, full-size statistical rule."""
    _vs_autograd(1024, 3, 4096, 0.2)


@pytest.mark.parametrize('tm', [8, 10, 12, 14, 16])
def test_monoloco_ragged_tiles(tm, monkeypatch):
    """Every rows-per-group with a ragged last row tile (padded DW tail), plain path."""
    monkeypatch.setenv('MLB_TRAIN_ROWS_PER_GROUP', str(tm))
    _vs_autograd(1024, 2, 301, 0.2)


@pytest.mark.parametrize('tm', [8, 16])
def test_monoloco_ragged_tiles_two_parts(tm, monkeypatch):
    monkeypatch.setenv('MLB_TRAIN_ROWS_PER_GROUP', str(tm))
    _vs_autograd(2048, 1, 301, 0.2)


def test_monoloco_more_tiles_than_sms():
    """Batch 6000: more row tiles than SMs, so CTAs walk several tiles per phase."""
    _vs_autograd(1024, 2, 6000, 0.2)


@pytest.mark.parametrize('L', [256, 300, 2048])
def test_monoloco_dropout_rng_consistency(L):
    """In-kernel counter RNG: a seed is reproducible and another differs; d sum(out) / d w2.bias is exactly B; and the
    backward draws the forward's masks: the central difference of the loss along w1's gradient matches its norm."""
    from monoloco_b200 import synthetic
    from monoloco_b200.train.fused import fused_train_forward
    model, _ = _model(34, 9, L, 2, 8, p_dropout=0.3)
    model.train()
    B = 500
    x = torch.from_numpy(synthetic.make_inputs(B, 34, seed=1)).cuda()
    y = torch.from_numpy(synthetic.make_labels(B, seed=2)).cuda()
    a = fused_train_forward(model, x, seed=11)
    b = fused_train_forward(model, x, seed=11)
    c = fused_train_forward(model, x, seed=12)
    assert torch.equal(a, b) and not torch.equal(a, c)
    d = fused_train_forward(model, x, seed=11)
    assert torch.equal(a, d)
    d.sum().backward()
    assert torch.equal(model.w2.bias.grad, torch.full((9,), float(B), device='cuda'))
    model.zero_grad()
    loss = monoloco_loss(fused_train_forward(model, x, seed=11), y)
    loss.backward()
    g = model.w1.weight.grad.detach().clone()
    gn = float(g.norm())
    assert gn > 0
    eps = 1e-3 * float(loss) / gn   # a step that moves the loss by ~0.1 %
    w0 = model.w1.weight.detach().clone()
    vals = []
    with torch.no_grad():
        for s in (1.0, -1.0):
            model.w1.weight.copy_(w0 + s * eps * g / gn)
            vals.append(float(monoloco_loss(fused_train_forward(model, x, seed=11), y).double()))
        model.w1.weight.copy_(w0)
    fd = (vals[0] - vals[1]) / (2 * eps)
    assert abs(fd - gn) <= 0.05 * gn, (fd, gn)


def test_monoloco_rejections_launch_nothing():
    """num_stage = 0, more than 16 outputs and train_step() are refused on the host before any launch; so are an output
    size out of range, a bad aux_block and the fused loss without an aux head at the C ABI."""
    import ctypes as C
    from monoloco_b200 import _lib as L_
    from monoloco_b200.network.architectures import MonolocoModel
    from monoloco_b200.train import train_step
    from monoloco_b200.train import fused
    x = torch.zeros(8, 34, device='cuda')
    n0 = _launches()
    with pytest.raises(ValueError, match='num_stage'):
        MonolocoModel(34, 2, 256, num_stage=0).cuda().train()(x)
    with pytest.raises(ValueError, match='num_stage'):
        MonolocoModel(34, 2, 128, num_stage=8).cuda().train()(x)
    with pytest.raises(ValueError, match='output_size'):
        MonolocoModel(34, 17, 256, num_stage=1).cuda().train()(x)
    model = MonolocoModel(34, 9, 256, num_stage=1).cuda().train()
    with pytest.raises(NotImplementedError, match='MonolocoModel'):
        train_step(model, x, torch.zeros(8, 10, device='cuda'), ('d',))
    assert _launches() == n0
    # the C entry points check the aux-less convention themselves
    ws = fused._workspace(model, 8, x.device)
    out = torch.empty(8, 9, device='cuda')
    lib = L_.lib()
    for field, val, fn, msg in (('output_size', 17, lib.mlb_train_forward, b'output_size'),
                                ('output_size', 0, lib.mlb_train_forward, b'output_size'),
                                ('aux_block', -2, lib.mlb_train_forward, b'aux_block'),
                                (None, None, lib.mlb_train_step, b'aux head')):
        a, blocks = fused._fill(model, ws, x, out)
        if field is not None:
            setattr(a, field, val)
        assert fn(ws.h, C.byref(a), blocks, fused._stream(x.device)) != 0
        assert msg in lib.mlb_last_error(), lib.mlb_last_error()
    assert _launches() == n0


def _rule_1e5(name, got, ref):
    """|a-b| <= 1e-5 max(|b|, column max) + 1e-6 (the forward tests' rule)."""
    colmax = np.abs(ref).max(axis=0, keepdims=True)
    tol = 1e-5 * np.maximum(np.abs(ref), colmax) + 1e-6
    assert (np.abs(got - ref) <= tol).all(), (name, float((np.abs(got - ref) / tol).max()))


@pytest.mark.parametrize('net,osz', [('monoloco', 2), ('monoloco_p', 9)])
def test_monoloco_train_end_to_end(net, osz, tmp_path):
    """MonolocoModel(34, osz, 256) trains 10 epochs on the KITTI-format fixture with FusedClipAdam and its loss goes
    down; the saved state_dict loads into Loco(net=...) and runs the pifpaf fixture (n_dropout 0 and 10) with finite
    outputs; the eval forward after the last step matches the torch oracle on the updated parameters."""
    from oracle import torch_port as T
    from monoloco_b200 import synthetic
    from monoloco_b200.network import Loco, preprocess_pifpaf
    from monoloco_b200.network.architectures import MonolocoModel
    from monoloco_b200.train import FusedClipAdam
    torch.manual_seed(0)
    sd = synthetic.make_state_dict('monoloco', 34, osz, 256, 3, 6)
    model = MonolocoModel(34, osz, 256, p_dropout=0.2, num_stage=3)
    model.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    model = model.cuda().train()
    kat = np.load(os.path.join(GOLDEN, 'kat_mono_train.npz'))
    x = torch.from_numpy(kat['X'].astype(np.float32)).cuda()
    y = torch.from_numpy(kat['Y'].astype(np.float32)).cuda()
    opt = FusedClipAdam(model.parameters(), lr=1e-3, max_norm=3.0)
    gen = torch.Generator().manual_seed(1)
    epoch_loss = []
    for _ in range(10):
        perm = torch.randperm(x.shape[0], generator=gen).cuda()
        tot, n = 0.0, 0
        for i in range(0, x.shape[0], 128):
            idx = perm[i:i + 128]
            opt.zero_grad()
            loss = monoloco_loss(model(x[idx]), y[idx])
            loss.backward()
            opt.step()
            tot, n = tot + float(loss) * len(idx), n + len(idx)
        epoch_loss.append(tot / n)
    assert all(np.isfinite(epoch_loss)) and epoch_loss[-1] < epoch_loss[0], epoch_loss
    # the eval forward on the trained parameters and running statistics
    model.eval()
    got = model(x).cpu().numpy()
    ref = T.model_forward(T.to_torch({k: v.detach().cpu() for k, v in model.state_dict().items()}), x.cpu(),
                          training=False).numpy()
    _rule_1e5(net, got, ref)
    path = str(tmp_path / ('%s.pkl' % net))
    torch.save(model.state_dict(), path)
    with open(os.path.join(GOLDEN, 'pifpaf_002282.json')) as fh:
        boxes, keypoints = preprocess_pifpaf(json.load(fh), im_size=(1238, 374))
    kk = synthetic.KITTI_K
    for n_dropout in (0, 10):
        loco = Loco(model=path, mode='mono', net=net, device=torch.device('cuda'), n_dropout=n_dropout, linear_size=256)
        assert isinstance(loco.model, MonolocoModel) and loco.model.output_size == osz
        dic = loco.forward(keypoints, kk)
        assert len(dic['d']) == len(keypoints)
        for k, v in dic.items():
            if isinstance(v, torch.Tensor):
                assert torch.isfinite(v).all(), (net, n_dropout, k)
