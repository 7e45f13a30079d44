"""CPU: MonolocoModel training, host side.  The torch-autograd oracle (oracle/torch_port.py) reproduces the live-reference
MonolocoModel training fixtures (tests/golden/ref_train_monoloco_*.npz: outputs, loss, every gradient, the buffers
after the step), and the fused step's block list and head mapping are checked for both network classes."""
import os

import numpy as np
import pytest

torch = pytest.importorskip('torch')
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
# legacy monoloco (2 outputs), monoloco_p (9), the BASELINE configuration MonolocoModel(34, 9, 1024), a padded width and
# a width run in two column parts (tools/gen_train_monoloco_golden.py)
FIXTURES = ['ref_train_monoloco_o2_l256_s3', 'ref_train_monoloco_o9_l256_s3', 'ref_train_monoloco_o9_l1024_s3',
            'ref_train_monoloco_o9_l300_s2', 'ref_train_monoloco_o9_l2048_s2']


def monoloco_loss(out, y):
    """The fixtures' loss: legacy monoloco, LaplacianLoss on (d, log b) against label column 3; monoloco_p,
    LaplacianLoss on 'zb' = out[:, 2:4] (process.py:340) against column 2 plus L1 on out[:, 4:9] (losses.py:104-142)."""
    def laplace(mu_si, xx):
        mu, si = mu_si[:, 0:1], mu_si[:, 1:2]
        return (torch.abs(1 - mu / xx) * torch.exp(-si) + 0.01 + si + 2).mean()
    if out.shape[1] == 2:
        return laplace(out[:, 0:2], y[:, 3:4])
    return laplace(out[:, 2:4], y[:, 2:3]) + torch.nn.functional.l1_loss(out[:, 4:9], y[:, 4:9])


def load_fixture(name):
    f = np.load(os.path.join(GOLDEN, name + '.npz'))
    isz, osz, L, st, seed, B = [int(v) for v in f['cfg']]
    return f, isz, osz, L, st, seed, B


def _tight(name, got, ref, scale):
    err = np.abs(got - ref)
    assert (err <= 1e-4 * np.abs(ref) + 2e-5 * scale + 2e-7).all(), (name, float(err.max()), scale)


@pytest.mark.parametrize('name', FIXTURES)
def test_oracle_reproduces_train_monoloco_fixture(name):
    from oracle import torch_port as T
    from monoloco_b200 import synthetic
    f, isz, osz, L, st, seed, B = load_fixture(name)
    assert B * L < (1 << 20)
    sd = synthetic.make_state_dict('monoloco', isz, osz, L, st, seed)
    checksum = float(sum(float(np.asarray(v, dtype=np.float64).sum()) for k, v in sorted(sd.items())))
    assert checksum == pytest.approx(float(f['checksum']), rel=1e-12, abs=1e-9)
    tsd = T.to_torch(sd, requires_grad=True)
    out = T.model_forward(tsd, torch.from_numpy(f['x']), training=True)
    assert out.shape == (B, osz)
    assert np.allclose(out.detach().numpy(), f['out'], rtol=1e-5, atol=1e-5)
    loss = monoloco_loss(out, torch.from_numpy(f['y']))
    assert abs(float(loss) - float(f['loss'])) <= 3e-6 * abs(float(f['loss']))
    loss.backward()
    n_grads = 0
    for k, t in tsd.items():
        if t.grad is None:
            continue
        g = t.grad.numpy().astype(np.float64)
        if 'grad.' + k in f.files:
            ref = f['grad.' + k].astype(np.float64)
            _tight(k, g, ref, max(float(np.abs(ref).max()), 1e-12))
        else:
            ref = f['gval.' + k].astype(np.float64)
            assert tuple(g.shape) == tuple(f['gshape.' + k]), k
            _tight(k, g.reshape(-1)[f['gidx.' + k]], ref, max(float(np.abs(ref).max()), 1e-12))
            nrm = float(f['gnorm.' + k])
            assert abs(float(np.linalg.norm(g)) - nrm) <= 1e-5 * nrm, k
        n_grads += 1
    assert n_grads == len([k for k in f.files if k.startswith(('grad.', 'gval.'))]) == 4 + 8 * st + 2
    for k in f.files:
        if k.startswith('buf.') and 'num_batches' not in k:
            assert np.allclose(tsd[k[4:]].detach().numpy(), f[k], rtol=1e-5, atol=1e-6), k


def test_block_list_and_heads_per_class():
    """The block description the fused step hands the kernel: LocoModel ends with the BatchNorm-free w2 (aux block) and
    w3; MonolocoModel ends with its last stage, whose w2 block carries the residual, and w2 is its final head."""
    from monoloco_b200.network.architectures import LocoModel, MonolocoModel
    from monoloco_b200.train.fused import _blocks_of, _heads_of
    loco = LocoModel(34, 9, 256, num_stage=2)
    assert _blocks_of(loco) == [('w1', 'batch_norm1', -1),
                                ('linear_stages.0.w1', 'linear_stages.0.batch_norm1', -1),
                                ('linear_stages.0.w2', 'linear_stages.0.batch_norm2', 0),
                                ('linear_stages.1.w1', 'linear_stages.1.batch_norm1', -1),
                                ('linear_stages.1.w2', 'linear_stages.1.batch_norm2', 2),
                                ('w2', None, -1), ('w3', 'batch_norm3', -1)]
    assert _heads_of(loco) == (34, 'w_aux', 'w_fin', 9)
    for st in (1, 3, 7):
        for osz in (2, 9):
            m = MonolocoModel(34, osz, 300, num_stage=st)
            blocks = _blocks_of(m)
            assert len(blocks) == 1 + 2 * st
            assert blocks[0] == ('w1', 'batch_norm1', -1)
            for i in range(st):
                pre = 'linear_stages.%d.' % i
                assert blocks[1 + 2 * i] == (pre + 'w1', pre + 'batch_norm1', -1)
                assert blocks[2 + 2 * i] == (pre + 'w2', pre + 'batch_norm2', 2 * i)
            assert blocks[-1][2] >= 0                       # the last block carries a residual
            assert all(bn is not None for _, bn, _ in blocks)  # one dropout site per block
            assert _heads_of(m) == (34, None, 'w2', osz)
            # every Linear and BatchNorm of the model appears once, the head aside
            names = {n.rsplit('.', 1)[0] for n, _ in m.named_parameters()}
            assert names == {x for b in blocks for x in b[:2]} | {'w2'}
