"""CPU: the torch-autograd oracle (oracle/torch_port.py) reproduces the live-reference training fixtures at padded and
two-part hidden widths (tests/golden/ref_train_wide_*.npz), and the fixtures were made from the weights
monoloco_b200.synthetic regenerates.  Pins the oracle the GPU tests compare the fused step with at these widths."""
import os

import numpy as np
import pytest

torch = pytest.importorskip('torch')
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
FIXTURES = ['ref_train_wide_mono_l2048_s3', 'ref_train_wide_stereo_l300_s2', 'ref_train_wide_mono_l1001_s1',
            'ref_train_wide_stereo_l1500_s1']
TASKS = {'mono': ('d', 'x', 'y', 'h', 'w', 'l', 'ori'), 'stereo': ('d', 'x', 'y', 'h', 'w', 'l', 'ori', 'aux')}


def _tight(name, got, ref, scale):
    err = np.abs(got - ref)
    assert (err <= 1e-4 * np.abs(ref) + 2e-5 * scale + 2e-7).all(), (name, float(err.max()), scale)


@pytest.mark.parametrize('name', FIXTURES)
def test_oracle_reproduces_train_wide_fixture(name):
    from oracle import torch_port as T
    from monoloco_b200 import synthetic
    f = np.load(os.path.join(GOLDEN, name + '.npz'))
    isz, osz, L, st, seed, B = [int(v) for v in f['cfg']]
    sd = synthetic.make_state_dict('loco', isz, osz, L, st, seed)
    checksum = float(sum(float(np.asarray(v, dtype=np.float64).sum()) for k, v in sorted(sd.items())))
    assert checksum == pytest.approx(float(f['checksum']), rel=1e-12, abs=1e-9)
    mode = 'stereo' if isz == 68 else 'mono'
    auto = bool(int(f['auto']))
    tsd = T.to_torch(sd, requires_grad=True)
    out = T.model_forward(tsd, torch.from_numpy(f['x']), training=True)
    assert np.allclose(out.detach().numpy(), f['out'], rtol=1e-5, atol=1e-5)
    ls = torch.from_numpy(f['log_sigmas']).requires_grad_(True) if auto else None
    loss, vals = T.multi_task_loss(out, torch.from_numpy(f['y']), TASKS[mode], log_sigmas=ls)
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
    assert n_grads == len([k for k in f.files if k.startswith(('grad.', 'gval.')) and k != 'grad.log_sigmas'])
    for k in f.files:
        if k.startswith('buf.') and 'num_batches' not in k:
            assert np.allclose(tsd[k[4:]].detach().numpy(), f[k], rtol=1e-5, atol=1e-6), k
