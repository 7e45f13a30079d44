"""CPU: the float64 training oracle and the conditioning of oracle/fp64_train.py, and what its rule notices.

* `step64` against a from-scratch numpy float64 forward + loss, and its gradients against central differences.
* `condition` is idempotent, clears < 1e-3 of the keep bits, and afterwards fp32 and float64 agree on every ReLU sign at
  the sizes where the unconditioned step flips units (DESIGN.md §9).
* The mutation table: defects of the kind a fused kernel can have at full batch, applied to the honest fp32 step, each
  measured in units of LIMITS and against the statistical rule the full-size tests use (DESIGN.md §2b)."""
import numpy as np
import pytest

torch = pytest.importorskip('torch')

from oracle import fp64_train as F64  # noqa: E402
from oracle import torch_port as T  # noqa: E402
from monoloco_b200 import synthetic  # noqa: E402
from test_train_wide_gpu import _cmp_grad_statistical  # noqa: E402

P = 0.2
MONO = ('d', 'x', 'y', 'h', 'w', 'l', 'ori')
STEREO = MONO + ('aux',)


def _problem(kind, isz, osz, L, st, B, seed=7, stereo=False):
    sd = synthetic.make_state_dict(kind, isz, osz, L, st, seed)
    x = synthetic.make_inputs(B, isz, seed=3)
    y = synthetic.make_labels(B, stereo=stereo, seed=4)
    masks = (np.random.RandomState(5).uniform(size=(len(F64.sites(sd)), B, L)) >= P).astype(np.uint8)
    return sd, x, y, masks


# ------------------------------------------------------------------------------------------------ step64 is right
def _np_step(sd, x, y, masks, tasks, log_sigmas=None):
    """Train-mode LocoModel forward + MultiTaskLoss in numpy float64, written from the definitions."""
    w = {k: np.asarray(v, dtype=np.float64) for k, v in sd.items()}
    it = iter(masks.astype(np.float64))
    run = {}

    def site(a, lin, bn):
        z = a @ w[lin + '.weight'].T + w[lin + '.bias']
        m, v = z.mean(0), ((z - z.mean(0)) ** 2).mean(0)
        run[bn + '.running_mean'] = 0.9 * w[bn + '.running_mean'] + 0.1 * m
        run[bn + '.running_var'] = 0.9 * w[bn + '.running_var'] + 0.1 * v * len(z) / (len(z) - 1)
        return np.maximum((z - m) / np.sqrt(v + 1e-5) * w[bn + '.weight'] + w[bn + '.bias'], 0) * next(it) / (1 - P)

    a = site(x.astype(np.float64), 'w1', 'batch_norm1')
    i = 0
    while 'linear_stages.%d.w1.weight' % i in w:
        pre = 'linear_stages.%d.' % i
        a = a + site(site(a, pre + 'w1', pre + 'batch_norm1'), pre + 'w2', pre + 'batch_norm2')
        i += 1
    a = a @ w['w2.weight'].T + w['w2.bias']
    aux = a @ w['w_aux.weight'].T + w['w_aux.bias']
    out = np.concatenate([site(a, 'w3', 'batch_norm3') @ w['w_fin.weight'].T + w['w_fin.bias'], aux], 1)
    y = y.astype(np.float64)
    vals = []
    for t in tasks:
        if t == 'd':
            v = (np.abs(1 - out[:, 2] / y[:, 3]) * np.exp(-out[:, 3]) + 0.01 + out[:, 3] + 2).mean()
        elif t == 'aux':
            o, g = out[:, 9], y[:, 10]
            v = (np.maximum(o, 0) - o * g + np.log1p(np.exp(-np.abs(o)))).mean()
        elif t == 'ori':
            v = np.abs(out[:, 7:9] - y[:, 7:9]).mean()
        else:
            c = {'x': 0, 'y': 1, 'h': 4, 'w': 5, 'l': 6}[t]
            v = np.abs(out[:, c] - y[:, c]).mean()
        vals.append(v)
    vals = np.array(vals)
    if log_sigmas is not None:
        vals = vals / (2 * np.exp(np.asarray(log_sigmas, dtype=np.float64)) ** 2)
        return out, vals.sum() + np.sum(log_sigmas), vals, run
    return out, vals.sum(), vals, run


@pytest.fixture(scope='module')
def small():
    sd, x, y, masks = _problem('loco', 68, 10, 48, 2, 64, stereo=True)
    masks, _ = F64.condition(sd, x, masks, P)
    ls = np.linspace(-0.3, 0.4, len(STEREO))
    out = F64.Forward(sd, x, masks, P).out.detach().numpy()
    y = F64.condition_labels(out, y, STEREO)
    return sd, x, y, masks, ls


def test_step64_equals_numpy_forward_and_loss(small):
    sd, x, y, masks, ls = small
    for log_sigmas in (None, ls):
        got = F64.step64(sd, x, masks, P, y, STEREO, log_sigmas=log_sigmas)
        out, loss, vals, run = _np_step(sd, x, y, masks, STEREO, log_sigmas)
        assert np.abs(got['out'] - out).max() <= 1e-12 * np.abs(out).max()
        assert abs(got['loss'] - loss) <= 1e-12 * abs(loss) and np.allclose(got['vals'], vals, rtol=1e-12, atol=0)
        for k, v in run.items():
            assert np.allclose(got['running'][k], v, rtol=1e-12, atol=1e-14), k
    # the walk that conditions is the same forward as the oracle that is differentiated
    with torch.no_grad():
        wout, _ = F64.walk(F64.leaves(sd), torch.as_tensor(x), masks, P)
    assert np.abs(wout.numpy() - got['out']).max() <= 1e-12 * np.abs(out).max()


def test_step64_gradients_match_central_differences(small):
    """Possible only because the conditioned problem is smooth: the probe moves no pre-ReLU value or residual by more
    than a small part of the margin conditioning left."""
    sd, x, y, masks, ls = small
    got = F64.step64(sd, x, masks, P, y, STEREO, log_sigmas=ls)
    rep = F64.margin_report(sd, x, masks, P, got['out'], y, STEREO)
    assert min(rep['relu']) > 1 and rep['loss'] > 1
    h = 1e-6   # a parameter step of 1e-6 moves a pre-ReLU value of RMS ~1 by ~1e-6 << tau = 1e-4
    rng = np.random.RandomState(0)

    def loss_at(name, idx, d):
        sd2 = dict(sd)
        v = np.array(sd[name], dtype=np.float64)
        v.reshape(-1)[idx] += d
        sd2[name] = v
        tsd = F64.leaves(sd2)
        out = T.model_forward(tsd, torch.as_tensor(x).double(), training=True, p_dropout=P,
                              masks=[torch.from_numpy(m) for m in masks])
        return float(T.multi_task_loss(out, torch.as_tensor(y).double(), STEREO, log_sigmas=torch.as_tensor(ls))[0])

    for name, g in got['grads'].items():
        scale = max(float(np.abs(g).max()), 1e-9)
        for idx in rng.choice(g.size, size=min(3, g.size), replace=False):
            fd = (loss_at(name, idx, h) - loss_at(name, idx, -h)) / (2 * h)
            assert abs(fd - g.reshape(-1)[idx]) <= 1e-6 * scale + 1e-9, (name, idx, fd, g.reshape(-1)[idx])
    # log_sigmas: d/d ls_t [v_t / (2 exp(2 ls_t)) + ls_t]
    for t in range(len(ls)):
        e = np.zeros_like(ls)
        e[t] = h
        fd = (F64.step64(sd, x, masks, P, y, STEREO, log_sigmas=ls + e)['loss'] -
              F64.step64(sd, x, masks, P, y, STEREO, log_sigmas=ls - e)['loss']) / (2 * h)
        assert abs(fd - got['g_log_sigmas'][t]) <= 1e-8


def test_condition_labels_moves_only_borderline_labels():
    rng = np.random.RandomState(1)
    y = synthetic.make_labels(64, stereo=True, seed=2)
    out = rng.standard_normal((64, 10))
    out[0, 0] = y[0, 0] + 3e-5          # x, within tau above
    out[1, 2] = y[1, 3] * (1 - 5e-5)    # d, within tau below
    out[2, 8] = y[2, 8]                 # ori cos, on the kink
    y2 = F64.condition_labels(out, y, STEREO)
    changed = np.argwhere(y2 != y)
    assert sorted(map(tuple, changed)) == [(0, 0), (1, 3), (2, 8)]
    assert min(float(np.abs(r).min()) for _, _, r in F64._residuals(out, y2, STEREO)) > F64.TAU_LABEL
    assert np.array_equal(F64.condition_labels(out, y2, STEREO), y2)


# ------------------------------------------------------------------------------------------------ conditioning
def _signs(sd, x, masks, dtype):
    with torch.no_grad():
        _, rec = F64.walk(F64.leaves(sd, dtype), torch.as_tensor(x), masks, P)
    return [r['pre'].numpy() > 0 for r in rec]


@pytest.fixture(scope='module')
def full():
    """LocoModel(34, 9, 1024), 3 stages, batch 4096: BASELINE's training size."""
    sd, x, y, masks0 = _problem('loco', 34, 9, 1024, 3, 4096)
    masks, cleared = F64.condition(sd, x, masks0, P)
    return sd, x, y, masks0, masks, cleared


def _check_conditioning(sd, x, masks0, masks, cleared):
    assert 0 < sum(cleared) < 1e-3 * masks0.size and (masks <= masks0).all()
    assert int(masks0.sum()) - int(masks.sum()) == sum(cleared)
    again, cleared2 = F64.condition(sd, x, masks, P)
    assert sum(cleared2) == 0 and np.array_equal(again, masks)
    assert min(F64.margin_report(sd, x, masks, P)['relu']) > 1
    flips = flips0 = 0
    for m, s32, s64 in zip(masks, _signs(sd, x, masks, torch.float32), _signs(sd, x, masks, torch.float64)):
        flips += int(((s32 != s64) & (m != 0)).sum())
    for m0, s32, s64 in zip(masks0, _signs(sd, x, masks0, torch.float32), _signs(sd, x, masks0, torch.float64)):
        flips0 += int(((s32 != s64) & (m0 != 0)).sum())
    return flips, flips0


def test_condition_full_size_no_sign_disagreement(full):
    sd, x, _, masks0, masks, cleared = full
    flips, flips0 = _check_conditioning(sd, x, masks0, masks, cleared)
    print('L=1024 B=4096: cleared %d of %d keep bits (%.1e); kept units whose ReLU sign differs between fp32 and float64: '
          '%d unconditioned, %d conditioned' % (sum(cleared), masks0.size, sum(cleared) / masks0.size, flips0, flips))
    assert flips == 0 and flips0 > 0


def test_condition_padded_width_no_sign_disagreement():
    """L=1500, B=300: the case DESIGN.md §9 records as flipping one unit in the fp32 oracle."""
    sd, x, _, masks0 = _problem('loco', 34, 9, 1500, 1, 300)
    masks, cleared = F64.condition(sd, x, masks0, P)
    flips, flips0 = _check_conditioning(sd, x, masks0, masks, cleared)
    print('L=1500 B=300: cleared %d, sign differences %d unconditioned, %d conditioned' % (sum(cleared), flips0, flips))
    assert flips == 0


def test_family_of_every_parameter():
    sd = synthetic.make_state_dict('loco', 34, 9, 64, 1, 0)
    fam = {n: F64.family(n, sd) for n in sd if 'running' not in n and 'num_batches' not in n}
    assert fam['w1.weight'] == 'dW input' and fam['w1.bias'] == 'zero' and fam['w3.bias'] == 'zero'
    assert fam['w2.bias'] == 'biases' and fam['w2.weight'] == 'dW hidden' and fam['w_aux.bias'] == 'head biases' and fam['w_fin.weight'] == 'heads'
    assert fam['linear_stages.0.w2.bias'] == 'zero' and fam['linear_stages.0.batch_norm2.bias'] == 'gamma/beta'
    sd = synthetic.make_state_dict('monoloco', 34, 2, 64, 1, 0)
    assert F64.family('w2.bias', sd) == 'head biases' and F64.family('w2.weight', sd) == 'heads' and len(F64.sites(sd)) == 3


# ------------------------------------------------------------------------------------------------ mutation table
class _WrongHalf(torch.autograd.Function):
    """Linear whose dX, for `rows`, multiplies the upper half of dZ's columns with the lower half's weights."""

    @staticmethod
    def forward(ctx, a, W, b, rows):
        ctx.save_for_backward(a, W)
        ctx.rows = rows
        return torch.nn.functional.linear(a, W, b)

    @staticmethod
    def backward(ctx, g):
        a, W = ctx.saved_tensors
        da, h, r = g @ W, W.shape[0] // 2, ctx.rows
        da[r] = g[r, :h] @ W[:h] + g[r, h:] @ W[:h]
        return da, g.t() @ a, g.sum(0), None


def _walk_step(sd, x, y, masks, tap=None):
    """The honest fp32 step through `walk` (so that a defect can be stated as a tap): grads, out, loss, rec."""
    tsd = F64.leaves(sd, torch.float32)
    out, rec = F64.walk(tsd, torch.as_tensor(x), masks, P, tap=tap)
    loss, _ = T.multi_task_loss(out, torch.as_tensor(y), MONO)
    loss.backward()
    grads = {k: v.grad.numpy().astype(np.float64) for k, v in tsd.items() if v.requires_grad}
    return grads, out.detach().numpy(), float(loss.detach()), rec


def _passes_statistical(sd, grads, ref):
    """Today's full-size rule (rel-L2 <= 3e-3, cosine >= 1 - 1e-5 against the fp32 oracle) on every gradient."""
    try:
        for n in ref:
            _cmp_grad_statistical(n, grads[n], ref[n])
    except AssertionError:
        return False
    return True


def _worst(sd, grads, r64, r32):
    """Worst excess over LIMITS of any gradient: max over tensors and both ratios of ratio / limit."""
    rat = F64.grad_ratios(sd, grads, r64, r32)
    n = max(rat, key=lambda k: max(rat[k][1] / F64.LIMITS[rat[k][0]][0], rat[k][2] / F64.LIMITS[rat[k][0]][1]))
    fam, l2, mx = rat[n]
    return n, max(l2 / F64.LIMITS[fam][0], mx / F64.LIMITS[fam][1])


def test_mutation_table(full):
    """Each defect applied to the honest fp32 step at batch 4096 must exceed the float64 rule's limit by >= 10x; the table
    printed (and kept in DESIGN.md §2b) also says which of them today's statistical rule accepts."""
    sd, x, y, _, masks, _ = full
    B = len(x)
    f64 = F64.Forward(sd, x, masks, P)
    y = F64.condition_labels(f64.out.detach().numpy(), y, MONO)
    r64 = F64.step64(sd, x, masks, P, y, MONO, fwd=f64)
    r32 = F64.step64(sd, x, masks, P, y, MONO, dtype=torch.float32)
    g32, out32, _, rec = _walk_step(sd, x, y, masks)
    # the walk under autograd is the honest step: same rule, no mutation -> within the limits
    assert not F64.over_limit(F64.grad_ratios(sd, g32, r64['grads'], r32['grads']))
    rows = slice(1000, 1008)     # one 8-row group
    tile = slice(2048, 2064)     # one 16-row tile
    table = []

    def row(label, grads, ref32=None):
        name, excess = _worst(sd, grads, r64['grads'], r32['grads'])
        table.append((label, name, excess, _passes_statistical(sd, grads, ref32 or r32['grads'])))

    # 1. one 8-row group's contribution missing from one dW
    s = 3
    lin = F64.sites(sd)[s][0]
    g = dict(g32)
    g[lin + '.weight'] = g32[lin + '.weight'] - (rec[s]['z'].grad[rows].t() @ rec[s]['a_in'][rows]).detach().numpy()
    row('dW: one 8-row group dropped', g)
    # 2. one group counted twice in one BatchNorm's sums (1/B unchanged)
    def moments(site, z):
        if site != s:
            return z.mean(0), z.var(0, unbiased=False)
        m = (z.sum(0) + z[rows].sum(0)) / B
        return m, (z.pow(2).sum(0) + z[rows].pow(2).sum(0)) / B - m * m
    g, _, _, _ = _walk_step(sd, x, y, masks, tap={'moments': moments})
    row('BatchNorm sums: one 8-row group twice', g)
    # 4. dgamma of one block without the dropout scale on one tile
    bn = F64.sites(sd)[s][1]
    zhat = ((rec[s]['pre'] - torch.as_tensor(sd[bn + '.bias'])) / torch.as_tensor(sd[bn + '.weight'])).detach()
    g = dict(g32)
    g[bn + '.weight'] = g32[bn + '.weight'] - P * (rec[s]['pre'].grad[tile] * zhat[tile]).sum(0).numpy()
    row('dgamma: dropout scale missing on one tile', g)
    # 5. the residual skip's gradient missing for one row tile
    def skip(stage, a):
        if stage != 1:
            return a
        keep = torch.ones(B, 1)
        keep[tile] = 0
        return a * keep + (a * (1 - keep)).detach()
    g, _, _, _ = _walk_step(sd, x, y, masks, tap={'skip': skip})
    row('skip gradient missing on one tile', g)
    # 3. running variance from the biased batch variance
    k = bn + '.running_var'
    biased = 0.9 * np.asarray(sd[k], dtype=np.float64) + 0.1 * rec[s]['var'].detach().numpy()
    l2, mx = F64.grad_rule(biased, r64['running'][k], r32['running'][k])
    lim = F64.LIMITS['running stats']
    table.append(('running_var: biased variance', k, max(l2 / lim[0], mx / lim[1]),
                  bool(np.allclose(biased, r32['running'][k], rtol=2e-5, atol=2e-6))))
    # 6. at 2048 (two column parts): one K half of dX against the other part's weights on one tile
    sd2, x2, y2, m2 = _problem('loco', 34, 9, 2048, 1, 4096)
    m2, _ = F64.condition(sd2, x2, m2, P)
    f2 = F64.Forward(sd2, x2, m2, P)
    y2 = F64.condition_labels(f2.out.detach().numpy(), y2, MONO)
    q64 = F64.step64(sd2, x2, m2, P, y2, MONO, fwd=f2)['grads']
    q32 = F64.step64(sd2, x2, m2, P, y2, MONO, dtype=torch.float32)['grads']
    g, _, _, _ = _walk_step(sd2, x2, y2, m2, tap={
        'linear': lambda site, a, W, b: _WrongHalf.apply(a, W, b, tile) if site == 2 else torch.nn.functional.linear(a, W, b)})
    name, excess = _worst(sd2, g, q64, q32)
    table.append(('dX at 2048: one K half against the wrong part on one tile', name, excess, _passes_statistical(sd2, g, q32)))

    print('\n%-60s %-36s %12s  %s' % ('defect (LocoModel 34->9, batch 4096, width 1024 / 2048)', 'worst tensor',
                                      'x the limit', 'statistical rule (3e-3, cos 1-1e-5)'))
    for label, name, excess, ok in table:
        print('%-60s %-36s %12.1f  %s' % (label, name, excess, 'accepts' if ok else 'rejects'))
    for label, name, excess, _ in table:
        assert excess >= 10, (label, name, excess)
