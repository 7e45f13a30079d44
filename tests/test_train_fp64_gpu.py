"""GPU: the fused training step against float64 at full batch, on problems conditioned by oracle/fp64_train.py so that no
ReLU sign and no |.| of the loss sits within rounding error of its threshold (DESIGN.md §2b).

Each case conditions the keep masks and the labels on the CPU, runs the kernel once, and holds every parameter gradient,
`log_sigmas.grad`, the loss values and the running statistics to LIMITS: the error against the float64 oracle in units
of the torch fp32 oracle's error against it.  Outputs are held to the forward's FFMA rule (fp64_ref.FFMA_RULE).

With MLB_FP64_TRAIN_RATIOS=<path> the measured ratios are written there as JSON (tools/fp64_train_ratios.py)."""
import functools
import json
import os

import numpy as np
import pytest

torch = pytest.importorskip('torch')
pytestmark = pytest.mark.gpu

from oracle import fp64_train as F64  # noqa: E402
from oracle import fp64_ref as R  # noqa: E402
from test_train_wide_gpu import _cmp_grad_statistical  # noqa: E402

P = 0.2
MONO = ('d', 'x', 'y', 'h', 'w', 'l', 'ori')
RATIOS = {}


@pytest.fixture(scope='module', autouse=True)
def _dump_ratios():
    yield
    path = os.environ.get('MLB_FP64_TRAIN_RATIOS')
    if path:
        with open(path, 'w') as f:
            json.dump(RATIOS, f, indent=1)


def _tasks(isz):
    return MONO + ('aux',) if isz == 68 else MONO


def _inputs(kind, isz, osz, L, st, B):
    from monoloco_b200 import synthetic
    sd = synthetic.make_state_dict(kind, isz, osz, L, st, 7)
    x = synthetic.make_inputs(B, isz, seed=3)
    y = synthetic.make_labels(B, stereo=isz == 68, seed=4)
    masks = (np.random.RandomState(5).uniform(size=(len(F64.sites(sd)), B, L)) >= P).astype(np.uint8)
    return sd, x, y, masks


@functools.lru_cache(maxsize=1)
def _problem(kind, isz, osz, L, st, B):
    """One conditioned problem per (topology, L, B, stages), shared by the entry points (cases of one problem are adjacent
    in every parametrize list below): masks and labels conditioned, no decision left within tau, and the float64 and
    fp32 forwards whose graphs serve every entry's backward."""
    sd, x, y, masks0 = _inputs(kind, isz, osz, L, st, B)
    masks, cleared = F64.condition(sd, x, masks0, P)
    assert sum(cleared) < 1e-3 * masks.size
    f64 = F64.Forward(sd, x, masks, P)
    f32 = F64.Forward(sd, x, masks, P, torch.float32)
    out64 = f64.out.detach().numpy()
    y = F64.condition_labels(out64, y, _tasks(isz)) if kind == 'loco' else y
    rep = F64.margin_report(sd, x, masks, P, out64, *((y, _tasks(isz)) if kind == 'loco' else ()))
    assert min(rep['relu']) > 1 and rep.get('loss', 2) > 1, rep
    return dict(sd=sd, x=x, y=y, masks=masks, f64=f64, f32=f32, cleared=sum(cleared) / masks.size)


def _model(kind, isz, osz, L, st, sd):
    from monoloco_b200.network.architectures import LocoModel, MonolocoModel
    m = (LocoModel if kind == 'loco' else MonolocoModel)(isz, osz, L, p_dropout=P, num_stage=st)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    return m.cuda().train()


def _g_out(B, cols):
    """Seeded output gradient of the drop-in entry, of the size a mean over the batch gives."""
    return (np.random.RandomState(6).standard_normal((B, cols)) / B).astype(np.float32)


def _log_sigmas(n):
    return np.linspace(-0.3, 0.4, n).astype(np.float32)


def _run_kernel(entry, model, pb, tasks, accumulate=False):
    """One fused step; returns what the kernel computed, as float64 numpy."""
    from monoloco_b200.train import train_step
    from monoloco_b200.train.fused import fused_train_forward
    x, dm = torch.from_numpy(pb['x']).cuda(), torch.from_numpy(pb['masks']).cuda()
    got = {}
    if entry == 'dropin':
        out = fused_train_forward(model, x, drop_mask=dm)
        out.backward(torch.from_numpy(_g_out(*out.shape)).cuda())
    else:
        ls = torch.nn.Parameter(torch.from_numpy(_log_sigmas(len(tasks))).cuda()) if entry == 'auto' else None
        loss, vals, out = train_step(model, x, torch.from_numpy(pb['y']).cuda(), tasks, log_sigmas=ls, drop_mask=dm,
                                     accumulate=accumulate)
        got['loss'] = np.array([float(loss)] + [float(v) for v in vals], dtype=np.float64)
        if ls is not None:
            got['g_log_sigmas'] = ls.grad.cpu().numpy().astype(np.float64)
    got['out'] = out.detach().cpu().numpy().astype(np.float64)
    got['grads'] = {n: p.grad.cpu().numpy().astype(np.float64) for n, p in model.named_parameters()}
    got['running'] = {n: b.cpu().numpy().astype(np.float64) for n, b in model.named_buffers() if 'running' in n}
    return got


def _oracles(entry, pb, tasks):
    kw = dict(g_out=_g_out(*pb['f64'].out.shape)) if entry == 'dropin' else dict(
        labels=pb['y'], tasks=tasks, log_sigmas=_log_sigmas(len(tasks)) if entry == 'auto' else None)
    return (F64.step64(pb['sd'], pb['x'], pb['masks'], P, fwd=pb['f64'], **kw),
            F64.step64(pb['sd'], pb['x'], pb['masks'], P, fwd=pb['f32'], **kw))


def _record(key, fam, l2, mx):
    old = RATIOS.setdefault(key, {}).get(fam, (0.0, 0.0))
    RATIOS[key][fam] = (max(old[0], l2), max(old[1], mx))


def _compare(key, sd, got, r64, r32):
    """Everything a step produced against float64 in units of the fp32 oracle's error; returns what is over a limit."""
    bad = {}
    ratios = F64.grad_ratios(sd, got['grads'], r64['grads'], r32['grads'])
    for n in r64['running']:
        ratios[n] = ('running stats',) + F64.grad_rule(got['running'][n], r64['running'][n], r32['running'][n])
    if 'loss' in got:
        ratios['loss'] = ('loss',) + F64.grad_rule(got['loss'], np.r_[r64['loss'], r64['vals']], np.r_[r32['loss'], r32['vals']])
    if 'g_log_sigmas' in got:
        ratios['log_sigmas'] = ('log_sigmas',) + F64.grad_rule(got['g_log_sigmas'], r64['g_log_sigmas'], r32['g_log_sigmas'])
    for n, (fam, l2, mx) in ratios.items():
        _record(key, fam, l2, mx)
    bad.update(F64.over_limit(ratios))
    mx, rms = R.fp64_rule(got['out'], r64['out'], r32['out'])
    _record(key, 'out', float(rms.max()), float(mx.max()))
    if mx.max() > R.FFMA_RULE[0] or rms.max() > R.FFMA_RULE[1]:
        bad['out'] = (mx.tolist(), rms.tolist())
    # absolute size of the error, for the record: the worst rel-L2 of any gradient with a scale
    worst = max((float(np.linalg.norm(got['grads'][n] - r64['grads'][n])) / float(np.linalg.norm(r64['grads'][n])), n)
                for n, r in ratios.items() if n in r64['grads'] and r[0] != 'zero')
    RATIOS[key]['worst rel-L2'] = max(RATIOS[key].get('worst rel-L2', (0.0, '')), worst)
    return bad


def _case(entry, kind, isz, osz, L, st, B):
    pb = _problem(kind, isz, osz, L, st, B)
    tasks = _tasks(isz)
    got = _run_kernel(entry, _model(kind, isz, osz, L, st, pb['sd']), pb, tasks)
    r64, r32 = _oracles(entry, pb, tasks)
    key = '%s %d->%d L=%d st=%d B=%d %s' % (kind, isz, osz, L, st, B, entry)
    RATIOS.setdefault(key, {})['cleared'] = pb['cleared']
    bad = _compare(key, pb['sd'], got, r64, r32)
    assert not bad, (key, bad)


# LocoModel: (input, output, width, stages, batch) paired with the entries run on it.  Widths 256, 300 (padded), 1024,
# 1500 (padded, two column parts) and 2048; batches 4096 (automatic rows-per-group), 4095 / 4097 (ragged last tile) and
# 6000 (two tiles per CTA); 3 stages (BASELINE) and 1; mono and stereo (the aux task).
LOCO = [(68, 10, 256, 1, 4097, ('step', 'auto')),
        (34, 9, 300, 3, 4095, ('step', 'dropin')),
        (34, 9, 1500, 1, 6000, ('step',)),
        (68, 10, 1024, 3, 6000, ('auto',)),
        (34, 9, 2048, 3, 4096, ('step', 'dropin')),
        (68, 10, 2048, 1, 4097, ('auto',)),
        (34, 9, 1024, 3, 4096, ('step', 'auto', 'dropin'))]


@pytest.mark.parametrize('isz,osz,L,st,B,entry', [c[:5] + (e,) for c in LOCO for e in c[5]])
def test_loco_step_vs_float64(isz, osz, L, st, B, entry):
    _case(entry, 'loco', isz, osz, L, st, B)


@pytest.mark.parametrize('tm', [8, 10, 12, 14, 16])
def test_rows_per_group_sweep_vs_float64(tm, monkeypatch):
    """Every rows-per-group at 4096 x 1024 (the automatic choice is one of them), same problem, same limits."""
    monkeypatch.setenv('MLB_TRAIN_ROWS_PER_GROUP', str(tm))
    pb = _problem('loco', 34, 9, 1024, 3, 4096)
    got = _run_kernel('step', _model('loco', 34, 9, 1024, 3, pb['sd']), pb, MONO)
    r64, r32 = _oracles('step', pb, MONO)
    bad = _compare('loco 34->9 L=1024 st=3 B=4096 step rows-per-group', pb['sd'], got, r64, r32)
    assert not bad, (tm, bad)


@pytest.mark.parametrize('osz,L,st,B', [(2, 256, 1, 4095), (9, 1024, 3, 4096), (9, 1500, 2, 4097), (9, 2048, 1, 6000)])
def test_monoloco_dropin_vs_float64(osz, L, st, B):
    """MonolocoModel trains through the drop-in: the legacy (34, 2, 256) net and the BASELINE (34, 9, 1024)."""
    _case('dropin', 'monoloco', 34, osz, L, st, B)


def test_unconditioned_step_keeps_the_statistical_rule():
    """What the full-size tests of test_train_gpu.py / test_train_wide_gpu.py mean, next to the rule above: on the
    unconditioned problem at 4096 x 1024 the fp32 and float64 oracles resolve some ReLU units differently, so their
    gradients are ~1e-3 apart and the fused step can only be held to rel-L2 <= 3e-3, cosine >= 1 - 1e-5."""
    from monoloco_b200.train import train_step
    sd, x, y, masks = _inputs('loco', 34, 9, 1024, 3, 4096)
    signs = []
    for dt in (torch.float32, torch.float64):
        with torch.no_grad():
            _, rec = F64.walk(F64.leaves(sd, dt), torch.as_tensor(x), masks, P)
        signs.append([r['pre'].numpy() > 0 for r in rec])
    flips = sum(int(((a != b) & (m != 0)).sum()) for a, b, m in zip(signs[0], signs[1], masks))
    assert flips > 0, 'no borderline unit in the unconditioned problem: the statistical rule is no longer needed here'
    model = _model('loco', 34, 9, 1024, 3, sd)
    train_step(model, torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), MONO, drop_mask=torch.from_numpy(masks).cuda())
    r32 = F64.step64(sd, x, masks, P, y, MONO, dtype=torch.float32)
    for n, p in model.named_parameters():
        _cmp_grad_statistical(n, p.grad.cpu().numpy(), r32['grads'][n])
    RATIOS['unconditioned 4096 x 1024'] = {'sign disagreements fp32 / float64': flips}


def test_accumulate_two_half_batches_vs_float64():
    """train_step(..., accumulate=True) over two conditioned micro-batches of different sizes: the gradients (and
    log_sigmas.grad) are the sum of the two float64 steps', the running statistics those of the two updates in turn."""
    from monoloco_b200.train import train_step
    from monoloco_b200 import synthetic
    L, st = 1024, 2
    sd = synthetic.make_state_dict('loco', 34, 9, L, st, 7)
    pbs = []
    for B, seed in ((2500, 3), (1596, 13)):
        pbs.append((B, synthetic.make_inputs(B, 34, seed=seed), synthetic.make_labels(B, seed=seed + 1),
                    (np.random.RandomState(seed + 2).uniform(size=(2 * st + 2, B, L)) >= P).astype(np.uint8)))
    model = _model('loco', 34, 9, L, st, sd)
    ls = torch.nn.Parameter(torch.from_numpy(_log_sigmas(len(MONO))).cuda())
    sums = [None, None]
    cur = [dict(sd), dict(sd)]    # the checkpoint each oracle sees: the running statistics move between the two steps
    g_ls = [0.0, 0.0]
    for B, x, y, masks in pbs:
        masks, _ = F64.condition(cur[0], x, masks, P)
        f64 = F64.Forward(cur[0], x, masks, P)
        y = F64.condition_labels(f64.out.detach().numpy(), y, MONO)
        rep = F64.margin_report(cur[0], x, masks, P, f64.out.detach().numpy(), y, MONO)
        assert min(rep['relu']) > 1 and rep['loss'] > 1, rep
        train_step(model, torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), MONO, log_sigmas=ls,
                   drop_mask=torch.from_numpy(masks).cuda(), accumulate=True)
        for i, dt in enumerate((torch.float64, torch.float32)):
            r = F64.step64(cur[i], x, masks, P, y, MONO, log_sigmas=_log_sigmas(len(MONO)), dtype=dt,
                           fwd=f64 if i == 0 else None)
            sums[i] = r['grads'] if sums[i] is None else {n: sums[i][n] + r['grads'][n] for n in sums[i]}
            g_ls[i] = g_ls[i] + r['g_log_sigmas']
            cur[i] = dict(cur[i], **r['running'])
    got = {'grads': {n: p.grad.cpu().numpy().astype(np.float64) for n, p in model.named_parameters()},
           'running': {n: b.cpu().numpy().astype(np.float64) for n, b in model.named_buffers() if 'running' in n}}
    ratios = F64.grad_ratios(sd, got['grads'], sums[0], sums[1])
    for n in got['running']:
        ratios[n] = ('running stats',) + F64.grad_rule(got['running'][n], cur[0][n], cur[1][n])
    ratios['log_sigmas'] = ('log_sigmas',) + F64.grad_rule(ls.grad.cpu().numpy(), g_ls[0], g_ls[1])
    for n, (fam, l2, mx) in ratios.items():
        _record('accumulate 2500 + 1596 L=1024 st=2', fam, l2, mx)
    bad = F64.over_limit(ratios)
    assert not bad, bad
