"""
Float64 parity of the fused training step on a problem without borderline decisions  --  TEST INFRASTRUCTURE ONLY.

At full batch any two correct evaluations of a training step differ by far more than rounding error, because a few of
the ~3e7 ReLU signs (and of the |.| signs in the L1 / Laplace losses) sit within rounding error of their threshold and
resolve differently in different summation orders (DESIGN.md §9).  This module removes those decisions with inputs the
kernels already take, instead of widening the tolerance:

  * `condition` walks the network forward in float64 (train-mode BatchNorm, the caller's keep masks applied) and clears
    the keep bit of every (row, unit) whose pre-ReLU value is within `tau` of zero.  A dropped unit contributes exactly 0
    forward and passes exactly 0 back whichever way its ReLU resolved.
  * `condition_labels` moves every label whose residual is within `tau` of a kink of the loss away from it.

On the conditioned problem the gradient is a smooth function of everything fp32 rounds, so the fused kernel, the torch
fp32 autograd oracle (`torch_port`, the "honest fp32" implementation) and the same oracle in float64 (taken as exact) can
be compared in units of the honest implementation's own error: `grad_rule`, `LIMITS`.

The step itself (`Forward`, `loss_grad`, `step64`) is `torch_port` run in float64 under torch autograd; `walk` is a second
statement of the forward only, needed to see the pre-ReLU values (tests/test_fp64_train_cpu.py holds the two together).
`monoloco_b200/` never imports this module.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import torch_port as T

BN_EPS = 1e-5
MOMENTUM = 0.1
TAU = 1e-4          # ReLU sites: a unit is borderline when |pre-ReLU| <= TAU * RMS of the site's pre-ReLU values
TAU_LABEL = 1e-4    # loss kinks: |out - y| <= TAU_LABEL (L1 tasks), |mu - y| <= TAU_LABEL |y| (Laplace d)
FLOOR = 2.0 ** -24

# Allowed (rel-L2, max-abs) ratios of `grad_rule` per tensor family: the fused step's error against float64 in units of
# the torch fp32 oracle's error against float64 on the same conditioned problem.  Set at 1.5x the worst value of
# two runs of tests/test_train_fp64_gpu.py on one H100 80GB HBM3 (700 W power limit); a few of the kernel's sums are float
# atomics, so the values move a little from run to run (DESIGN.md §5, §2b).  Worst measured (rel-L2, max) and where:
#   dW hidden      3.06, 4.74   LocoModel w2.weight, width 300 (padded), batch 4095, 3 stages, train_step
#   dW input       2.10, 2.32   width 2048, batch 4096, 3 stages
#   heads          3.57, 4.59   the family's limit was set with the head biases still in it (w_fin.bias, 8 values, width 300);
#                               the head weights alone stayed below 4.0
#   head biases    5.50, 5.50   w_aux.bias (one value), stereo, width 256, batch 4097, AutoTune: 1.7 in the first run, 5.5 in
#                               the second.  Tensors of 1 to 10 values, each a sum over the batch: the ratio is one error
#                               over another (or over the 2^-24 floor), and the worst of two runs is a poor estimate of
#                               its spread, so this family alone is held to 2x the worst, not 1.5x
#   biases         1.64, 1.91   LocoModel w2.bias, width 2048 drop-in / width 300
#   gamma/beta     2.19, 2.68   width 2048, batch 4096, 3 stages
#   running stats  1.01, 1.19   accumulate case (two steps); a single step 0.76, 1.06
#   zero           0.00         the Linear biases in front of a BatchNorm: at most 1e-9, against the floor of 2e-7
#   loss           0.89, 1.01   loss and task values; log_sigmas 1.09, 1.00.  A handful of fp32 scalars: their error is
#                               the last bit of the fp32 result, where 1.5x the worst of one run is less than one ulp, so
#                               both are held to the forward's FFMA rule (fp64_ref.FFMA_RULE) instead
# In absolute terms the fused step's worst gradient was 9.0e-6 rel-L2 from float64 (stereo, width 2048, batch 4097,
# AutoTune, w2.bias: the fp32 oracle is as far there), the worst of any other case 7.2e-6; outputs by fp64_ref.fp64_rule: max 2.67, RMS 2.18.
LIMITS = {
    'dW hidden': (4.6, 7.1),
    'dW input': (3.2, 3.5),
    'heads': (5.4, 6.9),
    'head biases': (11.0, 11.0),
    'biases': (2.5, 2.9),
    'gamma/beta': (3.3, 4.1),
    'running stats': (1.6, 1.8),
    'zero': (1.0, 1.0),
    'loss': (4.0, 4.0),
    'log_sigmas': (4.0, 4.0),
}


# ------------------------------------------------------------------------------------------------ topology
def sites(sd):
    """[(Linear, BatchNorm)] of every BatchNorm -> ReLU -> dropout site in forward order: 2 num_stage + 2 for LocoModel
    (w_fin in sd), 2 num_stage + 1 for MonolocoModel.  LocoModel.w2 has no site."""
    out = [('w1', 'batch_norm1')]
    i = 0
    while 'linear_stages.%d.w1.weight' % i in sd:
        out += [('linear_stages.%d.w%d' % (i, j), 'linear_stages.%d.batch_norm%d' % (i, j)) for j in (1, 2)]
        i += 1
    if 'w_fin.weight' in sd:
        out.append(('w3', 'batch_norm3'))
    return out


def family(name, sd):
    """Tensor family of a parameter for LIMITS.  'zero': Linear biases in front of a BatchNorm, whose true gradient is
    identically zero (the BatchNorm removes the column mean)."""
    lin, kind = name.rsplit('.', 1)
    if 'batch_norm' in lin:
        return 'gamma/beta'
    if kind == 'bias' and any(lin == s[0] for s in sites(sd)):
        return 'zero'
    if lin in ('w_fin', 'w_aux') or (lin == 'w2' and 'w_fin.weight' not in sd):
        return 'heads' if kind == 'weight' else 'head biases'
    if kind == 'bias':
        return 'biases'
    return 'dW input' if lin == 'w1' else 'dW hidden'


def leaves(sd, dtype=torch.float64):
    """The checkpoint as torch tensors of `dtype`; parameters are autograd leaves, running statistics are copies."""
    return {k: (v.to(dtype).detach().requires_grad_(v.requires_grad) if v.is_floating_point() else v)
            for k, v in T.to_torch(sd, requires_grad=True).items()}


# ------------------------------------------------------------------------------------------------ the sequential walk
def walk(tsd, x, masks, p, tau=None, tap=None):
    """Train-mode forward of `torch_port.model_forward`, site by site, in the dtype of `tsd` (from `leaves`).
    masks: uint8 [sites][B][L] keep masks.  With tau, the keep bit of every unit with |pre-ReLU| <= tau * RMS(pre-ReLU of
    the site) is cleared in place before the walk continues, so later sites see the activations the kernel will have.
    tap: optional {'linear': f(site, a, W, b) -> z, 'moments': f(site, z) -> (mean, biased var), 'skip': f(stage, y) -> y}
    replacing one step of the walk (the mutation tests of tests/test_fp64_train_cpu.py state defects with it).
    Returns (out, rec): rec[site] = dict(a_in, z, pre, mean, var, tau, cleared, margin), margin = min |pre| / tau over the
    units the site keeps."""
    tap = tap or {}
    rec = []
    dt = tsd['w1.weight'].dtype

    def site(y, s):
        lin, bn = sites(tsd)[s]
        W, b = tsd[lin + '.weight'], tsd[lin + '.bias']
        z = tap['linear'](s, y, W, b) if 'linear' in tap else F.linear(y, W, b)
        mean, var = tap['moments'](s, z) if 'moments' in tap else (z.mean(0), z.var(0, unbiased=False))
        pre = (z - mean) / torch.sqrt(var + BN_EPS) * tsd[bn + '.weight'] + tsd[bn + '.bias']
        with torch.no_grad():
            t = (tau if tau is not None else TAU) * float(pre.double().pow(2).mean().sqrt())
            keep = torch.from_numpy(masks[s])
            cleared = 0
            if tau is not None:
                near = (pre.abs() <= t) & (keep != 0)
                cleared = int(near.sum())
                keep[near] = 0          # shares memory with masks[s]
            kept = pre.abs()[keep != 0]
            margin = float(kept.min()) / t if kept.numel() else float('inf')
        for v in (z, pre):
            if v.requires_grad:
                v.retain_grad()
        rec.append(dict(a_in=y, z=z, pre=pre, mean=mean, var=var, tau=t, cleared=cleared, margin=margin))
        return F.relu(pre) * keep.to(dt) / (1.0 - p)

    y = site(x.to(dt), 0)
    s, i = 1, 0
    while 'linear_stages.%d.w1.weight' % i in tsd:
        z = site(site(y, s), s + 1)
        y = (tap['skip'](i, y) if 'skip' in tap else y) + z
        s, i = s + 2, i + 1
    if 'w_fin.weight' in tsd:
        y = F.linear(y, tsd['w2.weight'], tsd['w2.bias'])
        aux = F.linear(y, tsd['w_aux.weight'], tsd['w_aux.bias'])
        y = F.linear(site(y, s), tsd['w_fin.weight'], tsd['w_fin.bias'])
        return torch.cat((y, aux), dim=1), rec
    return F.linear(y, tsd['w2.weight'], tsd['w2.bias']), rec


def condition(sd, x, masks, p, tau=TAU):
    """Keep masks [sites][B][L] with every borderline ReLU unit dropped (one float64 pass, deterministic), and the number
    of bits cleared per site.  The input masks are not modified."""
    masks = np.array(masks, dtype=np.uint8, copy=True)
    assert masks.shape[0] == len(sites(sd)) and p > 0, (masks.shape, p)
    with torch.no_grad():
        _, rec = walk(leaves(sd), torch.as_tensor(x), masks, p, tau=tau)
    return masks, [r['cleared'] for r in rec]


# label column of each task's kink (torch_port.multi_task_loss): output column(s) -> label column(s); 'aux' is smooth
_KINKS = {'x': (0, 0), 'y': (1, 1), 'd': (2, 3), 'h': (4, 4), 'w': (5, 5), 'l': (6, 6), 'ori': ((7, 8), (7, 8))}


def _residuals(out64, labels, tasks):
    """[(label column, relative?, residual in the units tau is in)] of every loss kink: out - y for the L1 tasks,
    (mu - y) / |y| for the Laplace d task (|1 - mu / y| has its kink at y = mu)."""
    out64, labels = np.asarray(out64, dtype=np.float64), np.asarray(labels, dtype=np.float64)
    res = []
    for t in tasks:
        oc, lc = _KINKS.get(t, ((), ()))
        for o, c in zip(np.atleast_1d(oc), np.atleast_1d(lc)):
            r = out64[:, o] - labels[:, c]
            res.append((int(c), t == 'd', r / np.abs(labels[:, c]) if t == 'd' else r))
    return res


def condition_labels(out64, labels, tasks, tau=TAU_LABEL):
    """Labels (fp32) with every one whose residual is within tau of a kink moved 2 tau away from the output."""
    new = np.array(labels, dtype=np.float32, copy=True)
    for c, rel, r in _residuals(out64, labels, tasks):
        step = 2.0 * tau * (np.abs(new[:, c].astype(np.float64)) if rel else 1.0)
        moved = new[:, c] - np.where(r >= 0, 1.0, -1.0) * step
        new[:, c] = np.where(np.abs(r) <= tau, moved, new[:, c]).astype(np.float32)
    return new


def margin_report(sd, x, masks, p, out64=None, labels=None, tasks=None, tau=TAU, tau_label=TAU_LABEL):
    """After conditioning: per ReLU site the smallest |pre-ReLU| among kept units in units of the site's tau, and (with
    labels) the smallest loss residual in units of tau_label.  Every value must exceed 1."""
    with torch.no_grad():
        _, rec = walk(leaves(sd), torch.as_tensor(x), np.asarray(masks), p)
    rep = {'relu': [r['margin'] * TAU / tau for r in rec]}
    if labels is not None:
        rep['loss'] = min(float(np.abs(r).min()) for _, _, r in _residuals(out64, labels, tasks)) / tau_label
    return rep


# ------------------------------------------------------------------------------------------------ the step
class Forward:
    """`torch_port.model_forward` in train mode under autograd in `dtype`: outputs, updated running statistics (momentum
    0.1, unbiased variance), and the parameter gradients of any number of output gradients from the one forward."""

    def __init__(self, sd, x, masks, p, dtype=torch.float64):
        self.tsd = leaves(sd, dtype)
        self.out = T.model_forward(self.tsd, torch.as_tensor(x).to(dtype), training=True, p_dropout=p,
                                   masks=[torch.from_numpy(m) for m in np.asarray(masks)])
        self.names = [k for k, v in self.tsd.items() if v.requires_grad]
        self.running = {k: v.numpy().astype(np.float64) for k, v in self.tsd.items() if 'running' in k}

    def grads(self, g_out):
        g = torch.autograd.grad(self.out, [self.tsd[k] for k in self.names], torch.as_tensor(g_out).to(self.out.dtype),
                                retain_graph=True)
        return {k: v.numpy().astype(np.float64) for k, v in zip(self.names, g)}


def loss_grad(out, labels, tasks, log_sigmas=None):
    """MultiTaskLoss / AutoTuneMultiTaskLoss of `out` (a tensor; its dtype is the dtype of the evaluation) ->
    (loss, [weighted task values], d loss / d out, d loss / d log_sigmas or None)."""
    o = out.detach().clone().requires_grad_(True)
    ls = None if log_sigmas is None else torch.as_tensor(np.asarray(log_sigmas)).to(o.dtype).requires_grad_(True)
    loss, vals = T.multi_task_loss(o, torch.as_tensor(labels).to(o.dtype), tasks, log_sigmas=ls)
    loss.backward()
    return (float(loss.detach()), np.array([float(v.detach()) for v in vals]), o.grad,
            None if ls is None else ls.grad.numpy().astype(np.float64))


def step64(sd, x, masks, p, labels=None, tasks=None, log_sigmas=None, g_out=None, dtype=torch.float64, fwd=None):
    """One training step in `dtype` (float64: taken as exact; float32: the honest implementation): dict of out, running,
    grads, and with labels loss, vals, g_log_sigmas.  Either labels + tasks (the fused loss) or g_out (drop-in).  `fwd`: a
    `Forward` of the same (sd, x, masks, p, dtype) to reuse."""
    fwd = fwd or Forward(sd, x, masks, p, dtype)
    res = {'out': fwd.out.detach().numpy().astype(np.float64), 'running': fwd.running}
    if g_out is None:
        res['loss'], res['vals'], g_out, res['g_log_sigmas'] = loss_grad(fwd.out, labels, tasks, log_sigmas)
    res['grads'] = fwd.grads(g_out)
    return res


# ------------------------------------------------------------------------------------------------ comparison rule
def grad_rule(got, ref64, honest32, zero=False):
    """One tensor: (rel-L2(got - ref64) / max(rel-L2(honest32 - ref64), 2^-24), the same for the max-abs error over
    max |ref64|).  zero: the true value is identically zero, so there is no scale to be relative to; both ratios are then
    max |got| / max(max |honest32|, 2e-7), the honest implementation's own noise with an absolute floor."""
    got, ref, h = (np.asarray(v, dtype=np.float64).reshape(-1) for v in (got, ref64, honest32))
    assert got.shape == ref.shape == h.shape, (got.shape, ref.shape, h.shape)
    if not np.isfinite(got).all():
        return np.inf, np.inf
    if zero:
        r = float(np.abs(got).max()) / max(float(np.abs(h).max()), 2e-7)
        return r, r
    nrm, mx = max(float(np.linalg.norm(ref)), 1e-300), max(float(np.abs(ref).max()), 1e-300)
    l2 = float(np.linalg.norm(got - ref)) / nrm / max(float(np.linalg.norm(h - ref)) / nrm, FLOOR)
    mxr = float(np.abs(got - ref).max()) / mx / max(float(np.abs(h - ref).max()) / mx, FLOOR)
    return l2, mxr


def grad_ratios(sd, got, ref64, honest32):
    """{parameter: (family, rel-L2 ratio, max ratio)} of every gradient of a step."""
    out = {}
    for n in ref64:
        fam = family(n, sd)
        out[n] = (fam,) + grad_rule(got[n], ref64[n], honest32[n], zero=fam == 'zero')
    return out


def over_limit(ratios, limits=None):
    """The entries of `grad_ratios` outside LIMITS."""
    limits = limits or LIMITS
    return {n: r for n, r in ratios.items() if r[1] > limits[r[0]][0] or r[2] > limits[r[0]][1]}
