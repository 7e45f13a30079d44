"""
Fused training step for the LocoModel and MonolocoModel mirrors (monoloco_b200/csrc/train.cu).

Two ways in, both replacing trainer.py:153-161 (`outputs = model(inputs)`, `mt_loss`, `loss.backward()`):
  * drop-in: `model(inputs)` in train mode returns outputs that carry an autograd node (`_FusedTrainFn`);
    any loss built from them (the MultiTaskLoss mirror, or the reference's own) calls back into ONE backward
    kernel launch that writes every parameter gradient.  Two launches per step.
  * `train_step(model, inputs, labels, tasks, lambdas, log_sigmas)`: forward + multi-task loss + backward in a
    SINGLE cooperative kernel launch; `.grad` of every parameter (and of log_sigmas) is populated directly.
    LocoModel only: MultiTaskLoss indexes LocoModel's output columns, and MonolocoModel trains through the drop-in.
Optimizer / clip_grad_norm_ / scheduler stay PyTorch (trainer.py:159-161).
"""
import ctypes as C
import os
import weakref

import torch

from .. import _lib as L_

_WS = weakref.WeakKeyDictionary()


def _is_loco(model):
    from ..network.architectures import LocoModel
    return isinstance(model, LocoModel)


def _blocks_of(model):
    """(name of Linear, name of BatchNorm or None, res_src) in forward order: LocoModel (architectures.py:48-71) ends
    with the BatchNorm-free w2 and w3; MonolocoModel (:135-176) ends with its last stage, whose residual the head reads."""
    blocks = [('w1', 'batch_norm1', -1)]
    src = 0
    for i in range(model.num_stage):
        blocks.append(('linear_stages.%d.w1' % i, 'linear_stages.%d.batch_norm1' % i, -1))
        blocks.append(('linear_stages.%d.w2' % i, 'linear_stages.%d.batch_norm2' % i, src))
        src = len(blocks) - 1
    if _is_loco(model):
        blocks.append(('w2', None, -1))
        blocks.append(('w3', 'batch_norm3', -1))
    return blocks


def _heads_of(model):
    """(input size, aux head or None, final head, output columns): LocoModel's out = [w_fin | w_aux]; MonolocoModel's
    out = w2 (no aux head, mlb_train_args.aux_block = -1)."""
    if _is_loco(model):
        return model.stereo_size, 'w_aux', 'w_fin', model.output_size + 1
    return model.input_size, None, 'w2', model.output_size


class _Workspace:
    def __init__(self, model, max_rows, device):
        self.lib = L_.lib()
        self.h = C.c_void_p()
        self.max_rows = max_rows
        self.blocks = _blocks_of(model)
        self.in_size, self.aux, self.fin, self.out_cols = _heads_of(model)
        self.lambda_cache = {}
        self.generation = 0   # bumped by every launch that overwrites the saved activations (forward / train_step)
        L_.check(self.lib.mlb_train_create(device.index if device.index is not None else torch.cuda.current_device(),
                                           max_rows, self.in_size, model.linear_size, len(self.blocks),
                                           C.byref(self.h)), 'mlb_train_create')

    def __del__(self):
        try:
            if self.h.value:
                self.lib.mlb_train_destroy(self.h)
        except Exception:
            pass


def _workspace(model, n_rows, device):
    ws = _WS.get(model)
    if ws is None or ws.max_rows < n_rows:
        ws = _Workspace(model, max(n_rows, 512), device)
        _WS[model] = ws
    return ws


def _mod(model, dotted):
    m = model
    for part in dotted.split('.'):
        m = m[int(part)] if part.isdigit() else getattr(m, part)
    return m


def _fill(model, ws, x, out, grads=None, g_out=None, labels=None, tasks=None, scales=None, loss_vals=None,
          drop_seed=0, drop_mask=None, update_running=True):
    """Build the C structs from the live module parameters (device pointers, native layouts)."""
    nb = len(ws.blocks)
    blocks = (L_.MlbTrainBlock * nb)()
    for i, (lin, bn, res) in enumerate(ws.blocks):
        lm = _mod(model, lin)
        b = blocks[i]
        b.K, b.has_bn, b.res_src = lm.in_features, int(bn is not None), res
        b.W, b.b = lm.weight.data_ptr(), lm.bias.data_ptr()
        if grads is not None:
            b.dW, b.db = grads[lin + '.weight'].data_ptr(), grads[lin + '.bias'].data_ptr()
        if bn is not None:
            bm = _mod(model, bn)
            b.gamma, b.beta = bm.weight.data_ptr(), bm.bias.data_ptr()
            b.running_mean, b.running_var = bm.running_mean.data_ptr(), bm.running_var.data_ptr()
            if grads is not None:
                b.dgamma, b.dbeta = grads[bn + '.weight'].data_ptr(), grads[bn + '.bias'].data_ptr()
    a = L_.MlbTrainArgs()
    a.n_rows, a.input_size, a.output_size = x.shape[0], ws.in_size, ws.out_cols
    a.linear_size, a.n_blocks, a.aux_block = model.linear_size, nb, nb - 2 if ws.aux else -1
    a.update_running_stats = int(update_running)
    a.rows_per_group = int(os.environ.get('MLB_TRAIN_ROWS_PER_GROUP', '0'))  # 0 = auto; tests sweep 8..16
    a.p_dropout, a.bn_eps, a.bn_momentum = float(model.p_dropout), 1e-5, 0.1
    a.drop_seed = int(drop_seed)
    if drop_mask is not None:
        a.drop_mask = drop_mask.data_ptr()
    a.x, a.out = x.data_ptr(), out.data_ptr()
    fin = _mod(model, ws.fin)
    a.W_fin, a.b_fin = fin.weight.data_ptr(), fin.bias.data_ptr()
    if grads is not None:
        a.dW_fin, a.db_fin = grads[ws.fin + '.weight'].data_ptr(), grads[ws.fin + '.bias'].data_ptr()
    if ws.aux:   # MonolocoModel: no aux head, its pointers stay NULL
        aux = _mod(model, ws.aux)
        a.W_aux, a.b_aux = aux.weight.data_ptr(), aux.bias.data_ptr()
        if grads is not None:
            a.dW_aux, a.db_aux = grads[ws.aux + '.weight'].data_ptr(), grads[ws.aux + '.bias'].data_ptr()
    if g_out is not None:
        a.g_out = g_out.data_ptr()
    if labels is not None:
        a.labels, a.label_ld, a.n_tasks = labels.data_ptr(), labels.shape[1], len(tasks)
        for i, t in enumerate(tasks):
            a.tasks[i] = L_.TASK_IDS[t]
        if torch.is_tensor(scales):          # device tensor: the kernel reads it, nothing crosses to the host
            a.task_scale_dev = scales.data_ptr()
        else:
            for i in range(len(tasks)):
                a.task_scale[i] = float(scales[i])
        a.loss_vals = loss_vals.data_ptr()
    return a, blocks


def _stream(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _check_model(model, x):
    from ..network.architectures import LocoModel, MonolocoModel
    if not isinstance(model, (LocoModel, MonolocoModel)):
        raise NotImplementedError("fused training supports the LocoModel and MonolocoModel topologies")
    if isinstance(model, MonolocoModel):
        # 1 + 2 num_stage blocks; the kernel takes 2..MLB_MAX_BLOCKS (16) of them and at most 16 output columns
        if not 1 <= model.num_stage <= 7:
            raise ValueError("fused training of MonolocoModel needs num_stage in [1, 7] (got %d)" % model.num_stage)
        if not 1 <= model.output_size <= 16:
            raise ValueError("fused training of MonolocoModel needs output_size in [1, 16] (got %d)" % model.output_size)
    if not x.is_cuda or next(model.parameters()).device != x.device:
        raise RuntimeError("monoloco_b200 training runs on CUDA tensors only (no CPU fallback)")
    if x.shape[0] < 2:
        raise ValueError("Expected more than 1 value per channel when training (nn.BatchNorm1d)")


def _bump_batches_tracked(model):
    # nn.BatchNorm1d.num_batches_tracked of every layer, one multi-tensor launch
    torch._foreach_add_([m.num_batches_tracked for m in model.modules() if isinstance(m, torch.nn.BatchNorm1d)], 1)


class _FusedTrainFn(torch.autograd.Function):
    """outputs = model(inputs) in train mode; backward = one launch producing every parameter gradient."""

    @staticmethod
    def forward(ctx, x, model, seed, drop_mask, *params):
        ws = _workspace(model, x.shape[0], x.device)
        x = x.detach().float().contiguous()
        out = torch.empty((x.shape[0], ws.out_cols), dtype=torch.float32, device=x.device)
        a, blocks = _fill(model, ws, x, out, drop_seed=seed, drop_mask=drop_mask)
        L_.check(ws.lib.mlb_train_forward(ws.h, C.byref(a), blocks, _stream(x.device)), 'mlb_train_forward')
        _bump_batches_tracked(model)
        ws.generation += 1
        ctx.model, ctx.ws, ctx.x, ctx.seed, ctx.drop_mask, ctx.out = model, ws, x, seed, drop_mask, out
        ctx.generation = ws.generation
        return out

    @staticmethod
    def backward(ctx, g_out):
        model, ws, x = ctx.model, ctx.ws, ctx.x
        if ws.generation != ctx.generation:
            # the saved activations (Z / A / batch statistics) live in the per-model workspace, one set at a time: a later
            # train-mode forward or train_step() has overwritten the ones this graph needs
            raise RuntimeError(
                "monoloco_b200: backward through a train-mode forward whose saved activations were overwritten by a later "
                "train-mode forward of the same model (micro-batch accumulation, (loss1 + loss2).backward(), a no_grad "
                "train-mode forward in between).  Call backward() before the next train-mode forward, or use "
                "train_step(..., accumulate=True) per micro-batch.")
        grads = {n: torch.empty_like(p) for n, p in model.named_parameters()}
        g_out = g_out.float().contiguous()
        a, blocks = _fill(model, ws, x, ctx.out, grads=grads, g_out=g_out, drop_seed=ctx.seed, drop_mask=ctx.drop_mask,
                          update_running=False)
        L_.check(ws.lib.mlb_train_backward(ws.h, C.byref(a), blocks, _stream(x.device)), 'mlb_train_backward')
        return (None, None, None, None) + tuple(grads[n] for n, _ in model.named_parameters())


def _next_drop_seed(device):
    """Seed of the in-kernel dropout RNG for one step, taken from the device's default CUDA generator the way the
    reference's CUDA nn.Dropout consumes it: (initial seed, philox offset) hashed, offset advanced on the HOST (no kernel,
    no synchronisation).  The global CPU generator is never touched, so the DataLoader permutations that follow a
    `torch.manual_seed(s)` stay identical to the reference's in every epoch (ADVICE r1); `torch.manual_seed` re-seeds the
    CUDA generators too, so runs stay reproducible."""
    import hashlib
    idx = device.index if device.index is not None else torch.cuda.current_device()
    gen = torch.cuda.default_generators[idx]
    seed0, off = int(gen.initial_seed()), int(gen.get_offset())
    gen.set_offset(off + 4)   # philox offsets move in multiples of 4
    mix = hashlib.blake2b(seed0.to_bytes(8, 'little', signed=seed0 < 0) + off.to_bytes(8, 'little'), digest_size=8).digest()
    return int.from_bytes(mix, 'little') >> 2


def fused_train_forward(model, x, drop_mask=None, seed=None):
    """LocoModel.forward in train mode (called by the module mirror)."""
    _check_model(model, x)
    if seed is None:
        seed = _next_drop_seed(x.device)
    params = [p for _, p in model.named_parameters()]
    return _FusedTrainFn.apply(x, model, seed, drop_mask, *params)


def train_step(model, x, labels, tasks, lambdas=None, log_sigmas=None, drop_mask=None, seed=None, accumulate=False):
    """Forward + MultiTaskLoss (losses.py:59-73; AutoTune :28-43 when log_sigmas is given) + backward in ONE kernel
    launch.  Populates `.grad` of every model parameter (and of log_sigmas); returns (loss, [weighted task losses])
    exactly like `mt_loss(model(x), labels, phase='train')` followed by `loss.backward()`.  LocoModel only."""
    _check_model(model, x)
    if not _is_loco(model):
        raise NotImplementedError(
            "train_step() fuses MultiTaskLoss, which reads LocoModel's output columns (process.py:231-254); the reference "
            "defines no multi-task loss for MonolocoModel's outputs.  Train MonolocoModel through the drop-in instead: "
            "out = model(x) in train mode, any loss built in torch from `out`, loss.backward() (two launches).")
    if seed is None:
        seed = _next_drop_seed(x.device)
    tasks = tuple(tasks)
    lambdas = tuple(lambdas) if lambdas is not None else (1,) * len(tasks)
    ws = _workspace(model, x.shape[0], x.device)
    x = x.detach().float().contiguous()
    labels = labels.detach().float().contiguous()
    out = torch.empty((x.shape[0], ws.out_cols), dtype=torch.float32, device=x.device)
    # task weights as a device tensor (cached per lambdas; AutoTune's depend on log_sigmas and are computed on the device):
    # no host<->device synchronisation anywhere in the step, so consecutive steps queue back to back
    lam = ws.lambda_cache.get(lambdas)
    if lam is None:
        lam = ws.lambda_cache[lambdas] = torch.tensor([float(v) for v in lambdas], dtype=torch.float32, device=x.device)
    if log_sigmas is not None:
        scales = lam / (2.0 * torch.exp(log_sigmas.detach().float()) ** 2)   # losses.py:36-38
    else:
        scales = lam
    grads = {n: torch.empty_like(p) for n, p in model.named_parameters()}
    loss_vals = torch.zeros(8, dtype=torch.float32, device=x.device)
    a, blocks = _fill(model, ws, x, out, grads=grads, labels=labels, tasks=tasks, scales=scales, loss_vals=loss_vals,
                      drop_seed=seed, drop_mask=drop_mask)
    L_.check(ws.lib.mlb_train_step(ws.h, C.byref(a), blocks, _stream(x.device)), 'mlb_train_step')
    ws.generation += 1   # the workspace's saved activations now belong to this step
    _bump_batches_tracked(model)
    for n, p in model.named_parameters():
        p.grad = grads[n] if (p.grad is None or not accumulate) else p.grad + grads[n]
    weighted = loss_vals[:len(tasks)] * scales
    loss = weighted.sum()
    if log_sigmas is not None:
        loss = loss + log_sigmas.detach().sum()
        # d/d log_sigma_t [ lam L_t / (2 exp(2 ls_t)) + ls_t ] = -2 * weighted_t + 1
        g = 1.0 - 2.0 * weighted
        log_sigmas.grad = g if (log_sigmas.grad is None or not accumulate) else log_sigmas.grad + g
    return loss, [weighted[i] for i in range(len(tasks))], out


def phase_times(model):
    """[(phase type name, block, ms)] of the most recent train launch of `model` (profiling aid)."""
    ws = _WS.get(model)
    names = ['PACK', 'FWD', 'FWD_FINAL', 'BWD_INIT', 'BWD_HEAD', 'BWD', 'DW', 'PAD', 'UNPAD']
    ns = (C.c_double * 64)()
    ty = (C.c_int * 64)()
    bk = (C.c_int * 64)()
    n = ws.lib.mlb_train_phase_times(ws.h, 64, ns, ty, bk)
    return [(names[ty[i]], bk[i], ns[i] * 1e-6) for i in range(n)]


def subphase_times(model):
    """[(phase name, block, [[ms at point k for k in 0..7] for CTA first/middle/last])] of the most recent train launch:
    points are 0 input tile ready, 1 GEMM done, 2 epilogue done, 3 left the grid barrier, 4 statistics loaded, 5 tile rows finished (profiling aid)."""
    ws = _WS.get(model)
    ph = phase_times(model)
    ns = (C.c_double * (64 * 24))()
    n = ws.lib.mlb_train_subphase_times(ws.h, 64, ns)
    return [(ph[i][0], ph[i][1], [[ns[i * 24 + s * 8 + k] * 1e-6 for k in range(8)] for s in range(3)]) for i in range(n)]
