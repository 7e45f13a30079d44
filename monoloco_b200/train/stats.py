"""Loss statistics of the train / validate / evaluate loop on the device (csrc/task_stats.cu, `mlb_task_stats`).

`task_stats` adds, for every CSR row segment of (outputs, labels), what `MultiTaskLoss(..., phase='val')`,
`Trainer.epoch_logs` and `Trainer.compute_stats` (trainer.py:165-167, 193-197, 250-284) read from those rows into an fp64
device accumulator [n_seg, STATS_NACC]; columns are the `_lib.STAT_*` indices (include/monoloco_b200.h). One launch, no
host synchronisation. `task_stats_host` states the same sums in float64 numpy; the tests hold the kernel to it."""
import ctypes as C

import numpy as np
import torch

from .. import _lib as L_

TASK_ORDER = ('d', 'x', 'y', 'h', 'w', 'l', 'ori', 'aux')


def _mask(tasks):
    tasks = tuple(tasks)
    unknown = [t for t in tasks if t not in L_.TASK_IDS]
    if unknown:
        raise ValueError("task_stats: unknown tasks %s" % unknown)
    if list(tasks) != sorted(tasks, key=L_.TASK_IDS.get) or len(set(tasks)) != len(tasks):
        raise ValueError("task_stats: tasks must be distinct and in the order %s (log_sigmas are read in that order)"
                         % (TASK_ORDER,))
    return sum(1 << L_.TASK_IDS[t] for t in tasks)


def _seg_off(seg_off):
    off = [int(v) for v in seg_off]
    if not 2 <= len(off) <= L_.STATS_MAX_SEG + 1:
        raise ValueError("task_stats: seg_off needs 2..%d entries (got %d)" % (L_.STATS_MAX_SEG + 1, len(off)))
    return off


def task_stats(outputs, labels, seg_off, tasks, lambdas=None, log_sigmas=None, acc=None):
    """outputs [n, 9|10], labels [n, 10|11] (fp32 CUDA tensors), seg_off: host list of n_seg + 1 row offsets.
    Adds into `acc` (fp64 CUDA [n_seg, STATS_NACC]; a zeroed one is made when None) and returns it."""
    off = _seg_off(seg_off)
    mask = _mask(tasks)
    if not (outputs.is_cuda and labels.is_cuda):
        raise RuntimeError("task_stats runs on CUDA tensors only")
    if outputs.dim() != 2 or labels.dim() != 2 or outputs.shape[0] != labels.shape[0]:
        raise ValueError("task_stats: outputs [n, 9|10] and labels [n, 10|11] with the same n")
    if off[-1] > outputs.shape[0]:
        raise ValueError("task_stats: seg_off[-1] = %d exceeds the %d rows" % (off[-1], outputs.shape[0]))
    n_seg = len(off) - 1
    if acc is None:
        acc = torch.zeros((n_seg, L_.STATS_NACC), dtype=torch.float64, device=outputs.device)
    elif acc.dtype != torch.float64 or tuple(acc.shape) != (n_seg, L_.STATS_NACC) or not acc.is_contiguous() \
            or acc.device != outputs.device:
        raise ValueError("task_stats: acc must be a contiguous float64 [%d, %d] tensor on %s"
                         % (n_seg, L_.STATS_NACC, outputs.device))
    outputs = outputs.detach().float().contiguous()
    labels = labels.detach().float().contiguous()
    a = L_.MlbTaskStatsArgs()
    a.n_seg, a.out_cols, a.label_ld, a.task_mask = n_seg, outputs.shape[1], labels.shape[1], mask
    for i, v in enumerate(off):
        a.seg_off[i] = v
    lam = (1.0,) * len(tuple(tasks)) if lambdas is None else tuple(lambdas)
    for t, v in zip(tasks, lam):
        a.lambdas[L_.TASK_IDS[t]] = float(v)
    a.out, a.labels, a.acc = outputs.data_ptr(), labels.data_ptr(), acc.data_ptr()
    if log_sigmas is not None:
        if not log_sigmas.is_cuda or log_sigmas.dtype != torch.float32 or log_sigmas.numel() != len(tuple(tasks)):
            raise ValueError("task_stats: log_sigmas must be a float32 CUDA tensor with one entry per task")
        a.log_sigmas = log_sigmas.data_ptr()
    L_.check(L_.lib().mlb_task_stats(C.byref(a), C.c_void_p(torch.cuda.current_stream(outputs.device).cuda_stream)),
             'mlb_task_stats')
    return acc


def task_stats_host(outputs, labels, seg_off, tasks, lambdas=None, log_sigmas=None):
    """float64 numpy statement of mlb_task_stats (one fresh accumulator); fp32 where the reference compares in fp32."""
    out = np.asarray(outputs, dtype=np.float32)
    lab = np.asarray(labels, dtype=np.float32)
    tasks = tuple(tasks)
    lam = (1.0,) * len(tasks) if lambdas is None else tuple(lambdas)
    acc = np.zeros((len(seg_off) - 1, L_.STATS_NACC))
    for s in range(len(seg_off) - 1):
        o, y = out[seg_off[s]:seg_off[s + 1]], lab[seg_off[s]:seg_off[s + 1]]
        n = o.shape[0]
        if n == 0:
            continue
        o64, y64 = o.astype(np.float64), y.astype(np.float64)
        err = np.abs(o[:, 2] - y[:, 3])
        with np.errstate(over='ignore'):
            bi = np.exp(o[:, 3]) * o[:, 2]
        lap = np.abs(1.0 - o64[:, 2] / y64[:, 3]) * np.exp(-o64[:, 3]) + 0.01 + o64[:, 3] + 2.0
        val = {'d': err.astype(np.float64).sum(),
               'ori': np.abs(np.arctan2(o64[:, 7], o64[:, 8]) - np.arctan2(y64[:, 7], y64[:, 8])).sum()}
        for t, c in (('x', 0), ('y', 1), ('h', 4), ('w', 5), ('l', 6)):
            val[t] = np.abs(o64[:, c] - y64[:, c]).sum()
        ori_l1 = np.abs(o64[:, 7:9] - y64[:, 7:9]).sum()
        a = acc[s]
        if 'aux' in tasks:
            x, t = o64[:, 9], y64[:, 10]
            m = np.maximum(-x, 0.0)
            val['aux'] = ((1.0 - t) * x + m + np.log(np.exp(-m) + np.exp(-x - m))).sum()
            with np.errstate(over='ignore'):
                sig = np.float32(1.0) / (np.float32(1.0) + np.exp(-o[:, 9]))
            a[L_.STAT_AUX_MISS] = np.abs((sig >= 0.5).astype(np.float64) - t).sum()
        total, sum_ls = 0.0, 0.0
        for i, t in enumerate(tasks):
            w = float(np.float32(lam[i]))
            if log_sigmas is not None:
                ls = float(np.asarray(log_sigmas, dtype=np.float32)[i])
                w = w / (2.0 * np.exp(ls) ** 2)
                sum_ls += ls
            total += w * (lap.sum() if t == 'd' else 0.5 * ori_l1 if t == 'ori' else val[t])
        a[L_.STAT_N] = n
        a[L_.STAT_TOTAL] = total + n * sum_ls
        for t in tasks:
            a[L_.STAT_VAL + L_.TASK_IDS[t]] = val[t]
        a[L_.STAT_BI] = bi.astype(np.float64).sum()
        a[L_.STAT_BI_HIT] = float((err <= bi).sum())
        a[L_.STAT_ERR] = err.astype(np.float64).sum()
        a[L_.STAT_ERR2] = (err.astype(np.float64) ** 2).sum()
        a[L_.STAT_LAPLACE] = lap.sum()
        a[L_.STAT_ORI_L1] = ori_l1
    return acc


def val_values(acc_row, tasks):
    """CompositeLoss val-form means of one accumulator row (host numpy), in `tasks` order."""
    n = acc_row[L_.STAT_N]
    vals = []
    for t in tasks:
        v = acc_row[L_.STAT_VAL + L_.TASK_IDS[t]] / n
        vals.append(v * 180 / 3.14 if t == 'ori' else v)
    return vals


def err_std(acc_row):
    """Unbiased std of |d - d_gt| (torch's errs.std()): NaN for fewer than 2 rows."""
    n, s, s2 = acc_row[L_.STAT_N], acc_row[L_.STAT_ERR], acc_row[L_.STAT_ERR2]
    if n < 2:
        return float('nan')
    return float(np.sqrt(max(s2 - s * s / n, 0.0) / (n - 1)))
