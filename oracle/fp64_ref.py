"""
Float64 restatement of the inference hot path  --  TEST INFRASTRUCTURE ONLY.

`loco_oracle.py` is an fp32 restatement: it makes the same kind of rounding errors as the kernels, so a comparison
against it can only be as sharp as a rule written in units of the column maximum.  This module computes the same
operations in float64 from the fp32 values the engine actually sees -- fp32 weights, fp32 keypoints and the fp32 K^-1 of
`engine.kinv_from_kk` (float64 inverse rounded once, restated by `kinv32` below) -- taken as exact.  Against it, an fp32
implementation's error is measurable, and `fp64_rule` expresses a kernel's error in units of the error of an honest fp32
implementation (the numpy oracle) on the same rows.

Semantics follow `loco_oracle.py` (which cites the reference's file:line for each step): process.py preprocess_monoloco /
preprocess_monstereo, architectures.py LocoModel / MonolocoModel in eval mode with optional dropout keep-masks,
process.py extract_outputs / extract_outputs_mono, net.py's (d, bi) pair, camera.py xyz_from_distance.
`monoloco_b200/` never imports this module.
"""
import math

import numpy as np

F64 = np.float64
BN_EPS = 1e-5


def _f64(a):
    return np.asarray(a, dtype=np.float32).astype(F64)


def kinv32(kk):
    """K^-1 as the engine passes it to the kernels (engine.kinv_from_kk): float64 inverse of K as given, rounded once to
    fp32 (9,)."""
    k = np.asarray(kk, dtype=F64).reshape(3, 3)
    return np.linalg.inv(k).astype(np.float32).reshape(9)


# ------------------------------------------------------------------------------------------------ pre-process
def _centre(kps):
    """bbox centre (max - min) / 2 + min of the u and v rows: kps (m,3,17) -> (m,), (m,)."""
    u, v = kps[:, 0, :], kps[:, 1, :]
    return (u.max(1) - u.min(1)) / 2 + u.min(1), (v.max(1) - v.min(1)) / 2 + v.min(1)


def _to_camera(u, v, kinv, z_met):
    """rows 0/1 of [u v 1] K^-T times z_met, plus sum |terms| * z_met of each (the scale of its rounding error)."""
    k = _f64(kinv)
    x = (u * k[0] + v * k[1] + k[2]) * z_met
    y = (u * k[3] + v * k[4] + k[5]) * z_met
    bx = (np.abs(u * k[0]) + np.abs(v * k[1]) + abs(k[2])) * z_met
    by = (np.abs(u * k[3]) + np.abs(v * k[4]) + abs(k[5])) * z_met
    return x, y, bx, by


def preprocess_mono(kps, kinv, zero_center=False, z_met=10.0):
    """(m,3,17) keypoints -> ((m,34) inputs x0,y0,...,x16,y16, (m,34) componentwise error scale sum |terms| * z_met)."""
    kps = _f64(kps)
    x, y, bx, by = _to_camera(kps[:, 0, :], kps[:, 1, :], kinv, z_met)
    if zero_center:
        uc, vc = _centre(kps)
        cx, cy, _, _ = _to_camera(uc, vc, kinv, z_met)
        # the centre itself is rounded twice in fp32: its scale is |max| + |min|, not |centre|
        ub = np.abs(kps[:, 0, :]).max(1) * 2
        vb = np.abs(kps[:, 1, :]).max(1) * 2
        _, _, bcx, bcy = _to_camera(ub, vb, np.abs(_f64(kinv)), z_met)
        x, y = x - cx[:, None], y - cy[:, None]
        bx, by = bx + bcx[:, None] + np.abs(x), by + bcy[:, None] + np.abs(y)
    out = np.stack([x, y], axis=2).reshape(len(kps), 34)
    bound = np.stack([bx, by], axis=2).reshape(len(kps), 34)
    return out, bound


def preprocess_stereo(kps_l, kps_r, kinv, z_met=10.0):
    """all-vs-all rows l * R + r = cat(l, l - r) -> ((L*R, 68) inputs, (L*R, 68) componentwise error scale).  The
    difference cancels, so its scale is the sum of both sides' scales, not |l - r|."""
    xl, bl = preprocess_mono(kps_l, kinv, z_met=z_met)
    xr, br = preprocess_mono(kps_r, kinv, z_met=z_met)
    nl, nr = len(xl), len(xr)
    left, right = np.repeat(xl, nr, axis=0), np.tile(xr, (nl, 1))
    bleft, bright = np.repeat(bl, nr, axis=0), np.tile(br, (nl, 1))
    return np.concatenate([left, left - right], 1), np.concatenate([bleft, bleft + bright + np.abs(left - right)], 1)


# ------------------------------------------------------------------------------------------------ network (eval)
def _linear(x, sd, name):
    return x @ _f64(sd[name + '.weight']).T + _f64(sd[name + '.bias'])


def _bn(x, sd, name):
    inv = 1.0 / np.sqrt(_f64(sd[name + '.running_var']) + BN_EPS)
    return (x - _f64(sd[name + '.running_mean'])) * inv * _f64(sd[name + '.weight']) + _f64(sd[name + '.bias'])


def _drop(x, mask, p):
    return x if mask is None else x * np.asarray(mask, dtype=F64) / (1.0 - p)


def _num_stages(sd):
    n = 0
    while 'linear_stages.%d.w1.weight' % n in sd:
        n += 1
    return n


def _trunk(sd, x, m1, p):
    relu = lambda v: np.maximum(v, 0.0)  # noqa: E731
    y = _drop(relu(_bn(_linear(_f64(x), sd, 'w1'), sd, 'batch_norm1')), m1, p)
    for i in range(_num_stages(sd)):
        pre = 'linear_stages.%d.' % i
        z = relu(_bn(_linear(y, sd, pre + 'w1'), sd, pre + 'batch_norm1'))
        z = relu(_bn(_linear(z, sd, pre + 'w2'), sd, pre + 'batch_norm2'))
        y = y + z
    return y


def model_forward(sd, x, drop_masks=None, p_dropout=0.2):
    """LocoModel (w_fin in sd) or MonolocoModel eval forward in float64; drop_masks = keep masks after batch_norm1 and
    (LocoModel) after batch_norm3, as loco_oracle.loco_model_forward takes them."""
    m1, m3 = drop_masks if drop_masks is not None else (None, None)
    y = _trunk(sd, x, m1, p_dropout)
    if 'w_fin.weight' not in sd:
        return _linear(y, sd, 'w2')
    y = _linear(y, sd, 'w2')
    aux = _linear(y, sd, 'w_aux')
    y = _drop(np.maximum(_bn(_linear(y, sd, 'w3'), sd, 'batch_norm3'), 0.0), m3, p_dropout)
    return np.concatenate([_linear(y, sd, 'w_fin'), aux], axis=1)


# ------------------------------------------------------------------------------------------------ decode
DECODE_LOCO, DECODE_MONO, DECODE_DB = 1, 2, 3   # include/monoloco_b200.h


def _wrap(yaw):
    """camera.py back_correct_angles: one wrap by 2 pi in each direction."""
    yaw = np.where(yaw > math.pi, yaw - 2 * math.pi, yaw)
    return np.where(yaw < -math.pi, yaw + 2 * math.pi, yaw)


def decode(raw, kind):
    """Raw outputs -> (m,8) rows (x, y, z, d, bi, yaw_pred, yaw_orig, aux) in the layout of the engine's `dec` output:
    extract_outputs (kind 1, 9 or 10 columns), extract_outputs_mono (kind 2), net.py's (d, bi) (kind 3, 2 columns).
    Columns a kind does not define are 0; z of an inconsistent (d, theta, psi) is NaN, as in the reference."""
    o = np.asarray(raw, dtype=F64)
    m = o.shape[0]
    out = np.zeros((m, 8), dtype=F64)
    with np.errstate(invalid='ignore', over='ignore'):
        if kind == DECODE_LOCO:
            th, ps, d = o[:, 0], o[:, 1], o[:, 2]
            x = d * np.sin(ps) * np.cos(th)
            y = d * np.cos(ps)
            z = np.sqrt(d * d - x * x - y * y)
            out[:, 0:5] = np.stack([x, y, z, d, np.exp(o[:, 3]) * d], 1)
            if o.shape[1] == 10:
                out[:, 7] = 1.0 / (1.0 + np.exp(-o[:, 9]))
        elif kind == DECODE_MONO:
            x, y, z = o[:, 0], o[:, 1], o[:, 2]
            out[:, 0:5] = np.stack([x, y, z, np.sqrt(x * x + y * y + z * z), np.exp(o[:, 3]) * o[:, 2]], 1)
        elif kind == DECODE_DB:
            out[:, 3] = o[:, 0]
            out[:, 4] = np.exp(o[:, 1]) * o[:, 0]
        else:
            raise ValueError(kind)
        if kind in (DECODE_LOCO, DECODE_MONO):
            out[:, 5] = np.arctan2(o[:, 7], o[:, 8])
            out[:, 6] = _wrap(out[:, 5] + np.arctan2(out[:, 0], out[:, 2]))
    return out


# ------------------------------------------------------------------------------------------------ bbox-centre ray
def xyzc(kps, kinv, d):
    """net.py: xy_centers = pixel_to_camera(bbox centre, K, 1); xyz_from_distance(d, xy_centers) and its norm -> (m,4)."""
    kps = _f64(kps)
    k = _f64(kinv)
    uc, vc = _centre(kps)
    c = np.stack([uc * k[0] + vc * k[1] + k[2], uc * k[3] + vc * k[4] + k[5], uc * k[6] + vc * k[7] + k[8]], 1)
    xyz = c * np.asarray(d, dtype=F64).reshape(-1, 1) / np.sqrt(1.0 + c[:, 0:1] ** 2 + c[:, 1:2] ** 2)
    return np.concatenate([xyz, np.sqrt((xyz ** 2).sum(1, keepdims=True))], 1)


# ------------------------------------------------------------------------------------------------ comparison rule
# Allowed (max, RMS) ratios of fp64_rule for the FFMA kernel families and for the 3xTF32 tensor-core kernel, set from
# tests/test_forward_fp64_gpu.py on one H100 80GB HBM3 (400 W power limit; the kernels are deterministic, so these are
# fixed functions of the code).  Worst measured over every width, batch edge, feature and refresh case:
#   FFMA (row tiles, cluster, whole grid, wide2): max 2.75, RMS 2.51 (row tiles) -> 4.0.
#   tensor cores: max 41.2, RMS 49.4 (width 2048, one-element refreshes; fresh weights 17.4 / 23.5 at 2048, 6.0 / 10.8 at
#   1024) -> 75 = 1.5x the worst.  The emulation of the kernel's own scheme with a truncating accumulator
#   (tools/tf32x3_study.mm_tf32x3_split) gives 34-36 / 47-54 at 1536-2048: the excess is the wgmma accumulator's rounding
#   (DESIGN.md §2a; the accumulator change that would reduce it is a known gap, §9).
FFMA_RULE = (4.0, 4.0)
TC_RULE = (75.0, 75.0)


def _col_errors(x, ref64):
    x = np.asarray(x, dtype=F64).reshape(len(ref64), -1)
    ref64 = np.asarray(ref64, dtype=F64).reshape(x.shape)
    fin = np.isfinite(ref64)
    r = np.where(fin, ref64, 0.0)
    e = np.abs(np.where(fin, x - r, 0.0))
    n = np.maximum(fin.sum(0), 1)
    rms = np.sqrt((np.where(np.isfinite(e), e, 0.0) ** 2).sum(0) / n)
    return e, rms, fin, np.abs(r).max(0)


def fp64_rule(got, ref64, honest32, pool=None):
    """Per output column: (max |got - ref64| / max |honest32 - ref64|, rms |got - ref64| / rms |honest32 - ref64|).
    `honest32` is an fp32 implementation of the same operation on the same rows (the numpy oracle).  Both denominators
    are floored at 2^-24 * the column's max |ref64|, so an exactly computed column does not divide by zero.  Rows where
    ref64 is NaN are skipped; a NaN in `got` anywhere else makes that column's ratios infinite.
    pool = (ref64_pool, honest32_pool): take the denominators from these rows of the same operation instead (a superset
    of got's rows): the worst honest error of one or a few rows is too noisy a unit.
    Returns two float64 arrays of one ratio per column."""
    eg, rms_g, fin, _ = _col_errors(got, ref64)
    eh, rms_h, fin_h, cmax = _col_errors(*((honest32, ref64) if pool is None else (pool[1], pool[0])))
    eh = np.where(np.isfinite(eh), eh, 0.0)
    bad = (fin & ~np.isfinite(np.asarray(got, dtype=F64).reshape(eg.shape))).any(0)
    floor = np.maximum(2.0 ** -24 * cmax, np.finfo(F64).tiny)
    max_ratio = eg.max(0) / np.maximum(eh.max(0), floor)
    rms_ratio = rms_g / np.maximum(rms_h, floor)
    max_ratio[bad] = np.inf
    rms_ratio[bad] = np.inf
    return max_ratio, rms_ratio
