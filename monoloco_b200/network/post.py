"""`Loco.post_process` for MANY images in one device launch, and the KITTI rows of `save_txts` (SURVEY.md 8(f) row N3).

The reference post-processes one image at a time in Python loops (monoloco/network/net.py:164-248, one
`get_iou_matches` per image, monoloco/utils/iou.py:44-64) and evaluation drives it over a whole split
(monoloco/eval/generate_kitti.py:87-166).  Here the detections and ground truths of all images are concatenated
(CSR offsets) and `mlb_post_process` runs one CTA per image: bbox-centre rays, `xyz_from_distance`, the confidence,
IoU matching (fp64, same operation order as the reference's Python floats, so the match indices and the output order
are exact), the left-to-right reorder and `xyz_real`.  The host only assembles the result dictionaries.

No CPU fallback: without the CUDA library / a device these functions raise."""
import ctypes as C
from collections import defaultdict

import numpy as np
import torch

from .. import _lib as L_
from ..engine import kinv_from_kk


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def post_process_batch(items, iou_min=0.3, reorder=True, device=None):
    """items: list of (dic_in, boxes, keypoints, kk, dic_gt) exactly as `Loco.post_process` takes them (dic_gt may be
    None; a `dic_in` of None yields an empty dictionary).  Returns the list of per-image result dictionaries."""
    if not torch.cuda.is_available():
        raise RuntimeError("monoloco_b200: no CUDA device -- post_process_batch has no CPU fallback")
    lib = L_.lib()
    dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    live = [i for i, it in enumerate(items) if it[0] is not None and len(it[1]) > 0]
    results = [defaultdict(list) for _ in items]
    if not live:
        return results
    det_off, gt_off = [0], [0]
    boxes, kps, kinv, dec, gtb, gtd = [], [], [], [], [], []
    any_gt = False
    for i in live:
        dic_in, bx, kp, kk, dic_gt = items[i]
        m = len(bx)
        det_off.append(det_off[-1] + m)
        boxes.append(np.asarray(bx, dtype=np.float64).reshape(m, 5))
        kps.append(np.asarray(kp, dtype=np.float32).reshape(m, 3, 17))
        kinv.append(kinv_from_kk(kk))
        d = np.zeros((m, 8), dtype=np.float32)
        d[:, 3] = np.asarray(dic_in['d'], dtype=np.float32).reshape(-1)
        d[:, 4] = np.asarray(dic_in['bi'], dtype=np.float32).reshape(-1)
        dec.append(d)
        if dic_gt and len(dic_gt['boxes']):
            any_gt = True
            g = len(dic_gt['boxes'])
            gtb.append(np.asarray(dic_gt['boxes'], dtype=np.float64).reshape(g, -1)[:, :4])
            gtd.append(np.asarray([y[3] for y in dic_gt['ys']], dtype=np.float64))
            gt_off.append(gt_off[-1] + g)
        else:
            gt_off.append(gt_off[-1])
    M = det_off[-1]
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(dev, dtype=dt)  # noqa: E731
    d_boxes = t(np.concatenate(boxes), torch.float64)
    d_kps = t(np.concatenate(kps), torch.float32)
    d_kinv = t(np.stack(kinv), torch.float32)
    d_dec = t(np.concatenate(dec), torch.float32)
    d_doff = t(np.asarray(det_off, dtype=np.int32), torch.int32)
    d_goff = t(np.asarray(gt_off, dtype=np.int32), torch.int32) if any_gt else None
    d_gtb = t(np.concatenate(gtb), torch.float64) if any_gt else None
    d_gtd = t(np.concatenate(gtd), torch.float64) if any_gt else None
    o_xyz = torch.empty((M, 3), dtype=torch.float32, device=dev)
    o_ray = torch.empty((M, 4), dtype=torch.float32, device=dev)
    o_conf = torch.empty((M,), dtype=torch.float64, device=dev)
    o_uv = torch.empty((M, 6), dtype=torch.int32, device=dev)
    o_match = torch.empty((M,), dtype=torch.int32, device=dev)
    o_order = torch.empty((M,), dtype=torch.int32, device=dev)
    o_nm = torch.empty((len(live),), dtype=torch.int32, device=dev)
    o_xr = torch.zeros((M, 3), dtype=torch.float32, device=dev)
    p = lambda x: x.data_ptr() if x is not None else None  # noqa: E731
    a = L_.MlbPostArgs(len(live), max(det_off[i + 1] - det_off[i] for i in range(len(live))),
                       max(gt_off[i + 1] - gt_off[i] for i in range(len(live))), int(bool(reorder)), float(iou_min),
                       p(d_doff), p(d_goff), p(d_boxes), p(d_kps), p(d_kinv), p(d_dec), p(d_gtb), p(d_gtd), p(o_xyz),
                       p(o_ray), p(o_conf), p(o_uv), p(o_match), p(o_order), p(o_nm), p(o_xr))
    L_.check(lib.mlb_post_process(C.byref(a), _stream(dev)), 'mlb_post_process')
    xyz, conf, uv = o_xyz.cpu().numpy(), o_conf.cpu().numpy(), o_uv.cpu().numpy()
    match, order, nm, xr = o_match.cpu().numpy(), o_order.cpu().numpy(), o_nm.cpu().numpy(), o_xr.cpu().numpy()

    for li, i in enumerate(live):
        dic_in, bx, kp, kk, dic_gt = items[i]
        res = results[i]
        d0, m = det_off[li], det_off[li + 1] - det_off[li]
        n_match = int(nm[li])
        res['gt'] = [True] * n_match + [False] * (m - n_match)
        dd = np.asarray(dic_in['d'], dtype=np.float64).reshape(-1)
        bi = np.asarray(dic_in['bi'], dtype=np.float64).reshape(-1)
        epi = np.asarray(dic_in['epi'], dtype=np.float64).reshape(-1)
        has_yaw, has_aux = 'yaw' in dic_in, 'aux' in dic_in
        for pos in range(m):
            j = int(order[d0 + pos])
            res['boxes'].append(bx[j])
            res['confs'].append(float(conf[d0 + j]))
            res['dds_pred'].append(float(dd[j]))
            res['stds_ale'].append(float(bi[j]))
            res['stds_epi'].append(float(epi[j]))
            res['xyz_pred'].append(xyz[d0 + j].tolist())
            res['uv_kps'].append(kp[j])
            res['uv_centers'].append([int(uv[d0 + j, 0]), int(uv[d0 + j, 1])])
            res['uv_shoulders'].append([int(uv[d0 + j, 2]), int(uv[d0 + j, 3])])
            res['uv_heads'].append([int(uv[d0 + j, 4]), int(uv[d0 + j, 5])])
            res['angles']
            if not has_yaw:
                continue
            res['angles'].append(float(dic_in['yaw'][0][j]))
            res['angles_egocentric'].append(float(dic_in['yaw'][1][j]))
            res['aux']
            if has_aux:
                res['aux'].append(float(dic_in['aux'][j]))
        for pos in range(n_match):  # net.py:242-247, in the (re)ordered match order
            j = int(order[d0 + pos])
            jg = int(match[d0 + j])
            res['dds_real'].append(dic_gt['ys'][jg][3])
            res['boxes_gt'].append(dic_gt['boxes'][jg])
            res['xyz_real'].append(xr[d0 + j].tolist())
    return results


def kitti_rows_device(boxes, raw, dec, epi=None, net='monoloco_pp'):
    """eval/generate_kitti.py:202-253 for `net` in (monoloco_pp, monstereo): the 15 numbers of every label line, computed
    on the device from the forward's raw / decoded output tensors (CUDA, [n,out] / [n,8]) -> numpy [n, 15] fp64."""
    assert net in ('monoloco_pp', 'monstereo')
    lib = L_.lib()
    n = len(boxes)
    if n == 0:
        return np.zeros((0, 15))
    dev = raw.device
    d_boxes = torch.from_numpy(np.ascontiguousarray(np.asarray(boxes, dtype=np.float64).reshape(n, 5))).to(dev)
    d_epi = None
    if epi is not None and not isinstance(epi, list):
        d_epi = torch.as_tensor(epi, dtype=torch.float32).reshape(-1).to(dev).contiguous()
    elif isinstance(epi, list) and any(epi):
        d_epi = torch.tensor(epi, dtype=torch.float32, device=dev)
    rows = torch.empty((n, 15), dtype=torch.float64, device=dev)
    raw, dec = raw.contiguous(), dec.contiguous()
    L_.check(lib.mlb_kitti_rows(n, raw.shape[1], 0.035 if net == 'monoloco_pp' else 0.033, d_boxes.data_ptr(),
                                raw.data_ptr(), dec.data_ptr(), d_epi.data_ptr() if d_epi is not None else None,
                                rows.data_ptr(), _stream(dev)), 'mlb_kitti_rows')
    return rows.cpu().numpy()


# ------------------------------------------------------------------------------------------------ activity heuristics
_DRAW_TABLES = {}   # torch.device -> CUDA fp32 draw table (laplace_draw_table), grown on demand


def laplace_draw_table(n):
    """The draws behind the reference's social-distancing samples, as a table: T[k] = sign(u_k) * log1p(-|u_k|) for the
    first n values u of torch's seed-1 CPU stream `uniform_(eps - 1, 1)` (fp32).  laplace_sampling (process.py:101-122)
    reseeds with torch.manual_seed(1) on every call, so for an image of n people the S x n draws are
    dds[p] - |stds[p]| * T[s * n + p], bit for bit (Laplace.rsample computes loc - scale * u.sign() * log1p(-|u|)).  The
    stream is a prefix stream, so a longer table starts with every shorter one.  A private generator is used: the global
    CPU generator is left untouched.  torch computes log1p here because a device log1pf rounds differently."""
    g = torch.Generator().manual_seed(1)
    u = torch.empty(int(n), dtype=torch.float32).uniform_(torch.finfo(torch.float32).eps - 1, 1, generator=g)
    return u.sign() * torch.log1p(-u.abs())


def _draw_table(n, dev):
    t = _DRAW_TABLES.get(dev)
    if t is None or t.numel() < n:
        size = max(int(n), 6400, 2 * (t.numel() if t is not None else 0))
        t = _DRAW_TABLES[dev] = laplace_draw_table(size).to(dev)
    return t


def check_laplace_args(dds, stds):
    """Raise ValueError where the reference's torch.distributions.Laplace(dds, |stds|) would (fp32 values): a NaN
    distance or a scale that is not > 0 (zero, NaN, or too small for fp32)."""
    d = np.asarray(dds, dtype=np.float32).reshape(-1)
    s = np.abs(np.asarray(stds, dtype=np.float32).reshape(-1))
    if np.isnan(d).any():
        raise ValueError("social distance: a distance is NaN (Laplace loc must be real)")
    if not (s > 0).all():
        raise ValueError("social distance: a std is zero or NaN in fp32 (Laplace scale must be positive)")


def social_distance_device(xz, angles, dds, stds, img_off, *, threshold_prob, threshold_dist, radii, social_distance=False,
                           n_samples=100, max_people=None):
    """`social_interactions(idx, ...)` (activity.py:17-67) for every person of every image, in one launch
    (mlb_social_distance), flags identical to the reference's.  Device tensors in, a CUDA bool tensor [n] out, no host
    synchronisation.
      xz [n, 2] centres (x, z), angles [n] (fp64 on the device; other float dtypes are converted), dds [n], stds [n]
      (fp32, as torch.tensor(dds) makes them); people of all images concatenated, each image in its list order (the
      position selects the draw).  After LocoEngine.forward_images: xyzc[:, (0, 2)], dec[:, 5], dec[:, 3], dec[:, 4].
      img_off: CSR offsets [n_img + 1].  Host offsets (sequence, numpy, CPU tensor) are checked here and give the largest
      image; CUDA offsets need `max_people`, and the kernel clamps every image to it.
    The reference's validity check of Laplace(dds, stds) is not repeated here (it needs the values on the host):
    Loco.social_distance_batch does it."""
    lib = L_.lib()
    if not xz.is_cuda:
        raise ValueError("social_distance_device: inputs must be CUDA tensors")
    dev = xz.device
    n = xz.shape[0]
    if isinstance(img_off, torch.Tensor) and img_off.is_cuda:
        if max_people is None:
            raise ValueError("social_distance_device: max_people is required with device offsets")
        d_off = img_off.to(torch.int32).contiguous()
    else:
        off = np.asarray(img_off.cpu() if isinstance(img_off, torch.Tensor) else img_off, dtype=np.int64).reshape(-1)
        if off.size < 2 or off[0] != 0 or off[-1] != n or (np.diff(off) < 0).any():
            raise ValueError("social_distance_device: img_off must rise from 0 to %d" % n)
        if max_people is None:
            max_people = int(np.diff(off).max())
        d_off = torch.from_numpy(off.astype(np.int32)).to(dev, non_blocking=True)
    out = torch.empty((n,), dtype=torch.uint8, device=dev)
    radii = [float(r) for r in radii]
    a = L_.MlbSocialArgs()
    a.n_img, a.n_people, a.max_people, a.n_samples = d_off.numel() - 1, n, int(max_people), int(n_samples)
    a.n_radii, a.social_distance = len(radii), int(bool(social_distance))
    a.threshold_prob, a.threshold_dist = float(threshold_prob), float(threshold_dist)
    for i, r in enumerate(radii[:L_.SOCIAL_MAX_RADII]):
        a.radii[i] = r
    xz64 = xz.to(torch.float64).contiguous()
    ang64 = angles.to(torch.float64).contiguous()
    keep = [xz64, ang64]
    if n_samples >= 2:
        table = _draw_table(max(int(n_samples), 0) * min(max(int(max_people), 0), L_.SOCIAL_MAX_PEOPLE), dev)
        d32, s32 = dds.to(torch.float32).contiguous(), stds.to(torch.float32).contiguous()
        keep += [d32, s32]
        a.dds, a.stds, a.table, a.table_len = d32.data_ptr(), s32.data_ptr(), table.data_ptr(), table.numel()
    a.img_off, a.xz, a.angles, a.out = d_off.data_ptr(), xz64.data_ptr(), ang64.data_ptr(), out.data_ptr()
    L_.check(lib.mlb_social_distance(C.byref(a), _stream(dev)), 'mlb_social_distance')
    return out.view(torch.bool)


RAISING_HAND = (None, 'left', 'right', 'both')   # codes of mlb_raising_hand


def raising_hand_device(kps):
    """`is_raising_hand` (activity.py:70-117) for every pose: CUDA kps [n, 3, 17] (fp64 on the device) -> CUDA int8 codes
    [n] (0 None, 1 left, 2 right, 3 both; RAISING_HAND maps them back), one launch, no host synchronisation."""
    if not kps.is_cuda:
        raise ValueError("raising_hand_device: kps must be a CUDA tensor")
    k64 = kps.to(torch.float64).contiguous()
    n = k64.shape[0]
    if n and tuple(k64.shape[1:]) != (3, 17):
        raise ValueError("raising_hand_device: kps must be [n, 3, 17]")
    out = torch.empty((n,), dtype=torch.int8, device=kps.device)
    L_.check(L_.lib().mlb_raising_hand(k64.data_ptr(), n, out.data_ptr(), _stream(kps.device)), 'mlb_raising_hand')
    return out
