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
    dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    live = [i for i, it in enumerate(items) if it[0] is not None and len(it[1]) > 0]
    results = [defaultdict(list) for _ in items]
    if not live:
        return results
    det_off = [0]
    boxes, kps, kinv, dec = [], [], [], []
    for i in live:
        dic_in, bx, kp, kk, _ = items[i]
        m = len(bx)
        det_off.append(det_off[-1] + m)
        boxes.append(np.asarray(bx, dtype=np.float64).reshape(m, 5))
        kps.append(np.asarray(kp, dtype=np.float32).reshape(m, 3, 17))
        kinv.append(kinv_from_kk(kk))
        d = np.zeros((m, 8), dtype=np.float32)
        d[:, 3] = np.asarray(dic_in['d'], dtype=np.float32).reshape(-1)
        d[:, 4] = np.asarray(dic_in['bi'], dtype=np.float32).reshape(-1)
        dec.append(d)
    gt = gt_arrays([items[i][4] for i in live])
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(dev, dtype=dt)  # noqa: E731
    out = post_process_device(t(np.asarray(det_off, dtype=np.int32), torch.int32), t(np.concatenate(boxes), torch.float64),
                              t(np.concatenate(kps), torch.float32), t(np.stack(kinv), torch.float32),
                              t(np.concatenate(dec), torch.float32), max(np.diff(det_off)),
                              gt={k: torch.from_numpy(v).to(dev) if isinstance(v, np.ndarray) else v
                                  for k, v in gt.items()} if gt else None,
                              iou_min=iou_min, reorder=reorder)
    host = {k: v.cpu().numpy() for k, v in out.items()}
    for li, i in enumerate(live):
        dic_in, bx, kp, kk, dic_gt = items[i]
        a, b = det_off[li], det_off[li + 1]
        col = lambda v: np.asarray(v, dtype=np.float64).reshape(-1)  # noqa: E731
        yaw = (col(dic_in['yaw'][0]), col(dic_in['yaw'][1])) if 'yaw' in dic_in else None
        assemble_post(results[i], {k: host[k][a:b] for k in ('xyz', 'conf', 'uv', 'match', 'order', 'xyz_real')},
                      int(host['n_match'][li]), bx, kp, col(dic_in['d']), col(dic_in['bi']), col(dic_in['epi']), yaw,
                      col(dic_in['aux']) if 'aux' in dic_in else None, dic_gt)
    return results


def gt_arrays(dic_gt_list):
    """Ground truths of the images (dic_gt or None each) as the CSR arrays mlb_post_process reads: numpy gt_off [n_img + 1]
    int32, gt_boxes [n_gt, 4] fp64, gt_d [n_gt] fp64 (dic_gt['ys'][j][3]) and max_gt; None when no image has any."""
    gt_off, gtb, gtd = [0], [], []
    for dic_gt in dic_gt_list:
        g = len(dic_gt['boxes']) if dic_gt else 0
        if g:
            gtb.append(np.asarray(dic_gt['boxes'], dtype=np.float64).reshape(g, -1)[:, :4])
            gtd.append(np.asarray([y[3] for y in dic_gt['ys']], dtype=np.float64))
        gt_off.append(gt_off[-1] + g)
    if not gtb:
        return None
    return {'gt_off': np.asarray(gt_off, dtype=np.int32), 'gt_boxes': np.concatenate(gtb), 'gt_d': np.concatenate(gtd),
            'max_gt': int(np.diff(gt_off).max())}


def post_process_device(det_off, boxes, kps, kinv, dec, max_det, gt=None, iou_min=0.3, reorder=True):
    """`mlb_post_process` on device tensors, no host synchronisation: det_off [n_img + 1] int32 CSR, boxes [n, 5] fp64,
    kps [n, 3, 17] fp32, kinv [n_img, 9] fp32, dec [n, 8] fp32 (d at 3, bi at 4), max_det the largest image; gt the
    gt_arrays dictionary with its arrays as CUDA tensors, or None.  Returns CUDA tensors xyz [n, 3], conf [n], uv [n, 6],
    match [n] (image-local gt index or -1), order [n] (image-local detection at every output position), n_match [n_img]
    and xyz_real [n, 3]."""
    lib = L_.lib()
    dev = boxes.device
    n, n_img = boxes.shape[0], det_off.numel() - 1
    out = {'xyz': torch.empty((n, 3), dtype=torch.float32, device=dev),
           'ray': torch.empty((n, 4), dtype=torch.float32, device=dev),
           'conf': torch.empty((n,), dtype=torch.float64, device=dev),
           'uv': torch.empty((n, 6), dtype=torch.int32, device=dev),
           'match': torch.empty((n,), dtype=torch.int32, device=dev),
           'order': torch.empty((n,), dtype=torch.int32, device=dev),
           'n_match': torch.empty((n_img,), dtype=torch.int32, device=dev),
           'xyz_real': torch.zeros((n, 3), dtype=torch.float32, device=dev)}
    p = lambda x: x.data_ptr() if x is not None else None  # noqa: E731
    g = gt or {}
    a = L_.MlbPostArgs(n_img, int(max_det), int(g.get('max_gt', 0)), int(bool(reorder)), float(iou_min), p(det_off),
                       p(g.get('gt_off')), p(boxes), p(kps), p(kinv), p(dec), p(g.get('gt_boxes')), p(g.get('gt_d')),
                       p(out['xyz']), p(out['ray']), p(out['conf']), p(out['uv']), p(out['match']), p(out['order']),
                       p(out['n_match']), p(out['xyz_real']))
    L_.check(lib.mlb_post_process(C.byref(a), _stream(dev)), 'mlb_post_process')
    del out['ray']
    return out


def assemble_post(res, dev, n_match, boxes, keypoints, dd, bi, epi, yaw, aux, dic_gt):
    """Fill `res` (a defaultdict(list)) for one image of m >= 1 detections with the keys, key order and values of
    net.py:164-248.  dev: that image's rows of post_process_device's outputs as numpy arrays (image-local); boxes /
    keypoints the caller's lists (their elements are placed in the result as they are); dd, bi, epi fp64 columns by
    detection; yaw (angles, egocentric angles) or None; aux or None."""
    o = dev['order'].astype(np.int64)
    m = len(o)
    res['gt'] = [True] * n_match + [False] * (m - n_match)
    res['boxes'] = [boxes[j] for j in o]
    res['confs'] = dev['conf'][o].tolist()
    res['dds_pred'] = dd[o].tolist()
    res['stds_ale'] = bi[o].tolist()
    res['stds_epi'] = epi[o].tolist()
    res['xyz_pred'] = dev['xyz'][o].tolist()
    res['uv_kps'] = [keypoints[j] for j in o]
    uv = dev['uv'][o]
    res['uv_centers'], res['uv_shoulders'], res['uv_heads'] = uv[:, 0:2].tolist(), uv[:, 2:4].tolist(), uv[:, 4:6].tolist()
    res['angles']  # the reference's defaultdict access creates these keys even when the value is missing
    if yaw is not None:
        res['angles'] = yaw[0][o].tolist()
        res['angles_egocentric'] = yaw[1][o].tolist()
        res['aux']
        if aux is not None:
            res['aux'] = aux[o].tolist()
    if n_match:  # net.py:242-247, in the (re)ordered match order
        om = o[:n_match]
        jg = dev['match'][om].tolist()
        res['dds_real'] = [dic_gt['ys'][k][3] for k in jg]
        res['boxes_gt'] = [dic_gt['boxes'][k] for k in jg]
        res['xyz_real'] = dev['xyz_real'][om].tolist()
    return res


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
