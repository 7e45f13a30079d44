"""Reference-facing helpers of monoloco/network/process.py, backed by the CUDA kernels.

preprocess_monoloco / preprocess_monstereo / extract_outputs / unnormalize_bi / filter_outputs keep the
reference's names, argument meaning and error behaviour (asserts) but run on the GPU through
libmonoloco_b200.so; the host-side list munging (pifpaf json -> lists, calibration yaml) is plain Python.
"""
import ctypes as C
import json
import math
import os

import numpy as np
import torch

from .. import _lib as L_
from ..engine import preprocess_device

Sx, Sy = 7.2, 5.4  # nuScenes sensor size in mm (process.py:21-22)

# camera intrinsics of the reference (monoloco/network/intrinsics.yaml:1-21)
INTRINSICS = {
    'kitti': {'intrinsics': [[718.3351, 0., 600.3891], [0., 718.3351, 181.5122], [0., 0., 1.]], 'im_size': [1238, 374]},
    'wv': {'intrinsics': [[1070.9498, 0., 987.4846], [0., 1070.726, 605.5297], [0., 0., 1.]], 'im_size': [1920, 1200]},
    'nuscenes': {'intrinsics': [[1070.9498, 0., 987.4846], [0., 1070.726, 605.5297], [0., 0., 1.]],
                 'im_size': [1600, 900]},
}


def _cuda(t):
    if isinstance(t, (list, np.ndarray)):
        t = torch.tensor(t, dtype=torch.float32)
    if not t.is_cuda:
        if not torch.cuda.is_available():
            raise RuntimeError("monoloco_b200: no CUDA device -- the hot path has no CPU fallback")
        t = t.cuda()
    return t.float()


def preprocess_monoloco(keypoints, kk, zero_center=False):
    """process.py:47-67: (m,3,17) pixel keypoints + K -> (m,34) metres at z=10, on the GPU (mlb_preprocess)."""
    kps = _cuda(keypoints)
    assert kps.dim() == 3 and kps.shape[1] == 3 and kps.shape[2] == 17, "tensor dimensions not recognized"
    return preprocess_device(kps, kk, zero_center=zero_center)


def preprocess_monstereo(keypoints, keypoints_r, kk):
    """process.py:25-44: all-vs-all rows cat(l, l - r) -> ((L*R, 68), clusters).  (The fused forward builds these
    rows inside the kernel and never materialises them; this stand-alone form exists for dataset preparation.)"""
    inputs_l = preprocess_monoloco(keypoints, kk)
    inputs_r = preprocess_monoloco(keypoints_r, kk)
    n_l, n_r = inputs_l.shape[0], inputs_r.shape[0]
    left = inputs_l.repeat_interleave(n_r, dim=0)
    right = inputs_r.repeat(n_l, 1)
    return torch.cat((left, left - right), dim=1), [n_r] * n_l


def unnormalize_bi(loc):
    """process.py:125-133."""
    assert loc.size()[1] == 2, "size of the output tensor should be (m, 2)"
    return torch.exp(loc[:, 1:2]) * loc[:, 0:1]


def extract_outputs(outputs, tasks=()):
    """process.py:231-278.  With `tasks` returns the raw column views used by the losses; without, the decoded
    dictionary of CPU tensors.  The decode itself (spherical -> xyz, bi, yaw) is what the fused kernel's epilogue
    computes; for a raw [m,9|10] tensor handed in from outside it is re-done here with the same op order."""
    dic_out = {'x': outputs[:, 0:1], 'y': outputs[:, 1:2], 'd': outputs[:, 2:4], 'h': outputs[:, 4:5],
               'w': outputs[:, 5:6], 'l': outputs[:, 6:7], 'ori': outputs[:, 7:9]}
    if outputs.shape[1] == 10:
        dic_out['aux'] = outputs[:, 9:10]
    if len(tasks) >= 1:
        assert isinstance(tasks, tuple), "tasks need to be a tuple"
        return [dic_out[task] for task in tasks]
    from ..engine import decode_device
    return decode_device(outputs)


def extract_labels_aux(labels, tasks=None):
    """process.py:281-290."""
    dic = {'aux': labels[:, 0:1]}
    if tasks is not None:
        assert isinstance(tasks, tuple), "tasks need to be a tuple"
        return [dic[t] for t in tasks]
    return {k: v.detach().cpu() for k, v in dic.items()}


def extract_labels(labels, tasks=None):
    """process.py:293-304."""
    dic = {'x': labels[:, 0:1], 'y': labels[:, 1:2], 'z': labels[:, 2:3], 'd': labels[:, 3:4], 'h': labels[:, 4:5],
           'w': labels[:, 5:6], 'l': labels[:, 6:7], 'ori': labels[:, 7:9], 'aux': labels[:, 10:11]}
    if tasks is not None:
        assert isinstance(tasks, tuple), "tasks need to be a tuple"
        return [dic[t] for t in tasks]
    return {k: v.detach().cpu() for k, v in dic.items()}


def cluster_outputs(outputs, clusters):
    """process.py:307-316."""
    if clusters == 0:
        clusters = max(1, round(outputs.shape[0] / 2))
    assert outputs.shape[0] % clusters == 0, "Unexpected number of inputs"
    return outputs.view(-1, clusters, outputs.shape[1])


def load_calibration(calibration, im_size, focal_length=5.7):
    """process.py:70-86."""
    if calibration == 'custom':
        return [[im_size[0] * focal_length / Sx, 0., im_size[0] / 2],
                [0., im_size[1] * focal_length / Sy, im_size[1] / 2],
                [0., 0., 1.]]
    cfg = INTRINSICS[calibration]
    kk = [list(r) for r in cfg['intrinsics']]
    scale = [size / orig for size, orig in zip(im_size, cfg['im_size'])]
    kk[0] = [el * scale[0] for el in kk[0]]
    kk[1] = [el * scale[1] for el in kk[1]]
    return kk


def factory_for_gt(path_gt, name=None):
    """process.py:89-98."""
    assert os.path.exists(path_gt), "Ground-truth file not found"
    with open(path_gt, 'r') as f:
        dic_names = json.load(f)
    return dic_names[name], dic_names[name]['K']


def prepare_pif_kps(kps_in):
    """process.py:208-216: flat list of 51 -> [xs, ys, confs]."""
    assert len(kps_in) % 3 == 0, "keypoints expected as a multiple of 3"
    return [kps_in[0:][::3], kps_in[1:][::3], kps_in[2:][::3]]


def preprocess_pifpaf(annotations, im_size=None, enlarge_boxes=True, min_conf=0.):
    """process.py:155-205: pifpaf annotations -> (boxes [x1,y1,x2,y2,conf], keypoints [3][17])."""
    boxes, keypoints = [], []
    enlarge = 1 if enlarge_boxes else 2
    for dic in annotations:
        kps = prepare_pif_kps(dic['keypoints'])
        box = list(dic['bbox'])
        if 'score' in dic:
            conf = dic['score']
            delta_h = box[3] / (10 * enlarge)
            delta_w = box[2] / (5 * enlarge)
            box[2] += box[0]
            box[3] += box[1]
        else:
            conf = float(np.mean(np.array(kps[2])))
            delta_h = (box[3] - box[1]) / (7 * enlarge)
            delta_w = (box[2] - box[0]) / (3.5 * enlarge)
            assert delta_h > -5 and delta_w > -5, "Bounding box <=0"
        box[0] -= delta_w
        box[1] -= delta_h
        box[2] += delta_w
        box[3] += delta_h
        if im_size is not None:
            box[0] = max(0, box[0])
            box[1] = max(0, box[1])
            box[2] = min(box[2], im_size[0])
            box[3] = min(box[3], im_size[1])
        if conf >= min_conf:
            box.append(conf)
            boxes.append(box)
            keypoints.append(kps)
    return boxes, keypoints


# ------------------------------------------------------------------------------------------------ many images on the device
PIFPAF_FIELDS = (('kps', np.float64), ('bbox', np.float64), ('score', np.float64), ('im_size', np.float64),
                 ('ann_off', np.int32), ('has_score', np.uint8), ('has_size', np.uint8))


def check_pifpaf_options(enlarge_boxes, min_conf):
    """(enlarge, min_conf) as mlb_preprocess_pifpaf takes them; ValueError for a non-bool enlarge_boxes or a min_conf
    that is not a finite number."""
    if not isinstance(enlarge_boxes, (bool, np.bool_)):
        raise ValueError("enlarge_boxes must be True or False")
    try:
        mc = float(min_conf)
    except (TypeError, ValueError):
        raise ValueError("min_conf must be a finite number") from None
    if not math.isfinite(mc):
        raise ValueError("min_conf must be a finite number")
    return (1 if enlarge_boxes else 2), mc


def pack_pifpaf(annotations_list, im_size_list):
    """pifpaf annotations of many images -> the numpy arrays mlb_preprocess_pifpaf reads (PIFPAF_FIELDS): ann_off
    [n_img + 1] CSR, kps [n, 51] and bbox [n, 4] fp64, score [n] with has_score [n] (the 'score' key), im_size [n_img, 2]
    with has_size [n_img] (None: no clamping).  The annotation dictionaries are only read."""
    n_img = len(annotations_list)
    if len(im_size_list) != n_img:
        raise ValueError("one image size (or None) per image: %d for %d images" % (len(im_size_list), n_img))
    counts = [len(a) for a in annotations_list]
    anns = [d for a in annotations_list for d in a]
    n = len(anns)
    try:
        kps = np.asarray([d['keypoints'] for d in anns], dtype=np.float64).reshape(n, -1) if n else np.zeros((0, 51))
        bbox = np.asarray([d['bbox'] for d in anns], dtype=np.float64).reshape(n, -1) if n else np.zeros((0, 4))
    except (KeyError, TypeError, ValueError) as e:
        raise ValueError("every annotation needs 'keypoints' (51 numbers) and 'bbox' (4 numbers): %s" % e) from None
    if kps.shape[1] != 51 or bbox.shape[1] != 4:
        raise ValueError("every annotation needs 'keypoints' (51 numbers) and 'bbox' (4 numbers)")
    has_score = np.fromiter(('score' in d for d in anns), dtype=np.uint8, count=n)
    score = np.asarray([d['score'] if 'score' in d else 0.0 for d in anns], dtype=np.float64).reshape(n)
    im_size = np.zeros((n_img, 2), dtype=np.float64)
    has_size = np.zeros(n_img, dtype=np.uint8)
    for i, sz in enumerate(im_size_list):
        if sz is not None:
            if len(sz) != 2:
                raise ValueError("image size %d: (width, height) or None" % i)
            im_size[i] = (float(sz[0]), float(sz[1]))
            has_size[i] = 1
    ann_off = np.zeros(n_img + 1, dtype=np.int64)
    np.cumsum(counts, out=ann_off[1:])
    if ann_off[-1] > np.iinfo(np.int32).max:
        raise ValueError("more than 2^31 - 1 annotations")
    return {'kps': kps, 'bbox': bbox, 'score': score, 'im_size': im_size, 'ann_off': ann_off.astype(np.int32),
            'has_score': has_score, 'has_size': has_size}


def pifpaf_layout(packs):
    """Byte layout of several packs (pack_pifpaf) in one buffer: list of {field: (byte offset, shape, numpy dtype)} per
    pack, and the total size.  Every field starts on an 8-byte boundary."""
    out, pos = [], 0
    for p in packs:
        lay = {}
        for name, dt in PIFPAF_FIELDS:
            a = p[name]
            lay[name] = (pos, a.shape, np.dtype(dt))
            pos += -(-a.size * np.dtype(dt).itemsize // 8) * 8
        out.append(lay)
    return out, max(pos, 8)


def preprocess_pifpaf_device(arrays, n_img, n_ann, enlarge, min_conf):
    """mlb_preprocess_pifpaf on device tensors (`arrays`: the PIFPAF_FIELDS of one pack as CUDA tensors), no host
    synchronisation.  Returns CUDA tensors boxes [n_ann, 5] fp64, kps [n_ann, 3, 17] fp64, kps32 fp32, src [n_ann],
    kept_off [n_img + 1] and error [1]; rows beyond kept_off[-1] are unused."""
    dev = arrays['kps'].device
    e = lambda shape, dt: torch.empty(shape, dtype=dt, device=dev)  # noqa: E731
    out = {'boxes': e((n_ann, 5), torch.float64), 'kps': e((n_ann, 3, 17), torch.float64),
           'kps32': e((n_ann, 3, 17), torch.float32), 'src': e((n_ann,), torch.int32),
           'kept_off': e((n_img + 1,), torch.int32), 'error': e((1,), torch.int32)}
    scratch = e((n_img + 1,), torch.int64)
    p = lambda t: t.data_ptr() if t.numel() else None  # noqa: E731
    a = L_.MlbPifpafArgs()
    a.n_img, a.n_ann, a.enlarge, a.min_conf = n_img, n_ann, enlarge, min_conf
    a.ann_off, a.kps, a.bbox, a.score = p(arrays['ann_off']), p(arrays['kps']), p(arrays['bbox']), p(arrays['score'])
    a.has_score, a.im_size, a.has_size = p(arrays['has_score']), p(arrays['im_size']), p(arrays['has_size'])
    a.out_boxes, a.out_kps, a.out_kps32, a.out_src = p(out['boxes']), p(out['kps']), p(out['kps32']), p(out['src'])
    a.kept_off, a.error, a.scratch = p(out['kept_off']), p(out['error']), p(scratch)
    L_.check(L_.lib().mlb_preprocess_pifpaf(C.byref(a), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
             'mlb_preprocess_pifpaf')
    return out
