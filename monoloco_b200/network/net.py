"""
`Loco` -- the drop-in for monoloco/network/net.py:23-133 (same constructor, `forward`, `post_process`,
attributes), running pre-process + network + decode as one fused CUDA kernel per image.

Differences that are deliberate and documented (INTEGRATION.md):
  * the result tensors are produced on the GPU and returned as CPU float32 tensors, exactly the dict layout
    callers index (`dic_out['xyzd'][:, 0:3]`, `dic_out['yaw'][0][idx]`, ...), plus one extra key `xyz_c` =
    xyz_from_distance(d, bbox-centre ray) that `post_process` reuses;
  * MC-dropout epistemic std uses an in-kernel counter RNG + inverse-CDF Laplace sampling instead of torch's
    reseeded generator (equal in distribution, not sample-for-sample);
  * there is no CPU mode: `device=None` selects the current CUDA device.
"""
from collections import defaultdict

import torch

from .. import _lib as L_
from ..engine import dec_to_dict
from ..utils import get_iou_matches, reorder_matches, get_keypoints, pixel_to_camera, xyz_from_distance
from ..activity import social_interactions, is_raising_hand
from .architectures import MonolocoModel, LocoModel


class Loco:
    """Class for both MonoLoco and MonStereo (net.py:23-81)."""
    LINEAR_SIZE_MONO = 256
    N_SAMPLES = 100

    def __init__(self, model, mode, net=None, device=None, n_dropout=0, p_dropout=0.2, linear_size=1024):
        assert mode in ('mono', 'stereo'), "mode not recognized"
        self.mode = mode
        if net is None:
            self.net = 'monoloco_pp' if mode == 'mono' else 'monstereo'
        else:
            # net.py:41-44 is unreachable in the reference (reads self.net before assignment); here the documented
            # intent is implemented: legacy nets are mono-only
            assert net in ('monstereo', 'monoloco', 'monoloco_p', 'monoloco_pp')
            if net != 'monstereo':
                assert mode == 'mono', "Assert arguments mode and net are in conflict"
            self.net = net

        if self.net == 'monstereo':
            input_size, output_size = 68, 10
        elif self.net == 'monoloco_p':
            input_size, output_size, linear_size = 34, 9, 256
        elif self.net == 'monoloco_pp':
            input_size, output_size = 34, 9
        else:
            input_size, output_size = 34, 2

        if not torch.cuda.is_available():
            raise RuntimeError("monoloco_b200.Loco needs a CUDA device (H100); there is no CPU fallback")
        self.device = torch.device('cuda', torch.cuda.current_device()) if not device else torch.device(device)
        if self.device.type != 'cuda':
            raise RuntimeError("monoloco_b200.Loco runs on CUDA devices only")
        self.n_dropout = n_dropout
        self.epistemic = bool(self.n_dropout > 0)

        if isinstance(model, str):
            if self.net in ('monoloco', 'monoloco_p'):
                self.model = MonolocoModel(p_dropout=p_dropout, input_size=input_size, linear_size=linear_size,
                                           output_size=output_size)
            else:
                self.model = LocoModel(p_dropout=p_dropout, input_size=input_size, output_size=output_size,
                                       linear_size=linear_size, device=self.device)
            self.model.load_state_dict(torch.load(model, map_location=lambda storage, loc: storage))
        else:
            self.model = model
        self.model.eval()
        self.model.to(self.device)

    # ------------------------------------------------------------------------------------------- forward
    def forward(self, keypoints, kk, keypoints_r=None):
        """net.py:83-133: keypoints [m][3][17] lists (+ right keypoints for stereo) -> dict of CPU tensors."""
        if not keypoints:
            return None
        eng = self.model.engine()
        with torch.no_grad():
            if self.net == 'monstereo':
                kps = torch.tensor(keypoints, dtype=torch.float32).to(self.device)
                if keypoints_r:
                    kps_r = torch.tensor(keypoints_r, dtype=torch.float32).to(self.device)
                else:
                    kps_r = kps[0:1, :].clone()  # net.py:115-116
                out = eng.forward(kps, x_right=kps_r, kk=kk, kind=L_.IN_KPS_STEREO, want_xyzc=True)
                raw, dec, xyzc = eng.stereo_filter_host(out['raw'], out['dec'], out['xyzc'], kps.shape[0],
                                                        kps_r.shape[0])  # process.py:307-327, one sync
                dic_out = dec_to_dict(raw, dec, stereo=True)
                dic_out['xyz_c'] = xyzc[:, 0:3]
                n_out = kps.shape[0]  # net.py:130: outputs is the clustered 3-D tensor -> number of left poses
                inputs = None
            elif not self.epistemic and self.net != 'monoloco':
                # per-image fast path: one C call does H2D (pinned staging), the fused kernel, D2H and the sync
                out = self._forward_host_mono(eng, keypoints, kk)
                raw, dec = out['raw'], out['dec']
                if self.net == 'monoloco_p':
                    r, d = raw, dec
                    dic_out = {'xyz': r[:, 0:3], 'zb': r[:, 2:4], 'h': r[:, 4:5], 'w': r[:, 5:6], 'l': r[:, 6:7],
                               'ori': r[:, 7:9], 'xyzd': d[:, 0:4], 'd': d[:, 3:4], 'bi': d[:, 4:5],
                               'yaw': (d[:, 5:6], d[:, 6:7])}
                else:
                    dic_out = dec_to_dict(raw, dec, stereo=False)
                dic_out['xyz_c'] = out['xyzc'][:, 0:3]
                dic_out['epi'] = [0.] * raw.shape[0]
                return dic_out
            else:
                kps = torch.tensor(keypoints, dtype=torch.float32).to(self.device)
                zero_center = self.net == 'monoloco'
                out = eng.forward(kps, kk=kk, kind=L_.IN_KPS, want_xyzc=True, want_x=self.epistemic,
                                  zero_center=zero_center)
                raw, dec = out['raw'], out['dec']
                if self.net == 'monoloco':
                    dic_out = {'d': raw[:, 0:1].cpu(), 'bi': dec[:, 4:5].cpu()}  # net.py:95-100
                elif self.net == 'monoloco_p':
                    r, d = raw.cpu(), dec.cpu()  # extract_outputs_mono, process.py:330-360
                    dic_out = {'xyz': r[:, 0:3], 'zb': r[:, 2:4], 'h': r[:, 4:5], 'w': r[:, 5:6], 'l': r[:, 6:7],
                               'ori': r[:, 7:9], 'xyzd': d[:, 0:4], 'd': d[:, 3:4], 'bi': d[:, 4:5],
                               'yaw': (d[:, 5:6], d[:, 6:7])}
                else:
                    dic_out = dec_to_dict(raw, dec, stereo=False)
                dic_out['xyz_c'] = out['xyzc'][:, 0:3].cpu()
                n_out = raw.shape[0]
                inputs = out.get('x')
            if self.n_dropout > 0 and self.net != 'monstereo':
                dic_out['epi'] = self.epistemic_uncertainty(inputs)
            else:
                dic_out['epi'] = [0.] * n_out
        return dic_out

    def forward_batch(self, keypoints_list, kk_list, keypoints_r_list=None):
        """Loco.forward over many images with ONE network launch (plus two for the monstereo filter): image i gets the dict
        forward(keypoints_list[i], kk_list[i], keypoints_r_list[i]) returns, or None when it has no detections
        (net.py:88-89).  Inputs are staged through pinned memory, every copy back is asynchronous and the call ends in
        one stream synchronisation.  MC-dropout epistemic std (mono nets) adds one launch for all images' passes."""
        import numpy as np
        from ..engine import image_offsets
        n_img = len(keypoints_list)
        if len(kk_list) != n_img:
            raise ValueError("forward_batch: one camera matrix per image")
        n_l = [len(k) for k in keypoints_list]
        res = [None] * n_img
        if sum(n_l) == 0:
            return res
        eng = self.model.engine()
        stereo = self.net == 'monstereo'
        with torch.no_grad():
            kps_h = self._pinned('b_kps', (sum(n_l), 3, 17), torch.float32)
            kps_h.copy_(torch.from_numpy(np.concatenate([np.asarray(k, dtype=np.float32).reshape(-1, 3, 17)
                                                         for k in keypoints_list if len(k)])))
            kps = kps_h.to(self.device, non_blocking=True)
            if stereo:
                rights = []
                for i, k in enumerate(keypoints_list):
                    kr = keypoints_r_list[i] if keypoints_r_list is not None else None
                    if not len(k):
                        rights.append(np.zeros((0, 3, 17), dtype=np.float32))
                    elif kr is None or not len(kr):
                        rights.append(np.asarray(k[0:1], dtype=np.float32).reshape(1, 3, 17))  # net.py:115-116
                    else:
                        rights.append(np.asarray(kr, dtype=np.float32).reshape(-1, 3, 17))
                n_r = [r.shape[0] for r in rights]
                kr_h = self._pinned('b_kps_r', (sum(n_r), 3, 17), torch.float32)
                kr_h.copy_(torch.from_numpy(np.concatenate(rights)))
                kps_r = kr_h.to(self.device, non_blocking=True)
                left_off, right_off = image_offsets(n_l), image_offsets(n_r)
                row_off = image_offsets([a * b for a, b in zip(n_l, n_r)])
                out = eng.forward_images(kps, row_off, kk_list, kind=L_.IN_KPS_STEREO, x_right=kps_r, left_off=left_off,
                                         right_off=right_off, want_xyzc=True)
                sel = eng.stereo_filter_images(out['raw'], out['dec'], row_off, left_off, right_off, xyzc=out['xyzc'],
                                               trim=False)  # process.py:307-327 per image
                dev = {'raw': sel['sel_raw'], 'dec': sel['sel_dec'], 'xyzc': sel['sel_xyzc'], 'off': sel['sel_img_off']}
            else:
                row_off = image_offsets(n_l)
                zc = self.net == 'monoloco'
                out = eng.forward_images(kps, row_off, kk_list, kind=L_.IN_KPS, want_xyzc=True, zero_center=zc)
                dev = {'raw': out['raw'], 'dec': out['dec'], 'xyzc': out['xyzc']}
                if self.n_dropout > 0:
                    dev['epi'] = eng.epistemic_std(kps, self.n_dropout, n_samples=self.N_SAMPLES, seed=1, row_off=row_off,
                                                   kk_list=kk_list, zero_center=zc)
            host = {}
            for k, v in dev.items():
                host[k] = self._pinned('b_' + k, tuple(v.shape), v.dtype)
                host[k].copy_(v, non_blocking=True)
            torch.cuda.current_stream(self.device).synchronize()
        eng.check_error()
        off = host['off'].tolist() if stereo else row_off.tolist()
        for i in range(n_img):
            if not n_l[i]:
                continue
            a, b = off[i], off[i + 1]
            raw, dec = host['raw'][a:b].clone(), host['dec'][a:b].clone()
            if stereo:
                dic = dec_to_dict(raw, dec, stereo=True)
            elif self.net == 'monoloco':
                dic = {'d': raw[:, 0:1], 'bi': dec[:, 4:5]}  # net.py:95-100
            elif self.net == 'monoloco_p':
                dic = {'xyz': raw[:, 0:3], 'zb': raw[:, 2:4], 'h': raw[:, 4:5], 'w': raw[:, 5:6], 'l': raw[:, 6:7],
                       'ori': raw[:, 7:9], 'xyzd': dec[:, 0:4], 'd': dec[:, 3:4], 'bi': dec[:, 4:5],
                       'yaw': (dec[:, 5:6], dec[:, 6:7])}  # extract_outputs_mono, process.py:330-360
            else:
                dic = dec_to_dict(raw, dec, stereo=False)
            dic['xyz_c'] = host['xyzc'][a:b, 0:3].clone()
            dic['epi'] = host['epi'][a:b].clone() if 'epi' in host else [0.] * n_l[i]
            res[i] = dic
        return res

    def predict_batch(self, annotations_list, kk_list, im_size_list, *, annotations_r_list=None, dic_gt_list=None,
                      enlarge_boxes=False, min_conf=0., iou_min=0.3, reorder=True, activities=(), args=None):
        """The reference's per-image predict chain (predict.py:226-240, eval/eval_activity.py:173-179) for many images:
        res[i] = (boxes, keypoints, dic_out) of
            boxes, keypoints = preprocess_pifpaf(annotations_list[i], im_size_list[i], enlarge_boxes, min_conf)
            dic_out = post_process(forward(keypoints, kk_list[i][, keypoints_r]), boxes, keypoints, kk_list[i], dic_gt_list[i],
                                   iou_min, reorder)
            then social_distance(dic_out, args) if 'social_distance' in activities, raising_hand(dic_out, keypoints) if
            'raise_hand' in activities,
        with keypoints_r from preprocess_pifpaf(annotations_r_list[i], im_size_list[i]) in stereo (predict.py:244).
        Every stage is a device launch over all images: the pre-process (mlb_preprocess_pifpaf, left and right), the
        network (forward_images, the stereo filter, MC-dropout when n_dropout > 0), mlb_post_process, social distancing
        on the people in post-processed order and raised hands on the kept key points in caller order.  The annotations
        go up in one copy; the host waits twice: for the kept counts (they size the network launch) and for the results.
        The annotation dictionaries are not modified.  Raises AssertionError for the reference's degenerate-box assert
        (nothing after the pre-process is launched) and ValueError for bad arguments or where the reference's Laplace
        constructor would fail in social_distance."""
        import numpy as np
        from ..engine import image_offsets, kinv_images
        from .process import check_pifpaf_options, pack_pifpaf, pifpaf_layout, preprocess_pifpaf_device
        from .post import (post_process_device, gt_arrays, assemble_post, social_distance_device, raising_hand_device,
                           check_laplace_args, RAISING_HAND)
        n_img = len(annotations_list)
        if len(kk_list) != n_img or len(im_size_list) != n_img:
            raise ValueError("predict_batch: one camera matrix and one image size (or None) per image")
        if dic_gt_list is not None and len(dic_gt_list) != n_img:
            raise ValueError("predict_batch: one ground truth (or None) per image")
        stereo = self.net == 'monstereo'
        if annotations_r_list is not None and (not stereo or len(annotations_r_list) != n_img):
            raise ValueError("predict_batch: annotations_r_list is for stereo, one list per image")
        enlarge, min_conf = check_pifpaf_options(enlarge_boxes, min_conf)
        acts = tuple(activities)
        if set(acts) - {'social_distance', 'raise_hand'}:
            raise ValueError("predict_batch: activities are 'social_distance' and 'raise_hand'")
        want_sd, want_rh = 'social_distance' in acts, 'raise_hand' in acts
        if want_sd and (args is None or self.net == 'monoloco'):
            raise ValueError("predict_batch: social_distance needs args and a net with orientation outputs")
        packs = [pack_pifpaf(annotations_list, im_size_list)]
        if stereo:
            packs.append(pack_pifpaf(annotations_r_list if annotations_r_list is not None else [[]] * n_img, im_size_list))
        gt = gt_arrays(dic_gt_list) if dic_gt_list is not None else None

        def finish(res, flags=None, codes=None):   # social_distance / raising_hand in the reference's order
            if want_sd:
                res['angles'], res['dds_pred'], res['stds_ale'], res['xyz_pred']  # noqa: B018  (the reads create the keys)
                res['social_distance'] = flags if flags is not None else []
            if want_rh:
                res['raising_hand'] = codes if codes is not None else []
            return res

        if n_img == 0:
            return []
        if sum(int(p['ann_off'][-1]) for p in packs) == 0:
            return [([], [], finish(defaultdict(list))) for _ in range(n_img)]
        dev, eng = self.device, self.model.engine()
        with torch.no_grad():
            # ---- one upload of everything the pre-process reads, the pre-process, one read-back of the kept counts
            lays, nbytes = pifpaf_layout(packs)
            h_in = _pinned_host('pb_in', (nbytes,), torch.uint8)
            hn = h_in.numpy()
            for p, lay in zip(packs, lays):
                for name, (o, shape, dt) in lay.items():
                    a = np.ascontiguousarray(p[name], dtype=dt).reshape(-1).view(np.uint8)
                    hn[o:o + a.size] = a
            d_in = h_in.to(dev, non_blocking=True)
            tdt = {np.dtype(np.float64): torch.float64, np.dtype(np.int32): torch.int32, np.dtype(np.uint8): torch.uint8}
            pre = []
            for k, (p, lay) in enumerate(zip(packs, lays)):
                arrays = {name: d_in[o:o + int(np.prod(shape)) * dt.itemsize].view(tdt[dt]).view(shape)
                          for name, (o, shape, dt) in lay.items()}
                pre.append(preprocess_pifpaf_device(arrays, n_img, p['kps'].shape[0], *((enlarge, min_conf) if k == 0 else
                                                                                      (1, 0.))))
            h_rb = _pinned_host('pb_rb', (len(pre), n_img + 2), torch.int32)
            for k, o in enumerate(pre):
                h_rb[k, :n_img + 1].copy_(o['kept_off'], non_blocking=True)
                h_rb[k, n_img + 1:].copy_(o['error'], non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
            rb = h_rb.numpy().astype(np.int64)
            if (rb[:, -1] & L_.PIFPAF_ERR_TIMEOUT).any():
                raise RuntimeError("mlb_preprocess_pifpaf: the kept-offset scan timed out")
            if (rb[:, -1] & L_.PIFPAF_ERR_BOX).any():
                raise AssertionError("Bounding box <=0")
            koff = rb[0, :n_img + 1]
            n_l = np.diff(koff)
            n = int(koff[-1])
            if n == 0:
                return [([], [], finish(defaultdict(list))) for _ in range(n_img)]

            # ---- network
            kps32 = pre[0]['kps32'][:n]
            epi = None
            if stereo:
                n_r = np.diff(rb[1, :n_img + 1])
                n_re = np.where(n_l > 0, np.maximum(n_r, 1), 0)   # no right poses: the first left pose (net.py:115-116)
                n_rt = int(rb[1, n_img])
                src = np.concatenate([np.arange(rb[1, i], rb[1, i + 1]) if n_r[i] else [n_rt + koff[i]]
                                      for i in range(n_img) if n_l[i]]).astype(np.int64)
                x_right = torch.cat((pre[1]['kps32'][:n_rt], kps32)).index_select(0, torch.from_numpy(src).to(dev))
                row_off, right_off = image_offsets(n_l * n_re), image_offsets(n_re)
                out = eng.forward_images(kps32, row_off, kk_list, kind=L_.IN_KPS_STEREO, x_right=x_right, left_off=koff,
                                         right_off=right_off, want_xyzc=True)
                sel = eng.stereo_filter_images(out['raw'], out['dec'], row_off, koff, right_off, xyzc=out['xyzc'], trim=False)
                # post_process reads the first n_l rows of every image's filtered outputs (net.py:195-201)
                img = np.repeat(np.arange(n_img), n_l)
                local = np.arange(n) - koff[img]
                rows = torch.from_numpy(np.stack((img, local))).to(dev)
                gidx = (sel['sel_img_off'].long()[rows[0]] + rows[1]).clamp_(max=max(out['raw'].shape[0] - 1, 0))
                dec = sel['sel_dec'].index_select(0, gidx)
            else:
                zc = self.net == 'monoloco'
                dec = eng.forward_images(kps32, koff, kk_list, kind=L_.IN_KPS, want_xyzc=True, zero_center=zc)['dec']
                if self.n_dropout > 0:
                    epi = eng.epistemic_std(kps32, self.n_dropout, n_samples=self.N_SAMPLES, seed=1, row_off=koff,
                                            kk_list=kk_list, zero_center=zc)

            # ---- post-process, activities
            up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev, non_blocking=True)  # noqa: E731
            gt_dev = {k: up(v) if isinstance(v, np.ndarray) else v for k, v in gt.items()} if gt else None
            dev_out = post_process_device(pre[0]['kept_off'], pre[0]['boxes'][:n], kps32, up(kinv_images(kk_list)), dec,
                                          int(n_l.max()), gt=gt_dev, iou_min=iou_min, reorder=reorder)
            dev_out.update(dec=dec, boxes=pre[0]['boxes'][:n], kps=pre[0]['kps'][:n])
            if epi is not None:
                dev_out['epi'] = epi
            if want_sd:   # social_interactions(idx, ...) over dic_out['xyz_pred'], i.e. in post-processed order
                gidx = up(np.repeat(koff[:-1], n_l)) + dev_out['order'].long()
                xyz_o, dec_o = dev_out['xyz'].index_select(0, gidx), dec.index_select(0, gidx)
                dev_out['sd'] = social_distance_device(xyz_o[:, [0, 2]], dec_o[:, 5], dec_o[:, 3], dec_o[:, 4], koff,
                                                       threshold_prob=args.threshold_prob,
                                                       threshold_dist=args.threshold_dist, radii=args.radii,
                                                       n_samples=self.N_SAMPLES)
            if want_rh:   # net.py:267-271: the key points as preprocess_pifpaf returned them
                dev_out['rh'] = raising_hand_device(dev_out['kps'])

            # ---- one download of every result
            h = {}
            for k, v in dev_out.items():
                h[k] = _pinned_host('pb_' + k, tuple(v.shape), v.dtype)
                h[k].copy_(v, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
        eng.check_error()
        h = {k: v.numpy() for k, v in h.items()}
        dd, bi = h['dec'][:, 3].astype(np.float64), h['dec'][:, 4].astype(np.float64)
        if want_sd:
            check_laplace_args(dd, bi)   # laplace_sampling (process.py:101-122) in social_interactions
        epi = h['epi'].astype(np.float64) if 'epi' in h else np.zeros(n)
        has_yaw, has_aux = self.net != 'monoloco', stereo
        boxes, kps = h['boxes'].tolist(), h['kps'].tolist()
        sd = h['sd'].tolist() if want_sd else None
        rh = [RAISING_HAND[c] for c in h['rh'].tolist()] if want_rh else None
        results = []
        for i in range(n_img):
            a, b = int(koff[i]), int(koff[i + 1])
            res = defaultdict(list)
            if b > a:
                yaw = (h['dec'][a:b, 5].astype(np.float64), h['dec'][a:b, 6].astype(np.float64)) if has_yaw else None
                assemble_post(res, {k: h[k][a:b] for k in ('xyz', 'conf', 'uv', 'match', 'order', 'xyz_real')},
                              int(h['n_match'][i]), boxes[a:b], kps[a:b], dd[a:b], bi[a:b], epi[a:b], yaw,
                              h['dec'][a:b, 7].astype(np.float64) if has_aux else None,
                              dic_gt_list[i] if dic_gt_list is not None else None)
            results.append((boxes[a:b], kps[a:b], finish(res, sd[a:b] if want_sd else None, rh[a:b] if want_rh else None)))
        return results

    def _pinned(self, name, shape, dtype):
        """Pinned host buffer of this Loco, reused across calls (each call synchronises before it returns)."""
        import math
        n = math.prod(shape)
        st = self.__dict__.setdefault('_pin', {})
        buf = st.get(name)
        if buf is None or buf.numel() < n or buf.dtype != dtype:
            buf = st[name] = torch.empty((max(n, 64),), dtype=dtype).pin_memory()
        return buf[:n].view(shape)

    def _forward_host_mono(self, eng, keypoints, kk):
        """Python lists -> pinned staging -> mlb_forward_host -> fresh CPU tensors (caller owns them, net.py contract)."""
        import numpy as np
        m = len(keypoints)
        st = getattr(self, '_stage', None)
        if st is None or st['cap'] < m:
            cap = max(64, 1 << (m - 1).bit_length())
            st = {'cap': cap, 'kps': torch.empty((cap, 3, 17), dtype=torch.float32).pin_memory(),
                  'raw': torch.empty((cap, eng.output_size), dtype=torch.float32).pin_memory(),
                  'dec': torch.empty((cap, 8), dtype=torch.float32).pin_memory(),
                  'xyzc': torch.empty((cap, 4), dtype=torch.float32).pin_memory()}
            self._stage = st
        st['kps'][:m] = torch.from_numpy(np.asarray(keypoints, dtype=np.float32))
        out = {'raw': st['raw'][:m], 'dec': st['dec'][:m], 'xyzc': st['xyzc'][:m]}
        eng.forward_host(st['kps'][:m], kk=kk, kind=L_.IN_KPS, out=out)
        return {k: v.clone() for k, v in out.items()}

    def epistemic_uncertainty(self, inputs):
        """net.py:135-161: n_dropout stochastic passes (top-level dropout on) + Laplace sampling -> std per instance."""
        assert self.net in ('monoloco', 'monoloco_p', 'monoloco_pp'), "Not supported for MonStereo"
        eng = self.model.engine()
        return eng.epistemic_std(inputs, self.n_dropout, n_samples=self.N_SAMPLES, seed=1).cpu()

    # ------------------------------------------------------------------------------------------- post-process
    @staticmethod
    def post_process(dic_in, boxes, keypoints, kk, dic_gt=None, iou_min=0.3, reorder=True, verbose=False):
        """Final per-instance dictionary for visualisation / KITTI txt (same keys, order and values as net.py:163-248),
        computed column-wise: instances matched to ground truth come first (left to right), then the rest."""
        import numpy as np
        res = defaultdict(list)
        if dic_in is None:
            return res
        n = len(boxes)
        matches = get_iou_matches(boxes, dic_gt['boxes'], iou_min=iou_min) if dic_gt else []
        if verbose:
            print("found {} matches with ground-truth".format(len(matches)) if dic_gt else "NO ground-truth associated")
        taken = {i for i, _ in matches}
        if reorder and matches:
            matches = reorder_matches(matches, boxes, mode='left_right')
        order = [i for i, _ in matches] + [i for i in range(n) if i not in taken]
        res['gt'] = [True] * len(matches) + [False] * (n - len(matches))

        col = lambda key: np.asarray(dic_in[key], dtype=np.float64).reshape(-1)  # noqa: E731
        dd, bi, epi = col('d'), col('bi'), np.asarray(dic_in['epi'], dtype=np.float64).reshape(-1)
        centres = get_keypoints(keypoints, mode='center')
        rays = pixel_to_camera(centres, kk, 1)  # bbox-centre rays at z = 1 (net.py:195)
        if isinstance(dic_in, dict) and dic_in.get('xyz_c') is not None and len(dic_in['xyz_c']) == n:
            xyz = dic_in['xyz_c']  # xyz_from_distance already evaluated by the fused kernel's epilogue
        else:
            xyz = xyz_from_distance(torch.as_tensor(dd, dtype=torch.float32), rays)
        xyz64 = np.asarray(xyz, dtype=np.float64)
        conf = 0.035 * np.asarray([b[-1] for b in boxes], dtype=np.float64) / (bi / np.sqrt((xyz64 ** 2).sum(1)))
        pix = {name: np.asarray(get_keypoints(keypoints, mode=mode)).tolist()
               for name, mode in (('uv_centers', 'center'), ('uv_shoulders', 'shoulder'), ('uv_heads', 'head'))}
        has_yaw, has_aux = 'yaw' in dic_in, 'aux' in dic_in
        for i in order:
            res['boxes'].append(boxes[i])
            res['confs'].append(float(conf[i]))
            res['dds_pred'].append(float(dd[i]))
            res['stds_ale'].append(float(bi[i]))
            res['stds_epi'].append(float(epi[i]))
            res['xyz_pred'].append(np.asarray(xyz[i]).reshape(-1).tolist())
            res['uv_kps'].append(keypoints[i])
            for name, pts in pix.items():
                res[name].append([round(pts[i][0]), round(pts[i][1])])
            res['angles']  # the reference's defaultdict access creates these keys even when the value is missing
            if not has_yaw:
                continue
            res['angles'].append(float(dic_in['yaw'][0][i]))
            res['angles_egocentric'].append(float(dic_in['yaw'][1][i]))
            res['aux']
            if has_aux:
                res['aux'].append(float(dic_in['aux'][i]))
        for i, j in matches:
            d_real = dic_gt['ys'][j][3]
            res['dds_real'].append(d_real)
            res['boxes_gt'].append(dic_gt['boxes'][j])
            res['xyz_real'].append(xyz_from_distance(d_real, rays[i]).squeeze().tolist())
        return res

    @staticmethod
    def social_distance(dic_out, args):
        """net.py:250-265: flag every instance whose F-formation test fires."""
        angles, dds, stds = dic_out['angles'], dic_out['dds_pred'], dic_out['stds_ale']
        xz_centers = [[xx[0], xx[2]] for xx in dic_out['xyz_pred']]
        dic_out['social_distance'] = [bool(social_interactions(idx, xz_centers, angles, dds, stds=stds,
                                                               threshold_prob=args.threshold_prob,
                                                               threshold_dist=args.threshold_dist, radii=args.radii))
                                      for idx, _ in enumerate(dic_out['xyz_pred'])]
        return dic_out

    @staticmethod
    def raising_hand(dic_out, keypoints):
        """net.py:267-271."""
        dic_out['raising_hand'] = [is_raising_hand(keypoint) for keypoint in keypoints]
        return dic_out

    @staticmethod
    def social_distance_batch(dic_out_list, args):
        """Loco.social_distance over many images in ONE launch (social_distance_device): every dictionary gets the
        'social_distance' list the per-image method writes, flag for flag (same args.threshold_prob / threshold_dist /
        radii, social_distance=False, 100 samples).  An empty dictionary gets [], and a None entry becomes an empty
        defaultdict(list) with [] (what post_process gives an image without detections).  Inputs go through pinned
        memory and the call ends in one stream synchronisation.  Raises ValueError where the reference's Laplace
        constructor would, before anything is launched.  Returns the list of dictionaries."""
        import numpy as np
        from .post import social_distance_device, check_laplace_args
        res = [defaultdict(list) if d is None else d for d in dic_out_list]
        for d in res:
            if isinstance(d, defaultdict):   # the per-image method's reads create these keys on post_process's dicts
                d['angles'], d['dds_pred'], d['stds_ale'], d['xyz_pred']  # noqa: B018
        counts = [len(d['xyz_pred']) if 'xyz_pred' in d else 0 for d in res]
        n = sum(counts)
        if n == 0:
            for d in res:
                d['social_distance'] = []
            return res
        live = [d for d, c in zip(res, counts) if c]
        xz = np.concatenate([np.asarray(d['xyz_pred'], dtype=np.float64).reshape(-1, 3)[:, (0, 2)] for d in live])
        ang = np.concatenate([np.asarray(d['angles'], dtype=np.float64).reshape(-1) for d in live])
        dds = np.concatenate([np.asarray(d['dds_pred'], dtype=np.float32).reshape(-1) for d in live])
        stds = np.concatenate([np.asarray(d['stds_ale'], dtype=np.float32).reshape(-1) for d in live])
        if not (len(ang) == len(dds) == len(stds) == n):
            raise ValueError("social_distance_batch: angles, dds_pred and stds_ale need one entry per person")
        check_laplace_args(dds, stds)   # laplace_sampling (process.py:101-122) with the default 100 samples
        dev = torch.device('cuda', torch.cuda.current_device())
        h64, h32 = _pinned_host('sd64', (3 * n,), torch.float64), _pinned_host('sd32', (2 * n,), torch.float32)
        h64[:2 * n].copy_(torch.from_numpy(xz.reshape(-1)))
        h64[2 * n:].copy_(torch.from_numpy(ang))
        h32[:n].copy_(torch.from_numpy(dds))
        h32[n:].copy_(torch.from_numpy(stds))
        d64, d32 = h64.to(dev, non_blocking=True), h32.to(dev, non_blocking=True)
        flags = social_distance_device(d64[:2 * n].view(n, 2), d64[2 * n:], d32[:n], d32[n:], np.cumsum([0] + counts),
                                       threshold_prob=args.threshold_prob, threshold_dist=args.threshold_dist,
                                       radii=args.radii, n_samples=Loco.N_SAMPLES)
        h_out = _pinned_host('sd_out', (n,), torch.bool)
        h_out.copy_(flags, non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()
        vals = h_out.tolist()
        pos = 0
        for d, c in zip(res, counts):
            d['social_distance'] = vals[pos:pos + c]
            pos += c
        return res

    @staticmethod
    def raising_hand_batch(dic_out_list, keypoints_list):
        """Loco.raising_hand over many images in ONE launch (raising_hand_device): dictionary i gets
        [is_raising_hand(k) for k in keypoints_list[i]], in the caller's keypoint order as net.py:269-271 does.  None
        entries become an empty defaultdict(list).  Pinned staging, one stream synchronisation.  Returns the list."""
        import numpy as np
        from .post import raising_hand_device, RAISING_HAND
        if len(keypoints_list) != len(dic_out_list):
            raise ValueError("raising_hand_batch: one keypoint list per dictionary")
        res = [defaultdict(list) if d is None else d for d in dic_out_list]
        counts = [len(k) if k is not None else 0 for k in keypoints_list]
        n = sum(counts)
        if n == 0:
            for d in res:
                d['raising_hand'] = []
            return res
        kps = np.concatenate([np.asarray(k, dtype=np.float64).reshape(-1, 3, 17) for k, c in zip(keypoints_list, counts) if c])
        dev = torch.device('cuda', torch.cuda.current_device())
        h_kps = _pinned_host('rh_kps', (n, 3, 17), torch.float64)
        h_kps.copy_(torch.from_numpy(kps))
        codes = raising_hand_device(h_kps.to(dev, non_blocking=True))
        h_out = _pinned_host('rh_out', (n,), torch.int8)
        h_out.copy_(codes, non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()
        vals = [RAISING_HAND[c] for c in h_out.tolist()]
        pos = 0
        for d, c in zip(res, counts):
            d['raising_hand'] = vals[pos:pos + c]
            pos += c
        return res


_PINNED = {}


def _pinned_host(name, shape, dtype):
    """Pinned host buffer shared by the static batch methods, reused across calls (each call synchronises before it
    returns)."""
    import math
    n = math.prod(shape)
    buf = _PINNED.get(name)
    if buf is None or buf.numel() < n or buf.dtype != dtype:
        buf = _PINNED[name] = torch.empty((max(n, 64),), dtype=dtype).pin_memory()
    return buf[:n].view(shape)
