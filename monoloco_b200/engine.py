"""Thin Python owner of an `mlb_handle` (include/monoloco_b200.h).

PyTorch is used for device memory and streams only; every computation on the hot path is a kernel in
libmonoloco_b200.so.  There is no CPU fallback: constructing an engine without the library / an H100 raises.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib as L_
from .packing import pack_state_dict

DEC_COLS = ('x', 'y', 'z', 'd', 'bi', 'yaw_pred', 'yaw_orig', 'aux')


_KINV_CACHE = {}


def kinv_from_kk(kk):
    """K^-1 (utils/camera.py:25) computed once on the host in float64, rounded to fp32 (cached per K)."""
    k = np.asarray(kk.detach().cpu().numpy() if hasattr(kk, 'detach') else kk, dtype=np.float64).reshape(3, 3)
    key = k.tobytes()
    v = _KINV_CACHE.get(key)
    if v is None:
        if len(_KINV_CACHE) > 64:
            _KINV_CACHE.clear()
        v = _KINV_CACHE[key] = np.linalg.inv(k).astype(np.float32).reshape(9)
    return v


def kinv_images(kk_list):
    """K^-1 of every image (kinv_from_kk), packed [n_img, 9] fp32 as mlb_image_batch.kinv expects."""
    return np.stack([kinv_from_kk(kk) for kk in kk_list]).astype(np.float32).reshape(len(kk_list), 9)


def image_offsets(counts):
    """Per-image counts -> int32 CSR offsets [n_img + 1] (0, n_0, n_0 + n_1, ...)."""
    off = np.zeros(len(counts) + 1, dtype=np.int64)
    np.cumsum(np.asarray(counts, dtype=np.int64), out=off[1:])
    if off[-1] > np.iinfo(np.int32).max:
        raise ValueError("more than 2^31 - 1 rows")
    return off.astype(np.int32)


def check_image_batch(row_off, n_rows, left_off=None, right_off=None, n_left=None, n_right=None):
    """Host check of the offsets of mlb_forward_images (the kernels only clamp): int32 [n_img + 1] arrays, each starting at 0,
    non-decreasing and ending at its total; in stereo, image i owns (left_off[i+1] - left_off[i]) * (right_off[i+1] -
    right_off[i]) rows.  Returns the offsets as int32 numpy arrays."""
    def csr(name, off, total):
        off = np.asarray(off, dtype=np.int64).reshape(-1)
        if off.size < 2:
            raise ValueError("%s: at least one image needed (n_img + 1 >= 2 offsets)" % name)
        if off[0] != 0 or off[-1] != total or (np.diff(off) < 0).any():
            raise ValueError("%s must start at 0, be non-decreasing and end at %d" % (name, total))
        if total > np.iinfo(np.int32).max:
            raise ValueError("%s: more than 2^31 - 1 rows" % name)
        return off.astype(np.int32)
    row_off = csr('row_off', row_off, n_rows)
    if left_off is None:
        return row_off, None, None
    left_off, right_off = csr('left_off', left_off, n_left), csr('right_off', right_off, n_right)
    if not (left_off.size == right_off.size == row_off.size):
        raise ValueError("row_off, left_off and right_off must have n_img + 1 entries each")
    if (np.diff(row_off.astype(np.int64)) != np.diff(left_off.astype(np.int64)) * np.diff(right_off.astype(np.int64))).any():
        raise ValueError("stereo: image i must own n_left_i * n_right_i rows")
    return row_off, left_off, right_off


def _upload(arr, device):
    """Small host array -> device tensor through torch's pinned-memory cache (asynchronous, stream-ordered)."""
    return torch.from_numpy(np.ascontiguousarray(arr)).pin_memory().to(device, non_blocking=True)


class LocoEngine:
    def __init__(self, state_dict, p_dropout=0.2, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("monoloco_b200: no CUDA device -- the hot path has no CPU fallback")
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != 'cuda':
            raise RuntimeError("monoloco_b200: device must be a CUDA device")
        self.index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self._lib = L_.lib()
        self._h = C.c_void_p()
        self.p_dropout = p_dropout
        self._create(state_dict)

    # ---------------------------------------------------------------- lifetime
    def _create(self, state_dict):
        pm = pack_state_dict(state_dict, self.p_dropout)
        self.packed = pm
        d = pm.desc
        desc = L_.MlbModelDesc(L_.MLB_ABI_VERSION, d['input_size'], d['output_size'], d['linear_size'], d['n_ops'],
                               d['decode_kind'], d['p_dropout'], 0)
        ops = (L_.MlbOp * len(pm.ops))()
        for i, o in enumerate(pm.ops):
            ops[i] = L_.MlbOp(o['type'], o['K'], o['Kpad'], o['N'], o['flags'], o['out_col'], o['w_off'],
                              o['scale_off'], o['shift_off'])
        self._blob = pm.blob  # keep alive during the call
        L_.check(self._lib.mlb_create(C.byref(desc), ops, pm.blob.ctypes.data_as(C.c_void_p), pm.blob.size,
                                      self.index, C.byref(self._h)), 'mlb_create')
        self.input_size, self.output_size, self.linear_size = d['input_size'], d['output_size'], d['linear_size']
        self.decode_kind = d['decode_kind']
        self.n_sms = self._lib.mlb_num_sms(self._h)

    def update_weights(self, state_dict):
        """Re-pack and upload (same architecture), e.g. after an optimizer step / load_state_dict."""
        pm = pack_state_dict(state_dict, self.p_dropout)
        if pm.blob.size != self.packed.blob.size or pm.desc != self.packed.desc:
            self.close()
            self._create(state_dict)
            return
        self.packed = pm
        L_.check(self._lib.mlb_update_weights(self._h, pm.blob.ctypes.data_as(C.c_void_p), pm.blob.size,
                                              C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)),
                 'mlb_update_weights')
        torch.cuda.current_stream(self.device).synchronize()

    def close(self):
        if getattr(self, '_h', None) is not None and self._h.value:
            self._lib.mlb_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:  # interpreter shutdown
            pass

    def last_kernel(self):
        """(id, name) of the kernel the most recent forward launched."""
        k = self._lib.mlb_last_kernel(self._h)
        return k, L_.KERNEL_NAMES.get(k, '?')

    def kernel_times(self):
        """Per-wave kernel times measured at engine creation (ms) and the tensor-core kernel's co-resident CTA group count
        (`tc_resident_clusters`): what mlb_forward's kernel choice is based on."""
        t = (C.c_double * 4)()
        measured = self._lib.mlb_kernel_times(self._h, t)
        return {'measured': bool(measured), 'ffma_cluster_wave_ms': t[0], 'ffma_tile_wave_ms': '%.4f + %.4f * TM' % (t[1], t[2]),
                'tc_wave_ms': t[3], 'tc_resident_clusters': self._lib.mlb_tc_resident_clusters(self._h)}

    def check_error(self):
        """Raise if a kernel of this engine reported a protocol time-out (call after a stream synchronisation)."""
        err = self._lib.mlb_device_error(self._h)
        if err:
            raise RuntimeError("monoloco_b200: device error flag %d (1 TMA/mbarrier time-out, 3 grid barrier, "
                               "4 fused all-gather peer time-out)" % err)

    # ---------------------------------------------------------------- forward on device tensors
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def forward(self, x, x_right=None, kk=None, kind=L_.IN_X, want_dec=True, want_xyzc=False, want_x=False,
                zero_center=False, dropout=False, drop_mask=None, drop_seed=0, rows_per_group=0,
                gather_ptrs=None, gather_row0=0, gather_flags=None, gather_rank=0, gather_epoch=0, kernel=None):
        """x: float32 CUDA tensor ([B,in] | [B,3,17] | left [L,3,17]).  Returns dict of CUDA tensors."""
        assert x.is_cuda and x.dtype == torch.float32
        x = x.contiguous()
        a = L_.MlbForwardArgs()
        a.input_kind = kind
        a.flags = self._flags(zero_center, dropout, kernel)
        if kind == L_.IN_KPS_STEREO:
            x_right = x_right.contiguous()
            n_left, n_right = x.shape[0], x_right.shape[0]
            B = n_left * n_right
            a.n_left, a.n_right = n_left, n_right
            a.x_right = x_right.data_ptr()
        else:
            B = x.shape[0]
        if kind != L_.IN_X:
            kinv = kinv_from_kk(kk)
            for i in range(9):
                a.kinv[i] = float(kinv[i])
            a.z_met = 10.0
        a.n_rows = B
        a.rows_per_group = rows_per_group
        a.x = x.data_ptr()
        out = self._outputs(a, B, want_dec, want_xyzc, want_x, drop_mask, drop_seed)
        if gather_ptrs:
            a.n_gather = len(gather_ptrs)
            for i, ptr in enumerate(gather_ptrs):
                a.gather[i] = ptr
            a.gather_row0 = int(gather_row0)
            if gather_flags:  # device-side completion protocol (include/monoloco_b200.h: gather_epoch)
                for i, ptr in enumerate(gather_flags):
                    a.gather_flags[i] = ptr
                a.gather_rank = int(gather_rank)
                a.gather_epoch = int(gather_epoch) & 0xFFFFFFFF
        if B > 0 or (gather_ptrs and gather_flags and gather_epoch):  # an empty shard still signals its epoch
            L_.check(self._lib.mlb_forward(self._h, C.byref(a), self._stream()), 'mlb_forward')
        return out

    @staticmethod
    def _flags(zero_center, dropout, kernel):
        return (L_.FWD_ZERO_CENTER if zero_center else 0) | (L_.FWD_DROPOUT if dropout else 0) | \
            {None: 0, 'tile': L_.FWD_FORCE_TILE, 'cluster': L_.FWD_FORCE_CLUSTER, 'wide': L_.FWD_FORCE_WIDE,
             'tc': L_.FWD_FORCE_TC, 'wide2': L_.FWD_FORCE_WIDE2}[kernel]

    def _outputs(self, a, B, want_dec, want_xyzc, want_x, drop_mask, drop_seed):
        """Device output tensors of a forward of B rows, their pointers and the dropout arguments set in `a`."""
        out = {'raw': torch.empty((B, self.output_size), dtype=torch.float32, device=self.device)}
        a.out_raw = out['raw'].data_ptr()
        if want_dec:
            out['dec'] = torch.empty((B, 8), dtype=torch.float32, device=self.device)
            a.out_dec = out['dec'].data_ptr()
        if want_xyzc:
            out['xyzc'] = torch.empty((B, 4), dtype=torch.float32, device=self.device)
            a.out_xyzc = out['xyzc'].data_ptr()
        if want_x:
            out['x'] = torch.empty((B, self.input_size), dtype=torch.float32, device=self.device)
            a.out_x = out['x'].data_ptr()
        if drop_mask is not None:
            assert drop_mask.is_cuda and drop_mask.dtype == torch.uint8
            drop_mask = drop_mask.contiguous()
            a.drop_mask = drop_mask.data_ptr()
        a.drop_seed = int(drop_seed)
        return out

    def _image_batch(self, row_off, kk_list, B, left_off=None, right_off=None, n_left=None, n_right=None):
        """Checked host offsets + K^-1 per image (kk_list None: no intrinsics, the stereo filter) -> (mlb_image_batch,
        device tensors it points into)."""
        row_off, left_off, right_off = check_image_batch(row_off, B, left_off, right_off, n_left, n_right)
        n_img = row_off.size - 1
        if kk_list is not None and len(kk_list) != n_img:
            raise ValueError("one camera matrix per image: %d matrices for %d images" % (len(kk_list), n_img))
        offs = _upload(np.concatenate([row_off] + ([left_off, right_off] if left_off is not None else [])), self.device)
        kinv = _upload(kinv_images(kk_list), self.device) if kk_list is not None else None
        ib = L_.MlbImageBatch()
        ib.n_img = n_img
        ib.row_off = offs.data_ptr()
        if left_off is not None:
            ib.left_off = offs.data_ptr() + 4 * (n_img + 1)
            ib.right_off = offs.data_ptr() + 8 * (n_img + 1)
        ib.kinv = kinv.data_ptr() if kinv is not None else None
        return ib, (offs, kinv)

    def forward_images(self, x, row_off, kk_list, kind=L_.IN_KPS, x_right=None, left_off=None, right_off=None,
                       want_dec=True, want_xyzc=False, want_x=False, zero_center=False, dropout=False, drop_mask=None,
                       drop_seed=0, kernel=None):
        """Many images in ONE forward launch, each with its own camera matrix (mlb_forward_images).
        x: keypoints of all images concatenated (CUDA [B,3,17]; stereo: left poses [n_left,3,17] and x_right [n_right,3,17]).
        row_off (and in stereo left_off / right_off): host int CSR offsets [n_img + 1], checked here; kk_list: one K per
        image.  Returns the dict of CUDA tensors forward() returns, rows image-major (stereo: image-local pairs l * nr + r)."""
        assert x.is_cuda and x.dtype == torch.float32
        if kind not in (L_.IN_KPS, L_.IN_KPS_STEREO):
            raise ValueError("forward_images: keypoint inputs only (MLB_IN_X carries no camera intrinsics)")
        x = x.contiguous()
        a = L_.MlbForwardArgs()
        a.input_kind = kind
        a.flags = self._flags(zero_center, dropout, kernel)
        if kind == L_.IN_KPS_STEREO:
            if x_right is None or left_off is None or right_off is None:
                raise ValueError("forward_images: stereo needs x_right, left_off and right_off")
            x_right = x_right.contiguous()
            a.n_left, a.n_right = x.shape[0], x_right.shape[0]
            a.x_right = x_right.data_ptr()
            B = int(np.asarray(row_off)[-1])
            ib, keep = self._image_batch(row_off, kk_list, B, left_off, right_off, a.n_left, a.n_right)
        else:
            B = x.shape[0]
            ib, keep = self._image_batch(row_off, kk_list, B)
        a.n_rows = B
        a.z_met = 10.0
        a.x = x.data_ptr()
        out = self._outputs(a, B, want_dec, want_xyzc, want_x, drop_mask, drop_seed)
        if B > 0:
            L_.check(self._lib.mlb_forward_images(self._h, C.byref(a), C.byref(ib), self._stream()), 'mlb_forward_images')
        return out

    def forward_host(self, x, x_right=None, kk=None, kind=L_.IN_X, want_dec=True, want_xyzc=False, out=None,
                     rows_per_group=0):
        """Host (numpy / pinned torch CPU) buffers in, host buffers out; H2D + kernel + D2H + sync inside."""
        xt = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
        a = L_.MlbForwardArgs()
        a.input_kind = kind
        if kind == L_.IN_KPS_STEREO:
            xr = x_right if isinstance(x_right, torch.Tensor) else torch.from_numpy(
                np.ascontiguousarray(x_right, dtype=np.float32))
            a.n_left, a.n_right = xt.shape[0], xr.shape[0]
            B = a.n_left * a.n_right
            a.x_right = xr.data_ptr()
        else:
            B = xt.shape[0]
        if kind != L_.IN_X:
            kinv = kinv_from_kk(kk)
            for i in range(9):
                a.kinv[i] = float(kinv[i])
            a.z_met = 10.0
        a.n_rows = B
        a.rows_per_group = rows_per_group
        if out is None:
            out = {'raw': torch.empty((B, self.output_size), dtype=torch.float32)}
            if want_dec:
                out['dec'] = torch.empty((B, 8), dtype=torch.float32)
            if want_xyzc:
                out['xyzc'] = torch.empty((B, 4), dtype=torch.float32)
        a.x = xt.data_ptr()
        a.out_raw = out['raw'].data_ptr()
        if 'dec' in out:
            a.out_dec = out['dec'].data_ptr()
        if 'xyzc' in out:
            a.out_xyzc = out['xyzc'].data_ptr()
        if B > 0:
            L_.check(self._lib.mlb_forward_host(self._h, C.byref(a), self._stream()), 'mlb_forward_host')
        return out

    def stereo_filter(self, raw, dec, n_left, n_right, xyzc=None, trim=True):
        """process.py:307-327 on device (one warp per left pose, no host synchronisation inside).
        trim=True : (sel_raw, sel_dec, sel_idx[, sel_xyzc]) CUDA tensors cut to the kept rows (reads the count: one sync);
        trim=False: the full-capacity buffers plus the device count tensor `n_sel` as the last element, no sync."""
        B = n_left * n_right
        sel_raw = torch.empty_like(raw)
        sel_dec = torch.empty_like(dec) if dec is not None else None
        sel_xyzc = torch.empty_like(xyzc) if xyzc is not None else None
        sel_idx = torch.empty((B,), dtype=torch.int32, device=self.device)
        n_sel = torch.empty((1,), dtype=torch.int32, device=self.device)
        cnt = torch.empty((n_left,), dtype=torch.int32, device=self.device)
        best = torch.empty((n_left,), dtype=torch.float32, device=self.device)
        ptr = lambda t_: t_.data_ptr() if t_ is not None else None  # noqa: E731
        L_.check(self._lib.mlb_stereo_filter(raw.data_ptr(), ptr(dec), ptr(xyzc), n_left, n_right, raw.shape[1],
                                             sel_raw.data_ptr(), ptr(sel_dec), ptr(sel_xyzc), sel_idx.data_ptr(),
                                             n_sel.data_ptr(), cnt.data_ptr(), best.data_ptr(), self._stream()),
                 'mlb_stereo_filter')
        if not trim:
            res = (sel_raw, sel_dec, sel_idx)
            return res + ((sel_xyzc,) if xyzc is not None else ()) + (n_sel,)
        n = int(n_sel.item())
        res = (sel_raw[:n], (sel_dec[:n] if dec is not None else None), sel_idx[:n])
        return res + (sel_xyzc[:n],) if xyzc is not None else res

    def stereo_filter_images(self, raw, dec, row_off, left_off, right_off, xyzc=None, trim=True):
        """process.py:307-327 per image over the rows of a stereo forward_images (mlb_stereo_filter_images): kept rows
        image-major, each image in the order stereo_filter gives it.  Returns a dict of CUDA tensors sel_raw, sel_dec,
        sel_idx (row indices into raw), sel_xyzc, n_sel [1] and sel_img_off [n_img + 1]; trim=True cuts them to the
        kept rows and turns sel_img_off into a host list (one synchronisation)."""
        n_left, n_right = int(np.asarray(left_off)[-1]), int(np.asarray(right_off)[-1])
        B = raw.shape[0]
        ib, keep = self._image_batch(row_off, None, B, left_off, right_off, n_left, n_right)
        out = {'sel_raw': torch.empty_like(raw), 'sel_dec': torch.empty_like(dec) if dec is not None else None,
               'sel_xyzc': torch.empty_like(xyzc) if xyzc is not None else None,
               'sel_idx': torch.empty((B,), dtype=torch.int32, device=self.device),
               'n_sel': torch.empty((1,), dtype=torch.int32, device=self.device),
               'sel_img_off': torch.empty((ib.n_img + 1,), dtype=torch.int32, device=self.device)}
        cnt = torch.empty((max(n_left, 1),), dtype=torch.int32, device=self.device)
        best = torch.empty((max(n_left, 1),), dtype=torch.float32, device=self.device)
        ptr = lambda t_: t_.data_ptr() if t_ is not None else None  # noqa: E731
        L_.check(self._lib.mlb_stereo_filter_images(ptr(raw), ptr(dec), ptr(xyzc), C.byref(ib), n_left, n_right,
                                                    raw.shape[1], ptr(out['sel_raw']), ptr(out['sel_dec']),
                                                    ptr(out['sel_xyzc']), out['sel_idx'].data_ptr(),
                                                    out['n_sel'].data_ptr(), out['sel_img_off'].data_ptr(),
                                                    cnt.data_ptr(), best.data_ptr(), self._stream()),
                 'mlb_stereo_filter_images')
        if not trim:
            return out
        n = int(out['n_sel'].item())
        out['sel_img_off'] = out['sel_img_off'].cpu().tolist()
        for k in ('sel_raw', 'sel_dec', 'sel_xyzc', 'sel_idx'):
            if out[k] is not None:
                out[k] = out[k][:n]
        return out

    def stereo_filter_host(self, raw, dec, xyzc, n_left, n_right):
        """The filter for callers that want HOST tensors (Loco.forward): the count and the first n_left + 8 candidate rows
        travel in one batch of asynchronous copies followed by ONE synchronisation; only when ties push the kept-row
        count beyond that (process.py:321-326 keeps every tied row) is the remainder fetched."""
        sel_raw, sel_dec, sel_idx, sel_xyzc, n_sel = self.stereo_filter(raw, dec, n_left, n_right, xyzc=xyzc, trim=False)
        cap = min(n_left + 8, n_left * n_right)
        st = getattr(self, '_sf_stage', None)
        if st is None or st['raw'].shape[0] < cap or st['raw'].shape[1] != raw.shape[1]:
            st = {'n': torch.empty((1,), dtype=torch.int32).pin_memory(),
                  'raw': torch.empty((cap, raw.shape[1]), dtype=torch.float32).pin_memory(),
                  'dec': torch.empty((cap, 8), dtype=torch.float32).pin_memory(),
                  'xyzc': torch.empty((cap, 4), dtype=torch.float32).pin_memory()}
            self._sf_stage = st
        st['n'].copy_(n_sel, non_blocking=True)
        st['raw'][:cap].copy_(sel_raw[:cap], non_blocking=True)
        st['dec'][:cap].copy_(sel_dec[:cap], non_blocking=True)
        st['xyzc'][:cap].copy_(sel_xyzc[:cap], non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        n = int(st['n'][0])
        if n <= cap:
            return st['raw'][:n].clone(), st['dec'][:n].clone(), st['xyzc'][:n].clone()
        return sel_raw[:n].cpu(), sel_dec[:n].cpu(), sel_xyzc[:n].cpu()

    def epistemic_std(self, x, n_dropout, n_samples=100, seed=1, kind=L_.IN_X, kk=None, row_off=None, kk_list=None,
                      zero_center=False):
        """net.py:135-161: n_dropout stochastic forwards (top-level dropout on) -> (d, bi) -> Laplace sampling -> std.
        The passes are independent rows to the kernel: the inputs are replicated n_dropout times and run as ONE
        launch (the dropout mask is a function of (seed, site, row, column), so every replica draws its own mask and
        the weights are streamed once for all passes instead of once per pass).  Returns a CUDA tensor [B].
        Images form (row_off + kk_list, keypoints x of all images, mono; zero_center for the legacy monoloco): the image
        CSR is tiled n_dropout times on the host and the replicas run as one forward_images launch."""
        B = x.shape[0]
        reps = x.repeat((n_dropout,) + (1,) * (x.dim() - 1))
        if row_off is not None:
            row_off = np.asarray(row_off, dtype=np.int64)
            tiled = np.concatenate([[0]] + [row_off[1:] + p * B for p in range(n_dropout)])
            out = self.forward_images(reps, tiled, list(kk_list) * n_dropout, kind=L_.IN_KPS, zero_center=zero_center,
                                      dropout=True, drop_seed=seed)
        else:
            out = self.forward(reps, kk=kk, kind=kind, dropout=True, drop_seed=seed)
        c0 = 0 if self.output_size == 2 else 2  # net.py:146-149: db = outputs[:, 0:2] (monoloco) | outputs[:, 2:4]
        d_bi = torch.stack((out['raw'][:, c0], out['dec'][:, 4]), dim=1).contiguous()  # [n_dropout * B, 2] = [N, B, 2]
        std = torch.empty((B,), dtype=torch.float32, device=self.device)
        if B:
            L_.check(self._lib.mlb_laplace_std(d_bi.data_ptr(), n_dropout, B, n_samples, int(seed), std.data_ptr(),
                                               self._stream()), 'mlb_laplace_std')
        return std


def preprocess_device(kps, kk, zero_center=False):
    """process.py:47-67 as a stand-alone kernel: [B,3,17] CUDA tensor -> [B,34] CUDA tensor."""
    lib = L_.lib()
    assert kps.is_cuda and kps.dtype == torch.float32
    kps = kps.contiguous()
    B = kps.shape[0]
    out = torch.empty((B, 34), dtype=torch.float32, device=kps.device)
    kinv = (C.c_float * 9)(*[float(v) for v in kinv_from_kk(kk)])
    if B:
        L_.check(lib.mlb_preprocess(kps.data_ptr(), B, kinv, 10.0, int(zero_center), out.data_ptr(),
                                    C.c_void_p(torch.cuda.current_stream(kps.device).cuda_stream)), 'mlb_preprocess')
    return out


def dec_to_dict(raw, dec, stereo=None):
    """[B,out] raw + [B,8] decoded (CUDA or CPU tensors) -> the reference's dic_out of CPU tensors
    (process.py:231-278): h, w, l, ori, bi, xyzd, d, yaw=(alpha, ry)[, aux]."""
    raw, dec = raw.detach().cpu(), dec.detach().cpu()
    stereo = raw.shape[1] == 10 if stereo is None else stereo
    dic = {'h': raw[:, 4:5], 'w': raw[:, 5:6], 'l': raw[:, 6:7], 'ori': raw[:, 7:9], 'bi': dec[:, 4:5],
           'xyzd': dec[:, 0:4], 'd': dec[:, 3:4], 'yaw': (dec[:, 5:6], dec[:, 6:7])}
    if stereo:
        dic['aux'] = dec[:, 7:8]
    return dic


def decode_device(outputs, decode_kind=L_.DECODE_LOCO):
    """extract_outputs(outputs) for a raw [m,9|10] tensor: decode kernel, then the dictionary of CPU tensors."""
    lib = L_.lib()
    if not torch.cuda.is_available():
        raise RuntimeError("monoloco_b200: no CUDA device -- the hot path has no CPU fallback")
    raw = outputs.detach()
    raw = (raw if raw.is_cuda else raw.cuda()).float().contiguous()
    dec = torch.empty((raw.shape[0], 8), dtype=torch.float32, device=raw.device)
    if raw.shape[0]:
        L_.check(lib.mlb_decode(raw.data_ptr(), raw.shape[0], raw.shape[1], decode_kind, dec.data_ptr(),
                                C.c_void_p(torch.cuda.current_stream(raw.device).cuda_stream)), 'mlb_decode')
    if decode_kind == L_.DECODE_MONO:
        r, d = raw.cpu(), dec.cpu()
        return {'xyz': r[:, 0:3], 'zb': r[:, 2:4], 'h': r[:, 4:5], 'w': r[:, 5:6], 'l': r[:, 6:7], 'ori': r[:, 7:9],
                'xyzd': d[:, 0:4], 'd': d[:, 3:4], 'bi': d[:, 4:5], 'yaw': (d[:, 5:6], d[:, 6:7])}
    return dec_to_dict(raw, dec)


def probe_ffma_tflops(device_index=0, iters=4096, reps=5, packed=False):
    """Measured FP32-FFMA throughput of this GPU (roofline denominator in the fp32-bound regime)."""
    lib = L_.lib()
    n_sm = torch.cuda.get_device_properties(device_index).multi_processor_count
    blocks = n_sm * 4
    flops = C.c_double()
    st = torch.cuda.current_stream()
    best = 0.0
    for _ in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        L_.check(lib.mlb_probe_ffma(device_index, blocks, -iters if packed else iters, C.byref(flops),
                                    C.c_void_p(st.cuda_stream)), 'probe')
        e1.record(st)
        e1.synchronize()
        best = max(best, flops.value / (e0.elapsed_time(e1) * 1e-3) / 1e12)
    return best
