"""ctypes binding of include/monoloco_b200.h.  There is NO fallback: if the CUDA library is missing
or cannot be loaded every product entry point raises (the product path never runs on the CPU)."""
import ctypes as C
import os

from .build import LIB_PATH

MLB_ABI_VERSION = 2
MLB_MAX_OPS = 32
MLB_MAX_PEERS = 8
GATHER_LD = 20
GATHER_DEC = 12
GATHER_FLAG_STRIDE = 32
IPC_HANDLE_BYTES = 64
OP_GEMM, OP_HEAD = 0, 1
F_RELU, F_SAVE_RES, F_ADD_RES, F_DROPOUT, F_IN_XIN = 1, 2, 4, 8, 16
DECODE_NONE, DECODE_LOCO, DECODE_MONO, DECODE_DB = 0, 1, 2, 3
IN_X, IN_KPS, IN_KPS_STEREO = 0, 1, 2
FWD_ZERO_CENTER, FWD_DROPOUT, FWD_FORCE_TILE, FWD_FORCE_CLUSTER, FWD_FORCE_WIDE = 1, 2, 8, 16, 64
FWD_FORCE_TC = 128
FWD_FORCE_WIDE2 = 256
KERNEL_NAMES = {0: 'loco_forward_kernel (FFMA row tiles)', 1: 'loco_forward_cluster_kernel (FFMA, 8-CTA clusters)',
                2: 'loco_forward_wide_kernel (FFMA, whole grid)', 3: 'loco_forward_tc_kernel (wgmma 3xTF32)',
                4: 'loco_forward_wide2_kernel (FFMA, 4-CTA clusters, K x N split)'}

EXPORTS = ['mlb_create', 'mlb_update_weights', 'mlb_destroy', 'mlb_last_error', 'mlb_abi_version', 'mlb_num_sms', 'mlb_device_error', 'mlb_last_kernel', 'mlb_tc_resident_clusters', 'mlb_kernel_times',
           'mlb_forward', 'mlb_forward_host', 'mlb_forward_images', 'mlb_preprocess', 'mlb_stereo_filter', 'mlb_stereo_filter_images', 'mlb_post_process', 'mlb_kitti_rows', 'mlb_social_distance', 'mlb_raising_hand', 'mlb_preprocess_pifpaf', 'mlb_decode', 'mlb_laplace_std', 'mlb_ipc_alloc', 'mlb_ipc_open', 'mlb_ipc_close', 'mlb_ipc_free', 'mlb_train_create', 'mlb_train_destroy',
           'mlb_train_forward', 'mlb_train_backward', 'mlb_train_step', 'mlb_train_phase_times', 'mlb_train_subphase_times',
           'mlb_adam_clip_step', 'mlb_task_stats',
           'mlb_probe_ffma',
           'mlb_launch_count', 'mlb_debug_fwd_marks',
           ]


class MlbOp(C.Structure):
    _fields_ = [('type', C.c_int32), ('K', C.c_int32), ('Kpad', C.c_int32), ('N', C.c_int32), ('flags', C.c_int32),
                ('out_col', C.c_int32), ('w_off', C.c_int64), ('scale_off', C.c_int64), ('shift_off', C.c_int64)]


class MlbModelDesc(C.Structure):
    _fields_ = [('abi_version', C.c_int32), ('input_size', C.c_int32), ('output_size', C.c_int32),
                ('linear_size', C.c_int32), ('n_ops', C.c_int32), ('decode_kind', C.c_int32),
                ('p_dropout', C.c_float), ('reserved', C.c_int32)]


class MlbForwardArgs(C.Structure):
    _fields_ = [('input_kind', C.c_int32), ('flags', C.c_int32), ('n_rows', C.c_int32), ('n_left', C.c_int32),
                ('n_right', C.c_int32), ('rows_per_group', C.c_int32), ('kinv', C.c_float * 9), ('z_met', C.c_float),
                ('x', C.c_void_p), ('x_right', C.c_void_p), ('out_raw', C.c_void_p), ('out_dec', C.c_void_p),
                ('out_xyzc', C.c_void_p), ('out_x', C.c_void_p), ('drop_mask', C.c_void_p), ('drop_seed', C.c_uint64),
                ('gather', C.c_void_p * MLB_MAX_PEERS), ('n_gather', C.c_int32), ('gather_rank', C.c_int32),
                ('gather_row0', C.c_int64), ('gather_flags', C.c_void_p * MLB_MAX_PEERS), ('gather_epoch', C.c_uint32),
                ('reserved0', C.c_int32)]


class MlbImageBatch(C.Structure):
    _fields_ = [('n_img', C.c_int32), ('reserved', C.c_int32), ('row_off', C.c_void_p), ('left_off', C.c_void_p),
                ('right_off', C.c_void_p), ('kinv', C.c_void_p)]


class MlbPostArgs(C.Structure):
    _fields_ = [('n_img', C.c_int32), ('max_det', C.c_int32), ('max_gt', C.c_int32), ('reorder', C.c_int32),
                ('iou_min', C.c_double), ('det_off', C.c_void_p), ('gt_off', C.c_void_p), ('boxes', C.c_void_p),
                ('kps', C.c_void_p), ('kinv', C.c_void_p), ('dec', C.c_void_p), ('gt_boxes', C.c_void_p),
                ('gt_d', C.c_void_p), ('xyz', C.c_void_p), ('ray', C.c_void_p), ('conf', C.c_void_p), ('uv', C.c_void_p),
                ('match_gt', C.c_void_p), ('order', C.c_void_p), ('n_match', C.c_void_p), ('xyz_real', C.c_void_p)]


SOCIAL_MAX_PEOPLE = 1024
SOCIAL_MAX_RADII = 8


class MlbSocialArgs(C.Structure):
    _fields_ = [('n_img', C.c_int32), ('n_people', C.c_int32), ('max_people', C.c_int32), ('n_samples', C.c_int32),
                ('n_radii', C.c_int32), ('social_distance', C.c_int32), ('table_len', C.c_int64),
                ('threshold_prob', C.c_double), ('threshold_dist', C.c_double), ('radii', C.c_double * SOCIAL_MAX_RADII),
                ('img_off', C.c_void_p), ('xz', C.c_void_p), ('angles', C.c_void_p), ('dds', C.c_void_p),
                ('stds', C.c_void_p), ('table', C.c_void_p), ('out', C.c_void_p)]


class MlbPifpafArgs(C.Structure):
    _fields_ = [('n_img', C.c_int32), ('n_ann', C.c_int32), ('enlarge', C.c_int32), ('reserved', C.c_int32),
                ('min_conf', C.c_double), ('ann_off', C.c_void_p), ('kps', C.c_void_p), ('bbox', C.c_void_p),
                ('score', C.c_void_p), ('has_score', C.c_void_p), ('im_size', C.c_void_p), ('has_size', C.c_void_p),
                ('out_boxes', C.c_void_p), ('out_kps', C.c_void_p), ('out_kps32', C.c_void_p), ('out_src', C.c_void_p),
                ('kept_off', C.c_void_p), ('error', C.c_void_p), ('scratch', C.c_void_p)]


PIFPAF_ERR_BOX, PIFPAF_ERR_TIMEOUT = 1, 2   # bits of mlb_pifpaf_args.error


MLB_MAX_BLOCKS = 16
TASK_IDS = {'d': 0, 'x': 1, 'y': 2, 'h': 3, 'w': 4, 'l': 5, 'ori': 6, 'aux': 7}


class MlbTrainBlock(C.Structure):
    _fields_ = [('K', C.c_int32), ('has_bn', C.c_int32), ('res_src', C.c_int32), ('reserved', C.c_int32),
                ('W', C.c_void_p), ('b', C.c_void_p), ('gamma', C.c_void_p), ('beta', C.c_void_p),
                ('running_mean', C.c_void_p), ('running_var', C.c_void_p),
                ('dW', C.c_void_p), ('db', C.c_void_p), ('dgamma', C.c_void_p), ('dbeta', C.c_void_p)]


class MlbTrainArgs(C.Structure):
    _fields_ = [('n_rows', C.c_int32), ('input_size', C.c_int32), ('output_size', C.c_int32), ('linear_size', C.c_int32),
                ('n_blocks', C.c_int32), ('aux_block', C.c_int32), ('update_running_stats', C.c_int32),
                ('rows_per_group', C.c_int32),
                ('p_dropout', C.c_float), ('bn_eps', C.c_float), ('bn_momentum', C.c_float), ('flags', C.c_int32),
                ('drop_seed', C.c_uint64), ('drop_mask', C.c_void_p), ('x', C.c_void_p), ('out', C.c_void_p),
                ('g_out', C.c_void_p),
                ('W_aux', C.c_void_p), ('b_aux', C.c_void_p), ('W_fin', C.c_void_p), ('b_fin', C.c_void_p),
                ('dW_aux', C.c_void_p), ('db_aux', C.c_void_p), ('dW_fin', C.c_void_p), ('db_fin', C.c_void_p),
                ('labels', C.c_void_p), ('label_ld', C.c_int32), ('n_tasks', C.c_int32),
                ('tasks', C.c_int32 * 8), ('task_scale', C.c_float * 8), ('loss_vals', C.c_void_p),
                ('task_scale_dev', C.c_void_p)]


STATS_MAX_SEG = 16
STATS_NACC = 17
STAT_N, STAT_TOTAL, STAT_VAL, STAT_BI, STAT_BI_HIT, STAT_ERR, STAT_ERR2, STAT_AUX_MISS, STAT_LAPLACE, STAT_ORI_L1 = \
    0, 1, 2, 10, 11, 12, 13, 14, 15, 16


class MlbTaskStatsArgs(C.Structure):
    _fields_ = [('n_seg', C.c_int32), ('out_cols', C.c_int32), ('label_ld', C.c_int32), ('task_mask', C.c_int32),
                ('seg_off', C.c_int32 * (STATS_MAX_SEG + 1)), ('reserved', C.c_int32), ('lambdas', C.c_float * 8),
                ('out', C.c_void_p), ('labels', C.c_void_p), ('log_sigmas', C.c_void_p), ('acc', C.c_void_p)]


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "monoloco_b200: %s is missing -- build it with `python -m monoloco_b200.build` "
            "(there is no CPU fallback for the product path)" % LIB_PATH)
    l = C.CDLL(LIB_PATH)
    l.mlb_last_error.restype = C.c_char_p
    l.mlb_create.argtypes = [C.POINTER(MlbModelDesc), C.POINTER(MlbOp), C.c_void_p, C.c_size_t, C.c_int,
                             C.POINTER(C.c_void_p)]
    l.mlb_update_weights.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    l.mlb_destroy.argtypes = [C.c_void_p]
    l.mlb_destroy.restype = None
    l.mlb_num_sms.argtypes = [C.c_void_p]
    l.mlb_device_error.argtypes = [C.c_void_p]
    l.mlb_last_kernel.argtypes = [C.c_void_p]
    l.mlb_tc_resident_clusters.argtypes = [C.c_void_p]
    l.mlb_kernel_times.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
    l.mlb_forward.argtypes = [C.c_void_p, C.POINTER(MlbForwardArgs), C.c_void_p]
    l.mlb_forward_host.argtypes = [C.c_void_p, C.POINTER(MlbForwardArgs), C.c_void_p]
    l.mlb_forward_images.argtypes = [C.c_void_p, C.POINTER(MlbForwardArgs), C.POINTER(MlbImageBatch), C.c_void_p]
    l.mlb_preprocess.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_float), C.c_float, C.c_int, C.c_void_p, C.c_void_p]
    l.mlb_stereo_filter.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    l.mlb_stereo_filter_images.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(MlbImageBatch), C.c_int, C.c_int,
                                           C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p]
    l.mlb_post_process.argtypes = [C.POINTER(MlbPostArgs), C.c_void_p]
    l.mlb_kitti_rows.argtypes = [C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p]
    l.mlb_social_distance.argtypes = [C.POINTER(MlbSocialArgs), C.c_void_p]
    l.mlb_raising_hand.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    l.mlb_preprocess_pifpaf.argtypes = [C.POINTER(MlbPifpafArgs), C.c_void_p]
    l.mlb_decode.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    l.mlb_laplace_std.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_void_p, C.c_void_p]
    l.mlb_ipc_alloc.argtypes = [C.c_int, C.c_size_t, C.POINTER(C.c_void_p), C.c_char_p]
    l.mlb_ipc_open.argtypes = [C.c_int, C.c_char_p, C.POINTER(C.c_void_p)]
    l.mlb_ipc_close.argtypes = [C.c_void_p]
    l.mlb_ipc_free.argtypes = [C.c_void_p]
    l.mlb_train_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
    l.mlb_train_destroy.argtypes = [C.c_void_p]
    l.mlb_train_destroy.restype = None
    for fn in (l.mlb_train_forward, l.mlb_train_backward, l.mlb_train_step):
        fn.argtypes = [C.c_void_p, C.POINTER(MlbTrainArgs), C.POINTER(MlbTrainBlock), C.c_void_p]
    l.mlb_train_phase_times.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    l.mlb_train_subphase_times.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_double)]
    l.mlb_adam_clip_step.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int64,
                                     C.c_void_p, C.c_void_p]
    l.mlb_task_stats.argtypes = [C.POINTER(MlbTaskStatsArgs), C.c_void_p]
    l.mlb_probe_ffma.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double), C.c_void_p]
    l.mlb_launch_count.restype = C.c_uint64
    if l.mlb_abi_version() != MLB_ABI_VERSION:
        raise RuntimeError("monoloco_b200: ABI version mismatch between _lib.py and the shared library")
    _lib = l
    return l


def check(rc, what):
    if rc != 0:
        raise RuntimeError("%s failed: %s" % (what, lib().mlb_last_error().decode()))
