"""
Deterministic synthetic checkpoints and inputs (numpy only, identical on every machine).

There are no pretrained monoloco weights in the reference tree (they are downloaded from Google
Drive, monoloco/predict.py:36-39) and no network here, so tests / bench / smoke use random-init
weights of the reference architectures with the reference's state_dict key names
(SURVEY.md §8b "Checkpoint ABI") and synthetic 17-keypoint detections shaped like the reference's
fixture statistics (SURVEY.md §8d "Synthetic inputs").
"""
import math

import numpy as np

KITTI_K = [[718.3351, 0., 600.3891], [0., 718.3351, 181.5122], [0., 0., 1.]]  # network/intrinsics.yaml:1-6


def _linear(rng, out_f, in_f):
    bound = 1.0 / math.sqrt(in_f)  # nn.Linear default init (kaiming_uniform a=sqrt(5))
    w = rng.uniform(-bound, bound, size=(out_f, in_f)).astype(np.float32)
    b = rng.uniform(-bound, bound, size=(out_f,)).astype(np.float32)
    return w, b


def _bn(rng, n):
    return {
        'weight': rng.uniform(0.6, 1.4, size=n).astype(np.float32),
        'bias': rng.uniform(-0.3, 0.3, size=n).astype(np.float32),
        'running_mean': rng.uniform(-0.5, 0.5, size=n).astype(np.float32),
        'running_var': rng.uniform(0.3, 2.0, size=n).astype(np.float32),
        'num_batches_tracked': np.asarray(5, dtype=np.int64),
    }


def make_state_dict(kind='loco', input_size=34, output_size=9, linear_size=1024, num_stage=3, seed=0):
    """Random checkpoint with the reference's key names.

    kind='loco'     -> LocoModel      (monoloco/network/architectures.py:8-46)
    kind='monoloco' -> MonolocoModel  (architectures.py:111-133)
    Final-layer biases are set to typical label values so the decoded outputs (x,y,z,d,bi,yaw) are
    in a realistic range (theta~1.6, psi~1.4, d~20 m, ...).
    """
    rng = np.random.RandomState(seed)
    sd = {}

    def put_linear(name, out_f, in_f):
        w, b = _linear(rng, out_f, in_f)
        sd[name + '.weight'], sd[name + '.bias'] = w, b

    def put_bn(name, n):
        for k, v in _bn(rng, n).items():
            sd[name + '.' + k] = v

    L = linear_size
    put_linear('w1', L, input_size)
    put_bn('batch_norm1', L)
    for i in range(num_stage):
        p = 'linear_stages.%d' % i
        put_linear(p + '.w1', L, L)
        put_bn(p + '.batch_norm1', L)
        put_linear(p + '.w2', L, L)
        put_bn(p + '.batch_norm2', L)
    typical = np.array([1.57, 1.40, 20.0, -1.0, 1.70, 0.60, 0.80, 0.30, 0.50], dtype=np.float32)
    if kind == 'loco':
        put_linear('w2', L, L)
        put_linear('w3', L, L)
        put_bn('batch_norm3', L)
        put_linear('w_aux', 1, L)
        put_linear('w_fin', output_size - 1, L)
        nfin = output_size - 1
        sd['w_fin.bias'] = (sd['w_fin.bias'] + typical[:nfin]).astype(np.float32)
        sd['w_aux.bias'] = (sd['w_aux.bias'] + (0.5 if output_size == 9 else 0.0)).astype(np.float32)
    elif kind == 'monoloco':
        put_linear('w2', output_size, L)
        n = min(output_size, 9)
        if output_size >= 4:
            sd['w2.bias'][:n] = sd['w2.bias'][:n] + np.array(
                [0.5, 1.0, 20.0, -1.0, 1.70, 0.60, 0.80, 0.30, 0.50], dtype=np.float32)[:n]
        else:
            sd['w2.bias'][:n] = sd['w2.bias'][:n] + np.array([20.0, -1.0], dtype=np.float32)[:n]
    else:
        raise ValueError(kind)
    return sd


def make_keypoints(n, seed=0, right=False):
    """Raw detections [n,3,17] (u row, v row, confidence row), SURVEY.md §8d."""
    rng = np.random.RandomState(seed)
    u_c = rng.uniform(0, 1242, size=(n, 1))
    v_c = rng.uniform(150, 300, size=(n, 1))
    hh = rng.uniform(25, 250, size=(n, 1))
    u = u_c + 0.15 * hh * rng.standard_normal((n, 17))
    v = v_c + 0.30 * hh * rng.standard_normal((n, 17))
    c = rng.uniform(0, 1, size=(n, 17))
    kps = np.stack([u, v, c], axis=1).astype(np.float32)
    if right:
        z = rng.uniform(4, 60, size=(n, 1))
        kps_r = kps.copy()
        kps_r[:, 0, :] -= (0.54 * 721 / z).astype(np.float32)  # process.py:16-20 disparity model
        return kps, kps_r
    return kps


def make_inputs(n, input_size=34, seed=0):
    """Pre-processed network inputs X ~ N(0.40, 2.79^2) (fixture statistics, SURVEY.md §8d)."""
    rng = np.random.RandomState(seed)
    return (0.40 + 2.79 * rng.standard_normal((n, input_size))).astype(np.float32)


def make_labels(n, stereo=False, seed=0):
    """Training labels Y = [theta, psi, z, r, h, w, l, sin, cos, yaw(, s_match)]
    (prep/preprocess_kitti.py:363-369), ranges from the fixture (SURVEY.md §8d)."""
    rng = np.random.RandomState(seed)
    theta = rng.uniform(0.86, 2.28, n)
    psi = rng.uniform(1.22, 1.56, n)
    r = rng.uniform(4.2, 57.3, n)
    z = r * np.sin(psi) * np.sin(theta)
    h = rng.uniform(1.4, 1.95, n)
    w = rng.uniform(0.4, 0.9, n)
    ln = rng.uniform(0.4, 1.1, n)
    yaw = rng.uniform(-math.pi, math.pi, n)
    cols = [theta, psi, z, r, h, w, ln, np.sin(yaw), np.cos(yaw), yaw]
    if stereo:
        cols.append((rng.uniform(0, 1, n) > 0.5).astype(np.float64))
    return np.stack(cols, axis=1).astype(np.float32)


def make_joints_json(path, n_train=157, n_val=61, stereo=False, seed=5):
    """A small joints file in the reference's format (prep/preprocess_kitti.py output): X[:,0] carries the row id so a
    loader's batches reveal the sampling order."""
    rng = np.random.RandomState(seed)
    dic = {'version': 'synthetic-1'}
    for phase, n in (('train', n_train), ('val', n_val)):
        X = rng.uniform(-3, 3, size=(n, 68 if stereo else 34))
        X[:, 0] = np.arange(n)
        Y = rng.uniform(0.5, 30, size=(n, 11 if stereo else 10))
        kps = rng.uniform(0, 1000, size=(n, 3, 17))
        clst = {}
        for name, lo, hi in (('10', 0, 10), ('20', 10, 20), ('30', 20, 30), ('>30', 30, 1e9)):
            sel = [i for i in range(n) if lo <= Y[i, 3] < hi]
            clst[name] = {'X': X[sel].tolist(), 'Y': Y[sel].tolist()}
        dic[phase] = {'X': X.tolist(), 'Y': Y.tolist(), 'names': ['%06d.png' % i for i in range(n)], 'kps': kps.tolist(),
                      'clst': clst}
    import json
    with open(path, 'w') as f:
        json.dump(dic, f)
    return dic


def make_kitti_case(net, n=7, seed=0):
    """Arguments of `save_txts(path, boxes, all_outputs, params, net, cat)` (eval/generate_kitti.py:119-147) for one image
    with n detections: float32 tensors shaped like `Loco.forward`'s dictionary entries, python lists elsewhere."""
    import torch
    rng = np.random.RandomState(seed)
    f32 = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))  # noqa: E731
    boxes = [[float(v) for v in np.round(rng.uniform(0, 1200, 4), 2)] + [float(rng.uniform(0.1, 1.0))] for _ in range(n)]
    cat = [float(v) for v in rng.choice([0.0, 0.05, 0.3, 1.0], size=n)]
    d = rng.uniform(3, 60, size=(n, 1))
    xyz = rng.uniform(-1, 1, size=(n, 3)) * d
    bi, epi = rng.uniform(0.1, 5, size=(n, 1)), rng.uniform(0, 1, size=n)
    kk = [[718.3351, 0., 600.3891], [0., 718.3351, 181.5122], [0., 0., 1.]]
    tt = [float(v) for v in rng.uniform(-0.5, 0.5, 3)]
    if net in ('monoloco_pp', 'monstereo'):
        outs = [f32(np.concatenate([xyz, d], 1)), f32(bi), [0.] * n if seed % 2 else f32(epi),
                (f32(rng.uniform(-3, 3, (n, 1))), f32(rng.uniform(-3, 3, (n, 1)))),
                f32(rng.uniform(1.4, 2, (n, 1))), f32(rng.uniform(0.4, 0.9, (n, 1))), f32(rng.uniform(0.4, 1.2, (n, 1)))]
    else:
        centers = f32(np.concatenate([rng.uniform(-1, 1, (n, 2)), np.ones((n, 1))], 1))
        zzs = [float(v) for v in rng.uniform(3, 60, n)]
        first = [[float(v) for v in row] for row in xyz] if net == 'baseline' else f32(d)
        outs = [first, f32(bi), f32(epi), zzs, centers]
    return boxes, outs, [kk, tt], cat


def make_crowd(n, seed=0, spacing=(0.3, 3.0)):
    """One image's people for the activity heuristics (Loco.social_distance inputs): n centres (x, z) in metres, each
    new one `spacing` m from an earlier one and at least spacing[0] from all, orientations in (-pi, pi], distances
    near |centre| and Laplace scales in [0.2, 1].  Python lists of floats, as post_process writes them."""
    rng = np.random.RandomState(seed)
    pts = []
    while len(pts) < n:
        if not pts:
            c = (rng.uniform(-3.0, 3.0), rng.uniform(4.0, 12.0))
        else:
            base = pts[rng.randint(len(pts))]
            r, a = rng.uniform(*spacing), rng.uniform(-math.pi, math.pi)
            c = (base[0] + r * math.cos(a), base[1] + r * math.sin(a))
        if all(math.hypot(c[0] - p[0], c[1] - p[1]) >= spacing[0] for p in pts):
            pts.append(c)
    centers = [[float(x), float(z)] for x, z in pts]
    angles = rng.uniform(-math.pi, math.pi, n).tolist()
    dds = [math.hypot(x, z) * float(rng.uniform(0.95, 1.05)) for x, z in centers]
    stds = rng.uniform(0.2, 1.0, n).tolist()
    return centers, angles, dds, stds


TRAINER_CLUSTERS = (('10', 0, 10), ('20', 10, 20), ('30', 20, 30), ('40', 30, 40), ('>40', 40, 1e9))


def make_trainer_joints(path, n_train=600, n_val=150, stereo=False, seed=11):
    """A joints file for Trainer runs: inputs like normalised keypoints, labels with the reference's column meaning
    (x, y, z, d, h, w, l, sin, cos, yaw(, aux)), d in [2, 48) m so that every cluster 10 / 20 / 30 / 40 has rows."""
    import json
    rng = np.random.RandomState(seed)
    dic = {'version': 'synthetic-trainer-1'}
    for phase, n in (('train', n_train), ('val', n_val)):
        X = rng.uniform(-1.5, 1.5, size=(n, 68 if stereo else 34))
        d = rng.uniform(2, 48, size=n)
        yaw = rng.uniform(-math.pi, math.pi, size=n)
        # a learnable signal: the first input columns carry the targets up to noise
        X[:, 0] = d / 16 - 1.5 + rng.normal(0, 0.05, n)
        X[:, 1] = np.sin(yaw) + rng.normal(0, 0.05, n)
        cols = [rng.uniform(-0.6, 0.6, n), rng.uniform(-0.2, 0.2, n), d * 0.95, d, rng.uniform(1.4, 2.0, n),
                rng.uniform(0.4, 0.9, n), rng.uniform(0.4, 1.2, n), np.sin(yaw), np.cos(yaw), yaw]
        if stereo:
            cols.append(rng.randint(0, 2, n).astype(np.float64))
        Y = np.stack(cols, 1)
        clst = {}
        for name, lo, hi in TRAINER_CLUSTERS:
            sel = [i for i in range(n) if lo <= Y[i, 3] < hi]
            clst[name] = {'X': X[sel].tolist(), 'Y': Y[sel].tolist()}
        kps = rng.uniform(0, 1000, size=(n, 3, 17))
        dic[phase] = {'X': X.tolist(), 'Y': Y.tolist(), 'names': ['%06d.png' % i for i in range(n)],
                      'kps': kps.tolist(), 'clst': clst}
    with open(path, 'w') as f:
        json.dump(dic, f)
    return dic
