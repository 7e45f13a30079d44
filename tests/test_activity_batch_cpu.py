"""Batched activity heuristics without a GPU: the ctypes mirror of mlb_social_args against the header, the draw table
against the reference's Laplace samples (tests/golden/ref_activity_batch.npz, tools/gen_activity_golden.py), and the host
mirror (monoloco_b200.activity) against every flag and raised-hand code of that fixture."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


@pytest.fixture(scope='module')
def fix():
    return np.load(os.path.join(GOLDEN, 'ref_activity_batch.npz'))


def images(f):
    """(centers, angles, dds, stds, config dict, reference flags) per fixture image, as Python lists."""
    off = np.concatenate([[0], np.cumsum(f['n'])])
    for i in range(len(f['n'])):
        a, b, k = off[i], off[i + 1], int(f['cfg'][i])
        radii = tuple(float(r) for r in f['cfg_radii'][k] if not np.isnan(r))
        cfg = dict(social_distance=bool(f['cfg_social_distance'][k]), n_samples=int(f['cfg_n_samples'][k]),
                   threshold_prob=float(f['cfg_threshold_prob'][k]), threshold_dist=float(f['cfg_threshold_dist'][k]),
                   radii=radii)
        yield (f['xz'][a:b].tolist(), f['angles'][a:b].tolist(), f['dds'][a:b].tolist(), f['stds'][a:b].tolist(), cfg,
               f['flags'][a:b].tolist())


def test_social_args_layout_matches_header(tmp_path):
    from monoloco_b200 import _lib as L_
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "monoloco_b200.h"', 'int main(void) {',
             '  printf("sizeof %zu\\n", sizeof(mlb_social_args));',
             '  printf("MAX_PEOPLE %d\\n", MLB_SOCIAL_MAX_PEOPLE);', '  printf("MAX_RADII %d\\n", MLB_SOCIAL_MAX_RADII);']
    for fname, _ in L_.MlbSocialArgs._fields_:
        lines.append('  printf("%s %%zu\\n", offsetof(mlb_social_args, %s));' % (fname, fname))
    lines += ['  return 0;', '}']
    src = tmp_path / 'layout.c'
    src.write_text('\n'.join(lines))
    exe = tmp_path / 'layout'
    subprocess.run(['gcc', '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)],
                   check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], check=True, stdout=subprocess.PIPE,
                                                       text=True).stdout.splitlines())
    assert int(got['sizeof']) == C.sizeof(L_.MlbSocialArgs)
    for fname, _ in L_.MlbSocialArgs._fields_:
        assert int(got[fname]) == getattr(L_.MlbSocialArgs, fname).offset, fname
    assert int(got['MAX_PEOPLE']) == L_.SOCIAL_MAX_PEOPLE and int(got['MAX_RADII']) == L_.SOCIAL_MAX_RADII
    assert 'mlb_social_distance' in L_.EXPORTS and 'mlb_raising_hand' in L_.EXPORTS


def test_draw_table_equals_reference_stream(fix):
    from monoloco_b200.network.post import laplace_draw_table
    t = laplace_draw_table(fix['table'].size)
    assert t.dtype == torch.float32
    assert np.array_equal(t.numpy(), fix['table'])
    # a prefix stream: a longer table (as the device cache grows) starts with every shorter one
    assert np.array_equal(laplace_draw_table(150_000)[:fix['table'].size].numpy(), fix['table'])
    assert np.array_equal(laplace_draw_table(1).numpy(), fix['table'][:1])


def test_table_draws_equal_laplace_samples_per_image(fix):
    """For every fixture image: dds - |stds| * T[s * n + p] == Laplace(dds, |stds|).sample((S,)) under manual_seed(1),
    the draws laplace_sampling (process.py:101-122) makes, bit for bit."""
    from monoloco_b200.network.post import laplace_draw_table
    table = laplace_draw_table(100 * 64)
    checked = 0
    for _, _, dds, stds, cfg, _ in images(fix):
        n, S = len(dds), max(cfg['n_samples'], 7)
        if n == 0:
            continue
        mu, b = torch.tensor(dds), torch.abs(torch.tensor(stds))
        with torch.random.fork_rng(devices=[]):
            torch.manual_seed(1)
            ref = torch.distributions.Laplace(mu, b).sample((S,))
        got = mu[None, :] - b[None, :] * table[:S * n].view(S, n)
        assert torch.equal(got, ref), n
        checked += 1
    assert checked >= 50


def test_table_helper_leaves_global_generator_alone():
    from monoloco_b200.network.post import laplace_draw_table
    torch.manual_seed(1234)
    before = torch.get_rng_state().clone()
    laplace_draw_table(5000)
    assert torch.equal(torch.get_rng_state(), before)


def test_host_mirror_reproduces_fixture_flags(fix):
    """The per-image mirror behind Loco.social_distance on the whole corpus (sizes 0..64, every parameter set, the
    coincident centres): the yardstick the device flags are compared with in the GPU tests."""
    from monoloco_b200.activity import social_interactions
    seen = set()
    for centers, angles, dds, stds, cfg, ref in images(fix):
        got = [bool(social_interactions(i, centers, angles, dds, stds=stds, **cfg)) for i in range(len(centers))]
        assert got == ref, (len(centers), cfg)
        seen.add((cfg['n_samples'], cfg['social_distance'], cfg['radii']))
    assert len(seen) == 6
    assert 0 < int(fix['flags'].sum()) < fix['flags'].size


def test_host_mirror_reproduces_raising_hand_codes(fix):
    from monoloco_b200.activity import is_raising_hand
    names = (None, 'left', 'right', 'both')
    with np.errstate(invalid='ignore', divide='ignore'):
        got = [names.index(is_raising_hand(k.tolist())) for k in fix['kps']]
    assert got == fix['raising'].tolist()
    assert set(got) == {0, 1, 2, 3}


def test_laplace_argument_check_matches_reference_constructor():
    """check_laplace_args raises exactly where torch.distributions.Laplace(torch.tensor(dds), |torch.tensor(stds)|) does."""
    from monoloco_b200.network.post import check_laplace_args
    cases = [([5.0, 6.0], [0.3, -0.2]), ([5.0, 6.0], [0.3, 0.0]), ([float('nan'), 6.0], [0.3, 0.2]),
             ([5.0, 6.0], [0.3, float('nan')]), ([5.0, 6.0], [0.3, 1e-50]), ([float('inf'), 6.0], [0.3, 0.2]),
             ([5.0, 6.0], [0.3, float('inf')])]
    for dds, stds in cases:
        try:
            torch.distributions.Laplace(torch.tensor(dds), torch.abs(torch.tensor(stds)))
            ref_ok = True
        except ValueError:
            ref_ok = False
        if ref_ok:
            check_laplace_args(dds, stds)
        else:
            with pytest.raises(ValueError):
                check_laplace_args(dds, stds)
