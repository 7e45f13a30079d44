"""Print the float64-rule ratio table (family x test x width: worst max / RMS ratio over the output columns) of
tests/test_forward_fp64_gpu.py.  Runs that test file on the GPU with MLB_FP64_RATIOS set, then formats what it wrote.

    python tools/fp64_ratios.py [-k expr] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('-k', default='', help='pytest -k expression (default: the whole file)')
    ap.add_argument('--json', default=None, help='also keep the raw ratios here')
    args = ap.parse_args()
    out = args.json or os.path.join(tempfile.mkdtemp(prefix='fp64_ratios_'), 'ratios.json')
    cmd = [sys.executable, '-m', 'pytest', '-q', '-m', 'gpu', '-p', 'no:cacheprovider',
           os.path.join(ROOT, 'tests', 'test_forward_fp64_gpu.py')] + (['-k', args.k] if args.k else [])
    rc = subprocess.call(cmd, cwd=ROOT, env=dict(os.environ, MLB_FP64_RATIOS=out))
    if not os.path.exists(out):
        sys.exit("no ratios written (pytest exit code %d)" % rc)
    with open(out) as f:
        ratios = json.load(f)
    print('%-8s %-18s %6s %10s %10s  %s' % ('family', 'test', 'width', 'max ratio', 'RMS ratio', 'per column (max)'))
    for key in sorted(ratios, key=lambda k: (k.split('|')[1], k.split('|')[0], float(k.split('|')[2]))):
        fam, test, width = key.split('|')
        mx, rms = ratios[key]
        if test in ('matrix', 'xyzc', 'feature', 'refresh', 'user_path'):
            print('%-8s %-18s %6s %10.2f %10.2f  %s' % (fam, test, width, max(mx), max(rms), ' '.join('%.2f' % v for v in mx)))
        else:
            print('%-8s %-18s %6s  %s | %s' % (fam, test, width, mx, rms))
    sys.exit(rc)


if __name__ == '__main__':
    main()
