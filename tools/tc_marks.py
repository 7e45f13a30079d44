"""Timeline of CTA (0,0) inside the tensor-core forward kernel (mlb_debug_fwd_marks), us: per layer of its first tile, then
per tile of group 0 (prologue, layers, head partials, stores).
    python tools/tc_marks.py [B]     (env: MLB_TC_CLUSTERS caps the group count)"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
import numpy as np, torch
from monoloco_b200 import synthetic, _lib as L_
from monoloco_b200.engine import LocoEngine

B = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
eng = LocoEngine(synthetic.make_state_dict('loco', 34, 9, 1024, 3, 7))
kps = torch.from_numpy(synthetic.make_keypoints(B, seed=1)).cuda()
kw = dict(kk=synthetic.KITTI_K, kind=L_.IN_KPS, kernel='tc')
lib = L_.lib()
buf = torch.zeros(256, dtype=torch.int64, device='cuda')
for _ in range(3):
    eng.forward(kps, **kw)
torch.cuda.synchronize()
L_.check(lib.mlb_debug_fwd_marks(C.c_void_p(buf.data_ptr())), 'marks')
eng.forward(kps, **kw)
torch.cuda.synchronize()
L_.check(lib.mlb_debug_fwd_marks(C.c_void_p(0)), 'marks')
m = buf.cpu().numpy().astype(np.int64)
groups = lib.mlb_tc_resident_clusters(eng._h)
tiles = (B + 63) // 64
print('B=%d: %d tiles of 64 rows on %d co-resident CTA groups of 4 CTAs = %d tile round(s); %s' % (
    B, tiles, groups, -(-tiles // groups), torch.cuda.get_device_name()))
t0 = m[128]
print('first tile of group 0, per layer (us from the layer start; layer start from the tile start):')
for g in range(15):
    s, first, issued, acc, epi, bar, prod, xiss = m[8 * g:8 * g + 8]
    if s == 0:
        break
    # the producer lane runs ahead: its marks of layer g can precede the layer's start on thread 0 (negative)
    print('  layer %d @%7.1f: X copies issued %+6.1f | first stage +%5.1f | MMAs issued +%5.1f | accumulators done +%5.1f | '
          'epilogue end +%5.1f | group barrier +%5.1f | producer done %+6.1f' % (
              g, (s - t0) / 1e3, (xiss - s) / 1e3, (first - s) / 1e3, (issued - s) / 1e3, (acc - s) / 1e3, (epi - s) / 1e3,
              (bar - s) / 1e3, (prod - s) / 1e3))
print('tiles of group 0 (us from the kernel\'s first mark):')
for t in range(4):
    start, pro, heads, stored = m[128 + 4 * t:132 + 4 * t]
    if start == 0:
        break
    print('  tile %d @%7.1f: prologue + barrier %5.1f | layers + head partials gathered %6.1f | rows stored +%5.1f | '
          'tile %6.1f' % (t, (start - t0) / 1e3, (pro - start) / 1e3, (heads - pro) / 1e3, (stored - heads) / 1e3,
                          (stored - start) / 1e3))
