"""Times of_gn_stats / of_gn_finalize / of_gn_apply alone at the full B=32 size: achieved GB/s against the HBM peak.
usage: python tools/prof_gn.py ; env REPS"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from octfusion_b200 import octree_from_splits, DualOctree
from octfusion_b200.synth import synth_splits
from octfusion_b200._lib import lib, ptr, stream, check, dt

B = 32
l4, l5 = synth_splits(B, 0)
doc = DualOctree(octree_from_splits(l4, l5, B, device='cuda'))
reps = int(os.environ.get('REPS', 10))
flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')


def timed(fn):
    fn(); fn()
    tot = 0.0
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / reps * 1e3


for d, c0, c1 in ((6, 128, 0), (6, 128, 128), (5, 256, 0), (5, 256, 256), (4, 512, 0), (4, 512, 512)):
    p = doc.plan[d]
    n = p.rows
    x0 = torch.randn((n, c0), device='cuda').bfloat16()
    x1 = torch.randn((n, c1), device='cuda').bfloat16() if c1 else None
    c = c0 + c1
    scale = torch.ones((B, c), device='cuda'); shift = torch.zeros((B, c), device='cuda')
    gam = torch.ones((1, c), device='cuda'); bet = torch.zeros((1, c), device='cuda')
    out = torch.empty((n, c), dtype=torch.bfloat16, device='cuda')
    a1 = (ptr(x1), x1.stride(0), c1) if x1 is not None else (None, 0, 0)
    sp = p.stat
    part = sp.new_part(c, 4)
    st = lambda: check(lib.of_gn_stats(ptr(x0), x0.stride(0), c0, a1[0], a1[1], a1[2], ptr(sp.chunk_seg), ptr(sp.seg_slot),  # noqa: E731
                                       ptr(p.batch_id), 0, n, dt(x0), 4, ptr(part), stream()))
    scratch = torch.empty(B * 8 * c, dtype=torch.float64, device='cuda')
    ticket = torch.zeros(64, dtype=torch.int32, device='cuda')
    fi = lambda: check(lib.of_gn_finalize(ptr(part), c, 4, None, 0, 4, ptr(sp.sample_seg_off), sp.n_seg, ptr(p.rows_of_sample), 0,  # noqa: E731
                                          ptr(gam), ptr(bet), B, 32, 1e-5, 1e-5, ptr(scale), ptr(shift), ptr(scratch), ptr(ticket),
                                          stream()))
    ap = lambda: check(lib.of_gn_apply(ptr(x0), x0.stride(0), c0, a1[0], a1[1], a1[2], ptr(p.batch_id), 0, n, ptr(scale),  # noqa: E731
                                       ptr(shift), 1, dt(x0), ptr(out), out.stride(0), 0, stream()))
    ts, tf, ta = timed(st), timed(fi), timed(ap)
    byt = n * c * 2
    print('depth %d rows %7d C %3d+%3d: stats %7.1f us %6.0f GB/s | finalize %6.1f us | apply %7.1f us %6.0f GB/s' %
          (d, n, c0, c1, ts, byt / ts / 1e3, tf, ta, 2 * byt / ta / 1e3))
