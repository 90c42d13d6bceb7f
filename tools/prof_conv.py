"""One GraphConv (tensor-core tap-gather GEMM) at the full B=32 size, timed with CUDA events.
usage: python tools/prof_conv.py [depth cin cout] ; env REPS"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from octfusion_b200 import octree_from_splits, DualOctree
from octfusion_b200.synth import synth_splits
from octfusion_b200.modules import GraphConv

B = int(os.environ.get('BATCH', 32))
l4, l5 = synth_splits(B, 0)
doc = DualOctree(octree_from_splits(l4, l5, B, device='cuda'))
if os.environ.get('SHAPES'):                     # "6,128,128;6,256,256": several layers in one process
    shapes = [tuple(int(v) for v in sh.split(',')) for sh in os.environ['SHAPES'].split(';')]
else:
    shapes = [tuple(int(a) for a in (sys.argv[1:4] or (6, 128, 128)))]
for d, cin, cout in shapes:
    n = doc.plan[d].rows
    x = torch.randn((n, cin), device='cuda').bfloat16()
    conv = GraphConv(cin, cout, 7, 7, d - 1).cuda()
    reps = int(os.environ.get('REPS', 5))
    if os.environ.get('EPI'):          # EPI=stats,emb,resid: the epilogue extras of a GraphResBlockEmbed conv
        epi = {}
        p = doc.plan[d]
        if 'stats' in os.environ['EPI']: epi['stats'] = p.stat
        if 'emb' in os.environ['EPI']: epi.update(row_add=torch.randn((B, cout), device='cuda'), row_add_idx=p.batch_id)
        if 'resid' in os.environ['EPI']: epi['resid'] = torch.randn((n, cout), device='cuda').bfloat16()
        conv_ = conv
        conv = lambda x, doc, d: conv_.run(x, doc.plan[d], **epi)
    for _ in range(2):
        y = conv(x, doc, d)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        y = conv(x, doc, d)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    k = 7 * (cin + d - 1)
    print('depth %d rows %d K %d N %d: %.1f us  %.1f TFLOP/s' % (d, n, k, cout, ms * 1e3, 2.0 * n * k * cout / ms / 1e9))
