"""TEST INFRASTRUCTURE.  Regenerates tests/golden/metrics.npz from the UNMODIFIED reference
metrics/evaluation_metrics.py (imported from the checkout named by OCTFUSION_REFERENCE; its CUDA extension is not
built there, so it runs on its CPU paths):

    python -m oracle.gen_golden_metrics

Only this fixture is written.  It stores the input checksums and `distChamfer` on float64 clouds, `lgan_mmd_cov` and
`knn(..., 1)` on seeded matrices.  The reference's CPU `emd_approx` is an exact (Hungarian) EMD, a different quantity
from the approximate EMD of its CUDA kernels, so nothing is pinned against it.
"""
import importlib
import os
import sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_import                                    # noqa: E402
from oracle.gen_golden import OUT, checksum                      # noqa: E402


def metrics_inputs():
    """seeded inputs of metrics.npz: two batches of float64 clouds (uniform in the unit cube) and the blocks of a
    joint distance matrix (Mxx [10, 10], Mxy [10, 8], Myy [8, 8]) with its own [12, 9] sample x reference matrix"""
    g = torch.Generator().manual_seed(41)
    x = torch.rand(3, 64, 3, generator=g, dtype=torch.float64)
    y = torch.rand(3, 64, 3, generator=g, dtype=torch.float64)
    m = torch.rand(18, 18, generator=g)
    m = m + m.t()
    return {'x': x, 'y': y, 'mxx': m[:10, :10].contiguous(), 'mxy': m[:10, 10:].contiguous(),
            'myy': m[10:, 10:].contiguous(), 'all_dist': torch.rand(12, 9, generator=g)}


def main():
    torch.set_grad_enabled(False)
    ref_import.load()
    em = importlib.import_module('metrics.evaluation_metrics')
    inp = metrics_inputs()
    fx = {k + '_sum': checksum(v) for k, v in inp.items()}
    d1, d2 = em.distChamfer(inp['x'], inp['y'])
    fx['dist1'], fx['dist2'] = d1.numpy(), d2.numpy()
    for k, v in em.lgan_mmd_cov(inp['all_dist']).items():
        fx['lgan_' + k] = float(v)
    for k, v in em.knn(inp['mxx'], inp['mxy'], inp['myy'], 1).items():
        fx['knn_' + k] = float(v)
    np.savez_compressed(os.path.join(OUT, 'metrics.npz'), **fx)
    print('metrics.npz', os.path.getsize(os.path.join(OUT, 'metrics.npz')) // 1024, 'KB')


if __name__ == '__main__':
    main()
