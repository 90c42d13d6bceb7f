"""TEST INFRASTRUCTURE.  Regenerates tests/golden/metrics_emd_exact.npz from the UNMODIFIED reference
metrics/evaluation_metrics.py (imported from the checkout named by OCTFUSION_REFERENCE):

    python -m oracle.gen_golden_emd_exact

Its `from .StructuralLosses...` imports fail in a plain checkout, so every EMD it computes is the exact arm
`emd_approx` (scipy linear_sum_assignment on fp32 distances) and every CD is `distChamfer`.  Stored: input checksums,
`emd_approx` on paired batches of 1 .. 4096 points, `EMD_CD(accelerated_emd=False)` per pair and reduced,
`_pairwise_EMD_CD_` of the three matrices of compute_1_nna, `compute_cov_mmd` and `compute_1_nna`.

The clouds are ellipsoid shells on the dyadic grid 2^-10 inside the unit cube: distChamfer's |x|^2 + |y|^2 - 2 x.y
is then exact in fp32 (products carry 20 fractional bits, sums stay below 2^3), so its CD equals the per-point
nearest-neighbour CD up to the order of the mean, and the fixtures pin the EMD arm alone.
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

PAIRED = ((1, 4), (2, 4), (3, 4), (17, 4), (128, 3), (1000, 2), (2048, 2), (4096, 1))   # (points, pairs)


def shells(n, points, g):
    """[n, points, 3] fp32 noisy ellipsoid shells (semi-axes 0.2 .. 0.45, centre in [0.45, 0.55]^3) rounded to 2^-10"""
    d = torch.randn(n, points, 3, generator=g, dtype=torch.float64)
    d = d / d.norm(dim=-1, keepdim=True)
    axes = 0.2 + 0.25 * torch.rand(n, 1, 3, generator=g, dtype=torch.float64)
    centre = 0.45 + 0.1 * torch.rand(n, 1, 3, generator=g, dtype=torch.float64)
    radial = 1.0 + 0.01 * torch.randn(n, points, 1, generator=g, dtype=torch.float64)
    return (torch.round((centre + d * axes * radial) * 1024) / 1024).float().contiguous()


def emd_exact_inputs():
    """seeded inputs: 8 sample and 8 reference clouds of 512 points (the first three samples are noisy copies of
    references, so COV and 1-NNA are not trivial) and one paired batch (x, y) per entry of PAIRED"""
    g = torch.Generator().manual_seed(53)
    ref = shells(8, 512, g)
    smp = shells(8, 512, g)
    noise = 0.004 * torch.randn(3, 512, 3, generator=g, dtype=torch.float64)
    smp[:3] = (torch.round((ref[:3].double() + noise) * 1024) / 1024).float()
    inp = {'smp': smp.contiguous(), 'ref': ref}
    for n, b in PAIRED:
        inp['x%d' % n] = shells(b, n, g)
        inp['y%d' % n] = shells(b, n, g)
    return inp


def main():
    torch.set_grad_enabled(False)
    ref_import.load()
    em = importlib.import_module('metrics.evaluation_metrics')
    inp = emd_exact_inputs()
    fx = {k + '_sum': checksum(v) for k, v in inp.items()}
    for n, _ in PAIRED:
        fx['emd%d' % n] = em.emd_approx(inp['x%d' % n], inp['y%d' % n]).numpy()
    smp, ref = inp['smp'], inp['ref']
    per_pair = em.EMD_CD(smp, ref, 3, accelerated_emd=False, reduced=False)
    reduced = em.EMD_CD(smp, ref, 3, accelerated_emd=False)
    for k in ('MMD-CD', 'MMD-EMD'):
        fx['emd_cd_pairs_' + k] = per_pair[k].numpy()
        fx['emd_cd_' + k] = float(reduced[k])
    for tag, a, b in (('rs', ref, smp), ('rr', ref, ref), ('ss', smp, smp)):
        cd, emd = em._pairwise_EMD_CD_(a, b, 3)
        fx['m_%s_cd' % tag], fx['m_%s_emd' % tag] = cd.numpy(), emd.numpy()
    for k, v in em.compute_cov_mmd(smp, ref, 3).items():
        fx['cov_mmd_' + k] = float(v)
    for k, v in em.compute_1_nna(smp, ref, 3).items():
        fx['1nna_' + k] = float(v)
    path = os.path.join(OUT, 'metrics_emd_exact.npz')
    np.savez_compressed(path, **fx)
    print('metrics_emd_exact.npz', os.path.getsize(path) // 1024, 'KB')


if __name__ == '__main__':
    main()
