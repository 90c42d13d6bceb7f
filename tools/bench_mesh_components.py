"""Mesh connected components and the largest-component filter (the clean=True step of export_mesh) on one GPU:
`connected_components` and `keep_largest_component` over the marching-cubes meshes of B seeded 256^3 ellipsoid-shell
grids (bench_mesh.shell_grids) with small island spheres added near the corners, so each shape has several
components, and over one N(0, 1) noise grid, whose tens of millions of faces in a huge number of components are close
to the worst case.  The numpy + scipy restatement (oracle/restate_mesh_components.py) runs on one shell mesh on the
CPU (`kind: "port"`; trimesh is not measured).

Prints the card, its power limit and the SM clock sampled during the GPU runs, CUDA-event ms per shape of the labelling
(`connected_components`) and of the whole filter (labelling, selection, the host synchronisation and the
compaction), faces per second, and the ratio to `marching_cubes` of the same grids.

    python tools/bench_mesh_components.py [--batch 32] [--size 256] [--rounds 3] [--out result.json]
"""
from __future__ import annotations
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_metrics import smi, ClockSampler, timed  # noqa: E402
from bench_mesh import shell_grids  # noqa: E402


def add_islands(sdfs, seed, count=4):
    """min with `count` spheres of 2-6 voxels radius near random corners of each grid (index-space SDF)"""
    g = torch.Generator().manual_seed(seed)
    B, R = sdfs.shape[0], sdfs.shape[1]
    x = torch.arange(R, dtype=torch.float32, device=sdfs.device)
    X, Y, Z = torch.meshgrid(x, x, x, indexing='ij')
    for b in range(B):
        for _ in range(count):
            u = torch.rand(4, generator=g, dtype=torch.float64)
            corner = (torch.randint(0, 2, (3,), generator=g) * 2 - 1).to(torch.float64)
            c = (1 + corner * (0.88 + 0.06 * u[:3])) * (R - 1) / 2
            rad = 2.0 + 4.0 * float(u[3])
            s = torch.sqrt((X - float(c[0])) ** 2 + (Y - float(c[1])) ** 2 + (Z - float(c[2])) ** 2) - rad
            torch.minimum(sdfs[b], s, out=sdfs[b])
    return sdfs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--size', type=int, default=256)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_mesh_components needs a CUDA device'
    from octfusion_b200.mesh import marching_cubes, connected_components, keep_largest_component
    from oracle import restate_mesh_components as RC

    B, R = args.batch, args.size
    name, power_limit, max_clock = smi('name,power.limit,clocks.max.sm')
    sdfs, noise = shell_grids(B, R, 0)
    sdfs = add_islands(sdfs, 1)
    meshes = marching_cubes(sdfs)
    noise_mesh = marching_cubes(noise)
    keep_largest_component(marching_cubes(sdfs[:2]))        # warm-up of every kernel the timed window uses
    torch.cuda.synchronize()

    rounds = []
    with ClockSampler() as clk:
        for _ in range(args.rounds):
            _, mc_ms = timed(lambda: marching_cubes(sdfs))
            (_, counts), cc_ms = timed(lambda: connected_components(meshes))
            kept, keep_ms = timed(lambda: keep_largest_component(meshes))
            _, noise_mc_ms = timed(lambda: marching_cubes(noise))
            (_, ncounts), noise_cc_ms = timed(lambda: connected_components(noise_mesh))
            nkept, noise_keep_ms = timed(lambda: keep_largest_component(noise_mesh))
            rounds.append(dict(marching_cubes_ms=mc_ms, components_ms=cc_ms, keep_largest_ms=keep_ms,
                               noise_marching_cubes_ms=noise_mc_ms, noise_components_ms=noise_cc_ms,
                               noise_keep_largest_ms=noise_keep_ms))
    best = {k: min(r[k] for r in rounds) for k in rounds[0]}
    faces = meshes.faces.shape[0]
    comps = counts.cpu().tolist()

    v0, f0 = (t.cpu().numpy() for t in meshes.mesh(0))
    t0 = time.perf_counter()
    wv, wf = RC.largest_component(v0, f0)
    port_ms = (time.perf_counter() - t0) * 1e3
    kv, kf = kept.mesh(0)
    assert np.array_equal(kv.cpu().numpy(), wv) and np.array_equal(kf.cpu().numpy(), wf)

    res = {
        'card': name, 'power_limit_w': float(power_limit), 'sm_clock_mhz': clk.median(),
        'sm_clock_max_mhz': float(max_clock), 'batch': B, 'size': R,
        'faces_per_shape_mean': faces / B, 'components_per_shape_mean': float(np.mean(comps)),
        'components_per_shape_min': min(comps), 'kept_faces_per_shape_mean': kept.faces.shape[0] / B,
        'connected_components_ms_per_shape': best['components_ms'] / B,
        'keep_largest_component_ms_per_shape': best['keep_largest_ms'] / B,
        'keep_largest_faces_per_s': faces / (best['keep_largest_ms'] * 1e-3),
        'marching_cubes_ms_per_shape': best['marching_cubes_ms'] / B,
        'keep_largest_over_marching_cubes': best['keep_largest_ms'] / best['marching_cubes_ms'],
        'noise_grid': {'faces': noise_mesh.num_faces(0), 'components': int(ncounts[0]),
                       'kept_faces': nkept.num_faces(0),
                       'connected_components_ms': best['noise_components_ms'],
                       'keep_largest_component_ms': best['noise_keep_largest_ms'],
                       'keep_largest_faces_per_s': noise_mesh.num_faces(0) / (best['noise_keep_largest_ms'] * 1e-3),
                       'marching_cubes_ms': best['noise_marching_cubes_ms'],
                       'keep_largest_over_marching_cubes': best['noise_keep_largest_ms'] / best['noise_marching_cubes_ms']},
        'port': {'kind': 'port', 'what': 'oracle/restate_mesh_components.largest_component, numpy + scipy, one shell mesh',
                 'faces': len(f0), 'ms_per_shape': port_ms,
                 'speedup': port_ms / (best['keep_largest_ms'] / B)},
        'rounds': rounds,
    }
    print('%s, power limit %s W, SM clock %.0f MHz (max %s)' % (name, power_limit, res['sm_clock_mhz'], max_clock))
    print('%d meshes of %d^3 grids: %.0f faces, %.1f components per shape (min %d)'
          % (B, R, res['faces_per_shape_mean'], res['components_per_shape_mean'], res['components_per_shape_min']))
    print('connected_components %.3f ms/shape, keep_largest_component %.3f ms/shape (%.2f G faces/s), '
          '%.2f x marching_cubes (%.3f ms/shape)'
          % (res['connected_components_ms_per_shape'], res['keep_largest_component_ms_per_shape'],
             res['keep_largest_faces_per_s'] / 1e9, res['keep_largest_over_marching_cubes'],
             res['marching_cubes_ms_per_shape']))
    n = res['noise_grid']
    print('noise grid: %d faces, %d components; connected_components %.2f ms, keep_largest_component %.2f ms '
          '(%.2f G faces/s), %.2f x marching_cubes' % (n['faces'], n['components'], n['connected_components_ms'],
                                                       n['keep_largest_component_ms'],
                                                       n['keep_largest_faces_per_s'] / 1e9,
                                                       n['keep_largest_over_marching_cubes']))
    print('numpy + scipy port %.0f ms on one shell mesh (x%.0f)' % (port_ms, res['port']['speedup']))
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
