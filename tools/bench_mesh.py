"""Mesh and metric-point-cloud throughput on one GPU: `marching_cubes` and `pointclouds_from_sdfs(n=2048)` over a
batch of B seeded 256^3 SDF grids (ellipsoid shells like synth's) and on one Gaussian-noise grid (close to the most
triangles a grid can have), against the numpy restatement (oracle/restate_mesh.py) on one shell grid
on the CPU (`kind: "port"`; skimage is not measured).

Prints the card, its power limit and the SM clock sampled during the GPU runs, ms per shape, triangles per shape,
CUDA-event times of the count and emit passes with the grid bytes they read against the 3.35 TB/s data-sheet HBM
rate (each pass reads the 4 R^3-byte grid at least once), and the calc_sdf time of one 256^3 grid of the golden
depth-8 VAE octree (tests/golden/vae_decode.npz), so the share of the evaluation spent on meshes is visible.

    python tools/bench_mesh.py [--batch 32] [--size 256] [--rounds 3] [--out result.json]
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

HBM_BYTES_PER_S = 3.35e12


def shell_grids(batch, size, seed):
    """([batch, size, size, size] fp32 SDFs (index space) of random ellipsoid shells, [1, size, size, size] N(0, 1))"""
    g = torch.Generator().manual_seed(seed)
    x = torch.arange(size, dtype=torch.float32, device='cuda') / (size - 1) * 2 - 1
    X, Y, Z = torch.meshgrid(x, x, x, indexing='ij')
    out = torch.empty(batch, size, size, size, device='cuda')
    for b in range(batch):
        u = torch.rand(8, generator=g, dtype=torch.float64)
        centre = (u[0:3] * 2 - 1) * 0.15
        r = 0.45 + 0.30 * u[3]
        axes = (0.6 + 0.8 * u[4:7]) * r
        f = torch.sqrt(((X - centre[0]) / axes[0]) ** 2 + ((Y - centre[1]) / axes[1]) ** 2
                       + ((Z - centre[2]) / axes[2]) ** 2)
        out[b] = (f - 1.0) * float(axes.mean()) * (size - 1) / 2
    return out, torch.randn(1, size, size, size, generator=g).cuda()


def pass_times(sdfs):
    """(count pass ms, emit pass ms) over the batch, CUDA events around each shape's kernel"""
    from octfusion_b200._lib import lib, ptr, stream, check
    B, R = sdfs.shape[0], sdfs.shape[1]
    n = R ** 3
    vc, tc = (torch.empty(n, dtype=torch.int32, device='cuda') for _ in range(2))
    vs, ts = (torch.empty(n + 1, dtype=torch.int32, device='cuda') for _ in range(2))
    scratch = torch.empty(int(lib.of_scan_scratch_bytes(n)), dtype=torch.uint8, device='cuda')
    st = stream()
    count_ms = emit_ms = 0.0
    for b in range(B):
        g = sdfs[b]
        _, ms = timed(lambda: check(lib.of_mc_count(ptr(g), R, 0.0, ptr(vc), ptr(tc), st)))
        count_ms += ms
        check(lib.of_exclusive_scan_i32(ptr(vc), ptr(vs), n, None, ptr(scratch), st))
        check(lib.of_exclusive_scan_i32(ptr(tc), ptr(ts), n, None, ptr(scratch), st))
        nv, nf = int(vs[n]), int(ts[n])
        verts = torch.empty(max(nv, 1), 3, device='cuda')
        faces = torch.empty(max(nf, 1), 3, dtype=torch.int32, device='cuda')
        _, ms = timed(lambda: check(lib.of_mc_emit(ptr(g), R, 0.0, ptr(vs), ptr(ts), ptr(verts), ptr(faces), st)))
        emit_ms += ms
    return count_ms, emit_ms


def calc_sdf_ms(size):
    """one size^3 calc_sdf grid of the golden depth-8 VAE octree (random regression values)"""
    from tests import util as U
    from octfusion_b200 import graph_vae
    from octfusion_b200.mpu import NeuralMPU, calc_sdf
    g = np.load(os.path.join(U.GOLDEN, 'vae_decode.npz'))
    po = graph_vae.GraphVAE(**U.VAE).create_child_octree(U.product_doctree(1, 0).octree)
    for d in (6, 7, 8):
        po.octree_split(torch.from_numpy(np.unpackbits(g['label%d' % d])[: int(g['nnum'][d])].astype(np.int64)).cuda(), d)
        if d < 8:
            po.octree_grow(d + 1)
            po.depth += 1
    gen = torch.Generator().manual_seed(33)
    reg = {d: torch.randn(int(po.nnum[4:d + 1].sum()), 4, generator=gen).cuda() for d in (6, 7, 8)}
    mpu = NeuralMPU(4, 6, 8)

    def model(pos):
        return mpu(pos, reg, po)[8][0]
    model.mpu_args = (mpu, reg, po)
    calc_sdf(model, 1, size, 64 ** 3, -0.9, 0.9)
    return min(timed(lambda: calc_sdf(model, 1, size, 64 ** 3, -0.9, 0.9))[1] for _ in range(3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--size', type=int, default=256)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_mesh needs a CUDA device'
    from octfusion_b200.mesh import marching_cubes, pointclouds_from_sdfs
    from oracle import restate_mesh as RM

    B, R = args.batch, args.size
    name, power_limit, max_clock = smi('name,power.limit,clocks.max.sm')
    sdfs, noise = shell_grids(B, R, 0)
    marching_cubes(sdfs[:2])                           # warm-up of every kernel the timed window uses
    pointclouds_from_sdfs(sdfs[:2])
    torch.cuda.synchronize()

    rounds = []
    with ClockSampler() as clk:
        for _ in range(args.rounds):
            m, mc_ms = timed(lambda: marching_cubes(sdfs))
            _, pc_ms = timed(lambda: pointclouds_from_sdfs(sdfs, n=2048))
            count_ms, emit_ms = pass_times(sdfs)
            mn, noise_mc_ms = timed(lambda: marching_cubes(noise))
            _, noise_pc_ms = timed(lambda: pointclouds_from_sdfs(noise, n=2048))
            rounds.append(dict(marching_cubes_ms=mc_ms, pointclouds_ms=pc_ms, count_pass_ms=count_ms,
                               emit_pass_ms=emit_ms, noise_marching_cubes_ms=noise_mc_ms,
                               noise_pointclouds_ms=noise_pc_ms))
    sdf_ms = calc_sdf_ms(R)
    best = {k: min(r[k] for r in rounds) for k in rounds[0]}
    tris = [m.num_faces(b) for b in range(B)]
    grid_bytes = 4.0 * R ** 3 * B

    shell = sdfs[0].cpu().numpy()
    t0 = time.perf_counter()
    _, f_port = RM.marching_cubes(shell)
    port_ms = (time.perf_counter() - t0) * 1e3
    assert len(f_port) == tris[0]

    res = {
        'card': name, 'power_limit_w': float(power_limit), 'sm_clock_mhz': clk.median(),
        'sm_clock_max_mhz': float(max_clock), 'batch': B, 'size': R,
        'marching_cubes_ms_per_shape': best['marching_cubes_ms'] / B,
        'pointclouds_from_sdfs_ms_per_shape': best['pointclouds_ms'] / B,
        'triangles_per_shell_mean': float(np.mean(tris)), 'triangles_per_shell_max': max(tris),
        'noise_grid': {'triangles': mn.num_faces(0), 'marching_cubes_ms': best['noise_marching_cubes_ms'],
                       'pointclouds_from_sdfs_ms': best['noise_pointclouds_ms']},
        'count_pass': {'ms': best['count_pass_ms'], 'grid_GB_per_s': grid_bytes / best['count_pass_ms'] / 1e6,
                       'share_of_hbm': grid_bytes / best['count_pass_ms'] / 1e-3 / HBM_BYTES_PER_S},
        'emit_pass': {'ms': best['emit_pass_ms'], 'grid_GB_per_s': grid_bytes / best['emit_pass_ms'] / 1e6,
                      'share_of_hbm': grid_bytes / best['emit_pass_ms'] / 1e-3 / HBM_BYTES_PER_S},
        'calc_sdf_ms_per_shape': sdf_ms,
        'mesh_share_of_sdf_plus_pointclouds': (best['pointclouds_ms'] / B) / (best['pointclouds_ms'] / B + sdf_ms),
        'port': {'kind': 'port', 'what': 'oracle/restate_mesh.marching_cubes, numpy, one shell grid',
                 'ms_per_shape': port_ms, 'speedup': port_ms / (best['marching_cubes_ms'] / B)},
        'rounds': rounds,
    }
    print('%s, power limit %s W, SM clock %.0f MHz (max %s)' % (name, power_limit, res['sm_clock_mhz'], max_clock))
    print('%d grids of %d^3: marching_cubes %.2f ms/shape, pointclouds_from_sdfs(2048) %.2f ms/shape; calc_sdf %.2f ms'
          % (B, R, res['marching_cubes_ms_per_shape'], res['pointclouds_from_sdfs_ms_per_shape'], sdf_ms))
    print('triangles: %.0f per shell (max %d)' % (res['triangles_per_shell_mean'], max(tris)))
    print('noise grid: %d triangles, marching_cubes %.2f ms, pointclouds_from_sdfs(2048) %.2f ms'
          % (mn.num_faces(0), best['noise_marching_cubes_ms'], best['noise_pointclouds_ms']))
    for k in ('count_pass', 'emit_pass'):
        v = res[k]
        print('%-10s %8.2f ms  %7.0f GB/s of grid  %4.0f %% of 3.35 TB/s' % (k, v['ms'], v['grid_GB_per_s'],
                                                                              100 * v['share_of_hbm']))
    print('numpy port %.0f ms per shell grid (x%.0f)' % (port_ms, res['port']['speedup']))
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
