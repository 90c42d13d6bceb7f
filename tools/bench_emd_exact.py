"""Exact-EMD throughput on one GPU (csrc/emd_exact.cu through octfusion_b200.metrics) on the noisy ellipsoid shells of
tools/bench_metrics.py, against the reference's exact arm restated on the host (scipy linear_sum_assignment on fp32
distances, oracle/restate_emd_exact.py emd_exact, one process, `kind: "port"`).

Reports pairs/s of a paired batch and of an all-pairs and a symmetric (set against itself) matrix, the epsilon phases
and bidding rounds per pair from the status words, the certified gaps, the host solver's seconds per pair, the
projected time of compute_all_metrics(accelerated_emd=False) at --project x --project clouds, and the card, its power
limit and the SM clock sampled during the GPU runs.  Writes nothing unless --out is given.

    python tools/bench_emd_exact.py [--points 2048] [--batch 1024] [--side 128] [--host-pairs 3] [--out result.json]
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

import torch  # noqa: E402

from bench_metrics import smi, ClockSampler, timed  # noqa: E402


def per_pair_stats(status, gap):
    st = status.flatten().long().cpu()
    phases, rounds = (st >> 4) & 15, st >> 8
    r = rounds.double()
    return {'phases': int(phases.max()), 'rounds_mean': float(r.mean()), 'rounds_median': float(r.median()),
            'rounds_max': int(rounds.max()), 'gap_max': int(gap.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--points', type=int, default=2048)
    ap.add_argument('--batch', type=int, default=1024)
    ap.add_argument('--side', type=int, default=128)
    ap.add_argument('--host-pairs', type=int, default=3)
    ap.add_argument('--project', type=int, default=512)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_emd_exact needs a CUDA device'
    from octfusion_b200 import metrics as M
    from octfusion_b200.synth import synth_point_clouds
    from oracle import restate_emd_exact as R

    p = args.points
    x, y = synth_point_clouds(args.batch, p, 200).cuda(), synth_point_clouds(args.batch, p, 201).cuda()
    a, b = x[:args.side].contiguous(), y[:args.side].contiguous()
    name, power_limit, max_clock = smi('name,power.limit,clocks.max.sm')

    M.emd_exact(x[:4], y[:4])                                          # warm-up (module load, shared-memory attribute)
    torch.cuda.synchronize()
    runs = []
    for _ in range(args.rounds):
        r = {}
        with ClockSampler() as clk:
            (_, gap_p, st_p), r['paired_ms'] = timed(lambda: M.emd_exact(x, y, details=True))
            (_, gap_a, st_a), r['all_pairs_ms'] = timed(lambda: M.pairwise_emd_exact(a, b, details=True))
            (_, gap_s, st_s), r['symmetric_ms'] = timed(lambda: M.pairwise_emd_exact(a, a, details=True))
        r['sm_clock_mhz'] = clk.median()
        runs.append(r)
    best = {k: min(r[k] for r in runs) for k in ('paired_ms', 'all_pairs_ms', 'symmetric_ms')}
    n_paired, n_all, n_sym = args.batch, args.side * args.side, args.side * (args.side - 1) // 2

    # the reference's exact arm on the host: scipy on the fp32 distance matrix, one pair at a time
    xc, yc = x[:args.host_pairs].cpu(), y[:args.host_pairs].cpu()
    t0 = time.perf_counter()
    host = R.emd_exact(xc, yc)
    host_s = (time.perf_counter() - t0) / args.host_pairs
    dev = M.emd_exact(x[:args.host_pairs], y[:args.host_pairs]).cpu()

    # compute_all_metrics(accelerated_emd=False) at project x project: M_rs in full, M_rr and M_ss as triangles; the
    # reference solves all three matrices in full
    n = args.project
    sym_rate = n_sym / best['symmetric_ms'] * 1e3
    all_rate = n_all / best['all_pairs_ms'] * 1e3
    proj_s = n * n / all_rate + 2 * (n * (n - 1) // 2) / sym_rate
    ref_pairs = 3 * n * n
    res = {
        'card': name, 'power_limit_w': float(power_limit), 'sm_clock_mhz': runs[-1]['sm_clock_mhz'],
        'sm_clock_max_mhz': float(max_clock), 'points': p,
        'paired': dict(pairs=n_paired, ms=best['paired_ms'], pairs_per_s=n_paired / best['paired_ms'] * 1e3,
                       **per_pair_stats(st_p, gap_p)),
        'all_pairs': dict(shape=[args.side, args.side], pairs=n_all, ms=best['all_pairs_ms'], pairs_per_s=all_rate,
                          **per_pair_stats(st_a, gap_a)),
        'symmetric': dict(shape=[args.side, args.side], pairs_solved=n_sym, ms=best['symmetric_ms'],
                          pairs_per_s=sym_rate, **per_pair_stats(st_s, gap_s)),
        'host': {'kind': 'port', 'solver': 'scipy.optimize.linear_sum_assignment on fp32 distances, one core',
                 'pairs': args.host_pairs, 's_per_pair': host_s,
                 'max_abs_diff_to_gpu': float((host.double() - dev.double()).abs().max())},
        'projection': {'clouds_per_side': n, 'gpu_pairs_solved': n * n + n * (n - 1), 'gpu_s': proj_s,
                       'reference_pairs': ref_pairs, 'host_core_hours': ref_pairs * host_s / 3600.0},
        'runs': runs,
    }
    print('%s, power limit %s W, SM clock %.0f MHz (max %s); %d points per cloud'
          % (name, power_limit, res['sm_clock_mhz'], max_clock, p))
    for k in ('paired', 'all_pairs', 'symmetric'):
        v = res[k]
        print('%-9s %8.1f ms  %8.1f pairs/s  phases %d  rounds/pair mean %.0f median %.0f max %d  gap max %d'
              % (k, v['ms'], v['pairs_per_s'], v['phases'], v['rounds_mean'], v['rounds_median'], v['rounds_max'],
                 v['gap_max']))
    print('host scipy %.3f s/pair (max |diff| to GPU %.2e); compute_all_metrics(accelerated_emd=False) at %d x %d: '
          'GPU %.0f s projected, reference arm %.0f core-hours'
          % (host_s, res['host']['max_abs_diff_to_gpu'], n, n, proj_s, res['projection']['host_core_hours']))
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
