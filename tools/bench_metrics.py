"""Shape-metric throughput on one GPU: `compute_all_metrics` (MMD, COV, 1-NNA with CD and approximate EMD) at
N_s = N_r clouds of P points against the reference arm (the reference's own approxmatch / matchcost / nndistance
kernels driven like reference `_pairwise_EMD_CD_`, oracle/ref_metrics.py) on the same inputs, alternating runs.

The reference arm is timed on `--ref-rows` rows of each of the three matrices (M_rs, M_rr, M_ss) and scaled to the
full matrices; the output says so.  Prints the card, its power limit and the SM clock sampled during the product's
EMD run, per-metric pair rates, CUDA-event kernel times, the EMD kernel's rate against its MUFU / FP32 bound, and the
largest relative difference to the reference arm on the rows it computed.  Writes nothing unless --out is given.

    python tools/bench_metrics.py [--n 512] [--points 2048] [--ref-rows 2] [--rounds 2] [--out result.json]
"""
from __future__ import annotations
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

LEVELS = 9
MUFU_PER_ELEM_LEVEL = 4          # ex2 in each of the 3 passes + sqrt in the cost pass
FP32_PER_ELEM_LEVEL = 30         # 3 x (6 for |b - a|^2, level and log2(e) scaling, accumulate) + 3 in the cost pass
MUFU_PER_CLK_SM = 16
FP32_PER_CLK_SM = 128            # 67 TFLOP/s (FMA = 2) at 1980 MHz on 132 SMs


def smi(fields):
    r = subprocess.run(['nvidia-smi', '--query-gpu=' + fields, '--format=csv,noheader,nounits', '-i', '0'],
                       capture_output=True, text=True, check=True)
    return [v.strip() for v in r.stdout.strip().splitlines()[0].split(',')]


class ClockSampler:
    """SM clock (MHz) sampled every 0.5 s while a measurement runs"""

    def __enter__(self):
        self.samples, self._stop = [], threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        return self

    def _run(self):
        while not self._stop.wait(0.5):
            self.samples.append(float(smi('clocks.sm')[0]))

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()

    def median(self):
        s = sorted(self.samples)
        return s[len(s) // 2] if s else float('nan')


def timed(fn):
    """(result, milliseconds) of fn() between CUDA events"""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=512)
    ap.add_argument('--points', type=int, default=2048)
    ap.add_argument('--ref-rows', type=int, default=2)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_metrics needs a CUDA device'
    from octfusion_b200 import metrics as M
    from octfusion_b200.synth import synth_point_clouds
    from oracle import ref_metrics as RM
    RM.load()

    n, p = args.n, args.points
    smp, ref = synth_point_clouds(n, p, 100).cuda(), synth_point_clouds(n, p, 101).cuda()
    mats = (('rs', ref, smp), ('rr', ref, ref), ('ss', smp, smp))
    pairs = 3 * n * n
    elems = float(p) * p
    name, power_limit, max_clock = smi('name,power.limit,clocks.max.sm')
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    # warm-up of every shape the timed window uses
    M.compute_all_metrics(smp[:8], ref[:8])
    M.pairwise_cd(smp[:8], ref[:8])
    RM.pairwise_emd_cd(ref[:1], smp[:8])
    torch.cuda.synchronize()

    rounds = []
    for _ in range(args.rounds):
        r = {}
        with ClockSampler() as clk:
            _, r['all_metrics_ms'] = timed(lambda: M.compute_all_metrics(smp, ref))
            outs, r['emd_cd_kernel_ms'] = {}, 0.0
            for tag, a, b in mats:
                outs[tag], ms = timed(lambda: M.pairwise_emd_cd(a, b))
                r['emd_cd_kernel_ms'] += ms
        r['sm_clock_mhz'] = clk.median()
        r['cd_kernel_ms'] = sum(timed(lambda: M.pairwise_cd(a, b))[1] for _, a, b in mats)
        # reference arm on the first ref_rows rows of each matrix, its CD and EMD halves timed apart
        ref_cd_ms = ref_emd_ms = 0.0
        worst_cd = worst_emd = 0.0
        for tag, a, b in mats:
            for i in range(args.ref_rows):
                for j0 in range(0, n, 256):
                    bj = b[j0:j0 + 256]
                    ai = a[i].view(1, -1, 3).expand(bj.shape[0], -1, -1).contiguous()
                    (d1, d2), ms = timed(lambda: RM.nn_distance(ai, bj))
                    cd_ref = d1.mean(1) + d2.mean(1)
                    ref_cd_ms += ms
                    cost, ms = timed(lambda: RM.match_cost(ai, bj))
                    ref_emd_ms += ms
                    cd_got, emd_got = outs[tag][0][i, j0:j0 + 256], outs[tag][1][i, j0:j0 + 256]
                    worst_cd = max(worst_cd, float(((cd_got - cd_ref).abs() / cd_ref.abs().clamp_min(1e-30)).max()))
                    emd_ref = cost / float(p)
                    worst_emd = max(worst_emd, float(((emd_got - emd_ref).abs() / emd_ref.abs()).max()))
        scale = n / args.ref_rows
        r.update(ref_cd_ms_scaled=ref_cd_ms * scale, ref_emd_ms_scaled=ref_emd_ms * scale,
                 max_rel_diff_cd=worst_cd, max_rel_diff_emd=worst_emd)
        rounds.append(r)

    best = {k: min(r[k] for r in rounds) for k in ('all_metrics_ms', 'emd_cd_kernel_ms', 'cd_kernel_ms',
                                                    'ref_cd_ms_scaled', 'ref_emd_ms_scaled')}
    clock = rounds[-1]['sm_clock_mhz']
    bound_clk = pairs * LEVELS * elems * max(MUFU_PER_ELEM_LEVEL / MUFU_PER_CLK_SM, FP32_PER_ELEM_LEVEL / FP32_PER_CLK_SM) / sms
    bound_ms = bound_clk / (clock * 1e3)
    res = {
        'card': name, 'power_limit_w': float(power_limit), 'sm_clock_mhz_during_emd': clock,
        'sm_clock_max_mhz': float(max_clock), 'sms': sms, 'clouds_per_side': n, 'points': p, 'pairs': pairs,
        'reference_arm': 'timed on %d of %d rows per matrix, scaled x%.0f' % (args.ref_rows, n, n / args.ref_rows),
        'compute_all_metrics_ms': best['all_metrics_ms'],
        'cd': {'kernel_ms': best['cd_kernel_ms'], 'pairs_per_s': pairs / best['cd_kernel_ms'] * 1e3,
               'ms_per_1k_pairs': best['cd_kernel_ms'] / pairs * 1e3,
               'ref_ms_scaled': best['ref_cd_ms_scaled'], 'ref_pairs_per_s': pairs / best['ref_cd_ms_scaled'] * 1e3,
               'speedup': best['ref_cd_ms_scaled'] / best['cd_kernel_ms']},
        'emd': {'kernel_ms': best['emd_cd_kernel_ms'], 'pairs_per_s': pairs / best['emd_cd_kernel_ms'] * 1e3,
                'ms_per_1k_pairs': best['emd_cd_kernel_ms'] / pairs * 1e3,
                'ref_ms_scaled': best['ref_emd_ms_scaled'], 'ref_pairs_per_s': pairs / best['ref_emd_ms_scaled'] * 1e3,
                'speedup': best['ref_emd_ms_scaled'] / best['emd_cd_kernel_ms'],
                'bound_ms': bound_ms, 'bound': 'MUFU' if MUFU_PER_ELEM_LEVEL / MUFU_PER_CLK_SM >=
                FP32_PER_ELEM_LEVEL / FP32_PER_CLK_SM else 'FP32',
                'share_of_bound': bound_ms / best['emd_cd_kernel_ms']},
        'speedup_all_metrics': (best['ref_cd_ms_scaled'] + best['ref_emd_ms_scaled']) / best['all_metrics_ms'],
        'max_rel_diff_cd': max(r['max_rel_diff_cd'] for r in rounds),
        'max_rel_diff_emd': max(r['max_rel_diff_emd'] for r in rounds),
        'rounds': rounds,
    }
    print('%s, power limit %s W, SM clock %.0f MHz during the EMD run (max %s)' % (name, power_limit, clock, max_clock))
    print('%d x %d clouds of %d points, %d pairs over M_rs, M_rr, M_ss; %s' % (n, n, p, pairs, res['reference_arm']))
    for k in ('cd', 'emd'):
        v = res[k]
        print('%-3s product %9.1f ms  %10.0f pairs/s  %7.3f ms/1k pairs | reference %10.1f ms  %9.0f pairs/s | x%.1f'
              % (k.upper(), v['kernel_ms'], v['pairs_per_s'], v['ms_per_1k_pairs'], v['ref_ms_scaled'],
                 v['ref_pairs_per_s'], v['speedup']))
    print('EMD bound (%s) %.1f ms: kernel at %.0f %% of it' % (res['emd']['bound'], bound_ms,
                                                                100 * res['emd']['share_of_bound']))
    print('compute_all_metrics %.1f ms (x%.1f over the reference arm); max rel diff CD %.2e, EMD %.2e'
          % (res['compute_all_metrics_ms'], res['speedup_all_metrics'], res['max_rel_diff_cd'], res['max_rel_diff_emd']))
    print(json.dumps(res))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    t0 = time.time()
    main()
    print('wall %.0f s' % (time.time() - t0))
