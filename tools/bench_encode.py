"""Point clouds -> VAE latents on the GPU: CUDA-event times of Octree.build_octree (keys + radix sort + levels + fill +
node signal, csrc/points.cu), DualOctree, DualOctree.get_input_feature, the encoder network (encode_moments) and the
whole GraphVAE.extract_code, for B shapes x P points at depth 8 / full_depth 4 (reference configs/vae_snet_train.yaml).

The "port" arm is what the reference does in batch_to_cuda (models/octfusion_model_vae.py:135-146): one octree per
shape built by the ocnn restatement of oracle/restate_encode.py, run with CUDA tensors, then merge_octrees.  The two
arms alternate, repetition by repetition.  The card name and power limit are read in the same run.

The point count per shape is a parameter: ShapeNet's pointcloud.npz size is not available here, so 100 k seeded
ellipsoid-shell points with normals (octfusion_b200.synth.synth_shell_points) stand in for a shape.

usage: python tools/bench_encode.py [--batch 32] [--points 100000] [--reps 10] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

HBM_GBS = 3350.0        # H100 SXM data sheet, HBM3
DEPTH, FULL_DEPTH = 8, 4


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, power = [s.strip() for s in out.strip().split(',')[:2]]
        return {'name': name, 'power_limit': power}
    except Exception as e:  # noqa: BLE001
        return {'name': torch.cuda.get_device_name(), 'power_limit': 'unread (%s)' % e}


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1)


def build_bytes(octree, npts):
    """bytes the build must move at least: 24 B per point read (xyz + normal, fp32), the keys (8 B) and children
    (4 B) of every level it writes, and the per-node point and normal (24 B)"""
    out = 4 * int(octree.nnum[FULL_DEPTH]) + 12 * int(octree.nnum[FULL_DEPTH + 1:DEPTH + 1].sum())
    return 24 * npts + out + 24 * int(octree.nnum_nempty[DEPTH])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--points', type=int, default=100_000)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_encode: needs a CUDA device (there is no CPU measurement)')
    import bench
    from octfusion_b200 import Octree, Points, merge_points, DualOctree, graph_vae
    from octfusion_b200.synth import synth_shell_points
    from oracle import restate_encode as RE
    from tests.encode_util import assert_same_structure
    from tests.util import VAE
    torch.set_grad_enabled(False)
    dev = torch.device('cuda')
    shapes = [(x.to(dev), n.to(dev)) for x, n in synth_shell_points(args.batch, args.points, 0)]
    npts = args.batch * args.points
    pts = merge_points([Points(x, n) for x, n in shapes])
    net = bench.randomise_(graph_vae.GraphVAE(**VAE), 3).to(dev).eval()

    def ours():
        return Octree(DEPTH, FULL_DEPTH, args.batch, dev).build_octree(pts)

    def port():
        return RE.merge_octrees([RE.Octree(DEPTH, FULL_DEPTH, 1, dev).build_octree(RE.Points(x, n))
                                 for x, n in shapes])

    octree, port_octree = ours(), port()                    # warm-up of both arms, and the same octree from both
    assert_same_structure(octree, port_octree, DEPTH)
    doc = DualOctree(octree)
    feat = doc.get_input_feature()
    net.encode_moments(feat, doc)
    net.extract_code(octree)
    t = {k: [] for k in ('build', 'port_build', 'dual_octree', 'get_input_feature', 'encoder', 'extract_code')}
    for _ in range(args.reps):
        octree, ms = timed(ours)
        t['build'].append(ms)
        t['port_build'].append(timed(port)[1])
        doc, ms = timed(lambda: DualOctree(octree))
        t['dual_octree'].append(ms)
        feat, ms = timed(doc.get_input_feature)
        t['get_input_feature'].append(ms)
        t['encoder'].append(timed(lambda: net.encode_moments(feat, doc))[1])
        t['extract_code'].append(timed(lambda: net.extract_code(octree))[1])
    med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
    nbytes = build_bytes(octree, npts)
    line = {'what': 'point clouds -> octree -> ND features -> GraphVAE encoder (extract_code), fp32',
            'card': card(), 'batch': args.batch, 'points_per_shape': args.points, 'depth': DEPTH,
            'full_depth': FULL_DEPTH, 'nnum': octree.nnum.tolist(), 'nnum_nempty': octree.nnum_nempty.tolist(),
            'note': '%d seeded ellipsoid-shell points per shape stand in for a ShapeNet pointcloud.npz, whose size is '
                    'not available here' % args.points,
            'median_ms': med, 'min_ms': {k: min(v) for k, v in t.items()}, 'reps': args.reps,
            'build_points_per_s': npts / (med['build'] * 1e-3),
            'port_over_build': med['port_build'] / med['build'],
            'build_hbm': {'bound': 'HBM bandwidth, %.0f GB/s (H100 SXM data sheet)' % HBM_GBS, 'bytes': nbytes,
                          'share': nbytes / (HBM_GBS * 1e9) / (med['build'] * 1e-3)}}
    text = json.dumps(line)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(text + '\n')


if __name__ == '__main__':
    main()
