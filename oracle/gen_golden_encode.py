"""TEST INFRASTRUCTURE.  Writes tests/golden/vae_encode_points.npz by running the UNMODIFIED reference (imported under
the ocnn shim, see oracle/gen_golden.py) on seeded point clouds:

    python -m oracle.gen_golden_encode

points -> ocnn Octree.build_octree (oracle/restate_encode.py: parity UNPINNED at the ocnn boundary, SURVEY.md
Appendix B) -> reference DualOctree.get_input_feature (dual_octree.py:343-360) -> reference GraphVAE.extract_code
(graph_vae.py:291-298) and GraphVAE.forward(evaluate=True) (:246-289), each after torch.manual_seed.  Octrees are
stored as digests, float results as row samples, so that the fixture stays far below 1 MB.
"""
import os
import sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_import, restate_encode as RE              # noqa: E402
from tests.util import VAE, vae_state_dict, digest               # noqa: E402
from tests.encode_util import (FIXTURE, CODE_SEED, FORWARD_SEED, ROW_STEP, fixture_shapes,  # noqa: E402
                               oracle_build)


def main():
    import importlib
    ref_import.load()
    torch.set_grad_enabled(False)
    shapes = fixture_shapes()
    octree = oracle_build(shapes, VAE['depth'], VAE['full_depth'])
    D, fd = VAE['depth'], VAE['full_depth']
    fx = {'xyz_sum': float(sum(x.double().abs().sum() for x, _ in shapes)),
          'normal_sum': float(sum(n.double().abs().sum() for _, n in shapes)),
          'nnum': octree.nnum.numpy(), 'nnum_nempty': octree.nnum_nempty.numpy(),
          'points': octree.points[D][::ROW_STEP].numpy(), 'normals': octree.normals[D][::ROW_STEP].numpy()}
    for d in range(fd, D + 1):
        fx['keys%d' % d] = digest(octree.keys[d])
        fx['children%d' % d] = digest(octree.children[d])
    dual_octree = importlib.import_module('models.networks.dualoctree_networks.dual_octree')
    # the reference's source is untouched: only the third-party name it imported (dual_octree.py:14) is bound to the
    # restatement, which the ocnn shim does not provide
    dual_octree.InputFeature = RE.InputFeature
    doc = dual_octree.DualOctree(octree)
    doc.post_processing_for_docnn()
    feat = doc.get_input_feature()
    fx['feature_rows'] = feat.shape[0]
    fx['feature'] = feat[::ROW_STEP].numpy()
    gv = importlib.import_module('models.networks.dualoctree_networks.graph_vae')
    net = gv.GraphVAE(**VAE).eval()
    net.load_state_dict(vae_state_dict())
    torch.manual_seed(CODE_SEED)
    z, _ = net.extract_code(octree)
    fx['code'] = z[::4].numpy()
    fx['code_rows'] = z.shape[0]
    torch.manual_seed(FORWARD_SEED)
    out = net.forward(octree, evaluate=True)
    fx['kl_loss'], fx['code_max'], fx['code_min'] = (float(out[k]) for k in ('kl_loss', 'code_max', 'code_min'))
    fx['out_nnum'] = out['octree_out'].nnum.numpy()
    for d in (6, 7, 8):
        lg = out['logits'][d]
        fx['label%d' % d] = np.packbits(lg.argmax(1).numpy().astype(np.uint8))
        fx['margin%d' % d] = float((lg[:, 0] - lg[:, 1]).abs().min())
        fx['logit%d' % d] = lg[::ROW_STEP].numpy()
        fx['reg%d' % d] = out['reg_voxs'][d][::ROW_STEP].numpy()
    path = FIXTURE
    np.savez_compressed(path, **fx)
    print('nnum', fx['nnum'].tolist(), 'nempty', fx['nnum_nempty'].tolist(), 'out nnum', fx['out_nnum'].tolist(),
          'kl %.5f' % fx['kl_loss'], os.path.getsize(path) // 1024, 'KB')


if __name__ == '__main__':
    main()
