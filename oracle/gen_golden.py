"""TEST INFRASTRUCTURE.  Regenerates tests/golden/*.npz by running the UNMODIFIED reference
(a checkout of octree-nn/octfusion, imported under the ocnn shim; its location is OCTFUSION_REFERENCE):

    python -m oracle.gen_golden

The fixtures are all the tests ever see of the reference: they pin both the oracle (`-m "not gpu"`) and the CUDA
path (`-m gpu`).  Inputs are regenerated from seeds by the tests; the stored input checksums guard against a drifting
generator.  Large integer results (graphs, octrees) are stored as sha256 digests (tests.util.digest), large float
results as a fixed row sample, so that every fixture stays below 1 MB.
"""
import os
import sys
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_import, restate as R                      # noqa: E402
from oracle.octree_util import octree_from_splits                # noqa: E402
from octfusion_b200.synth import synth_splits                    # noqa: E402
from tests.util import UNCOND, SMALL, COND, digest               # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden')


def checksum(t: torch.Tensor) -> float:
    return float(t.double().abs().sum())


def seeded_inputs(n, c, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, c, generator=g)


def mpu_inputs(octree, npts=2000, seed=21):
    """seeded query points (half near occupied depth-8 cells, half uniform) and regression values for mpu tests."""
    gen = torch.Generator().manual_seed(seed)
    reg = {d: torch.randn(int(octree.nnum[4:d + 1].sum()), 4, generator=gen) for d in (6, 7, 8)}
    x, y, z, b = octree.xyzb(8)
    pick = torch.randperm(x.numel(), generator=gen)[:npts]
    near = (torch.stack([x, y, z], 1)[pick].float() + torch.rand(npts, 3, generator=gen)) / 128.0 - 1.0
    uni = torch.rand(npts, 3, generator=gen) * 2 - 1
    pos = torch.cat([torch.cat([near, uni]), torch.zeros(2 * npts, 1)], 1)
    return pos, reg


def mpu_fixture():
    """outputs of the unmodified reference NeuralMPU (mpu.py:143-155; its hard-coded `.cuda()` patched to identity)."""
    import importlib
    from tests import util as U
    ref_import.load()
    mpu = importlib.import_module('models.networks.dualoctree_networks.mpu')
    g = np.load(os.path.join(OUT, 'vae_decode.npz'))
    labels = {d: torch.from_numpy(np.unpackbits(g['label%d' % d])[: int(g['nnum'][d])].astype(np.int64)) for d in (6, 7, 8)}
    octree = U.oracle_grown_octree(labels)
    pos, reg = mpu_inputs(octree)
    orig = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        out = mpu.NeuralMPU(4, 6, 8)(pos, reg, octree)
    finally:
        torch.Tensor.cuda = orig
    fx = {'pos_sum': checksum(pos), 'reg_sum': sum(checksum(v) for v in reg.values())}
    for d in (6, 7, 8):
        fx['fval%d' % d] = out[d][0].numpy()
        fx['flag%d' % d] = np.packbits(out[d][1].numpy())
    return fx


# round-2 additions to UNET_CASES (tests/util.py): the benchmarked 8-channel config and the cond config at the shard
# size of BASELINE.json configs[4] (B = 4 per GPU)
from tests.util import UNET_CASES, UNET_TS, UNET_LABEL           # noqa: E402


def unet_row_step(y):
    """every row of a U-Net output up to ~700 KB, else every second row"""
    return 1 if y.numel() * 4 <= 700 * 1024 else 2


def graph_digests(doc):
    """the dual graph of a doctree (reference or oracle) as digests: canonical sorted (row*7+dir, col), node types and
    batch ids per depth"""
    out = {}
    for d in range(4, 7):
        k, c = R.edge_set(doc.graph[d])
        out['key%d' % d], out['col%d' % d] = digest(k), digest(c)
        out['node_type%d' % d], out['batch_id%d' % d] = digest(doc.graph[d]['node_type']), digest(doc.batch_id(d))
    return out


def octree_digests(octree, depths):
    out = {}
    for d in depths:
        out['keys%d' % d], out['children%d' % d] = digest(octree.keys[d]), digest(octree.children[d])
    return out


OPERATOR_GN_CHANNELS = (24, 64, 384)


def operator_inputs(dg1, dg2):
    """seeded inputs of the operator parity cases; dg1 / dg2: doctrees of one and two shapes (seed 0)"""
    n6 = dg2.batch_id(6).shape[0]
    return {'conv8_w': seeded_inputs(56, 8, 31) / np.sqrt(56.0), 'conv8_x': seeded_inputs(2 * 4096, 8, 32),
            'conv16_w': seeded_inputs(7 * 21, 24, 33) / np.sqrt(147.0), 'conv16_x': seeded_inputs(n6, 16, 34),
            'gn': {c: (1 + 0.1 * seeded_inputs(1, c, 35 + c), 0.1 * seeded_inputs(1, c, 36 + c),
                       seeded_inputs(dg2.batch_id(5).shape[0], c, 37 + c) * 2 + 0.5) for c in OPERATOR_GN_CHANNELS},
            'qkv': seeded_inputs(8 * 96, 64, 38).reshape(8, 96, 64), 't': torch.tensor([9.2, -2.3, 0.1])}


def split_signal():
    """the random split signal of the stage-1 -> stage-2 handoff case"""
    g = torch.Generator().manual_seed(4)
    split = torch.randn(2, 8, 16, 16, 16, generator=g)
    split[torch.rand(split.shape, generator=g) < 0.6] = -1.0            # sparse, like a surface
    return split


# inputs of the full-forward parity cases, distinct from UNET_CASES': other weights, latent, timesteps and labels
PARITY_UNET = {'small': 2, 'uncond': 1, 'cond': 1}          # name -> batch
PARITY_UNET_TS, PARITY_UNET_LABEL, PARITY_UNET_ROW_STEP = [0.8, -1.2], [2, 4], 8


def parity_unet_inputs(name, total_num):
    """(config, state-dict seed, latent, timesteps, labels) of a full-forward parity case"""
    from tests.util import UNET_CASES
    cfg, _, cc = UNET_CASES[name]
    batch = PARITY_UNET[name]
    label = torch.tensor(PARITY_UNET_LABEL)[:batch] if cfg.get('num_classes') else None
    return cfg, 2, seeded_inputs(total_num, cc, 17), torch.tensor(PARITY_UNET_TS)[:batch], label


def reference_parity(ref):
    """outputs of the reference's own modules for tests/test_oracle_vs_reference.py -> reference_parity.npz"""
    import importlib
    from tests import util as U
    fx = {}
    # full HR forwards (every PARITY_UNET_ROW_STEP-th output row)
    for name, batch in PARITY_UNET.items():
        doc = _ref_doctree(ref, batch, 0)
        cfg, wseed, x, ts, label = parity_unet_inputs(name, doc.total_num)
        net = ref.union.UNet3DModel('hr', **cfg).eval()
        net.load_state_dict(R.seeded_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, wseed))
        y = net(unet_type='hr', x=x, doctree=doc, timesteps=ts, unet_lr=net.unet_lr, label=label)
        fx['unet_%s_y' % name], fx['unet_%s_absmax' % name] = y[::PARITY_UNET_ROW_STEP].numpy(), float(y.abs().max())
    # dual graphs of several batches
    for batch, seed in ((1, 0), (2, 0), (3, 5)):
        doc = _ref_doctree(ref, batch, seed)
        for k, v in graph_digests(doc).items():
            fx['graph_b%d_s%d_%s' % (batch, seed, k)] = v
        fx['graph_b%d_s%d_nnum' % (batch, seed)] = doc.nnum.numpy()
        fx['graph_b%d_s%d_lnum' % (batch, seed)] = doc.lnum.numpy()
    # operators
    m = ref.modules
    doc2 = _ref_doctree(ref, 2, 0)
    inp = operator_inputs(doc2, doc2)
    conv = m.GraphConv(8, 8, 7, 7, 0)
    conv.weights.data.copy_(inp['conv8_w'])
    fx['conv8_y'] = conv(inp['conv8_x'], doc2, 4)[::4].numpy()
    conv = m.GraphConv(16, 24, 7, 7, 5)
    conv.weights.data.copy_(inp['conv16_w'])
    fx['conv16_y'] = conv(inp['conv16_x'], doc2, 6)[::32].numpy()
    for c, (gam, bet, x) in inp['gn'].items():
        gn = m.DualOctreeGroupNorm(c)
        gn.weights.data.copy_(gam); gn.bias.data.copy_(bet)
        fx['gn%d_y' % c] = gn(x, doc2, 5)[::256].numpy()
    fx['attn_y'] = m.QKVAttention()(inp['qkv']).numpy()
    fx['temb_y'] = ref.util.timestep_embedding(inp['t'], 128).numpy()
    fx['log_snr_0.3'] = float(ref.util.beta_linear_log_snr(torch.tensor(0.3)))
    # GraphVAE decode (octree grown by the reference) and encode
    gv = importlib.import_module('models.networks.dualoctree_networks.graph_vae')
    net = gv.GraphVAE(**U.VAE).eval()
    net.load_state_dict(U.vae_state_dict(5))
    doc = _ref_doctree(ref, 2, 3)
    out = net.decode_code(U.vae_code(doc.total_num, 2), doc, update_octree=True)
    fx['vae_nnum'] = out['octree_out'].nnum.numpy()
    for k, v in octree_digests(out['octree_out'], (6, 7, 8)).items():
        fx['vae_' + k] = v
    for d in (6, 7, 8):
        fx['vae_label%d' % d] = np.packbits(out['logits'][d].argmax(1).numpy().astype(np.uint8))
        fx['vae_logit%d' % d] = out['logits'][d][::32].numpy()
        fx['vae_reg%d' % d] = out['reg_voxs'][d][::32].numpy()
    net.load_state_dict(U.vae_state_dict())
    g = np.load(os.path.join(OUT, 'vae_decode.npz'))
    labels = {d: torch.from_numpy(np.unpackbits(g['label%d' % d])[: int(g['nnum'][d])].astype(np.int64)) for d in (6, 7, 8)}
    octree = U.oracle_grown_octree(labels)
    doc = ref.dual_octree.DualOctree(octree)
    doc.post_processing_for_docnn()
    data = torch.randn(doc.total_num, 4, generator=torch.Generator().manual_seed(9))
    net._get_input_feature = lambda doctree: data
    fx['vae_encode_y'] = net.KL_conv(net.octree_encoder_step(octree, doc)[6])[::32].numpy()
    # stage-1 -> stage-2 handoff
    util = ref_import.load_util()
    want = util.split2octree_small(split_signal(), 6, 4)
    for k, v in octree_digests(want, (4, 5, 6)).items():
        fx['split_' + k] = v
    fx['split_nnum'], fx['split_nnum_nempty'] = np.array(want.nnum.tolist()), np.array(want.nnum_nempty.tolist())
    fx['split_back'] = digest(util.octree2split_small(want, 4).flatten().long())
    fx['split_back_sum'] = checksum(util.octree2split_small(want, 4))
    # NeuralMPU on more query points than mpu_eval.npz
    mpu = importlib.import_module('models.networks.dualoctree_networks.mpu')
    pos, reg = mpu_inputs(octree, 4000, 22)
    orig = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        out = mpu.NeuralMPU(4, 6, 8)(pos, reg, octree)
    finally:
        torch.Tensor.cuda = orig
    for d in (6, 7, 8):
        fx['mpu_fval%d' % d] = out[d][0].numpy()
        fx['mpu_flag%d' % d] = np.packbits(out[d][1].numpy())
    np.savez_compressed(os.path.join(OUT, 'reference_parity.npz'), **fx)


def _ref_doctree(ref, batch, seed):
    l4, l5 = synth_splits(batch, seed)
    doc = ref.dual_octree.DualOctree(octree_from_splits(l4, l5, batch))
    doc.post_processing_for_docnn()
    return doc


def unet_fixture(ref, name):
    """full HR forward of the unmodified reference on seeded inputs -> tests/golden/unet_<name>.npz"""
    cfg, batch, cc = UNET_CASES[name]
    net = ref.union.UNet3DModel('hr', **cfg).eval()
    sd = R.seeded_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, 1)
    net.load_state_dict(sd)
    d = _ref_doctree(ref, batch, 0)
    x = seeded_inputs(d.total_num, cc, 7)
    ts = torch.tensor(UNET_TS)[:batch]
    label = torch.tensor(UNET_LABEL)[:batch] if cfg.get('num_classes') else None
    y = net(unet_type='hr', x=x, doctree=d, timesteps=ts, unet_lr=net.unet_lr, label=label)
    row_step = unet_row_step(y)
    np.savez_compressed(os.path.join(OUT, 'unet_%s.npz' % name), y=y[::row_step].numpy(), row_step=row_step,
                        x_sum=checksum(x), w_sum=sum(checksum(v) for v in sd.values()), batch=batch)
    print(name, 'out absmax', float(y.abs().max()), 'N', d.total_num)


def state_shapes(ref):
    """state_dict shapes of the unmodified reference nets -> tests/golden/state_shapes.json (lets bench.py's CPU arm
    build seeded weights on hosts without the reference tree and without importing the product package)."""
    import json
    import importlib
    from tests import util as U
    out = {}
    for name in ('uncond', 'uncond8', 'cond'):
        cfg = UNET_CASES[name][0]
        with torch.device('meta'):
            net = ref.union.UNet3DModel('hr', **cfg)
        out[name] = {k: list(v.shape) for k, v in net.state_dict().items()}
    gv = importlib.import_module('models.networks.dualoctree_networks.graph_vae')
    with torch.device('meta'):
        net = gv.GraphVAE(**U.VAE)
    out['vae'] = {k: list(v.shape) for k, v in net.state_dict().items()}
    with open(os.path.join(OUT, 'state_shapes.json'), 'w') as f:
        json.dump(out, f)
    print('state_shapes.json', {k: len(v) for k, v in out.items()})


def main():
    ref = ref_import.load()
    os.makedirs(OUT, exist_ok=True)
    torch.set_grad_enabled(False)
    if 'shapes' in sys.argv[1:]:
        state_shapes(ref)
        return
    if 'parity' in sys.argv[1:]:
        reference_parity(ref)
        return
    only = [a for a in sys.argv[1:] if a in UNET_CASES]
    if only:                                   # python -m oracle.gen_golden uncond8 cond_b4: just these fixtures
        for name in only:
            unet_fixture(ref, name)
        return

    def ref_doctree(batch, seed):
        return _ref_doctree(ref, batch, seed)

    # 1. dual graph of one shape: canonical sorted (row*7+dir, col) per depth
    doc = ref_doctree(1, 0)
    g = graph_digests(doc)
    g['nnum'], g['lnum'] = doc.nnum.numpy(), doc.lnum.numpy()
    np.savez_compressed(os.path.join(OUT, 'dual_graph_b1_s0.npz'), **g)

    # 2. BASELINE.json configs[0] analogue: one GraphConv 8->8 on the depth-4 full layer of one octree
    conv = ref.modules.GraphConv(8, 8, 7, 7, 0)
    w = seeded_inputs(56, 8, 11) / np.sqrt(56.0)
    conv.weights.data.copy_(w)
    x = seeded_inputs(4096, 8, 12)
    np.savez_compressed(os.path.join(OUT, 'graphconv_config1.npz'), x=x.numpy(), w=w.numpy(),
                        y=conv(x, doc, 4).numpy())

    # 3. operators at depth 6 with node types / ragged norm / attention
    conv = ref.modules.GraphConv(64, 32, 7, 7, 5)
    w = seeded_inputs(7 * 69, 32, 13) / np.sqrt(7 * 69.0)
    conv.weights.data.copy_(w)
    n6 = doc.total_num
    x = seeded_inputs(n6, 64, 14)
    ops = {'conv_y': conv(x, doc, 6)[::16].numpy(),      # every 16th row keeps the fixture small
            'conv_x_sum': checksum(x), 'conv_w_sum': checksum(w)}
    gn = ref.modules.DualOctreeGroupNorm(64)
    gam, bet = 1 + 0.1 * seeded_inputs(1, 64, 15), 0.1 * seeded_inputs(1, 64, 16)
    gn.weights.data.copy_(gam); gn.bias.data.copy_(bet)
    doc2 = ref_doctree(2, 0)
    x2 = seeded_inputs(doc2.batch_id(5).shape[0], 64, 17) * 2 + 0.5
    ops['gn_y'] = gn(x2, doc2, 5)[::16].numpy()
    qkv = seeded_inputs(8 * 96, 64, 18).reshape(8, 96, 64)
    ops['attn_y'] = ref.modules.QKVAttention()(qkv).numpy()
    np.savez_compressed(os.path.join(OUT, 'operators.npz'), **ops)

    # 4. full U-Net forwards (weights from the shared seeded_state_dict)
    for name in UNET_CASES:
        unet_fixture(ref, name)
    state_shapes(ref)
    # 5. GraphVAE decoder (SURVEY.md 8f rank 1): decode_code(update_octree=True) of the unmodified reference
    import importlib
    from tests import util as U
    gv = importlib.import_module('models.networks.dualoctree_networks.graph_vae')
    vae = gv.GraphVAE(**U.VAE).eval()
    sd = U.vae_state_dict()
    vae.load_state_dict(sd)
    d_in = ref_doctree(1, 0)
    code = U.vae_code(d_in.total_num)
    out = vae.decode_code(code, d_in, update_octree=True)
    fx = {'code_sum': checksum(code), 'w_sum': sum(checksum(v) for v in sd.values()),
          'nnum': out['octree_out'].nnum.numpy(), 'nnum_nempty': out['octree_out'].nnum_nempty.numpy()}
    for d in (6, 7, 8):
        lg = out['logits'][d]
        fx['label%d' % d] = np.packbits(lg.argmax(1).numpy().astype(np.uint8))
        fx['margin%d' % d] = float((lg[:, 0] - lg[:, 1]).abs().min())
        fx['logit%d' % d] = lg[::16].numpy()
        fx['reg%d' % d] = out['reg_voxs'][d][::16].numpy()
    np.savez_compressed(os.path.join(OUT, 'vae_decode.npz'), **fx)
    print('vae nnum', fx['nnum'].tolist(), 'margins', [fx['margin%d' % d] for d in (6, 7, 8)])
    # 6. NeuralMPU (SURVEY.md 8f rank 4) on the octree grown above, random per-node regression values
    fx = mpu_fixture()
    np.savez_compressed(os.path.join(OUT, 'mpu_eval.npz'), **fx)
    # 7. the remaining parity cases of tests/test_oracle_vs_reference.py (reads vae_decode.npz)
    reference_parity(ref)
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)) // 1024, 'KB')


if __name__ == '__main__':
    main()
