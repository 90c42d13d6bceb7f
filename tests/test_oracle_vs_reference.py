"""Pins the oracle (oracle/restate.py) against outputs of the UNMODIFIED reference modules, stored in
tests/golden/reference_parity.npz by oracle/gen_golden.py (the reference itself is not needed to run these)."""
import os
import numpy as np
import pytest
import torch

from oracle import restate as R
from oracle.gen_golden import graph_digests, octree_digests, operator_inputs, split_signal, mpu_inputs, OPERATOR_GN_CHANNELS
from tests.util import relerr, oracle_doctree, digest, GOLDEN


@pytest.fixture(scope='module')
def ref():
    return np.load(os.path.join(GOLDEN, 'reference_parity.npz'))


@pytest.mark.parametrize('batch,seed', [(1, 0), (2, 0), (3, 5)])
def test_dual_graph_equals_reference(ref, batch, seed):
    dg, _ = oracle_doctree(batch, seed)
    pre = 'graph_b%d_s%d_' % (batch, seed)
    for k, v in graph_digests(dg).items():
        assert v == ref[pre + k], k
    assert np.array_equal(dg.nnum.numpy(), ref[pre + 'nnum']) and np.array_equal(dg.lnum.numpy(), ref[pre + 'lnum'])


@pytest.mark.parametrize('name', ['small', 'uncond', 'cond'])
def test_full_unet_equals_reference(ref, name):
    """full HR forward of the oracle against the reference's UNet3DModel.  Its own inputs (weights, latent, timesteps,
    labels: oracle/gen_golden.py parity_unet_inputs), not those of the unet_<name>.npz fixtures."""
    from oracle.gen_golden import PARITY_UNET, PARITY_UNET_ROW_STEP, parity_unet_inputs
    from tests.util import model_shapes
    dg, _ = oracle_doctree(PARITY_UNET[name], 0)
    cfg, wseed, x, ts, label = parity_unet_inputs(name, dg.total_num)
    lr_cfg, hr_cfg = R.split_cfg(cfg)
    got = R.hr_forward(x, dg, ts, R.seeded_state_dict(model_shapes(cfg), wseed), hr_cfg, lr_cfg, label=label)
    assert float(ref['unet_%s_absmax' % name]) > 0.1          # the seeded weights must not leave the net at zero
    assert relerr(got[::PARITY_UNET_ROW_STEP], torch.from_numpy(ref['unet_%s_y' % name])) < 2e-5


def test_operators_equal_reference(ref):
    dg, _ = oracle_doctree(2, 0)
    inp = operator_inputs(dg, dg)
    # config-1 analogue: GraphConv 8->8 on the depth-4 full layer
    assert relerr(R.graph_conv(inp['conv8_x'], dg.graph[4], inp['conv8_w'], 0)[::4], torch.from_numpy(ref['conv8_y'])) < 1e-6
    assert relerr(R.graph_conv(inp['conv16_x'], dg.graph[6], inp['conv16_w'], 5)[::32], torch.from_numpy(ref['conv16_y'])) < 1e-6
    for c in OPERATOR_GN_CHANNELS:
        gam, bet, x = inp['gn'][c]
        assert relerr(R.doctree_group_norm(x, dg.batch_id(5), 2, gam, bet)[::256], torch.from_numpy(ref['gn%d_y' % c])) < 1e-5
    assert relerr(R.qkv_attention(inp['qkv']), torch.from_numpy(ref['attn_y'])) < 1e-6
    assert relerr(R.timestep_embedding(inp['t'], 128), torch.from_numpy(ref['temb_y'])) < 1e-6
    assert abs(float(R.beta_linear_log_snr(torch.tensor(0.3))) - float(ref['log_snr_0.3'])) < 1e-6


def test_vae_decode_equals_reference(ref):
    """GraphVAE (SURVEY.md 8f rank 1): state_dict parity of the product class with the reference's, and
    decode_code(update_octree=True) of the oracle against the reference on two shapes; the oracle grows its octree with
    the reference's labels."""
    import json
    from tests import util as U
    with open(os.path.join(GOLDEN, 'state_shapes.json')) as f:
        assert {k: tuple(v) for k, v in json.load(f)['vae'].items()} == U.vae_shapes()
    nnum = ref['vae_nnum']
    labels = {d: torch.from_numpy(np.unpackbits(ref['vae_label%d' % d])[: int(nnum[d])].astype(np.int64)) for d in (6, 7, 8)}
    dg, _ = oracle_doctree(2, 3)
    mine = R.DualGraph(U.oracle_child_octree(dg.octree))
    code = U.vae_code(dg.total_num, 2)
    logits, regs, octree = R.vae_decode(code, mine, U.vae_state_dict(5), 6, 8, 2, update_octree=True, labels=labels)
    assert np.array_equal(octree.nnum.numpy(), nnum)
    for k, v in octree_digests(octree, (6, 7, 8)).items():
        assert v == ref['vae_' + k], k
    for d in (6, 7, 8):
        assert relerr(logits[d][::32], torch.from_numpy(ref['vae_logit%d' % d])) < 1e-5
        assert relerr(regs[d][::32], torch.from_numpy(ref['vae_reg%d' % d])) < 1e-5


def test_vae_encode_equals_reference(ref):
    """GraphVAE.octree_encoder_step + KL_conv on given input features (the reference builds them from point clouds
    with ocnn InputFeature, which is outside the path: `_get_input_feature` was replaced by a seeded tensor)."""
    from tests import util as U
    g = np.load(os.path.join(GOLDEN, 'vae_decode.npz'))
    labels = {d: torch.from_numpy(np.unpackbits(g['label%d' % d])[: int(g['nnum'][d])].astype(np.int64)) for d in (6, 7, 8)}
    octree = U.oracle_grown_octree(labels)
    dg = R.DualGraph(octree)
    data = torch.randn(dg.total_num, 4, generator=torch.Generator().manual_seed(9))
    mine = R.vae_encode(data, dg, U.vae_state_dict(), 8, 6, 2)
    assert relerr(mine[::32], torch.from_numpy(ref['vae_encode_y'])) < 1e-5


def test_split_octree_handoff_equals_reference(ref):
    """stage-1 -> stage-2 handoff (SURVEY.md 8f rank 2): split2octree_small / octree2split_small of the product
    (device-agnostic index ops) against the reference's, on a random split signal and its round trip."""
    from octfusion_b200 import octree as P
    got = P.split2octree_small(split_signal(), 6, 4)
    assert got.depth == 6
    for k, v in octree_digests(got, (4, 5, 6)).items():
        assert v == ref['split_' + k], k
    assert got.nnum.tolist() == ref['split_nnum'].tolist() and got.nnum_nempty.tolist() == ref['split_nnum_nempty'].tolist()
    back = P.octree2split_small(got, 4)
    assert digest(back.flatten().long()) == ref['split_back']
    assert abs(float(back.double().abs().sum()) - float(ref['split_back_sum'])) < 1e-6
    # round trip: the octree built from its own split signal is the same octree
    again = P.split2octree_small(back, 6, 4)
    for d in range(4, 7):
        assert torch.equal(again.keys[d], got.keys[d]) and torch.equal(again.children[d], got.children[d])


def test_neural_mpu_equals_reference(ref):
    """NeuralMPU (SURVEY.md 8f rank 4, oracle only): per-point restatement against reference mpu.py on the octree of the
    VAE fixture case, query points near occupied depth-8 cells and uniform ones."""
    from tests import util as U
    g = np.load(os.path.join(GOLDEN, 'vae_decode.npz'))
    labels = {d: torch.from_numpy(np.unpackbits(g['label%d' % d])[: int(g['nnum'][d])].astype(np.int64)) for d in (6, 7, 8)}
    octree = U.oracle_grown_octree(labels)
    pos, reg = mpu_inputs(octree, 4000, 22)
    mine = R.mpu_eval(pos, reg, octree, 4, 6, 8)
    for d in (6, 7, 8):
        assert np.array_equal(np.packbits(mine[d][1].numpy()), ref['mpu_flag%d' % d])
        assert relerr(mine[d][0], torch.from_numpy(ref['mpu_fval%d' % d])) < 1e-5, d
    flag8 = np.unpackbits(ref['mpu_flag8'])[: mine[8][1].numel()]
    assert flag8.any() and not flag8.all()
