"""-m gpu parity of the composed operators and of the full denoising U-Net against the oracle.
Tolerances are the north star's: 1e-3 relative (fp32), 2e-2 relative (bf16), max-abs error over max-abs
reference value."""
import pytest
import torch

from oracle import restate as R
from tests.util import (relerr, oracle_doctree, product_doctree, model_shapes, build_product, UNCOND, COND, SMALL,
                        UNET_CASES, UNET_TS, UNET_LABEL)

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g) * scale


def _sub(sd, prefix):
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


@pytest.fixture(scope='module')
def uncond():
    shapes = model_shapes(UNCOND)
    sd = R.seeded_state_dict(shapes, 0)
    return sd, build_product(UNCOND, sd)


@pytest.mark.parametrize('dtype,tol', [(torch.float32, 1e-4), (torch.bfloat16, 2e-2)])
def test_resblock_and_resample(uncond, dtype, tol):
    sd, net = uncond
    hr = net.unet_hr
    dg, _ = oracle_doctree(2, 0)
    doc = product_doctree(2, 0)
    emb = _rand((2, 512), 3)
    sub = _sub(sd, 'unet_hr.')
    # input_blocks.1: 128->128 at depth 6 (identity skip); input_blocks.3: 128->256 at depth 5 (Conv1x1 skip)
    for idx, d, cin in ((1, 6, 128), (3, 5, 128)):
        n = dg.batch_id(d).shape[0]
        x = _rand((n, cin), 10 + idx)
        ref = R.res_block_embed(x, emb, dg, d, sub, 'input_blocks.%d.' % idx, d - 1)
        y = hr.input_blocks[idx](x.to(DEV).to(dtype), emb.to(DEV), doc, d)
        assert relerr(y.float().cpu(), ref) < tol, (idx, relerr(y.float().cpu(), ref))
    # GraphDownsample 6->5 and GraphUpsample 5->6
    x = _rand((dg.batch_id(6).shape[0], 128), 20)
    ref = R.graph_downsample(x, dg, 6, sub['input_blocks.2.downsample.weights'], sub['input_blocks.2.conv.weights'], 4)
    y = hr.input_blocks[2](x.to(DEV).to(dtype), doc, 6)
    assert relerr(y.float().cpu(), ref) < tol
    x = _rand((dg.batch_id(5).shape[0], 256), 21)
    ref = R.graph_upsample(x, dg, 5, sub['output_blocks.4.upsample.weights'], sub['output_blocks.4.conv.weights'], 5)
    y = hr.output_blocks[4](x.to(DEV).to(dtype), doc, 5)
    assert relerr(y.float().cpu(), ref) < tol


# The LR middle block alone is an *intermediate* (post-GroupNorm+SiLU features after ~20 bf16 stages).  Since round 2 the
# norm statistics are deterministic (no atomics), so its bf16 error is a fixed number: max-norm 2.2e-2, relative L2 1.6e-2
# (round 1: 2 % .. 3.5 % from run to run, asserted at 6e-2).  The north-star 2e-2 max-norm tolerance is asserted on the U-Net
# OUTPUT below; the intermediate is held to 2.5e-2 max-norm and 2e-2 L2.
@pytest.mark.parametrize('dtype,tol', [(torch.float32, 1e-4), (torch.bfloat16, 2.5e-2)])
def test_lr_middle(uncond, dtype, tol):
    sd, net = uncond
    dg, _ = oracle_doctree(2, 0)
    doc = product_doctree(2, 0)
    lr_cfg, _ = R.split_cfg(UNCOND)
    h = _rand((2 * 4096, 64), 5)
    ts = torch.tensor([1.5, -0.5])
    ref = R.lr_forward_as_middle(h, dg, ts, sd, lr_cfg)
    y = net.unet_lr.forward_as_middle(h.to(DEV).to(dtype), doc, ts.to(DEV), None, None).float().cpu()
    print('ERR lr_middle %s max %.3e l2 %.3e' % (str(dtype), relerr(y, ref), float((y - ref).norm() / ref.norm())))
    assert relerr(y, ref) < tol
    if dtype == torch.bfloat16:
        assert float((y - ref).norm() / ref.norm()) < 2e-2


@pytest.mark.parametrize('cfg_name', ['uncond', 'cond', 'small'])
@pytest.mark.parametrize('dtype,tol', [(torch.float32, 1e-3), (torch.bfloat16, 2e-2)])
def test_full_unet_forward(cfg_name, dtype, tol):
    cfg = {'uncond': UNCOND, 'cond': COND, 'small': SMALL}[cfg_name]
    sd = R.seeded_state_dict(model_shapes(cfg), 1)
    net = build_product(cfg, sd)
    dg, _ = oracle_doctree(2, 0)
    doc = product_doctree(2, 0)
    lr_cfg, hr_cfg = R.split_cfg(cfg)
    x = _rand((dg.total_num, 3), 7)
    ts = torch.tensor([1.5, -0.5])
    label = torch.tensor([1, 3]) if cfg.get('num_classes') else None
    ref = R.hr_forward(x, dg, ts, sd, hr_cfg, lr_cfg, label=label)
    y = net(unet_type='hr', x=x.to(DEV).to(dtype), doctree=doc, timesteps=ts.to(DEV), unet_lr=net.unet_lr,
            label=label.to(DEV) if label is not None else None)
    assert y.dtype == torch.float32
    e = relerr(y.cpu(), ref)
    print('ERR full_unet %s %s %.3e' % (cfg_name, str(dtype), e))
    assert e < tol, e


def test_forward_is_bit_reproducible_and_fusion_neutral():
    """No floating-point atomics anywhere on the path (norm statistics are per-segment partials summed in fixed order):
    two forwards give bit-identical results in fp32 and bf16.  Switching the epilogue statistics off (stand-alone
    statistics pass over the stored bf16 tensor instead of the fp32 accumulators) moves the bf16 result by no more than the
    bf16 tolerance itself."""
    from octfusion_b200 import ops
    cfg = SMALL
    sd = R.seeded_state_dict(model_shapes(cfg), 1)
    net = build_product(cfg, sd)
    doc = product_doctree(2, 0)
    x = _rand((doc.total_num, 3), 7)
    ts = torch.tensor([1.5, -0.5]).to(DEV)
    outs = {}
    for dtype in (torch.float32, torch.bfloat16):
        run = lambda: net(unet_type='hr', x=x.to(DEV).to(dtype), doctree=doc, timesteps=ts, unet_lr=net.unet_lr, label=None)  # noqa: E731
        a, b = run(), run()
        assert torch.equal(a, b), str(dtype)
        outs[dtype] = a
    ops._FUSE_STATS = False
    try:
        c = net(unet_type='hr', x=x.to(DEV).bfloat16(), doctree=doc, timesteps=ts, unet_lr=net.unet_lr, label=None)
    finally:
        ops._FUSE_STATS = True
    assert relerr(c, outs[torch.bfloat16]) < 2e-2


def test_sampler_cuda_graph_matches_eager_and_oracle():
    from octfusion_b200.sampler import sample_loop, sampling_log_snr
    cfg = SMALL
    sd = R.seeded_state_dict(model_shapes(cfg), 2)
    net = build_product(cfg, sd)
    dg, _ = oracle_doctree(2, 0)
    doc = product_doctree(2, 0)
    lr_cfg, hr_cfg = R.split_cfg(cfg)
    steps = 4
    noise = _rand((dg.total_num, 3), 9)
    x = noise.clone()
    ls = sampling_log_snr(steps)
    for i in range(steps):
        t = torch.full((2,), ls[i])
        eps = R.hr_forward(x, dg, t, sd, hr_cfg, lr_cfg)
        x = R.ddim_eps_update(x, eps, torch.tensor(ls[i]), torch.tensor(ls[i + 1]))
    for graph in (False, True):
        y = sample_loop(net.unet_hr, net.unet_lr, doc, ddim_steps=steps, noise=noise.to(DEV), act_dtype=torch.float32,
                        use_cuda_graph=graph)
        assert relerr(y.cpu(), x) < 2e-3, (graph, relerr(y.cpu(), x))
    yb = sample_loop(net.unet_hr, net.unet_lr, doc, ddim_steps=steps, noise=noise.to(DEV), act_dtype=torch.bfloat16)
    print('ERR sampler4 bf16 %.3e' % relerr(yb.cpu(), x))
    assert relerr(yb.cpu(), x) < 1e-2


# ------------------------------------------------------------------------------------------------
# against the committed golden vectors (outputs of the unmodified reference, tests/golden/)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(UNET_CASES))
@pytest.mark.parametrize('dtype,tol', [(torch.float32, 1e-3), (torch.bfloat16, 2e-2)])
def test_unet_against_reference_golden(name, dtype, tol):
    """includes `uncond8` = the benchmarked configuration (8 latent channels: first conv K = 7*(8+5), output conv
    128 -> 8 on the N=16 tile) at B=2 and `cond_b4` = the cond config at the 4-shapes-per-GPU shard of configs[4]."""
    import os
    import numpy as np
    from tests.util import GOLDEN
    cfg, batch, cc = UNET_CASES[name]
    g = np.load(os.path.join(GOLDEN, 'unet_%s.npz' % name))
    assert batch == int(g['batch'])
    sd = R.seeded_state_dict(model_shapes(cfg), 1)
    net = build_product(cfg, sd)
    doc = product_doctree(batch, 0)
    x = _rand((doc.total_num, cc), 7)
    ts = torch.tensor(UNET_TS)[:batch]
    label = torch.tensor(UNET_LABEL)[:batch].to(DEV) if cfg.get('num_classes') else None
    y = net(unet_type='hr', x=x.to(DEV).to(dtype), doctree=doc, timesteps=ts.to(DEV), unet_lr=net.unet_lr, label=label)
    e = relerr(y.cpu()[::int(g['row_step']) if 'row_step' in g else 1], torch.from_numpy(g['y']))
    print('ERR golden %s %s %.3e' % (name, str(dtype), e))
    assert e < tol, e


def test_graph_and_config1_against_reference_golden():
    import os
    import numpy as np
    from tests.util import GOLDEN, digest
    from octfusion_b200.modules import GraphConv
    doc = product_doctree(1, 0)
    g = np.load(os.path.join(GOLDEN, 'dual_graph_b1_s0.npz'))
    for d in range(4, 7):
        k, c = R.edge_set({'edge_idx': doc.graph[d]['edge_idx'].cpu(), 'edge_dir': doc.graph[d]['edge_dir'].cpu()})
        assert digest(k) == g['key%d' % d] and digest(c) == g['col%d' % d]
        assert digest(doc.plan[d].node_type) == g['node_type%d' % d]
        assert digest(doc.plan[d].batch_id) == g['batch_id%d' % d]
    g = np.load(os.path.join(GOLDEN, 'graphconv_config1.npz'))
    conv = GraphConv(8, 8, 7, 7, 0)
    conv.weights.data.copy_(torch.from_numpy(g['w']))
    y = conv.to(DEV)(torch.from_numpy(g['x']).to(DEV), doc, 4)
    assert relerr(y.cpu(), torch.from_numpy(g['y'])) < 1e-5


# ------------------------------------------------------------------------------------------------
# SURVEY.md 8f-3 ("next" row): the dense LR U-Net as a stand-alone stage-1 denoiser
# (reference graph_unet_lr.py:184-230, called with unet_type="lr" by octfusion_model_union.py:373)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype,tol', [(torch.float32, 1e-3), (torch.bfloat16, 2e-2)])
def test_lr_unet_standalone_stage1(uncond, dtype, tol):
    sd, net = uncond
    lr_cfg, _ = R.split_cfg(UNCOND)
    x = _rand((2, 8, 16, 16, 16), 31)
    ts = torch.tensor([0.7, -1.2])
    ref = R.lr_forward_dense(x, ts, sd, lr_cfg, as_middle=False)
    y = net(unet_type='lr', x=x.to(DEV).to(dtype), timesteps=ts.to(DEV))
    assert y.shape == ref.shape
    print('ERR lr_standalone %s %.3e' % (str(dtype), relerr(y.float().cpu(), ref)))
    assert relerr(y.float().cpu(), ref) < tol


def test_stage1_sample_loop_x0_branch(uncond):
    """reference sample_loop 'x0' branch (octfusion_model_union.py:300-344) with explicit noises: self-conditioning,
    sign() truncation below t=0.7, ancestral noise above.  sign() is discontinuous, so the comparison is teacher-forced:
    at every step the product's network and update kernel run on the ORACLE's state (continuous prediction compared at
    1e-3; the update -- sign included -- on identical inputs at 1e-5).  The free-running loop must then agree with the
    oracle everywhere except on the few voxels whose prediction sat within rounding of zero at a sign() step."""
    from octfusion_b200 import ops
    from octfusion_b200.sampler import sample_loop_lr, beta_linear_log_snr
    sd, net = uncond
    lr_cfg, _ = R.split_cfg(UNCOND)
    steps, b = 4, 2
    noises = [_rand((b, 8, 16, 16, 16), 100 + i) for i in range(steps + 1)]
    times = torch.linspace(1.0, 0.0, steps + 1)
    x, x_start = noises[0].clone(), None
    for i in range(steps):
        t, tn = float(times[i]), float(times[i + 1])
        ls, lsn = torch.tensor(beta_linear_log_snr(t)), torch.tensor(beta_linear_log_snr(tn))
        inp = torch.cat([x, torch.zeros_like(x) if x_start is None else x_start], 1)
        pred = R.lr_forward_dense(F_conv_in(inp, sd), torch.full((b,), float(ls)), sd, lr_cfg, as_middle=True)
        pred = torch.nn.functional.conv3d(pred, sd['unet_lr.out.weight'], sd['unet_lr.out.bias'], padding=1)
        # product network on the oracle's state
        ts = torch.full((b,), float(ls), device=DEV)
        mine = net.unet_lr(x=x.to(DEV), timesteps=ts, x_self_cond=None if x_start is None else x_start.to(DEV), label=None)
        assert relerr(mine.float().cpu(), pred) < 1e-3, i
        # product update kernel on the oracle's prediction
        noise = noises[i + 1] if tn > 0.7 else None
        xp, pp = x.clone().to(DEV).contiguous(), pred.clone().to(DEV).contiguous()
        ops.ddpm_x0_update(xp, pp, ls.reshape(1).to(DEV), lsn.reshape(1).to(DEV),
                           noise=None if noise is None else noise.to(DEV).contiguous(), do_sign=(t < 0.7))
        x, x_start = R.ddpm_x0_update(x, pred, ls, lsn, noise, t < 0.7)
        assert relerr(xp.cpu(), x) < 1e-5 and relerr(pp.cpu(), x_start) < 1e-5, i
    y = sample_loop_lr(net.unet_lr, b, ddim_steps=steps, act_dtype=torch.float32, noises=noises)
    off = ((y.cpu() - x).abs() > 2e-3 * float(x.abs().max())).float().mean()
    assert float(off) < 1e-3, float(off)


def F_conv_in(inp, sd):
    """input_emb of the stand-alone LR net applied to (x | x_self_cond) (graph_unet_lr.py:198-200)."""
    return torch.nn.functional.conv3d(inp, sd['unet_lr.input_emb.weight'], sd['unet_lr.input_emb.bias'], padding=1)


def test_stepper_recaptures_when_weights_change():
    """The captured CUDA graph holds packed copies of the weights; an in-place parameter update must invalidate it
    (ADVICE round 1): the next replay equals an eager step with the new weights, not the stale graph."""
    from octfusion_b200.sampler import HRStepper, sampling_log_snr
    cfg = SMALL
    sd = R.seeded_state_dict(model_shapes(cfg), 2)
    net = build_product(cfg, sd)
    doc = product_doctree(1, 0)
    ls = sampling_log_snr(4)
    noise = _rand((doc.total_num, 3), 9).to(DEV)

    def one_step(use_graph, stepper=None):
        st = stepper or HRStepper(net.unet_hr, net.unet_lr, doc, torch.float32, None, use_cuda_graph=use_graph)
        st.set_latent(noise)
        st.step(ls[0], ls[1])
        return st, st.x.clone()
    st, a = one_step(True)
    with torch.no_grad():
        net.unet_hr.out.weights.mul_(1.5)                   # in-place: bumps the parameter's version
    _, b_graph = one_step(True, st)                          # same stepper: must notice and re-capture
    _, b_eager = one_step(False)
    assert not torch.equal(a, b_graph)
    assert torch.equal(b_graph, b_eager)


def test_stepper_host_latents_pipeline_matches_serial():
    """HRStepper.step_host: latents in pinned host memory, copies double-buffered on side streams beside the compute of
    the neighbouring calls -- every result equals the serial set_latent / step / read-back of the same latent, bit for
    bit (five calls: both staging buffers are re-used)."""
    from octfusion_b200.sampler import HRStepper, sampling_log_snr
    cfg = SMALL
    sd = R.seeded_state_dict(model_shapes(cfg), 2)
    net = build_product(cfg, sd)
    doc = product_doctree(1, 0)
    ls = sampling_log_snr(8)
    st = HRStepper(net.unet_hr, net.unet_lr, doc, torch.bfloat16, None, use_cuda_graph=True)
    xs = [_rand((doc.total_num, 3), 20 + i).pin_memory() for i in range(5)]
    want = []
    for i, x in enumerate(xs):
        st.set_latent(x.to(DEV))
        st.step(ls[i], ls[i + 1])
        want.append(st.x.cpu())
    outs = [torch.empty_like(x).pin_memory() for x in xs]
    for i, x in enumerate(xs):
        st.step_host(x, ls[i], ls[i + 1], outs[i])
    st.sync_host()
    torch.cuda.synchronize()
    for i in range(5):
        assert torch.equal(outs[i], want[i]), i
