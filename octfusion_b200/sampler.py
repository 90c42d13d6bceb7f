"""The stage-2 ("hr") sampling loop: drop-in for reference models/octfusion_model_union.py
`sample_loop` (:300-352, df_type "eps") with the log-SNR schedule of ldm_diffusion_util.py:300-309.

One step = U-Net forward (epsilon prediction) + eps-DDIM update.  The dual octree is constant across
steps, so all shapes are static: the whole step (~400 kernels) is captured once in a CUDA graph and
replayed; the per-step scalars (log-SNR of t and t_next) live in device tensors that are refreshed before
each replay.  The reference's per-sample Python loop (modules.py:757-758) and its ~300 ATen launches per
step disappear.
"""
from __future__ import annotations
import math
import torch

from . import ops


def beta_linear_log_snr(t: float) -> float:
    """reference ldm_diffusion_util.py:300-301, evaluated on the host in float64."""
    return -math.log(math.expm1(1e-4 + 10.0 * t * t))


def sampling_log_snr(steps: int):
    """log-SNR at the steps+1 times linspace(1, 0, steps+1) (octfusion_model_union.py:292-298)."""
    ts = torch.linspace(1.0, 0.0, steps + 1, dtype=torch.float32)
    return [beta_linear_log_snr(float(t)) for t in ts]


class HRStepper:
    """Holds the static buffers of one (model, doctree) pair and runs denoising steps."""

    def __init__(self, unet_hr, unet_lr, doctree, act_dtype=torch.bfloat16, label=None, use_cuda_graph=True):
        self.hr, self.lr, self.doctree = unet_hr, unet_lr, doctree
        self.act_dtype = act_dtype
        dev = doctree.device
        n = doctree.total_num
        c = unet_hr.in_channels
        self.x = torch.zeros((n, c), dtype=torch.float32, device=dev)          # the latent, always fp32
        self.x_act = torch.zeros((n, c), dtype=act_dtype, device=dev) if act_dtype != torch.float32 else None
        self.ts = torch.zeros(doctree.batch_size, dtype=torch.float32, device=dev)
        self.ls = torch.zeros(1, dtype=torch.float32, device=dev)
        self.ls_next = torch.zeros(1, dtype=torch.float32, device=dev)
        self.label = label
        self.eps = None
        self.graph = None
        self._graph_key = None
        self.use_cuda_graph = use_cuda_graph
        self.kernels_per_step = 0
        self._pipe = None

    def _weights_key(self):
        """fingerprint of every parameter of the two nets: the captured graph bakes in device copies of the weights
        (packed tensor-core images, concatenated embedding projections, padded first conv), so an in-place update, a
        load_state_dict or an EMA swap must force a re-capture"""
        key = []
        for net in (self.hr, self.lr):
            if net is not None:
                key += [(p.data_ptr(), p._version) for p in net.parameters()]
        return tuple(key)

    def invalidate(self):
        """drop the captured CUDA graph (next step re-captures it)"""
        self.graph, self._graph_key = None, None

    def set_latent(self, x):
        self.x.copy_(x)
        if self.x_act is not None:
            ops.copy_rows(self.x, self.x_act, self.x.shape[0], self.x.shape[1])

    # ---- latents that live in (pinned) host memory: one step per call, copies overlapped with the previous / next step ----
    def step_host(self, x_host, log_snr: float, log_snr_next: float, out_host):
        """One denoising step of a latent in pinned host memory: x_host -> device, step, result -> out_host.

        Asynchronous and double-buffered: the host->device copy of THIS call runs on a copy stream while the previous
        call's step is still computing, and the device->host copy of this call's result runs on a second copy stream
        while the next call computes (PCIe is full duplex).  Independent latents only -- a call does not see the
        previous call's output.  Call sync_host() before reading out_host."""
        cur = torch.cuda.current_stream()
        if self._pipe is None:
            mk = lambda: torch.empty_like(self.x)                       # noqa: E731
            ev = lambda: [torch.cuda.Event(), torch.cuda.Event()]       # noqa: E731
            self._pipe = dict(h2d=torch.cuda.Stream(), d2h=torch.cuda.Stream(), xin=[mk(), mk()], out=[mk(), mk()],
                              loaded=ev(), consumed=ev(), produced=ev(), drained=ev(), n=0)
        q = self._pipe
        i, s = q['n'], q['n'] & 1
        with torch.cuda.stream(q['h2d']):
            if i >= 2:
                q['h2d'].wait_event(q['consumed'][s])                   # step i-2 has read this staging buffer
            q['xin'][s].copy_(x_host, non_blocking=True)
            q['loaded'][s].record(q['h2d'])
        cur.wait_event(q['loaded'][s])
        self.set_latent(q['xin'][s])
        q['consumed'][s].record(cur)
        self.step(log_snr, log_snr_next)
        if i >= 2:
            cur.wait_event(q['drained'][s])                             # the result of step i-2 has left this buffer
        q['out'][s].copy_(self.x)
        q['produced'][s].record(cur)
        with torch.cuda.stream(q['d2h']):
            q['d2h'].wait_event(q['produced'][s])
            out_host.copy_(q['out'][s], non_blocking=True)
            q['drained'][s].record(q['d2h'])
        q['n'] = i + 1

    def sync_host(self):
        """make the current stream wait for every outstanding result copy of step_host()"""
        if self._pipe is not None:
            cur = torch.cuda.current_stream()
            for k in range(min(2, self._pipe['n'])):
                cur.wait_event(self._pipe['drained'][k])

    def forward_eps(self):
        xin = self.x if self.x_act is None else self.x_act
        return self.hr(x=xin, doctree=self.doctree, unet_lr=self.lr, timesteps=self.ts, label=self.label,
                       out_f32=True)

    def _body(self):
        self.eps = self.forward_eps()
        ops.ddim_eps_update(self.x, self.eps, self.ls, self.ls_next, self.x_act)

    def _set_scalars(self, log_snr, log_snr_next):
        self.ts.fill_(log_snr)
        self.ls.fill_(log_snr)
        self.ls_next.fill_(log_snr_next)

    def step(self, log_snr: float, log_snr_next: float):
        from . import _lib
        self._set_scalars(log_snr, log_snr_next)
        if not self.use_cuda_graph:
            c0 = _lib.launch_count()
            self._body()
            self.kernels_per_step = _lib.launch_count() - c0
            return
        if self.graph is not None and self._graph_key != self._weights_key():
            self.invalidate()                    # weights changed since capture: the graph holds stale packed copies
        if self.graph is None:
            # eager warm-up on a side copy of the state (builds packed weights, tables, func attributes)
            keep = self.x.clone()
            self._body()
            self.set_latent(keep)
            c0 = _lib.launch_count()             # second pass: the steady-state launches only (no weight packing)
            self._body()
            self.kernels_per_step = _lib.launch_count() - c0
            self.set_latent(keep)
            torch.cuda.synchronize()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self._body()
            self._graph_key = self._weights_key()
            self.set_latent(keep)        # capture does not execute; restore is a no-op safety
        self.graph.replay()


@torch.no_grad()
def sample_loop(unet_hr, unet_lr, doctree, ddim_steps=200, label=None, noise=None, seed=0,
                act_dtype=torch.bfloat16, use_cuda_graph=True, stepper=None):
    """Returns the denoised latent [total_num, code_channel] fp32 (reference :300-352, 'eps' branch)."""
    if stepper is not None:
        # a caller-provided stepper carries its own label / dtype / graph switch: refuse silently different arguments
        same_label = (label is None and stepper.label is None) or (label is not None and stepper.label is not None
                                                                   and torch.equal(label.to(stepper.label.device), stepper.label))
        if stepper.act_dtype != act_dtype or not same_label or stepper.doctree is not doctree:
            raise ValueError('sample_loop: the stepper was built for another doctree / label / act_dtype')
    st = stepper or HRStepper(unet_hr, unet_lr, doctree, act_dtype, label, use_cuda_graph)
    if noise is None:
        g = torch.Generator(device=doctree.device).manual_seed(seed)
        noise = torch.randn(st.x.shape, generator=g, device=doctree.device)
    st.set_latent(noise)
    ls = sampling_log_snr(ddim_steps)
    for i in range(ddim_steps):
        st.step(ls[i], ls[i + 1])
    return st.x.clone()


TRUNCATED_TIME = 0.7        # reference models/octfusion_model_union.py:39


def truncation_flags(ddim_steps: int, truncated_index: float = TRUNCATED_TIME):
    """Per step (do_sign, add_noise) of the stage-1 loop, decided exactly as the reference does: on the float32 time
    tensors (`t[0] < truncated_index`, octfusion_model_union.py:324; `t_next > truncated_index`, :339).  torch casts
    the Python scalar to the tensor's dtype, so 0.7 is compared as float32(0.7) = 0.699999988, which
    linspace(1, 0, steps+1) hits exactly for steps = 10, 50, 100, 200, 1000 -- a float64 compare would apply sign()
    one step early there."""
    times = torch.linspace(1.0, 0.0, ddim_steps + 1, dtype=torch.float32)
    do_sign = [bool(times[i] < truncated_index) for i in range(ddim_steps)]
    add_noise = [bool(times[i + 1] > truncated_index) for i in range(ddim_steps)]
    return do_sign, add_noise


@torch.no_grad()
def sample_loop_lr(unet_lr, batch_size, z_shape=(8, 16, 16, 16), ddim_steps=200, label=None, seed=0,
                   truncated_index=TRUNCATED_TIME, act_dtype=torch.bfloat16, device='cuda', noises=None):
    """Stage 1 ("lr", df_type "x0") of reference sample_loop (octfusion_model_union.py:300-344): the dense 16^3 U-Net
    with self-conditioning predicts x0; below `truncated_index` the prediction is replaced by its sign and no noise
    is added.  `noises` (list of steps+1 tensors: initial latent, then one per step) makes the run reproducible for
    tests; otherwise a seeded device generator is used.  Returns the split signal [B, 8, 16, 16, 16] fp32."""
    dev = torch.device(device)
    g = torch.Generator(device=dev).manual_seed(seed)
    shape = (batch_size, *z_shape)
    draw = (lambda i: noises[i].to(dev).float().contiguous()) if noises is not None else \
        (lambda i: torch.randn(shape, generator=g, device=dev))
    x = draw(0).clone()
    x_start = None
    times = torch.linspace(1.0, 0.0, ddim_steps + 1)
    do_sign, add_noise = truncation_flags(ddim_steps, truncated_index)
    ls_dev = torch.zeros(1, device=dev)
    lsn_dev = torch.zeros(1, device=dev)
    ts = torch.zeros(batch_size, device=dev)
    for i in range(ddim_steps):
        t, t_next = float(times[i]), float(times[i + 1])
        ls, lsn = beta_linear_log_snr(t), beta_linear_log_snr(t_next)
        ts.fill_(ls); ls_dev.fill_(ls); lsn_dev.fill_(lsn)
        xin = x if act_dtype == torch.float32 else x.to(act_dtype)
        sc = None if x_start is None else (x_start if act_dtype == torch.float32 else x_start.to(act_dtype))
        pred = unet_lr(x=xin, timesteps=ts, x_self_cond=sc, label=label).float().contiguous()
        noise = draw(i + 1) if add_noise[i] else None
        ops.ddpm_x0_update(x, pred, ls_dev, lsn_dev, noise=noise, do_sign=do_sign[i])
        x_start = pred
    return x


@torch.no_grad()
def sample_shapes(stage1_unet_lr, unet_hr, unet_lr, vae, batch_size, ddim_steps=200, label=None, seed=0,
                  act_dtype=torch.bfloat16, full_depth=4, octree_depth=6, split_small=None, device='cuda'):
    """The reference's `OctFusionModel.sample` flow without mesh export (octfusion_model_union.py:354-400), every stage
    on the device: stage-1 dense sampler -> split signal -> octree (`split2octree_small`) -> dual graph -> stage-2
    latent sampler (CUDA graph per step) -> GraphVAE decoder growing the octree to depth 8.
    Returns {'split_small', 'octree_small', 'doctree_small', 'samples', 'logits', 'reg_voxs', 'octree_out'}; the
    reference's NeuralMPU / marching cubes keep consuming `reg_voxs` and `octree_out`."""
    from .octree import split2octree_small
    from .dual_octree import DualOctree
    if split_small is None:
        split_small = sample_loop_lr(stage1_unet_lr, batch_size, ddim_steps=ddim_steps, label=label, seed=seed,
                                     act_dtype=act_dtype, device=device)
    octree_small = split2octree_small(split_small, octree_depth, full_depth)
    doctree_small = DualOctree(octree_small)
    doctree_small.post_processing_for_docnn()
    samples = sample_loop(unet_hr, unet_lr, doctree_small, ddim_steps=ddim_steps, label=label, seed=seed,
                          act_dtype=act_dtype)
    out = {'split_small': split_small, 'octree_small': octree_small, 'doctree_small': doctree_small, 'samples': samples}
    if vae is not None:
        code = samples if act_dtype == torch.float32 else samples.to(act_dtype)
        out.update(vae.decode_code(code, doctree_small, update_octree=True))
    return out
