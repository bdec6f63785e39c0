"""Run-to-run determinism of the training path: the backward kernels that gather instead of using atomics give the same
bits on identical inputs, the training step never asks for the one gradient that still uses atomics, and a whole eager
training step is bitwise reproducible.

Left out on purpose: the gradient w.r.t. the SOURCE image of the sampler (csrc/warp.cu scatter_level and
mip_down_bwd_kernel) accumulates with atomicAdd, so its rounding depends on the order the atomics land in.  Training never
needs it (the STN's input is the frozen generator's output), which test_training_step_never_requests_the_source_gradient
enforces."""
import dataclasses

import pytest
import torch
import torch.nn.functional as F

from demod_reference import demod_inputs
from fp64_contract import grid_stride_batch
from oracle import flow as FL
from oracle import sampling as S

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _twice(fn):
    """fn() -> tuple of tensors, evaluated twice on identical inputs; every pair must be bitwise equal."""
    a, b = fn(), fn()
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), "output %d differs between two runs (max diff %.3e)" % (i, (x - y).abs().max().item())


def _inputs(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 3, 128, 128, generator=g).to(DEV)
    theta = (torch.eye(2, 3)[None] * (0.5 + 1.5 * torch.rand(n, 1, 1, generator=g)) + 0.15 * torch.randn(n, 2, 3, generator=g)).to(DEV)
    go = torch.randn(n, 3, 128, 128, generator=g).to(DEV)
    low = (0.0125 * torch.randn(n, 16, 16, 2, generator=g)).to(DEV)
    mask = (2.0 * torch.randn(n, 576, 16, 16, generator=g)).to(DEV)
    base = (torch.eye(2, 3)[None] * 1.4 + 0.1 * torch.randn(n, 2, 3, generator=g)).to(DEV)
    alpha = torch.rand(n, generator=g).to(DEV)
    gf = torch.randn(n, 128, 128, 2, generator=g).to(DEV)
    return x, theta, go, low, mask, base, alpha, gf


def test_sampler_grid_gradients_are_deterministic():
    """grad_grid of MipmapWarp and the grid-generator gradients of both one-pass samplers, at a batch beyond one trip of
    the grid-stride loops (the source does not require grad: its gradient uses atomics, see the module docstring)."""
    from gangealing_b200.stn import sampling as GS
    n = grid_stride_batch(128, 128)
    x, theta, go, low, mask, base, alpha, gf = _inputs(n)
    ident = S.affine_grid_ref(torch.eye(2, 3)[None], (1, 1, 128, 128)).to(DEV)
    grid = (F.affine_grid(theta, (n, 3, 128, 128), align_corners=False) + 0.02 * gf).detach()

    def mipmap():
        gr = grid.clone().requires_grad_(True)
        return torch.autograd.grad(GS.mipmap_warp(x, gr, 4, 0.0, "border")[0], gr, go)

    def affine():
        th = theta.clone().requires_grad_(True)
        out, gr, _ = GS.stn_sample_affine(x, th, (128, 128), 4, 0.0, "reflection")
        return torch.autograd.grad((out * go).sum(), th)

    def flow():
        leaves = [t.clone().requires_grad_(True) for t in (low, mask, base)]
        out, fl, delta, _ = GS.stn_sample_flow(x, leaves[0], leaves[1], ident, leaves[2], alpha, 8, 4, 0.0, "border")
        return torch.autograd.grad((out * go).sum() + (fl * gf).sum() + delta.square().sum(), leaves)

    for fn in (mipmap, affine, flow):
        _twice(fn)


def test_flow_compose_gradients_are_deterministic():
    """g_low (warp-per-entry gather), g_mask and g_base (per-sample block reduction) of flow_compose."""
    from gangealing_b200 import stn
    n = grid_stride_batch(128, 128)
    _, _, _, low, mask, base, alpha, gf = _inputs(n, seed=1)
    ident = FL.identity_flow_ref(128, 128).to(DEV)

    def run():
        leaves = [t.clone().requires_grad_(True) for t in (low, mask, base)]
        delta, fl = stn.flow_compose(leaves[0], leaves[1], ident, leaves[2], alpha, 8)
        return torch.autograd.grad((fl * gf).sum() + (delta * gf.flip(1)).sum(), leaves)

    _twice(run)


def test_demodulation_is_deterministic():
    """The demodulation coefficients (single-layer and batched launches) and their style gradients."""
    from gangealing_b200.op import style_path
    from gangealing_b200.op.modconv import demod_coefficients
    w, s, scale = demod_inputs(65, 200, 257)
    w2, s2, scale2 = demod_inputs(65, 512, 512, seed=1)
    gd = torch.randn(65, 200, device=DEV)

    def single():
        sg = s.to(DEV).requires_grad_(True)
        d = demod_coefficients(w.to(DEV), sg, scale)
        return (d,) + torch.autograd.grad(d, sg, gd)

    def batched():
        sg = [s.to(DEV).requires_grad_(True), s2.to(DEV).requires_grad_(True)]
        d = style_path.all_demod([w.to(DEV), w2.to(DEV)], sg, [scale, scale2])
        return tuple(d) + torch.autograd.grad(d[0].sum() + (d[1] * 0.5).sum(), sg)

    _twice(single)
    _twice(batched)


def _config():
    from gangealing_b200.training.step import TrainConfig
    return TrainConfig(gen_size=64, flow_size=64, dim_latent=32, n_mlp=2, batch=8, inject=3, seed=4)


@pytest.fixture
def deterministic_cudnn():
    """cuDNN with a fixed algorithm choice, as bench.py runs the step (the autotuner's choice varies from run to run)."""
    old = torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    yield
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = old


def test_training_step_never_requests_the_source_gradient(monkeypatch, deterministic_cudnn):
    """Every sampler backward of a training step passes a null grad_src: the step's determinism rests on it."""
    from gangealing_b200 import _lib
    from gangealing_b200.training.step import Trainer
    lib = _lib.load()
    real = lib.gg_mipmap_warp_backward
    grad_src_args = []

    def recording(*args):
        grad_src_args.append(args[0])
        return real(*args)

    monkeypatch.setattr(lib, "gg_mipmap_warp_backward", recording)
    tr = Trainer(_config(), DEV)
    tr.step()
    torch.cuda.synchronize()
    assert grad_src_args, "the step ran no sampler backward"
    assert all(a is None for a in grad_src_args), "a training step asked the sampler for the source-image gradient"


def test_training_step_is_bitwise_reproducible(deterministic_cudnn):
    """Two Trainers from the same seed, fed the same latents and reseeded before every step: after 3 eager steps the STN,
    its EMA, the latent learner and the whole Adam state are bitwise equal."""
    from gangealing_b200.training.step import Trainer
    cfg = _config()
    trainers = [Trainer(cfg, DEV), Trainer(dataclasses.replace(cfg), DEV)]
    zs = torch.randn(3, cfg.batch, cfg.dim_latent, generator=torch.Generator().manual_seed(11)).to(DEV)
    for tr in trainers:
        for k in range(3):
            torch.manual_seed(100 + k)
            tr.step(z=zs[k])
    torch.cuda.synchronize()
    a, b = trainers
    for name, ma, mb in (("stn", a.t_module, b.t_module), ("stn_ema", a.t_ema, b.t_ema), ("latent_learner", a.ll_module, b.ll_module)):
        for (k, pa), (_, pb) in zip(ma.named_parameters(), mb.named_parameters()):
            assert torch.equal(pa, pb), "%s.%s differs between two identical runs" % (name, k)
    sa, sb = a.t_optim.state_dict()["state"], b.t_optim.state_dict()["state"]
    assert sa.keys() == sb.keys() and sa
    for k in sa:
        for field, va in sa[k].items():
            vb = sb[k][field]
            assert torch.equal(va, vb) if torch.is_tensor(va) else va == vb, "Adam state %s[%s] differs" % (k, field)
