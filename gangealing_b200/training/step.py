"""One GANgealing training iteration (reference train.py:89-136) as a reusable object.

Trainer.step() = gangealing_loss forward (G x2, STN, perceptual) -> TV / identity regularisers -> backward
(DDP all-reduces the STN gradients over NCCL) -> Adam x2 -> EMA of the STN -> loss reduce.  It is what bench.py
times for the "train images/sec at 256^2" metric.
"""
import contextlib
import dataclasses

import torch
from torch import nn, optim

from ..stn import BilinearDownsample, get_stn
from ..stylegan2 import Generator
from . import distributed as gdist
from .latent_learner import PCA, DirectionInterpolator, kmeans_plusplus
from .losses import flow_identity_loss, gangealing_cluster_loss, gangealing_loss, total_variation_loss
from .perceptual import get_perceptual_loss


def requires_grad(model, flag=True):
    for p in model.parameters():
        p.requires_grad = flag


def accumulate(model1, model2, decay=0.999):
    """EMA of parameters (reference models/__init__.py:19-24), as two fused multi-tensor ops."""
    p1 = dict(model1.named_parameters())
    p2 = dict(model2.named_parameters())
    keys = list(p1.keys())
    a = [p1[k].data for k in keys]
    b = [p2[k].data for k in keys]
    torch._foreach_mul_(a, decay)
    torch._foreach_add_(a, b, alpha=1 - decay)


@dataclasses.dataclass
class TrainConfig:
    """Defaults = BASELINE config 2 (LSUN Cats 256^2, unimodal similarity+flow STN, fp32);
    reference utils/base_argparse.py + scripts/training/lsun_cats_lpips.sh."""
    gen_size: int = 256
    flow_size: int = 128
    dim_latent: int = 512
    n_mlp: int = 8
    gen_channel_multiplier: int = 2
    stn_channel_multiplier: float = 0.5
    transform: tuple = ("similarity", "flow")
    num_heads: int = 1
    flips: bool = False
    ndirs: int = 1
    inject: int = 5
    batch: int = 5                    # per GPU (reference default)
    padding_mode: str = "border"
    sample_from_full_res: bool = False
    tv_weight: float = 2500.0
    flow_identity_weight: float = 0.0
    stn_lr: float = 1e-3
    ll_lr: float = 1e-2
    freeze_ll: bool = False
    psi: float = 0.5
    seed: int = 0
    channels_last: bool = True        # generator + STN-trunk activations NHWC on CUDA (no cuDNN layout conversions)
    dtype: str = "f32"                # "f32" (BASELINE config 2) or "bf16" (config 3): STORAGE type of the generator / STN
    #                                   trunk / VGG activations; fp32 master weights, fp32 arithmetic in the fused kernels,
    #                                   bf16 tensor-core convolutions, fp32 images / grids / losses / optimiser
    fused_optimizer: bool = True      # CUDA: Adam x2 + EMA as ONE multi-tensor kernel (training/fused_optim.py)
    fused_weight_scaling: bool = True  # CUDA: the STN's 62 `weight * scale` products (and their backward) as a few multi-tensor
    #                                    launches per step (op/scaled_weights.py)
    grad_compression: str = "none"    # DDP gradient all-reduce: "none" (fp32) or "bf16" (compressed on the wire)
    bucket_cap_mb: int = 25


class Trainer:
    """Builds G (frozen), STN (+EMA copy), latent learner, perceptual loss and optimisers; `step()` runs one iteration.
    `ops`: None = the sm_90a op set; tests/bench's CPU legs pass the oracle's."""

    def __init__(self, cfg, device, ops=None, distributed=False, seed_offset=0):
        self.cfg, self.device, self.distributed, self.ops = cfg, device, distributed, ops
        torch.manual_seed(cfg.seed)  # identical weights on every rank (stands in for the shared checkpoint)
        self.generator = Generator(cfg.gen_size, cfg.dim_latent, cfg.n_mlp, channel_multiplier=cfg.gen_channel_multiplier,
                                   ops=ops).to(device).eval()
        self.generator.channels_last = torch.device(device).type == "cuda" and ops is None and cfg.channels_last
        kw = dict(flow_size=cfg.flow_size, supersize=cfg.gen_size if cfg.sample_from_full_res else cfg.flow_size,
                  channel_multiplier=cfg.stn_channel_multiplier, num_heads=cfg.num_heads, ops=ops)
        self.stn = get_stn(list(cfg.transform), **kw).to(device)
        self.t_ema = get_stn(list(cfg.transform), **kw).to(device)
        self.t_ema.load_state_dict(self.stn.state_dict())
        if cfg.dtype not in ("f32", "bf16"):
            raise ValueError("TrainConfig.dtype must be 'f32' or 'bf16'")
        act_dtype = torch.bfloat16 if cfg.dtype == "bf16" else torch.float32
        if act_dtype != torch.float32 and not self.generator.channels_last:
            raise RuntimeError("bf16 activations need the channels-last sm_90a path (CUDA device, channels_last=True)")
        self.generator.act_dtype = act_dtype
        if self.generator.channels_last:
            # 4-D STN parameters are STORED channels-last (KRSC): cuDNN's NHWC kernels take them as they are (no per-call
            # weight re-layout copies), weight gradients come back in the same layout, and DDP's bucket views -- created
            # from the parameters' strides -- match the gradients (round 1's "grad strides differ from bucket view" copies)
            self.stn.to(memory_format=torch.channels_last)
            self.t_ema.to(memory_format=torch.channels_last)
            for m in list(self.stn.modules()) + list(self.t_ema.modules()):
                if hasattr(m, "channels_last") and hasattr(m, "stn_in_size"):
                    m.channels_last = True
                    m.act_dtype = act_dtype
        self.ll = DirectionInterpolator(None, cfg.ndirs, cfg.inject, self.generator.n_latent, num_heads=cfg.num_heads,
                                        dim_latent=cfg.dim_latent).to(device)
        self.loss_fn = get_perceptual_loss(device, seed=cfg.seed + 1, ops=ops)
        if act_dtype != torch.float32:
            # frozen VGG16: bf16 filters and feature maps; biases stay fp32 (applied by the fused bias+ReLU kernel, which
            # takes fp32 per-channel constants); fp32 distance
            for m in self.loss_fn.net.modules():
                if isinstance(m, nn.Conv2d):
                    m.weight.data = m.weight.data.to(act_dtype)
        self.resize_fake2stn = (BilinearDownsample(cfg.gen_size // cfg.flow_size, 3, ops=ops).to(device)
                                if cfg.gen_size > cfg.flow_size else nn.Sequential())
        requires_grad(self.generator, False)
        requires_grad(self.stn, True)
        requires_grad(self.ll, True)
        requires_grad(self.t_ema, False)
        self.t_module, self.ll_module = self.stn, self.ll
        self._side = None
        if distributed:
            on_gpu = device != "cpu" and torch.device(device).type == "cuda"
            ids = [torch.cuda.current_device()] if on_gpu else None

            def wrap():
                self.stn = nn.parallel.DistributedDataParallel(self.stn, device_ids=ids, broadcast_buffers=False,
                                                               gradient_as_bucket_view=True, bucket_cap_mb=cfg.bucket_cap_mb)
                self.ll = nn.parallel.DistributedDataParallel(self.ll, device_ids=ids, broadcast_buffers=False)
                if cfg.grad_compression == "bf16":   # halves the bytes of the one exchange step (172 MB of fp32 STN gradients)
                    from torch.distributed.algorithms.ddp_comm_hooks import default_hooks
                    self.stn.register_comm_hook(None, default_hooks.bf16_compress_hook)
            if on_gpu:
                # DDP stashes the AccumulateGrad nodes, which stay pinned to the stream they were created on: build the
                # wrapper on the ONE side stream the step will be warmed up and captured on (capture()), so that inside the
                # captured graph gradients are accumulated on the capturing stream itself (no cross-stream joins)
                self._side = torch.cuda.Stream()
                self._side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(self._side):
                    wrap()
                torch.cuda.current_stream().wait_stream(self._side)
                torch.autograd.graph.set_warn_on_accumulate_grad_stream_mismatch(False)   # eager steps run on the default stream
            else:
                wrap()
        fused = torch.device(device).type == "cuda"
        # capturable: the optimiser state AND the learning rates live on the device, psi too, so ONE captured CUDA graph
        # serves the whole schedule (psi 1 -> 0, cyclic lr: reference train.py:89-96,129-132); `step(psi=, lr=, ll_lr=)`
        # copies new values into these scalars before the replay
        self.psi_t = torch.tensor(float(cfg.psi), device=device)
        self.accum = 0.5 ** (32 / (10 * 1000))
        self.fused_optim = None
        if fused and ops is None and cfg.fused_optimizer:
            # train.py:126-134 in one kernel: Adam for the STN and the latent learner + the EMA of the STN
            from .fused_optim import FusedAdamEMA
            groups = [{"params": list(self.t_module.parameters()), "lr": cfg.stn_lr}]
            if not cfg.freeze_ll:
                groups.append({"params": list(self.ll_module.parameters()), "lr": cfg.ll_lr})
            ema = dict(self.t_ema.named_parameters())
            pairs = {p: ema[k] for k, p in self.t_module.named_parameters()}
            self.fused_optim = FusedAdamEMA(groups, betas=(0.9, 0.999), eps=1e-8, ema_pairs=pairs, ema_decay=self.accum)
            self.t_optim = self.ll_optim = self.fused_optim
            self.stn_lr_t = self.fused_optim.lr_tensor(0)
            self.ll_lr_t = self.fused_optim.lr_tensor(1) if not cfg.freeze_ll else None
        else:
            self.stn_lr_t = torch.tensor(float(cfg.stn_lr), device=device) if fused else None
            self.ll_lr_t = torch.tensor(float(cfg.ll_lr), device=device) if fused else None
            self.t_optim = optim.Adam(self.t_module.parameters(), lr=self.stn_lr_t if fused else cfg.stn_lr, betas=(0.9, 0.999),
                                      eps=1e-8, fused=fused, capturable=fused)
            self.ll_optim = optim.Adam(self.ll_module.parameters(), lr=self.ll_lr_t if fused else cfg.ll_lr, betas=(0.9, 0.999),
                                       eps=1e-8, fused=fused, capturable=fused)
        self.weight_scaler = None
        if fused and ops is None and cfg.fused_weight_scaling:
            from ..op.scaled_weights import WeightScaler, equalized_layers
            layers = equalized_layers(self.t_module)
            if layers:
                self.weight_scaler = WeightScaler(layers)
                for module, _ in layers:
                    module.scaler = self.weight_scaler
        self._graph = None
        self.zero = torch.tensor(0.0, device=device)
        # each rank draws its own latents (reference train.py:193: seed*world + rank)
        torch.manual_seed(cfg.seed * max(1, gdist.get_world_size()) + gdist.get_rank() + seed_offset)

    def losses(self, z=None):
        cfg = self.cfg
        if cfg.num_heads > 1 or cfg.flips:
            perceptual, delta_flow = gangealing_cluster_loss(
                self.generator, self.stn, self.ll, self.loss_fn, self.resize_fake2stn, self.psi_t, cfg.batch, cfg.dim_latent,
                cfg.freeze_ll, cfg.num_heads, cfg.flips, self.device, sample_from_full_res=cfg.sample_from_full_res, z=z,
                padding_mode=cfg.padding_mode)
        else:
            perceptual, delta_flow = gangealing_loss(
                self.generator, self.stn, self.ll, self.loss_fn, self.resize_fake2stn, self.psi_t, cfg.batch, cfg.dim_latent,
                cfg.freeze_ll, self.device, sample_from_full_res=cfg.sample_from_full_res, z=z,
                padding_mode=cfg.padding_mode)
        tv = total_variation_loss(delta_flow) if cfg.tv_weight > 0 else self.zero
        idt = flow_identity_loss(delta_flow) if cfg.flow_identity_weight > 0 else self.zero
        return {"p": perceptual, "tv": tv, "f": idt}

    def set_schedule(self, psi=None, lr=None, ll_lr=None):
        """Update the truncation psi and the two learning rates (plain floats or 0-dim tensors).  They live in device
        scalars, so this works before AND after `capture()` -- the captured graph reads them at replay time."""
        if psi is not None:
            self.psi_t.fill_(psi) if not torch.is_tensor(psi) else self.psi_t.copy_(psi, non_blocking=True)
        for value, scalar, optimiser in ((lr, self.stn_lr_t, self.t_optim), (ll_lr, self.ll_lr_t, self.ll_optim)):
            if value is None:
                continue
            if scalar is not None:
                scalar.fill_(value) if not torch.is_tensor(value) else scalar.copy_(value, non_blocking=True)
            elif optimiser is not self.fused_optim:
                for group in optimiser.param_groups:
                    group["lr"] = float(value)

    def set_iteration(self, i, **recipe):
        """psi and learning rates of iteration `i` of the reference recipe (training/schedule.py:schedule_at)."""
        from .schedule import schedule_at
        s = schedule_at(i, self.cfg.stn_lr, self.cfg.ll_lr, **recipe)
        self.set_schedule(psi=s["psi"], lr=s["stn_lr"], ll_lr=s["ll_lr"])
        return s

    # ---- checkpoints in the reference's layout (train.py:20-27 `save_state_dict`, :214-224 restore) -----------------------
    def checkpoint(self, iteration=None):
        """-> dict with the reference's keys: `g_ema`, `t`, `t_ema`, `t_optim`, `ll`, `ll_optim` (optimiser dicts in
        torch.optim.Adam's layout, whichever optimiser runs here).  The reference's `t_sched` / `ll_sched` entries have no
        counterpart: the schedule is a closed form of the iteration (training/schedule.py), stored as `iteration`."""
        if self.fused_optim is not None:
            from .fused_optim import split_adam_state_dict
            parts = split_adam_state_dict(self.fused_optim.state_dict())
            t_sd, ll_sd = parts[0], (parts[1] if len(parts) > 1 else None)
        else:
            t_sd, ll_sd = self.t_optim.state_dict(), self.ll_optim.state_dict()
        return {"g_ema": self.generator.state_dict(), "t": self.t_module.state_dict(), "t_ema": self.t_ema.state_dict(),
                "t_optim": t_sd, "ll": self.ll_module.state_dict(), "ll_optim": ll_sd, "iteration": iteration}

    def load_checkpoint(self, ckpt, load_G_only=False):
        """Restore from a reference checkpoint (or one of `checkpoint()`): the generator always, and -- unless `load_G_only`
        or the checkpoint holds nothing else (train.py:216-225 falls through the same way) -- STN, EMA, latent learner and the
        Adam state.  In place: parameters, moments and the step counter keep their addresses (the fused kernels' pointer
        tables stay valid).  A captured CUDA graph is nevertheless RELEASED: the frozen generator's derived filter banks
        (`scale * W` re-laid out, `sum W^2`: memoised per parameter version, op/modconv.py) are constants of the capture, and
        a replay would keep synthesising with the old generator -- call `capture()` again.
        -> True when the full training state was restored."""
        if self._graph is not None:
            self.release_graph()
        self.generator.load_state_dict(ckpt["g_ema"])
        if load_G_only or "t" not in ckpt:
            return False
        self.t_module.load_state_dict(ckpt["t"])
        self.t_ema.load_state_dict(ckpt["t_ema"])
        self.ll_module.load_state_dict(ckpt["ll"])
        if self.fused_optim is not None:
            from .fused_optim import merge_adam_state_dicts
            parts = [ckpt["t_optim"]] + ([ckpt["ll_optim"]] if len(self.fused_optim.param_groups) > 1 else [])
            self.fused_optim.load_state_dict(merge_adam_state_dicts(parts))
        else:
            self.t_optim.load_state_dict(ckpt["t_optim"])
            if ckpt.get("ll_optim") is not None:
                self.ll_optim.load_state_dict(ckpt["ll_optim"])
            for scalar, optimiser in ((self.stn_lr_t, self.t_optim), (self.ll_lr_t, self.ll_optim)):
                if scalar is not None:      # capturable Adam: the learning rate must stay the device scalar the graph reads
                    for group in optimiser.param_groups:
                        scalar.copy_(group["lr"]) if torch.is_tensor(group["lr"]) else scalar.fill_(float(group["lr"]))
                        group["lr"] = scalar
        if ckpt.get("iteration") is not None:
            self.set_iteration(int(ckpt["iteration"]))
        return True

    @torch.no_grad()
    def init_target_mode(self, n_pca=1_000_000, n_kmeans=50_000, debug=False):
        """Initialise the latent learner from the generator, as reference train.py:228-243 does after loading only
        `g_ema`: an IncrementalPCA of n_pca generated latents (n_pca // world per rank, all-gathered) gives `directions`
        and `lat_mean`; with several heads, k-means++ over n_kmeans latents (or, with `debug`, num_heads random latents)
        gives the centroids whose PCA codes become `coefficients`.  `debug` also sets n_pca = 1000.
        The three tensors are written in place: the fused optimiser's pointer table and a captured graph stay valid.
        -> the fitted PCA."""
        cfg = self.cfg
        if debug:
            n_pca = 1000
        batch_w = gdist.all_gather(self.generator.batch_latent(n_pca // gdist.get_world_size()))
        pca = PCA(cfg.ndirs, batch_w, ops=self.ops)
        ll = self.ll_module
        ll.directions.copy_(torch.from_numpy(pca.components_).float())
        ll.lat_mean.copy_(torch.from_numpy(pca.mean_[None]).float())
        if cfg.num_heads > 1:
            if debug:
                centroids = self.generator.batch_latent(cfg.num_heads)
            else:
                centroids = kmeans_plusplus(cfg.num_heads, n_kmeans, self.generator, self.loss_fn, cfg.inject)
            ll.assign_coefficients(pca.encode(centroids))
        return pca

    def step(self, z=None, psi=None, lr=None, ll_lr=None):
        """-> dict of (rank-0 averaged) scalar loss tensors, still on the device (no host sync here).
        After `capture()` the iteration is replayed from a CUDA graph (z, if given, is copied into its static input;
        psi / lr / ll_lr, if given, into the device scalars the graph reads)."""
        if psi is not None or lr is not None or ll_lr is not None:
            self.set_schedule(psi, lr, ll_lr)
        if self._graph is not None:
            if z is None:
                self._static_z.normal_()
            else:
                self._static_z.copy_(z, non_blocking=True)
            self._graph.replay()
            return self._static_out
        return self._eager_step(z)

    def capture(self, warmup=3):
        """Capture one whole iteration (G x2, STN, loss, backward, Adam x2, EMA) into a CUDA graph.

        The reference's loop is launch-bound at its recipe's per-GPU batch (thousands of launches per step,
        SURVEY.md 8e "scaling risk"); every op on this path is graph-safe: static shapes, no host sync (the fused
        sampler drops MipmapWarp's `.item()`), device-side RNG and optimiser state.  Under DDP the NCCL bucket
        all-reduces and the loss reduce are captured as graph nodes too."""
        if self.distributed:
            warmup = max(warmup, 11)  # DDP needs >= 11 eager iterations on the side stream before capture (PyTorch docs)
        self.release_graph()          # re-capture: the warm-up below runs eagerly (see the guard in _eager_step)
        cfg = self.cfg
        self._static_z = torch.randn(cfg.batch, cfg.dim_latent, device=self.device)
        side = self._side if self._side is not None else torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self._eager_step(self._static_z)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        self.t_optim.zero_grad(set_to_none=True)
        self.ll_optim.zero_grad(set_to_none=True)
        with torch.cuda.graph(graph, stream=side):
            out = self._eager_step(self._static_z)
            self._static_out = {k: v.detach() for k, v in out.items()}
        self._graph = graph
        return self

    def release_graph(self):
        """Drop the captured graph (before tearing down the process group whose collectives it references)."""
        self._graph = None
        self._static_out = None

    def _eager_step(self, z=None):
        if self._graph is not None:
            # the captured graph re-reads the pinned pointer tables of the multi-tensor kernels (optimiser, weight scaler) at
            # every replay; an eager step rewrites those tables with ITS tensors' addresses -- later replays would scatter
            # into freed memory.  step() never mixes the two; refuse a direct call that would.
            raise RuntimeError("Trainer: an eager step while a captured graph is held; call release_graph() first")
        cfg = self.cfg
        # the scaled-weight cache is valid for exactly one forward + backward: the optimiser below changes the parameters
        scope = self.weight_scaler.step() if self.weight_scaler is not None else contextlib.nullcontext()
        with scope:
            loss_dict = self.losses(z)
            self.t_optim.zero_grad(set_to_none=True)
            self.ll_optim.zero_grad(set_to_none=True)
            full = loss_dict["p"] + cfg.tv_weight * loss_dict["tv"] + cfg.flow_identity_weight * loss_dict["f"]
            full.backward()
        if self.fused_optim is not None:
            self.fused_optim.step()               # Adam (both groups) + EMA: one multi-tensor kernel
        else:
            self.t_optim.step()
            if not cfg.freeze_ll:
                self.ll_optim.step()
            accumulate(self.t_ema, self.t_module, self.accum)
        # detached: a caller that keeps the returned dict must not keep the iteration's autograd graph (and its
        # AccumulateGrad nodes, which are pinned to the stream they were created on) alive
        return gdist.reduce_loss_dict({k: v.detach() for k, v in loss_dict.items()})
