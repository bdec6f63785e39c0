"""Time one round of training visuals at the reference's defaults (gen 256, flow 128, n_mean 8000, n_sample 64,
vis_batch_size 250) for K = 1 and K = 4 heads: the port (gangealing_b200.training.visuals) against the reference's
formulation on this repository's networks (utils/vis_tools/training_vis.py: every congealed real image kept in a host
list, one .cpu() per assigned fake, host sums, numpy flow images, images2grid per grid).

    python tools/trainvisbench.py [--heads 1 4] [--n-mean 8000] [--out DIR]

Every (K, leg) runs in a process of its own so that its peak host memory (ru_maxrss) is its own; each prints one JSON
line and the driver prints them with the card's name and power limit.  Weights are random (seeded): the work does not
depend on them.  Writes nothing but --out (default: a temporary directory)."""
import argparse
import json
import os
import resource
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _setup(k, n_mean, real_batch):
    import torch
    from gangealing_b200.training import TrainConfig, Trainer
    cfg = TrainConfig(num_heads=k)                      # gen 256, flow 128 (BASELINE config 2), k heads
    tr = Trainer(cfg, "cuda")
    g = torch.Generator(device="cuda").manual_seed(1)
    z = torch.randn(64, cfg.dim_latent, device="cuda", generator=g)
    big_z = torch.randn(n_mean, cfg.dim_latent, device="cuda", generator=g)
    # real images at the STN's input size, as the reference's real loader yields them at flow size
    reals = torch.randn(64, 3, cfg.flow_size, cfg.flow_size, device="cuda", generator=g).clamp(-1, 1)
    loader = [torch.randn(real_batch, 3, cfg.flow_size, cfg.flow_size, device="cuda", generator=g).clamp(-1, 1)
              for _ in range(-(-n_mean // real_batch))]
    return tr, z, big_z, reals, loader


def _reference_round(tr, z, big_z, reals, loader, n_mean, n_sample, vis_batch_size):
    """create_training_visuals / create_training_cluster_visuals as the reference runs them, on this repo's networks."""
    import numpy as np
    import torch
    from oracle.training_vis import flow_colors
    from torchvision.utils import make_grid
    from gangealing_b200.training import assign_fake_images_to_clusters, sample_gan_supervised_pairs
    cfg, k, dev = tr.cfg, tr.cfg.num_heads, "cuda"
    kw = dict(padding_mode=cfg.padding_mode)
    grids = {}

    def log(images, name, range=(-1, 1), scale_each=False):
        nrow = max(1, int(images.size(0) ** 0.5))
        g = make_grid(images, nrow=nrow, padding=2, pad_value=0, normalize=True, value_range=range, scale_each=scale_each)
        grids[name] = g.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to("cpu", torch.uint8).numpy()

    out, total = [], 0                                   # run_loader_mean: every congealed image on the host
    for x in loader:
        out.append(tr.t_ema(x, unfold=True, **kw).cpu())
        total += x.size(0)
        if total >= n_mean:
            break
    out = torch.cat(out, 0)
    means = out.sum(0).to(dev) / out.size(0)
    log(means.reshape(-1, *means.shape[-3:]), "mean_EMA_transformed_real_sample", None, True)
    if k == 1:
        transformed, flow = tr.t_ema(reals, return_flow=True, **kw)
        log(transformed[:n_sample], "EMA_transformed_real_sample")
        colors = torch.from_numpy(flow_colors(flow.cpu().numpy())).float().div(255.0).permute(0, 3, 1, 2)
        log(colors[:n_sample], "flow_real", (0, 1))
    else:
        log(out.view(-1, *out.shape[2:])[:n_sample], "EMA_transformed_real_sample")
        for h in range(k):
            log(out[:, h][:n_sample], "EMA_head_%d" % h)
        heads, total, vb = [[] for _ in range(k)], 0, max(1, vis_batch_size // k)
        while True:                                      # generate_cluster_congeal: one .cpu() per assigned image
            z_in = big_z[total:total + vb]
            a, aligned, _, _, _, _ = assign_fake_images_to_clusters(
                tr.generator, tr.t_ema, tr.ll_module, tr.loss_fn, tr.resize_fake2stn, tr.psi_t, z_in.size(0), None, True,
                k, cfg.flips, dev, sample_from_full_res=True, z=z_in, **kw)
            aligned = aligned.view(z_in.size(0), k, *aligned.shape[1:])
            for warp, c in zip(aligned[torch.arange(z_in.size(0), device=dev), a.indices], a.indices):
                heads[c.item() % k].append(warp.cpu())
            total += z_in.size(0)
            if total >= n_mean:
                break
        size = aligned.size(-1)
        for h in heads:
            h.extend([torch.zeros(3, size, size)] * max(0, n_sample - len(h)))
        stacked = [torch.stack(h, 0) for h in heads]
        cm = torch.stack([h.sum(0) for h in stacked]).to(dev) / torch.tensor([float(h.size(0)) for h in stacked],
                                                                              device=dev).view(k, 1, 1, 1)
        log(cm, "mean_generated_EMA_transformed_assigned", None, True)
        for h in range(k):
            log(stacked[h][:n_sample], "generated_EMA_assigned_head_%d" % h)
    sample, truncated = sample_gan_supervised_pairs(tr.generator, tr.ll_module, lambda x: x, tr.psi_t, n_sample, None, True,
                                                    dev, z=z)
    transformed = tr.t_ema(tr.resize_fake2stn(sample), **kw)
    for images, name in ((sample, "sample"), (transformed, "transformed_sample"), (truncated, "truncated_sample")):
        log(images[:n_sample], name)
        log(images.mean(0, keepdim=True), "mean_" + name, None, True)
    return grids


def _leg(args):
    import torch
    from gangealing_b200.training import visuals as V
    tr, z, big_z, reals, loader = _setup(args.k, args.n_mean, args.real_batch)
    kw = dict(n_mean=args.n_mean, n_sample=args.n_sample, vis_batch_size=args.vis_batch_size)

    def port():
        grids = V.training_visuals(tr, z, big_z if args.k > 1 else None, reals, loader, **kw)
        return {n: g.cpu() for n, g in grids.items()}

    def reference():
        with torch.no_grad():
            return _reference_round(tr, z, big_z, reals, loader, **kw)

    fn = port if args.leg == "port" else reference
    fn()                                                 # warm-up round: modules, cuDNN algorithms
    torch.cuda.synchronize()
    times = []
    for _ in range(args.rounds):
        t0 = time.perf_counter()
        grids = fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    print(json.dumps({"k": args.k, "leg": args.leg, "seconds": times, "grids": len(grids),
                      "peak_host_mb": resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024.0}))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--heads", type=int, nargs="+", default=[1, 4])
    p.add_argument("--n-mean", type=int, default=8000)
    p.add_argument("--n-sample", type=int, default=64)
    p.add_argument("--vis-batch-size", type=int, default=250)
    p.add_argument("--real-batch", type=int, default=50)
    p.add_argument("--rounds", type=int, default=2)
    p.add_argument("--out", default=None)
    p.add_argument("--leg", choices=["port", "reference"], default=None)
    p.add_argument("--k", type=int, default=1)
    args = p.parse_args()
    if args.leg:
        return _leg(args)
    out = args.out or tempfile.mkdtemp(prefix="trainvisbench_")
    os.makedirs(out, exist_ok=True)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    results = []
    for k in args.heads:
        for leg in ("port", "reference"):
            cmd = [sys.executable, os.path.abspath(__file__), "--leg", leg, "--k", str(k), "--n-mean", str(args.n_mean),
                   "--n-sample", str(args.n_sample), "--vis-batch-size", str(args.vis_batch_size),
                   "--real-batch", str(args.real_batch), "--rounds", str(args.rounds)]
            res = subprocess.run(cmd, capture_output=True, text=True, cwd=out)
            line = [l for l in res.stdout.splitlines() if l.startswith("{")]
            if res.returncode != 0 or not line:
                raise RuntimeError("leg %s K=%d failed:\n%s" % (leg, k, res.stderr[-3000:]))
            r = json.loads(line[-1])
            r["card"] = card
            results.append(r)
            print(json.dumps(r), flush=True)
    with open(os.path.join(out, "trainvisbench.json"), "w") as fh:
        json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
