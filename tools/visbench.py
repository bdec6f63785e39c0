"""Time the congealing visualisations on the GPU against the reference's per-frame formulation on this repository's
cuda_ops() mirror.  Seeded weights (flow 128, channel multiplier 0.5) and images.

    python tools/visbench.py [--frames-window 4] [--n-mean 1000]

Average-image animation, 512^2 source and output, two STN stages x 240 frames, batches of 50:
  * the reference formulation (create_average_image: flip inference + STN + lerp + warp + sum, again for every frame), per
    frame and per batch of 50, timed over a window of frames (a per-frame figure, not a total);
  * congealing_average_frames end to end at n_mean images;
  * the mean kernel (gg_mipmap_warp_lerp_mean) per (sample, frame), with its DRAM bytes.
Point tracking, N = 4, P = 40000, patch 9, 512^2 grids, 240 frames: track_points_lerp against the per-frame Unfold
composition (oracle.vis.nearest_neighbor_within_patch on the device).
Label propagation, N = 4, 512^2, 2 x 240 frames, a 256^2 label (65 536 points) at sigma 1.2: splat_composite_grid over all
480 frames against the reference formulation (visualize_label_propagation: chunks of 100 (frame, image) pairs, two
splat2d, the composite, .cpu(), then images2grid per frame on the host), timed over --label-chunks chunks and given per
frame.  --labels-only runs this section alone.
--propagate runs only the edits-on-real-images comparison at 512^2, sigma 1.3, for N = 9 (the script's usual
--dset_indices count) and N = 50 images and labels of P = 25 233 and 403 533 points (BASELINE config 4): the reference
composition on the mirror (determine_flips, t(flipped), uncongeal_points, the x mirror, splat_points, then make_grid and the
uint8 cast of each grid on the host) against propagate_to_images, in ms per batch, with the STN forwards (images through
the flow STN) and C-ABI launches of each.  Needs a CUDA device.
"""
import argparse
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gangealing_b200.evaluation import congealing_average_frames  # noqa: E402
from gangealing_b200.evaluation import visuals as V  # noqa: E402
from gangealing_b200.stn import get_stn  # noqa: E402
from gangealing_b200.stn.sampling import MipmapWarp, mipmap_warp_lerp_mean  # noqa: E402
from gangealing_b200.splat2d import splat2d, splat_composite_grid, track_points_lerp  # noqa: E402
from oracle import opset  # noqa: E402
from oracle import vis as OV  # noqa: E402


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # the timing does not depend on it
        q = "nvidia-smi unavailable (%s)" % exc
    return q or torch.cuda.get_device_name()


def _events(fn, reps=1):
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / reps


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames-window", type=int, default=4)
    ap.add_argument("--n-mean", type=int, default=1000)
    ap.add_argument("--label-chunks", type=int, default=2)
    ap.add_argument("--labels-only", action="store_true")
    ap.add_argument("--propagate", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("visbench: needs a CUDA device")
    print("card: %s" % _card())
    if args.propagate:
        propagate()
        return
    label_propagation(args.label_chunks)
    if not args.labels_only:
        congealing(args)


def propagate():
    """propagate_to_images against the reference's make_visuals composition on the mirror."""
    from torchvision.utils import make_grid
    from gangealing_b200 import _lib
    from gangealing_b200.evaluation import propagate_to_images
    from gangealing_b200.evaluation.propagate import label_queries
    dev, res, sigma, opacity = "cuda", 512, 1.3, 0.75
    t = opset.fill_parameters(get_stn(["similarity", "flow"], flow_size=128, supersize=res, channel_multiplier=0.5).eval(),
                              51, gain=0.6).to(dev)
    ops = t.ops
    seen = [0]
    t.stns[-1].register_forward_hook(lambda m, inp, out: seen.__setitem__(0, seen[0] + inp[0].size(0)))
    g = torch.Generator().manual_seed(0)

    def host_grid(x, nrow):
        grid = make_grid(x.cpu(), nrow=nrow, padding=3, pad_value=-1.0, normalize=True, value_range=(-1, 1))
        return grid.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to(torch.uint8)

    for n in (9, 50):
        images = torch.nn.functional.interpolate(torch.randn(n, 3, 32, 32, generator=g), size=(res, res), mode="bilinear",
                                                 align_corners=False).to(dev)
        nrow = int(n ** 0.5)
        for p in (25233, 403533):
            side = int(p ** 0.5) + 1    # the label: P pixels of a side x side image at resolution = side
            idx = torch.randperm(side * side, generator=g)[:p].sort().values
            label = torch.stack([idx % side, idx // side], -1)
            colors = (torch.rand(1, p, 3, generator=g) * 2 - 1).to(dev)
            alpha = torch.rand(1, p, 1, generator=g).to(dev)

            def reference():
                flipped, flips, policy = V.determine_flips(t, None, images)
                congealed = t(flipped, warp_policy=policy, output_resolution=res)
                queries, _ = label_queries(label.to(dev), side, res)
                pts = t.uncongeal_points(flipped, queries.expand(n, p, 2), warp_policy=policy)
                pts[:, :, 0] = torch.where(flips.view(-1, 1), res - 1 - pts[:, :, 0], pts[:, :, 0])
                out = V._splat_points(ops, images, pts, colors, alpha, sigma, opacity)
                return [host_grid(x, nrow) for x in (images, congealed, out)]

            def fused():
                r = propagate_to_images(t, images, label, colors, alpha, sigma, opacity, resolution=side)
                return [r["input_images"], r["congealed_images"], r["propagated"]]

            row = []
            for name, fn in (("reference", reference), ("propagate_to_images", fused)):
                fn()
                seen[0], calls = 0, _lib.CALLS
                fn()
                torch.cuda.synchronize()
                fwd, launches = seen[0], _lib.CALLS - calls
                start = time.perf_counter()
                for _ in range(3):
                    fn()
                torch.cuda.synchronize()
                row.append((name, (time.perf_counter() - start) / 3 * 1e3, fwd, launches))
            print("propagate N %d, P %d, %d^2: " % (n, p, res) + "; ".join(
                "%s %.1f ms per batch, %d STN images, %d C-ABI calls" % r for r in row) +
                  "; speed-up %.2fx" % (row[0][1] / row[1][1]))


def label_propagation(chunks):
    """visualize_label_propagation's splat + grid loop against splat_composite_grid."""
    from torchvision.utils import make_grid
    dev, n, res, frames, side, batch = "cuda", 4, 512, 480, 256, 100
    g = torch.Generator().manual_seed(1)
    images = (torch.rand(frames, n, 3, res, res, generator=g) * 2 - 1).to(dev)
    ys, xs = torch.meshgrid(torch.arange(side), torch.arange(side), indexing="ij")
    label = (torch.stack([xs.flatten(), ys.flatten()], -1).float() * ((res - 1) / (side - 1))).to(dev)
    drift = torch.randn(frames, n, 1, 2, generator=g).to(dev) * 20
    points = (label.view(1, 1, -1, 2) + drift).contiguous()
    p = label.size(0)
    colors = (torch.rand(1, p, 3, generator=g) * 2 - 1).to(dev)
    alpha = torch.rand(1, p, 1, generator=g).to(dev)
    splat_composite_grid(images[:2], points[:2], colors, alpha, 1.2, 0.7, 2)
    fused = _events(lambda: splat_composite_grid(images, points, colors, alpha, 1.2, 0.7, 2))
    print("splat_composite_grid: N %d, %d^2, %d frames, %d points: %.1f ms per call = %.3f ms per frame" %
          (n, res, frames, p, fused, fused / frames))

    flat_images, flat_points = images.view(-1, 3, res, res), points.view(-1, p, 2)
    col, al = colors.repeat(batch, 1, 1), alpha.repeat(batch, 1, 1)
    sig = torch.full((batch,), 1.2, device=dev)

    def reference(c):
        sl = slice(c * batch, (c + 1) * batch)
        obj = splat2d(torch.zeros(batch, 3, res, res, device=dev), flat_points[sl], col, sig, False)
        mask = splat2d(torch.zeros(batch, 1, res, res, device=dev), flat_points[sl], al, sig, True) * 0.7
        out = (mask * obj + (1 - mask) * flat_images[sl]).cpu().view(-1, n, 3, res, res)
        return [make_grid(f, nrow=2, normalize=True, value_range=(-1, 1)).mul(255).add_(0.5).clamp_(0, 255)
                .permute(1, 2, 0).to("cpu", torch.uint8).numpy() for f in out]

    reference(0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for c in range(chunks):
        reference(c)
    ref = (time.perf_counter() - t0) * 1e3 / (chunks * batch // n)
    print("reference formulation (chunks of %d pairs: 2 splat2d + composite + .cpu() + images2grid per frame): %.2f ms per "
          "frame (%d chunks); fused %.1fx" % (batch, ref, chunks, ref / (fused / frames)))


def congealing(args):
    dev = "cuda"
    res, batch, length = 512, 50, 240
    t = opset.fill_parameters(get_stn(["similarity", "flow"], flow_size=128, supersize=res, channel_multiplier=0.5).eval(),
                              51, gain=0.6).to(dev)
    g = torch.Generator().manual_seed(0)
    data = torch.randn(batch, 3, res, res, generator=g).to(dev)

    # the reference formulation: every frame re-runs the flips and the STN over the batch, then lerps, warps and sums
    identity = V._identity(1, res, data)
    warper = MipmapWarp(3.5)
    alphas = V.cosine_alphas(length, dev)

    def ref_frame(i):
        flipped, flips, policy = V.determine_flips(t, None, data)
        _, grids = t(flipped, warp_policy=policy, return_intermediates=True)
        grid = V._resize(V.flip_grid(grids[1], flips), res)
        base = V._resize(V.flip_grid(grids[0], flips), res)
        return warper(data, base.lerp(grid, alphas[i])).sum(dim=0, keepdim=True)

    ref_frame(0)
    w = args.frames_window
    ms = _events(lambda: [ref_frame(i) for i in range(w)]) / w
    print("reference formulation (per-frame flips + STN + warp + sum), batch %d at %d^2: %.1f ms per frame per batch "
          "(window of %d frames)" % (batch, res, ms, w))

    # end to end
    n_batches = args.n_mean // batch
    batches = [torch.randn(batch, 3, res, res, generator=g).to(dev) for _ in range(min(n_batches, 4))]
    loader = [batches[i % len(batches)] for i in range(n_batches)]
    congealing_average_frames(t, loader[:1], batch, length=4, vis_in_stages=True, output_resolution=res)   # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    frames = congealing_average_frames(t, loader, args.n_mean, length=length, vis_in_stages=True, output_resolution=res)
    torch.cuda.synchronize()
    e2e = time.perf_counter() - t0
    print("congealing_average_frames: n_mean %d, 2 stages x %d frames at %d^2: %.2f s end to end (%s)" %
          (args.n_mean, length, res, e2e, tuple(frames.shape)))
    del frames

    # the mean kernel alone: one stage of one batch
    flipped, flips, policy = V.determine_flips(t, None, data)
    _, grids = t(flipped, warp_policy=policy, return_intermediates=True)
    target = V._resize(V.flip_grid(grids[1], flips), res)
    base = V._resize(V.flip_grid(grids[0], flips), res)
    acc = torch.zeros(length, 3, res, res, device=dev)
    mipmap_warp_lerp_mean(data, base, target, alphas, acc, 3.5)
    kms = _events(lambda: mipmap_warp_lerp_mean(data, base, target, alphas, acc, 3.5), 3)
    per = kms * 1e3 / (batch * length)
    dram = 4 * (batch * 3 * res * res * 4 / 3 + 2 * batch * res * res * 2 + 2 * length * 3 * res * res)   # src + pyramid, grids, acc
    print("mean kernel: %.2f ms per call (%d samples x %d frames) = %.2f us per (sample, frame); DRAM bytes %.2f GB -> "
          "%.0f GB/s (%.1f%% of 3.35 TB/s): bound by the per-pixel gathers (L1/L2), not DRAM" %
          (kms, batch, length, per, dram / 1e9, dram / kms / 1e6, 100 * dram / kms / 1e6 / 3350))

    # point tracking
    n, p, ps = 4, 40000, 9
    tb, tt = base[:n].contiguous(), target[:n].contiguous()
    pts = torch.rand(n, p, 2, generator=g).to(dev) * 1.6 - 0.8
    centers = torch.randint(0, res, (n, p, 2), generator=g).to(dev)
    track_points_lerp(tb, tt, alphas, pts, centers, ps)
    kt = _events(lambda: track_points_lerp(tb, tt, alphas, pts, centers, ps), 3)
    c = centers

    def unfold_frames():
        nonlocal c
        for i in range(w):
            c = OV.nearest_neighbor_within_patch(tb.lerp(tt, alphas[i]), pts, c, ps)

    unfold_frames()
    uf = _events(unfold_frames) / w
    print("tracker: N %d, P %d, patch %d, %d^2, %d frames: %.2f ms per launch (%.3f ms per frame); per-frame Unfold "
          "composition %.2f ms per frame (window of %d frames)" % (n, p, ps, res, length, kt, kt / length, uf, w))


if __name__ == "__main__":
    main()
