"""Time dataset congealing on the GPU: congeal_images against the reference's composition on this repository's
cuda_ops() (per image: PIL's border_pad twice on the host, the fp32 padded squares uploaded, determine_flips, the
similarity stage and four .item() reads), and the letterbox kernel on its own.

    python tools/congealbench.py [--images 64] [--batch 32] [--runs 7]

Seeded similarity -> flow STN (flow 128, channel multiplier 0.5, the fixture's head re-centring) and seeded uint8 images
whose sides are drawn from 200-1500 px; output resolution 256.  Reports images/s end to end for both paths: after a
warm-up pass of each, --runs timed passes over all images alternate between the two paths (a host clock around each pass,
which ends in a device synchronise), and the median, minimum and maximum per path are printed; the spread between runs
comes from the shared host (PIL, packing, launch latency) as much as from the GPU.  Also the letterbox kernel's time per batch with the
bytes it must move (uint8 pixels read once, fp32 squares written once) over that time.  Needs a CUDA device.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gangealing_b200.evaluation import congeal_images, determine_flips  # noqa: E402
from gangealing_b200.op.letterbox import letterbox  # noqa: E402
from gangealing_b200.opset import cuda_ops  # noqa: E402
from gangealing_b200.stn import get_stn  # noqa: E402
from oracle import congeal as OC  # noqa: E402
from oracle import make_golden_congeal as GC  # noqa: E402
from oracle import opset  # noqa: E402

FLOW, OUT_RES, MIN_RES = 128, 256, 192


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # the timing does not depend on it
        q = "nvidia-smi unavailable (%s)" % exc
    return q or torch.cuda.get_device_name()


def _images(n, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        h, w = (int(v) for v in rng.integers(200, 1501, 2))
        low = rng.integers(0, 256, (h // 8 + 1, w // 8 + 1, 3), dtype=np.uint8)
        out.append(np.ascontiguousarray(np.repeat(np.repeat(low, 8, 0), 8, 1)[:h, :w]))   # blocky, any content works
    return out


def _reference(t, images):
    """congeal_dataset.py:35-61 on cuda_ops, image by image."""
    from PIL import Image
    t_sim = t.stns[0]
    one_hot = torch.tensor([[[0, 0, 1]]], dtype=torch.float, device="cuda")
    kept = []
    for img in images:
        x = Image.fromarray(img)
        w, h = x.size
        x_big = OC.prepro(OC.border_pad(x, max(w, h), resize=False)).cuda()
        x_in = OC.prepro(OC.border_pad(x, FLOW)).cuda()
        x_in, flip, _ = determine_flips(t, None, x_in)
        x_big = torch.where(flip.view(-1, 1, 1, 1), x_big.flip(3), x_big)
        bounds = torch.tensor([[h, w]], dtype=torch.float, device="cuda")
        aligned, M, oob = t_sim(x_in, return_flow=True, return_out_of_bounds=True, input_img_for_sampling=x_big,
                                output_resolution=OUT_RES, image_bounds=bounds)
        scale = torch.det(torch.cat([M, one_hot], 1)).sqrt_()
        if not (scale.item() * min(w, h) < MIN_RES or oob.item()):
            kept.append(aligned.clamp(-1, 1).add(1).div(2).mul(255).add_(0.5).clamp_(0, 255).permute(0, 2, 3, 1)
                        .to("cpu", torch.uint8))
    return kept


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--runs", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("congealbench needs a CUDA device")
    t = opset.fill_parameters(get_stn(["similarity", "flow"], flow_size=FLOW, supersize=FLOW, channel_multiplier=0.5,
                                      ops=cuda_ops()).eval(), GC.WEIGHT_SEED, gain=GC.WEIGHT_GAIN).cuda()
    images = _images(args.images)
    with torch.no_grad():
        GC.set_head(t, *GC.tune_head(t, letterbox(images[:16], FLOW)))

    def ours():
        for s in range(0, len(images), args.batch):
            congeal_images(t, images[s:s + args.batch], OUT_RES, MIN_RES, FLOW)["aligned"].cpu()

    def ref():
        _reference(t, images)

    res = {"card": _card(), "images": len(images), "batch": args.batch, "runs": args.runs}
    paths = (("congeal_images", ours), ("reference_composition", ref))
    rates = {name: [] for name, _ in paths}
    with torch.no_grad():
        for _, fn in paths:
            fn()
        for _ in range(args.runs):
            for name, fn in paths:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                rates[name].append(len(images) / (time.perf_counter() - t0))
        for name, r in rates.items():
            res[name + "_images_per_s"] = {"median": round(float(np.median(r)), 2), "min": round(min(r), 2),
                                           "max": round(max(r), 2)}
        res["speedup_median"] = round(float(np.median(rates["congeal_images"]) / np.median(rates["reference_composition"])), 2)
        batch = images[:args.batch]
        for name, size, resize in (("letterbox_flow", FLOW, True), ("letterbox_native", None, False)):
            imgs = batch if resize else [batch[0]]
            s = size or max(imgs[0].shape[:2])
            out = letterbox(imgs, s, resize)
            torch.cuda.synchronize()
            # the kernels alone, from a profiler run of their own
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(10):
                    letterbox(imgs, s, resize)
                torch.cuda.synchronize()
            us = sum(e.device_time_total for e in prof.key_averages() if "letterbox" in e.key) / 10
            nbytes = sum(x.size for x in imgs) + out.numel() * 4
            res[name + "_kernel_us"] = round(us, 1)
            res[name + "_GBps"] = round(nbytes / (us * 1e-6) / 1e9, 1) if us > 0 else None
            res[name + "_images"] = len(imgs)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
