"""Time PCK-Transfer evaluation on the GPU: the single-forward batch core (eager and replayed from a CUDA graph) against
the reference's composition -- match_flows, then transfer_points once per direction -- on this repository's cuda_ops()
mirror (oracle.pck.pck_transfer_ref).  N = 50 pairs (the reference's evaluation batch), S = 256, F = 128,
P in {15, 30} (CUB, SPair), iters in {1, 3}, seeded weights and images.

    python tools/evalbench.py [--reps 20] [--warmup 3]

Prints the card and its power limit, then per configuration: ms per batch, pairs/s, STN forwards per batch and C-ABI
launches per batch.  Needs a CUDA device.
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gangealing_b200 import _lib  # noqa: E402
from gangealing_b200.evaluation import pck_transfer_batch  # noqa: E402
from gangealing_b200.stn import get_stn  # noqa: E402
from oracle import opset  # noqa: E402
from oracle import pck as OP  # noqa: E402


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # the timing does not depend on it
        q = "nvidia-smi unavailable (%s)" % exc
    return q or torch.cuda.get_device_name()


def _time(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("evalbench: needs a CUDA device")
    dev = "cuda"
    print("card: %s" % _card())
    n, s, f = 50, 256, 128
    t = opset.fill_parameters(get_stn(["similarity", "flow"], flow_size=f, supersize=s, channel_multiplier=0.5).eval(), 51,
                              gain=0.6).to(dev)
    seen = [0]
    sim_forward = t.stns[0].forward

    def counting_forward(input_img, *a, **k):   # an instance attribute: also counts congeal_points' direct self.forward
        seen[0] += input_img.size(0)
        return sim_forward(input_img, *a, **k)
    t.stns[0].forward = counting_forward
    alphas_l = [0.1, 0.05, 0.01]
    alphas = torch.tensor(alphas_l, device=dev)
    g = torch.Generator().manual_seed(0)
    for p in (15, 30):
        for iters in (1, 3):
            imgsA = torch.randn(n, 3, s, s, generator=g).to(dev)
            imgsB = torch.randn(n, 3, s, s, generator=g).to(dev)
            kpsA = (torch.rand(n, p, 2, generator=g) * (s - 9) + 4).to(dev)
            kpsB = (torch.rand(n, p, 2, generator=g) * (s - 9) + 4).to(dev)
            perm = torch.randperm(p, generator=g).to(dev)
            kw = dict(iters=iters, padding_mode="border")
            batch = dict(imgsA=imgsA, imgsB=imgsB, kpsA=kpsA, kpsB=kpsB)
            core = lambda: pck_transfer_batch(t, imgsA, imgsB, kpsA, kpsB, alphas, permutation=perm, **kw)
            ref = lambda: OP.pck_transfer_ref(t, iter([batch]), alphas_l, num_pairs=n, device=dev, permutation=perm, **kw)
            with torch.no_grad():
                rows = []
                for label, fn in (("reference composition (8N)", ref), ("pck_transfer_batch eager", core)):
                    fn()
                    seen[0], calls = 0, _lib.CALLS
                    fn()
                    fwd, launches = seen[0], _lib.CALLS - calls
                    ms = _time(fn, args.reps, args.warmup)
                    rows.append((label, ms, fwd, launches))
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    core()
                side.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph, stream=side):
                    core()
                rows.append(("pck_transfer_batch graph replay", _time(graph.replay, args.reps, args.warmup), rows[1][2], rows[1][3]))
            print("N=%d S=%d F=%d P=%d iters=%d" % (n, s, f, p, iters))
            for label, ms, fwd, launches in rows:
                print("  %-34s %8.2f ms/batch %9.0f pairs/s   STN forwards %4d   C-ABI launches %4d  (%.2fx)"
                      % (label, ms, n * 1000.0 / ms, fwd, launches, rows[0][1] / ms))


if __name__ == "__main__":
    main()
