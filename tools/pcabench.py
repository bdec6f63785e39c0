"""Time the latent learner's initialisation on the GPU (Trainer.init_target_mode, reference train.py:228-243).

    python tools/pcabench.py [--n 1000000] [--n-kmeans 50000] [--reps 10] [--no-sklearn]

On n seeded latents of the config-2 generator's mapping network (512 wide) it reports:
  * the `batch_gram` kernels (csrc/pca.cu) with CUDA events: ms, the FLOP rate of the fp64 tensor-core MMAs they issue
    (upper-triangle tiles only) against the data-sheet H100 SXM FP64 tensor peak (67 TFLOP/s), the bytes they must move
    (the latents once, the Grams and means written once) against 3.35 TB/s, and which of the two bounds the kernel;
  * the chain of float64 eigensolves that consumes the Grams (PCA with the Grams precomputed), for ndirs 1 and 5;
  * end-to-end init_target_mode for config 2 (ndirs 1) and config 5 (K 4, ndirs 5, inject 6; k-means++ over n_kmeans);
  * sklearn's IncrementalPCA(1).fit on the host cores on the same latents, or "not available".
Prints the card and its power limit first.  Needs a CUDA device.
"""
import argparse
import os
import subprocess
import sys
import time
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gangealing_b200.op.pca import batch_gram  # noqa: E402
from gangealing_b200.training import TrainConfig, Trainer  # noqa: E402
from gangealing_b200.training.latent_learner import PCA, gen_batches  # noqa: E402

FP64_TENSOR_PEAK = 67e12      # H100 SXM data sheet, dense FP64 tensor core
HBM_PEAK = 3.35e12            # H100 SXM data sheet, HBM3


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # the timing does not depend on it
        q = "nvidia-smi unavailable (%s)" % exc
    return q or torch.cuda.get_device_name()


def _events(fn, reps, warmup=2):
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


def _wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--n-kmeans", type=int, default=50_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--no-sklearn", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pcabench: needs a CUDA device")
    dev = "cuda"
    print("card: %s" % _card())
    tr2 = Trainer(TrainConfig(), dev)
    torch.manual_seed(0)
    with torch.no_grad():
        w = torch.cat([tr2.generator.batch_latent(min(100_000, args.n - i)) for i in range(0, args.n, 100_000)])
    n, d = w.shape

    # 1. the batch_gram kernels
    off = gen_batches(n, 5 * d, 5)
    sizes = [b - a for a, b in zip(off[:-1], off[1:])]
    t_tiles = d // 64
    flops = sum(2.0 * s * 64 * 64 * t_tiles * (t_tiles + 1) / 2 for s in sizes)   # 2 FLOP per product, upper tiles
    nbytes = n * d * 4 + len(sizes) * (d * d + d) * 8
    ms = _events(lambda: batch_gram(w, off), args.reps)
    t_flop, t_byte = flops / FP64_TENSOR_PEAK, nbytes / HBM_PEAK
    bound = "FP64 tensor" if t_flop >= t_byte else "HBM"
    print("batch_gram   n=%d D=%d blocks=%d: %.3f ms  %.1f TFLOP/s (%.0f%% of 67)  %.2f TB/s (%.0f%% of 3.35)  "
          "%s-bound: %.0f%% of the bound's minimum time"
          % (n, d, len(sizes), ms, flops / ms / 1e9, 100 * flops / ms / 1e9 / 67, nbytes / ms / 1e9,
             100 * nbytes / ms / 1e9 / 3.35, bound, 100 * max(t_flop, t_byte) * 1e3 / ms))

    # 2. the eigensolve chain alone (Grams precomputed)
    gram, mean = batch_gram(w, off)
    pre = types.SimpleNamespace(batch_gram=lambda *_: (gram, mean))
    for k in (1, 5):
        PCA(k, w, ops=pre)
        ms_chain, _ = _wall(lambda: PCA(k, w, ops=pre))
        ms_pca, _ = _wall(lambda: PCA(k, w))
        print("eigensolve chain ndirs=%d: %d float64 %dx%d eigh: %.1f ms (%.2f ms each); whole PCA %.1f ms"
              % (k, len(sizes), d, d, ms_chain, ms_chain / len(sizes), ms_pca))
    del gram, mean

    # 3. end to end
    for name, cfg, kw in (("config 2", TrainConfig(), {}),
                          ("config 5", TrainConfig(num_heads=4, ndirs=5, inject=6), {"n_kmeans": args.n_kmeans})):
        tr = tr2 if name == "config 2" else Trainer(cfg, dev)
        ms_init, _ = _wall(lambda: tr.init_target_mode(n_pca=args.n, **kw))
        extra = " (k-means++ over %d latents)" % args.n_kmeans if kw else ""
        print("init_target_mode %s n_pca=%d%s: %.1f ms" % (name, args.n, extra, ms_init))
        del tr
        torch.cuda.empty_cache()

    # 4. sklearn on the host cores
    if args.no_sklearn:
        print("sklearn IncrementalPCA: skipped")
        return
    try:
        from sklearn.decomposition import IncrementalPCA
    except ImportError:
        print("sklearn IncrementalPCA: not available")
        return
    x = w.cpu().numpy()
    t = time.perf_counter()
    IncrementalPCA(1).fit(x)
    print("sklearn IncrementalPCA(1).fit on %d host cores: %.1f s" % (os.cpu_count(), time.perf_counter() - t))


if __name__ == "__main__":
    main()
