"""Per-op microbenchmark on one H100: achieved algorithmic GB/s of each hot-path kernel at the
BASELINE config-2 shapes (per-GPU batch B), CUDA-event timed, inputs rotated through a pool larger than L2.
Usage: python tools/opbench.py [--batch 5] [--json out.json]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gangealing_b200 import op  # noqa: E402
from gangealing_b200.op.fused_act import bias_act_backward_raw  # noqa: E402


def peak_gbs():
    return 3350.0, "H100 SXM data sheet"


GRAPH = False   # --graph: time a captured CUDA graph of `iters` calls (device time only; no Python / launch overhead)


def timeit(fn, pools, iters=20, warmup=3):
    """fn(i) runs on input set i (rotating) -> ms per call (mean over iters).  With --graph the `iters` calls are captured
    into ONE CUDA graph and the replay is timed: what a kernel costs inside the captured training step (both this repo's
    ops and the reference's pybind kernels launch on the current stream, so both capture)."""
    for i in range(warmup):
        fn(i % pools)
    torch.cuda.synchronize()
    st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if GRAPH:
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for i in range(iters):
                fn(i % pools)
        graph.replay()
        torch.cuda.synchronize()
        st.record()
        graph.replay()
        en.record()
        torch.cuda.synchronize()
        del graph
        return st.elapsed_time(en) / iters
    st.record()
    for i in range(iters):
        fn(i % pools)
    en.record()
    torch.cuda.synchronize()
    return st.elapsed_time(en) / iters


def nhwc_family(B, dev, k4, timeit, report, pool_count):
    """The channels-last kernels (csrc/nhwc.cu) at the generator's shapes."""
    from gangealing_b200.op.modconv import channel_scale_raw, _ToRGB
    CL = torch.channels_last
    for C, H in [(128, 256), (256, 128), (512, 64), (512, 32), (512, 16), (512, 8)]:
        hin = H + 1
        nbytes = 4 * B * C * (hin * hin + H * H)
        P = pool_count(nbytes)
        xs = [torch.randn(B, C, hin, hin, device=dev).contiguous(memory_format=CL) for _ in range(P)]
        noise = torch.randn(B, 1, H, H, device=dev)
        nw = torch.tensor([0.1], device=dev)
        bias = torch.randn(C, device=dev)
        rs = torch.rand(B, C, device=dev) + 0.5
        ms = timeit(lambda i: op.upfirdn2d(xs[i], k4, pad=(1, 1)), P)
        report("nhwc blur C=%d %d->%d" % (C, hin, H), nbytes, ms)
        ms = timeit(lambda i: op.blur_noise_bias_act(xs[i], k4, (1, 1), noise, nw, bias, row_scale=rs), P)
        report("nhwc fused blur+noise+bias+act C=%d %d->%d" % (C, hin, H), nbytes + 4 * B * H * H, ms)
        del xs
        ys = [torch.randn(B, C, H, H, device=dev).contiguous(memory_format=CL) for _ in range(P)]
        nb2 = 4 * B * C * H * H * 2
        ms = timeit(lambda i: op.noise_bias_act(ys[i], noise, nw, bias, row_scale=rs), P)
        report("nhwc noise+bias+act C=%d %d^2" % (C, H), nb2 + 4 * B * H * H, ms)
        ms = timeit(lambda i: bias_act_backward_raw(ys[i], ys[(i + 1) % P], 0.2, 1.4, True), P)
        report("nhwc bias_act backward(+bias grad) C=%d %d^2" % (C, H), 4 * B * C * H * H * 3, ms)
        ms = timeit(lambda i: channel_scale_raw(ys[i], rs), P)
        report("nhwc channel_scale C=%d %d^2" % (C, H), nb2, ms)
        ms = timeit(lambda i: channel_scale_raw(ys[i], rs, y=ys[(i + 1) % P]), P)
        report("nhwc channel_scale + row_dot C=%d %d^2" % (C, H), 4 * B * C * H * H * 3, ms)
        wm = torch.randn(B, 3, C, device=dev)
        b3 = torch.randn(1, 3, 1, 1, device=dev)
        skip = torch.randn(B, 3, H, H, device=dev)
        ms = timeit(lambda i: _ToRGB.apply(ys[i], wm, b3, skip), P)
        report("nhwc to_rgb forward C=%d %d^2" % (C, H), 4 * B * H * H * (C + 6), ms)
        g3 = torch.randn(B, 3, H, H, device=dev)
        lib = __import__("gangealing_b200._lib", fromlist=["x"])
        gx = torch.empty_like(ys[0]); gw = torch.empty(B, 3, C, device=dev)
        ws = torch.empty(max(1, lib.load().gg_to_rgb_nhwc_workspace(B, C, H * H) // 4), device=dev)
        ms = timeit(lambda i: lib.check(lib.load().gg_to_rgb_nhwc_backward(gx.data_ptr(), gw.data_ptr(), ws.data_ptr(), g3.data_ptr(),
                    ys[i].data_ptr(), wm.data_ptr(), B, C, H * H, lib.stream()), "to_rgb bwd"), P)
        report("nhwc to_rgb backward C=%d %d^2" % (C, H), 4 * B * H * H * (2 * C + 3), ms)
        ms = timeit(lambda i: ys[(i + 1) % P].copy_(ys[i]), P)
        report("  torch copy_ (roofline probe) C=%d %d^2" % (C, H), nb2, ms)
        del ys


def reference_bar(B, dev, k4, timeit, pool_count, peak, json_path):
    """The kernel bar (BASELINE.md section 3 / SURVEY.md 8d): the reference's own CUDA kernels recompiled for sm_90a
    (oracle/_ref/*.so: upfirdn2d_kernel.cu:209-369, fused_bias_act_kernel.cu:52-99, splat_gpu_impl.cu:41-96) timed at the
    hot-path shapes on this GPU, next to this repo's kernels on the same inputs.  tools/ is test infrastructure."""
    from oracle import build_ref
    from gangealing_b200.splat2d import splat2d
    up_ref, fused_ref, splat_ref = build_ref.load_ref("upfirdn2d_ref"), build_ref.load_ref("fused_ref"), build_ref.load_splat_ref()
    if up_ref is None or fused_ref is None:
        raise SystemExit("oracle/_ref/*.so not built (python -m oracle.build_ref in the build container)")
    CL = torch.channels_last
    rows = []

    def add(name, nbytes, ms_ref, ms_nchw, ms_nhwc):
        row = {"op": name, "MB": nbytes / 1e6, "reference_ms": ms_ref, "ours_nchw_ms": ms_nchw, "ours_nhwc_ms": ms_nhwc,
               "reference_GBs": nbytes / ms_ref / 1e6,
               "ours_nchw_GBs": nbytes / ms_nchw / 1e6 if ms_nchw else None,
               "ours_nhwc_GBs": nbytes / ms_nhwc / 1e6 if ms_nhwc else None}
        best = min(m for m in (ms_nchw, ms_nhwc) if m)
        row["speedup_best"] = ms_ref / best
        row["ours_best_frac_of_peak"] = nbytes / best / 1e6 / peak
        rows.append(row)
        print("%-52s ref %8.3f ms | ours nchw %8s  nhwc %8s ms | x%5.2f  (%4.1f%% of peak)" % (
            name, ms_ref, "%.3f" % ms_nchw if ms_nchw else "-", "%.3f" % ms_nhwc if ms_nhwc else "-", row["speedup_best"],
            100 * row["ours_best_frac_of_peak"]))

    def ref_up(x, up=1, down=1, pad=(1, 1)):
        n, c, h, w = x.shape
        return up_ref.upfirdn2d(x.reshape(-1, h, w, 1), k4, up, up, down, down, pad[0], pad[1], pad[0], pad[1])

    only = os.environ.get("GG_OPBENCH_ONLY", "")      # e.g. "splat": just those rows (kernel experiments)
    for C, H in ([] if only else [(128, 256), (256, 128), (512, 64), (512, 32), (512, 16), (512, 8)]):
        hin = H + 1
        nbytes = 4 * B * C * (hin * hin + H * H)
        P = pool_count(nbytes)
        xs = [torch.randn(B, C, hin, hin, device=dev) for _ in range(P)]
        xl = [x.contiguous(memory_format=CL) for x in xs]
        noise = torch.randn(B, 1, H, H, device=dev)
        nw = torch.tensor([0.1], device=dev)
        bias = torch.randn(C, device=dev)
        empty = xs[0].new_empty(0)
        add("upfirdn2d blur C=%d %d->%d" % (C, hin, H), nbytes,
            timeit(lambda i: ref_up(xs[i]), P), timeit(lambda i: op.upfirdn2d(xs[i], k4, pad=(1, 1)), P),
            timeit(lambda i: op.upfirdn2d(xl[i], k4, pad=(1, 1)), P))

        def ref_tail(i):    # Blur -> NoiseInjection -> FusedLeakyReLU, networks.py:266,291-298,346-348
            t = ref_up(xs[i]).view(B, C, H, H)
            t = t + nw * noise
            return fused_ref.fused_bias_act(t, bias, empty, 3, 0, 0.2, 2 ** 0.5)
        add("StyledConv-up tail (blur+noise+bias+lrelu) C=%d %d" % (C, H), nbytes + 4 * B * H * H,
            timeit(ref_tail, P), timeit(lambda i: op.blur_noise_bias_act(xs[i], k4, (1, 1), noise, nw, bias), P),
            timeit(lambda i: op.blur_noise_bias_act(xl[i], k4, (1, 1), noise, nw, bias), P))
        del xs, xl
        ys = [torch.randn(B, C, H, H, device=dev) for _ in range(P)]
        yl = [y.contiguous(memory_format=CL) for y in ys]
        nb2 = 4 * B * C * H * H * 2
        add("fused_bias_act fwd C=%d %d^2" % (C, H), nb2,
            timeit(lambda i: fused_ref.fused_bias_act(ys[i], bias, empty, 3, 0, 0.2, 2 ** 0.5), P),
            timeit(lambda i: op.fused_leaky_relu(ys[i], bias), P), timeit(lambda i: op.fused_leaky_relu(yl[i], bias), P))

        def ref_plain_tail(i):
            return fused_ref.fused_bias_act(ys[i] + nw * noise, bias, empty, 3, 0, 0.2, 2 ** 0.5)
        add("StyledConv tail (noise+bias+lrelu) C=%d %d^2" % (C, H), nb2 + 4 * B * H * H,
            timeit(ref_plain_tail, P), timeit(lambda i: op.noise_bias_act(ys[i], noise, nw, bias), P),
            timeit(lambda i: op.noise_bias_act(yl[i], noise, nw, bias), P))

        def ref_bwd(i):     # fused_act.py:29-38: act-grad kernel, then a second pass for the bias gradient
            gx = fused_ref.fused_bias_act(ys[i], empty, ys[(i + 1) % P], 3, 1, 0.2, 2 ** 0.5)
            return gx, gx.sum([0, 2, 3])
        add("fused_bias_act bwd (+bias grad) C=%d %d^2" % (C, H), 4 * B * C * H * H * 3,
            timeit(ref_bwd, P), timeit(lambda i: bias_act_backward_raw(ys[i], ys[(i + 1) % P], 0.2, 2 ** 0.5, True), P),
            timeit(lambda i: bias_act_backward_raw(yl[i], yl[(i + 1) % P], 0.2, 2 ** 0.5, True), P))
        del ys, yl
    for H in ([] if only else (128, 64)):
        x = torch.randn(B, 3, H, H, device=dev)
        add("upfirdn2d rgb up2 %d->%d" % (H, 2 * H), 4 * B * 3 * 5 * H * H,
            timeit(lambda i: ref_up(x, 2, 1, (2, 1)), 1), timeit(lambda i: op.upfirdn2d(x, k4, up=2, pad=(2, 1)), 1), None)
    for C, H, pad in ([] if only else [(64, 128, (2, 2)), (64, 128, (1, 1)), (128, 64, (2, 2)), (512, 32, (2, 2))]):
        x = [torch.randn(B, C, H, H, device=dev) for _ in range(4)]
        xl = [t.contiguous(memory_format=CL) for t in x]
        ho = H + 2 * pad[0] - 3
        add("upfirdn2d stn blur C=%d %d pad%s" % (C, H, pad), 4 * B * C * (H * H + ho * ho),
            timeit(lambda i: ref_up(x[i], 1, 1, pad), 4), timeit(lambda i: op.upfirdn2d(x[i], k4, pad=pad), 4),
            timeit(lambda i: op.upfirdn2d(xl[i], k4, pad=pad), 4))
    # splat2d, BASELINE config 4: a dense disc of P points into 512^2, sigma 0.3 / 1.3 (propagate_to_images.py:44-78)
    if splat_ref is not None:
        for R, sigma in [(256, 0.3), (256, 1.3), (1024, 0.3), (1024, 1.3)]:
            ys_, xs_ = torch.meshgrid(torch.arange(float(R)), torch.arange(float(R)), indexing="ij")
            disc = ((ys_ - R / 2) ** 2 + (xs_ - R / 2) ** 2) < (0.35 * R) ** 2
            pts = (torch.stack([xs_[disc], ys_[disc]], 1) * (511.0 / (R - 1)) + 0.25)[None].to(dev).contiguous()
            Pn = pts.shape[1]
            vals = torch.randn(1, Pn, 3, device=dev)
            sig = torch.tensor([sigma], device=dev)
            blank = torch.zeros(1, 3, 512, 512, device=dev)
            alpha = torch.zeros(1, 512, 512, device=dev)

            def ref_splat(i):   # splat_gpu.c:20-41 host sequence around the reference kernel
                alpha.zero_()
                acc = blank.clone()
                splat_ref.SplatForwardGpu(torch.cuda.current_stream().cuda_stream, pts.data_ptr(), vals.data_ptr(), sig.data_ptr(),
                                          alpha.data_ptr(), acc.data_ptr(), Pn, 3, 512, 512, Pn)
                return acc / (alpha.view(1, 1, 512, 512) + 1e-8)
            nbytes = 4 * (Pn * 5 + 4 * 512 * 512 + 2 * 3 * 512 * 512)
            add("splat2d 512^2 P=%d sigma=%.1f" % (Pn, sigma), nbytes, timeit(ref_splat, 1),
                timeit(lambda i: splat2d(blank, pts, vals, sig, False), 1), None)
    if json_path:
        os.makedirs(os.path.dirname(os.path.abspath(json_path)), exist_ok=True)
        json.dump({"batch": B, "dtype": "float32", "peak_gbs": peak,
                   "timing": "CUDA graph replay of 20 calls (device time)" if GRAPH else "eager calls (includes launch overhead)",
                   "what": "reference CUDA kernels (recompiled sm_90a) vs this repo, same inputs, CUDA events, >L2 input pools",
                   "rows": rows}, open(json_path, "w"), indent=1)


def stn_rows(B, dev, timeit, peak, json_path):
    """The STN's sampling path (SURVEY.md 8a rows a8-a10): reference sequence (its own MipmapWarp run from the byte-compiled
    oracle/_ref/refpy + F.affine_grid / the ATen flow composition of warping_heads.py) vs this repo's two-pass ops
    (flow_compose -> grid in HBM -> pyramid + warp) vs the ONE-pass sampler (grid generated inside the sampler).
    GB/s by the SURVEY.md 8(d) formula: 4*N*(C*Hs*Ws + C*Ho*Wo + 2*Hf*Wf + 6) (+ 4*N*2*Ho*Wo for the returned grid)."""
    import importlib.util
    import torch.nn.functional as F
    from oracle import build_ref
    from gangealing_b200.stn import sampling as S
    from gangealing_b200.stn.flow import flow_compose
    ref_cls = None
    pyc = os.path.join(build_ref.REFPY, "models", "spatial_transformers", "antialiased_sampling.pyc")
    if os.path.exists(pyc):
        spec = importlib.util.spec_from_file_location("ref_antialiased_sampling", pyc)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        ref_cls = mod.MipmapWarp
    rows = []
    g = torch.Generator(device=dev).manual_seed(0)
    for tag, hs, ho, kind in [("similarity 128->128", 128, 128, "sim"), ("flow 128->128", 128, 128, "flow"),
                              ("similarity 256->128 (sample_from_full_res)", 256, 128, "sim"),
                              ("flow 256->128 (sample_from_full_res)", 256, 128, "flow"),
                              ("flow 512->512 (config 4)", 512, 512, "flow")]:
        n = B if hs < 512 else max(1, B // 8)
        img = torch.rand(n, 3, hs, hs, device=dev, generator=g) * 2 - 1
        theta = torch.eye(2, 3, device=dev)[None].repeat(n, 1, 1) + 0.05 * torch.randn(n, 2, 3, device=dev, generator=g)
        s = 8
        lh = ho // s
        low = 0.02 * torch.randn(n, lh, lh, 2, device=dev, generator=g)
        mask = torch.randn(n, 9 * s * s, lh, lh, device=dev, generator=g)
        ident = F.affine_grid(torch.eye(2, 3, device=dev)[None], (1, 1, ho, ho), align_corners=False)
        alg = 4 * n * (3 * hs * hs + 3 * ho * ho + 2 * ho * ho + (2 * lh * lh + 9 * s * s * lh * lh if kind == "flow" else 0) + 6)
        ref_warp = ref_cls(max_num_levels=3.5).to(dev) if ref_cls is not None else None

        def ref_path(i):
            if kind == "sim":
                grid = F.affine_grid(theta, (n, 3, ho, ho), align_corners=False)
            else:   # warping_heads.py:180-193 (upsample_flow), :239-244, :268-277
                m = mask.view(n, 1, 9, s, s, lh, lh).softmax(dim=2)
                up = F.unfold(s * low.permute(0, 3, 1, 2), [3, 3], padding=1).view(n, 2, 9, 1, 1, lh, lh)
                delta = (m * up).sum(dim=2).permute(0, 1, 4, 2, 5, 3).reshape(n, 2, ho, ho).permute(0, 2, 3, 1)
                flow = ident + delta
                flat = flow.reshape(n, -1, 2)
                grid = (flat @ theta[:, :, :2].transpose(1, 2) + theta[:, None, :, 2]).reshape(n, ho, ho, 2)
            return ref_warp(img, grid, padding_mode="border")

        def two_pass(i):
            if kind == "sim":
                grid = F.affine_grid(theta, (n, 3, ho, ho), align_corners=False)
            else:
                grid = flow_compose(low, mask, ident, theta, None, s)[1]
            return S.mipmap_warp(img, grid, 3.5, 0.0, "border")[0]

        def one_pass(i):
            if kind == "sim":
                return S.stn_sample_affine(img, theta, (ho, ho), 3.5, 0.0, "border")[0]
            return S.stn_sample_flow(img, low, mask, ident, theta, None, s, 3.5, 0.0, "border")[0]
        ms_ref = timeit(ref_path, 1) if ref_warp is not None else None
        ms_two, ms_one = timeit(two_pass, 1), timeit(one_pass, 1)
        err = (one_pass(0) - two_pass(0)).abs().max().item()
        row = {"op": tag, "batch": n, "MB": alg / 1e6, "reference_ms": ms_ref, "two_pass_ms": ms_two, "one_pass_ms": ms_one,
               "one_pass_GBs": alg / ms_one / 1e6, "one_pass_frac_of_peak": alg / ms_one / 1e6 / peak,
               "speedup_vs_reference": (ms_ref / ms_one) if ms_ref else None, "one_vs_two_pass_max_abs_diff": err}
        rows.append(row)
        print("%-46s N=%-3d ref %s ms | two-pass %.3f | one-pass %.3f ms  %7.1f GB/s (%.1f%% of peak)  x%s vs ref" % (
            tag, n, "%.3f" % ms_ref if ms_ref else "   -  ", ms_two, ms_one, row["one_pass_GBs"], 100 * row["one_pass_frac_of_peak"],
            "%.1f" % row["speedup_vs_reference"] if ms_ref else "-"))
    if json_path:
        os.makedirs(os.path.dirname(os.path.abspath(json_path)), exist_ok=True)
        json.dump({"batch": B, "peak_gbs": peak, "what": "STN sampling path: reference MipmapWarp sequence vs two-pass vs one-pass",
                   "rows": rows}, open(json_path, "w"), indent=1)


FP32_PEAK_TFLOPS = 67.0   # H100 SXM data sheet, dense FP32 (700 W)


def blend_rows(dev, timeit, peak, json_path):
    """Laplacian pyramid blending (splat_points(blend_alg='laplacian*')): the reference's formulation (2-D depthwise
    convolution per level, materialised stacks; oracle.blend.laplacian_blend_conv2d_ref on the GPU) vs the fused op,
    forward and forward+backward.  Bounds per call: FMA = 2 (2C+1) (L-1) width per pixel (separable blur, both passes),
    bytes = 4 N H W (3C+1) (read img0, img1, mask, write out); each as a share of the data-sheet peak."""
    from oracle import blend as OB
    from gangealing_b200.splat2d import laplacian_blend
    props = torch.cuda.get_device_properties(0)
    try:
        import subprocess
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001 -- report, do not fail the measurement
        power = "unknown (%s)" % e
    print("card: %s | power limit, max SM clock: %s" % (props.name, power))
    presets = {"laplacian": (5, 45, 1.0), "laplacian_light": (3, 11, 0.5)}
    rows = []
    g = torch.Generator(device=dev).manual_seed(0)
    for n, res in [(4, 1024), (8, 512)]:
        c = 3
        img0 = torch.rand(n, c, res, res, device=dev, generator=g) * 2 - 1
        img1 = torch.rand(n, c, res, res, device=dev, generator=g) * 2 - 1
        mask = torch.rand(n, 1, res, res, device=dev, generator=g)
        gout = torch.rand(n, c, res, res, device=dev, generator=g)
        for name, (levels, k, s) in presets.items():
            fma = 2 * (2 * c + 1) * (levels - 1) * k * n * res * res
            nbytes = 4 * n * res * res * (3 * c + 1)
            t_fma, t_mem = fma / (FP32_PEAK_TFLOPS * 0.5e12) * 1e3, nbytes / (peak * 1e6)   # ms at peak (1 FMA = 2 FLOP)
            ms_ref = timeit(lambda i: OB.laplacian_blend_conv2d_ref(img0, img1, mask, levels, k, s), 1, iters=5, warmup=2)
            ms_fwd = timeit(lambda i: laplacian_blend(img0, img1, mask, levels, k, s), 1, iters=20, warmup=3)
            leaves = [t.clone().requires_grad_(True) for t in (img0, img1, mask)]

            def fwd_bwd(i):
                out = laplacian_blend(*leaves, levels, k, s)
                return torch.autograd.grad(out, leaves, gout)
            ms_fb = timeit(fwd_bwd, 1, iters=10, warmup=3)
            err = (laplacian_blend(img0, img1, mask, levels, k, s)
                   - OB.laplacian_blend_conv2d_ref(img0, img1, mask, levels, k, s)).abs().max().item()
            bound = "FMA" if t_fma >= t_mem else "HBM"
            row = {"preset": name, "N": n, "res": res, "reference_ms": ms_ref, "fused_fwd_ms": ms_fwd,
                   "fused_fwd_bwd_ms": ms_fb, "fma_G": fma / 1e9, "MB": nbytes / 1e6,
                   "fwd_fma_frac_of_peak": t_fma / ms_fwd, "fwd_bytes_frac_of_peak": t_mem / ms_fwd, "binding": bound,
                   "speedup_vs_reference": ms_ref / ms_fwd, "max_abs_diff_vs_reference": err}
            rows.append(row)
            print("%-16s N=%d %4d^2  ref %8.3f ms | fused fwd %7.3f ms  fwd+bwd %7.3f ms | x%5.1f vs ref | fwd: FMA %.1f G "
                  "= %4.1f%% of FP32 peak, bytes %.0f MB = %4.1f%% of HBM peak -> %s-bound | max|diff| %.2e" % (
                      name, n, res, ms_ref, ms_fwd, ms_fb, ms_ref / ms_fwd, fma / 1e9, 100 * t_fma / ms_fwd, nbytes / 1e6,
                      100 * t_mem / ms_fwd, bound, err))
    if json_path:
        os.makedirs(os.path.dirname(os.path.abspath(json_path)), exist_ok=True)
        json.dump({"card": props.name, "power_limit_and_max_sm_clock": power, "fp32_peak_tflops": FP32_PEAK_TFLOPS,
                   "peak_gbs": peak, "what": "Laplacian blending: reference 2-D conv formulation vs fused op (CUDA events)",
                   "rows": rows}, open(json_path, "w"), indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stn", action="store_true", help="the STN sampling path: reference / two-pass / one-pass")
    ap.add_argument("--blend", action="store_true", help="Laplacian blending: reference formulation vs the fused op")
    ap.add_argument("--ref", action="store_true", help="time the reference's own CUDA kernels (oracle/_ref) next to ours")
    ap.add_argument("--graph", action="store_true", help="time CUDA-graph replays (device time without launch overhead)")
    ap.add_argument("--batch", type=int, default=5)
    ap.add_argument("--json", default=None)
    ap.add_argument("--dtype", default="float32")
    ap.add_argument("--layout", default="nchw", choices=["nchw", "nhwc"])
    args = ap.parse_args()
    global GRAPH
    GRAPH = args.graph
    dt = getattr(torch, args.dtype)
    es = torch.empty(0, dtype=dt).element_size()
    B = args.batch
    dev = "cuda"
    peak, src = peak_gbs()
    k4 = torch.tensor([1., 3., 3., 1.])
    k4 = (k4[None] * k4[:, None]); k4 = (k4 / k4.sum() * 4).to(dev)
    rows = []

    def report(name, nbytes, ms):
        gbs = nbytes / ms / 1e6
        rows.append({"op": name, "ms": ms, "GB/s": gbs, "frac": gbs / peak, "MB": nbytes / 1e6})
        print("%-46s %9.3f ms %9.1f MB %8.1f GB/s  %5.1f%% of %s peak" % (name, ms, nbytes / 1e6, gbs, 100 * gbs / peak, src))

    def pool_count(nbytes):
        return max(2, min(8, int(400e6 // max(nbytes, 1)) + 1))

    if args.stn:
        stn_rows(B, dev, timeit, peak, args.json)
        return
    if args.blend:
        blend_rows(dev, timeit, peak, args.json)
        return
    if args.ref:
        reference_bar(B, dev, k4, timeit, pool_count, peak, args.json)
        return
    if args.layout == "nhwc":
        nhwc_family(B, dev, k4, timeit, report, pool_count)
        if args.json:
            os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
            json.dump({"batch": B, "dtype": "float32", "layout": "nhwc", "peak_gbs": peak, "peak_source": src, "rows": rows},
                      open(args.json, "w"), indent=1)
        return
    for C, H in [(128, 256), (256, 128), (512, 64), (512, 32), (512, 16), (512, 8)]:
        hin = H + 1
        nbytes = es * B * C * (hin * hin + H * H)
        P = pool_count(nbytes)
        xs = [torch.randn(B, C, hin, hin, device=dev, dtype=dt) for _ in range(P)]
        ms = timeit(lambda i: op.upfirdn2d(xs[i], k4, pad=(1, 1)), P)
        report("upfirdn2d blur C=%d %d->%d" % (C, hin, H), nbytes, ms)
        noise = torch.randn(B, 1, H, H, device=dev, dtype=dt)
        nw = torch.tensor([0.1], device=dev)
        bias = torch.randn(C, device=dev)
        ms = timeit(lambda i: op.blur_noise_bias_act(xs[i], k4, (1, 1), noise, nw, bias), P)
        report("fused blur+noise+bias+act C=%d %d->%d" % (C, hin, H), nbytes + es * B * H * H, ms)
        ys = [torch.randn(B, C, H, H, device=dev, dtype=dt) for _ in range(P)]
        nb2 = es * B * C * H * H * 2
        ms = timeit(lambda i: op.fused_leaky_relu(ys[i], bias.to(dt)), P)
        report("fused_leaky_relu C=%d %d^2" % (C, H), nb2, ms)
        ms = timeit(lambda i: op.noise_bias_act(ys[i], noise, nw, bias), P)
        report("noise+bias+act C=%d %d^2" % (C, H), nb2 + es * B * H * H, ms)
        ms = timeit(lambda i: bias_act_backward_raw(ys[i], ys[(i + 1) % P], 0.2, 1.4, True), P)
        report("bias_act backward(+bias grad) C=%d %d^2" % (C, H), es * B * C * H * H * 3, ms)
        ms = timeit(lambda i: ys[(i + 1) % P].copy_(ys[i]), P)
        report("  torch copy_ (roofline probe) C=%d %d^2" % (C, H), nb2, ms)
        del xs, ys
    # RGB skip upsample and its backward
    for H in (128, 64):
        x = torch.randn(B, 3, H, H, device=dev, dtype=dt)
        ms = timeit(lambda i: op.upfirdn2d(x, k4, up=2, pad=(2, 1)), 1)
        report("upfirdn2d rgb up2 %d->%d" % (H, 2 * H), es * B * 3 * (H * H + 4 * H * H), ms)
        g = torch.randn(B, 3, 2 * H, 2 * H, device=dev, dtype=dt)
        ms = timeit(lambda i: op.upfirdn2d(g, k4, down=2, pad=(1, 1)), 1)
        report("upfirdn2d rgb-up bwd dn2 %d->%d" % (2 * H, H), es * B * 3 * (H * H + 4 * H * H), ms)
    # STN blurs
    for C, H, pad in [(64, 128, (2, 2)), (64, 128, (1, 1)), (128, 64, (2, 2)), (512, 32, (2, 2))]:
        x = [torch.randn(B, C, H, H, device=dev, dtype=dt) for _ in range(4)]
        ho = H + 2 * pad[0] - 3
        ms = timeit(lambda i: op.upfirdn2d(x[i], k4, pad=pad), 4)
        report("upfirdn2d stn blur C=%d %d pad%s" % (C, H, pad), es * B * C * (H * H + ho * ho), ms)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump({"batch": B, "dtype": args.dtype, "peak_gbs": peak, "peak_source": src, "rows": rows},
                  open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
