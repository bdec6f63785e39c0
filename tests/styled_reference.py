"""The fused StyledConv / ToRGB tails' test inputs and bf16 storage contract (not collected: the name does not match
test_*.py).  test_styled_fused_gpu.py holds the general route to them, test_const_style_tails_gpu.py the sign-mask route
of the layers whose styles are constants."""
import torch

from fp64_contract import BF16, DEV, blur_k, blur_plan, check_once, check_sum, fir64, library, lrelu64, rowwise_c, slope_gain
from oracle import stylegan2_ops as so
from oracle.rounding import U32, ulp


def inputs(n, c, h, w, blur, with_rgb, with_next, seed):
    g = torch.Generator().manual_seed(seed)
    oh, ow = (h - 1, w - 1) if blur else (h, w)
    t = {"raw": torch.randn(n, c, h, w, generator=g), "demod": torch.rand(n, c, generator=g) + 0.5,
         "noise": torch.randn(n, 1, oh, ow, generator=g), "nw": torch.randn(1, generator=g) * 0.3, "bias": torch.randn(c, generator=g) * 0.5}
    t["s_next"] = torch.randn(n, c, generator=g) + 1.0 if with_next else None
    t["wm"] = torch.randn(n, 3, c, generator=g) / c ** 0.5 if with_rgb else None
    t["rgb_bias"] = torch.randn(3, generator=g) if with_rgb else None
    t["skip"] = torch.randn(n, 3, oh, ow, generator=g) if with_rgb else None
    t["g_xs"] = torch.randn(n, c, oh, ow, generator=g) if with_next else None
    t["g_rgb"] = torch.randn(n, 3, oh, ow, generator=g) if with_rgb else None
    return t


def dekink(t, blur, dtype, margin=2e-3):
    """Leaky-ReLU is not differentiable at 0: a pre-activation within rounding of 0 takes a different slope in two correct
    implementations, and the flip shows up at full size in the gradients.  Move `raw` a little wherever the oracle's
    pre-activation is closer to 0 than `margin`, so every comparison below is taken away from the kink."""
    k = so.make_kernel([1, 3, 3, 1]) * 4 if blur else None
    for _ in range(8):
        raw = t["raw"].to(dtype).float()
        if blur:
            pre = so.blur_noise_bias_act_ref(raw, k, (1, 1), t["noise"], t["nw"], t["bias"], negative_slope=1.0, scale=1.0, row_scale=t["demod"])
        else:
            pre = so.noise_bias_act_ref(raw * t["demod"][:, :, None, None], t["noise"], t["nw"], t["bias"], negative_slope=1.0, scale=1.0)
        bad = (pre.abs() < margin).nonzero()
        if bad.shape[0] == 0:
            return t
        off = 1 if blur else 0
        for n, c, y, x in bad.tolist():
            t["raw"][n, c, y + off, x + off] += 0.0625 * (1 + (y + x) % 3)
        t["raw"] = t["raw"].to(dtype).float()
    raise AssertionError("could not move the test inputs away from the activation kink")


def bf16_tail_contract(t, blur, xs, rgb, gg, slope=0.2, gain=2 ** 0.5):
    """bf16 storage contract of the public fused tail (tests/test_bf16_storage_gpu.py): float64 reference on the stored raw /
    g_xs.  At this level the backward also reads the forward's stored activation `out` (allowance: half an ulp of o per
    element it enters), and the blur layers hand g_t = lrelu'(out)*gain*g_xs*s_next from one launch to the next as a bf16
    tensor (DESIGN.md, deviations): g_raw and d_demod are allowed B^T(1/2 ulp(g_t)) on top of the fp32 bound."""
    d = {nm: (v.double().to(DEV) if isinstance(v, torch.Tensor) else v) for nm, v in t.items()}
    raw = t["raw"].to(torch.bfloat16).double().to(DEV)
    n, c = raw.shape[:2]
    dm = d["demod"][:, :, None, None]
    k = (so.make_kernel([1, 3, 3, 1]) * 4).to(DEV) if blur else None
    b = d["bias"][:, None, None]
    noise = d["nw"] * d["noise"]
    if blur:
        pre = fir64(raw, k, (1, 1, 1, 1)) * dm + b + noise
        apre = fir64(raw.abs(), k.abs(), (1, 1, 1, 1)) * dm.abs() + b.abs() + noise.abs()
        k_o = blur_k(k) + 5
    else:
        pre, apre, k_o = raw * dm + b + noise, (raw * dm).abs() + b.abs() + noise.abs(), 6
    o, ao = lrelu64(pre, slope, gain), apre * slope_gain(slope, gain)
    h_o = 0.5 * ulp(o, torch.bfloat16) + k_o * U32 * ao           # stored `out` vs o
    oh, ow = o.shape[2:]
    if xs is not None:
        s = d["s_next"][:, :, None, None]
        check_once(xs, o * s, ao * s.abs(), k_o + 1, "fused_tail xs")
    if rgb is not None:
        wm = d["wm"]
        ref = torch.einsum("noc,nchw->nohw", wm, o) + d["rgb_bias"].reshape(1, 3, 1, 1) + d["skip"]
        ab = torch.einsum("noc,nchw->nohw", wm.abs(), ao) + d["rgb_bias"].abs().reshape(1, 3, 1, 1) + d["skip"].abs()
        check_sum(rgb, ref, ab, c // 8 + 11, "fused_tail rgb")
    gxs = d["g_xs"].to(torch.bfloat16).double() if t["g_xs"] is not None else torch.zeros_like(o)
    s = d["s_next"][:, :, None, None] if t["s_next"] is not None else torch.zeros(n, c, 1, 1, dtype=torch.float64, device=DEV)
    go, goa = gxs * s, (gxs * s).abs()
    if t["g_rgb"] is not None:
        go = go + torch.einsum("noc,nohw->nchw", d["wm"], d["g_rgb"])
        goa = goa + torch.einsum("noc,nohw->nchw", d["wm"].abs(), d["g_rgb"].abs())
    sl = torch.where(pre > 0, 1.0, slope) * gain                   # dekink keeps every pre-activation off the kink
    gt, gta = go * sl, goa * sl.abs()
    c_tail = rowwise_c(n, c, oh * ow, 0, True, BF16, library().sm_count())
    if blur:
        kf, gp = torch.flip(k, [0, 1]), (2, 2, 2, 2)
        h_t = 0.5 * ulp(gt, torch.bfloat16) + 4 * U32 * gta         # g_t: g*s, *slope, *gain, the bf16 store
        tr, tra, trh = fir64(gt, kf, gp), fir64(gta, kf.abs(), gp), fir64(h_t, kf.abs(), gp)
        check_once(gg["raw"], tr * dm, tra * dm.abs(), blur_k(k) + 1, "fused_tail g_raw (blur)", extra=trh * dm.abs())
        if "demod" in gg:
            p = blur_plan(BF16, n, c, oh, ow, 4, 4, gp, library().sm_count())
            check_sum(gg["demod"], (tr * raw).sum((2, 3)), (tra * raw.abs()).sum((2, 3)),
                      blur_k(k) + 1 + p["seg_rows"] + 32 + p["xblocks"] * p["segs"] // 32 + 35, "fused_tail d_demod (blur)", extra=(trh * raw.abs()).sum((2, 3)))
    else:
        check_once(gg["raw"], gt * dm, gta * dm.abs(), 7, "fused_tail g_raw")
        if "demod" in gg:
            check_sum(gg["demod"], (gt * raw).sum((2, 3)), (gta * raw.abs()).sum((2, 3)), c_tail + 6, "fused_tail d_demod")
    if "s_next" in gg:
        check_sum(gg["s_next"], (gxs * o).sum((2, 3)), (gxs * o).abs().sum((2, 3)), c_tail, "fused_tail d_s_next",
                  extra=(gxs.abs() * h_o).sum((2, 3)))
    if "wm" in gg:
        gr = d["g_rgb"]
        check_sum(gg["wm"], torch.einsum("nohw,nchw->noc", gr, o), torch.einsum("nohw,nchw->noc", gr.abs(), o.abs()), c_tail,
                  "fused_tail d_wm", extra=torch.einsum("nohw,nchw->noc", gr.abs(), h_o))
    if "skip" in gg:
        assert torch.equal(gg["skip"].cpu(), t["g_rgb"])
