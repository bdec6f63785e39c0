"""Torch restatement of Laplacian pyramid blending (test infrastructure -- see oracle/__init__.py).

Reference: utils/laplacian_blending.py:13-107 (`LaplacianBlender`), called by splat_points(blend_alg='laplacian' |
'laplacian_light') in utils/vis_tools/helpers.py:186-193.  Every level blurs with the same width k + a and sigma s * m^l,
replicate padding of width // 2; the blurred mask weights a lerp of the two Laplacian stacks, and the stack is summed.

`laplacian_blend_ref` restates it with the 2-D blur split into two clamped 1-D passes (exact: the kernel is an outer
product and replicate padding clamps each axis on its own).  It runs in the dtype and on the device of its inputs, so in
float64 its autograd is the gradient reference of the CUDA op.  `laplacian_blend_conv2d_ref` keeps the reference's own
formulation (fp32 2-D taps, one depthwise 2-D convolution per level, materialised stacks): the bar tools/opbench.py times.
"""
import numpy as np
import torch
import torch.nn.functional as F

# splat_points' presets (helpers.py:188-193)
PRESETS = {
    "laplacian": dict(levels=5, kernel_size=45, sigma=1.0),
    "laplacian_light": dict(levels=3, kernel_size=11, sigma=0.5),
}


def gaussian_taps(width, sigma):
    """cv2.getGaussianKernel(width, sigma) for sigma > 0: exp(-(i - (width-1)/2)^2 / (2 sigma^2)), normalised, float64."""
    if sigma <= 0:
        raise ValueError("gaussian_taps: sigma must be positive")
    x = np.arange(width, dtype=np.float64) - (width - 1) * 0.5
    g = np.exp(-0.5 / (sigma * sigma) * x * x)
    return g / g.sum()


def level_taps(levels, kernel_size, sigma, level_size_adder=0, level_sigma_multiplier=2):
    """(levels - 1, width) float64: the 1-D taps of every blurring level (laplacian_blending.py:34-39)."""
    width = kernel_size + level_size_adder
    rows = [gaussian_taps(width, sigma * level_sigma_multiplier ** level) for level in range(levels - 1)]
    return torch.from_numpy(np.stack(rows)) if rows else torch.zeros(0, width, dtype=torch.float64)


def blur_ref(x, taps):
    """One level: replicate pad + 1-D blur along W, then along H.  x: (N, C, H, W); taps: (width,)."""
    width = taps.numel()
    r, c = width // 2, x.shape[1]
    kh = taps.reshape(1, 1, 1, width).expand(c, 1, 1, width)
    kv = taps.reshape(1, 1, width, 1).expand(c, 1, width, 1)
    x = F.conv2d(F.pad(x, (r, r, 0, 0), mode="replicate"), kh, groups=c)
    return F.conv2d(F.pad(x, (0, 0, r, r), mode="replicate"), kv, groups=c)


def laplacian_blend_ref(img0, img1, mask, levels, kernel_size, sigma, level_size_adder=0, level_sigma_multiplier=2,
                        taps=None):
    """out = sum_{l<L-1} lerp(A_l - A_{l+1}, B_l - B_{l+1}, M_l) + lerp(A_{L-1}, B_{L-1}, M_{L-1}), G_{l+1} = blur_l(G_l)."""
    if taps is None:
        taps = level_taps(levels, kernel_size, sigma, level_size_adder, level_sigma_multiplier)
    taps = taps.to(device=img0.device, dtype=img0.dtype)

    def stack(x):
        out = [x]
        for level in range(levels - 1):
            out.append(blur_ref(out[-1], taps[level]))
        return out
    a, b, m = stack(img0), stack(img1), stack(mask)
    out = None
    for level in range(levels):
        if level < levels - 1:
            term = torch.lerp(a[level] - a[level + 1], b[level] - b[level + 1], m[level])
        else:
            term = torch.lerp(a[level], b[level], m[level])
        out = term if out is None else out + term
    return out


def laplacian_blend_conv2d_ref(img0, img1, mask, levels, kernel_size, sigma, level_size_adder=0,
                               level_sigma_multiplier=2):
    """The reference's formulation: fp32 2-D taps (the float64 outer product, rounded), a depthwise 2-D convolution per
    level, three (levels, N, C, H, W) stacks, lerp, sum over levels."""
    taps = level_taps(levels, kernel_size, sigma, level_size_adder, level_sigma_multiplier)
    k2d = [torch.outer(t, t).float().to(img0.device) for t in taps]
    r = taps.shape[1] // 2

    def stacks(x):
        lap, gauss = [], []
        c = x.shape[1]
        for level in range(levels):
            gauss.append(x)
            if level < levels - 1:
                k = k2d[level].reshape(1, 1, *k2d[level].shape).expand(c, 1, -1, -1)
                blurred = F.conv2d(F.pad(x, (r, r, r, r), mode="replicate"), k, groups=c)
                lap.append(x - blurred)
                x = blurred
            else:
                lap.append(x)
        return torch.stack(lap), torch.stack(gauss)
    lp0, _ = stacks(img0)
    lp1, _ = stacks(img1)
    _, gm = stacks(mask)
    return lp0.lerp(lp1, gm).sum(dim=0)


def splat_points_ref(images, points, sigma, opacity, colors, alpha_channel=None, blend_alg="alpha", splat_fn=None):
    """splat_points with every blend branch (helpers.py:184-193): 'alpha' is oracle.splat.splat_points_ref itself; the
    Laplacian branches make the same two splats (colours, soft-normalised alpha) and blend them into `images` with
    laplacian_blend_ref and the preset's parameters."""
    from . import splat as _splat
    splat_fn = splat_fn or _splat.splat2d_ref
    if blend_alg == "alpha":
        return _splat.splat_points_ref(images, points, sigma, opacity, colors, alpha_channel, splat_fn=splat_fn)
    if blend_alg not in PRESETS:
        raise ValueError("blend_alg must be 'alpha', 'laplacian' or 'laplacian_light' (got %r)" % (blend_alg,))
    n, _, h, w = images.shape
    if alpha_channel is None:
        alpha_channel = torch.ones(points.shape[0], points.shape[1], 1, device=points.device)
    sig = torch.full((n,), float(sigma), device=points.device) if not torch.is_tensor(sigma) else sigma
    prop_obj = splat_fn(torch.zeros(n, colors.shape[-1], h, w, device=images.device), points, colors, sig, False)
    prop_mask = splat_fn(torch.zeros(n, 1, h, w, device=images.device), points, alpha_channel, sig, True) * opacity
    return laplacian_blend_ref(images, prop_obj.to(images.device), prop_mask.to(images.device), **PRESETS[blend_alg])


def cpu_ops():
    """oracle.opset.cpu_ops() plus `laplacian_blend` (laplacian_blend_ref): the op set that runs
    ComposedSTN.uncongeal_and_splat(blend_alg='laplacian*') on the CPU restatement."""
    import types
    from . import opset
    return types.SimpleNamespace(**vars(opset.cpu_ops()), laplacian_blend=laplacian_blend_ref)


def fixture_inputs(seed, n, c, h, w):
    """Seeded (img0, img1, mask, grad_out) float32 built from a splitmix64 hash in integer arithmetic, so the golden fixture
    need not store its inputs.  The mask is 1 inside a soft-edged disc, 0 far outside, with exact 0 and 1 regions."""
    def uniform(k, count):
        z = (np.arange(count, dtype=np.uint64) + np.uint64(seed * 1_000_003 + k * 7919)) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
        return ((z >> np.uint64(40)).astype(np.float64) / float(1 << 24)).astype(np.float32)   # 24-bit uniforms in [0, 1)
    img0 = torch.from_numpy(uniform(1, n * c * h * w).reshape(n, c, h, w) * 2 - 1)
    img1 = torch.from_numpy(uniform(2, n * c * h * w).reshape(n, c, h, w) * 2 - 1)
    gout = torch.from_numpy(uniform(3, n * c * h * w).reshape(n, c, h, w) * 2 - 1)
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing="ij")
    rad = np.sqrt((ys - 0.45 * h) ** 2 + (xs - 0.55 * w) ** 2) / (0.3 * min(h, w))
    noise = uniform(4, n * h * w).reshape(n, 1, h, w)
    mask = np.clip(2.0 - 2.0 * rad[None, None] + 0.4 * (noise - 0.5), 0.0, 1.0).astype(np.float32)
    return img0, img1, torch.from_numpy(mask), gout
