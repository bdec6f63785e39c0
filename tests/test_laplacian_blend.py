"""Laplacian pyramid blending (csrc/blend.cu, splat2d.laplacian_blend / LaplacianBlender / splat_points).

CPU: the float64 oracle (oracle/blend.py) against the reference's own LaplacianBlender (tests/golden/laplacian_blend.npz),
the splat_points composition, the C ABI's argument checks and the call site on the oracle op set.
GPU: the kernel's output and gradients against the reference fixture, bitwise reproducibility and CUDA-graph replay,
splat_points and uncongeal_and_splat against the oracle, and the error behaviour.  Every kernel instantiation is checked
element by element against float64 in test_blend_family_gpu.py."""
import pytest
import torch

from conftest import assert_close, golden_cases, load_golden
from oracle import blend as OB
from oracle import splat as SP

DEV = "cuda"

CONFIGS = {   # laplacian_blend(levels, kernel_size, sigma, level_size_adder, level_sigma_multiplier)
    "laplacian": (5, 45, 1.0, 0, 2),
    "laplacian_light": (3, 11, 0.5, 0, 2),
    "custom": (4, 11, 1.0, 2, 1.5),
    "single_level": (1, 45, 1.0, 0, 2),
}
FWD_RTOL = 2e-6       # 10x the fp32 CPU error of the separable restatement (1.1-1.6e-7 of the output's max-abs)
GRAD_RTOL = 5e-6
MAX_ERR = {}          # largest relative errors seen, printed at the end of the GPU sweep (pytest -s)


def _rel_err(actual, expected):
    actual, expected = actual.detach().double().cpu(), expected.detach().double().cpu()
    return ((actual - expected).abs().max() / expected.abs().max().clamp_min(1e-12)).item()


def _record(key, err):
    MAX_ERR[key] = max(MAX_ERR.get(key, 0.0), err)


def _oracle64(img0, img1, mask, cfg, grad_out=None):
    """float64 oracle output (and input gradients for grad_out) on the tensors' device."""
    args = [t.detach().double().requires_grad_(grad_out is not None) for t in (img0, img1, mask)]
    out = OB.laplacian_blend_ref(*args, *cfg)
    if grad_out is None:
        return out.detach()
    return out.detach(), torch.autograd.grad(out, args, grad_out.double())


# ------------------------------------------------------------------------------------------------ CPU
def _fixture_cfg(blob, name):
    v = blob[name + ".cfg"].tolist()
    cfg = (int(v[0]), int(v[1]), float(v[2]), int(v[3]), float(v[4]))
    return cfg, int(v[5]), tuple(int(s) for s in v[6:])


def test_oracle_reproduces_the_reference_fixture():
    """The separable float64 restatement against the reference's LaplacianBlender (fp32 2-D convolutions): outputs and the
    three gradients, both presets, a custom (a=2, m=1.5) configuration, an image smaller than the halo and 144x201."""
    blob = load_golden("laplacian_blend")
    names = golden_cases(blob)
    assert len(names) == 4
    for name in names:
        cfg, seed, shape = _fixture_cfg(blob, name)
        img0, img1, mask, gout = OB.fixture_inputs(seed, *shape)
        out, grads = _oracle64(img0, img1, mask, cfg, gout)
        assert_close(out, blob[name + ".out"], rtol=1e-6, what=name + " out")
        for key, g in zip(("g0", "g1", "gm"), grads):
            assert_close(g, blob[name + "." + key], rtol=1e-6, what=name + " " + key)


def test_fixture_masks_have_exact_zero_and_one_regions():
    _, _, mask, _ = OB.fixture_inputs(4, 1, 1, 144, 201)
    assert (mask == 0).float().mean() > 0.2 and (mask == 1).float().mean() > 0.05


def test_separable_restatement_equals_the_conv2d_formulation():
    img0, img1, mask, _ = OB.fixture_inputs(7, 2, 3, 40, 56)
    for cfg in CONFIGS.values():
        assert_close(OB.laplacian_blend_ref(img0.double(), img1.double(), mask.double(), *cfg),
                     OB.laplacian_blend_conv2d_ref(img0, img1, mask, *cfg), rtol=2e-6, what="conv2d formulation %s" % (cfg,))


def _splat_case(seed, n=2, p=60, h=40, w=48):
    g = torch.Generator().manual_seed(seed)
    imgs = torch.rand(n, 3, h, w, generator=g) * 2 - 1
    pts = torch.rand(n, p, 2, generator=g) * torch.tensor([w - 1.0, h - 1.0])
    colors = torch.rand(n, p, 3, generator=g) * 2 - 1
    return imgs, pts, colors


@pytest.mark.parametrize("blend_alg", ["laplacian", "laplacian_light"])
def test_splat_points_ref_blend_branches(blend_alg):
    """helpers.py:184-193: the two splats, then LaplacianBlender(preset)(images, prop_obj, prop_mask)."""
    imgs, pts, colors = _splat_case(1)
    sig = torch.full((2,), 1.1)
    prop_obj = SP.splat2d_ref(torch.zeros(2, 3, 40, 48), pts, colors, sig, False)
    prop_mask = SP.splat2d_ref(torch.zeros(2, 1, 40, 48), pts, torch.ones(2, 60, 1), sig, True) * 0.8
    levels, k, s = {"laplacian": (5, 45, 1), "laplacian_light": (3, 11, 0.5)}[blend_alg]
    expect = OB.laplacian_blend_conv2d_ref(imgs, prop_obj, prop_mask, levels, k, s)
    got = OB.splat_points_ref(imgs, pts, 1.1, 0.8, colors, blend_alg=blend_alg)
    assert_close(got, expect, rtol=2e-6, what="splat_points_ref " + blend_alg)
    alpha = OB.splat_points_ref(imgs, pts, 1.1, 0.8, colors)
    assert torch.equal(alpha, prop_mask * prop_obj + (1 - prop_mask) * imgs)
    with pytest.raises(ValueError):
        OB.splat_points_ref(imgs, pts, 1.1, 0.8, colors, blend_alg="poisson")


def test_abi_rejects_bad_arguments():
    from gangealing_b200 import _lib
    dll = _lib.load()
    one = 1   # non-null pointer value: validation must reject these calls before dereferencing anything
    fwd = dll.gg_laplacian_blend_forward
    bwd = dll.gg_laplacian_blend_backward
    assert fwd(one, one, one, one, one, one, 1, 3, 8, 8, 5, 44, None) == -1            # even width
    assert b"odd" in dll.gg_last_error()
    assert fwd(one, one, one, one, one, one, 1, 3, 8, 8, 5, 65, None) == -2            # above the cap of 63
    assert b"63" in dll.gg_last_error()
    assert fwd(one, one, one, one, one, one, 1, 3, 8, 8, 0, 45, None) == -1            # levels < 1
    assert b"levels" in dll.gg_last_error()
    assert fwd(one, one, one, one, one, None, 1, 3, 8, 8, 5, 45, None) == -1           # null taps
    assert fwd(None, one, one, one, one, one, 1, 3, 8, 8, 5, 45, None) == -1           # null output
    assert b"null" in dll.gg_last_error()
    assert fwd(one, one, one, one, one, one, 0, 3, 8, 8, 5, 45, None) == -1            # non-positive sizes
    assert fwd(one, one, one, one, one, one, 1, 3, 8, -8, 5, 45, None) == -1
    assert b"positive" in dll.gg_last_error()
    assert bwd(one, one, one, one, one, one, one, one, one, 1, 3, 8, 8, 3, 12, None) == -1
    assert bwd(one, one, None, one, one, one, one, one, one, 1, 3, 8, 8, 3, 11, None) == -1
    assert bwd(one, one, one, one, one, one, one, one, one, 1, 3, 8, 8, 3, 101, None) == -2
    assert dll.gg_laplacian_blend_workspace(2, 3, 8, 8, 1, 1) == 0                    # one level: elementwise, no workspace
    assert dll.gg_laplacian_blend_workspace(2, 3, 8, 8, 5, 0) == 4 * 2 * 7 * 2 * 64
    assert dll.gg_laplacian_blend_workspace(2, 3, 8, 8, 5, 1) == 4 * (12 + 9) * 2 * 64


def test_ops_refuse_cpu_tensors_and_bad_configurations():
    from gangealing_b200.splat2d import LaplacianBlender, laplacian_blend
    x = torch.zeros(1, 3, 8, 8)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        laplacian_blend(x, x, torch.zeros(1, 1, 8, 8), 5, 45, 1.0)
    with pytest.raises(AssertionError):
        LaplacianBlender(gaussian_kernel_size=44)
    with pytest.raises(AssertionError):
        LaplacianBlender(level_size_adder=1)
    with pytest.raises(RuntimeError, match="outside"):
        LaplacianBlender(gaussian_kernel_size=61, level_size_adder=4)
    with pytest.raises(RuntimeError, match="levels"):
        LaplacianBlender(levels=0)


def test_laplacian_taps_match_the_oracle():
    from gangealing_b200.splat2d.blend import level_taps
    for cfg in CONFIGS.values():
        if cfg[0] > 1:
            assert torch.equal(level_taps(*cfg, device="cpu"), OB.level_taps(*cfg).float())


def test_compat_registers_the_blender():
    import sys
    from gangealing_b200 import compat
    from gangealing_b200.splat2d import LaplacianBlender
    saved = sys.modules.pop("utils.laplacian_blending", None)
    try:
        compat.install()
        assert sys.modules["utils.laplacian_blending"].LaplacianBlender is LaplacianBlender
    finally:
        sys.modules.pop("utils.laplacian_blending", None)
        if saved is not None:
            sys.modules["utils.laplacian_blending"] = saved


def _disc_points(n, res=64):
    ys, xs = torch.meshgrid(torch.arange(float(res)), torch.arange(float(res)), indexing="ij")
    disc = ((ys - res / 2) ** 2 + (xs - res / 2) ** 2) < (0.35 * res) ** 2
    return torch.stack([xs[disc], ys[disc]], dim=1)[None].repeat(n, 1, 1)


def test_uncongeal_and_splat_laplacian_on_the_oracle_op_set():
    from gangealing_b200.stn import get_stn
    from oracle import opset
    stn = get_stn(["similarity", "flow"], flow_size=64, supersize=64, channel_multiplier=0.25, num_heads=1,
                  ops=OB.cpu_ops()).eval()
    opset.fill_parameters(stn, 21, gain=0.2)
    g = torch.Generator().manual_seed(3)
    imgs = torch.rand(1, 3, 64, 64, generator=g) * 2 - 1
    pts = _disc_points(1, 32)[:, ::7]
    colors = torch.randn(1, pts.shape[1], 3, generator=g)
    with torch.no_grad():
        got, got_pts = stn.uncongeal_and_splat(imgs, pts, colors, 1.3, 0.75, normalize_input_points=True,
                                               blend_alg="laplacian")
        two_pts = stn.uncongeal_points(imgs, pts, normalize_input_points=True)
        expect = OB.splat_points_ref(imgs, two_pts, 1.3, 0.75, colors, blend_alg="laplacian")
    assert_close(got_pts, two_pts, atol=1e-5, what="points")
    assert_close(got, expect, rtol=1e-5, what="laplacian-blended image")
    with pytest.raises(ValueError):
        stn.uncongeal_and_splat(imgs, pts, colors, 1.3, 0.75, blend_alg="poisson")


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_forward_and_gradients_vs_reference_fixture():
    from gangealing_b200.splat2d import laplacian_blend
    blob = load_golden("laplacian_blend")
    for name in golden_cases(blob):
        cfg, seed, shape = _fixture_cfg(blob, name)
        img0, img1, mask, gout = [t.to(DEV) for t in OB.fixture_inputs(seed, *shape)]
        args = [t.clone().requires_grad_(True) for t in (img0, img1, mask)]
        out = laplacian_blend(*args, *cfg)
        grads = torch.autograd.grad(out, args, gout)
        err = _rel_err(out, blob[name + ".out"])
        _record("fixture forward", err)
        assert err <= FWD_RTOL, "%s: %.3g" % (name, err)
        for key, g in zip(("g0", "g1", "gm"), grads):
            err = _rel_err(g, blob[name + "." + key])
            _record("fixture " + key, err)
            assert err <= GRAD_RTOL, "%s %s: %.3g" % (name, key, err)


@pytest.mark.gpu
def test_bitwise_reproducible_and_cuda_graph_replay():
    from gangealing_b200.splat2d import laplacian_blend
    cfg = CONFIGS["laplacian"]
    img0, img1, mask, gout = [t.to(DEV) for t in OB.fixture_inputs(5, 2, 3, 200, 260)]
    def step(args):
        out = laplacian_blend(*args, *cfg)
        return (out,) + torch.autograd.grad(out, args, gout)
    eager_args = [t.clone().requires_grad_(True) for t in (img0, img1, mask)]
    first = [t.clone() for t in step(eager_args)]
    second = step(eager_args)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    # capture: leaves first used on the capture stream (their gradient accumulators live there), warmed up there
    args = [t.clone().requires_grad_(True) for t in (img0, img1, mask)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step(args)
    side.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        captured = step(args)
    with torch.no_grad():                      # replay on other inputs first, then on the originals
        for t, value in zip(args, (img1, img0, mask.flip(-1))):
            t.copy_(value)
    graph.replay()
    torch.cuda.synchronize()
    assert not torch.equal(captured[0], first[0])
    with torch.no_grad():
        for t, value in zip(args, (img0, img1, mask)):
            t.copy_(value)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(captured, first):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("blend_alg", ["alpha", "laplacian", "laplacian_light"])
def test_splat_points_vs_oracle(blend_alg):
    from gangealing_b200.splat2d import splat2d, splat_points
    imgs, pts, colors = _splat_case(2, n=2, p=300, h=96, w=128)
    imgs, pts, colors = imgs.to(DEV), pts.to(DEV), colors.to(DEV)
    sig = torch.tensor([1.3, 0.8], device=DEV)
    got = splat_points(imgs, pts, sig, 0.75, colors, blend_alg=blend_alg)
    expect = OB.splat_points_ref(imgs, pts, sig, 0.75, colors, blend_alg=blend_alg, splat_fn=splat2d)
    assert_close(got, expect, rtol=1e-4, what="splat_points " + blend_alg)
    # (N, K, P, 2) points and a float sigma
    got4 = splat_points(imgs, pts.reshape(2, 3, 100, 2), 1.1, 0.75, colors, blend_alg=blend_alg)
    expect4 = OB.splat_points_ref(imgs, pts, 1.1, 0.75, colors, blend_alg=blend_alg, splat_fn=splat2d)
    assert_close(got4, expect4, rtol=1e-4, what="splat_points (N, K, P, 2) " + blend_alg)
    with pytest.raises(ValueError):
        splat_points(imgs, pts, 1.1, 0.75, None, blend_alg=blend_alg)


@pytest.mark.gpu
def test_uncongeal_and_splat_laplacian_vs_two_step_oracle():
    from gangealing_b200.splat2d import splat2d
    from gangealing_b200.stn import get_stn
    from oracle import opset
    stn = get_stn(["similarity", "flow"], flow_size=64, supersize=128, channel_multiplier=0.25, num_heads=1).eval()
    opset.fill_parameters(stn, 21, gain=0.2).to(DEV)
    g = torch.Generator().manual_seed(3)
    imgs = (torch.rand(2, 3, 128, 128, generator=g) * 2 - 1).to(DEV)
    pts = _disc_points(2).to(DEV)
    colors = torch.randn(2, pts.shape[1], 3, generator=g).to(DEV)
    with torch.no_grad():
        img, got_pts = stn.uncongeal_and_splat(imgs, pts, colors, 1.3, 0.75, output_resolution=128,
                                               normalize_input_points=True, padding_mode="border", blend_alg="laplacian")
        two_pts = stn.uncongeal_points(imgs, pts, normalize_input_points=True, output_resolution=128, padding_mode="border")
        two_img = OB.splat_points_ref(imgs, two_pts, 1.3, 0.75, colors, blend_alg="laplacian", splat_fn=splat2d)
    assert_close(got_pts, two_pts, atol=2e-3, what="points")
    assert_close(img, two_img, rtol=2e-3, what="laplacian-propagated image")


@pytest.mark.gpu
def test_error_behaviour_on_the_gpu():
    from gangealing_b200.splat2d import LaplacianBlender, laplacian_blend
    x = torch.zeros(2, 3, 16, 16, device=DEV)
    m = torch.zeros(2, 1, 16, 16, device=DEV)
    for dtype in (torch.float16, torch.bfloat16, torch.float64):
        with pytest.raises(RuntimeError, match="float32"):
            laplacian_blend(x.to(dtype), x.to(dtype), m.to(dtype), 5, 45, 1.0)
    with pytest.raises(RuntimeError, match="num_channels"):
        laplacian_blend(x, x, x, 5, 45, 1.0)
    with pytest.raises(RuntimeError):
        laplacian_blend(x, x[:, :, :8], m, 5, 45, 1.0)
    with pytest.raises(RuntimeError):
        laplacian_blend(x, x, m[:1], 5, 45, 1.0)
    with pytest.raises(RuntimeError):
        laplacian_blend(x[0], x[0], m[0], 5, 45, 1.0)
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        laplacian_blend(x, x, m.cpu(), 5, 45, 1.0)
    with torch.inference_mode():                                   # splat_points runs under inference_mode
        out = LaplacianBlender()(x + 1, x - 1, m + 0.25)
    assert_close(out, torch.full_like(x, 0.5), atol=1e-6, what="constant images")     # lerp(1, -1, 0.25)


@pytest.mark.gpu
def test_zz_report_largest_errors():
    """Prints the largest relative errors of the sweep above (run with -s)."""
    for key in sorted(MAX_ERR):
        print("laplacian_blend max relative error  %-22s %.3e" % (key, MAX_ERR[key]))
