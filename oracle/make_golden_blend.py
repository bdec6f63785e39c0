"""Generate tests/golden/laplacian_blend.npz from the reference's LaplacianBlender and pin oracle/blend.py against it.

Run where the reference checkout is (GG_REFERENCE_ROOT; its module imports cv2):  python -m oracle.make_golden_blend
Like oracle/make_golden.py: the REFERENCE's own CPU implementation runs on seeded inputs, the float64 oracle must
reproduce it (outputs and the three input gradients, 1e-6 relative), and the reference's results are stored.  The inputs
are rebuilt from their seed by oracle.blend.fixture_inputs, so only results are stored.  The other fixtures are untouched.
"""
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import blend as B, refimport  # noqa: E402
from oracle.make_golden import _close, _save  # noqa: E402

BLEND_CASES = [
    # name, (N, C, H, W), LaplacianBlender kwargs, fixture_inputs seed
    ("laplacian_40x56", (1, 3, 40, 56), dict(), 1),                       # splat_points' 'laplacian' preset; image < halo
    ("light_40x56", (1, 3, 40, 56), dict(levels=3, gaussian_kernel_size=11, gaussian_sigma=0.5), 2),   # 'laplacian_light'
    ("custom_40x56", (1, 3, 40, 56), dict(levels=4, gaussian_kernel_size=11, gaussian_sigma=1.0, level_size_adder=2,
                                          level_sigma_multiplier=1.5), 3),
    ("laplacian_144x201", (1, 1, 144, 201), dict(), 4),
]


def gen_laplacian_blend():
    """Laplacian pyramid blending (utils/laplacian_blending.py:13-107): the reference's LaplacianBlender (fp32, CPU) on
    seeded inputs -- output and the three input gradients for a seeded upstream gradient."""
    spec = importlib.util.spec_from_file_location("ref_laplacian_blending",
                                                  os.path.join(refimport.REFERENCE_ROOT, "utils", "laplacian_blending.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    out = {}
    for name, shape, kw, seed in BLEND_CASES:
        img0, img1, mask, gout = B.fixture_inputs(seed, *shape)
        args = [t.clone().requires_grad_(True) for t in (img0, img1, mask)]
        res = ref.LaplacianBlender(**kw)(*args)
        grads = torch.autograd.grad(res, args, gout)
        cfg = dict(levels=kw.get("levels", 5), kernel_size=kw.get("gaussian_kernel_size", 45),
                   sigma=kw.get("gaussian_sigma", 1), level_size_adder=kw.get("level_size_adder", 0),
                   level_sigma_multiplier=kw.get("level_sigma_multiplier", 2))
        args64 = [t.double().requires_grad_(True) for t in (img0, img1, mask)]
        res64 = B.laplacian_blend_ref(*args64, **cfg)
        grads64 = torch.autograd.grad(res64, args64, gout.double())
        _close(res64, res.detach().double(), 1e-6, "laplacian_blend/%s out" % name)
        for what, g64, g in zip(("g0", "g1", "gm"), grads64, grads):
            _close(g64, g.double(), 1e-6, "laplacian_blend/%s %s" % (name, what))
        out[name + ".cfg"] = np.array([cfg["levels"], cfg["kernel_size"], cfg["sigma"], cfg["level_size_adder"],
                                       cfg["level_sigma_multiplier"], seed] + list(shape), dtype=np.float64)
        out[name + ".out"] = res.detach()
        out[name + ".g0"], out[name + ".g1"], out[name + ".gm"] = grads
    _save("laplacian_blend", **out)


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen_laplacian_blend()
