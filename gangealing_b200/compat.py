"""Drop-in shim: makes the UNMODIFIED reference tree (`models/stylegan2/networks.py`,
`models/spatial_transformers/*.py`, `models/losses/loss.py`, `train.py` ...) run on libgg_b200's kernels.

    import gangealing_b200.compat as compat
    compat.install()                  # before the first `import models`
    sys.path.insert(0, "/path/to/gangealing")
    from models import Generator, get_stn     # reference code, sm_90a kernels underneath

It pre-registers, under the reference's module names, the modules that sit directly on the kernel boundary:
  models.stylegan2.op (+ .upfirdn2d, .fused_act, .conv2d_gradfix)   <- gangealing_b200.op
  models.spatial_transformers.antialiased_sampling                  <- gangealing_b200.stn.sampling
  utils.splat2d_cuda (+ .functional, .splat)                        <- gangealing_b200.splat2d
  utils.laplacian_blending (LaplacianBlender)                       <- gangealing_b200.splat2d.blend
  utils.vis_tools.flow_vis (flow_to_image)                          <- gangealing_b200.training.visuals
so the reference never reaches its import-time JIT builds (`torch.utils.cpp_extension.load`, op/upfirdn2d.py:9-16,
op/fused_act.py:10-17, utils/splat2d_cuda/functional.py:9-27 -- the last of which no longer compiles on modern
torch).  Everything above those modules is the reference's own code, untouched.
"""
import sys
import types


def install(force=False):
    from . import op as _op
    from . import splat2d as _splat
    from .op import conv2d_gradfix as _gradfix
    from .op import fused_act as _fused
    from .op import upfirdn2d as _upfirdn
    from .stn import sampling as _sampling

    def register(name, module):
        if force or name not in sys.modules:
            sys.modules[name] = module

    pkg = types.ModuleType("models.stylegan2.op")
    pkg.__path__ = []  # a package: `from models.stylegan2.op import conv2d_gradfix` resolves through sys.modules
    pkg.FusedLeakyReLU = _op.FusedLeakyReLU
    pkg.fused_leaky_relu = _op.fused_leaky_relu
    pkg.upfirdn2d = _op.upfirdn2d
    pkg.conv2d_gradfix = _gradfix
    register("models.stylegan2.op", pkg)
    register("models.stylegan2.op.upfirdn2d", _upfirdn)
    register("models.stylegan2.op.fused_act", _fused)
    register("models.stylegan2.op.conv2d_gradfix", _gradfix)
    register("models.spatial_transformers.antialiased_sampling", _sampling)
    register("utils.splat2d_cuda", _splat)
    register("utils.splat2d_cuda.functional", _splat.functional)
    splat_mod = types.ModuleType("utils.splat2d_cuda.splat")
    splat_mod.Splat2D, splat_mod.splat2d = _splat.Splat2D, _splat.splat2d
    register("utils.splat2d_cuda.splat", splat_mod)
    blend_mod = types.ModuleType("utils.laplacian_blending")     # the reference's needs cv2 for its 1-D Gaussians
    blend_mod.LaplacianBlender = _splat.LaplacianBlender
    register("utils.laplacian_blending", blend_mod)
    from .training import visuals as _visuals
    flow_vis = types.ModuleType("utils.vis_tools.flow_vis")       # train.py's flow images, colour wheel on the device
    flow_vis.flow_to_image = _visuals.flow_to_image
    register("utils.vis_tools.flow_vis", flow_vis)
    return pkg
