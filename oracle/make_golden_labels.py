"""Generate tests/golden/label_propagation.npz from the reference's labelled videos.

Run where the reference checkout is (GG_REFERENCE_ROOT):  python -m oracle.make_golden_labels
The reference's own smoothly_congeal_and_propagate (with visualize_label_propagation and visualize_correspondence) and
average_and_congeal (with its labelled tail) run on CPU on make_golden_pck's seeded STN, on make_golden_vis' cases (output
resolution 96, lengths 60 and 6, both stage_flip settings), with N = 4 and N = 1 images and a 40-point label with and
without an alpha channel.  Their splat2d is oracle.splat.splat2d_ref; their utils/vis_tools/helpers.py is loaded from its
file with its video, colour-scale, ray and Laplacian-blending imports stubbed, and its make_grid's `range=` keyword passed
on as torchvision's `value_range=`.  save_video is replaced by a capture of the frames it is given.  Stored: the label's
colours and alpha, a few frames of every video and every frame's per-channel sums.
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refimport  # noqa: E402
from oracle import splat as OS  # noqa: E402
from oracle.make_golden import _save  # noqa: E402
from oracle.make_golden_pck import STN_KW, _stub_modules, make_stn  # noqa: E402
from oracle import make_golden_vis as GV  # noqa: E402

SIGMA, OPACITY = 1.2, 0.7
LABEL_CASES = [   # name, make_golden_vis.SMOOTH_CASES index, images, alpha channel
    ("labels_stages_flip", 0, 4, True),
    ("labels_final_n1", 1, 1, False),
]
AVERAGE_CASE = ("labeled_average", 0, True)   # name, make_golden_vis.AVG_CASES index, alpha channel
VIDEOS = ("congealing", "propagation", "correspondence")


def label_colors(seed=11):
    """(1, P, 3) colours in [-1, 1] and (1, P, 1) opacities in [0, 1] for make_golden_vis.label_points()."""
    g = torch.Generator().manual_seed(seed)
    return torch.rand(1, GV.P, 3, generator=g) * 2 - 1, torch.rand(1, GV.P, 1, generator=g)


def kept_frames(video, counts):
    """A few frames of each video: the ends and the middle; in the correspondence video also the middle of the blend."""
    f = counts[video]
    if video == "correspondence":
        return [counts["congealing"] + 60 + 30, f - 1]
    return [0, f // 2, f - 1]


def _stub_devices():
    GV._stub_devices()

    def cpu(x):
        return "cpu" if (x == "cuda" or (isinstance(x, torch.device) and x.type == "cuda")) else x

    for name in ("zeros", "ones", "linspace", "full"):
        fn = getattr(torch, name)
        setattr(torch, name, lambda *a, _fn=fn, **k: _fn(*a, **{key: cpu(v) for key, v in k.items()}))


def _load_helpers():
    """utils/vis_tools/helpers.py itself, loaded from its file, with splat2d = oracle.splat.splat2d_ref."""
    stubs = {"moviepy": {}, "moviepy.editor": {}, "plotly": {}, "plotly.graph_objects": {}, "plotly.colors": {}, "ray": {},
             "utils.splat2d_cuda": {"splat2d": OS.splat2d_ref}, "utils.laplacian_blending": {"LaplacianBlender": None}}
    for name, attrs in stubs.items():
        mod = types.ModuleType(name)
        mod.__dict__.update(attrs)
        mod.__getattr__ = lambda attr: (lambda *a, **k: None)
        sys.modules[name] = mod
    path = os.path.join(refimport.REFERENCE_ROOT, "utils", "vis_tools", "helpers.py")
    spec = importlib.util.spec_from_file_location("utils.vis_tools.helpers", path)
    helpers = importlib.util.module_from_spec(spec)
    sys.modules["utils.vis_tools.helpers"] = helpers
    spec.loader.exec_module(helpers)
    make_grid = helpers.make_grid

    def make_grid_range(*a, range=None, **k):    # the installed torchvision calls it value_range
        return make_grid(*a, value_range=range, **k)

    helpers.make_grid = make_grid_range
    return helpers


def _capture(vc):
    videos = {}
    vc.save_video = lambda frames, fps, out_path, **k: videos.__setitem__(os.path.basename(out_path),
                                                                          torch.from_numpy(np.stack(frames)))
    vc.save_image = lambda *a, **k: None
    return videos


def _congealed_points(pts, n):
    from models.spatial_transformers.spatial_transformer import SpatialTransformer as ST
    points = pts.unsqueeze(0).repeat(n, 1, 1)
    return points, ST.normalize(points, GV.RES, GV.RESOLUTION), ST.convert(points, GV.RESOLUTION, GV.RES).round().long()


def ref_videos(vc, ref_t, data, pts, colors, alpha, stages, stage_flip, length, flip_length, iters):
    """smoothly_congeal_and_propagate (:208-298) on the reference's functions: -> {video name: (F, H, W, 3) uint8}."""
    args = GV._args(iters=iters, label_path="label", objects=True, output_resolution=GV.RES, flow_size=STN_KW["flow_size"],
                    resolution=GV.RESOLUTION, vis_in_stages=stages, stage_flip=stage_flip, length=length,
                    flip_length=flip_length, sigma=SIGMA, opacity=OPACITY, splat_batch=100, fps=60, out="visuals")

    def sample_images_and_points(args, t, classifier, device):     # :33-56 on `data` instead of a dataset
        data_flipped, flip_indices, warp_policy = vc.determine_flips(args, t, classifier, data, cluster=args.cluster)
        _, normalized, points = _congealed_points(pts, data.size(0))
        return data, data_flipped, flip_indices, warp_policy, points, normalized, colors, alpha

    vc.sample_images_and_points = sample_images_and_points
    videos = _capture(vc)
    vc.smoothly_congeal_and_propagate(args, ref_t, None)
    return {"congealing": videos["smoothly_congeal.mp4"], "propagation": videos["smoothly_propagate.mp4"],
            "correspondence": videos["smooth_correspondence.mp4"]}


def ref_average(vc, ref_t, batches, pts, colors, alpha, stages, stage_flip, length, flip_length, iters, n_mean):
    """average_and_congeal (:384-437) with its labelled tail: -> (F, R, R, 3) uint8."""
    args = GV._args(iters=iters, n_mean=n_mean, stage_flip=stage_flip, vis_in_stages=stages, length=length,
                    flip_length=flip_length, output_resolution=GV.RES, real_data_path=None, real_size=GV.SIZE,
                    distributed=False, label_path="label", objects=True, sigma=SIGMA, opacity=OPACITY, fps=60,
                    out="visuals")
    vc.img_dataloader = lambda *a, **k: batches
    _, _, points = _congealed_points(pts, GV.N)
    vc.sample_images_and_points = lambda *a, **k: (None, None, None, None, points, None, colors, alpha)
    videos = _capture(vc)
    vc.average_and_congeal(args, ref_t, None)
    return videos["smoothly_average.mp4"]


def _store(out, name, video, frames, counts):
    kept = kept_frames(video, counts)
    out["%s.%s.kept" % (name, video)] = frames[kept]
    out["%s.%s.sums" % (name, video)] = frames.long().sum((1, 2))


@torch.no_grad()
def gen_label_propagation():
    refimport.import_reference()
    _stub_devices()
    _load_helpers()
    _stub_modules()
    GV._load_training_vis()
    from models.spatial_transformers.spatial_transformer import get_stn
    from applications import vis_correspondence as vc
    ref_t = make_stn(get_stn)
    pts = GV.label_points()
    colors, alpha = label_colors()
    out = {"colors": colors, "alpha": alpha}
    for name, smooth, n, with_alpha in LABEL_CASES:
        _, stages, stage_flip, length, flip_length, iters, seed = GV.SMOOTH_CASES[smooth]
        data = GV.case_batches(seed, 1)[0][:n]
        videos = ref_videos(vc, ref_t, data, pts, colors, alpha if with_alpha else torch.ones_like(alpha), stages,
                            stage_flip, length, flip_length, iters)
        counts = {k: v.size(0) for k, v in videos.items()}
        print("%s: %s" % (name, {k: tuple(v.shape) for k, v in videos.items()}))
        out[name + ".cfg"] = torch.tensor([smooth, n, int(with_alpha)])
        for video in VIDEOS:
            _store(out, name, video, videos[video], counts)
    name, avg, with_alpha = AVERAGE_CASE
    _, stages, stage_flip, length, flip_length, iters, n_mean, seed = GV.AVG_CASES[avg]
    frames = ref_average(vc, ref_t, GV.case_batches(seed), pts, colors, alpha if with_alpha else torch.ones_like(alpha),
                         stages, stage_flip, length, flip_length, iters, n_mean)
    print("%s: %s" % (name, tuple(frames.shape)))
    out[name + ".cfg"] = torch.tensor([avg, int(with_alpha)])
    out[name + ".kept"] = frames[[frames.size(0) - 126, frames.size(0) - 35, frames.size(0) - 1]]
    out[name + ".sums"] = frames.long().sum((1, 2))
    _save("label_propagation", **out)


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen_label_propagation()
