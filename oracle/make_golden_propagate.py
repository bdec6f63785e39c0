"""Generate tests/golden/propagate_to_images.npz from the reference's propagate_to_images.py.

Run where the reference checkout is (GG_REFERENCE_ROOT):  python -m oracle.make_golden_propagate
The reference's own make_visuals (with vis_correspondence.sample_images_and_points and helpers.load_dense_label) and
average run on CPU on a seeded similarity -> flow STN with flow size 128 and images of 256 (so the congealed images'
grid is resized from the lookup's), with the stubs of make_golden_labels.py.  The dataset is the case's images; the
Plotly colour scale of a label loaded without --objects is replaced by seeded colours, which are stored.  save_image is
captured: it writes the PNG with torchvision's own save_image (its `range=` passed on as `value_range=`), and the PNG
is read back.  Stored per case: the label PNG, the loader's points / colours / alpha, the flips, the correspondences
and every grid PNG; with n_mean, average.png and the annotated average.
"""
import os
import sys
import tempfile

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refimport  # noqa: E402
from oracle import opset  # noqa: E402
from oracle.make_golden import _save  # noqa: E402
from oracle.make_golden_pck import WEIGHT_GAIN, WEIGHT_SEED, _stub_modules  # noqa: E402
from oracle import make_golden_labels as GL  # noqa: E402
from oracle import make_golden_vis as GV  # noqa: E402

STN_KW = dict(flow_size=128, supersize=256, channel_multiplier=0.25, num_heads=1)
SIZE, SIGMA, OPACITY = 256, 1.3, 0.75
CASES = [   # name, images, image seed, --objects, iters, label --resolution, label PNG size, n_mean (-1: no average)
    ("objects_average", 4, 61, True, 1, 64, 64, 8),
    ("plain_iters3", 3, 62, False, 3, 96, 80, -1),
]
GRIDS = ("input_images", "congealed_images", "propagated", "average_annotated")


def make_stn(get_stn, **kw):
    return opset.fill_parameters(get_stn(["similarity", "flow"], **STN_KW, **kw).eval(), WEIGHT_SEED, gain=WEIGHT_GAIN)


def case_images(seed, n):
    """Smooth seeded images in [-1, 1]-ish: bilinear 16 -> 256 noise (smooth fields keep the fixture small)."""
    g = torch.Generator().manual_seed(seed)
    low = torch.randn(n, 3, 16, 16, generator=g) * 0.8
    return F.interpolate(low, size=(SIZE, SIZE), mode="bilinear", align_corners=False)


def label_png(seed, size):
    """(size, size, 4) uint8 RGBA label: an ellipse and a bar with random alpha (some pixels fully transparent inside)."""
    g = torch.Generator().manual_seed(seed)
    ys, xs = torch.meshgrid(torch.arange(size).float(), torch.arange(size).float(), indexing="ij")
    c = (size - 1) / 2
    inside = ((xs - c) / (0.38 * size)) ** 2 + ((ys - 0.45 * size) / (0.3 * size)) ** 2 <= 1
    inside |= (ys > 0.8 * size) & (ys < 0.88 * size) & (xs > 0.1 * size)
    rgba = torch.randint(0, 256, (size, size, 4), generator=g, dtype=torch.int64)
    for ch in range(3):   # smooth colour ramps (a small fixture); the alpha stays random
        rgba[..., ch] = ((xs * (2 + ch) + ys * (5 - ch) + 60 * ch) % 256).long()
    rgba[..., 3] = torch.where(inside, rgba[..., 3].clamp_min(1), torch.zeros_like(rgba[..., 3]))
    rgba[..., 3][::7, ::5] = 0
    return rgba.to(torch.uint8)


def plotly_colors(p, seed=13):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(1, p, 3, generator=g) * 2 - 1


@torch.no_grad()
def gen_propagate():
    from PIL import Image
    import torchvision.utils as tvu
    refimport.import_reference()
    GL._stub_devices()
    helpers = GL._load_helpers()
    _stub_modules()
    GV._load_training_vis()
    from models.spatial_transformers.spatial_transformer import get_stn
    from applications import vis_correspondence as vc
    from applications import propagate_to_images as pti
    ref_t = make_stn(get_stn)
    written = {}

    def save_image(img, path, range=None, **k):      # torchvision's save_image, `range` spelled as it is today
        tvu.save_image(img, path, value_range=range, **k)
        written[os.path.basename(path)] = np.asarray(Image.open(path))

    pti.save_image = save_image
    out = {}
    flips_seen = set()
    for name, n, seed, objects, iters, resolution, png_size, n_mean in CASES:
        data = case_images(seed, n)
        with tempfile.TemporaryDirectory() as tmp:
            label = label_png(seed + 100, png_size)
            label_path = os.path.join(tmp, "label.png")
            Image.fromarray(label.numpy()).save(label_path)
            args = GV._args(iters=iters, n_mean=n_mean, output_resolution=SIZE, real_data_path=None, real_size=SIZE,
                            distributed=False, out=tmp, label_path=label_path, objects=objects, resolution=resolution,
                            sigma=SIGMA, opacity=OPACITY, dset_indices=list(range(n)), flow_scores=None,
                            save_individual_images=False, average_path=None)
            vc.MultiResolutionDataset = lambda *a, **k: list(data)
            pti.args = args
            loaded = helpers.load_dense_label(label_path, resolution=resolution, load_colors=objects)
            colors = loaded[1] if objects else plotly_colors(loaded[0].size(1))
            helpers.get_plotly_colors = lambda num_points, colorscale, _c=colors: _c
            flips = {}
            determine = vc.determine_flips

            def determine_flips(*a, _d=determine, **k):
                res = _d(*a, **k)
                flips["f"] = res[1].flatten().clone()
                return res

            vc.determine_flips = determine_flips
            uncongeal = ref_t.uncongeal_points
            ref_t.uncongeal_points = lambda *a, _u=uncongeal, **k: flips.__setitem__("u", _u(*a, **k)) or flips["u"]
            written.clear()
            if n_mean > 0:
                pti.img_dataloader = lambda *a, **k: [case_images(seed + 1000 + i, 4) for i in range(3)]
                pti.average(args, ref_t, None)
            pti.make_visuals(args, ref_t, None)
            vc.determine_flips = determine
            del ref_t.uncongeal_points
        upoints = flips["u"]    # the script mirrors these in place (:67-69)
        flips_seen.update(flips["f"].tolist())
        out[name + ".cfg"] = torch.tensor([n, seed, int(objects), iters, resolution, png_size, n_mean])
        out[name + ".label"] = label
        out[name + ".label_points"] = loaded[0]
        out[name + ".label_alpha"] = loaded[2]
        out[name + ".colors"] = colors
        if objects:
            out[name + ".label_colors"] = loaded[1]
        out[name + ".flips"] = flips["f"]
        out[name + ".correspondences"] = upoints
        for g in GRIDS:
            if g + "_grid.png" in written:
                out[name + "." + g] = torch.from_numpy(written[g + "_grid.png"].copy())
        if "average.png" in written:
            out[name + ".average_png"] = torch.from_numpy(written["average.png"].copy())
        print("%s: flips %s, %d label points, grids %s" % (name, flips["f"].tolist(), loaded[0].size(1),
                                                          sorted(k for k in written)))
    assert flips_seen == {False, True}, "the fixture must see both flip outcomes (got %s)" % sorted(flips_seen)
    _save("propagate_to_images", **out)


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen_propagate()
