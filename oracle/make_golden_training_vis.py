"""Generate tests/golden/training_vis.npz from the reference's own training visuals.

Run where the reference checkout is (GG_REFERENCE_ROOT):  python -m oracle.make_golden_training_vis
The reference's create_training_visuals, create_training_cluster_visuals and create_training_cluster_classifier_visuals
(utils/vis_tools/training_vis.py, with its real flow_vis.py) run on CPU on make_golden.classifier_setup's seeded generator
(128²), similarity -> flow STN (flow 64), latent learner and cluster classifier, loaded the same way into both trees, with
make_golden's per-sample MSE as the assignment loss.  GANgealingWriter._log_image_grid's arrays are captured instead of
written (images2grid with its make_grid `range=` passed on as torchvision's `value_range=`), and the reference's devices
are stubbed as make_golden_labels.py stubs them.  The assignments of every generate_cluster_congeal batch and their
per-slot losses are captured too.  Cases: K = 1 (n_mean 7 over batches of 3: 9 real images used), K = 2 with flips (7
fakes in batches of 3: a cluster gets fewer than n_sample = 4) and the classifier's real-image visuals.  Stored: every
grid's per-channel sums, the grids at the STN's size, the 128² grids decimated, and the assignments.  The generator's
noise comes from the global RNG, seeded with NOISE_SEED before each case.
"""
import importlib.util
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refimport  # noqa: E402
from oracle.make_golden import _mse, _save, classifier_setup  # noqa: E402

N_SAMPLE, PSI, PADDING = 4, 0.5, "reflection"
NOISE_SEED = 77      # torch.manual_seed before each case: the generator draws its noise from the global RNG
CASES = [   # name, K, flips, n_mean, vis_batch_size (train.py divides it by K), kind
    ("unimodal", 1, False, 7, 6, "training"),
    ("cluster", 2, True, 7, 6, "training"),
    ("classifier", 2, True, 5, 6, "classifier"),
]
GEN_SIZE_GRIDS = ("sample", "truncated_sample")      # 128² images: stored decimated


def inputs(seed=5, dim_latent=512, size=128):
    """z (N_SAMPLE latents), big_z (7 latents), reals (N_SAMPLE images) and three real batches of 3 images."""
    g = torch.Generator().manual_seed(seed)
    z, big_z = torch.randn(N_SAMPLE, dim_latent, generator=g), torch.randn(7, dim_latent, generator=g)
    reals = torch.randn(N_SAMPLE, 3, size, size, generator=g)
    loader = [torch.randn(3, 3, size, size, generator=g) for _ in range(3)]
    return z, big_z, reals, loader


def decimate(name, grid):
    return grid[::4, ::4] if name in GEN_SIZE_GRIDS else grid


def _load_file(name, *parts):
    path = os.path.join(refimport.REFERENCE_ROOT, *parts)
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def _reference():
    from oracle import make_golden_labels as GL
    from oracle import make_golden_pck as GP
    from oracle import make_golden_vis as GV
    refimport.import_reference()
    GL._stub_devices()
    helpers = GL._load_helpers()
    make_grid = helpers.make_grid

    def make_grid_no_pil(*a, return_as_PIL=None, **k):    # the writer's return_as_PIL is not a make_grid argument
        return make_grid(*a, **k)

    helpers.make_grid = make_grid_no_pil
    GP._stub_modules()
    _load_file("utils.vis_tools.flow_vis", "utils", "vis_tools", "flow_vis.py")
    GV._load_training_vis()
    return sys.modules["utils.vis_tools.training_vis"]


def _writer(tv, grids):
    w = tv.GANgealingWriter.__new__(tv.GANgealingWriter)
    helpers = sys.modules["utils.vis_tools.helpers"]

    def log(images, logging_name, prefix, itr, range=(-1, 1), scale_each=False):   # _log_image_grid without the file
        nrow = max(1, int(images.size(0) ** 0.5))
        grids[logging_name] = torch.from_numpy(helpers.images2grid(images, nrow=nrow, padding=2, pad_value=0, normalize=True,
                                                                    range=range, scale_each=scale_each))

    w._log_image_grid = log
    return w


def _capture_assignments(tv, record):
    assign = tv.assign_fake_images_to_clusters

    def wrapped(*a, **k):
        out = assign(*a, **k)
        record.append((out[0].indices.clone(), out[5].clone()))
        return out

    tv.assign_fake_images_to_clusters = wrapped


@torch.no_grad()
def gen_training_vis():
    tv = _reference()
    from models import ResnetClassifier
    from models.latent_learner import DirectionInterpolator
    from models.spatial_transformers.antialiased_sampling import BilinearDownsample
    from models.spatial_transformers.spatial_transformer import get_stn
    from models.stylegan2.networks import Generator
    mods = dict(Generator=Generator, get_stn=get_stn, DirectionInterpolator=DirectionInterpolator,
                ResnetClassifier=ResnetClassifier, BilinearDownsample=BilinearDownsample)
    record = []
    _capture_assignments(tv, record)
    out = {}
    for name, k, flips, n_mean, vb, kind in CASES:
        g, stn, ll, cls, resize, _ = classifier_setup(mods, heads=k, flips=flips)
        z, big_z, reals, loader = inputs()
        grids = {}
        w = _writer(tv, grids)
        record.clear()
        torch.manual_seed(NOISE_SEED)
        if kind == "classifier":
            tv.create_training_cluster_classifier_visuals(stn, cls, loader, k, n_mean, N_SAMPLE, "cpu", 0, w,
                                                          padding_mode=PADDING)
        elif k > 1:
            tv.create_training_cluster_visuals(g, stn, ll, _mse, loader, resize, z, big_z, PSI, "cpu", n_mean, N_SAMPLE, k,
                                               flips, vb // k, 64, 0, w, padding_mode=PADDING)
        else:
            tv.create_training_visuals(g, stn, ll, loader, reals, resize, z, PSI, "cpu", n_mean, N_SAMPLE, 0, w,
                                       padding_mode=PADDING)
        out[name + ".names"] = torch.tensor([ord(c) for c in ",".join(sorted(grids))])
        for gname, grid in grids.items():
            out["%s.%s.sums" % (name, gname)] = grid.long().sum((0, 1))
            out["%s.%s.shape" % (name, gname)] = torch.tensor(grid.shape)
            out["%s.%s" % (name, gname)] = decimate(gname, grid)
        for i, (idx, dist) in enumerate(record):
            out["%s.assign%d" % (name, i)], out["%s.dist%d" % (name, i)] = idx, dist
        print("%s: %s, %d assignment batches" % (name, sorted(grids), len(record)))
    _save("training_vis", **out)


def grid_names(blob, case):
    return "".join(chr(c) for c in blob[case + ".names"].tolist()).split(",")


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen_training_vis()
