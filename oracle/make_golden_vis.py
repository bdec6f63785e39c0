"""Generate tests/golden/congealing_vis.npz from the reference's congealing visualisations and pin oracle/vis.py against it.

Run where the reference checkout is (GG_REFERENCE_ROOT):  python -m oracle.make_golden_vis
The reference's own create_average_image (the average-image animation, frame by frame), smoothly_sample_image (the
congealing animation with its points, forward and reverse) and propagate_to_images.average's STN calls run on CPU on
make_golden_pck's seeded similarity -> flow STN (flow 64, supersize 128) at output resolution 96 (neither the flow size
nor a tile multiple).  Their device moves ('cuda') and the vis-only modules (video / image writing) are stubbed here, and
only here.  The oracle's per-frame compositions on the mirror STN must reproduce every result.  Stored: the seeds, the label
points, the average-image frames, a subset of the congealing frames, every frame's per-channel sums, and the points.
"""
import math
import os
import sys
import types

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refimport  # noqa: E402
from oracle import vis as OV  # noqa: E402
from oracle.make_golden import _save  # noqa: E402
from oracle.make_golden_pck import STN_KW, WEIGHT_GAIN, WEIGHT_SEED, _stub_modules, make_stn  # noqa: E402

SIZE, N, RES, P, RESOLUTION = 128, 4, 96, 40, 64
AVG_CASES = [   # name, vis_in_stages, stage_flip, length, flip_length, iters, n_mean, image seed
    ("avg_stages_flip", True, True, 6, 4, 1, 8, 31),
    ("avg_final_iters3", False, False, 6, 4, 3, 8, 32),
]
SMOOTH_CASES = [   # name, vis_in_stages, stage_flip, length, flip_length, iters, image seed
    ("smooth_stages_flip", True, True, 60, 4, 1, 41),
    ("smooth_final_iters3", False, False, 60, 4, 3, 42),
]
MEAN_CASE = ("average", 6, 1, 51)   # name, n_mean (batches of 4: the reference averages 8), iters, image seed
KEPT_FRAMES = [0, 3, 30, 63, 64, 90, 123]


def tolerance(iters):
    """Relative tolerance of results that go through the mirror STN against the reference's.  The two STNs round their
    convolutions in different orders (~1e-7 of a grid coordinate); with iters > 1 the similarity STN warps its own output
    again, and the difference compounds: 1e-5 for one pass, 5e-5 for three (measured: 2.5e-5)."""
    return 1e-5 if iters == 1 else 5e-5


def case_batches(seed, n_batches=2):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(N, 3, SIZE, SIZE, generator=g) for _ in range(n_batches)]


def label_points(seed=7):
    """(P, 2) integer label pixels at RESOLUTION, the first eight on the border so that windows leave the padded grid."""
    g = torch.Generator().manual_seed(seed)
    pts = torch.randint(0, RESOLUTION, (P, 2), generator=g)
    edge = torch.tensor([[0, 0], [RESOLUTION - 1, 0], [0, RESOLUTION - 1], [RESOLUTION - 1, RESOLUTION - 1],
                         [0, 20], [RESOLUTION - 1, 33], [17, 0], [40, RESOLUTION - 1]])
    pts[:8] = edge
    return pts


def _stub_devices():
    to = torch.Tensor.to

    def cpu(x):
        return "cpu" if (x == "cuda" or (isinstance(x, torch.device) and x.type == "cuda")) else x

    torch.Tensor.to = lambda self, *a, **k: to(self, *[cpu(x) for x in a], **{key: cpu(v) for key, v in k.items()})
    torch.Tensor.cuda = lambda self, *a, **k: self
    tensor = torch.tensor
    torch.tensor = lambda *a, **k: tensor(*a, **{key: cpu(v) for key, v in k.items()})
    torch.nn.Module.to = lambda self, *a, **k: self


def _load_training_vis():
    """utils/vis_tools/training_vis.py itself (run_loader_mean), its package stubbed: loaded from its file, with the
    tensorboard writer and flow colouring it imports stubbed."""
    import importlib.util
    for name in ("utils.vis_tools.flow_vis", "torch.utils.tensorboard"):
        if name not in sys.modules:
            mod = types.ModuleType(name)
            mod.__getattr__ = lambda attr: type(attr, (), {"__init__": lambda self, *a, **k: None})
            sys.modules[name] = mod
    path = os.path.join(refimport.REFERENCE_ROOT, "utils", "vis_tools", "training_vis.py")
    spec = importlib.util.spec_from_file_location("utils.vis_tools.training_vis", path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules["utils.vis_tools.training_vis"] = mod
    spec.loader.exec_module(mod)


def _args(**kw):
    base = dict(cluster=None, num_heads=1, no_flip_inference=False, padding_mode="border", batch=N)
    base.update(kw)
    return types.SimpleNamespace(**base)


def _close(got, want, what, tol=1e-5, scale=None):
    """Relative error.  Averages (scale = the images' magnitude): the largest difference over scale.  Frames: the norm of
    the difference over the norm of `want`, and every difference within 10 tol of its magnitude -- the two STNs compute
    the grids in different orders, so a pixel where the image is steep may move by more than the norm."""
    d = got.double() - want.double()
    if scale is not None:
        err = (d.abs().max() / scale).item()
        ok = err <= tol
    else:
        err = (d.norm() / want.double().norm().clamp_min(1e-12)).item()
        ok = err <= tol and (d.abs().max() / want.double().abs().max().clamp_min(1e-12)).item() <= 10 * tol
    assert ok, "%s: rel err %.3e > %.0e" % (what, err, tol)
    return err


@torch.inference_mode()
def ref_smooth(vc, ref_t, data, pts, vis_in_stages, stage_flip, length, flip_length, iters):
    """smoothly_congeal_and_propagate (:208-298) without its video writing, on the reference's own functions."""
    from models.spatial_transformers.antialiased_sampling import MipmapWarp
    from models.spatial_transformers.spatial_transformer import SpatialTransformer as ST
    args = _args(iters=iters)
    data_flipped, flip_indices, warp_policy = vc.determine_flips(args, ref_t, None, data, cluster=None)
    points = pts.unsqueeze(0).repeat(data.size(0), 1, 1)
    points_normalized = ST.normalize(points, RES, RESOLUTION)
    points = ST.convert(points, RESOLUTION, RES).round().long()
    _, grids = ref_t(data_flipped, return_intermediates=True, warp_policy=warp_policy, padding_mode="border", iters=iters)
    if not vis_in_stages:
        grids = [grids[-1]]
    grids = vc.flip_grid(torch.stack(grids), flip_indices.view(1, -1, 1, 1))
    fs = STN_KW["flow_size"]
    grids = grids.reshape(-1, fs, fs, 2)
    grids = F.interpolate(grids.permute(0, 3, 1, 2), scale_factor=RES / fs, mode="bilinear").permute(0, 2, 3, 1)
    grids = grids.reshape(-1, data.size(0), RES, RES, 2)
    identity_grid = F.affine_grid(torch.eye(2, 3).unsqueeze(0).repeat(data.size(0), 1, 1), (data.size(0), 3, RES, RES))
    num_stages = grids.size(0)
    flipping_grid = vc.flip_grid(identity_grid, flip_indices)
    grids = torch.cat([flipping_grid.unsqueeze(0), grids], 0)
    warper = MipmapWarp(3.5)
    full_grid = grids[-1]
    nua = F.grid_sample(full_grid.permute(0, 3, 1, 2), points_normalized.unsqueeze(2).float(),
                        padding_mode="border").squeeze(3).permute(0, 2, 1)
    unaligned = ST.unnormalize(nua, RES, RES)
    centers = unaligned.round().long().clamp(0, RES - 1)
    centers[..., 0] = torch.where(flip_indices.view(-1, 1), RES - 1 - centers[..., 0], centers[..., 0])
    congealed_centers = points
    images, propagated = [], []
    if stage_flip:
        images.append(vc.smoothly_sample_image(flipping_grid, identity_grid, warper, data, flip_length, 2)[2])
    for i in range(num_stages):
        _, pp, im, centers = vc.smoothly_sample_image(grids[i + 1], grids[i], warper, data, length, 2, nua, centers)
        propagated.append(pp)
        images.append(im)
    for i in range(num_stages):
        alpha = torch.linspace(0, 1, steps=length).view(length, 1, 1, 1)
        _, rev, _, congealed_centers = vc.smoothly_sample_image(grids[-i - 2], grids[-i - 1], warper, data, length, 2, nua,
                                                                congealed_centers)
        propagated[-i - 1].lerp_(rev.flip(0), alpha)
    return torch.cat(images, 0), torch.cat(propagated, 0), unaligned, flip_indices.flatten()


@torch.no_grad()
def gen_congealing_vis():
    refimport.import_reference()
    _stub_devices()
    _stub_modules()
    _load_training_vis()
    from models.spatial_transformers.antialiased_sampling import MipmapWarp
    from models.spatial_transformers.spatial_transformer import get_stn
    from applications import vis_correspondence as vc
    from applications import propagate_to_images as pti
    from gangealing_b200.stn import get_stn as mirror_get_stn
    from oracle import opset
    ref_t = make_stn(get_stn)
    mirror = opset.fill_parameters(mirror_get_stn(["similarity", "flow"], ops=OV.cpu_ops(), **STN_KW).eval(), WEIGHT_SEED,
                                   gain=WEIGHT_GAIN)
    out = {"label_points": label_points(), "kept_frames": torch.tensor(KEPT_FRAMES)}
    flips_seen = set()
    name, n_mean, iters, seed = MEAN_CASE
    batches = case_batches(seed)
    args = _args(iters=iters, n_mean=n_mean, output_resolution=RES, real_data_path=None, real_size=SIZE,
                 distributed=False, out="visuals")
    captured = {}
    pti.save_image = lambda img, *a, **k: captured.setdefault("avg", img)
    pti.img_dataloader = lambda *a, **k: batches
    pti.args = args
    pti.average(args, ref_t, None)
    want = captured["avg"]
    err = _close(OV.average_ref(mirror, batches, n_mean, RES, iters), want, "average image", tolerance(iters),
                 scale=torch.stack(batches).abs().max())
    print("%s: oracle rel err %.1e" % (name, err))
    out[name + ".cfg"] = torch.tensor([n_mean, iters, seed])
    out[name + ".image"] = want
    for ci, (name, stages, stage_flip, length, flip_length, iters, n_mean, seed) in enumerate(AVG_CASES):
        batches = case_batches(seed)
        args = _args(iters=iters, n_mean=n_mean, stage_flip=stage_flip)
        identity_grid = F.affine_grid(torch.eye(2, 3).unsqueeze(0), (1, 3, RES, RES))
        warper = MipmapWarp(3.5)
        num_stages = (len(ref_t.stns) if stages else 1) + int(stage_flip)
        frames = []
        for i in range(num_stages):     # average_and_congeal (:403-417)
            n_frames = length if not stage_flip or i > 0 else flip_length
            for frame_ix in range(n_frames):
                alpha = 1 - 0.5 * (1 + torch.cos(torch.tensor(math.pi * frame_ix / (n_frames - 1))))
                frames.append(vc.create_average_image(args, ref_t, None, batches, warper, alpha, warp_index=i - int(stage_flip),
                                                      identity_grid=identity_grid, flip=(i == 0) and stage_flip, iters=iters,
                                                      output_resolution=RES, padding_mode="border"))
        frames = torch.stack(frames, 0)
        mine = OV.average_frames_ref(mirror, batches, n_mean, length, flip_length, stages, stage_flip, RES, iters)
        err = _close(mine, frames, name + " frames", tolerance(iters), scale=torch.stack(batches).abs().max())
        print("%s: oracle rel err %.1e" % (name, err))
        for b in batches:
            flips_seen.update(vc.determine_flips(args, ref_t, None, b)[1].flatten().tolist())
        out[name + ".cfg"] = torch.tensor([int(stages), int(stage_flip), length, flip_length, iters, n_mean, seed])
        out[name + ".frames"] = frames
    pts = out["label_points"]
    for name, stages, stage_flip, length, flip_length, iters, seed in SMOOTH_CASES:
        data = case_batches(seed, 1)[0]
        images, points, unaligned, flips = ref_smooth(vc, ref_t, data, pts, stages, stage_flip, length, flip_length, iters)
        flips_seen.update(flips.tolist())
        o_images, o_points, o_unaligned = OV.smooth_congealing_ref(mirror, data, pts, RESOLUTION, length, flip_length, stages,
                                                                   stage_flip, RES, iters)
        err = _close(o_images, images, name + " frames", tolerance(iters))
        _close(o_unaligned, unaligned, name + " unaligned points", tolerance(iters))
        # the mirror STN's grids differ from the reference's by rounding, so a near-tie of the window search can go the
        # other way and move that point's later frames; at most 1 % of the (frame, image, point) positions may differ
        differ = int((o_points != points).any(-1).sum())
        assert differ <= 0.01 * points[..., 0].numel(), "%s: %d tracked points differ from the reference" % (name, differ)
        print("%s: frames rel err %.1e, %d of %d tracked positions differ" % (name, err, differ, points[..., 0].numel()))
        kept = [f for f in KEPT_FRAMES if f < images.size(0)]
        out[name + ".cfg"] = torch.tensor([int(stages), int(stage_flip), length, flip_length, iters, seed])
        out[name + ".frames_kept"] = images[kept, :2]
        out[name + ".frame_sums"] = images.double().sum((3, 4))
        out[name + ".points"] = points
        out[name + ".unaligned"] = unaligned
        out[name + ".flips"] = flips
    assert flips_seen == {False, True}, "the fixture must see both flip outcomes (got %s)" % sorted(flips_seen)
    _save("congealing_vis", **out)


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen_congealing_vis()
