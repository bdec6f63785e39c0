"""Generate tests/golden/congeal_dataset.npz from the reference's congeal_dataset.py.

Run where the reference checkout is (GG_REFERENCE_ROOT):  python -m oracle.make_golden_congeal
The reference's own apply_congealing and write_image_batch run on CPU on a seeded similarity -> flow STN (flow size 64,
weights of the other fixtures' seed; the similarity head's layer re-centred and its spread widened by tune_head so that
the scales and shifts vary, and stored) over ten seeded images of
varied sizes: landscape, portrait and square, odd and even padding, smaller than the flow size (Lanczos upsampling) and
up to 600 pixels, and sizes whose letterbox skips one resampling pass.  prepare_data's imports (lmdb, pandas, cv2,
utils.download) are stubbed, Image.ANTIALIAS is Pillow's LANCZOS (the name Pillow 10 removed), and the script's
hard-coded 'cuda' is sent to the CPU with make_golden_labels' stubs.  Stored per case (iters 1 and 3): the images, the
used indices, every image's flip, scale and out-of-bounds flag, and the PNGs write_image_batch wrote, read back.
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refimport  # noqa: E402
from oracle import opset  # noqa: E402
from oracle.make_golden import _save  # noqa: E402
from oracle.make_golden_pck import WEIGHT_SEED  # noqa: E402
from oracle import make_golden_labels as GL  # noqa: E402

WEIGHT_GAIN = 0.6
HEAD_TARGET = (0.0, -0.35, 0.0, 0.0)   # rotation, log scale, x and y shift the tuned head regresses on average
HEAD_SPREAD = 3.0
STN_KW = dict(flow_size=64, supersize=64, channel_multiplier=0.25, num_heads=1)
OUTPUT_RESOLUTION = 64
MIN_EFFECTIVE_RESOLUTION = 60
SIZES = [(48, 80), (90, 37), (64, 64), (33, 64), (64, 41), (300, 331), (600, 563), (257, 257), (121, 500), (17, 20),
         (130, 117), (200, 190)]
CASES = [("iters1", 1), ("iters3", 3)]


def make_stn(get_stn, **kw):
    return opset.fill_parameters(get_stn(["similarity", "flow"], **{**STN_KW, **kw}).eval(), WEIGHT_SEED, gain=WEIGHT_GAIN)


def tune_head(t, x_in):
    """(weight, bias) of the similarity head's linear layer that regress HEAD_TARGET on average over the batch x_in and
    HEAD_SPREAD times the seeded weights' spread around it: seeded weights alone shift every image past the border."""
    head = t.stns[0].warp_head.linear
    seen = []
    handle = head.register_forward_hook(lambda m, inp, out: seen.append(out.detach().clone()))
    t.stns[0](x_in)
    handle.remove()
    params = seen[0] - head.bias
    weight = head.weight.detach() * HEAD_SPREAD
    bias = torch.tensor(HEAD_TARGET, device=params.device) - HEAD_SPREAD * params.mean(0)
    return weight, bias


def set_head(t, weight, bias):
    with torch.no_grad():
        t.stns[0].warp_head.linear.weight.copy_(weight)
        t.stns[0].warp_head.linear.bias.copy_(bias)
    return t


def case_images(seed=5):
    """Smooth seeded uint8 (H, W, 3) images: bilinear noise from 8 x 8 (smooth images keep the fixture small)."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for h, w in SIZES:
        low = torch.rand(1, 3, 8, 8, generator=g) * 255
        img = F.interpolate(low, size=(h, w), mode="bilinear", align_corners=False)[0].permute(1, 2, 0)
        out.append(img.round().clamp(0, 255).to(torch.uint8))
    return out


def _stub_prepare_data():
    from PIL import Image
    Image.ANTIALIAS = Image.LANCZOS
    for name in ("lmdb", "pandas", "cv2", "utils.download", "tqdm"):
        mod = types.ModuleType(name)
        mod.__getattr__ = lambda attr: (lambda *a, **k: None)
        sys.modules[name] = mod
    sys.modules["tqdm"].tqdm = lambda x, *a, **k: x


@torch.no_grad()
def gen_congeal():
    from PIL import Image
    refimport.import_reference()
    _stub_prepare_data()
    GL._stub_devices()
    from models.spatial_transformers.spatial_transformer import get_stn
    from applications import congeal_dataset as cd
    ref_t = make_stn(get_stn)
    t_sim = ref_t.stns[0]
    images = case_images()
    dataset = [Image.fromarray(img.numpy()) for img in images]
    from oracle.congeal import letterbox_ref
    weight, bias = tune_head(ref_t, letterbox_ref(images, STN_KW["flow_size"]))
    set_head(ref_t, weight, bias)
    out = {"sizes": torch.tensor(SIZES), "cfg": torch.tensor([OUTPUT_RESOLUTION, MIN_EFFECTIVE_RESOLUTION]),
           "head_weight": weight, "head_bias": bias}
    for k, img in enumerate(images):
        out["image%d" % k] = img
    for name, iters in CASES:
        rec = {"flips": [], "M": [], "oob": []}
        determine = cd.determine_flips

        def determine_flips(*a, _d=determine, **k):
            res = _d(*a, **k)
            rec["flips"].append(res[1].flatten().clone())
            return res

        def stn(*a, **k):
            res = t_sim(*a, **k)
            rec["M"].append(res[1].clone())
            rec["oob"].append(res[2].clone())
            return res

        cd.determine_flips = determine_flips
        args = types.SimpleNamespace(flow_size=STN_KW["flow_size"], output_resolution=OUTPUT_RESOLUTION,
                                     min_effective_resolution=MIN_EFFECTIVE_RESOLUTION, no_flip_inference=False,
                                     padding_mode="border", iters=iters, num_heads=1)
        with tempfile.TemporaryDirectory() as tmp:
            used = cd.apply_congealing(args, dataset, stn, ref_t, tmp, "cpu", 0, 1, iters=iters, padding_mode="border")
            pngs = sorted(f for f in os.listdir(tmp) if f.endswith(".png"))
            written = torch.stack([torch.from_numpy(np.asarray(Image.open(os.path.join(tmp, f))).copy()) for f in pngs])
        cd.determine_flips = determine
        one_hot = torch.tensor([[[0.0, 0.0, 1.0]]])
        scale = torch.cat([torch.det(torch.cat([m, one_hot], 1)).sqrt_() for m in rec["M"]])
        oob = torch.cat(rec["oob"]).flatten()
        flips = torch.cat(rec["flips"])
        too_low = torch.tensor([s * min(w, h) < MIN_EFFECTIVE_RESOLUTION for s, (h, w) in zip(scale.tolist(), SIZES)])
        assert bool(too_low.any()) and bool(oob.any()), "both filters must reject an image (%s, %s)" % (too_low, oob)
        out[name + ".used"] = used
        out[name + ".flips"] = flips
        out[name + ".scale"] = scale
        out[name + ".oob"] = oob
        out[name + ".pngs"] = written
        print("%s: used %s, flips %s, scale %s, oob %s, too low %s" % (name, used.tolist(), flips.int().tolist(),
                                                                    [round(s, 3) for s in scale.tolist()],
                                                                    oob.int().tolist(), too_low.int().tolist()))
    _save("congeal_dataset", **out)


if __name__ == "__main__":
    torch.set_num_threads(8)
    gen_congeal()
