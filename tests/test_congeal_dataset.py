"""Dataset congealing (gangealing_b200.evaluation.congeal and the letterbox kernel, csrc/letterbox.cu) against the
reference fixture (oracle/make_golden_congeal.py), Pillow itself (oracle/congeal.py) and the reference's per-image
composition on the device.

The STN here and the reference's round their convolutions in different orders, and the flips are decided on the whole
batch rather than image by image, so an aligned value near a quantisation step may round the other way: at most 0.5 % of
the stored bytes may differ, each by 1 (by 2 at iters 3, where the similarity stage warps its own output again and the
rounding compounds)."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

from conftest import load_golden
from oracle import congeal as OC
from oracle import make_golden_congeal as GC
from oracle import opset
from vis_reference import fp32_stn

DEV = "cuda"
CASES = [c[0] for c in GC.CASES]
DIFFER_BOUND = 0.005


def _mirror(ops, blob=None, **kw):
    from gangealing_b200.stn import get_stn
    t = opset.fill_parameters(get_stn(["similarity", "flow"], ops=ops, **{**GC.STN_KW, **kw}).eval(), GC.WEIGHT_SEED,
                              gain=GC.WEIGHT_GAIN)
    if blob is not None:
        GC.set_head(t, blob["head_weight"], blob["head_bias"])
    return t


def _images(blob):
    return [blob["image%d" % k] for k in range(len(GC.SIZES))]


def _run(ops, blob, name, device="cpu"):
    from gangealing_b200.evaluation import congeal_images
    iters = dict(GC.CASES)[name]
    t = _mirror(ops, blob).to(device)
    return congeal_images(t, _images(blob), output_resolution=GC.OUTPUT_RESOLUTION,
                          min_effective_resolution=GC.MIN_EFFECTIVE_RESOLUTION, iters=iters)


def _check_fixture(blob, name, res, exact=False):
    """exact: every PNG byte equal (the CPU op set at iters 1, where the only rounding left is the convolutions' own)."""
    iters = dict(GC.CASES)[name]
    assert torch.equal(res["flips"], blob[name + ".flips"].bool()), (res["flips"], blob[name + ".flips"])
    assert res["keep"].nonzero().flatten().tolist() == blob[name + ".used"].tolist()
    assert torch.equal(res["out_of_bounds"], blob[name + ".oob"].bool())
    assert (res["scale"] - blob[name + ".scale"]).abs().max().item() <= 1e-4
    got, want = res["aligned"].cpu(), blob[name + ".pngs"]
    assert got.shape == want.shape and got.dtype == torch.uint8
    d = (got.int() - want.int()).abs()
    differ = int((d > 0).sum())
    step = 0 if exact else 1 if iters == 1 else 2
    assert int(d.max()) <= step and differ <= DIFFER_BOUND * want.numel(), "%s: %d of %d bytes differ (max %d)" % (
        name, differ, want.numel(), int(d.max()))
    print("%s: %d of %d PNG bytes differ from the reference" % (name, differ, want.numel()))


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", CASES)
def test_api_on_the_oracle_reproduces_the_reference_fixture(name):
    """congeal_images on oracle.congeal.cpu_ops(): the kept set, flips, scales, out-of-bounds flags and PNG bytes of the
    reference's apply_congealing + write_image_batch; at iters 1 every byte is equal."""
    blob = load_golden("congeal_dataset")
    _check_fixture(blob, name, _run(OC.cpu_ops(), blob, name), exact=dict(GC.CASES)[name] == 1)


def test_oracle_letterbox_is_border_pad_then_prepro():
    """The restatement is the script's own composition: a landscape, a portrait and a flip of the unresized square."""
    g = torch.Generator().manual_seed(3)
    for h, w in ((20, 33), (41, 17)):
        img = torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8)
        pil = Image.fromarray(img.numpy())
        want = OC.prepro(OC.border_pad(pil, 16))
        assert torch.equal(OC.letterbox_ref([img], 16), want)
        big = OC.prepro(OC.border_pad(pil, max(h, w), resize=False))
        assert torch.equal(OC.letterbox_ref([img], None, False, torch.tensor([True])), big.flip(3))


def test_refusals():
    """Clustering STNs, a non-similarity first stage, empty batches and images that are not (H, W, 3) uint8."""
    from gangealing_b200.evaluation import congeal_images
    from gangealing_b200.stn import get_stn
    ops = OC.cpu_ops()
    img = torch.zeros(20, 30, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="num_heads"):
        congeal_images(_mirror(ops, num_heads=2), [img])
    with pytest.raises(ValueError, match="similarity"):
        congeal_images(get_stn(["flow"], flow_size=64, supersize=64, channel_multiplier=0.25, ops=ops), [img])
    with pytest.raises(ValueError, match="no images"):
        congeal_images(_mirror(ops), [])
    for bad in (torch.zeros(20, 30, 4, dtype=torch.uint8), torch.zeros(20, 30, 3), np.zeros((20, 30), np.uint8)):
        with pytest.raises(ValueError, match="uint8"):
            congeal_images(_mirror(ops), [bad])


def _driver_worker(rank, world, ret):
    from gangealing_b200.evaluation import congeal_dataset
    blob = load_golden("congeal_dataset")
    images = _images(blob)
    dataset = [Image.fromarray(x.numpy()) if k % 2 else x.numpy() for k, x in enumerate(images)]  # PIL and arrays
    out = os.environ["GG_CONGEAL_OUT"]
    used = congeal_dataset(_mirror(OC.cpu_ops(), blob), dataset, out, batch=4, output_resolution=GC.OUTPUT_RESOLUTION,
                           min_effective_resolution=GC.MIN_EFFECTIVE_RESOLUTION)
    ret[rank] = used.tolist()


def test_driver_on_two_ranks(tmp_path):
    """congeal_dataset on two gloo ranks: rank r congeals items r, r + 2, ...; its kept images are {a, b}0000000.png,
    ...; dataset_indices.pt holds both ranks' kept indices, sorted.  Both ranks' kept sets are the fixture's."""
    from ranks import run_ranks
    out = str(tmp_path / "aligned")
    os.environ["GG_CONGEAL_OUT"] = out
    try:
        ret = run_ranks(_driver_worker, timeout=600)
    finally:
        del os.environ["GG_CONGEAL_OUT"]
    blob = load_golden("congeal_dataset")
    n = len(GC.SIZES)
    for rank in range(2):
        assert all(i % 2 == rank and 0 <= i < n for i in ret[rank])
        names = sorted(f for f in os.listdir(out) if f.startswith(chr(ord("a") + rank)))
        assert names == ["%s%07d.png" % (chr(ord("a") + rank), k) for k in range(len(ret[rank]))]
    indices = torch.load(os.path.join(out, "dataset_indices.pt"))
    assert indices.tolist() == sorted(ret[0] + ret[1]) == blob["iters1.used"].tolist()


def test_all_gatherv_on_one_process_is_the_input():
    from gangealing_b200.training.distributed import all_gatherv
    x = torch.arange(5)
    assert all_gatherv(x) is x


def test_abi_rejects_bad_arguments():
    """gg_letterbox_plan and gg_letterbox validate before any device work; the dummy device pointers are never read."""
    import ctypes
    from gangealing_b200 import _lib
    from gangealing_b200.op.letterbox import LetterboxImage
    dll = _lib.load()
    one = 16

    def err():
        return dll.gg_last_error().decode()

    def table(sizes, offsets=None):
        info = (LetterboxImage * len(sizes))()
        off = 0
        for k, (h, w) in enumerate(sizes):
            info[k].offset, info[k].h, info[k].w = (off if offsets is None else offsets[k]), h, w
            off += h * w * 3
        return info, off

    def plan(info, n, S=64, resize=1, nbytes=None):
        ws = ctypes.c_int64()
        return dll.gg_letterbox_plan(info, n, S, resize, nbytes, ctypes.byref(ws)), ws.value

    info, nbytes = table([(30, 40), (50, 20)])
    assert plan(info, 2, nbytes=nbytes)[0] == 0
    assert (info[0].nh, info[0].nw, info[0].order) == (48, 64, 3) and (info[1].nh, info[1].nw) == (64, 26)
    ws = plan(info, 2, nbytes=nbytes)[1]

    def call(out=one, ws_ptr=one, ws_bytes=ws, images=one, nbytes=nbytes, info_host=info, info_dev=one, n=2, S=64,
             resize=1):
        return dll.gg_letterbox(out, ws_ptr, ws_bytes, images, nbytes, info_host, info_dev, None, n, S, resize, None)

    assert call(out=None) == -1 and "null" in err()
    assert call(images=None) == -1 and "null" in err()
    assert call(info_host=None) == -1 and "null" in err()
    assert call(info_dev=None) == -1 and "null" in err()
    assert call(info_dev=one + 4) == -1 and "8-byte" in err()
    assert call(n=0) == -1 and "N" in err()
    assert call(S=0) == -1 and "S >= 1" in err()
    assert call(resize=2) == -1 and "resize" in err()
    assert call(nbytes=nbytes - 1) == -1 and "outside" in err()
    assert call(ws_bytes=ws - 1) == -1 and "workspace" in err()
    assert call(ws_ptr=None) == -1 and "workspace" in err()
    assert call(ws_ptr=one + 4) == -1 and "16-byte" in err()
    assert call(S=128) == -1 and "differs" in err()          # the table was planned for S = 64
    assert call(resize=0) == -1 and "max(h, w)" in err()
    bad, _ = table([(30, 40), (50, 20)], offsets=[0, -3])
    assert plan(bad, 2, nbytes=nbytes)[0] == -1 and "outside" in err()
    empty, _ = table([(0, 40)])
    assert plan(empty, 1, nbytes=nbytes)[0] == -1 and "empty" in err()
    thin, thin_bytes = table([(1, 200)])
    assert plan(thin, 1, S=64, nbytes=thin_bytes)[0] == -1 and "empty image" in err()   # Pillow refuses height 0 too
    for (h, w), S, order in ((((201, 2), 128, 4), ((202, 2), 256, 3), ((200, 2), 128, 3), ((901, 9), 256, 4),
                             ((900, 9), 256, 3), ((2, 201), 128, 3))):   # Pillow's pass order on both sides of each bound
        tall, tall_bytes = table([(h, w)])
        assert plan(tall, 1, S=S, nbytes=tall_bytes)[0] == 0 and tall[0].order == order, (h, w, S, tall[0].order)
    square, square_bytes = table([(50, 40)])
    assert plan(square, 1, S=50, resize=0, nbytes=square_bytes)[0] == 0 and square[0].order == 0


# ------------------------------------------------------------------------------------------------ GPU
def _sweep_sizes():
    """At least 200 seeded sizes from 1 x 1 to 2000 x 1500: both orientations, up- and downsampling, one-pass sizes
    (the long side already S) and images more than 100 times as tall as wide, whose vertical pass shrinks (Pillow's
    vertical-first order: 201 x 2 at S = 128) or grows (horizontal first: 202 x 2 at S = 256)."""
    rng = np.random.default_rng(2024)
    sizes = [(1, 1), (2000, 1500), (1500, 2000), (1, 2), (2, 1), (7, 7), (300, 2), (1000, 3), (2000, 13), (13, 2000),
             (200, 2), (201, 2), (202, 2), (203, 2), (204, 2), (240, 2), (255, 2), (301, 3), (900, 9), (901, 9)]
    for S in (64, 128, 256):
        sizes += [(S, S), (S // 2, S), (S, S // 3), (S, S + 1), (3 * S, S), (S - 1, S - 1)]
    while len(sizes) < 230:
        h, w = (int(v) for v in np.exp(rng.uniform(0, np.log(2000), 2)))
        sizes.append((max(1, h), max(1, min(w, 1500 if h > 1500 else 2000))))
    return sizes


@pytest.mark.gpu
def test_letterbox_is_bitwise_pillow():
    """Every value of letterbox(resize=True) equals prepro(border_pad(img, S)) under the installed Pillow, for the sweep's
    sizes at S = 64, 128 and 256, in ragged batches; sizes that resize to an empty image are refused as Pillow does."""
    from gangealing_b200.op.letterbox import letterbox
    rng = np.random.default_rng(7)
    sizes = _sweep_sizes()
    differ = total = cases = 0
    for S in (64, 128, 256):
        batch = []
        for k, (h, w) in enumerate(sizes):
            nh, nw = (S, int(np.around(S * w / h))) if h > w else (int(np.around(S * h / w)), S)
            if min(nh, nw) < 1:
                with pytest.raises(RuntimeError, match="empty image"):
                    letterbox([np.zeros((h, w, 3), np.uint8)], S)
                continue
            batch.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
            if len(batch) == 24 or k == len(sizes) - 1:
                got = letterbox(batch, S).cpu()
                want = OC.letterbox_ref(batch, S)
                differ += int((got.view(torch.int32) != want.view(torch.int32)).sum())
                total += want.numel()
                cases += len(batch)
                batch = []
    print("letterbox vs Pillow: %d of %d values differ over %d images" % (differ, total, cases))
    assert cases >= 600 and differ == 0


@pytest.mark.gpu
def test_letterbox_without_resize_pads_and_mirrors_the_square():
    """resize=False: x_big, and torch.where(flip, x_big.flip(3), x_big) where a flip flag is set (asymmetric pads)."""
    from gangealing_b200.op.letterbox import letterbox
    rng = np.random.default_rng(9)
    for h, w in ((37, 60), (60, 37), (45, 45), (1, 8), (9, 2)):
        imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(3)]
        flip = torch.tensor([True, False, True], device=DEV)
        big = OC.letterbox_ref(imgs, None, False)
        assert torch.equal(letterbox(imgs, None, resize=False).cpu(), big)
        assert torch.equal(letterbox(imgs, max(h, w), resize=False, flip=flip).cpu(),
                           torch.where(flip.cpu().view(-1, 1, 1, 1), big.flip(3), big))


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_api_on_the_gpu_reproduces_the_fixture(name):
    """The API on cuda_ops with the STN's convolutions in fp32 against the CPU fixture."""
    from gangealing_b200.opset import cuda_ops
    blob = load_golden("congeal_dataset")
    with fp32_stn():
        res = _run(cuda_ops(), blob, name, DEV)
    assert res["aligned"].is_cuda
    _check_fixture(blob, name, res)


@pytest.mark.gpu
@pytest.mark.parametrize("iters", [1, 3])
def test_api_matches_the_per_image_composition(iters):
    """The script's order on cuda_ops: per image, letterbox, determine_flips on a batch of one, the flipped native
    square, the similarity stage and the filters.  The kept sets are equal; flips decided on the batch may differ from
    batch-1 flips only at a near-tie of the two flows' smoothness, and the test reports how many do."""
    from gangealing_b200.evaluation import congeal_images, determine_flips
    from gangealing_b200.op.letterbox import letterbox
    from gangealing_b200.opset import cuda_ops
    blob = load_golden("congeal_dataset")
    t = _mirror(cuda_ops(), blob).to(DEV)
    images = _images(blob)
    with torch.no_grad(), fp32_stn():
        res = congeal_images(t, images, output_resolution=GC.OUTPUT_RESOLUTION,
                             min_effective_resolution=GC.MIN_EFFECTIVE_RESOLUTION, iters=iters)
        keep, flips = [], []
        for img in images:
            h, w = img.shape[:2]
            x_in, flip, _ = determine_flips(t, None, letterbox([img], GC.STN_KW["flow_size"]), iters=iters)
            x_big = letterbox([img], max(h, w), resize=False)
            x_big = torch.where(flip.view(-1, 1, 1, 1), x_big.flip(3), x_big)
            bounds = torch.tensor([[h, w]], dtype=torch.float, device=DEV)
            _, M, oob = t.stns[0](x_in, return_flow=True, return_out_of_bounds=True, input_img_for_sampling=x_big,
                                  output_resolution=GC.OUTPUT_RESOLUTION, image_bounds=bounds, iters=iters)
            scale = torch.det(torch.cat([M, torch.tensor([[[0.0, 0.0, 1.0]]], device=DEV)], 1)).sqrt_()
            keep.append(not (scale.item() * min(w, h) < GC.MIN_EFFECTIVE_RESOLUTION or oob.item()))
            flips.append(bool(flip.item()))
    assert res["keep"].tolist() == keep
    print("iters %d: %d of %d flips differ from batch-1 flips" % (iters, sum(a != b for a, b in zip(res["flips"].tolist(),
                                                                                                     flips)), len(flips)))
