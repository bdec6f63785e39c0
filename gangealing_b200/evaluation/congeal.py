"""Dataset congealing (reference applications/congeal_dataset.py:21-107): align a dataset of images of any size at their
native resolution with the similarity stage of a trained STN, and keep the images it aligns well.

The reference puts every image through PIL twice on the host (prepare_data.border_pad), uploads the fp32 copy of its
full-resolution padded square and reads four values back per image.  Here the op set's `letterbox` letterboxes a whole
batch to the flow size in one launch and each native square on the device (the flip applied there, with no host read),
the flips are decided once per batch, and the keep decisions are made on the device and read back once per batch.  The
similarity stage still runs once per image: with iters > 1 each intermediate is sampled from that image's native square.
"""
import contextlib
import os

import torch

from ..op.letterbox import hwc_uint8
from .flips import determine_flips
from .flow_scores import filter_dataset


def _similarity_stage(t):
    from ..stn.heads import SimilarityHead
    from ..stn.transformer import ComposedSTN
    if getattr(t, "num_heads", 1) > 1 or getattr(getattr(t, "warp_head", None), "num_heads", 1) > 1:
        raise ValueError("congeal_images: clustering STNs (num_heads > 1) are not supported")
    t_sim = t.stns[0] if isinstance(t, ComposedSTN) else t
    if not isinstance(t_sim.warp_head, SimilarityHead):
        raise ValueError("congeal_images: only similarity transformations are supported (the first stage is not one)")
    return t_sim


@torch.no_grad()
def congeal_images(t, images, output_resolution=256, min_effective_resolution=192, flow_size=None, iters=1,
                   padding_mode="border", no_flip_inference=False):
    """apply_congealing (congeal_dataset.py:21-64) on a batch of images: a list of (H, W, 3) uint8 tensors or arrays, or PIL
    images, of any sizes.  t: the STN (a ComposedSTN, whose similarity stage t.stns[0] aligns, or a similarity STN);
    flow_size: the letterbox size the STN reads (None: t.stn_in_size).

    Each image is letterboxed to flow_size, the flips are decided on the batch by determine_flips, and the similarity
    stage aligns the image from its (flipped) native square padded to max(H, W), at output_resolution.  The reference's
    filters are kept as they are: image n is kept unless scale * min(W, H) < min_effective_resolution or the warp samples
    outside the image, where scale = sqrt(det([M; 0 0 1])) is the similarity's scale relative to the padded square (not
    to the image's short side), and the bounds passed to the out-of-bounds test are (H, W), which it reads as the height
    and width of the content inside the square.
    -> dict: aligned (M, R, R, 3) uint8, the kept images quantised as write_image_batch stores them; keep (N,) bool,
    scale (N,) fp32, out_of_bounds (N,) bool and flips (N,) bool, on the host."""
    t_sim = _similarity_stage(t)
    imgs = [hwc_uint8(x) for x in images]
    n = len(imgs)
    if n == 0:
        raise ValueError("congeal_images: no images")
    flow_size = flow_size or t.stn_in_size
    dev = next(t.parameters()).device
    # the C-ABI ops launch on the current device's stream: make the STN's device current for the whole batch
    with torch.cuda.device(dev) if dev.type == "cuda" else contextlib.nullcontext():
        return _congeal_batch(t, t_sim, imgs, dev, output_resolution, min_effective_resolution, flow_size, iters,
                              padding_mode, no_flip_inference)


def _congeal_batch(t, t_sim, imgs, dev, output_resolution, min_effective_resolution, flow_size, iters, padding_mode,
                   no_flip_inference):
    ops = t.ops
    n = len(imgs)
    sizes = torch.tensor([list(img.shape[:2]) for img in imgs], dtype=torch.float).to(dev)   # (h, w), one copy
    x_in = ops.letterbox(imgs, flow_size, device=dev)
    x_in, flips, _ = determine_flips(t, None, x_in, no_flip_inference=no_flip_inference, iters=iters,
                                     padding_mode=padding_mode)
    flips = flips.reshape(n).bool()
    aligned, mats, oobs = [], [], []
    for k, img in enumerate(imgs):
        x_big = ops.letterbox([img], max(img.shape[:2]), resize=False, flip=flips[k:k + 1], device=dev)
        out, M, oob = t_sim(x_in[k:k + 1], return_flow=True, return_out_of_bounds=True, input_img_for_sampling=x_big,
                            output_resolution=output_resolution, image_bounds=sizes[k:k + 1], iters=iters,
                            padding_mode=padding_mode)
        aligned.append(out)
        mats.append(M)
        oobs.append(oob)
    one_hot = torch.zeros(n, 1, 3, device=dev)
    one_hot[:, :, 2] = 1
    scale = torch.det(torch.cat([torch.cat(mats, 0), one_hot], 1)).sqrt_()
    oob = torch.cat(oobs, 0).reshape(n).bool()
    # scale.item() * min(w, h) in the reference: a Python float times an int, i.e. in float64
    too_low_res = scale.double() * sizes.min(dim=1).values.double() < min_effective_resolution
    keep = ~(too_low_res | oob)
    host = torch.cat([keep.float(), scale, oob.float(), flips.float()]).cpu()    # the batch's one host sync
    keep, scale, oob, flips = host[:n].bool(), host[n:2 * n], host[2 * n:3 * n].bool(), host[3 * n:].bool()
    kept = keep.nonzero().flatten().tolist()
    r = aligned[0].size(-1)
    if kept:
        x = torch.cat([aligned[k] for k in kept], 0)
        ranges = torch.ones(len(kept), 2, device=dev)
        ranges[:, 0] = -1
        # write_image_batch: clamp(-1, 1), (x + 1) / 2, * 255 + 0.5, clamp(0, 255), truncation -- image_grid's quantisation
        # with the range (-1, 1); one column without padding lays the images out back to back
        images_u8 = ops.image_grid(x, ranges, 1, padding=0).reshape(len(kept), r, r, 3)
    else:
        images_u8 = torch.empty(0, r, r, 3, dtype=torch.uint8, device=dev)
    return {"aligned": images_u8, "keep": keep, "scale": scale, "out_of_bounds": oob, "flips": flips}


def image_name(rank, count):
    """write_image_batch's file name of the count-th image a rank writes: the rank's letter and seven digits."""
    return "%s%07d.png" % (chr(ord("a") + rank), count)


@torch.no_grad()
def congeal_dataset(t, dataset, out, batch=50, flow_scores=None, fraction_retained=1.0, **kw):
    """align_and_filter_dataset (congeal_dataset.py:80-107) without the LMDB: every rank congeals the items
    arange(rank, len(dataset), world) of `dataset` (PIL images or (H, W, 3) uint8 arrays), `batch` at a time with
    congeal_images(**kw), and writes its kept images to `out` as PNGs named a0000000.png, a0000001.png, ... (b... on rank
    1).  The primary rank writes `out`/dataset_indices.pt: the kept indices of every rank, sorted.  As in the reference
    they index `dataset` after the flow-score filter (flow_scores: scores or their path; fraction_retained).
    -> this rank's kept indices (int64, on the STN's device)."""
    from PIL import Image
    from ..training.distributed import all_gatherv, get_rank, get_world_size, primary, synchronize
    if flow_scores is not None:
        dataset = filter_dataset(dataset, flow_scores, fraction_retained)
    rank, world = get_rank(), get_world_size()
    if primary():
        os.makedirs(out, exist_ok=True)
    synchronize()
    indices = list(range(rank, len(dataset), world))
    used, total = [], 0
    for start in range(0, len(indices), batch):
        idx = indices[start:start + batch]
        res = congeal_images(t, [dataset[i] for i in idx], **kw)
        for img in res["aligned"].cpu().numpy():
            Image.fromarray(img).save(os.path.join(out, image_name(rank, total)))
            total += 1
        used += [idx[j] for j in res["keep"].nonzero().flatten().tolist()]
    device = next(t.parameters()).device
    used = torch.tensor(used, dtype=torch.long).to(device)
    synchronize()
    gathered = all_gatherv(used)
    if primary():
        torch.save(gathered.sort().values.cpu(), os.path.join(out, "dataset_indices.pt"))
    return used
