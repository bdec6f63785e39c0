"""Dataset congealing's pre-processing on the device (csrc/letterbox.cu): prepare_data.border_pad (Pillow's LANCZOS
resize + edge padding) followed by congeal_dataset.py's prepro, for a ragged list of uint8 RGB images, in one host-to-
device copy and three launches."""
import ctypes

import numpy as np
import torch

from .. import _lib

__all__ = ["letterbox", "LetterboxImage"]


class LetterboxImage(ctypes.Structure):
    """GGLetterboxImage (include/gg_b200.h)."""
    _fields_ = [("offset", ctypes.c_int64), ("h", ctypes.c_int32), ("w", ctypes.c_int32), ("nh", ctypes.c_int32),
                ("nw", ctypes.c_int32), ("order", ctypes.c_int32), ("ksize_h", ctypes.c_int32),
                ("ksize_v", ctypes.c_int32), ("reserved", ctypes.c_int32), ("tmp_offset", ctypes.c_int64),
                ("coef_h", ctypes.c_int64), ("coef_v", ctypes.c_int64)]


def hwc_uint8(image):
    """A (H, W, 3) uint8 CPU tensor from a tensor, an array or a PIL image; anything else is refused."""
    t = image if torch.is_tensor(image) else torch.from_numpy(np.array(image))
    if t.dtype != torch.uint8 or t.dim() != 3 or t.size(2) != 3:
        raise ValueError("letterbox: images must be (H, W, 3) uint8 RGB (got %s %s)" % (t.dtype, tuple(t.shape)))
    return t.cpu()


@torch.no_grad()
def letterbox(images, size=None, resize=True, flip=None, device=None):
    """border_pad(img, size, resize) then prepro (congeal_dataset.py:23-26) of every image, on a CUDA device.
    images: a list of (H, W, 3) uint8 tensors or arrays of any sizes.  resize=True: Pillow 12.2's LANCZOS resize of the
    long side to `size`, bitwise; resize=False: the edge pad alone to size = max(H, W), which every image must share
    (None: the first image's).  flip: (N,) bool device tensor or None; where set, the mirror of the padded square is
    written (x_big.flip(3)), decided on the device without a host sync.  device: the CUDA device of the output (None:
    flip's, else the current device).  -> (N, 3, size, size) fp32 in [-1, 1]."""
    imgs = [hwc_uint8(x) for x in images]
    n = len(imgs)
    if n == 0:
        raise ValueError("letterbox: no images")
    if size is None:
        if resize:
            raise ValueError("letterbox: resize needs a target size")
        size = max(imgs[0].shape[:2])
    if device is None:
        device = flip.device if flip is not None else torch.device("cuda", torch.cuda.current_device())
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("letterbox: the output device must be a CUDA device (got %s)" % dev)
    with torch.cuda.device(dev):
        return _letterbox(imgs, n, int(size), bool(resize), flip, dev)


def _letterbox(imgs, n, size, resize, flip, dev):
    if flip is not None:
        _lib.require_cuda(flip)
        if flip.numel() != n:
            raise RuntimeError("letterbox: flip must hold one flag per image (%d), got %d" % (n, flip.numel()))
        flip = flip.reshape(n).to(torch.uint8).contiguous()
    lib = _lib.load()
    info = (LetterboxImage * n)()
    offset = 0
    for k, t in enumerate(imgs):
        info[k].offset, info[k].h, info[k].w = offset, t.size(0), t.size(1)
        offset += t.numel()
    ws_bytes = ctypes.c_int64()
    _lib.check(lib.gg_letterbox_plan(info, n, int(size), int(bool(resize)), offset, ctypes.byref(ws_bytes)),
               "gg_letterbox_plan")
    table = ctypes.sizeof(info)    # 64 bytes per image: the images start 16-byte aligned
    host = torch.empty(table + offset, dtype=torch.uint8, pin_memory=True)
    ctypes.memmove(host.data_ptr(), info, table)
    for k, t in enumerate(imgs):
        host.narrow(0, table + info[k].offset, t.numel()).copy_(t.reshape(-1))
    buf = host.to(dev, non_blocking=True)   # the one host-to-device copy: table and pixels
    ws = torch.empty(max(16, ws_bytes.value), dtype=torch.uint8, device=dev)
    out = torch.empty(n, 3, size, size, dtype=torch.float32, device=dev)
    _lib.check(lib.gg_letterbox(out.data_ptr(), ws.data_ptr(), ws.numel(), buf.data_ptr() + table, offset,
                                host.data_ptr(), buf.data_ptr(), _lib.ptr(flip), n, int(size), int(bool(resize)),
                                _lib.stream()), "gg_letterbox")
    return out
