"""CPU restatement of dataset congealing's pre-processing (test infrastructure -- see oracle/__init__.py).

Reference: prepare_data.py:53-77 (`border_pad`: Pillow's resize with ANTIALIAS, which is LANCZOS, and np.pad(mode='edge'))
and applications/congeal_dataset.py:23-26 (`prepro`), called literally on each image.
"""
import types

import numpy as np
import torch
from PIL import Image

from . import propagate as _propagate


def border_pad(img, target_res, resize=True):
    """prepare_data.border_pad(img, target_res, resize, to_pil=False) on a PIL image."""
    original_width, original_height = img.size
    if original_height <= original_width:
        if resize:
            img = img.resize((target_res, int(np.around(target_res * original_height / original_width))), Image.LANCZOS)
        width, height = img.size
        img = np.asarray(img)
        half_height = (target_res - height) / 2
        int_half_height = int(half_height)
        lh = int_half_height
        rh = int_half_height + (half_height > int_half_height)
        img = np.pad(img, mode="edge", pad_width=[(lh, rh), (0, 0), (0, 0)])
    else:
        if resize:
            img = img.resize((int(np.around(target_res * original_width / original_height)), target_res), Image.LANCZOS)
        width, height = img.size
        img = np.asarray(img)
        half_width = (target_res - width) / 2
        int_half_width = int(half_width)
        lw = int_half_width
        rw = int_half_width + (half_width > int_half_width)
        img = np.pad(img, mode="edge", pad_width=[(0, 0), (lw, rw), (0, 0)])
    return img


def prepro(x):
    """congeal_dataset.py:23-26 without the device move: (H, W, 3) uint8 -> (1, 3, H, W) fp32."""
    return torch.from_numpy(np.ascontiguousarray(x)).float().div_(255.0).add_(-0.5).mul_(2.0).permute(2, 0, 1).unsqueeze_(0)


def letterbox_ref(images, size=None, resize=True, flip=None, device=None):
    """The op set's letterbox: prepro(border_pad(img, size, resize)) of each image, mirrored where flip."""
    from gangealing_b200.op.letterbox import hwc_uint8
    imgs = [Image.fromarray(hwc_uint8(x).numpy()) for x in images]
    if size is None:
        size = max(imgs[0].size)
    out = torch.cat([prepro(border_pad(img, size, resize)) for img in imgs], 0)
    if flip is not None:
        out = torch.where(flip.reshape(-1, 1, 1, 1).cpu().bool(), out.flip(3), out)
    return out if device is None else out.to(device)


def cpu_ops():
    """oracle.propagate.cpu_ops() plus `letterbox`: the op set that runs gangealing_b200.evaluation.congeal on the CPU."""
    return types.SimpleNamespace(**vars(_propagate.cpu_ops()), letterbox=letterbox_ref)
