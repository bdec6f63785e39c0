"""The sm_90a op of the latent learner's PCA initialiser (csrc/pca.cu), registered in `cuda_ops()` as `batch_gram`;
oracle/opset.py restates it in float64 torch with the same signature."""
import torch

from .. import _lib


def batch_gram(w, offsets):
    """Per-block fp64 column means and centred Gram matrices of a (n, D) float32 matrix, one C-ABI call (gg_batch_gram).

    offsets: B + 1 strictly increasing row offsets (a sequence of ints or a CPU int64 tensor); block b is the rows
    [offsets[b], offsets[b+1]).  D must be a multiple of 64, at most 1024.
    -> (gram (B, D, D) float64: sum over the block's rows of (x - mean_b)(x - mean_b)^T, mean (B, D) float64)."""
    _lib.require_cuda(w)
    if w.dim() != 2 or w.dtype != torch.float32:
        raise RuntimeError("batch_gram: expected a (n, D) float32 matrix, got %s %s" % (tuple(w.shape), w.dtype))
    off = torch.as_tensor(offsets, dtype=torch.int64, device="cpu").contiguous()   # read on the host by the C entry
    if off.dim() != 1 or off.numel() < 2:
        raise RuntimeError("batch_gram: offsets must hold B + 1 >= 2 entries")
    if int(off[-1]) > w.size(0):
        raise RuntimeError("batch_gram: offsets[-1] = %d exceeds the %d rows of w" % (int(off[-1]), w.size(0)))
    w = w.contiguous()
    b, d = off.numel() - 1, w.size(1)
    gram = torch.empty(b, d, d, dtype=torch.float64, device=w.device)
    mean = torch.empty(b, d, dtype=torch.float64, device=w.device)
    _lib.check(_lib.load().gg_batch_gram(gram.data_ptr(), mean.data_ptr(), w.data_ptr(), off.data_ptr(), b, d,
                                         _lib.stream()), "gg_batch_gram")
    return gram, mean
