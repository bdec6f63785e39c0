"""Flow-smoothness scores for dataset filtering (reference applications/flow_scores.py:25-70).  Scores come one batch at
a time; the caller owns the loader, the gathering across ranks and any file it keeps them in."""
import torch

from .flips import determine_flips


@torch.inference_mode()
def flow_scores(t, batch, iters=1, padding_mode="border", no_flip_inference=False):
    """-(per-sample smoothness) of the residual flow the STN produces for each image of `batch` (N, C, H, W), after the
    flip decision: lower (more negative) scores mark images to drop.  -> (N,) float32."""
    if getattr(t, "num_heads", 1) > 1:
        raise ValueError("flow_scores: clustering STNs (num_heads > 1) are not supported")
    batch, _, _ = determine_flips(t, None, batch, no_flip_inference=no_flip_inference, iters=iters, padding_mode=padding_mode)
    _, flows = t(batch, return_flow=True, iters=iters, padding_mode=padding_mode)
    return -t.ops.tv_per_sample(flows)


def get_high_score_indices(scores, fraction_retained):
    """Indices of the scores strictly above the (1 - fraction_retained) quantile."""
    min_score = torch.quantile(scores, 1 - fraction_retained)
    high_score_indices, = torch.where(scores > min_score)
    return high_score_indices.tolist()


def filter_dataset(dataset, scores, fraction_retained):
    """`dataset` without its lowest-scoring images: a Subset keeping `fraction_retained` of it.  scores: 1-D tensor with
    one score per item, or the path of a saved one."""
    from torch.utils.data import Subset
    if isinstance(scores, str):
        scores = torch.load(scores)
    return Subset(dataset, get_high_score_indices(scores, fraction_retained))
