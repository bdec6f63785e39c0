"""Test-time flip decision (reference applications/__init__.py:57-84)."""
import torch


def determine_flips(t, classifier, input_imgs, cluster=None, return_cluster_assignments=False, num_heads=1,
                    no_flip_inference=False, iters=1, padding_mode="border"):
    """Decide per image whether to mirror it before congealing.  With a cluster classifier (clustering models) the flip is
    predicted directly (run_flip, or run_flip_target for a given `cluster`); otherwise, unless no_flip_inference, the image
    and its mirror both run through the STN and the smoother residual flow wins (forward_with_flip).  The reference's
    `args` fields are keyword arguments here.
    -> (images, flip_indices (N, 1, 1, 1) or (N,) bool, warp_policy[, clusters])."""
    if classifier is not None:
        if cluster is None:
            data_flipped, _, clusters, flip_indices = classifier.run_flip(input_imgs)
            clusters = clusters % num_heads
        else:
            data_flipped, flip_indices = classifier.run_flip_target(input_imgs, cluster)
            clusters = torch.full((input_imgs.size(0),), int(cluster), dtype=torch.long, device=input_imgs.device)
        warp_policy = torch.eye(num_heads, device=input_imgs.device)[clusters]
    elif not no_flip_inference:
        _, data_flipped, flip_indices = t.forward_with_flip(input_imgs, return_inputs=True, return_flip_indices=True,
                                                            padding_mode=padding_mode, iters=iters)
        warp_policy = "cartesian"
        clusters = torch.zeros(input_imgs.size(0), dtype=torch.long, device=input_imgs.device)
    else:
        data_flipped = input_imgs
        flip_indices = torch.zeros(input_imgs.size(0), 1, 1, 1, device=input_imgs.device, dtype=torch.bool)
        warp_policy = "cartesian"
        clusters = torch.zeros(input_imgs.size(0), dtype=torch.long, device=input_imgs.device)
    if return_cluster_assignments:
        return data_flipped, flip_indices, warp_policy, clusters
    return data_flipped, flip_indices, warp_policy
