"""GAN-supervised pair sampling and the GANgealing losses -- host-side mirror of reference
models/losses/loss.py (callers of the hot path; plain tensor logic above the op boundary)."""
import torch

from ..stn.transformer import total_variation_loss  # noqa: F401  (re-exported, as the reference's loss.py does)


def flow_identity_loss(delta_flow):
    return delta_flow.pow(2).mean()


def sample_gan_supervised_pairs(generator, ll, resize_fake2stn, psi, batch, dim_latent, freeze_ll, device, z=None):
    """One (unaligned input, aligned target) batch: G(z) and G(truncated w), reference loss.py:21-29."""
    with torch.set_grad_enabled(not freeze_ll):
        if z is None:
            z = torch.randn(batch, dim_latent, device=device)
        unaligned_in, w_noise = generator([z], noise=None, return_latents=True)
        # the latent learner's output in the generator's two-latent form: the rows above the inject index are w itself
        w_aligned = ll([w_noise[:, 0, :]], psi=psi, split=True)
        inject = getattr(ll, "module", ll).inject_index
        aligned_target, _ = generator(w_aligned, input_is_latent=True, inject_index=inject, noise=None)
        aligned_target = resize_fake2stn(aligned_target)
    return unaligned_in, aligned_target


def gangealing_loss(generator, stn, ll, loss_fn, resize_fake2stn, psi, batch, dim_latent, freeze_ll, device,
                    sample_from_full_res=False, z=None, **stn_kwargs):
    """Unimodal reconstruction loss (reference loss.py:64-75)."""
    unaligned_in, aligned_target = sample_gan_supervised_pairs(generator, ll, resize_fake2stn, psi, batch, dim_latent,
                                                               freeze_ll, device, z=z)
    source = unaligned_in if sample_from_full_res else None
    aligned_pred, delta_flow = stn(resize_fake2stn(unaligned_in), return_flow=True, input_img_for_sampling=source,
                                   **stn_kwargs)
    return loss_fn(aligned_pred, aligned_target).mean(), delta_flow


def assign_fake_images_to_clusters(generator, stn, ll, loss_fn, resize_fake2stn, psi, batch, dim_latent, freeze_ll,
                                   num_heads, flips, device, sample_from_full_res=True, z=None, **stn_kwargs):
    """Congeal fake images with every head (and optionally their mirrors), score, assign (reference loss.py:32-61)."""
    unaligned_in, aligned_target = sample_gan_supervised_pairs(generator, ll, resize_fake2stn, psi, batch, dim_latent,
                                                               freeze_ll, device, z)
    if flips:
        unaligned_in = torch.cat([unaligned_in, unaligned_in.flip(3,)], 0)
        aligned_target = aligned_target.repeat(2, 1, 1, 1)
        loss_size = (2, batch, num_heads)
    else:
        loss_size = (batch, num_heads)
    source = unaligned_in if sample_from_full_res else None
    resized = resize_fake2stn(unaligned_in)
    aligned_pred, delta_flow = stn(resized, return_flow=True, input_img_for_sampling=source, **stn_kwargs)
    perceptual = loss_fn(aligned_pred, aligned_target).view(*loss_size)
    collapsed = perceptual.permute(1, 0, 2).reshape(batch, 2 * num_heads) if flips else perceptual
    return collapsed.min(dim=1), aligned_pred, delta_flow, unaligned_in, resized, collapsed


def gangealing_cluster_loss(generator, stn, ll, loss_fn, resize_fake2stn, psi, batch, dim_latent, freeze_ll, num_heads,
                            flips, device, sample_from_full_res=True, z=None, **stn_kwargs):
    """Clustering reconstruction loss: only the assigned head's flow is regularised (reference loss.py:78-92)."""
    assignments, _, delta_flow, _, _, _ = assign_fake_images_to_clusters(
        generator, stn, ll, loss_fn, resize_fake2stn, psi, batch, dim_latent, freeze_ll, num_heads, flips, device,
        sample_from_full_res, z=z, **stn_kwargs)
    hw2 = delta_flow.size()[1:]
    if flips:
        delta_flow = delta_flow.view(2, batch, num_heads, *hw2).permute(1, 0, 2, 3, 4, 5).reshape(batch, 2 * num_heads, *hw2)
    else:
        delta_flow = delta_flow.view(batch, num_heads, *hw2)
    return assignments.values.mean(), delta_flow[torch.arange(batch, device=delta_flow.device), assignments.indices]
