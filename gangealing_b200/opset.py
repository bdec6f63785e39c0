"""The op namespace the host-side networks are written against.

`cuda_ops()` is the product: every entry goes through libgg_b200.so (or cuDNN for the convolutions).  The
networks take an optional `ops=` argument so that test infrastructure (oracle/) can run the SAME host code
on its CPU restatement for parity checks and for the timed CPU baseline; nothing in this package ever
selects anything but `cuda_ops()` by itself.
"""
import types

_cached = None


def cuda_ops():
    global _cached
    if _cached is None:
        from . import op as _op
        from .op import modconv as _mod
        from .stn import flow as _flow
        from .stn import sampling as _smp
        from .splat2d import nn_argmin as _nn_argmin
        from .splat2d import splat2d as _splat2d
        from .splat2d import splat2d_lookup as _splat2d_lookup
        from .splat2d import track_points_lerp as _track_points_lerp
        from .splat2d import splat_composite_grid as _splat_composite_grid
        from .splat2d import splat_lookup_composite_grid as _splat_lookup_composite_grid
        from .splat2d import laplacian_blend as _laplacian_blend
        from .op import feature_distance as _fd
        from .op import vgg_pool as _vp
        from .evaluation import ops as _ev
        from .op import pca as _pca
        from .op import grids as _grids
        from .op import letterbox as _letterbox
        _cached = types.SimpleNamespace(
            name="sm_90a",
            upfirdn2d=_op.upfirdn2d,
            fused_leaky_relu=_op.fused_leaky_relu,
            noise_bias_act=_op.noise_bias_act,
            blur_noise_bias_act=_op.blur_noise_bias_act,
            conv2d=_op.conv2d_gradfix.conv2d,
            conv_transpose2d=_op.conv2d_gradfix.conv_transpose2d,
            modulated_weight=_mod.modulated_weight,
            modulated_conv2d=_mod.modulated_conv2d,
            channel_scale=_mod.channel_scale,
            mipmap_warp=_smp.mipmap_warp,
            grid_sample=_smp.grid_sample_bilinear,
            bilinear_downsample=_smp.bilinear_downsample,
            flow_compose=_flow.flow_compose,
            stn_sample_affine=_smp.stn_sample_affine,     # one-pass sampling (grid generated inside the sampler)
            stn_sample_flow=_smp.stn_sample_flow,
            splat2d=_splat2d,
            splat2d_lookup=_splat2d_lookup,               # uncongeal_points' grid lookup fused into the splat
            nn_argmin=_nn_argmin,                         # congeal_points' brute-force search without the distance tensor
            laplacian_blend=_laplacian_blend,             # splat_points(blend_alg='laplacian*'): fused Gaussian stacks
            feature_distance=_fd.feature_distance,
            feature_distance_stacked=_fd.feature_distance_stacked,   # both images' features from ONE backbone pass
            bias_relu_pool=_vp.bias_relu_pool,            # VGG slice boundary: bias + ReLU + 2x2 max-pool, one pass each way
            bias_relu_pool_supported=_vp.supported,
            tv_per_sample=_ev.tv_per_sample,              # match_flows / flow_scores: per-sample smoothness, one launch
            pck_transfer_points=_ev.pck_transfer_points,  # PCK-Transfer: congeal + search + lookup + score, one call
            batch_gram=_pca.batch_gram,                   # IncrementalPCA's per-batch means + centred Grams, fp64 DMMA
            mipmap_warp_lerp=_smp.mipmap_warp_lerp,       # congealing animation: T lerped-grid warps from one pyramid
            mipmap_warp_lerp_mean=_smp.mipmap_warp_lerp_mean,   # ... and their per-frame batch sums, frames never written
            track_points_lerp=_track_points_lerp,         # dense point tracking over a stage's frames, one launch
            splat_composite_grid=_splat_composite_grid,   # label propagation: splats + composite + uint8 grid per frame
            splat_lookup_composite_grid=_splat_lookup_composite_grid,   # edits on real images: lookup + flip + splat + grid
            flow_image_grid=_grids.flow_image_grid,       # training visuals: colour-wheel flow images as a uint8 grid
            image_grid=_grids.image_grid,                 # ... min/max-normalised uint8 grid (per-image ranges)
            cluster_accumulate=_grids.cluster_accumulate,  # ... per-cluster sums of routed images, in order, on the device
            letterbox=_letterbox.letterbox,               # dataset congealing: ragged uint8 -> Lanczos + edge pad, fp32
        )
    return _cached
