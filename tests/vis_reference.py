"""What the visualisation tests share (not collected: the name does not match test_*.py): the fp32 switch for STN runs
held to a CPU fixture, and the mirror models, grids and fixture comparison of the training-visual tests on the CPU and
the GPU (test_training_vis.py, test_training_vis_gpu.py)."""
import contextlib

import torch

from oracle import make_golden_training_vis as GT

DIFFER_BOUND = 0.005


@contextlib.contextmanager
def fp32_stn():
    """The STN's cuDNN convolutions and matmuls in fp32, not TF32, so that the GPU run can be held to the CPU fixture
    (as the other fixture tests on the GPU do)."""
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def mirror_models(ops, k, flips, device="cpu"):
    """This repo's generator, STN, latent learner and classifier with the fixture's seeded weights, as the duck-typed
    trainer / classifier trainer training_visuals and classifier_visuals read."""
    import types
    from oracle.make_golden import _mse, classifier_setup
    from gangealing_b200.cluster_classifier import ResnetClassifier
    from gangealing_b200.stn import BilinearDownsample, get_stn
    from gangealing_b200.stylegan2 import Generator
    from gangealing_b200.training import DirectionInterpolator

    def with_ops(cls):
        return lambda *a, **kw: cls(*a, ops=ops, **kw)
    mods = dict(Generator=with_ops(Generator), get_stn=with_ops(get_stn), DirectionInterpolator=DirectionInterpolator,
                ResnetClassifier=with_ops(ResnetClassifier), BilinearDownsample=with_ops(BilinearDownsample))
    g, stn, ll, cls, resize, _ = classifier_setup(mods, heads=k, flips=flips)
    g, stn, ll, cls, resize = [m.to(device) for m in (g, stn, ll, cls, resize)]
    cfg = types.SimpleNamespace(num_heads=k, flips=flips, padding_mode=GT.PADDING)
    trainer = types.SimpleNamespace(cfg=cfg, generator=g, t_ema=stn, ll=ll, ll_module=ll, loss_fn=_mse, resize_fake2stn=resize,
                                    psi_t=GT.PSI, device=device)
    return trainer, types.SimpleNamespace(trainer=trainer, classifier=cls)


def case_grids(ops, case, device="cpu", vis_ops=None):
    from gangealing_b200.training import visuals as V
    name, k, flips, n_mean, vb, kind = case
    trainer, ct = mirror_models(ops, k, flips, device)
    z, big_z, reals, loader = [x.to(device) if torch.is_tensor(x) else [b.to(device) for b in x] for x in GT.inputs()]
    torch.manual_seed(GT.NOISE_SEED)
    if kind == "classifier":
        return V.classifier_visuals(ct, loader, n_mean, GT.N_SAMPLE, ops=vis_ops)
    return V.training_visuals(trainer, z, big_z if k > 1 else None, reals, loader, n_mean, GT.N_SAMPLE, vb, ops=vis_ops)


def compare_to_fixture(grids, blob, case, skip=()):
    """Every grid's shape and sums, and its stored pixels: at most 0.5 % differ, each by one step (pixels that pass
    through the mirror STN / generator may land on the other side of a quantisation step).  -> (differing, total)."""
    names = GT.grid_names(blob, case)
    assert sorted(grids) == names, "%s: grids %s, the reference logs %s" % (case, sorted(grids), names)
    differ = total = 0
    for name in names:
        got = grids[name].cpu()
        assert tuple(got.shape) == tuple(blob["%s.%s.shape" % (case, name)].tolist()), "%s.%s shape" % (case, name)
        if name in skip:
            continue
        want = blob["%s.%s" % (case, name)]
        d = (GT.decimate(name, got).long() - want.long()).abs()
        n = int((d > 0).sum())
        print("%s.%s: %d of %d stored values differ (max %d)" % (case, name, n, d.numel(), int(d.max())))
        assert int(d.max()) <= 1 and n <= DIFFER_BOUND * d.numel(), "%s.%s: %d values differ, max %d" % (case, name, n,
                                                                                                        int(d.max()))
        pixels = got.size(0) * got.size(1)
        assert (got.long().sum((0, 1)) - blob["%s.%s.sums" % (case, name)]).abs().max() <= DIFFER_BOUND * pixels
        differ, total = differ + n, total + d.numel()
    return differ, total
