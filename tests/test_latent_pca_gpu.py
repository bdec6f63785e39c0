"""GPU: the latent learner's initialisers on the device.  `batch_gram` (csrc/pca.cu, fp64 tensor cores) against float64
numpy, its repeatability and argument errors; the device PCA against the Gram-form oracle and the reference's sklearn
fixture; k-means++ against the reference's per-round distances; Trainer.init_target_mode in place."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import make_golden_pca as MG
from oracle import pca as OP

DEV = "cuda"
GRAM_RTOL = 1e-12          # fp64 sums of <= 5120 products: rounding ~ n * 2^-53 of the largest entry, with margin
SKLEARN_COMPONENTS = 1e-5  # measured oracle vs sklearn: <= 3.9e-6 (float32 batch centring in sklearn, float64 here)

GRAM_CASES = [
    # n, D, offsets
    (5, 64, [0, 5]),                          # fewer rows than one 32-row stage
    (100, 64, [0, 37, 38, 100]),              # ragged blocks, one of a single row
    (777, 512, [0, 777]),                     # one block
    (3000, 512, [0, 1000, 2000, 3000]),
    (2600, 512, [3, 2563, 2600]),             # rows before the first offset are not read
]


def _latents(n, d, seed):
    return MG.case_latents(seed, n, d)


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(GRAM_CASES)))
def test_batch_gram_equals_float64_numpy(case):
    from gangealing_b200.op.pca import batch_gram
    n, d, off = GRAM_CASES[case]
    w = _latents(n, d, 100 + case) + 3.0         # an offset mean: centring must happen before the products
    gram, mean = batch_gram(w.to(DEV), off)
    assert gram.dtype == torch.float64 and gram.shape == (len(off) - 1, d, d) and mean.shape == (len(off) - 1, d)
    x = w.numpy().astype(np.float64)
    for b, (a, e) in enumerate(zip(off[:-1], off[1:])):
        mu = x[a:e].mean(0)
        g = (x[a:e] - mu).T @ (x[a:e] - mu)
        np.testing.assert_allclose(mean[b].cpu().numpy(), mu, rtol=0, atol=GRAM_RTOL * np.abs(mu).max())
        scale = max(np.abs(g).max(), 1e-300)
        err = np.abs(gram[b].cpu().numpy() - g).max()
        assert err <= GRAM_RTOL * scale, "block %d: %.3e > %.1e * %.3e" % (b, err, GRAM_RTOL, scale)
    assert torch.equal(gram, gram.transpose(1, 2))


@pytest.mark.gpu
def test_batch_gram_is_bitwise_repeatable():
    from gangealing_b200.op.pca import batch_gram
    w = _latents(6000, 512, 7).to(DEV)
    off = OP.gen_batches(6000, 2560, 5)
    g1, m1 = batch_gram(w, off)
    g2, m2 = batch_gram(w, off)
    assert torch.equal(g1, g2) and torch.equal(m1, m2)


@pytest.mark.gpu
def test_batch_gram_argument_errors():
    from gangealing_b200 import _lib
    from gangealing_b200.op.pca import batch_gram
    dll = _lib.load()
    w = torch.zeros(64, 128, device=DEV)
    g = torch.empty(2, 128, 128, dtype=torch.float64, device=DEV)
    m = torch.empty(2, 128, dtype=torch.float64, device=DEV)

    def call(off, d=128, wp=None, gp=None):
        arr = (ctypes.c_int64 * len(off))(*off)
        return dll.gg_batch_gram(g.data_ptr() if gp is None else gp, m.data_ptr(), w.data_ptr() if wp is None else wp,
                                 ctypes.cast(arr, ctypes.c_void_p), len(off) - 1, d, None)

    assert call([0, 32, 64]) == 0
    torch.cuda.synchronize()
    assert call([0, 32, 64], d=96) == -2 and b"multiple of 64" in dll.gg_last_error()
    assert call([0, 32], d=1088) == -2
    assert call([0, 32, 32]) == -1 and b"increase" in dll.gg_last_error()
    assert call([0, 40, 32]) == -1
    assert call([-1, 32]) == -1
    assert call([0, 32], gp=0) == -1 and b"null" in dll.gg_last_error()
    assert call([0, 32], wp=w.data_ptr() + 4) == -1 and b"aligned" in dll.gg_last_error()
    assert call([0], d=128) == -1
    with pytest.raises(RuntimeError, match="exceeds"):
        batch_gram(w, [0, 65])
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        batch_gram(w.cpu(), [0, 64])
    with pytest.raises(RuntimeError, match="float32"):
        batch_gram(w.double(), [0, 64])


@pytest.mark.gpu
def test_device_pca_equals_the_oracle_and_the_reference_fixture():
    from gangealing_b200.training.latent_learner import PCA
    blob = load_golden("latent_pca")
    for name, n, d, k, n_upd, seed in MG.PCA_CASES:
        w = MG.case_latents(seed, n + n_upd + MG.ENCODE_ROWS, d)
        fit, upd, enc = w[:n], w[n:n + n_upd], w[n + n_upd:]
        pca = PCA(k, fit.to(DEV))
        st = OP.ipca(fit.numpy(), k)
        assert pca.components_.dtype == np.float64
        np.testing.assert_allclose(pca.components_, st["components"], rtol=0, atol=1e-9, err_msg=name)
        np.testing.assert_allclose(pca.mean_, st["mean"], rtol=0, atol=1e-12, err_msg=name)
        np.testing.assert_allclose(pca.components_, blob[name + ".components"].numpy(), rtol=0, atol=SKLEARN_COMPONENTS,
                                   err_msg=name + " vs sklearn")
        np.testing.assert_allclose(pca.singular_values_, blob[name + ".singular_values"].numpy(), rtol=1e-6)
        if n_upd:
            pca.update(upd.to(DEV))
            st = OP.ipca(upd.numpy(), k, state=st)
            np.testing.assert_allclose(pca.components_, st["components"], rtol=0, atol=1e-9, err_msg=name + " update")
            np.testing.assert_allclose(pca.components_, blob[name + ".update.components"].numpy(), rtol=0,
                                       atol=SKLEARN_COMPONENTS, err_msg=name + " update vs sklearn")
        code = pca.encode(enc.to(DEV))
        assert code.device.type == "cuda" and code.dtype == torch.float64
        np.testing.assert_allclose(code.cpu().numpy(), OP.encode(st, enc.numpy()), rtol=0, atol=1e-8)
        if not n_upd:
            ref = blob[name + ".encode"].numpy()
            np.testing.assert_allclose(code.cpu().numpy(), ref, rtol=0, atol=1e-4 * np.abs(ref).max())


@pytest.mark.gpu
def test_kmeans_plusplus_on_the_device_matches_the_reference():
    from gangealing_b200.opset import cuda_ops
    blob = load_golden("latent_pca")
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        w, centroids, dists, probs = MG.run_kmeans(blob, DEV, cuda_ops())
    finally:
        torch.backends.cudnn.allow_tf32 = old
    ref_d, ref_p = blob["kmeans.dists"], blob["kmeans.logits"]
    assert dists.shape == ref_d.shape and probs.shape == ref_p.shape
    assert (dists - ref_d).abs().max() <= 1e-3 * ref_d.abs().max()
    assert (probs - ref_p).abs().max() <= 1e-3 * ref_p.abs().max()
    assert centroids.is_cuda and torch.equal(centroids, w[blob["kmeans.draws"].to(DEV).long()])


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["config2", "config5"])
def test_init_target_mode_on_the_device_in_place(config):
    from gangealing_b200.training import TrainConfig, Trainer
    cfg = TrainConfig() if config == "config2" else TrainConfig(num_heads=4, ndirs=5, inject=6)
    tr = Trainer(cfg, DEV)
    ll = tr.ll_module
    ptrs = [t.data_ptr() for t in (ll.directions, ll.lat_mean, ll.coefficients)]
    state = torch.cuda.get_rng_state()
    w = tr.generator.batch_latent(1000)
    centroids = tr.generator.batch_latent(cfg.num_heads) if cfg.num_heads > 1 else None
    torch.cuda.set_rng_state(state)
    assert not tr.load_checkpoint({"g_ema": tr.generator.state_dict()}, load_G_only=True)
    pca = tr.init_target_mode(debug=True)
    st = OP.ipca(w.detach().cpu().numpy(), cfg.ndirs)
    assert [t.data_ptr() for t in (ll.directions, ll.lat_mean, ll.coefficients)] == ptrs
    np.testing.assert_allclose(pca.components_, st["components"], rtol=0, atol=1e-9)
    assert torch.equal(ll.directions.cpu(), torch.from_numpy(pca.components_).float())
    assert torch.equal(ll.lat_mean.cpu(), torch.from_numpy(pca.mean_[None]).float())
    if centroids is not None:
        want = torch.from_numpy(OP.encode(st, centroids.detach().cpu().numpy())).float()
        assert (ll.coefficients.detach().cpu() - want).abs().max() <= 1e-5 * want.abs().max()
    out = tr.step()                                   # the fused optimiser's pointer table still addresses the learner
    assert all(torch.isfinite(v).item() for v in out.values())
