"""CPU: the latent learner's initialisers (reference train.py:228-243).  The Gram-form IncrementalPCA oracle against the
reference-generated fixture (sklearn), the package's PCA on the oracle op set against the oracle, k-means++ against the
reference's per-round distances, Trainer.init_target_mode in place, and a 2-rank gloo run."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import make_golden_pca as MG
from oracle import pca as OP
from ranks import run_ranks

SKLEARN_COMPONENTS = 1e-5     # oracle (float64 batches) vs sklearn (float32 batch centring, float32 first SVD)


def _case_inputs(blob, name):
    n, d, k, n_upd, seed = [int(v) for v in blob[name + ".shape"]]
    w = MG.case_latents(seed, n + n_upd + MG.ENCODE_ROWS, d)
    return w[:n], w[n:n + n_upd], w[n + n_upd:], k


def _names(blob):
    return [c[0] for c in MG.PCA_CASES if c[0] + ".shape" in blob]


def test_oracle_matches_the_reference_incremental_pca():
    blob = load_golden("latent_pca")
    assert len(_names(blob)) == len(MG.PCA_CASES)
    for name in _names(blob):
        fit, upd, enc, k = _case_inputs(blob, name)
        st = OP.ipca(fit.numpy(), k)
        np.testing.assert_allclose(st["components"], blob[name + ".components"].numpy(), rtol=0, atol=SKLEARN_COMPONENTS,
                                   err_msg=name)
        np.testing.assert_allclose(st["mean"], blob[name + ".mean"].numpy(), rtol=0, atol=1e-12, err_msg=name)
        np.testing.assert_allclose(st["singular_values"], blob[name + ".singular_values"].numpy(), rtol=1e-6, err_msg=name)
        if len(upd):
            st2 = OP.ipca(upd.numpy(), k, state=st)
            np.testing.assert_allclose(st2["components"], blob[name + ".update.components"].numpy(), rtol=0,
                                       atol=SKLEARN_COMPONENTS, err_msg=name + " update")
            np.testing.assert_allclose(st2["mean"], blob[name + ".update.mean"].numpy(), rtol=0, atol=1e-12)
        else:
            # encode is stored for the fit when no update follows
            ref = blob[name + ".encode"].numpy()
            np.testing.assert_allclose(OP.encode(st, enc.numpy()), ref, rtol=0, atol=1e-4 * np.abs(ref).max(), err_msg=name)


def test_batch_offsets_are_sklearns_gen_batches():
    from gangealing_b200.training.latent_learner import gen_batches
    assert gen_batches(2 * 2560 + 3, 2560, 5) == [0, 2560, 5123]            # remainder < k: absorbed into the last batch
    assert gen_batches(2 * 2560 + 900, 2560, 5) == [0, 2560, 5120, 6020]    # kept as a batch of its own
    assert gen_batches(1000, 2560, 1) == [0, 1000]
    assert gen_batches(7, 3, 3) == [0, 3, 7]
    for n, bs, k in ((10, 3, 2), (12000, 2560, 20), (5, 2560, 1)):
        assert gen_batches(n, bs, k) == OP.gen_batches(n, bs, k)


def test_pca_on_the_oracle_op_set_equals_the_oracle():
    from gangealing_b200.training.latent_learner import PCA
    blob = load_golden("latent_pca")
    for name in ("absorbed_k5", "d64_k5", "n1000_k1"):
        fit, upd, enc, k = _case_inputs(blob, name)
        pca = PCA(k, fit, ops=OP.cpu_ops())
        st = OP.ipca(fit.numpy(), k)
        assert pca.pca is pca and pca.n_samples_seen_ == len(fit)
        assert pca.components_.dtype == np.float64 and pca.components_.shape == (k, fit.shape[1])
        np.testing.assert_allclose(pca.components_, st["components"], rtol=0, atol=1e-12, err_msg=name)
        np.testing.assert_allclose(pca.mean_, st["mean"], rtol=0, atol=1e-12)
        np.testing.assert_allclose(pca.singular_values_, st["singular_values"], rtol=1e-12)
        if len(upd):
            pca.update(upd)
            st = OP.ipca(upd.numpy(), k, state=st)
            np.testing.assert_allclose(pca.components_, st["components"], rtol=0, atol=1e-12, err_msg=name + " update")
            np.testing.assert_allclose(pca.mean_, st["mean"], rtol=0, atol=1e-12)
        code = pca.encode(enc)
        assert code.dtype == torch.float64 and code.shape == (len(enc), k)
        np.testing.assert_allclose(code.numpy(), OP.encode(st, enc.numpy()), rtol=0, atol=1e-9)
    with pytest.raises(ValueError, match="batch number of samples"):
        PCA(5, fit[:3], ops=OP.cpu_ops())


def test_assign_buffers_takes_the_package_pca():
    from gangealing_b200.training.latent_learner import PCA, DirectionInterpolator
    blob = load_golden("latent_pca")
    fit, _, _, k = _case_inputs(blob, "d64_k5")
    pca = PCA(k, fit, ops=OP.cpu_ops())
    ll = DirectionInterpolator(None, k, 3, 8, num_heads=2, dim_latent=64)
    ll.assign_buffers(pca)
    assert torch.equal(ll.directions, torch.from_numpy(pca.components_).float())
    assert torch.equal(ll.lat_mean, torch.from_numpy(pca.mean_[None]).float())
    ptr = ll.coefficients.data_ptr()
    ll.assign_coefficients(torch.arange(2 * k, dtype=torch.float64).reshape(2, k))
    assert ll.coefficients.data_ptr() == ptr and ll.coefficients.requires_grad
    assert torch.equal(ll.coefficients.detach(), torch.arange(2 * k, dtype=torch.float32).reshape(2, k))


def test_kmeans_plusplus_on_the_oracle_op_set_matches_the_reference():
    from oracle import opset
    blob = load_golden("latent_pca")
    w, centroids, dists, probs = MG.run_kmeans(blob, "cpu", opset.cpu_ops())
    ref_d, ref_p = blob["kmeans.dists"], blob["kmeans.logits"]
    assert dists.shape == ref_d.shape and probs.shape == ref_p.shape
    assert (dists - ref_d).abs().max() <= 1e-4 * ref_d.abs().max()
    assert (probs - ref_p).abs().max() <= 1e-4 * ref_p.abs().max()
    assert torch.equal(centroids, w[blob["kmeans.draws"].long()])
    assert (centroids - blob["kmeans.centroids"]).abs().max() <= 1e-4 * blob["kmeans.centroids"].abs().max()


def _small_config(**kw):
    from gangealing_b200.training import TrainConfig
    base = dict(gen_size=64, flow_size=64, dim_latent=64, n_mlp=1, batch=1, inject=3, stn_channel_multiplier=0.25,
                gen_channel_multiplier=1, seed=7)
    base.update(kw)
    return TrainConfig(**base)


@pytest.mark.parametrize("heads,ndirs", [(1, 1), (3, 2)])
def test_init_target_mode_writes_the_reference_initialisation_in_place(heads, ndirs):
    from gangealing_b200.training import Trainer
    tr = Trainer(_small_config(num_heads=heads, ndirs=ndirs), "cpu", ops=OP.cpu_ops())
    ll = tr.ll_module
    ptrs = [t.data_ptr() for t in (ll.directions, ll.lat_mean, ll.coefficients)]
    state = torch.random.get_rng_state()
    w = tr.generator.batch_latent(1000)
    centroids = tr.generator.batch_latent(heads) if heads > 1 else None
    torch.random.set_rng_state(state)
    assert not tr.load_checkpoint({"g_ema": tr.generator.state_dict()}, load_G_only=True)
    pca = tr.init_target_mode(n_pca=10 ** 9, debug=True)       # debug: 1000 latents, random centroids
    st = OP.ipca(w.detach().numpy(), ndirs)
    assert [t.data_ptr() for t in (ll.directions, ll.lat_mean, ll.coefficients)] == ptrs
    np.testing.assert_allclose(pca.components_, st["components"], rtol=0, atol=1e-10)
    assert torch.equal(ll.directions, torch.from_numpy(pca.components_).float())
    assert torch.equal(ll.lat_mean, torch.from_numpy(pca.mean_[None]).float())
    if heads > 1:
        want = torch.from_numpy(OP.encode(st, centroids.detach().numpy())).float()
        assert (ll.coefficients.detach() - want).abs().max() <= 1e-5 * want.abs().max()
    else:
        assert torch.equal(ll.coefficients.detach(), torch.zeros(1, ndirs))


def _worker(rank, world, ret):
    from oracle import pca as OP_
    from gangealing_b200.training import Trainer
    from gangealing_b200.training import distributed as gdist
    tr = Trainer(_small_config(num_heads=2, ndirs=2), "cpu", ops=OP_.cpu_ops(), distributed=True)
    state = torch.random.get_rng_state()
    mine = tr.generator.batch_latent(3000 // world)
    torch.random.set_rng_state(state)
    pca = tr.init_target_mode(n_pca=3000, n_kmeans=8)
    everyone = gdist.all_gather(mine.detach())
    ll = tr.ll_module
    params = gdist.all_gather(torch.cat([ll.directions.reshape(-1), ll.lat_mean.reshape(-1),
                                         ll.coefficients.detach().reshape(-1)])[None])
    if rank == 0:
        st = OP_.ipca(everyone.numpy(), 2)
        ret["components_err"] = float(np.abs(pca.components_ - st["components"]).max())
        ret["mean_err"] = float(np.abs(pca.mean_ - st["mean"]).max())
        ret["seen"] = pca.n_samples_seen_
        ret["ranks_equal"] = bool(torch.equal(params[0], params[1]))


@pytest.mark.timeout(600)
def test_two_rank_init_target_mode_equals_the_fit_over_the_gathered_latents_gloo():
    ret = run_ranks(_worker, 560)
    assert ret["seen"] == 3000
    assert ret["components_err"] <= 1e-10 and ret["mean_err"] <= 1e-12
    assert ret["ranks_equal"]
