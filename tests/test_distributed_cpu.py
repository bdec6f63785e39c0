"""CPU, world_size 2 over gloo: the data-parallel logic of the train step (per-rank latents, DDP gradient
all-reduce keeps replicas identical, rank-0 loss reduce)."""
import pytest
import torch

from ranks import run_ranks


def _worker(rank, world, ret):
    from oracle import opset
    from gangealing_b200.training import TrainConfig, Trainer
    from gangealing_b200.training import distributed as gdist
    cfg = TrainConfig(gen_size=64, flow_size=64, dim_latent=16, n_mlp=1, batch=1, inject=3, seed=3)
    tr = Trainer(cfg, "cpu", ops=opset.cpu_ops(), distributed=True)
    z_probe = torch.randn(2)                      # the per-rank RNG stream differs (train.py:193)
    for _ in range(2):
        out = tr.step()
    flat = torch.cat([p.detach().reshape(-1) for p in tr.t_module.parameters()])
    gathered = gdist.all_gather(flat[None], cat=True)
    probes = gdist.all_gather(z_probe[None], cat=True)
    if rank == 0:
        ret["replicas_equal"] = bool(torch.equal(gathered[0], gathered[1]))
        ret["latents_differ"] = bool(not torch.equal(probes[0], probes[1]))
        ret["loss_keys"] = sorted(out.keys())
        ret["loss_finite"] = bool(all(torch.isfinite(v) for v in out.values()))


@pytest.mark.timeout(600)
def test_two_rank_data_parallel_step_gloo():
    ret = run_ranks(_worker, 560)
    assert ret["replicas_equal"], "DDP replicas diverged"
    assert ret["latents_differ"]
    assert ret["loss_keys"] == ["f", "p", "tv"] and ret["loss_finite"]


def _worker_cluster(rank, world, ret):
    from oracle import opset
    from gangealing_b200.training import ClassifierTrainer, TrainConfig, Trainer
    from gangealing_b200.training import distributed as gdist
    # the exchange helpers on known per-rank values (reference utils/distributed.py:87-100,140-162)
    mine = torch.tensor([1.0 + rank, 10.0 * (rank + 1)])
    mean = gdist.all_reduce_mean(mine)
    red = gdist.reduce_loss_dict({"b": mine[1], "a": mine[0]})
    parts = gdist.all_gather(mine[None], cat=False)
    # BASELINE config 5's shape of work, shrunk: K = 2 heads + flips through gangealing_cluster_loss, then the classifier step
    cfg = TrainConfig(gen_size=64, flow_size=64, dim_latent=16, n_mlp=1, batch=2, inject=3, seed=5, num_heads=2, flips=True,
                      ndirs=2, stn_channel_multiplier=0.25, gen_channel_multiplier=1, padding_mode="reflection")
    tr = Trainer(cfg, "cpu", ops=opset.cpu_ops(), distributed=True)
    out = tr.step()
    ct = ClassifierTrainer(tr, ops=opset.cpu_ops(), distributed=True)
    cout = ct.step()
    stn_flat = torch.cat([p.detach().reshape(-1) for p in tr.t_module.parameters()])
    cls_flat = torch.cat([p.detach().reshape(-1) for p in ct.module.parameters()])
    stn_all, cls_all = gdist.all_gather(stn_flat[None]), gdist.all_gather(cls_flat[None])
    if rank == 0:
        ret["mean"] = mean.tolist()
        ret["reduced"] = {k: float(v) for k, v in red.items()}
        ret["gathered"] = [p.tolist() for p in parts]
        ret["stn_equal"] = bool(torch.equal(stn_all[0], stn_all[1]))
        ret["cls_equal"] = bool(torch.equal(cls_all[0], cls_all[1]))
        ret["finite"] = bool(all(torch.isfinite(v) for v in out.values()) and torch.isfinite(cout["cross_entropy"]))
        ret["hist"] = sum(float(cout["head_%d" % c]) for c in range(4))


@pytest.mark.timeout(900)
def test_two_rank_cluster_step_classifier_step_and_exchange_helpers_gloo():
    ret = run_ranks(_worker_cluster, 860)
    assert ret["mean"] == [1.5, 15.0]
    assert ret["reduced"] == {"a": 1.5, "b": 15.0}                 # rank 0 holds the mean over ranks
    assert ret["gathered"] == [[[1.0, 10.0]], [[2.0, 20.0]]]
    assert ret["stn_equal"], "DDP replicas of the clustering STN diverged"
    assert ret["cls_equal"], "DDP replicas of the classifier diverged"
    assert ret["finite"] and abs(ret["hist"] - 1.0) < 1e-6        # rank-0 mean of per-rank histograms still sums to one
