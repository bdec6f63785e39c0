"""Generate tests/golden/latent_pca.npz from the reference's latent-learner initialisers and pin oracle/pca.py against it.

Run where the reference checkout and sklearn are (GG_REFERENCE_ROOT):  python -m oracle.make_golden_pca
  * PCA: the reference's own models.latent_learner.PCA (sklearn IncrementalPCA) fitted to seeded latents (`case_latents`),
    then `update` and `encode`; the Gram-form oracle must reproduce every fit.  Cases: n = 1000 (one batch, the debug
    path), a ragged remainder smaller than k absorbed into the last batch and one kept as its own batch, k = 1, 5, 20,
    D = 512 and 64.  Every component's two largest |entries| differ by at least 1e-4, so the sign rule cannot flip on
    rounding.
  * k-means++: the reference's kmeans_plusplus on the CPU ('cuda' device strings mapped to 'cpu') with a seeded
    Generator(64) whose noise strengths are zero (its images are a function of the latents), the seeded-VGG perceptual
    loss of oracle.make_golden.gen_perceptual_loss, 48 latents, K = 3.  The latents are unit-normal draws (`kmeans_w`):
    the seeded mapping network's outputs are ~1e-3 wide, too alike for the distances to say anything.  torch.randint
    and torch.multinomial are patched: their draws are seeded and stored, with the distances and probabilities of every
    round.
Inputs are rebuilt from seeds (case_latents, kmeans_w, kmeans_generator); only results are stored.
"""
import contextlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import opset  # noqa: E402
from oracle import pca as OP  # noqa: E402

PCA_CASES = [
    # name, n, D, k, rows of the partial_fit update, seed
    ("n1000_k1", 1000, 512, 1, 0, 1),
    ("absorbed_k5", 2 * 2560 + 3, 512, 5, 700, 2),
    ("kept_k5", 2 * 2560 + 900, 512, 5, 0, 3),
    ("k20", 3 * 2560 + 41, 512, 20, 0, 4),
    ("d64_k5", 5 * 320 + 77, 64, 5, 130, 5),
]
ENCODE_ROWS = 4
KMEANS = dict(size=64, style_dim=64, n_mlp=2, channel_multiplier=1, weight_seed=61, latent_seed=62, draw_seed=63,
              num_latent=48, num_heads=3, inject_index=6, batch_size=20, vgg_seed=4242)


def case_latents(seed, n, d):
    """n latents of width d from a seeded random mapping network (pixel norm, 4 x (linear, lrelu * sqrt 2)), float32."""
    g = torch.Generator().manual_seed(seed)
    layers = [torch.randn(d, d, generator=g) / d ** 0.5 for _ in range(4)]
    x = torch.randn(n, d, generator=g)
    x = x * torch.rsqrt(x.square().mean(1, keepdim=True) + 1e-8)
    for W in layers:
        x = torch.nn.functional.leaky_relu(x @ W.T, 0.2) * 2 ** 0.5
    return x.float()


def kmeans_generator(Generator, **kw):
    """The k-means fixture's generator: seeded weights, noise strengths zero."""
    k = KMEANS
    G = Generator(k["size"], k["style_dim"], k["n_mlp"], channel_multiplier=k["channel_multiplier"], **kw).eval()
    opset.fill_parameters(G, k["weight_seed"], gain=0.5)
    with torch.no_grad():
        for name, p in G.named_parameters():
            if name.endswith("noise.weight"):
                p.zero_()
    return G


def kmeans_w():
    return torch.randn(KMEANS["num_latent"], KMEANS["style_dim"], generator=torch.Generator().manual_seed(KMEANS["latent_seed"]))


class FixedLatents:
    """A generator whose batch_latent returns the given latents (the fixture's in place of fresh draws)."""

    def __init__(self, G, w):
        self.G, self.w = G, w

    def batch_latent(self, n):
        assert n == len(self.w)
        return self.w.clone()

    def __call__(self, *args, **kwargs):
        return self.G(*args, **kwargs)


@contextlib.contextmanager
def injected_draws(initial, draws, record=None):
    """torch.randint -> [initial]; torch.multinomial -> draws[i] in order (or, with `record`, a seeded draw appended to
    record["draws"] and the probabilities to record["logits"])."""
    randint, multinomial = torch.randint, torch.multinomial
    calls = [0]
    g = torch.Generator().manual_seed(KMEANS["draw_seed"])

    def fake_randint(*args, device=None, **kwargs):
        if record is not None:        # generating the fixture: the reference's device='cuda' runs on the CPU
            device = "cpu"
        return torch.tensor([int(initial)], device=device)

    def fake_multinomial(p, num_samples=1, **kwargs):
        if record is not None:
            record["logits"].append(p.detach().cpu().clone())
            idx = int(multinomial(p.detach().cpu(), 1, generator=g))
            record["draws"].append(idx)
        else:
            idx = int(draws[calls[0]])
        calls[0] += 1
        return torch.tensor([idx], device=p.device)

    torch.randint, torch.multinomial = fake_randint, fake_multinomial
    try:
        yield
    finally:
        torch.randint, torch.multinomial = randint, multinomial


def kmeans_setup(device, ops):
    """The fixture's generator, perceptual loss and latents, built with this package's modules."""
    from gangealing_b200.stylegan2 import Generator
    from gangealing_b200.training.perceptual import PerceptualLoss
    G = kmeans_generator(Generator, ops=ops).to(device)
    loss = opset.fill_convs_in_order(PerceptualLoss(ops=ops), KMEANS["vgg_seed"]).to(device)
    if device != "cpu":
        loss = loss.to(memory_format=torch.channels_last)
    return G, loss, kmeans_w().to(device)


def run_kmeans(blob, device, ops):
    """This package's kmeans_plusplus with the draws stored in `blob` (the loaded fixture) injected -> (latents,
    centroids, per-round distances, per-round probabilities)."""
    from gangealing_b200.training.latent_learner import kmeans_plusplus
    k = KMEANS
    G, loss, w = kmeans_setup(device, ops)
    dists, probs = [], []

    def loss_fn(a, b):
        d = loss(a, b)
        dists.append(d.detach().reshape(-1).cpu())
        return d

    draws = blob["kmeans.draws"]
    with injected_draws(int(draws[0]), [int(v) for v in draws[1:]]):
        inner = torch.multinomial

        def spy(p, num_samples=1, **kw):       # records each round's probabilities, then returns the stored draw
            probs.append(p.detach().cpu())
            return inner(p, num_samples, **kw)

        torch.multinomial = spy
        try:
            centroids = kmeans_plusplus(k["num_heads"], k["num_latent"], FixedLatents(G, w), loss_fn, k["inject_index"],
                                        k["batch_size"])
        finally:
            torch.multinomial = inner
    per_round = -(-k["num_latent"] // k["batch_size"])
    rounds = torch.stack([torch.cat(dists[r * per_round:(r + 1) * per_round]) for r in range(k["num_heads"] - 1)])
    return w, centroids, rounds, torch.stack(probs)


def gen_pca(ref_ll, out):
    for name, n, d, k, n_upd, seed in PCA_CASES:
        w = case_latents(seed, n + n_upd + ENCODE_ROWS, d)
        fit, upd, enc = w[:n], w[n:n + n_upd], w[n + n_upd:]
        pca = ref_ll.PCA(k, fit)
        oracle = OP.ipca(fit.numpy(), k)
        _check(name, pca.pca, oracle, k)
        out[name + ".components"], out[name + ".singular_values"] = pca.pca.components_, pca.pca.singular_values_
        out[name + ".mean"] = pca.pca.mean_
        if n_upd:
            pca.update(upd)
            oracle = OP.ipca(upd.numpy(), k, state=oracle)
            _check(name + " update", pca.pca, oracle, k)
            out[name + ".update.components"], out[name + ".update.mean"] = pca.pca.components_, pca.pca.mean_
            out[name + ".update.singular_values"] = pca.pca.singular_values_
        out[name + ".encode"] = pca.encode(enc).numpy()
        out[name + ".shape"] = np.array([n, d, k, n_upd, seed])


def _check(name, sk, oracle, k):
    srt = np.sort(np.abs(sk.components_), axis=1)
    margin = (srt[:, -1] - srt[:, -2]).min()
    assert margin >= 1e-4, "%s: sign margin %.2e" % (name, margin)
    err = np.abs(sk.components_ - oracle["components"]).max()
    assert err <= 1e-5, "%s: oracle components off by %.2e" % (name, err)
    assert np.abs(sk.mean_ - oracle["mean"]).max() <= 1e-12
    rel = np.abs(sk.singular_values_ - oracle["singular_values"]).max() / sk.singular_values_.max()
    assert rel <= 1e-6, "%s: singular values off by %.2e" % (name, rel)
    print("%-18s k=%-2d oracle vs sklearn: components %.1e, singular values %.1e (rel), sign margin %.1e"
          % (name, k, err, rel, margin))


def gen_kmeans(ref_ll, out):
    from models.stylegan2.networks import Generator
    import models.losses.lpips as L
    k = KMEANS
    G = kmeans_generator(Generator)
    net = L.LPIPS(net="vgg", lpips=False, pnet_rand=True, verbose=False)
    opset.fill_convs_in_order(net, k["vgg_seed"])
    w = kmeans_w()
    initial = int(torch.randint(0, k["num_latent"], (1,), generator=torch.Generator().manual_seed(k["draw_seed"] + 1)))
    record = dict(logits=[], draws=[])
    dists = []

    def loss_fn(a, b):
        d = net(a, b) / 18.0
        dists.append(d.detach().reshape(-1).clone())
        return d

    to = torch.Tensor.to

    def to_cpu(self, *args, **kwargs):
        return to(self, *["cpu" if a == "cuda" else a for a in args], **kwargs)

    torch.Tensor.to = to_cpu
    try:
        with injected_draws(initial, None, record):
            centroids = ref_ll.kmeans_plusplus(k["num_heads"], k["num_latent"], FixedLatents(G, w), loss_fn,
                                               k["inject_index"], k["batch_size"])
    finally:
        torch.Tensor.to = to
    per_round = k["num_latent"] // k["batch_size"] + (k["num_latent"] % k["batch_size"] > 0)
    out["kmeans.dists"] = torch.stack([torch.cat(dists[r * per_round:(r + 1) * per_round])
                                       for r in range(k["num_heads"] - 1)]).numpy()
    out["kmeans.logits"] = torch.stack(record["logits"]).numpy()
    out["kmeans.draws"] = np.array([initial] + record["draws"])
    out["kmeans.centroids"] = centroids.numpy()
    print("kmeans++: centroids %s" % out["kmeans.draws"].tolist())


def main():
    from oracle import refimport
    from oracle.make_golden import _save
    refimport.import_reference()
    import models.latent_learner as ref_ll
    out = {}
    gen_pca(ref_ll, out)
    gen_kmeans(ref_ll, out)
    _save("latent_pca", **out)


if __name__ == "__main__":
    main()
