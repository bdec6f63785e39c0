"""DirectionInterpolator -- learned truncation of the aligned target's latent (host-side mirror of reference
models/latent_learner.py:25-82; buffers `directions`, `lat_mean`, parameter `coefficients`) -- and the initialisers that
fill it from a pre-trained generator (reference train.py:228-243): `PCA` (reference :8-22) and `kmeans_plusplus`
(reference :85-123).  Offline benchmarks use seeded random `directions`/`lat_mean` buffers."""
import numpy as np
import torch
import torch.nn as nn

from . import distributed as gdist


def gen_batches(n, batch_size, min_batch_size=0):
    """Row offsets of sklearn.utils.gen_batches(n, batch_size, min_batch_size), the batches IncrementalPCA.fit takes:
    full batches, with a remainder smaller than min_batch_size absorbed into the last of them."""
    offsets, start = [0], 0
    for _ in range(n // batch_size):
        end = start + batch_size
        if end + min_batch_size > n:
            continue
        offsets.append(end)
        start = end
    if start < n:
        offsets.append(n)
    return offsets


class PCA:
    """sklearn's IncrementalPCA(n_components) fitted to `w_batch` (reference models/latent_learner.py:8-22), computed on
    the tensor's device.

    IncrementalPCA keeps only the top k directions between its batches of 5 * D rows, so its result is not the exact PCA.
    Each partial_fit step is an SVD whose right singular vectors are the eigenvectors of the Gram matrix
        A = V^T diag(s^2) V + G_b + c^2 d d^T,   G_b = sum_rows (x - mean_b)(x - mean_b)^T,   d = mean - mean_b,
    c^2 = seen * b / (seen + b) (A = G_b for the first batch).  The per-batch means and Grams do not depend on the running
    fit: ONE `batch_gram` call computes all of them (fp64 tensor cores), then a chain of float64 eigensolves on the device
    consumes them.  Batches are centred in float64 where sklearn centres float32 batches in float32.

    `components_` (k, D), `singular_values_` (k,) and `mean_` (D,) are float64 numpy arrays, as sklearn's; `pca.pca` is
    the object itself, so reference callers that reach the sklearn estimator through it (`assign_buffers`) work unchanged.
    `ops`: None = the sm_90a op set; tests pass the oracle's (oracle.pca.cpu_ops())."""

    def __init__(self, n_components, w_batch, ops=None):
        self.n_components = int(n_components)
        self.ops = ops
        self.n_samples_seen_ = 0
        self._V = self._s = self._mu = None
        self._fit(w_batch, gen_batches(w_batch.size(0), 5 * w_batch.size(1), self.n_components))

    @property
    def pca(self):
        return self

    def update(self, w_batch):
        """Continue the fit with `w_batch` as one batch (IncrementalPCA.partial_fit)."""
        self._fit(w_batch, [0, w_batch.size(0)])

    def encode(self, x):
        """IncrementalPCA.transform: (x - mean_) @ components_^T, float64, on x's device."""
        mean = torch.from_numpy(self.mean_).to(x.device)
        comps = torch.from_numpy(self.components_).to(x.device)
        return (x.detach().to(torch.float64) - mean) @ comps.T

    def _fit(self, w, offsets):
        k = self.n_components
        if w.dim() != 2 or not 1 <= k <= w.size(1):
            raise ValueError("PCA: n_components=%d must be between 1 and the %s latents' width" % (k, tuple(w.shape)))
        sizes = [b - a for a, b in zip(offsets[:-1], offsets[1:])]
        if not sizes or min(sizes) < k:
            raise ValueError("PCA: n_components=%d must be less or equal to the batch number of samples %d"
                             % (k, min(sizes) if sizes else 0))
        ops = self.ops
        if ops is None:
            from ..opset import cuda_ops
            ops = cuda_ops()
        gram, mean = ops.batch_gram(w.detach().float(), offsets)
        V, s, mu, seen = self._V, self._s, self._mu, self.n_samples_seen_
        for b, nb in enumerate(sizes):
            if seen == 0:
                A, mu = gram[b], mean[b]
            else:
                delta = mu - mean[b]
                A = (V.T * s.square()) @ V + gram[b] + (seen * nb / (seen + nb)) * torch.outer(delta, delta)
                mu = (seen * mu + nb * mean[b]) / (seen + nb)
            lam, E = torch.linalg.eigh(A)
            V = E[:, -k:].flip(1).T.contiguous()
            s = lam[-k:].flip(0).clamp_min(0).sqrt()
            seen += nb
        self._V, self._s, self._mu, self.n_samples_seen_ = V, s, mu, seen
        # sklearn's svd_flip(u_based_decision=False): the largest |entry| of every component is positive
        signs = V.gather(1, V.abs().argmax(1, keepdim=True)).sign()
        self.components_ = (V * signs).cpu().numpy()
        self.singular_values_ = s.cpu().numpy()
        self.mean_ = mu.cpu().numpy()


class DirectionInterpolator(nn.Module):
    def __init__(self, pca_path, n_comps, inject_index, n_latent, num_heads=1, initializer=None, dim_latent=512):
        super().__init__()
        if pca_path is not None:
            with np.load(pca_path) as data:
                self.register_buffer("lat_mean", torch.from_numpy(data["lat_mean"]))
                self.register_buffer("directions", torch.from_numpy(data["lat_comp"].squeeze(axis=1))[:n_comps])
        else:
            self.register_buffer("directions", torch.randn(n_comps, dim_latent))
            self.register_buffer("lat_mean", torch.randn(1, dim_latent))
        if initializer is None:
            initializer = torch.zeros(num_heads, n_comps)
        self.coefficients = nn.Parameter(initializer.detach().clone())
        self.n_latent, self.inject_index, self.num_heads = n_latent, inject_index, num_heads

    def forward(self, styled_latent, psi=None, lat_mean=None, pca=None, unfold=False, split=False):
        if pca is not None:
            return self.assign_buffers(pca)
        return self.interpolate(styled_latent, psi, lat_mean, unfold, split)

    def interpolate(self, styled_latent, psi, lat_mean=None, unfold=False, split=False):
        """-> [(N*K, n_latent, D)], the reference's return value.  split=True: the same latent as the generator's two-latent
        form [(N*K, D) truncated, (N*K, D) fixed] for `inject_index=self.inject_index`: the generator then sees that the
        rows from the inject index up are constants (only `truncated` depends on the coefficients)."""
        assert len(styled_latent) == 1
        w = styled_latent[0]
        n = w.size(0)
        mean = self.lat_mean if lat_mean is None else lat_mean
        target = (mean + self.coefficients @ self.directions).repeat(n, 1)          # (N*K, D)
        w = w.repeat_interleave(self.num_heads, dim=0)
        if split:
            if unfold:
                raise ValueError("DirectionInterpolator: unfold and split are exclusive")
            return [target.lerp(w, psi), w]
        truncated = target.lerp(w, psi).unsqueeze(1).repeat(1, self.inject_index, 1)
        fixed = w.unsqueeze(1).repeat(1, self.n_latent - self.inject_index, 1)
        out = torch.cat([truncated, fixed], dim=1)
        if unfold:
            out = out.reshape(n, self.num_heads, self.n_latent, out.size(-1))
        return [out]

    @torch.no_grad()
    def assign_buffers(self, pca):
        dev = self.directions.device
        self.register_buffer("directions", torch.from_numpy(pca.pca.components_).float().to(dev))
        self.register_buffer("lat_mean", torch.from_numpy(pca.pca.mean_[None]).float().to(dev))

    @torch.no_grad()
    def assign_coefficients(self, initializer):
        """Copy `initializer` (num_heads, n_comps) into the coefficients in place (reference :79-82)."""
        self.coefficients.copy_(initializer)


@torch.no_grad()
def kmeans_plusplus(num_heads, num_latent, G, loss_fn, inject_index=6, batch_size=100):
    """k-means++ seeding of `num_heads` centroids among `num_latent` generated latents (reference :85-123, same
    statements), with the perceptual distance between their images.  The images stay on the device; every rank draws
    num_latent // world latents, the centroid draws are rank 0's.  -> (num_heads, D) centroid latents."""
    num_w_per_gpu = num_latent // gdist.get_world_size()
    batch_w = G.batch_latent(num_w_per_gpu)
    dev = batch_w.device
    mean_w = gdist.all_gather(batch_w.mean(dim=0, keepdim=True)).mean(dim=0, keepdim=True)
    batch_fakes = None    # written batch by batch: 50,000 images at 256^2 are 39 GB, a concatenation would double that
    for i in range(0, num_w_per_gpu, batch_size):
        batch_w_in = batch_w[i:i + batch_size]
        fakes, _ = G([batch_w_in, mean_w.expand_as(batch_w_in)], input_is_latent=True, randomize_noise=True,
                     inject_index=inject_index)
        if batch_fakes is None:
            batch_fakes = fakes.new_empty((num_w_per_gpu,) + tuple(fakes.shape[1:]))
        batch_fakes[i:i + batch_size] = fakes
    batch_w = gdist.all_gather(batch_w)
    # randomly pick the first centroid from the data
    initial_w_idx = torch.randint(low=0, high=num_latent, size=(1,), device=dev)
    initial_w_idx = gdist.rank0_to_all(initial_w_idx).item()
    dists = []
    centroid_idx = [initial_w_idx]
    for _ in range(num_heads - 1):
        # the previous centroid's image, recomputed on every rank, against every data point's
        G_w, _ = G([batch_w[centroid_idx[-1]].unsqueeze(0), mean_w], input_is_latent=True, randomize_noise=True,
                   inject_index=inject_index)
        dist = []
        for i in range(0, num_w_per_gpu, batch_size):
            dist.append(loss_fn(G_w.expand_as(batch_fakes[i:i + batch_size]), batch_fakes[i:i + batch_size]).squeeze())
        dist = gdist.all_gather(torch.cat(dist, 0))
        dists.append(dist)
        # distance of every data point to its nearest centroid; sample the next centroid favouring poorly covered points
        closest = torch.stack(dists).min(dim=0).values
        logits_sqr = closest ** 2
        logits = logits_sqr / logits_sqr.sum()
        next_idx = gdist.rank0_to_all(torch.multinomial(logits, num_samples=1)).item()
        centroid_idx.append(next_idx)
    print("Centroids: %s" % centroid_idx)
    return batch_w[centroid_idx]
