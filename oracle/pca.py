"""CPU restatement of the latent learner's PCA initialiser (test infrastructure).

sklearn's IncrementalPCA (reference models/latent_learner.py:8-22) keeps only the top k directions between batches of
5 * D rows.  Each of its partial_fit steps is an SVD of M = [s * V; X_b - mean_b; c (mean - mean_b)], c^2 = seen * b /
(seen + b); its right singular vectors are the eigenvectors of the Gram matrix

    A = V^T diag(s^2) V + G_b + c^2 d d^T,   G_b = sum_rows (x - mean_b)(x - mean_b)^T,   d = mean - mean_b

(A = G_b for the first batch), and the singular values are the square roots of the eigenvalues.  `ipca` runs that chain
in numpy float64; `batch_gram_ref` is the float64 torch restatement of the sm_90a `batch_gram` op, and `cpu_ops()` the
oracle op set with it added, so that the package's PCA and Trainer.init_target_mode run on the CPU.
"""
import types

import numpy as np
import torch

from . import opset


def gen_batches(n, batch_size, min_batch_size=0):
    """Row offsets of sklearn.utils.gen_batches(n, batch_size, min_batch_size): full batches, a remainder smaller than
    min_batch_size absorbed into the last of them."""
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


def batch_gram_ref(w, offsets):
    """Float64 restatement of cuda_ops().batch_gram: (gram (B, D, D), mean (B, D)) of the row blocks of w."""
    off = [int(o) for o in offsets]
    x = w.detach().to(torch.float64)
    grams, means = [], []
    for a, b in zip(off[:-1], off[1:]):
        mu = x[a:b].mean(0)
        xc = x[a:b] - mu
        grams.append(xc.T @ xc)
        means.append(mu)
    return torch.stack(grams), torch.stack(means)


def ipca(w, k, state=None, offsets=None):
    """Gram-form IncrementalPCA in numpy float64.  w: (n, D) array; state: the dict a previous call returned (continue
    the fit like partial_fit) or None (fit: batches of 5 * D rows); offsets: explicit row blocks (default: gen_batches
    for a fit, one block when continuing).  -> dict(components (k, D), singular_values (k,), mean (D,), seen)."""
    w = np.asarray(w, dtype=np.float64)
    n, d = w.shape
    if offsets is None:
        offsets = gen_batches(n, 5 * d, k) if state is None else [0, n]
    V, s, mu, seen = (None, None, None, 0) if state is None else (state["components"], state["singular_values"],
                                                                   state["mean"], state["seen"])
    for a, b in zip(offsets[:-1], offsets[1:]):
        x = w[a:b]
        nb = b - a
        mb = x.mean(0)
        G = (x - mb).T @ (x - mb)
        if seen == 0:
            A, mu = G, mb
        else:
            delta = mu - mb
            A = (V.T * s ** 2) @ V + G + (seen * nb / (seen + nb)) * np.outer(delta, delta)
            mu = (seen * mu + nb * mb) / (seen + nb)
        lam, E = np.linalg.eigh(A)
        V = E[:, ::-1][:, :k].T.copy()
        s = np.sqrt(np.maximum(lam[::-1][:k], 0.0))
        seen += nb
    # sklearn's svd_flip(u_based_decision=False): the largest |entry| of every component is positive
    V = V * np.sign(V[np.arange(k), np.abs(V).argmax(1)])[:, None]
    return dict(components=V, singular_values=s, mean=mu, seen=seen)


def encode(state, x):
    """IncrementalPCA.transform: (x - mean) @ components^T in float64."""
    return (np.asarray(x, dtype=np.float64) - state["mean"]) @ state["components"].T


_ops = None


def cpu_ops():
    """oracle.opset.cpu_ops() plus `batch_gram`."""
    global _ops
    if _ops is None:
        _ops = types.SimpleNamespace(**vars(opset.cpu_ops()))
        _ops.batch_gram = batch_gram_ref
    return _ops
