"""NumPy pieces of the IVF tests: a seeded clustered fixture and the fp64 spherical k-means update."""
import numpy as np


def gaussian_mixture(n, d, clusters, seed, spread=0.3):
    """float32 [n, d]: rows drawn around `clusters` Gaussian centres (the centres from a fixed seed, so two calls with
    different seeds sample the same mixture)."""
    centres = np.random.default_rng(1000 + clusters * 7 + d).standard_normal((clusters, d))
    rng = np.random.default_rng(seed)
    pick = rng.integers(0, clusters, n)
    return (centres[pick] + spread * rng.standard_normal((n, d))).astype(np.float32)


def update_fp64(X, assign, prev, nlist):
    """New centroids from an assignment: the normalised sum of the members' unit rows; an empty list (or a zero sum)
    keeps its previous centroid."""
    X = X.astype(np.float64)
    nrm = np.sqrt((X ** 2).sum(1, keepdims=True))
    U = np.divide(X, nrm, out=np.zeros_like(X), where=nrm > 0)
    S = np.zeros((nlist, X.shape[1]))
    np.add.at(S, assign, U)
    n = np.sqrt((S ** 2).sum(1, keepdims=True))
    out = prev.astype(np.float64).copy()
    keep = n[:, 0] > 0
    out[keep] = S[keep] / n[keep]
    return out
