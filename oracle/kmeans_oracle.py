"""Float64 numpy restatement of the k-means kernels (unispeech_b200/csrc/kmeans.cu) and of KMeans.fit's Lloyd loop.

assign   labels = argmin_k (|c_k|^2 - 2 x . c_k), ties to the lowest k (np.argmin); score = that minimum
update   counts, sums per cluster; inertia = sum (|x|^2 + score)
centres  sum / count; an empty cluster keeps its previous centre (scipy.cluster.vq.kmeans2's rule)
lloyd    assign -> update -> centres, stopping when no label changes (then the last labels belong to the final centres) or after
         max_iter iterations (then one more assign with the final centres gives the labels and the inertia); n_iter counts updates.
"""
from __future__ import annotations

import numpy as np


def scores(x, centers):
    x = np.asarray(x, dtype=np.float64)
    c = np.asarray(centers, dtype=np.float64)
    return (c * c).sum(1)[None, :] - 2.0 * (x @ c.T)


def assign(x, centers):
    s = scores(x, centers)
    lab = np.argmin(s, axis=1)
    return lab.astype(np.int64), s[np.arange(s.shape[0]), lab]


def update(x, labels, score, K):
    x = np.asarray(x, dtype=np.float64)
    counts = np.bincount(labels, minlength=K)
    sums = np.zeros((K, x.shape[1]))
    np.add.at(sums, labels, x)
    inertia = float((x * x).sum() + np.sum(score))
    return counts, sums, inertia


def new_centers(sums, counts, centers):
    out = np.array(centers, dtype=np.float64, copy=True)
    nz = counts > 0
    out[nz] = sums[nz] / counts[nz, None]
    return out


def inertia(x, centers, labels):
    x = np.asarray(x, dtype=np.float64)
    d = x - np.asarray(centers, dtype=np.float64)[labels]
    return float((d * d).sum())


def lloyd(x, centers, max_iter=100):
    """Returns (centres, labels, inertia, n_iter).  The inertia is the direct sum of squared distances."""
    x = np.asarray(x, dtype=np.float64)
    c = np.asarray(centers, dtype=np.float64)
    K = c.shape[0]
    prev = np.full(x.shape[0], -1)
    for it in range(max_iter):
        lab, sc = assign(x, c)
        counts, sums, _ = update(x, lab, sc, K)
        c = new_centers(sums, counts, c)
        if np.array_equal(lab, prev):
            return c, lab, inertia(x, c, lab), it + 1
        prev = lab
    lab, _ = assign(x, c)
    return c, lab, inertia(x, c, lab), max_iter
