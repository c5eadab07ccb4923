"""K-means without a GPU: the float64 oracle (oracle/kmeans_oracle.py) against scipy.cluster.vq.kmeans2 and scikit-learn's
Lloyd, and the host-side argument checks of unispeech_b200.kmeans.KMeans."""
import warnings

import numpy as np
import pytest
import torch

from oracle import kmeans_oracle as KO


def blobs(n_per, centers, spread, seed):
    rng = np.random.default_rng(seed)
    c = np.asarray(centers, dtype=np.float64)
    x = np.concatenate([ci + spread * rng.standard_normal((n_per, c.shape[1])) for ci in c])
    return x[rng.permutation(x.shape[0])]


def blob_problem(K=6, D=16, n_per=200, seed=0, spread=1.0):
    """Well-separated blobs and starting centres one per blob, off its mean (no cluster empties: scikit-learn would relocate it)."""
    rng = np.random.default_rng(seed + 100)
    truth = 10.0 * rng.standard_normal((K, D))
    x = blobs(n_per, truth, spread, seed)
    init = truth + 1.5 * spread * rng.standard_normal((K, D))
    return x, init


def test_oracle_lloyd_equals_kmeans2():
    from scipy.cluster.vq import kmeans2
    x, init = blob_problem()
    c, lab, _, n_iter = KO.lloyd(x, init, max_iter=50)
    assert n_iter < 50   # converged: further kmeans2 iterations change nothing
    c2, lab2 = kmeans2(x, init.copy(), iter=50, minit="matrix", missing="warn")
    np.testing.assert_allclose(c, c2, rtol=0, atol=1e-10)
    assert np.array_equal(lab, lab2)


def test_oracle_empty_cluster_keeps_its_centre_like_kmeans2():
    from scipy.cluster.vq import kmeans2
    x, init = blob_problem(K=4, D=8, n_per=100, seed=3)
    init = np.concatenate([init, np.full((1, 8), 1e3)])   # a centre no point is nearest to
    c, lab, _, _ = KO.lloyd(x, init, max_iter=30)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        c2, lab2 = kmeans2(x, init.copy(), iter=30, minit="matrix", missing="warn")
    assert not np.any(lab == 4)
    np.testing.assert_array_equal(c[4], init[4])
    np.testing.assert_allclose(c, c2, rtol=0, atol=1e-10)
    assert np.array_equal(lab, lab2)


@pytest.mark.parametrize("max_iter", [1, 100])
def test_oracle_lloyd_equals_sklearn(max_iter):
    from sklearn.cluster import KMeans as SkKMeans
    x, init = blob_problem(K=8, D=32, n_per=150, seed=5)
    c, lab, inertia, n_iter = KO.lloyd(x, init, max_iter=max_iter)
    sk = SkKMeans(n_clusters=8, init=init, n_init=1, max_iter=max_iter, tol=0.0, algorithm="lloyd").fit(x)
    np.testing.assert_allclose(c, sk.cluster_centers_, rtol=0, atol=1e-9)
    assert np.array_equal(lab, sk.labels_)
    assert inertia == pytest.approx(sk.inertia_, rel=1e-10)
    assert n_iter == sk.n_iter_


def test_oracle_assign_equals_sklearn_predict():
    from sklearn.cluster import KMeans as SkKMeans
    x, init = blob_problem(K=5, D=24, n_per=120, seed=7)
    sk = SkKMeans(n_clusters=5, init=init, n_init=1, max_iter=3, algorithm="lloyd").fit(x)
    q = np.random.default_rng(1).standard_normal((500, 24)) * 12.0
    lab, sc = KO.assign(q, sk.cluster_centers_)
    assert np.array_equal(lab, sk.predict(q))
    d = ((q[:, None, :] - sk.cluster_centers_[None]) ** 2).sum(-1)
    np.testing.assert_allclose(sc + (q * q).sum(1), d.min(1), rtol=1e-9, atol=1e-9)


def test_oracle_assign_ties_go_to_the_lowest_index():
    c = np.array([[1.0, 0.0], [0.0, 1.0], [1.0, 0.0], [0.0, 1.0]])
    x = np.array([[1.0, 1.0], [2.0, 0.0], [0.0, 3.0]])
    lab, _ = KO.assign(x, c)
    assert lab.tolist() == [0, 0, 1]


def test_host_argument_checks():
    from unispeech_b200.kmeans import KMeans
    for bad in (dict(n_clusters=0), dict(n_clusters=1025), dict(n_clusters=4, max_iter=0), dict(n_clusters=4, n_init=0),
                dict(n_clusters=4, tol=-1.0), dict(n_clusters=4, init_size=3), dict(n_clusters=4, seed=-1)):
        with pytest.raises(ValueError):
            KMeans(**bad)
    km = KMeans(1024, max_iter=5, tol=1e-4, init_size=2048, n_init=3, seed=7)
    assert (km.n_clusters, km.max_iter, km.tol, km.init_size, km.n_init, km.seed) == (1024, 5, 1e-4, 2048, 3, 7)
    with pytest.raises(ValueError):
        KMeans.from_centers(np.zeros((4, 39)))          # D % 64 != 0: zero-pad first
    with pytest.raises(ValueError):
        KMeans.from_centers(np.zeros(64))
    km = KMeans.from_centers(np.arange(3 * 64, dtype=np.float64).reshape(3, 64))
    assert km.n_clusters == 3 and km.cluster_centers_.dtype == torch.float32 and km.cluster_centers_.shape == (3, 64)
    assert KMeans.from_centers(torch.ones(2, 128, dtype=torch.float16)).cluster_centers_.dtype == torch.float32
    # no CPU fallback: host tensors are refused before any kernel call
    with pytest.raises(TypeError, match="no CPU fallback"):
        km.predict(torch.zeros(5, 64, dtype=torch.bfloat16))
    with pytest.raises(TypeError):
        KMeans(2).fit(torch.zeros(8, 64))
    with pytest.raises(RuntimeError, match="not fitted"):
        KMeans(2)._device_centers(torch.device("cpu"))
