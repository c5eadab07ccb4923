"""K-means pseudo-labels on the library's kernels (`csrc/kmeans.cu`): the label stage of HuBERT-style pre-training.

The HuBERT recipe dumps one layer's features with `extract_features(..., output_layer=L)`, fits scikit-learn's `MiniBatchKMeans`
on the CPU and labels every frame with `argmin(|x|^2 - 2 x.C + |C|^2)`.  Here both steps run on the GPU::

    km = KMeans(500, max_iter=100, init_size=100_000, seed=0).fit(feats)      # feats: CUDA bf16 [N, D] of valid frames
    x, pm = model.extract_features(wav, padding_mask=pad, output_layer=L)     # model.eval(), torch.no_grad()
    labels = km.predict(x, pm)                                                # int32 [B, T], -1 at padded frames

These are not scikit-learn's labels: the fit is full-batch Lloyd (not mini-batch) and the seeding uses the library's
counter-based generator, so compare the quality of two fits by their inertia.  An existing k-means model (for example
`joblib.load(km_path).cluster_centers_` from the recipe) labels on the GPU through `KMeans.from_centers`.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import ops

MAX_CLUSTERS = 1024   # B200S_KMEANS_MAX_K: the pre-training heads' label-set limit
TILE = 256            # centroid tile of the assignment kernel: the bf16 centres are padded to a multiple of it


def _check_features(x: torch.Tensor, dims, what: str):
    if not isinstance(x, torch.Tensor) or not x.is_cuda or x.dtype != torch.bfloat16:
        raise TypeError(f"{what}: expected a CUDA bf16 tensor, got {getattr(x, 'dtype', type(x))} on "
                        f"{getattr(x, 'device', '?')} (no CPU fallback)")
    if x.dim() not in dims:
        raise ValueError(f"{what}: expected {' or '.join(f'{d}-D' for d in dims)} features, got shape {list(x.shape)}")
    if x.shape[-1] % 64 != 0:
        raise ValueError(f"{what}: feature size {x.shape[-1]} is not a multiple of 64 (zero-pad it: distances do not change)")
    if x.stride(-1) != 1:
        raise ValueError(f"{what}: the feature dimension must be contiguous")


class KMeans:
    """Lloyd's k-means over bf16 features on the GPU, k-means++ seeding, scikit-learn-like attributes.

    fit(x) stops after `max_iter` iterations, when no label changes, or when the relative inertia improvement of an iteration is
    <= `tol` (0 disables that test).  Each iteration reads back one small tensor (the changed-label count and the inertia) to
    decide whether to go on: a host synchronisation per iteration, which an offline fit can afford.  `init_size`: rows of a
    random subsample the seeding runs on (None: every row); `n_init` seedings are drawn and the one with the lowest inertia on
    that subsample is kept.  An empty cluster keeps its previous centre (scipy.cluster.vq.kmeans2's rule).

    After fit: `cluster_centers_` (fp32 [K, D] on the device), `labels_` (int32 [N]), `inertia_` (sum of squared distances to
    the assigned centres, from the bf16 features and the bf16 centres), `n_iter_`.
    """

    def __init__(self, n_clusters: int, max_iter: int = 100, tol: float = 0.0, init_size: Optional[int] = None,
                 n_init: int = 1, seed: int = 0):
        if not (1 <= int(n_clusters) <= MAX_CLUSTERS):
            raise ValueError(f"n_clusters={n_clusters} outside [1, {MAX_CLUSTERS}]")
        if int(max_iter) < 1 or int(n_init) < 1:
            raise ValueError(f"max_iter={max_iter} and n_init={n_init} must be >= 1")
        if not tol >= 0.0:
            raise ValueError(f"tol={tol} must be >= 0")
        if init_size is not None and int(init_size) < int(n_clusters):
            raise ValueError(f"init_size={init_size} must be at least n_clusters={n_clusters}")
        if not (0 <= int(seed) < 2 ** 32):
            raise ValueError(f"seed={seed} must fit in 32 bits")
        self.n_clusters = int(n_clusters)
        self.max_iter = int(max_iter)
        self.tol = float(tol)
        self.init_size = None if init_size is None else int(init_size)
        self.n_init = int(n_init)
        self.seed = int(seed)
        self.cluster_centers_: Optional[torch.Tensor] = None
        self.labels_: Optional[torch.Tensor] = None
        self.inertia_: Optional[float] = None
        self.n_iter_ = 0
        self._dev = None   # (centres, bf16 copy [Kp, D], cnorm [Kp]) on the device the assignment last ran on

    @classmethod
    def from_centers(cls, centers) -> "KMeans":
        """A fitted model from existing centres: numpy or torch [K, D] (e.g. the recipe's `joblib.load(km_path).cluster_centers_`)."""
        c = torch.as_tensor(np.asarray(centers.detach().cpu() if isinstance(centers, torch.Tensor) else centers),
                            dtype=torch.float32)
        if c.dim() != 2:
            raise ValueError(f"centers must be [K, D], got shape {list(c.shape)}")
        if c.shape[1] % 64 != 0:
            raise ValueError(f"feature size {c.shape[1]} is not a multiple of 64 (zero-pad centres and features alike)")
        km = cls(c.shape[0])
        km.cluster_centers_ = c.contiguous()
        return km

    # ------------------------------------------------------------------------------------------------------------ internals
    def _device_centers(self, dev: torch.device):
        c = self.cluster_centers_
        if c is None:
            raise RuntimeError("KMeans: not fitted (call fit or use KMeans.from_centers)")
        if self._dev is None or self._dev[0] is not c or self._dev[1].device != dev:
            K, D = c.shape
            cd = c.to(dev).contiguous()
            cbf = torch.empty(-(-K // TILE) * TILE, D, dtype=torch.bfloat16, device=dev)
            cnorm = torch.empty(cbf.shape[0], dtype=torch.float32, device=dev)
            ops.kmeans_centers(None, None, K, D, cd, cbf, cnorm)
            self._dev = (c, cbf, cnorm)
        return self._dev[1], self._dev[2]

    def _seed_centers(self, x: torch.Tensor) -> torch.Tensor:
        N, D = x.shape
        K = self.n_clusters
        n = N if self.init_size is None else min(N, self.init_size)
        xs = x
        if n < N:
            g = torch.Generator().manual_seed(self.seed)
            idx = torch.randperm(N, generator=g)[:n].sort().values.to(x.device)
            xs = x.index_select(0, idx)
        d2 = torch.empty(n, dtype=torch.float32, device=x.device)
        cand = torch.empty(self.n_init, K, D, dtype=torch.float32, device=x.device)
        inertia = torch.empty(self.n_init, dtype=torch.float64, device=x.device)
        for trial in range(self.n_init):
            ops.kmeanspp_init(xs, xs.stride(0), n, D, K, (self.seed, trial), d2, cand[trial], inertia[trial:trial + 1])
        return cand[int(inertia.argmin())].contiguous() if self.n_init > 1 else cand[0]

    # ------------------------------------------------------------------------------------------------------------ public API
    def fit(self, x: torch.Tensor, init_centers=None) -> "KMeans":
        """Fit on `x`: CUDA bf16 [N, D] of valid frames (N >= n_clusters, D a multiple of 64).  `init_centers` ([K, D]) starts
        Lloyd from given centres instead of k-means++."""
        _check_features(x, (2,), "KMeans.fit")
        N, D = x.shape
        K = self.n_clusters
        if N < K:
            raise ValueError(f"KMeans.fit: {N} rows for {K} clusters")
        dev = x.device
        if init_centers is not None:
            centers = torch.as_tensor(init_centers, dtype=torch.float32).to(dev).clone().contiguous()
            if tuple(centers.shape) != (K, D):
                raise ValueError(f"init_centers must be [{K}, {D}], got {list(centers.shape)}")
        else:
            centers = self._seed_centers(x)
        cbf = torch.empty(-(-K // TILE) * TILE, D, dtype=torch.bfloat16, device=dev)
        cnorm = torch.empty(cbf.shape[0], dtype=torch.float32, device=dev)
        ops.kmeans_centers(None, None, K, D, centers, cbf, cnorm)

        labels = torch.empty(N, dtype=torch.int32, device=dev)
        prev = torch.full((N,), -1, dtype=torch.int32, device=dev)
        score = torch.empty(N, dtype=torch.float32, device=dev)
        changed = torch.zeros(1, dtype=torch.int32, device=dev)
        counts = torch.empty(K, dtype=torch.int32, device=dev)
        sums = torch.empty(K, D, dtype=torch.float32, device=dev)
        inertia = torch.empty(1, dtype=torch.float64, device=dev)
        ws = torch.empty(ops.kmeans_update_workspace(N, K, D), dtype=torch.uint8, device=dev)
        rs = x.stride(0)

        converged, last, n_iter = False, None, 0
        for it in range(self.max_iter):
            changed.zero_()
            ops.kmeans_assign(x, 0, rs, N, 1, D, None, cbf, cnorm, K, labels, score, prev, changed)
            ops.kmeans_update(x, rs, N, D, labels, score, K, ws, counts, sums, inertia)
            ops.kmeans_centers(sums, counts, K, D, centers, cbf, cnorm)
            n_changed, cur = torch.cat([changed.to(torch.float64), inertia]).tolist()   # the one read-back per iteration
            n_iter = it + 1
            labels, prev = prev, labels   # prev now holds this iteration's labels
            if n_changed == 0:
                converged = True           # same labels: the update left the centres bit-identical
                break
            if self.tol > 0.0 and last is not None and last - cur <= self.tol * last:
                break
            last = cur
        if not converged:
            # the labels and inertia of the final centres (the last update moved them)
            ops.kmeans_assign(x, 0, rs, N, 1, D, None, cbf, cnorm, K, labels, score)
            ops.kmeans_update(x, rs, N, D, labels, score, K, ws, counts, sums, inertia)
            cur = float(inertia.item())
            prev = labels
        self.cluster_centers_ = centers
        self.labels_ = prev
        self.inertia_ = float(cur)
        self.n_iter_ = n_iter
        self._dev = (centers, cbf, cnorm)
        return self

    def predict(self, x: torch.Tensor, padding_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Nearest-centre labels (int32) of `x`: [N, D], or [B, T, D] with the frame padding mask `extract_features` returns
        (bool [B, T], True = padded).  Padded frames get -1; 128-frame tiles past an utterance's last valid frame are not read."""
        _check_features(x, (2, 3), "KMeans.predict")
        if self.cluster_centers_ is not None and self.cluster_centers_.shape[1] != x.shape[-1]:
            raise ValueError(f"KMeans.predict: features of size {x.shape[-1]}, centres of size {self.cluster_centers_.shape[1]}")
        cbf, cnorm = self._device_centers(x.device)
        K, D = self.cluster_centers_.shape
        if x.dim() == 2:
            if padding_mask is not None:
                raise ValueError("KMeans.predict: padding_mask goes with [B, T, D] features")
            labels = torch.empty(x.shape[0], dtype=torch.int32, device=x.device)
            ops.kmeans_assign(x, 0, x.stride(0), x.shape[0], 1, D, None, cbf, cnorm, K, labels)
            return labels
        B, T, _ = x.shape
        labels = torch.empty(B, T, dtype=torch.int32, device=x.device)
        valid = None
        if padding_mask is not None:
            if tuple(padding_mask.shape) != (B, T):
                raise ValueError(f"KMeans.predict: padding_mask must be [{B}, {T}], got {list(padding_mask.shape)}")
            padding_mask = padding_mask.to(x.device)
            valid = getattr(padding_mask, "_b200_valid", None)   # set by extract_features: frames up to the last valid one
            if valid is None:
                valid = ((~padding_mask).to(torch.int32) * torch.arange(1, T + 1, dtype=torch.int32, device=x.device)) \
                    .amax(1).to(torch.int32).contiguous()
        ops.kmeans_assign(x, x.stride(0), x.stride(1), T, B, D, valid, cbf, cnorm, K, labels)
        if padding_mask is not None:
            labels.masked_fill_(padding_mask, -1)   # padded frames before an utterance's last valid one, if the mask has any
        return labels
