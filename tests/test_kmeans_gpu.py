"""K-means kernels (csrc/kmeans.cu) and unispeech_b200.kmeans.KMeans on the GPU, against float64 restatements on the same bf16
values (oracle/kmeans_oracle.py for the Lloyd loop) and scikit-learn.  Outputs start as NaN / sentinels.

Error bound of a score.  The kernel computes |c|^2 - 2 x.c with the bf16 products accumulated in fp32 over D terms, and |c|^2 of
the bf16 centre in fp32 over D terms.  A sum of n terms in fp32 (in any order, rounding or truncating: u = 2^-23) is within
(n - 1) u sum|terms| of the exact sum, so for every row and centre
    |score_kernel - score_fp64| <= bound = 2 D u max_k sum_d |x_d c_kd| + D u max_k |c_k|^2 (+ the final rounding, inside).
The chosen centre's fp64 score is then within 2 * bound of the fp64 minimum, and the label equals the fp64 arg-min on every row
whose best-to-second fp64 gap exceeds 2 * bound."""
import numpy as np
import pytest
import torch

from oracle import kmeans_oracle as KO
from oracle import wavlm_oracle as O

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
SENT = -7


def _ops():
    from unispeech_b200 import ops
    return ops


def prep_centers(c32):
    """fp32 [K, D] -> (bf16 [Kp, D], cnorm [Kp]) through the library's centres kernel."""
    ops = _ops()
    K, D = c32.shape
    Kp = -(-K // 256) * 256
    cbf = torch.full((Kp, D), float("nan"), dtype=torch.bfloat16, device=c32.device)
    cn = torch.full((Kp,), float("nan"), dtype=torch.float32, device=c32.device)
    ops.kmeans_centers(None, None, K, D, c32.contiguous(), cbf, cn)
    return cbf, cn


def fp64_scores(x, cbf, K):
    xd, cd = x.double(), cbf[:K].double()
    s = (cd * cd).sum(1)[None, :] - 2.0 * xd @ cd.T
    bound = 2 * x.shape[1] * U * (xd.abs() @ cd.abs().T).amax(1) + x.shape[1] * U * (cd * cd).sum(1).max()
    return s, bound


def check_labels(x, cbf, K, labels, score=None):
    """Every row: chosen fp64 score within 2 bound of the minimum; label = fp64 arg-min where the gap exceeds 2 bound.
    Returns the share of rows compared exactly."""
    s, bound = fp64_scores(x, cbf, K)
    lab = labels.long()
    assert bool(((lab >= 0) & (lab < K)).all())
    best = s.min(1).values
    chosen = s.gather(1, lab[:, None])[:, 0]
    assert bool((chosen - best <= 2 * bound).all()), float((chosen - best - 2 * bound).max())
    if score is not None:
        assert bool(((score.double() - chosen).abs() <= bound).all())
    if K == 1:
        return 1.0
    top2 = s.topk(2, dim=1, largest=False).values
    clear = (top2[:, 1] - top2[:, 0]) > 2 * bound
    assert torch.equal(lab[clear], s.argmin(1)[clear])
    return float(clear.double().mean())


def rand_bf16(shape, seed, dev, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(torch.bfloat16).to(dev)


SHAPES = [(n, 768, k) for n in (1, 127, 128, 129, 100_003) for k in (1, 2, 255, 256, 257, 500, 1024)] + \
         [(1000, d, k) for d in (64, 1024) for k in (1, 257, 1024)] + [(100_003, 1024, 1024), (100_003, 64, 500)]


@pytest.mark.parametrize("N,D,K", SHAPES)
def test_assign_contiguous(cuda_device, N, D, K):
    ops = _ops()
    dev = cuda_device
    x = rand_bf16((N, D), 11 * N + D + K, dev)
    cbf, cn = prep_centers(rand_bf16((K, D), 7 * K + D, dev).float())
    labels = torch.full((N,), SENT, dtype=torch.int32, device=dev)
    score = torch.full((N,), float("nan"), device=dev)
    ops.kmeans_assign(x, 0, D, N, 1, D, None, cbf, cn, K, labels, score)
    share = check_labels(x, cbf, K, labels, score)
    print(f"N={N} D={D} K={K}: labels compared exactly on {100 * share:.2f}% of rows")
    if N >= 100_000 and K > 1:
        # i.i.d. Gaussian rows and centres are the hardest case for the worst-case bound: every distance is 2 D +- O(sqrt D),
        # so the best two are close (measured on an H100: 97-99.7% of rows compared exactly)
        assert share >= 0.95


def test_assign_clustered_features_compared_exactly(cuda_device):
    """The recipe's shape (D = 768, K = 500) on random rows drawn around random centres (noise 4x the centre spread), as
    encoder features cluster: the exact label comparison covers >= 99% of the rows."""
    ops = _ops()
    dev = cuda_device
    N, D, K = 100_003, 768, 500
    c = rand_bf16((K, D), 31, dev).float()
    g = torch.Generator(device="cpu").manual_seed(32)
    z = torch.randint(0, K, (N,), generator=g).to(dev)
    x = (c[z] + 4.0 * rand_bf16((N, D), 33, dev).float()).to(torch.bfloat16)
    cbf, cn = prep_centers(c)
    labels = torch.full((N,), SENT, dtype=torch.int32, device=dev)
    score = torch.full((N,), float("nan"), device=dev)
    ops.kmeans_assign(x, 0, D, N, 1, D, None, cbf, cn, K, labels, score)
    share = check_labels(x, cbf, K, labels, score)
    print(f"clustered N={N} D={D} K={K}: labels compared exactly on {100 * share:.2f}% of rows")
    assert share >= 0.99


def test_assign_strided_ragged_encoder_view(cuda_device):
    """[B, T, D] view of a wider, longer buffer (batch and row strides), ragged `valid`: padded rows hold NaN and must change
    nothing; their labels are -1 and their scores are not written."""
    ops = _ops()
    dev = cuda_device
    B, T, Tp, D, Dp, K = 5, 700, 720, 768, 832, 500
    buf = rand_bf16((B, Tp, Dp), 3, dev)
    valid = torch.tensor([700, 1, 0, 130, 257], dtype=torch.int32, device=dev)
    for b in range(B):
        buf[b, int(valid[b]):] = float("nan")
    x = buf[:, :T, :D]
    cbf, cn = prep_centers(rand_bf16((K, D), 4, dev).float())
    labels = torch.full((B, T), SENT, dtype=torch.int32, device=dev)
    score = torch.full((B, T), float("nan"), device=dev)
    ops.kmeans_assign(x, x.stride(0), x.stride(1), T, B, D, valid, cbf, cn, K, labels, score)
    for b in range(B):
        v = int(valid[b])
        assert bool((labels[b, v:] == -1).all()) and bool(score[b, v:].isnan().all())
        if v:
            check_labels(x[b, :v], cbf, K, labels[b, :v], score[b, :v])
    # the same rows as one contiguous call give the same labels
    rows = torch.cat([x[b, :int(valid[b])] for b in range(B)]).contiguous()
    flat = torch.full((rows.shape[0],), SENT, dtype=torch.int32, device=dev)
    ops.kmeans_assign(rows, 0, D, rows.shape[0], 1, D, None, cbf, cn, K, flat)
    assert torch.equal(flat, torch.cat([labels[b, :int(valid[b])] for b in range(B)]))


def test_assign_duplicated_centres_resolve_to_the_lowest_index(cuda_device):
    ops = _ops()
    dev = cuda_device
    D, half = 256, 300
    lo = rand_bf16((half, D), 5, dev).float()
    c = torch.cat([lo, lo])                     # centre k + 300 == centre k, across the 256-wide tiles
    cbf, cn = prep_centers(c)
    idx = torch.arange(0, half, 3, device=dev)
    x = torch.cat([cbf[idx], rand_bf16((4000, D), 6, dev)])   # rows equal to a centre, and random rows
    labels = torch.full((x.shape[0],), SENT, dtype=torch.int32, device=dev)
    ops.kmeans_assign(x, 0, D, x.shape[0], 1, D, None, cbf, cn, 2 * half, labels)
    assert bool((labels < half).all())
    assert torch.equal(labels[:idx.numel()].long(), idx)


def test_assign_changed_count(cuda_device):
    ops = _ops()
    dev = cuda_device
    N, D, K = 50_000, 128, 300
    x = rand_bf16((N, D), 8, dev)
    cbf, cn = prep_centers(rand_bf16((K, D), 9, dev).float())
    lab = torch.full((N,), SENT, dtype=torch.int32, device=dev)
    ops.kmeans_assign(x, 0, D, N, 1, D, None, cbf, cn, K, lab)
    prev = lab.clone()
    flip = torch.arange(0, N, 7, device=dev)
    prev[flip] = (prev[flip] + 1) % K
    changed = torch.zeros(1, dtype=torch.int32, device=dev)
    lab2 = torch.full((N,), SENT, dtype=torch.int32, device=dev)
    ops.kmeans_assign(x, 0, D, N, 1, D, None, cbf, cn, K, lab2, None, prev, changed)
    assert torch.equal(lab2, lab) and int(changed) == flip.numel()


def test_assign_limits_are_errors(cuda_device):
    ops = _ops()
    dev = cuda_device
    x = rand_bf16((256, 128), 1, dev)
    cbf, cn = prep_centers(rand_bf16((4, 128), 2, dev).float())
    lab = torch.full((256,), SENT, dtype=torch.int32, device=dev)
    big = torch.zeros(1280, 128, dtype=torch.bfloat16, device=dev)
    bign = torch.zeros(1280, device=dev)
    for args in ((x, 0, 128, 256, 1, 128, None, cbf, cn, 0, lab),          # K = 0
                 (x, 0, 128, 256, 1, 128, None, big, bign, 1025, lab),     # K > 1024
                 (x, 0, 128, 256, 1, 96, None, cbf, cn, 4, lab)):          # D % 64 != 0
        with pytest.raises(RuntimeError):
            ops.kmeans_assign(*args)
    assert bool((lab == SENT).all())
    with pytest.raises(RuntimeError):
        ops.kmeans_centers(None, None, 0, 128, torch.zeros(1, 128, device=dev), cbf, cn)
    with pytest.raises(RuntimeError):
        ops.kmeanspp_init(x, 128, 256, 96, 4, (0, 0), torch.empty(256, device=dev), torch.empty(4, 96, device=dev))


def run_update(x, labels, score, K):
    ops = _ops()
    N, D = x.shape
    counts = torch.full((K,), SENT, dtype=torch.int32, device=x.device)
    sums = torch.full((K, D), float("nan"), device=x.device)
    inertia = torch.full((1,), float("nan"), dtype=torch.float64, device=x.device)
    ws = torch.empty(ops.kmeans_update_workspace(N, K, D), dtype=torch.uint8, device=x.device)
    ops.kmeans_update(x, x.stride(0), N, D, labels, score, K, ws, counts, sums, inertia)
    return counts, sums, inertia


@pytest.mark.parametrize("N,D,K", [(200_003, 768, 500), (7, 64, 3), (65_536, 1024, 1024)])
def test_update_counts_sums_inertia(cuda_device, N, D, K):
    """Half of all rows in cluster 0, the last two clusters empty, some rows unlabelled (-1).  Counts exact; sums within the
    fp32 bound of the partial sums (2048-row pieces, then fp64); inertia within fp64 accumulation of fp32 row terms."""
    dev = cuda_device
    x = rand_bf16((N, D), N + K, dev)
    g = torch.Generator(device="cpu").manual_seed(N)
    lab = torch.randint(1, max(K - 2, 2), (N,), generator=g, dtype=torch.int32)
    lab[::2] = 0
    lab[torch.arange(N) % 97 == 5] = -1
    lab = lab.to(dev)
    score = (torch.randn(N, generator=g) * 50).to(dev)
    counts, sums, inertia = run_update(x, lab, score, K)
    keep = lab >= 0
    ref_counts = torch.bincount(lab[keep].long(), minlength=K)
    assert torch.equal(counts.long(), ref_counts)
    assert int(counts[K - 1]) == 0 and int(counts[0]) > N // 3
    xd = x.double()
    ref = torch.zeros(K, D, dtype=torch.float64, device=dev).index_add_(0, lab[keep].long(), xd[keep])
    ref_abs = torch.zeros(K, D, dtype=torch.float64, device=dev).index_add_(0, lab[keep].long(), xd[keep].abs())
    err = (sums.double() - ref).abs()
    assert bool((err <= 2048 * U * ref_abs + U * ref.abs() + 1e-30).all()), float((err / (ref_abs + 1e-30)).max())
    want = float((xd[keep] ** 2).sum() + score[keep].double().sum())
    scale = float((xd[keep] ** 2).sum() + score[keep].double().abs().sum())
    assert abs(float(inertia) - want) <= 4096 * U * scale   # fp32 |x|^2 sums over <= 2048 terms per thread, then fp64
    # bit-identical on a second call
    c2, s2, i2 = run_update(x, lab, score, K)
    assert torch.equal(c2, counts) and torch.equal(s2.view(torch.int32), sums.view(torch.int32)) and float(i2) == float(inertia)


def test_centres_update_keeps_empty_clusters(cuda_device):
    ops = _ops()
    dev = cuda_device
    K, D = 300, 128
    prev = torch.randn(K, D, device=dev)
    sums = torch.randn(K, D, device=dev) * 100
    counts = torch.randint(1, 1000, (K,), dtype=torch.int32, device=dev)
    counts[::7] = 0
    c = prev.clone()
    cbf = torch.full((512, D), float("nan"), dtype=torch.bfloat16, device=dev)
    cn = torch.full((512,), float("nan"), device=dev)
    ops.kmeans_centers(sums, counts, K, D, c, cbf, cn)
    empty = counts == 0
    assert torch.equal(c[empty], prev[empty])
    want = sums[~empty].double() / counts[~empty].double()[:, None]
    assert bool(((c[~empty].double() - want).abs() <= 2 * U * want.abs()).all())
    assert torch.equal(cbf[:K], c.to(torch.bfloat16)) and bool((cbf[K:] == 0).all()) and bool((cn[K:] == 0).all())
    ref = (cbf[:K].double() ** 2).sum(1)
    assert bool(((cn[:K].double() - ref).abs() <= D * U * ref).all())


def blob_data(dev, K=20, D=64, n_per=500, spread=1.0, sep=10.0, seed=0):
    rng = np.random.default_rng(seed)
    truth = sep * rng.standard_normal((K, D))
    x = np.concatenate([t + spread * rng.standard_normal((n_per, D)) for t in truth])
    x = x[rng.permutation(x.shape[0])]
    xb = torch.tensor(x, dtype=torch.float32).to(torch.bfloat16)
    init = truth + 1.5 * spread * rng.standard_normal((K, D))
    return xb.to(dev), xb.double().numpy(), truth, init


def test_fit_from_given_centres_matches_oracle_and_sklearn(cuda_device):
    from sklearn.cluster import KMeans as SkKMeans

    from unispeech_b200.kmeans import KMeans
    dev = cuda_device
    K = 20
    x, x64, _, init = blob_data(dev, K=K)
    km = KMeans(K, max_iter=100).fit(x, init_centers=init)
    c, lab, inertia, n_iter = KO.lloyd(x64, init, max_iter=100)
    sk = SkKMeans(n_clusters=K, init=init, n_init=1, max_iter=100, tol=0.0, algorithm="lloyd").fit(x64)
    got = km.labels_.cpu().numpy()
    assert np.array_equal(got, lab) and np.array_equal(got, sk.labels_)
    assert km.n_iter_ == n_iter == sk.n_iter_
    # centres: fp32 sums of ~500 bf16 rows of magnitude <= ~40 (rounding error ~sqrt(500) * 2^-24 * 500 * 40 / 500 ~ 5e-5);
    # inertia: the kernels measure distances to the bf16 centres (each coordinate moved by up to |c| 2^-9 ~ 0.03) and take
    # |x|^2 + score in fp32, which cancels about 100:1 here, so a few 1e-3 relative
    np.testing.assert_allclose(km.cluster_centers_.cpu().numpy(), c, rtol=0, atol=1e-3)
    np.testing.assert_allclose(km.cluster_centers_.cpu().numpy(), sk.cluster_centers_, rtol=0, atol=1e-3)
    assert km.inertia_ == pytest.approx(inertia, rel=5e-3) and km.inertia_ == pytest.approx(sk.inertia_, rel=5e-3)
    assert torch.equal(km.predict(x), km.labels_)
    # an iteration cap: labels and inertia belong to the final centres (scikit-learn's rule)
    km1 = KMeans(K, max_iter=1).fit(x, init_centers=init)
    c1, lab1, inertia1, _ = KO.lloyd(x64, init, max_iter=1)
    assert km1.n_iter_ == 1 and np.array_equal(km1.labels_.cpu().numpy(), lab1)
    assert km1.inertia_ == pytest.approx(inertia1, rel=5e-3)


def test_kmeanspp_one_centre_per_blob_seeded(cuda_device):
    ops = _ops()
    dev = cuda_device
    K, D = 8, 128
    x, _, truth, _ = blob_data(dev, K=K, D=D, n_per=1000, spread=1.0, sep=30.0, seed=4)
    n = x.shape[0]

    def draw(seed):
        c = torch.full((K, D), float("nan"), device=dev)
        d2 = torch.empty(n, device=dev)
        inertia = torch.full((1,), float("nan"), dtype=torch.float64, device=dev)
        ops.kmeanspp_init(x, D, n, D, K, seed, d2, c, inertia)
        return c, float(inertia)

    c1, i1 = draw((1, 0))
    near = ((c1.double().cpu()[:, None, :] - torch.tensor(truth)[None]) ** 2).sum(-1).argmin(1)
    assert sorted(near.tolist()) == list(range(K))
    rows = set(map(tuple, x.float().cpu().numpy().tolist()))
    assert all(tuple(r) in rows for r in c1.cpu().numpy().tolist())   # every centre is a data row
    lab, _ = KO.assign(x.double().cpu().numpy(), c1.double().cpu().numpy())
    assert i1 == pytest.approx(KO.inertia(x.double().cpu().numpy(), c1.double().cpu().numpy(), lab), rel=1e-4)
    c2, i2 = draw((1, 0))
    assert torch.equal(c1, c2) and i1 == i2
    c3, _ = draw((2, 0))
    assert not torch.equal(c1, c3)


def test_fit_is_bit_reproducible(cuda_device):
    from unispeech_b200.kmeans import KMeans
    dev = cuda_device
    x = rand_bf16((60_000, 256), 21, dev)
    runs = [KMeans(100, max_iter=8, init_size=20_000, n_init=3, seed=5).fit(x) for _ in range(2)]
    a, b = runs
    assert torch.equal(a.cluster_centers_.view(torch.int32), b.cluster_centers_.view(torch.int32))
    assert torch.equal(a.labels_, b.labels_) and a.inertia_ == b.inertia_ and a.n_iter_ == b.n_iter_
    other = KMeans(100, max_iter=8, init_size=20_000, n_init=3, seed=6).fit(x)
    assert not torch.equal(other.cluster_centers_, a.cluster_centers_)
    # inertia_ is the sum of squared distances of the bf16 rows to the bf16 centres under labels_
    cbf = a.cluster_centers_.to(torch.bfloat16).double()
    d = x.double() - cbf[a.labels_.long()]
    assert a.inertia_ == pytest.approx(float((d * d).sum()), rel=1e-4)


def test_labels_from_wavlm_features_feed_a_hubert_step(cuda_device):
    """extract_features(output_layer=1) of a small WavLM on a ragged batch -> fit on the valid frames -> predict: padded frames
    get -1, valid frames the fp64 arg-min (gap rule); the labels (padding set to 0) are the targets of one HubertModel step."""
    from unispeech_b200.hubert import HubertConfig, HubertModel
    from unispeech_b200.kmeans import KMeans
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    dev = cuda_device
    cfg = O.tiny_config(pre_ln=False)
    m = WavLM(WavLMConfig(vars(cfg)))
    m.load_state_dict(O.deterministic_state_dict(cfg), strict=True)
    m = m.to(dev).eval()
    B, L = 4, 32000
    wav, pmask = O.deterministic_waveform(B, L, seed=3, lengths=[32000, 20000, 9000, 25000])
    with torch.no_grad():
        x, pm = m.extract_features(wav.to(dev), padding_mask=pmask.to(dev), output_layer=1)
    assert x.dtype == torch.bfloat16 and pm is not None and bool(pm.any())
    T = x.shape[1]
    valid = x[~pm].contiguous()
    K = 16
    km = KMeans(K, max_iter=20, seed=1).fit(valid)
    labels = km.predict(x, pm)
    assert labels.shape == (B, T) and labels.dtype == torch.int32
    assert bool((labels[pm] == -1).all())
    cbf, _ = km._device_centers(dev)
    check_labels(valid, cbf, K, labels[~pm])

    hcfg = O.tiny_config(pre_ln=True, relative_position_embedding=False, gru_rel_pos=False)
    h = HubertModel(HubertConfig(dict(vars(hcfg), final_dim=64)), [K])
    h.load_state_dict(O.deterministic_state_dict(hcfg), strict=False)
    h = h.to(dev).train()
    target = labels.long().clamp(min=0)
    np.random.seed(0)
    out = h(wav.to(dev), target_list=[target], padding_mask=pmask.to(dev), mask=True)
    loss, ss, _ = h.criterion(out)
    assert bool(torch.isfinite(loss)) and float(ss) > 0
    loss.backward()
