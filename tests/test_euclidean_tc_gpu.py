"""GPU tests of Euclidean user x item scoring on the tensor-core kernels: trk_score_dense_euclid_f16x3 and
trk_score_topk_euclid_f16x3 through the ABI, predict() / predict_rank() and predict_top_k against the oracle
(oracle.OracleModel(prediction='euclidean'), tests/masked_topk.py).  Integer fixtures match bit for bit; float
fixtures are compared on the d^2 scale at the similar-items tolerance |got^2 - ref^2| <= 8 * 2^-20 (|u|^2 + |i|^2)."""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from tests import helpers as H
from tests.masked_topk import SENTINEL_ID, masked_top_k

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def T():
    import torch
    import tensorrec_b200
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    torch.cuda.set_device(0)
    return tensorrec_b200


def make_model(T, U, I, d, integer, n_tastes=1, biased=True, seed=0, itf=None):
    """-> (model, user features, item features, oracle scores, user reprs [T, U, d], item repr [I, d])."""
    uf = H.tag_features(U, 200, 20, seed=seed + 1, integer=integer)
    itf = H.tag_features(I, 200, 20, seed=seed + 2, integer=integer) if itf is None else itf
    wus = [H.linear_weights(200, d, seed=seed + 10 + t, integer=integer) for t in range(n_tastes)]
    wi = H.linear_weights(200, d, seed=seed + 4, integer=integer)
    model = T.TensorRec(n_components=d, n_tastes=n_tastes, biased=biased,
                        prediction_graph=T.prediction_graphs.EuclideanSimilarityPredictionGraph())
    weights = {'linear_weights_item': wi}
    for t in range(n_tastes):
        weights['linear_weights_user_%d' % t] = wus[t]
    bu = bi = None
    if biased:
        bu, bi = H.feature_biases(200, seed=seed + 5, integer=integer), H.feature_biases(200, seed=seed + 6,
                                                                                         integer=integer)
        weights.update({'feature_biases_user': bu[:, None], 'feature_biases_item': bi[:, None]})
    model.set_weights(weights)
    om = oracle.OracleModel(wus, wi, bu, bi, prediction='euclidean')
    return model, uf, itf, om.predict(uf, itf), om.user_representation(uf), om.item_representation(itf)


def exclusion(scores, k, seed):
    """Rows cycle through: empty; the row's own unmasked top-k; heavy (> half of the catalogue); everything; fewer than
    k eligible items; a random light history with duplicates -- plus explicit zeros, which exclude nothing."""
    rng = np.random.default_rng(seed)
    U, I = scores.shape
    own = oracle.top_k_from_scores(scores, k)[0]
    rows, cols, vals = [], [], []
    for u in range(U):
        kind = u % 6
        if kind == 1:
            c = own[u]
        elif kind == 2:
            c = np.nonzero(rng.random(I) < 0.6)[0]
        elif kind == 3:
            c = np.arange(I)
        elif kind == 4:
            c = np.setdiff1d(np.arange(I), rng.choice(I, max(k // 2, 0), replace=False))
        elif kind == 5:
            c = rng.integers(0, I, 40)
        else:
            continue
        rows.append(np.full(len(c), u))
        cols.append(c)
        vals.append(np.ones(len(c)))
    rows.append([0, 5])
    cols.append([1, 2])
    vals.append([0.0, 0.0])
    return sp.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(U, I))


def n_items_exact(T, extra=37):
    return max(T.tensorrec.EUCLIDEAN_MIN_ITEMS, 1024) + extra       # not a multiple of 128


def assert_same(a, b):
    assert np.array_equal(np.asarray(a.items), np.asarray(b.items))
    assert np.array_equal(np.asarray(a.scores), np.asarray(b.scores))


def assert_d2_close(got, user_repr, item_repr):
    """got: unbiased scores -sqrt(max(d^2, 1e-16)), compared with d^2 in float64."""
    u = user_repr.astype(np.float64)
    i = item_repr.astype(np.float64)
    su, si = (u * u).sum(1), (i * i).sum(1)
    ref = np.maximum(su[:, None] - 2 * u @ i.T + si[None, :], 0.0)
    tol = 8 * 2.0 ** -20 * (su[:, None] + si[None, :]) + 1e-15
    assert np.all(np.abs(got.astype(np.float64) ** 2 - ref) <= tol)


# ---- dense, through the ABI ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('d', [64, 128])
@pytest.mark.parametrize('biased', [True, False])
@pytest.mark.parametrize('store', ['tma', 'direct'])
def test_abi_dense_integer_fixture_is_exact(T, d, biased, store):
    import torch
    from tensorrec_b200 import kernels
    rng = np.random.default_rng(d + 2 * biased)
    U, I = 300, 1000 + 37
    user = rng.integers(-3, 4, size=(U, d)).astype(np.float32)
    item = rng.integers(-3, 4, size=(I, d)).astype(np.float32)
    user[0] = 0.0                           # a zero row
    user[1] = item[5]                       # d^2 = 0: clamps to 1e-16, score -1e-8
    user[2] = item[I - 1]
    ub = rng.integers(-5, 6, size=U).astype(np.float32) if biased else None
    ib = rng.integers(-5, 6, size=I).astype(np.float32) if biased else None
    expect = oracle.euclidean_dense(user, item)
    if biased:
        expect = oracle.bias_prediction_dense(expect, ub, ib)
    dev = torch.device('cuda')
    us, usc = kernels.split_f32(torch.from_numpy(user).to(dev), d_pad=d)
    its, isc = kernels.split_f32(torch.from_numpy(item).to(dev), d_pad=d)
    dub = None if ub is None else torch.from_numpy(ub).to(dev)
    dib = None if ib is None else torch.from_numpy(ib).to(dev)
    items = kernels.SideOperands(None, its, isc, dib, I, d, d)
    meta = kernels.pack_item_meta(isc, dib, I)
    sq = (kernels.operand_half_sqnorm(us, usc, d), kernels.item_half_sqnorm(items))
    width = (I + 3) // 4 * 4 if store == 'tma' else I + 2    # 1040: TMA stores; 1039 (not a multiple of 4): direct
    buf = torch.full((U, width), float('nan'), dtype=torch.float32, device=dev)
    out = buf[:, :I]
    kernels.score_dense_tc(us, usc, dub, its, meta, U, I, d, out=out, sqnorms=sq)
    got = out.cpu().numpy()
    assert np.array_equal(got, expect)


def test_abi_topk_matches_the_oracle(T):
    import torch
    from tensorrec_b200 import kernels
    rng = np.random.default_rng(3)
    U, I, d, k = 200, 700 + 5, 64, 10
    user = rng.integers(-3, 4, size=(U, d)).astype(np.float32)
    item = rng.integers(-3, 4, size=(I, d)).astype(np.float32)
    ub = rng.integers(-5, 6, size=U).astype(np.float32)
    ib = rng.integers(-5, 6, size=I).astype(np.float32)
    scores = oracle.bias_prediction_dense(oracle.euclidean_dense(user, item), ub, ib)
    dev = torch.device('cuda')
    us, usc = kernels.split_f32(torch.from_numpy(user).to(dev), d_pad=d)
    its, isc = kernels.split_f32(torch.from_numpy(item).to(dev), d_pad=d)
    users = kernels.SideOperands(None, us, usc, torch.from_numpy(ub).to(dev), U, d, d)
    items = kernels.SideOperands(None, its, isc, torch.from_numpy(ib).to(dev), I, d, d)
    for n_splits in (1, 3):
        top = kernels.topk_exact(users, items, k, n_splits=n_splits, item_hsq=kernels.item_half_sqnorm(items))
        exp_i, exp_s = oracle.top_k_from_scores(scores, k)
        assert np.array_equal(top.items.cpu().numpy(), exp_i) and np.array_equal(top.scores.cpu().numpy(), exp_s)


# ---- dense, through the model ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('d', [64, 128])
@pytest.mark.parametrize('biased', [True, False])
def test_predict_integer_fixture_is_exact(T, d, biased):
    model, uf, itf, scores, _, _ = make_model(T, 300, 1000 + 37, d, integer=True, biased=biased, seed=d)
    assert model._euclidean_tensor_ok()
    got = model.predict(uf, itf)
    assert np.array_equal(got, scores)
    out = np.empty_like(scores)                          # streamed in user blocks into a caller's array
    model.predict(uf, itf, out=out, user_batch_size=128)
    assert np.array_equal(out, scores)
    assert np.array_equal(model.predict_rank(uf, itf), oracle.rank_predictions(scores))


def test_predict_float_fixture_on_the_d2_scale(T, monkeypatch):
    model, uf, itf, _, ureps, irepr = make_model(T, 257, 1500, 128, integer=False, biased=False, seed=5)
    got = model.predict(uf, itf)
    assert_d2_close(got, ureps[0], irepr)
    monkeypatch.setattr(T.tensorrec, 'SCORE_PATH', 'exact')          # the CUDA-core kernel
    exact = model.predict(uf, itf)
    assert_d2_close(exact, ureps[0], irepr)
    u, i = ureps[0].astype(np.float64), irepr.astype(np.float64)
    tol = 8 * 2.0 ** -20 * ((u * u).sum(1)[:, None] + (i * i).sum(1)[None, :]) + 1e-15
    assert np.all(np.abs(got.astype(np.float64) ** 2 - exact.astype(np.float64) ** 2) <= 2 * tol)


def test_score_path_tensor_accepts_euclidean_models(T, monkeypatch):
    monkeypatch.setattr(T.tensorrec, 'SCORE_PATH', 'tensor')
    model, uf, itf, scores, _, _ = make_model(T, 150, 300, 64, integer=True, seed=6)
    assert np.array_equal(model.predict(uf, itf), scores)


# ---- top-k -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('d', [64, 128])
@pytest.mark.parametrize('k', [1, 10, 32])
def test_topk_integer_fixture_is_exact(T, d, k):
    model, uf, itf, scores, _, _ = make_model(T, 300, n_items_exact(T), d, integer=True, seed=k + d)
    top = model.predict_top_k(uf, itf, k)
    assert model.last_topk_info['path'] == 'exact3'
    exp_i, exp_s = oracle.top_k_from_scores(scores, k)
    assert np.array_equal(top.items, exp_i) and np.array_equal(top.scores, exp_s)
    assert_same(model.predict_rank(uf, itf, k=k), top)


def test_tie_heavy_catalogue_keeps_the_lower_id_first(T):
    """Every item row appears several times: equal distances everywhere, ordered by id as tf.nn.top_k orders them."""
    I = n_items_exact(T)
    distinct = H.tag_features(9, 200, 20, seed=7, integer=True)
    itf = sp.vstack([distinct[j % 9] for j in range(I)]).tocsr()
    model, uf, itf, scores, _, _ = make_model(T, 260, I, 64, integer=True, seed=8, itf=itf)
    for k in (10, 32):
        top = model.predict_top_k(uf, itf, k)
        assert model.last_topk_info['path'] == 'exact3'
        exp_i, exp_s = oracle.top_k_from_scores(scores, k)
        assert np.array_equal(top.items, exp_i) and np.array_equal(top.scores, exp_s)


@pytest.mark.parametrize('n_tastes', [1, 3])
def test_exclusion_matches_the_masked_oracle(T, n_tastes):
    k = 10
    model, uf, itf, scores, _, _ = make_model(T, 300, n_items_exact(T), 64, integer=True, n_tastes=n_tastes, seed=9)
    exclude = exclusion(scores, k, seed=10)
    top = model.predict_top_k(uf, itf, k, exclude=exclude)
    assert model.last_topk_info['path'] == 'exact3'
    exp_i, exp_s = masked_top_k(scores, exclude, k)
    assert np.array_equal(top.items, exp_i) and np.array_equal(top.scores, exp_s)
    assert (top.items == SENTINEL_ID).any()              # rows with fewer than k eligible items
    if n_tastes > 1:
        plain = model.predict_top_k(uf, itf, k)
        exp_i, exp_s = oracle.top_k_from_scores(scores, k)
        assert np.array_equal(plain.items, exp_i) and np.array_equal(plain.scores, exp_s)


def test_user_blocks_and_item_shards(T):
    import torch
    from tensorrec_b200 import kernels
    k, I = 10, n_items_exact(T, extra=1037)
    model, uf, itf, scores, _, _ = make_model(T, 333, I, 128, integer=True, n_tastes=2, seed=11)
    exclude = exclusion(scores, k, seed=12)
    whole = model.predict_top_k(uf, itf, k, exclude=exclude)
    for size in (128, 200):
        assert_same(model.predict_top_k(uf, itf, k, exclude=exclude, user_batch_size=size), whole)
    bounds = [0, I - 700, I]        # the second shard, below EUCLIDEAN_MIN_ITEMS, still takes exact3 (rank-invariant)
    parts = []
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        ex = exclude if lo > 0 else sp.csr_matrix(exclude)[:, :hi]
        top = model.predict_top_k(uf, itf.tocsr()[lo:hi], k, item_id_offset=lo, to_host=False, exclude=ex)
        assert model.last_topk_info['path'] == 'exact3'
        parts.append(torch.cat([top.scores.view(torch.int32), top.items], dim=1))
    merged = kernels.topk_merge_received(torch.stack(parts).contiguous(), uf.shape[0], len(parts), k)
    assert np.array_equal(merged.items.cpu().numpy(), whole.items)
    assert np.array_equal(merged.scores.cpu().numpy(), whole.scores)


def test_float_fixture_differs_only_at_near_ties(T):
    k = 10
    model, uf, itf, scores, ureps, irepr = make_model(T, 300, n_items_exact(T), 128, integer=False, biased=False,
                                                      seed=13)
    got = model.predict_top_k(uf, itf, k)
    assert model.last_topk_info['path'] == 'exact3'
    # the fused top-k of exactly the scores the dense kernel writes
    dense_i, dense_s = oracle.top_k_from_scores(model.predict(uf, itf), k)
    assert np.array_equal(got.items, dense_i) and np.array_equal(got.scores, dense_s)
    # against the oracle: a slot may differ only where the two items' float64 distances nearly tie
    exp_i, _ = oracle.top_k_from_scores(scores, k)
    u, i = ureps[0].astype(np.float64), irepr.astype(np.float64)
    d2 = np.maximum((u * u).sum(1)[:, None] - 2 * u @ i.T + (i * i).sum(1)[None, :], 0.0)
    rows = np.arange(len(u))[:, None]
    tol = 8 * 2.0 ** -20 * ((u * u).sum(1)[:, None] + (i * i).sum(1)[got.items])
    differ = got.items != exp_i
    assert np.all(np.abs(d2[rows, got.items] - d2[rows, exp_i])[differ] <= 2 * tol[differ])
    assert differ.mean() < 0.01


def test_dense_rank_route_equals_exact3(T, monkeypatch):
    k = 10
    model, uf, itf, scores, _, _ = make_model(T, 250, n_items_exact(T), 64, integer=True, seed=14)
    exclude = exclusion(scores, k, seed=15)
    fused = model.predict_top_k(uf, itf, k, exclude=exclude)
    assert model.last_topk_info['path'] == 'exact3'
    monkeypatch.setattr(T.tensorrec, 'EUCLIDEAN_MIN_ITEMS', 10 ** 9)
    dense = model.predict_top_k(uf, itf, k, exclude=exclude)
    assert model.last_topk_info['path'] == 'dense+rank'
    assert_same(dense, fused)
    big = model.predict_top_k(uf, itf, 40)                # k > 32: dense+rank, scored on tensor cores
    exp_i, exp_s = oracle.top_k_from_scores(scores, 40)
    assert np.array_equal(big.items, exp_i) and np.array_equal(big.scores, exp_s)
