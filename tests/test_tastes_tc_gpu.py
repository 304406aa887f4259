"""GPU tests of mixture-of-tastes and attention scoring on the tensor-core kernels: trk_score_dense_tastes_f16x3 and
trk_score_topk_tastes_f16x3 through the ABI, predict() / predict_rank() / predict_top_k through the model, against
the oracle (oracle.OracleModel, tests/masked_topk.py).

Exact fixtures are integer-valued.  With attention, every (user, item) pair has one attention logit that leads the
others by at least 110: expf(-110) and below round to 0 in fp32, so the softmax weights are exactly one-hot and the
scores stay exact.  Float fixtures are held to the bound of float_reference()."""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from tests import helpers as H
from tests.masked_topk import SENTINEL_ID, masked_top_k

pytestmark = pytest.mark.gpu

LEAD = 200          # the winning attention logit; the others lie within +-15 of 0


@pytest.fixture(scope='module')
def T():
    import torch
    import tensorrec_b200
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    torch.cuda.set_device(0)
    return tensorrec_b200


def crafted(U, I, d, n_tastes, attention, seed, biased=True):
    """Integer representations: (u [T, U, d], a [T, U, d] or None, item [I, d], ub, ib).  Items carry a one-hot
    selector in components [0, T); a_t puts LEAD on the selector of taste t's turn, (w(i) + c_u) % T == t, so the
    winning taste varies with the user and the item.  Component T adds a small spread to the other logits.  User 0 is
    a zero row."""
    rng = np.random.default_rng(seed)
    nsel = n_tastes if attention else 0
    u = rng.integers(-3, 4, size=(n_tastes, U, d)).astype(np.float32)
    item = rng.integers(-3, 4, size=(I, d)).astype(np.float32)
    a = None
    if attention:
        assert d > n_tastes
        item[:, :nsel] = 0
        item[np.arange(I), rng.integers(0, n_tastes, I)] = 1
        item[:, nsel] = rng.integers(-3, 4, size=I)
        a = np.zeros((n_tastes, U, d), dtype=np.float32)
        shift = rng.integers(0, n_tastes, U)
        for t in range(n_tastes):
            for s in range(n_tastes):
                a[t, (s + shift) % n_tastes == t, s] = LEAD
        a[:, :, nsel] = rng.integers(-5, 6, size=(n_tastes, U))
        a[:, 0] = 0.0
    u[:, 0] = 0.0
    ub = rng.integers(-5, 6, size=U).astype(np.float32) if biased else None
    ib = rng.integers(-5, 6, size=I).astype(np.float32) if biased else None
    return u, a, item, ub, ib


def oracle_scores(u, a, item, ub, ib):
    preds = [u[t] @ item.T for t in range(u.shape[0])]
    atts = None if a is None else [a[t] @ item.T for t in range(a.shape[0])]
    s = oracle.collapse_mixture_of_tastes(preds, atts)
    if ub is not None:
        s = oracle.bias_prediction_dense(s, ub, ib)
    return s


def stacked_operand(u, a, d_pad):
    """The stacked split operand of the ABI, each slice written by trk_split_f32_to_f16x2."""
    import torch
    from tensorrec_b200 import kernels
    ops = list(u) + ([] if a is None else list(a))
    U = u.shape[1]
    split = torch.empty((len(ops), U, 2 * d_pad), dtype=torch.float16, device='cuda')
    scale = torch.empty((len(ops), U), dtype=torch.float32, device='cuda')
    for j, op in enumerate(ops):
        kernels.split_f32(torch.from_numpy(np.ascontiguousarray(op)).cuda(), d_pad=d_pad, out=(split[j], scale[j]))
    return split, scale


def identity_model(T, u, a, item, ub, ib, prediction='dot'):
    """A TensorRec whose representations ARE the given rows: identity features, the rows as linear weights."""
    n_tastes, U, d = u.shape
    R, P = T.representation_graphs, T.prediction_graphs
    preds = {'dot': P.DotProductPredictionGraph, 'cosine': P.CosineSimilarityPredictionGraph}
    model = T.TensorRec(n_components=d, n_tastes=n_tastes, biased=ub is not None, prediction_graph=preds[prediction](),
                        attention_graph=R.LinearRepresentationGraph() if a is not None else None)
    weights = {'linear_weights_item': item}
    for t in range(n_tastes):
        weights['linear_weights_user_%d' % t] = u[t]
        if a is not None:
            weights['linear_weights_attn_%d' % t] = a[t]
    if ub is not None:
        weights.update({'feature_biases_user': ub[:, None], 'feature_biases_item': ib[:, None]})
    model.set_weights(weights)
    uf = sp.identity(U, dtype=np.float32, format='csr')
    itf = sp.identity(item.shape[0], dtype=np.float32, format='csr')
    return model, uf, itf


def float_model(T, U, I, d, n_tastes, attention, prediction='dot', biased=True, seed=0):
    """Tag features and normalised random weights (tests/helpers.py) -> (model, uf, itf, oracle model)."""
    R, P = T.representation_graphs, T.prediction_graphs
    preds = {'dot': P.DotProductPredictionGraph, 'cosine': P.CosineSimilarityPredictionGraph}
    uf, itf = H.tag_features(U, 200, 20, seed=seed + 1), H.tag_features(I, 200, 20, seed=seed + 2)
    wu = [H.linear_weights(200, d, seed=seed + 10 + t) for t in range(n_tastes)]
    wa = [H.linear_weights(200, d, seed=seed + 100 + t) for t in range(n_tastes)] if attention else None
    wi = H.linear_weights(200, d, seed=seed + 3)
    bu = H.feature_biases(200, seed=seed + 4) if biased else None
    bi = H.feature_biases(200, seed=seed + 5) if biased else None
    model = T.TensorRec(n_components=d, n_tastes=n_tastes, biased=biased, prediction_graph=preds[prediction](),
                        attention_graph=R.LinearRepresentationGraph() if attention else None)
    weights = {'linear_weights_item': wi}
    for t in range(n_tastes):
        weights['linear_weights_user_%d' % t] = wu[t]
        if attention:
            weights['linear_weights_attn_%d' % t] = wa[t]
    if biased:
        weights.update({'feature_biases_user': bu[:, None], 'feature_biases_item': bi[:, None]})
    model.set_weights(weights)
    om = oracle.OracleModel(wu, wi, bu, bi, attention_weights=wa, prediction=prediction)
    return model, uf, itf, om


def float_reference(om, uf, itf):
    """(float64 reference scores, |got - ref| bound) of a float fixture.  The reference evaluates the model's formula in
    float64 from the oracle's fp32 representations.  Each 3-pass dot product is within E = 2^-21 |x||i| of the exact
    one (x = u_t or a_t).  Since the softmax weights sum to 1, logit errors of at most E_a = max_t E |a_t||i| move pred
    by at most 2 E_a sum_t w_t |p_t - pred|; the prediction errors add sum_t w_t E |u_t||i| (max: max_t E |u_t||i|).
    The fp32 roundings of the collapse and the biases add a few ulps of the magnitudes involved.  The bound is capped at
    rtol = atol = 2e-5, the tolerance of test_api_gpu's attention case."""
    E = 2.0 ** -21
    uc, ic = oracle.coo_from_sparse(uf), oracle.coo_from_sparse(itf)
    cosine = om.prediction == 'cosine'

    def rep(kind, coo, w):
        x = om._repr(kind, coo, w).astype(np.float64)
        return x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-6) if cosine else x

    item = rep(om.item_repr, ic, om.item_weights)
    ni = np.linalg.norm(item, axis=1)
    users = [rep(om.user_repr, uc, w) for w in om.user_weights]
    p = np.stack([x @ item.T for x in users])
    eu = np.stack([E * np.linalg.norm(x, axis=1)[:, None] * ni[None, :] for x in users])
    if om.attention_weights is None:
        pred, bound = p.max(0), eu.max(0)
    else:
        atts = [rep(om.attention_repr, uc, w) for w in om.attention_weights]
        a = np.stack([x @ item.T for x in atts])
        ea = np.max([E * np.linalg.norm(x, axis=1)[:, None] * ni[None, :] for x in atts], axis=0)
        w = np.exp(a - a.max(0))
        w /= w.sum(0)
        pred = (w * p).sum(0)
        bound = (w * eu).sum(0) + 2 * ea * (w * np.abs(p - pred)).sum(0)
    mag = np.abs(pred) + np.abs(p).max(0)
    if om.user_bias is not None:
        ub = oracle.project_biases(uc, om.user_bias).astype(np.float64)
        ib = oracle.project_biases(ic, om.item_bias).astype(np.float64)
        pred = pred + ub[:, None] + ib[None, :]
        mag = mag + np.abs(ub)[:, None] + np.abs(ib)[None, :]
    bound = bound + 4 * len(users) * 2.0 ** -24 * mag
    return pred, np.minimum(bound, 2e-5 + 2e-5 * np.abs(pred))


def n_items_exact(T, extra=37):
    return max(T.tensorrec.ATTENTION_MIN_ITEMS, 1024) + extra        # not a multiple of 128


def assert_same(a, b):
    assert np.array_equal(np.asarray(a.items), np.asarray(b.items))
    assert np.array_equal(np.asarray(a.scores), np.asarray(b.scores))


TASTE_CASES = [(2, False), (3, False), (5, False), (64, False), (2, True), (3, True), (5, True), (32, True)]


# ---- dense, through the ABI ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n_tastes,attention', TASTE_CASES)
@pytest.mark.parametrize('d', [40, 128])
@pytest.mark.parametrize('store', ['tma', 'direct'])
def test_abi_dense_integer_fixture_is_exact(T, n_tastes, attention, d, store):
    import torch
    from tensorrec_b200 import kernels
    U, I = 301, 1000 + 37            # U is a multiple of no block size; I of no tile
    biased = n_tastes % 2 == 1
    u, a, item, ub, ib = crafted(U, I, d, n_tastes, attention, seed=n_tastes + d, biased=biased)
    expect = oracle_scores(u, a, item, ub, ib)
    d_pad = kernels.d_pad_for(d)
    split, scale = stacked_operand(u, a, d_pad)
    its, isc = kernels.split_f32(torch.from_numpy(item).cuda(), d_pad=d_pad)
    dub = None if ub is None else torch.from_numpy(ub).cuda()
    dib = None if ib is None else torch.from_numpy(ib).cuda()
    users = kernels.SideOperands(None, split, scale, dub, U, d, d_pad)
    meta = kernels.pack_item_meta(isc, dib, I)
    width = (I + 3) // 4 * 4 if store == 'tma' else I + 2
    buf = torch.full((U, width), float('nan'), dtype=torch.float32, device='cuda')
    out = buf[:, :I]
    kernels.score_dense_tastes(users, its, meta, I, n_tastes, attention, out=out)
    assert np.array_equal(out.cpu().numpy(), expect)
    if store == 'direct':
        assert torch.isnan(buf[:, I:]).all()                 # nothing written past the matrix


def test_abi_rejects_unsupported_shapes(T):
    import torch
    from tensorrec_b200 import _lib, kernels
    U, I, d = 10, 200, 64
    item = torch.zeros((I, d), device='cuda')
    its, isc = kernels.split_f32(item, d_pad=64)
    meta = kernels.pack_item_meta(isc, None, I)
    for n_tastes, attention in ((65, False), (33, True)):
        n_ops = n_tastes * (2 if attention else 1)
        users = kernels.SideOperands(None, torch.zeros((n_ops, U, 128), dtype=torch.float16, device='cuda'),
                                     torch.ones((n_ops, U), device='cuda'), None, U, d, 64)
        with pytest.raises(_lib.TrkUnsupportedError):
            kernels.score_dense_tastes(users, its, meta, I, n_tastes, attention)
        with pytest.raises(_lib.TrkUnsupportedError):
            kernels.topk_tastes(users, kernels.SideOperands(None, its, isc, None, I, d, 64), n_tastes, attention, 5)
    users = kernels.SideOperands(None, torch.zeros((2, U, 128), dtype=torch.float16, device='cuda'),
                                 torch.ones((2, U), device='cuda'), None, U, d, 64)
    with pytest.raises(ValueError):
        kernels.score_dense_tastes(users, its, meta, I, 0, False)


# ---- dense, through the model ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('attention', [False, True])
@pytest.mark.parametrize('d', [10, 64, 128])
def test_predict_integer_fixture_is_exact(T, attention, d):
    u, a, item, ub, ib = crafted(250, 700 + 3, d, 3, attention, seed=d)
    model, uf, itf = identity_model(T, u, a, item, ub, ib)
    assert model._tastes_tensor_ok()
    expect = oracle_scores(u, a, item, ub, ib)
    assert np.array_equal(model.predict(uf, itf), expect)
    out = np.empty_like(expect)                               # streamed in user blocks into a caller's array
    model.predict(uf, itf, out=out, user_batch_size=100)
    assert np.array_equal(out, expect)
    assert np.array_equal(model.predict_rank(uf, itf), oracle.rank_predictions(expect))


@pytest.mark.parametrize('prediction', ['dot', 'cosine'])
@pytest.mark.parametrize('attention', [False, True])
@pytest.mark.parametrize('biased', [True, False])
def test_predict_float_fixture_within_the_bound(T, monkeypatch, prediction, attention, biased):
    model, uf, itf, om = float_model(T, 257, 1500, 64, 3, attention, prediction=prediction, biased=biased, seed=7)
    ref, tol = float_reference(om, uf, itf)
    got = model.predict(uf, itf)
    assert np.all(np.abs(got - ref) <= tol)
    monkeypatch.setattr(T.tensorrec, 'SCORE_PATH', 'exact')           # the CUDA-core kernel, same bound
    exact = model.predict(uf, itf)
    assert np.all(np.abs(exact - ref) <= tol)


@pytest.mark.parametrize('d', [10, 128])
def test_float_fixture_at_the_api_test_shapes(T, d):
    """The shapes of test_api_gpu's attention case (15 users, 30 items, three tastes)."""
    uf, itf = H.tag_features(15, 200, 20, seed=1), H.tag_features(30, 200, 20, seed=2)
    model, _, _, om = float_model(T, 15, 30, d, 3, True, seed=0)
    ref, tol = float_reference(om, uf, itf)
    assert np.all(np.abs(model.predict(uf, itf) - ref) <= tol)


def test_score_path_exact_keeps_the_cuda_core_kernel(T, monkeypatch):
    from tensorrec_b200 import kernels
    calls = []
    real = kernels.score_exact
    monkeypatch.setattr(kernels, 'score_exact', lambda *a, **kw: calls.append(1) or real(*a, **kw))
    u, a, item, ub, ib = crafted(100, 300, 64, 3, True, seed=1)
    model, uf, itf = identity_model(T, u, a, item, ub, ib)
    expect = oracle_scores(u, a, item, ub, ib)
    assert np.array_equal(model.predict(uf, itf), expect) and not calls
    monkeypatch.setattr(T.tensorrec, 'SCORE_PATH', 'exact')
    assert not model._tastes_tensor_ok()
    assert np.array_equal(model.predict(uf, itf), expect) and calls


def test_score_path_tensor_accepts_tastes_and_attention(T, monkeypatch):
    monkeypatch.setattr(T.tensorrec, 'SCORE_PATH', 'tensor')
    for attention in (False, True):
        u, a, item, ub, ib = crafted(100, 300, 64, 4, attention, seed=2)
        model, uf, itf = identity_model(T, u, a, item, ub, ib)
        assert np.array_equal(model.predict(uf, itf), oracle_scores(u, a, item, ub, ib))


# ---- attention top-k -------------------------------------------------------------------------------------------------
def exclusion(scores, k, seed):
    """Rows cycle through: empty; the row's own unmasked top-k; heavy; everything; a random light history."""
    rng = np.random.default_rng(seed)
    U, I = scores.shape
    own = oracle.top_k_from_scores(scores, k)[0]
    rows, cols = [], []
    for r in range(U):
        kind = r % 5
        c = {0: [], 1: own[r], 2: np.nonzero(rng.random(I) < 0.6)[0], 3: np.arange(I),
             4: rng.integers(0, I, 40)}[kind]
        rows.append(np.full(len(c), r))
        cols.append(np.asarray(c))
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    return sp.coo_matrix((np.ones(len(rows)), (rows, cols)), shape=(U, I))


@pytest.mark.parametrize('k', [1, 10, 32])
@pytest.mark.parametrize('d', [64, 128])
def test_attention_topk_integer_fixture_is_exact(T, k, d):
    u, a, item, ub, ib = crafted(300, n_items_exact(T), d, 3, True, seed=k + d)
    model, uf, itf = identity_model(T, u, a, item, ub, ib)
    scores = oracle_scores(u, a, item, ub, ib)
    top = model.predict_top_k(uf, itf, k)
    assert model.last_topk_info['path'] == 'exact3'
    exp_i, exp_s = oracle.top_k_from_scores(scores, k)
    assert np.array_equal(top.items, exp_i) and np.array_equal(top.scores, exp_s)
    assert_same(model.predict_rank(uf, itf, k=k), top)
    exclude = exclusion(scores, k, seed=k)
    top = model.predict_top_k(uf, itf, k, exclude=exclude)
    assert model.last_topk_info['path'] == 'exact3'
    exp_i, exp_s = masked_top_k(scores, exclude, k)
    assert np.array_equal(top.items, exp_i) and np.array_equal(top.scores, exp_s)
    assert (top.items == SENTINEL_ID).any()


def test_attention_user_blocks_and_item_shards(T):
    import torch
    from tensorrec_b200 import kernels
    k, I = 10, n_items_exact(T, extra=1037)
    u, a, item, ub, ib = crafted(333, I, 128, 5, True, seed=11)
    model, uf, itf = identity_model(T, u, a, item, ub, ib)
    scores = oracle_scores(u, a, item, ub, ib)
    exclude = exclusion(scores, k, seed=12)
    whole = model.predict_top_k(uf, itf, k, exclude=exclude)
    exp_i, exp_s = masked_top_k(scores, exclude, k)
    assert np.array_equal(whole.items, exp_i) and np.array_equal(whole.scores, exp_s)
    for size in (100, 128, 200):
        assert_same(model.predict_top_k(uf, itf, k, exclude=exclude, user_batch_size=size), whole)
    bounds = [0, I - 700, I]          # the second shard, below ATTENTION_MIN_ITEMS, still takes exact3
    parts = []
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        ex = exclude if lo > 0 else sp.csr_matrix(exclude)[:, :hi]
        top = model.predict_top_k(uf, itf.tocsr()[lo:hi], k, item_id_offset=lo, to_host=False, exclude=ex)
        assert model.last_topk_info['path'] == 'exact3'
        parts.append(torch.cat([top.scores.view(torch.int32), top.items], dim=1))
    merged = kernels.topk_merge_received(torch.stack(parts).contiguous(), uf.shape[0], len(parts), k)
    assert np.array_equal(merged.items.cpu().numpy(), whole.items)
    assert np.array_equal(merged.scores.cpu().numpy(), whole.scores)


def test_attention_dense_rank_on_tensor_cores(T, monkeypatch):
    from tensorrec_b200 import kernels
    u, a, item, ub, ib = crafted(200, n_items_exact(T), 64, 3, True, seed=14)
    model, uf, itf = identity_model(T, u, a, item, ub, ib)
    scores = oracle_scores(u, a, item, ub, ib)
    calls = []
    real = kernels.score_dense_tastes
    monkeypatch.setattr(kernels, 'score_dense_tastes', lambda *a_, **kw: calls.append(1) or real(*a_, **kw))
    big = model.predict_top_k(uf, itf, 100)
    assert model.last_topk_info['path'] == 'dense+rank' and calls
    exp_i, exp_s = oracle.top_k_from_scores(scores, 100)
    assert np.array_equal(big.items, exp_i) and np.array_equal(big.scores, exp_s)
    exclude = exclusion(scores, 10, seed=15)
    fused = model.predict_top_k(uf, itf, 10, exclude=exclude)
    monkeypatch.setattr(T.tensorrec, 'ATTENTION_MIN_ITEMS', 10 ** 9)
    dense = model.predict_top_k(uf, itf, 10, exclude=exclude)
    assert model.last_topk_info['path'] == 'dense+rank'
    assert_same(dense, fused)


@pytest.mark.parametrize('prediction', ['dot', 'cosine'])
def test_attention_float_topk_differs_only_at_near_ties(T, prediction):
    k = 10
    model, uf, itf, om = float_model(T, 300, n_items_exact(T), 128, 3, True, prediction=prediction, seed=13)
    got = model.predict_top_k(uf, itf, k)
    assert model.last_topk_info['path'] == 'exact3'
    # the fused top-k of exactly the scores the dense kernel writes
    dense_i, dense_s = oracle.top_k_from_scores(model.predict(uf, itf), k)
    assert np.array_equal(got.items, dense_i) and np.array_equal(got.scores, dense_s)
    # against the oracle: a slot may differ only where the two items' reference scores are within the bounds
    exp_i, _ = oracle.top_k_from_scores(om.predict(uf, itf), k)
    ref, tol = float_reference(om, uf, itf)
    rows = np.arange(ref.shape[0])[:, None]
    differ = got.items != exp_i
    gap = np.abs(ref[rows, got.items] - ref[rows, exp_i])
    assert np.all(gap[differ] <= 2 * (tol[rows, got.items] + tol[rows, exp_i])[differ])
    assert differ.mean() < 0.01


# ---- mixtures of tastes without attention: the top-k routes stay, dense+rank scores on tensor cores ------------------
def test_tastes_without_attention_keep_their_topk_routes(T, monkeypatch):
    from tensorrec_b200 import kernels
    u, a, item, ub, ib = crafted(200, n_items_exact(T), 64, 3, False, seed=16)
    model, uf, itf = identity_model(T, u, a, item, ub, ib)
    scores = oracle_scores(u, a, item, ub, ib)
    top = model.predict_top_k(uf, itf, 10)
    assert model.last_topk_info['path'] == 'filter'
    exp_i, exp_s = oracle.top_k_from_scores(scores, 10)
    assert np.array_equal(top.items, exp_i) and np.array_equal(top.scores, exp_s)
    calls = []
    real = kernels.score_dense_tastes
    monkeypatch.setattr(kernels, 'score_dense_tastes', lambda *a_, **kw: calls.append(1) or real(*a_, **kw))
    big = model.predict_top_k(uf, itf, 100)
    assert model.last_topk_info['path'] == 'dense+rank' and calls
    exp_i, exp_s = oracle.top_k_from_scores(scores, 100)
    assert np.array_equal(big.items, exp_i) and np.array_equal(big.scores, exp_s)
