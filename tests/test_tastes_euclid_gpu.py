"""GPU tests of Euclidean mixtures of tastes on the taste-collapsing tensor-core kernel (DESIGN §3.12):
trk_score_{dense,topk,topk_wide,count}_tastes_euclid_f16x3 through kernels.py and the model.

Max form: bit for bit against the elementwise maximum over the tastes of the one-taste Euclidean tensor-core scores
(rounding is monotone, so the maximum commutes with the biases), and against the oracle on integer fixtures.
Attention form: integer fixtures whose winning attention similarity leads the others by >= 110 (one-hot softmax) are
exact against the oracle; float fixtures lie within the bound of float_bound().  Routes: predict_rank_at on
'exact3_count' equals predict_rank(), and the attention top-k routes equal forced 'dense+rank' bit for bit."""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from tests import helpers as H
from tests.masked_topk import SENTINEL_ID
from tests.test_euclidean_tc_gpu import exclusion
from tests.test_rank_at_gpu import assert_same_matrix, expect_at, make_pairs, masked_ranks

pytestmark = pytest.mark.gpu

SELECT = 120        # the attention selector: a winning attention row is >= 110 closer to the item than the others


@pytest.fixture(scope='module')
def T():
    import torch
    import tensorrec_b200
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    torch.cuda.set_device(0)
    return tensorrec_b200


# ---- fixtures -------------------------------------------------------------------------------------------------------
def crafted(U, I, d, n_tastes, attention, seed, biased=True):
    """Integer representations (u [T, U, d], a [T, U, d] or None, item [I, d], ub, ib).  With attention, items hold
    SELECT in one selector component of [0, T) and every a_t holds SELECT in one of them (a permutation per user):
    the taste whose selector matches the item's is at distance sqrt(R), the others at sqrt(2 SELECT^2 + R), R <=
    9 (d - T) from the remaining components, so the winner leads by >= 110 and expf rounds the others' weights to 0.
    Without attention, user 1's taste 0 row equals item 0 (d^2 = 0) and user 2's rows are items 1 .. T."""
    rng = np.random.default_rng(seed)
    u = rng.integers(-3, 4, size=(n_tastes, U, d)).astype(np.float32)
    item = rng.integers(-3, 4, size=(I, d)).astype(np.float32)
    a = None
    if attention:
        assert d > n_tastes
        item[:, :n_tastes] = 0
        item[np.arange(I), rng.integers(0, n_tastes, I)] = SELECT
        a = np.zeros((n_tastes, U, d), dtype=np.float32)
        shift = rng.integers(0, n_tastes, U)
        for t in range(n_tastes):
            for s in range(n_tastes):
                a[t, (s + shift) % n_tastes == t, s] = SELECT
    else:
        u[0, 1] = item[0]
        for t in range(n_tastes):
            u[t, 2] = item[1 + t]
    ub = rng.integers(-5, 6, size=U).astype(np.float32) if biased else None
    ib = rng.integers(-5, 6, size=I).astype(np.float32) if biased else None
    return u, a, item, ub, ib


def oracle_scores(u, a, item, ub, ib):
    """The reference order: EuclideanSimilarityPredictionGraph dense per taste and attention row, the collapse, the
    biases."""
    preds = [oracle.euclidean_dense(u[t], item) for t in range(u.shape[0])]
    atts = None if a is None else [oracle.euclidean_dense(a[t], item) for t in range(a.shape[0])]
    s = oracle.collapse_mixture_of_tastes(preds, atts)
    if ub is not None:
        s = oracle.bias_prediction_dense(s, ub, ib)
    return s


def device_operands(T, u, a, item, ub, ib):
    """(stacked users with their half norms, items, item half norms) as the model forms them."""
    import torch
    from tensorrec_b200 import kernels
    from tests.test_tastes_tc_gpu import stacked_operand
    n_tastes, U, d = u.shape
    d_pad = kernels.d_pad_for(d)
    split, scale = stacked_operand(u, a, d_pad)
    n_ops = split.shape[0]
    hsq = kernels.operand_half_sqnorm(split.view(n_ops * U, 2 * d_pad), scale.view(-1), d_pad).view(n_ops, U)
    dev = lambda x: None if x is None else torch.from_numpy(x).cuda()   # noqa: E731
    users = kernels.SideOperands(None, split, scale, dev(ub), U, d, d_pad, hsq=hsq)
    its, isc = kernels.split_f32(torch.from_numpy(item).cuda(), d_pad=d_pad)
    items = kernels.SideOperands(None, its, isc, dev(ib), item.shape[0], d, d_pad)
    return users, items, kernels.item_half_sqnorm(items)


def per_taste_max(T, users, items):
    """max_t of the one-taste Euclidean tensor-core dense scores of every taste slice of `users`."""
    from tensorrec_b200 import kernels
    meta = kernels.pack_item_meta(items.scale, items.bias, items.n_rows)
    best = None
    for t in range(users.hsq.shape[0]):
        s = kernels.score_dense_tc(users.split[t], users.scale[t], users.bias, items.split, meta, users.n_rows,
                                   items.n_rows, users.d_pad, sqnorms=(users.hsq[t], kernels.item_half_sqnorm(items)))
        s = s.cpu().numpy()
        best = s if best is None else np.maximum(best, s)
    return best


def model_of(T, U, I, d, n_tastes, attention, integer, seed, biased=True):
    """A Euclidean TensorRec on tag features -> (model, uf, itf, oracle model)."""
    R, P = T.representation_graphs, T.prediction_graphs
    uf = H.tag_features(U, 200, 20, seed=seed + 1, integer=integer)
    itf = H.tag_features(I, 200, 20, seed=seed + 2, integer=integer)
    wu = [H.linear_weights(200, d, seed=seed + 10 + t, integer=integer) for t in range(n_tastes)]
    wa = [H.linear_weights(200, d, seed=seed + 100 + t, integer=integer) for t in range(n_tastes)] if attention else None
    wi = H.linear_weights(200, d, seed=seed + 3, integer=integer)
    bu = H.feature_biases(200, seed=seed + 4, integer=integer) if biased else None
    bi = H.feature_biases(200, seed=seed + 5, integer=integer) if biased else None
    model = T.TensorRec(n_components=d, n_tastes=n_tastes, biased=biased,
                        prediction_graph=P.EuclideanSimilarityPredictionGraph(),
                        attention_graph=R.LinearRepresentationGraph() if attention else None)
    weights = {'linear_weights_item': wi}
    for t in range(n_tastes):
        weights['linear_weights_user_%d' % t] = wu[t]
        if attention:
            weights['linear_weights_attn_%d' % t] = wa[t]
    if biased:
        weights.update({'feature_biases_user': bu[:, None], 'feature_biases_item': bi[:, None]})
    model.set_weights(weights)
    return model, uf, itf, oracle.OracleModel(wu, wi, bu, bi, attention_weights=wa, prediction='euclidean')


def float_bound(om, uf, itf):
    """(float64 reference scores, |got - ref| bound) of a float fixture (DESIGN §3.12).  Every squared distance is within
    D_j = 8 * 2^-20 (|x_j|^2 + |i|^2) of the exact one (the one-taste Euclidean tolerance: the 3-pass dot product, the
    norms from the split operands, K1's fp32 representations); through the root, |e_j - e_j*| <= min(D_j / |e_j*|,
    sqrt(D_j)).  The softmax weights sum to 1, so logit errors of at most E_a = max_t |ea_t - ea_t*| move pred by at most
    2 E_a sum_t w_t |e_t - pred|, and the taste errors add sum_t w_t |e_t - e_t*|; the fp32 roundings of the roots, the
    collapse and the biases add 4 n_ops 2^-24 of the magnitudes involved."""
    uc, ic = oracle.coo_from_sparse(uf), oracle.coo_from_sparse(itf)
    item = om._repr(om.item_repr, ic, om.item_weights).astype(np.float64)
    isq = (item ** 2).sum(1)

    def sims(weights):
        xs = [om._repr(om.user_repr, uc, w).astype(np.float64) for w in weights]
        e, err = [], []
        for x in xs:
            xsq = (x ** 2).sum(1)
            d2 = np.maximum(xsq[:, None] - 2 * x @ item.T + isq[None, :], 1e-16)
            dd = 8 * 2.0 ** -20 * (xsq[:, None] + isq[None, :])
            e.append(-np.sqrt(d2))
            err.append(np.minimum(dd / np.sqrt(d2), np.sqrt(dd)))
        return np.stack(e), np.stack(err)

    e, ee = sims(om.user_weights)
    n_ops = len(om.user_weights)
    if om.attention_weights is None:
        pred, bound = e.max(0), ee.max(0)
    else:
        ea, eea = sims(om.attention_weights)
        n_ops *= 2
        w = np.exp(ea - ea.max(0))
        w /= w.sum(0)
        pred = (w * e).sum(0)
        bound = (w * ee).sum(0) + 2 * eea.max(0) * (w * np.abs(e - pred)).sum(0)
    mag = np.abs(pred) + np.abs(e).max(0)
    if om.user_bias is not None:
        ub = oracle.project_biases(uc, om.user_bias).astype(np.float64)
        ib = oracle.project_biases(ic, om.item_bias).astype(np.float64)
        pred = pred + ub[:, None] + ib[None, :]
        mag = mag + np.abs(ub)[:, None] + np.abs(ib)[None, :]
    return pred, bound + 4 * n_ops * 2.0 ** -24 * mag


# ---- the max form, dense ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n_tastes', [2, 3, 64])
@pytest.mark.parametrize('d', [40, 64, 128])
@pytest.mark.parametrize('biased', [True, False])
def test_max_dense_is_the_max_of_the_one_taste_scores(T, n_tastes, d, biased):
    from tensorrec_b200 import kernels
    U, I = 301 if n_tastes < 64 else 67, 1000 + 37
    u, _, item, ub, ib = crafted(U, I, d, n_tastes, False, seed=n_tastes + d, biased=biased)
    users, items, ihsq = device_operands(T, u, None, item, ub, ib)
    meta = kernels.pack_item_meta(items.scale, items.bias, I)
    got = kernels.score_dense_tastes(users, items.split, meta, I, n_tastes, False, item_hsq=ihsq).cpu().numpy()
    assert np.array_equal(got, oracle_scores(u, None, item, ub, ib))
    assert np.array_equal(got, per_taste_max(T, users, items))
    # d^2 = 0: the floor, -sqrtf(1e-16f), before the biases
    e0 = -np.sqrt(np.float32(1e-16))
    assert got[1, 0] == (e0 if ub is None else (e0 + ub[1]) + ib[0])
    # float operands: still the max of the one-taste scores, bit for bit
    rng = np.random.default_rng(d)
    fu = rng.standard_normal(u.shape).astype(np.float32)
    fi = rng.standard_normal(item.shape).astype(np.float32)
    users, items, ihsq = device_operands(T, fu, None, fi, ub, ib)
    meta = kernels.pack_item_meta(items.scale, items.bias, I)
    got = kernels.score_dense_tastes(users, items.split, meta, I, n_tastes, False, item_hsq=ihsq).cpu().numpy()
    assert np.array_equal(got, per_taste_max(T, users, items))


# ---- the attention form ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n_tastes', [2, 3, 32])
@pytest.mark.parametrize('d', [40, 128])
def test_attention_integer_fixture_is_exact(T, n_tastes, d):
    from tensorrec_b200 import kernels
    if d <= n_tastes:
        pytest.skip('the selectors need d > n_tastes')
    U, I = 150, 1000 + 37
    u, a, item, ub, ib = crafted(U, I, d, n_tastes, True, seed=n_tastes + d, biased=n_tastes != 3)
    expect = oracle_scores(u, a, item, ub, ib)
    users, items, ihsq = device_operands(T, u, a, item, ub, ib)
    meta = kernels.pack_item_meta(items.scale, items.bias, I)
    got = kernels.score_dense_tastes(users, items.split, meta, I, n_tastes, True, item_hsq=ihsq)
    assert np.array_equal(got.cpu().numpy(), expect)
    # the one-sweep top-k routes score through the same collapse
    for k, topk in ((10, kernels.topk_tastes), (300, kernels.topk_tastes_wide)):
        top = topk(users, items, n_tastes, True, k, item_hsq=ihsq)
        exp_i, exp_s = oracle.top_k_from_scores(expect, k)
        assert np.array_equal(top.items.cpu().numpy(), exp_i)
        assert np.array_equal(top.scores.cpu().numpy(), exp_s)
    # without attention there is no one-sweep top-k
    with pytest.raises(kernels._lib.TrkUnsupportedError):
        kernels.topk_tastes(users, items, 2 * n_tastes, False, 10, item_hsq=ihsq)


@pytest.mark.parametrize('attention', [False, True])
@pytest.mark.parametrize('d', [40, 128])
def test_float_fixture_within_the_bound(T, attention, d):
    model, uf, itf, om = model_of(T, 200, 1100, d, 3, attention, False, seed=d)
    assert model._tensor_score_form() == 'tastes_euclid'
    got = model.predict(uf, itf)
    ref, bound = float_bound(om, uf, itf)
    assert np.all(np.abs(got - ref) <= bound)


def test_model_integer_fixture_is_exact(T):
    model, uf, itf, om = model_of(T, 200, 1100, 64, 3, False, True, seed=1)
    assert np.array_equal(model.predict(uf, itf), om.predict(uf, itf))


# ---- consistency on one model ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('attention', [False, True])
def test_rank_at_equals_predict_rank(T, monkeypatch, attention):
    monkeypatch.setattr(T.tensorrec, 'RANK_AT_MIN_ITEMS', 0)
    monkeypatch.setattr(T.tensorrec, 'RANK_AT_EUCLID_ATTENTION_MIN_ITEMS', 0)
    model, uf, itf, _ = model_of(T, 300, 1000, 64, 3, attention, False, seed=3)
    pairs, listed = make_pairs(4)
    got = model.predict_rank_at(uf, itf, pairs)
    assert model.last_rank_info['path'] == 'exact3_count'
    assert_same_matrix(got, expect_at(model.predict_rank(uf, itf), listed))
    excl = sp.random(300, 1000, density=0.1, format='csr', random_state=6, dtype=np.float32)
    got = model.predict_rank_at(uf, itf, pairs, exclude=excl)
    assert_same_matrix(got, masked_ranks(model.predict(uf, itf), excl, listed))
    if not attention:
        # a pair of rank r <= k is at slot r of the per-taste top-k
        k = 10
        monkeypatch.setattr(T.tensorrec, 'EUCLIDEAN_MIN_ITEMS', 0)
        top = model.predict_top_k(uf, itf, k, exclude=excl)
        assert model.last_topk_info['path'] == 'exact3'
        ex = excl.toarray() != 0
        r, c = got.nonzero()
        checked = 0
        for uu, i, rank in zip(r, c, got[r, c].A1):
            if not ex[uu, i] and rank <= k:
                assert top.items[uu, rank - 1] == i
                checked += 1
        assert checked > 0


def forced(T, monkeypatch, model, uf, itf, k, route, **kw):
    floor = 0 if route != 'dense+rank' else 10 ** 9
    monkeypatch.setattr(T.tensorrec, 'ATTENTION_MIN_ITEMS', floor)
    monkeypatch.setattr(T.tensorrec, 'EXACT_WIDE_MIN_ITEMS', floor)
    top = model.predict_top_k(uf, itf, k, **kw)
    assert model.last_topk_info['path'] == route
    return top


@pytest.mark.parametrize('k', [1, 10, 32, 33, 100, 1000])
def test_attention_routes_equal_dense_rank(T, monkeypatch, k):
    model, uf, itf, _ = model_of(T, 150, 1200 + 37, 40, 3, True, False, seed=k)
    route = 'exact3' if k <= 32 else 'exact3_wide'
    dense = forced(T, monkeypatch, model, uf, itf, k, 'dense+rank')
    fused = forced(T, monkeypatch, model, uf, itf, k, route)
    assert np.array_equal(fused.items, dense.items) and np.array_equal(fused.scores, dense.scores)
    # exclusion and user blocks
    exclude = exclusion(model.predict(uf, itf), k, seed=k + 1)
    dense = forced(T, monkeypatch, model, uf, itf, k, 'dense+rank', exclude=exclude)
    fused = forced(T, monkeypatch, model, uf, itf, k, route, exclude=exclude, user_batch_size=64)
    assert np.array_equal(fused.items, dense.items) and np.array_equal(fused.scores, dense.scores)
    assert (fused.items[3::6] == SENTINEL_ID).all()
    # an item shard at offset 5000 (the exclusion's columns are global ids): the same lists, ids shifted
    offset = 5000
    shifted = sp.hstack([sp.csr_matrix((exclude.shape[0], offset)), sp.csr_matrix(exclude)]).tocsr()
    shard = forced(T, monkeypatch, model, uf, itf, k, route, exclude=shifted, item_id_offset=offset)
    ids = np.where(dense.items == SENTINEL_ID, SENTINEL_ID, dense.items + offset)
    assert np.array_equal(shard.items, ids) and np.array_equal(shard.scores, dense.scores)
