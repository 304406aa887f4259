"""GPU tests of predict_rank_at: the exact kernel's counting mode ('exact3_count') against predict_rank() bit for bit
for every score form, against the oracle on integer fixtures, with exclusion against the masked closed form and
predict_top_k, and the 'dense+rank' route against the same matrix."""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from tests import helpers as H

pytestmark = pytest.mark.gpu

U, I = 300, 1000        # neither a multiple of a user block (128, 2P) nor of an item tile (128)


@pytest.fixture(scope='module')
def T():
    import torch
    import tensorrec_b200
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    torch.cuda.set_device(0)
    return tensorrec_b200


def make_model(T, form, d, integer, seed=0):
    """-> (model, user features, item features, oracle scores or None).  form: 'dot', 'cosine', 'euclidean', 'max'
    (three tastes) or 'attention' (three tastes)."""
    n_tastes = 3 if form in ('max', 'attention') else 1
    uf = H.tag_features(U, 200, 20, seed=seed + 1, integer=integer)
    itf = H.tag_features(I, 200, 20, seed=seed + 2, integer=integer)
    wu = [H.linear_weights(200, d, seed=seed + 10 + t, integer=integer) for t in range(n_tastes)]
    wa = [H.linear_weights(200, d, seed=seed + 20 + t, integer=integer) for t in range(n_tastes)]
    wi = H.linear_weights(200, d, seed=seed + 4, integer=integer)
    bu, bi = H.feature_biases(200, seed=seed + 5, integer=integer), H.feature_biases(200, seed=seed + 6, integer=integer)
    P, R = T.prediction_graphs, T.representation_graphs
    pred = {'euclidean': P.EuclideanSimilarityPredictionGraph(), 'cosine': P.CosineSimilarityPredictionGraph()}.get(
        form, P.DotProductPredictionGraph())
    model = T.TensorRec(n_components=d, n_tastes=n_tastes, prediction_graph=pred,
                        attention_graph=R.LinearRepresentationGraph() if form == 'attention' else None)
    weights = {'linear_weights_item': wi, 'feature_biases_user': bu[:, None], 'feature_biases_item': bi[:, None]}
    for t in range(n_tastes):
        weights['linear_weights_user_%d' % t] = wu[t]
        if form == 'attention':
            weights['linear_weights_attn_%d' % t] = wa[t]
    model.set_weights(weights)
    scores = None
    if integer and form in ('dot', 'euclidean', 'max'):
        om = oracle.OracleModel(wu, wi, bu, bi, prediction='euclidean' if form == 'euclidean' else 'dot')
        scores = om.predict(uf, itf)
    return model, uf, itf, scores


def make_pairs(seed, n_users=U, n_items=I):
    """(pairs, listed): an unsummed COO matrix with rows of 0, 1, 32, 33 and 100+ listed pairs, duplicate entries of
    listed pairs, explicit zeros and duplicates that cancel to zero (neither listed), and the boolean CSR of the pairs
    it lists."""
    rng = np.random.default_rng(seed)
    per_row = rng.integers(0, 12, n_users)
    per_row[:6] = [0, 1, 32, 33, 150, 400]
    rows = np.repeat(np.arange(n_users), per_row)
    cols = np.concatenate([rng.choice(n_items, k, replace=False) for k in per_row])
    vals = rng.integers(1, 3, rows.size).astype(np.float32)
    listed = sp.csr_matrix((np.ones(rows.size, bool), (rows, cols)), shape=(n_users, n_items))
    dup = rng.random(rows.size) < 0.1                       # a second entry of a listed pair: the sum stays > 0
    free_r, free_c = rng.integers(0, n_users, 200), rng.integers(0, n_items, 200)
    free = ~np.asarray(listed[free_r, free_c]).reshape(-1)
    free_r, free_c = free_r[free][:100], free_c[free][:100]
    zr, zc, cr, cc = free_r[:50], free_c[:50], free_r[50:], free_c[50:]
    all_r = np.concatenate([rows, rows[dup], zr, cr, cr])
    all_c = np.concatenate([cols, cols[dup], zc, cc, cc])
    all_v = np.concatenate([vals, vals[dup], np.zeros(zr.size, np.float32), np.full(cr.size, 2, np.float32),
                            np.full(cr.size, -2, np.float32)])
    pairs = sp.coo_matrix((all_v, (all_r, all_c)), shape=(n_users, n_items))
    assert dup.any() and (pairs.data == 0).sum() >= 40 and cr.size >= 40
    return pairs, listed


def expect_at(full, listed):
    r, c = listed.nonzero()
    return sp.csr_matrix((full[r, c].astype(np.int32), (r, c)), shape=listed.shape)


def assert_same_matrix(got, want):
    assert isinstance(got, sp.csr_matrix) and got.dtype == np.int32 and got.has_sorted_indices
    assert got.shape == want.shape and got.nnz == want.nnz
    want = sp.csr_matrix(want)
    want.sort_indices()
    assert np.array_equal(got.indptr, want.indptr) and np.array_equal(got.indices, want.indices)
    assert np.array_equal(got.data, want.data)


def masked_ranks(scores, excl, listed):
    out = []
    ex = excl.toarray() != 0
    for r, c in zip(*listed.nonzero()):
        s = scores[r]
        ok = ~ex[r]
        ok[c] = False
        j = np.arange(s.shape[0])
        out.append(1 + int(np.sum(ok & ((s > s[c]) | ((s == s[c]) & (j < c))))))
    r, c = listed.nonzero()
    return sp.csr_matrix((np.array(out, np.int32), (r, c)), shape=listed.shape)


def force(monkeypatch, T, route):
    monkeypatch.setattr(T.tensorrec, 'RANK_AT_MIN_ITEMS', 0 if route == 'exact3_count' else 10 ** 9)


@pytest.mark.parametrize('form', ['dot', 'cosine', 'euclidean', 'max', 'attention'])
@pytest.mark.parametrize('d', [40, 128])
@pytest.mark.parametrize('integer', [True, False])
def test_counting_mode_equals_predict_rank(T, monkeypatch, form, d, integer):
    force(monkeypatch, T, 'exact3_count')
    model, uf, itf, scores = make_model(T, form, d, integer, seed=d)
    pairs, listed = make_pairs(d + (1 if integer else 0))
    got = model.predict_rank_at(uf, itf, pairs)
    assert model.last_rank_info == {'path': 'exact3_count', 'passes': 13}
    full = model.predict_rank(uf, itf)
    assert_same_matrix(got, expect_at(full, listed))
    if scores is not None:
        assert_same_matrix(got, expect_at(oracle.rank_predictions(scores), listed))


@pytest.mark.parametrize('form', ['dot', 'euclidean', 'max', 'attention'])
def test_exclusion_equals_the_masked_closed_form_and_the_top_k(T, monkeypatch, form):
    force(monkeypatch, T, 'exact3_count')
    model, uf, itf, _ = make_model(T, form, 64, True, seed=3)
    pairs, listed = make_pairs(5)
    excl = sp.random(U, I, density=0.1, format='csr', random_state=6, dtype=np.float32)
    excl = excl + sp.csr_matrix(listed.multiply(sp.random(U, I, density=0.5, format='csr', random_state=7) != 0))
    scores = model.predict(uf, itf)
    got = model.predict_rank_at(uf, itf, pairs, exclude=excl)
    assert_same_matrix(got, masked_ranks(scores, excl, listed))
    k = 10
    top = model.predict_top_k(uf, itf, k, exclude=excl)
    ex = excl.toarray() != 0
    r, c = got.nonzero()
    checked = 0
    for u, i, rank in zip(r, c, got[r, c].A1):
        if not ex[u, i] and rank <= k:
            assert top.items[u, rank - 1] == i
            checked += 1
    assert checked > 0


def test_splits_user_blocks_and_the_dense_route_agree(T, monkeypatch):
    from tensorrec_b200 import kernels
    model, uf, itf, _ = make_model(T, 'dot', 128, False, seed=9)
    pairs, listed = make_pairs(11)
    excl = sp.random(U, I, density=0.05, format='csr', random_state=12, dtype=np.float32)
    force(monkeypatch, T, 'exact3_count')
    base = model.predict_rank_at(uf, itf, pairs)
    base_ex = model.predict_rank_at(uf, itf, pairs, exclude=excl)
    assert_same_matrix(base, expect_at(model.predict_rank(uf, itf), listed))
    with monkeypatch.context() as m:
        m.setattr(kernels, 'default_splits', lambda *_: 5)
        assert_same_matrix(model.predict_rank_at(uf, itf, pairs), base)
        assert_same_matrix(model.predict_rank_at(uf, itf, pairs, exclude=excl), base_ex)
    assert_same_matrix(model.predict_rank_at(uf, itf, pairs, user_batch_size=200), base)     # rounded down to 128
    force(monkeypatch, T, 'dense+rank')
    assert_same_matrix(model.predict_rank_at(uf, itf, pairs), base)
    assert model.last_rank_info['path'] == 'dense+rank'
    assert_same_matrix(model.predict_rank_at(uf, itf, pairs, exclude=excl), base_ex)
    assert_same_matrix(model.predict_rank_at(uf, itf, pairs, exclude=excl, user_batch_size=100), base_ex)


def test_tastes_blocks_and_empty_pairs(T, monkeypatch):
    force(monkeypatch, T, 'exact3_count')
    model, uf, itf, _ = make_model(T, 'max', 40, False, seed=13)
    pairs, listed = make_pairs(14)
    full = model.predict_rank(uf, itf)
    assert_same_matrix(model.predict_rank_at(uf, itf, pairs, user_batch_size=100), expect_at(full, listed))  # 2P = 42
    empty = model.predict_rank_at(uf, itf, sp.csr_matrix((U, I), dtype=np.float32))
    assert empty.nnz == 0 and empty.shape == (U, I)


def test_recall_from_rank_at_equals_recall_from_predict_rank(T, monkeypatch):
    from tensorrec_b200 import eval as tr_eval
    force(monkeypatch, T, 'exact3_count')
    model, uf, itf, _ = make_model(T, 'dot', 64, False, seed=15)
    test = sp.random(U, I, density=0.01, format='csr', random_state=16, dtype=np.float32)
    ranks = model.predict_rank_at(uf, itf, test)
    full = model.predict_rank(uf, itf)
    for k in (1, 10, 100, 1000):
        np.testing.assert_array_equal(tr_eval.recall_at_k(ranks, test, k=k), tr_eval.recall_at_k(full, test, k=k))
