"""GPU tests of predict_at: the exact kernel's pairs mode ('exact3_pairs') against predict() bit for bit (int32 views:
the sign of zero counts) for every score form, biased or not, float or integer-valued; the independence of a pair's
score from the other slots of its gathered tiles; and the 'dense+gather' route of the models the pairs mode does not
score."""
import numpy as np
import pytest
import scipy.sparse as sp

from tests import helpers as H

pytestmark = pytest.mark.gpu

U = 300                 # not a multiple of a user block (128, 2P): the last block is partial
FORMS = ['dot', 'cosine', 'euclidean', 'max', 'attention', 'euclid_max', 'euclid_attention']


@pytest.fixture(autouse=True)
def pairs_mode_on_small_catalogues(monkeypatch):
    """The fixtures' catalogues lie below PREDICT_AT_MIN_ITEMS: the pairs mode is forced on them (the dense+gather
    test forces the other route on its own)."""
    import tensorrec_b200
    monkeypatch.setattr(tensorrec_b200.tensorrec, 'PREDICT_AT_MIN_ITEMS', 0)


@pytest.fixture(scope='module')
def T():
    import torch
    import tensorrec_b200
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    torch.cuda.set_device(0)
    return tensorrec_b200


def make_model(T, form, d, n_items, biased=True, integer=False, seed=0, prediction_graph=None):
    """-> (model, user features, item features).  form: 'dot', 'cosine', 'euclidean', or a three-taste 'max' /
    'attention' of dot products or ('euclid_...') of Euclidean similarities."""
    n_tastes = 3 if form in ('max', 'attention', 'euclid_max', 'euclid_attention') else 1
    attention = form in ('attention', 'euclid_attention')
    uf = H.tag_features(U, 200, 20, seed=seed + 1, integer=integer)
    itf = H.tag_features(n_items, 200, 20, seed=seed + 2, integer=integer)
    P, R = T.prediction_graphs, T.representation_graphs
    pred = prediction_graph
    if pred is None:
        pred = (P.EuclideanSimilarityPredictionGraph() if form in ('euclidean', 'euclid_max', 'euclid_attention')
                else P.CosineSimilarityPredictionGraph() if form == 'cosine' else P.DotProductPredictionGraph())
    model = T.TensorRec(n_components=d, n_tastes=n_tastes, prediction_graph=pred, biased=biased,
                        attention_graph=R.LinearRepresentationGraph() if attention else None)
    weights = {'linear_weights_item': H.linear_weights(200, d, seed=seed + 4, integer=integer)}
    if biased:
        weights['feature_biases_user'] = H.feature_biases(200, seed=seed + 5, integer=integer)[:, None]
        weights['feature_biases_item'] = H.feature_biases(200, seed=seed + 6, integer=integer)[:, None]
    for t in range(n_tastes):
        weights['linear_weights_user_%d' % t] = H.linear_weights(200, d, seed=seed + 10 + t, integer=integer)
        if attention:
            weights['linear_weights_attn_%d' % t] = H.linear_weights(200, d, seed=seed + 20 + t, integer=integer)
    model.set_weights(weights)
    return model, uf, itf


def make_pairs(seed, n_items, heavy=False):
    """An unsummed COO listing: an empty row, rows of 1 .. 400 pairs, duplicates, explicit zeros (not listed) and, with
    heavy, a row of 150 items of one residue and an item listed by every row of the second user block."""
    rng = np.random.default_rng(seed)
    per_row = rng.integers(0, 12, U)
    per_row[:5] = [0, 1, 33, 150, 400]
    rows = np.repeat(np.arange(U), per_row)
    cols = np.concatenate([rng.choice(n_items, k, replace=False) for k in per_row])
    if heavy:
        rows = np.concatenate([rows, np.full(150, 7), np.arange(128, 256)])
        cols = np.concatenate([cols, 3 + 128 * np.arange(150), np.full(128, 4097)])
    vals = np.ones(rows.size, np.float32)
    zr, zc = rng.integers(0, U, 50), rng.integers(0, n_items, 50)
    pairs = sp.coo_matrix((np.concatenate([vals, np.zeros(50, np.float32)]),
                           (np.concatenate([rows, zr]), np.concatenate([cols, zc]))), shape=(U, n_items))
    listed = sp.csr_matrix((np.ones(rows.size, bool), (rows, cols)), shape=(U, n_items))
    listed.sum_duplicates()
    listed.sort_indices()
    return pairs, listed


def assert_scores_equal_predict(got, full, listed):
    assert isinstance(got, sp.csr_matrix) and got.dtype == np.float32 and got.has_sorted_indices
    assert got.shape == listed.shape and got.nnz == listed.nnz
    assert np.array_equal(got.indptr, listed.indptr) and np.array_equal(got.indices, listed.indices)
    r, c = listed.nonzero()
    want = np.ascontiguousarray(full[r, c], dtype=np.float32)
    assert np.array_equal(got.data.view(np.int32), want.view(np.int32))


@pytest.mark.parametrize('form', FORMS)
@pytest.mark.parametrize('d', [10, 64, 100, 128])
@pytest.mark.parametrize('biased', [True, False])
@pytest.mark.parametrize('integer', [False, True])
def test_predict_at_equals_predict(T, form, d, biased, integer):
    n_items = 2600 + 7
    model, uf, itf = make_model(T, form, d, n_items, biased=biased, integer=integer, seed=d)
    pairs, listed = make_pairs(d + 1, n_items)
    full = model.predict(uf, itf)
    got = model.predict_at(uf, itf, pairs)
    assert model.last_predict_at_info['path'] == 'exact3_pairs' and model.last_predict_at_info['tiles'] > 0
    assert_scores_equal_predict(got, full, listed)
    assert_scores_equal_predict(model.predict_at(uf, itf, pairs, user_batch_size=200), full, listed)


@pytest.mark.parametrize('form', FORMS)
def test_many_tiles_rows_equal_predict(T, form):
    n_items = 150 * 128 + 5
    model, uf, itf = make_model(T, form, 64, n_items, seed=3)
    pairs, listed = make_pairs(4, n_items, heavy=True)
    full = model.predict(uf, itf)
    got = model.predict_at(uf, itf, pairs)
    assert model.last_predict_at_info['tiles'] >= 150
    assert_scores_equal_predict(got, full, listed)


@pytest.mark.parametrize('form', FORMS)
def test_a_pairs_score_does_not_depend_on_its_tiles_other_slots(T, form):
    """The same pairs scored in calls whose other listings differ: their gathered tiles hold different neighbours (and
    tile indices), the bits stay."""
    n_items = 5000 + 3
    model, uf, itf = make_model(T, form, 100, n_items, seed=7)
    rng = np.random.default_rng(8)
    base_r, base_c = rng.integers(0, U, 400), rng.integers(0, n_items, 400)
    base = sp.csr_matrix((np.ones(400, np.float32), (base_r, base_c)), shape=(U, n_items))
    base.data[:] = 1
    got = []
    for seed in (9, 10, 11):
        g = np.random.default_rng(seed)
        k = 3000 * (seed - 8)
        other = sp.csr_matrix((np.ones(k, np.float32), (g.integers(0, U, k), g.integers(0, n_items, k))),
                              shape=(U, n_items))
        listing = (base + other).astype(bool).astype(np.float32)
        out = model.predict_at(uf, itf, listing).tocsr()
        got.append(np.asarray(out[base_r, base_c]).reshape(-1).view(np.int32).copy())
    assert np.array_equal(got[0], got[1]) and np.array_equal(got[0], got[2])
    full = model.predict(uf, itf)
    assert np.array_equal(got[0], np.ascontiguousarray(full[base_r, base_c]).view(np.int32))


def user_dot_graph(T):
    import torch

    class UserDot(T.prediction_graphs.AbstractPredictionGraph):
        def connect_dense_prediction_graph(self, tf_user_representation, tf_item_representation):
            return torch.matmul(tf_user_representation, tf_item_representation.t())
    return UserDot()


@pytest.mark.parametrize('route', ['user_graph', 'd200', 'score_path_exact', 'below_min_items'])
def test_dense_gather_route_equals_predict(T, monkeypatch, route):
    n_items = 1000 + 3
    if route == 'score_path_exact':
        monkeypatch.setattr(T.tensorrec, 'SCORE_PATH', 'exact')
    if route == 'below_min_items':     # a tensor-scored model on a catalogue below the pairs mode's floor
        monkeypatch.setattr(T.tensorrec, 'PREDICT_AT_MIN_ITEMS', n_items + 1)
    model, uf, itf = make_model(T, 'dot', 200 if route == 'd200' else 32, n_items, seed=12,
                                prediction_graph=user_dot_graph(T) if route == 'user_graph' else None)
    pairs, listed = make_pairs(13, n_items)
    full = model.predict(uf, itf)
    got = model.predict_at(uf, itf, pairs, user_batch_size=200)
    assert model.last_predict_at_info == {'path': 'dense+gather', 'tiles': 0}
    assert_scores_equal_predict(got, full, listed)
