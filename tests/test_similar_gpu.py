"""GPU tests of predict_similar_items_top_k: the filter and exact 3-pass kernels (dot, cosine and Euclidean through
-1/2 |row|^2 biases), the device-side fallback, exclusion, query blocks and the dense+rank route, against the oracle of
tests/similar_topk.py.  Integer fixtures match bit for bit; float fixtures use the tolerances of test_api_gpu.py
(Euclidean on the d^2 scale)."""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from tests import helpers as H
from tests.masked_topk import SENTINEL_ID
from tests.similar_topk import similar_items_top_k
from tests.test_exclude_gpu import exclusion

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def T():
    import torch
    import tensorrec_b200
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    torch.cuda.set_device(0)
    return tensorrec_b200


def make_model(T, I, d, integer, prediction='dot', seed=0, prediction_graph=None):
    """A model with injected weights and its item representations as the oracle computes them."""
    P = T.prediction_graphs
    graphs = {'dot': P.DotProductPredictionGraph, 'cosine': P.CosineSimilarityPredictionGraph,
              'euclidean': P.EuclideanSimilarityPredictionGraph}
    itf = H.tag_features(I, 200, 20, seed=seed + 2, integer=integer)
    wi = H.linear_weights(200, d, seed=seed + 4, integer=integer)
    model = T.TensorRec(n_components=d, prediction_graph=prediction_graph or graphs[prediction]())
    model.set_weights({'linear_weights_user_0': H.linear_weights(200, d, seed=seed + 10, integer=integer),
                       'linear_weights_item': wi,
                       'feature_biases_user': H.feature_biases(200, seed=seed + 5, integer=integer)[:, None],
                       'feature_biases_item': H.feature_biases(200, seed=seed + 6, integer=integer)[:, None]})
    return model, itf, oracle.OracleModel([wi], wi).item_representation(itf)


def query_ids(I, n_queries, seed):
    ids = np.random.default_rng(seed).integers(0, I, n_queries)
    ids[1] = ids[0]                                                     # a duplicate query
    return ids


def assert_same(a, b):
    assert np.array_equal(a.items, b.items) and np.array_equal(a.scores, b.scores)


def check_float(top, prediction, item_repr, ids, n, exclude=None, exclude_self=False):
    """ids differ from the oracle in < 1 % of the slots; every reported score is the oracle's score of that item within
    the fp32 tolerance (dot / cosine: 1e-5 |q||i|; Euclidean: |got^2 - ref^2| <= 8 * 2^-20 (|q|^2 + |i|^2))."""
    exp_i, _ = similar_items_top_k(prediction, item_repr, ids, n, exclude=exclude, exclude_self=exclude_self)
    got_i = np.asarray(top.items)
    real = got_i != SENTINEL_ID
    assert np.array_equal(real, exp_i != SENTINEL_ID)
    assert (got_i != exp_i).mean() < 0.01
    scores = oracle.predict_similar_items(prediction, item_repr, ids)
    q = np.nonzero(real)[0]
    i = got_i[real]
    got, ref = np.asarray(top.scores)[real].astype(np.float64), scores[q, i].astype(np.float64)
    r = oracle.l2_normalize(item_repr) if prediction == 'cosine' else item_repr
    nq, ni = np.linalg.norm(r[ids[q]].astype(np.float64), axis=1), np.linalg.norm(r[i].astype(np.float64), axis=1)
    if prediction == 'euclidean':
        assert np.all(np.abs(got * got - ref * ref) <= 8 * 2.0 ** -20 * (nq * nq + ni * ni) + 1e-12)
    else:
        assert np.all(np.abs(got - ref) <= 1e-5 * nq * ni + 2e-6)


def expected_path(n, path):
    return 'filter' if (path == 'auto' and n <= 12) else 'exact3'


@pytest.mark.parametrize('prediction', ['dot', 'euclidean'])
@pytest.mark.parametrize('d', [10, 64, 128])
@pytest.mark.parametrize('n', [1, 10, 12, 20])
@pytest.mark.parametrize('cluster', ['1', '2'])
@pytest.mark.parametrize('path', ['auto', 'exact'])
def test_integer_fixture_is_bit_identical_to_the_oracle(T, monkeypatch, prediction, d, n, cluster, path):
    monkeypatch.setenv('TRK_FILTER_CLUSTER', cluster)
    monkeypatch.setattr(T.tensorrec, 'TOPK_PATH', path)
    I = 1000 + 37                                                       # n_items not a multiple of 128
    model, itf, item_repr = make_model(T, I, d, integer=True, prediction=prediction, seed=d)
    ids = query_ids(I, 300, seed=n)
    top = model.predict_similar_items_top_k(itf, n, item_ids=ids)
    assert model.last_topk_info['path'] == expected_path(n, path)
    exp_i, exp_s = similar_items_top_k(prediction, item_repr, ids, n)
    assert np.array_equal(top.items, exp_i) and np.array_equal(top.scores, exp_s)
    assert top.items.dtype == np.int32 and top.scores.dtype == np.float32 and top.items.shape == (300, n)


@pytest.mark.parametrize('prediction', ['dot', 'cosine', 'euclidean'])
@pytest.mark.parametrize('d,n', [(64, 10), (128, 12), (128, 20)])
def test_float_fixture_within_tolerance(T, prediction, d, n):
    I = 3000 + 5
    model, itf, item_repr = make_model(T, I, d, integer=False, prediction=prediction, seed=1)
    ids = query_ids(I, 400, seed=2)
    top = model.predict_similar_items_top_k(itf, n, item_ids=ids)
    assert model.last_topk_info['path'] == expected_path(n, 'auto')
    check_float(top, prediction, item_repr, ids, n)


@pytest.mark.parametrize('prediction', ['dot', 'cosine', 'euclidean'])
def test_exclude_self(T, prediction):
    I = 2000
    model, itf, item_repr = make_model(T, I, 64, integer=False, prediction=prediction, seed=3)
    ids = query_ids(I, 300, seed=4)
    top = model.predict_similar_items_top_k(itf, 10, item_ids=ids, exclude_self=True)
    assert not (top.items == ids[:, None]).any()
    check_float(top, prediction, item_repr, ids, 10, exclude_self=True)
    with_self = model.predict_similar_items_top_k(itf, 10, item_ids=ids)
    if prediction != 'dot':        # cosine / Euclidean: an item is its own best match (tie-free fixture)
        assert np.array_equal(with_self.items[:, 0], ids)
    if prediction == 'cosine':
        assert np.all(np.abs(with_self.scores[:, 0] - 1.0) <= 1e-5)


@pytest.mark.parametrize('prediction', ['dot', 'euclidean'])
@pytest.mark.parametrize('n,path', [(10, 'auto'), (12, 'auto'), (10, 'exact'), (20, 'auto')])
def test_exclusion_patterns(T, monkeypatch, prediction, n, path):
    """empty, own top-k, heavy, everything (all sentinels), fewer than n eligible, duplicates and explicit zeros --
    together with exclude_self, whose union with a -1 entry on the query's own id still excludes it."""
    monkeypatch.setattr(T.tensorrec, 'TOPK_PATH', path)
    I = 1500 + 3
    model, itf, item_repr = make_model(T, I, 64, integer=True, prediction=prediction, seed=5)
    ids = query_ids(I, 240, seed=6)
    scores = oracle.predict_similar_items(prediction, item_repr, ids)
    exclude = exclusion(scores, n, seed=n)
    rows = np.arange(len(ids))
    for exclude_self in (False, True):
        ex = exclude
        if exclude_self:      # plus -1 on every own id: where the pattern already holds it, the entries sum to 0
            ex = sp.coo_matrix((np.concatenate([exclude.data, -np.ones(len(ids))]),
                                (np.concatenate([exclude.row, rows]), np.concatenate([exclude.col, ids]))),
                               shape=(len(ids), I))
        top = model.predict_similar_items_top_k(itf, n, item_ids=ids, exclude=ex, exclude_self=exclude_self)
        assert model.last_topk_info['path'] == expected_path(n, path)
        exp_i, exp_s = similar_items_top_k(prediction, item_repr, ids, n, exclude=ex, exclude_self=exclude_self)
        assert np.array_equal(top.items, exp_i) and np.array_equal(top.scores, exp_s)
        assert (top.items[3::6] == SENTINEL_ID).all()                 # "everything" rows
    plain = model.predict_similar_items_top_k(itf, n, item_ids=ids)
    for empty in (sp.csr_matrix((len(ids), I)), sp.coo_matrix(([0.0], ([3], [7])), shape=(len(ids), I))):
        assert_same(model.predict_similar_items_top_k(itf, n, item_ids=ids, exclude=empty), plain)


@pytest.mark.parametrize('prediction', ['dot', 'euclidean'])
def test_tie_heavy_rows_take_the_device_fallback(T, prediction):
    """All-equal item vectors: every score of a row ties (Euclidean: every distance is 0 and clamps), the filter's
    buffer overflows and the rows go through the exact kernel on the device."""
    I, d, n = 2000, 64, 10
    P = T.prediction_graphs
    graph = P.EuclideanSimilarityPredictionGraph() if prediction == 'euclidean' else P.DotProductPredictionGraph()
    itf = sp.csr_matrix(np.ones((I, 1), np.float32))
    wi = np.ones((1, d), np.float32)
    model = T.TensorRec(n_components=d, biased=False, prediction_graph=graph)
    model.set_weights({'linear_weights_user_0': wi, 'linear_weights_item': wi})
    item_repr = oracle.OracleModel([wi], wi).item_representation(itf)
    ids = query_ids(I, 700, seed=7)
    scores = oracle.predict_similar_items(prediction, item_repr, ids)
    for exclude in (None, exclusion(scores, n, seed=8)):
        top = model.predict_similar_items_top_k(itf, n, item_ids=ids, exclude=exclude)
        assert model.last_topk_info['path'] == 'filter' and model.last_topk_info['fallback_rows'] > 0
        exp_i, exp_s = similar_items_top_k(prediction, item_repr, ids, n, exclude=exclude)
        assert np.array_equal(top.items, exp_i) and np.array_equal(top.scores, exp_s)


@pytest.mark.parametrize('prediction', ['dot', 'cosine', 'euclidean'])
def test_call_forms_are_bit_identical(T, prediction):
    import torch
    I = 1000 + 21
    model, itf, _ = make_model(T, I, 128, integer=False, prediction=prediction, seed=9)
    whole = model.predict_similar_items_top_k(itf, 10)
    assert whole.items.shape == (I, 10)
    assert_same(model.predict_similar_items_top_k(itf, 10, item_ids=np.arange(I)), whole)
    assert_same(model.predict_similar_items_top_k(itf, 10, item_batch_size=128), whole)
    assert_same(model.predict_similar_items_top_k(itf, 10, item_ids=list(range(I)), item_batch_size=300), whole)
    assert_same(model.predict_similar_items_top_k(itf, 10), whole)                         # repeated call
    dev = model.predict_similar_items_top_k(itf, 10, to_host=False)
    assert isinstance(dev.items, torch.Tensor) and dev.items.is_cuda
    assert np.array_equal(dev.items.cpu().numpy(), whole.items)
    ids = np.array([7, 3, 7, 1020, 3, 7], dtype=np.int32)                # duplicate queries give identical rows
    dup = model.predict_similar_items_top_k(itf, 10, item_ids=ids)
    assert np.array_equal(dup.items, whole.items[ids]) and np.array_equal(dup.scores, whole.scores[ids])
    empty = model.predict_similar_items_top_k(itf, 10, item_ids=[])
    assert empty.items.shape == (0, 10) and empty.scores.shape == (0, 10)


def user_dot_graph(T):
    """A user-defined prediction graph (the dot product written by hand): only the dense form is needed here."""
    import torch

    class UserDot(T.prediction_graphs.AbstractPredictionGraph):
        def connect_dense_prediction_graph(self, tf_user_representation, tf_item_representation):
            return torch.matmul(tf_user_representation, tf_item_representation.t())
    return UserDot()


@pytest.mark.parametrize('route', ['score_path_exact', 'n40', 'n40_euclidean', 'user_graph'])
def test_dense_rank_route(T, monkeypatch, route):
    prediction = 'euclidean' if route == 'n40_euclidean' else 'dot'
    n = 40 if route.startswith('n40') else 10
    graph = user_dot_graph(T) if route == 'user_graph' else None
    if route == 'score_path_exact':
        monkeypatch.setattr(T.tensorrec, 'SCORE_PATH', 'exact')
    I = 900 + 11
    model, itf, item_repr = make_model(T, I, 32, integer=True, prediction=prediction, seed=10, prediction_graph=graph)
    ids = query_ids(I, 200, seed=11)
    scores = oracle.predict_similar_items(prediction, item_repr, ids)
    exclude = exclusion(scores, n, seed=12)
    for kw in ({}, {'exclude': exclude, 'exclude_self': True}, {'item_batch_size': 64}):
        top = model.predict_similar_items_top_k(itf, n, item_ids=ids, **kw)
        assert model.last_topk_info['path'] == 'dense+rank'
        exp_i, exp_s = similar_items_top_k(prediction, item_repr, ids, n, exclude=kw.get('exclude'),
                                           exclude_self=kw.get('exclude_self', False))
        assert np.array_equal(top.items, exp_i) and np.array_equal(top.scores, exp_s)


def test_tensor_score_path_insists(T, monkeypatch):
    monkeypatch.setattr(T.tensorrec, 'SCORE_PATH', 'tensor')
    model, itf, _ = make_model(T, 300, 32, integer=True, prediction_graph=user_dot_graph(T))
    with pytest.raises(RuntimeError, match='tensor'):
        model.predict_similar_items_top_k(itf, 10)


@pytest.mark.parametrize('prediction', ['dot', 'cosine', 'euclidean'])
def test_agrees_with_predict_similar_items(T, prediction):
    I, n = 500, 8
    model, itf, _ = make_model(T, I, 48, integer=False, prediction=prediction, seed=13)
    ids = np.array([0, 17, 250, 499])
    top = model.predict_similar_items_top_k(itf, n, item_ids=ids)
    old = model.predict_similar_items(itf, ids, n)
    for q in range(len(ids)):
        old_ids = [int(i) for i, _ in old[q]]
        old_scores = dict((int(i), float(s)) for i, s in old[q])
        assert set(old_ids) == set(top.items[q].tolist())
        for i, s in zip(top.items[q], top.scores[q]):
            assert abs(float(s) - old_scores[int(i)]) <= 1e-5 * max(1.0, abs(old_scores[int(i)]))
