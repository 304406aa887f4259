"""GPU tests of the wide filter route (32 < k <= 1024): predict_top_k / predict_rank(k) and predict_similar_items_top_k
against the masked oracle (tests/masked_topk.py, tests/similar_topk.py), and the user blocks of the dense+rank route.
The route is reached at small shapes by lowering tensorrec.WIDE_MIN_ITEMS.  Integer fixtures match bit for bit; float
fixtures use the tolerances of test_exclude_gpu.py and test_similar_gpu.py."""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from tests import helpers as H
from tests.masked_topk import SENTINEL_ID, masked_top_k
from tests.similar_topk import similar_items_top_k
from tests.test_exclude_gpu import check, exclusion, make_model
from tests.test_similar_gpu import check_float, query_ids
from tests.test_similar_gpu import make_model as make_item_model

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def T():
    import torch
    import tensorrec_b200
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    torch.cuda.set_device(0)
    return tensorrec_b200


@pytest.fixture
def wide(T, monkeypatch):
    monkeypatch.setattr(T.tensorrec, 'WIDE_MIN_ITEMS', 0)
    return T


def assert_same(a, b):
    assert np.array_equal(a.items, b.items) and np.array_equal(a.scores, b.scores)


@pytest.mark.parametrize('d', [64, 128])
@pytest.mark.parametrize('k', [33, 100, 256, 1024])
@pytest.mark.parametrize('cluster', ['1', '2'])
def test_integer_fixture_is_bit_identical_to_the_masked_oracle(wide, monkeypatch, d, k, cluster):
    monkeypatch.setenv('TRK_FILTER_CLUSTER', cluster)
    model, uf, itf, scores = make_model(wide, 300, 3000 + 37, d, integer=True, seed=k)
    exclude = exclusion(scores, k, seed=d + k)        # includes rows with fewer than k eligible items
    top = model.predict_top_k(uf, itf, k, exclude=exclude)
    assert model.last_topk_info['path'] == 'wide'
    check(top, scores, exclude, k, integer=True)
    plain = model.predict_rank(uf, itf, k=k)
    exp_i, exp_s = oracle.top_k_from_scores(scores, k)
    assert np.array_equal(plain.items, exp_i) and np.array_equal(plain.scores, exp_s)


def test_thousands_of_excluded_items_among_the_best(wide):
    k = 100
    model, uf, itf, scores = make_model(wide, 260, 9000, 128, integer=True, seed=3)
    best = oracle.top_k_from_scores(scores, 4000)[0]
    rng = np.random.default_rng(4)
    rows, cols = [], []
    for u in range(scores.shape[0]):
        c = best[u, :3000] if u % 2 == 0 else rng.choice(best[u], 2500, replace=False)
        rows.append(np.full(len(c), u))
        cols.append(c)
    exclude = sp.csr_matrix((np.ones(sum(map(len, cols))), (np.concatenate(rows), np.concatenate(cols))),
                            shape=scores.shape)
    top = model.predict_top_k(uf, itf, k, exclude=exclude)
    assert model.last_topk_info['path'] == 'wide'
    check(top, scores, exclude, k, integer=True)


def test_tie_heavy_rows_go_through_the_fallback(wide):
    """Every item has the same features: all scores of a row tie, no row can be certified, every row is scored dense,
    ranked and still returned in reference order (ties by id)."""
    T = wide
    U, I, k = 200, 2500, 100
    uf = H.tag_features(U, 200, 20, seed=1, integer=True)
    one = H.tag_features(1, 200, 20, seed=2, integer=True)
    itf = sp.vstack([one] * I).tocsr()
    wu, wi = H.linear_weights(200, 64, seed=3, integer=True), H.linear_weights(200, 64, seed=4, integer=True)
    bu = H.feature_biases(200, seed=5, integer=True)
    model = T.TensorRec(n_components=64)
    model.set_weights({'linear_weights_user_0': wu, 'linear_weights_item': wi, 'feature_biases_user': bu[:, None],
                       'feature_biases_item': np.zeros((200, 1), np.float32)})
    scores = oracle.OracleModel([wu], wi, bu, np.zeros(200, np.float32)).predict(uf, itf)
    exclude = exclusion(scores, k, seed=6)
    top = model.predict_top_k(uf, itf, k, exclude=exclude)
    assert model.last_topk_info['path'] == 'wide'
    assert model.last_topk_info['fallback_rows'] > 0
    check(top, scores, exclude, k, integer=True)


@pytest.mark.parametrize('prediction', ['dot', 'cosine'])
@pytest.mark.parametrize('k', [50, 300])
def test_float_fixture_within_tolerance(wide, prediction, k):
    P = wide.prediction_graphs
    graph = P.CosineSimilarityPredictionGraph() if prediction == 'cosine' else None
    model, uf, itf, _ = make_model(wide, 400, 5000, 128, integer=False, seed=7, prediction=graph)
    scores = model.predict(uf, itf)
    exclude = exclusion(scores, k, seed=8)
    top = model.predict_top_k(uf, itf, k, exclude=exclude)
    assert model.last_topk_info['path'] == 'wide'
    check(top, scores, exclude, k, integer=False)
    # the dense fallback is exact, so the oracle comparison alone would pass even if no row were ever certified: on
    # continuous scores the certificate must accept (almost) every row, with and without exclusion
    assert model.last_topk_info['fallback_rows'] < scores.shape[0] // 10
    model.predict_top_k(uf, itf, k)
    assert model.last_topk_info['fallback_rows'] < scores.shape[0] // 10


def test_user_blocks_equal_one_block(wide):
    model, uf, itf, scores = make_model(wide, 700, 4000, 128, integer=False, seed=9)
    exclude = exclusion(scores, 200, seed=10)
    whole = model.predict_top_k(uf, itf, 200, exclude=exclude)
    for size in (128, 300):
        assert_same(model.predict_top_k(uf, itf, 200, exclude=exclude, user_batch_size=size), whole)


def test_shards_merged_equal_the_whole(wide):
    import torch
    from tensorrec_b200 import kernels
    k = 150
    model, uf, itf, scores = make_model(wide, 333, 4100, 128, integer=True, seed=11)
    whole = model.predict_top_k(uf, itf, k)
    bounds = [0, 1000, 4100]       # a shard smaller than WIDE_MIN_ITEMS still takes the wide route (rank-invariant)
    parts = []
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        top = model.predict_top_k(uf, itf.tocsr()[lo:hi], k, item_id_offset=lo, to_host=False)
        assert model.last_topk_info['path'] == 'wide'
        parts.append(torch.cat([top.scores.view(torch.int32), top.items], dim=1))
    merged = kernels.topk_merge_received(torch.stack(parts).contiguous(), uf.shape[0], len(parts), k)
    assert np.array_equal(merged.items.cpu().numpy(), whole.items)
    assert np.array_equal(merged.scores.cpu().numpy(), whole.scores)


def test_route_of_sharded_calls_ignores_the_shard_size(T, monkeypatch):
    monkeypatch.setattr(T.tensorrec, 'WIDE_MIN_ITEMS', 10 ** 9)
    model, uf, itf, scores = make_model(T, 100, 1500, 64, integer=True, seed=12)
    model.predict_top_k(uf, itf, 64)
    assert model.last_topk_info['path'] == 'dense+rank'
    top = model.predict_top_k(uf, itf.tocsr()[500:], 64, item_id_offset=500)
    assert model.last_topk_info['path'] == 'wide'
    exp_i, exp_s = oracle.top_k_from_scores(scores[:, 500:], 64)
    assert np.array_equal(top.items, np.where(exp_i == SENTINEL_ID, exp_i, exp_i + 500))
    assert np.array_equal(top.scores, exp_s)


def test_smaller_k_is_a_prefix_of_a_larger_one(wide):
    model, uf, itf, _ = make_model(wide, 300, 3000, 128, integer=True, seed=13)
    big = model.predict_top_k(uf, itf, 400)
    for k in (33, 100):
        small = model.predict_top_k(uf, itf, k)
        assert np.array_equal(small.items, big.items[:, :k]) and np.array_equal(small.scores, big.scores[:, :k])


@pytest.mark.parametrize('prediction', ['dot', 'cosine', 'euclidean'])
@pytest.mark.parametrize('n', [50, 100])
def test_similar_items(wide, prediction, n):
    integer = prediction != 'cosine'
    I = 3000 + 5
    model, itf, item_repr = make_item_model(wide, I, 64, integer=integer, prediction=prediction, seed=14)
    ids = query_ids(I, 300, seed=15)
    scores = oracle.predict_similar_items(prediction, item_repr, ids)
    exclude = exclusion(scores, n, seed=16)
    for kw in ({}, {'exclude_self': True}, {'exclude': exclude, 'exclude_self': True}, {'item_batch_size': 100}):
        top = model.predict_similar_items_top_k(itf, n, item_ids=ids, **kw)
        assert model.last_topk_info['path'] == 'wide'
        if integer:
            exp_i, exp_s = similar_items_top_k(prediction, item_repr, ids, n, exclude=kw.get('exclude'),
                                               exclude_self=kw.get('exclude_self', False))
            assert np.array_equal(top.items, exp_i) and np.array_equal(top.scores, exp_s)
        else:
            check_float(top, prediction, item_repr, ids, n, exclude=kw.get('exclude'),
                        exclude_self=kw.get('exclude_self', False))


def test_dense_route_blocks_are_bit_identical_to_one_block(T, monkeypatch):
    model, uf, itf, scores = make_model(T, 257, 1500, 64, integer=False, seed=17)
    exclude = exclusion(scores, 100, seed=18)
    whole = model.predict_top_k(uf, itf, 100, exclude=exclude)
    assert model.last_topk_info['path'] == 'dense+rank'
    monkeypatch.setattr(T.TensorRec, 'PREDICT_BLOCK_BYTES', 35 * 1500 * 40)    # 40 users per block
    assert_same(model.predict_top_k(uf, itf, 100, exclude=exclude), whole)
    exp_i, _ = masked_top_k(scores, exclude, 100)
    assert (np.asarray(whole.items) != exp_i).mean() < 0.01
