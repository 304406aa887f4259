"""GPU tests of predict_top_k / predict_rank(k) with exclude=: the filter kernel, the exact 3-pass kernel, the
device-side fallback over gathered rows, tastes, item shards, user blocks and the dense+rank path, against the masked
oracle (tests/masked_topk.py).  Integer fixtures match exactly; float fixtures use the tolerances of test_api_gpu.py."""
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


def make_model(T, U, I, d, integer, n_tastes=1, prediction=None, seed=0):
    uf = H.tag_features(U, 200, 20, seed=seed + 1, integer=integer)
    itf = H.tag_features(I, 200, 20, seed=seed + 2, integer=integer)
    wus = [H.linear_weights(200, d, seed=seed + 10 + t, integer=integer) for t in range(n_tastes)]
    wi = H.linear_weights(200, d, seed=seed + 4, integer=integer)
    bu, bi = H.feature_biases(200, seed=seed + 5, integer=integer), H.feature_biases(200, seed=seed + 6, integer=integer)
    kw = {} if prediction is None else {'prediction_graph': prediction}
    model = T.TensorRec(n_components=d, n_tastes=n_tastes, **kw)
    weights = {'linear_weights_item': wi, 'feature_biases_user': bu[:, None], 'feature_biases_item': bi[:, None]}
    for t in range(n_tastes):
        weights['linear_weights_user_%d' % t] = wus[t]
    model.set_weights(weights)
    om = oracle.OracleModel(wus, wi, bu, bi, prediction='dot' if prediction is None else 'euclidean')
    return model, uf, itf, om.predict(uf, itf)


def exclusion(scores, k, seed):
    """Rows cycle through: empty; the row's own unmasked top-k (theta has to go deeper); heavy (> half of the
    catalogue); everything; fewer than k eligible items; a random light history with duplicates and explicit zeros."""
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
            c = rng.integers(0, I, 40)                                   # duplicates
        else:
            continue
        rows.append(np.full(len(c), u))
        cols.append(c)
        vals.append(np.ones(len(c)))
    rows.append([0, 5])                                                  # explicit zeros: exclude nothing
    cols.append([1, 2])
    vals.append([0.0, 0.0])
    return sp.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(U, I))


def check(top, scores, exclude, k, integer, tol=1e-5 * 40 + 2e-6):
    exp_i, exp_s = masked_top_k(scores, exclude, k)
    mask = sp.csr_matrix(exclude)
    mask.sum_duplicates()
    dense = mask.toarray() != 0
    got_i = np.asarray(top.items)
    real = got_i != SENTINEL_ID
    rows = np.nonzero(real)[0]
    assert not dense[rows, got_i[real]].any()                           # an excluded item is never reported
    assert np.array_equal(got_i == SENTINEL_ID, exp_i == SENTINEL_ID)    # sentinel slots where too few are eligible
    if integer:
        assert np.array_equal(got_i, exp_i) and np.array_equal(top.scores, exp_s)
    else:
        assert np.all(np.abs(np.where(real, top.scores - scores[np.arange(len(got_i))[:, None],
                                                                   np.where(real, got_i, 0)], 0)) <= tol)
        assert (got_i != exp_i).mean() < 0.01


@pytest.mark.parametrize('d', [64, 128])
@pytest.mark.parametrize('k', [1, 10, 12])
@pytest.mark.parametrize('cluster', ['1', '2'])
@pytest.mark.parametrize('path', ['auto', 'exact'])
def test_exclusion_matches_the_masked_oracle(T, monkeypatch, d, k, cluster, path):
    integer = k != 12
    monkeypatch.setenv('TRK_FILTER_CLUSTER', cluster)
    monkeypatch.setattr(T.tensorrec, 'TOPK_PATH', path)
    model, uf, itf, scores = make_model(T, 300, 1000 + 37, d, integer)   # n_items not a multiple of 128
    exclude = exclusion(scores, k, seed=d + k)
    top = model.predict_top_k(uf, itf, k, exclude=exclude)
    assert model.last_topk_info['path'] == ('filter' if path == 'auto' else 'exact3')
    check(top, scores, exclude, k, integer)
    again = model.predict_rank(uf, itf, k=k, exclude=exclude)         # repeated calls are bit-identical
    assert np.array_equal(top.items, again.items) and np.array_equal(top.scores, again.scores)


def test_empty_exclude_is_bit_identical_to_none(T):
    model, uf, itf, scores = make_model(T, 517, 3001, 128, integer=False)
    plain = model.predict_top_k(uf, itf, 10)
    for empty in (sp.csr_matrix((517, 3001)), sp.coo_matrix(([0.0], ([3], [7])), shape=(517, 3001))):
        top = model.predict_top_k(uf, itf, 10, exclude=empty)
        assert np.array_equal(top.items, plain.items) and np.array_equal(top.scores, plain.scores)


def test_tie_heavy_rows_take_the_device_fallback_with_the_row_map(T):
    """All-equal item vectors: every row overflows the filter's buffer and goes through the exact kernel over gathered
    rows, which reads its lists through excl_row_map."""
    U, I, d, k = 700, 2000, 64, 10
    uf = H.tag_features(U, 200, 20, seed=1, integer=True)
    itf = sp.csr_matrix(np.ones((I, 1), np.float32))
    wu = H.linear_weights(200, d, seed=3, integer=True)
    wi = np.ones((1, d), np.float32)
    model = T.TensorRec(n_components=d, biased=False)
    model.set_weights({'linear_weights_user_0': wu, 'linear_weights_item': wi})
    scores = oracle.OracleModel([wu], wi).predict(uf, itf)
    exclude = exclusion(scores, k, seed=5)
    top = model.predict_top_k(uf, itf, k, exclude=exclude)
    assert model.last_topk_info['path'] == 'filter' and model.last_topk_info['fallback_rows'] > 0
    check(top, scores, exclude, k, integer=True)


@pytest.mark.parametrize('integer', [True, False])
def test_tastes_shards_and_user_blocks(T, integer):
    import torch
    from tensorrec_b200 import kernels
    from tensorrec_b200.distributed import shard_bounds
    U, I, d, k, world = 300, 4000, 64, 10, 3
    model, uf, itf, scores = make_model(T, U, I, d, integer, n_tastes=3)
    exclude = exclusion(scores, k, seed=11)
    whole = model.predict_top_k(uf, itf, k, exclude=exclude)
    assert model.last_topk_info['path'] == 'filter'
    check(whole, scores, exclude, k, integer)
    assert all(len(set(r[r != SENTINEL_ID])) == (r != SENTINEL_ID).sum() for r in whole.items)   # no item twice
    blocks = model.predict_top_k(uf, itf, k, exclude=exclude, user_batch_size=128)
    assert np.array_equal(blocks.items, whole.items) and np.array_equal(blocks.scores, whole.scores)
    per_shard = []
    for r in range(world):
        lo, hi = shard_bounds(I, world, r)
        ex = exclude if lo > 0 else sp.csr_matrix(exclude)[:, :hi]     # (offset 0 without a group: exactly n_items)
        top = model.predict_top_k(uf, sp.csr_matrix(itf)[lo:hi], k, item_id_offset=lo, to_host=False, exclude=ex)
        per_shard.append(torch.cat([top.scores.view(torch.int32), top.items], dim=1))
    merged = kernels.topk_merge_received(torch.stack(per_shard).contiguous(), U, world, k)
    assert np.array_equal(merged.items.cpu().numpy(), whole.items)
    assert np.array_equal(merged.scores.cpu().numpy(), whole.scores)


def test_dense_rank_path_and_recall(T):
    from tensorrec_b200.eval import recall_at_k
    U, I, k = 200, 700, 10
    model, uf, itf, scores = make_model(T, U, I, 16, integer=True,
                                        prediction=T.prediction_graphs.EuclideanSimilarityPredictionGraph())
    exclude = exclusion(scores, k, seed=2)
    top = model.predict_top_k(uf, itf, k, exclude=exclude)
    assert model.last_topk_info['path'] == 'dense+rank'
    check(top, scores, exclude, k, integer=True)
    # held-out protocol: the excluded (training) items never count as hits, even when they are also test items
    test = sp.csr_matrix(exclude).astype(np.float32)
    test.data[:] = 1.0
    assert np.all(recall_at_k(top, test, k=k) == 0.0)
