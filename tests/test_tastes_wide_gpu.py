"""GPU tests of the wide route for mixtures of tastes (32 < k <= 1024): trk_topk_merge_dedup_pair against the numpy model
of tests/test_tastes_wide_cpu.py, and predict_top_k of 2-5 tastes against the masked oracle of the max-collapsed
scores.  The route is reached at small shapes by lowering tensorrec.WIDE_MIN_ITEMS.  Integer fixtures match bit for
bit; float fixtures use the tolerances of test_exclude_gpu.py."""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from tests import helpers as H
from tests.masked_topk import SENTINEL_ID
from tests.test_exclude_gpu import check, exclusion, make_model
from tests.test_tastes_wide_cpu import merge_pair

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


# ---- the merge kernel -----------------------------------------------------------------------------------------------
def sorted_list(ids, scores, k):
    order = np.lexsort((ids, -scores.astype(np.float64)))
    items = np.full(k, SENTINEL_ID, np.int32)
    vals = np.full(k, -np.inf, np.float32)
    items[:len(ids)], vals[:len(ids)] = ids[order], scores[order]
    return items, vals


def list_pair(rng, n_rows, k, overlap):
    """Rows of two sorted lists.  Row kinds cycle: both full; a sentinel tail in A, in B, in both; A all sentinels;
    B all sentinels; both all sentinels.  `overlap` of B's real ids are A's, half of those at A's score (a duplicate
    with equal scores), the others one higher or lower.  Scores are small integers: many equal scores on different
    items."""
    lists = []
    for r in range(n_rows):
        kind = r % 7
        n_a = {1: k // 3, 3: k // 2, 4: 0, 6: 0}.get(kind, k)
        n_b = {2: k // 4, 3: k - 1, 5: 0, 6: 0}.get(kind, k)
        pool = rng.permutation(20 * k)[:n_a + n_b].astype(np.int32)
        a_ids = pool[:n_a]
        a_s = rng.integers(-20, 20, n_a).astype(np.float32)
        n_dup = min(n_a, int(round(overlap * n_b)))
        pick = rng.choice(n_a, n_dup, replace=False) if n_dup else np.zeros(0, np.int64)
        b_ids = np.concatenate([a_ids[pick], pool[n_a:n_a + n_b - n_dup]])
        b_s = rng.integers(-20, 20, n_b).astype(np.float32)
        shift = rng.choice(np.array([-1, 1], np.float32), n_dup)
        shift[::2] = 0
        b_s[:n_dup] = a_s[pick] + shift
        lists.append((sorted_list(a_ids, a_s, k), sorted_list(b_ids, b_s, k)))
    a_i = np.stack([x[0][0] for x in lists])
    a_s = np.stack([x[0][1] for x in lists])
    b_i = np.stack([x[1][0] for x in lists])
    b_s = np.stack([x[1][1] for x in lists])
    return a_i, a_s, b_i, b_s


def packed(kernels, items, scores):
    import torch
    top = kernels.PackedTopK(items.shape[0], items.shape[1], 'cuda')
    top.scores.copy_(torch.from_numpy(scores))
    top.items.copy_(torch.from_numpy(items))
    return top


@pytest.mark.parametrize('k', [33, 100, 512, 1024])
@pytest.mark.parametrize('overlap', [0.0, 0.3, 1.0])
def test_merge_kernel_is_bit_identical_to_the_model(T, k, overlap):
    from tensorrec_b200 import kernels
    rng = np.random.default_rng(k + int(10 * overlap))
    n_rows = 7 * 5 + 2                                  # every row kind, not a multiple of anything
    a_i, a_s, b_i, b_s = list_pair(rng, n_rows, k, overlap)
    exp_i, exp_s = merge_pair(a_i, a_s, b_i, b_s, k)
    out = kernels.topk_merge_dedup(packed(kernels, a_i, a_s), packed(kernels, b_i, b_s))
    assert np.array_equal(out.items.cpu().numpy(), exp_i)
    assert np.array_equal(out.scores.cpu().numpy(), exp_s)
    # the result is symmetric up to which copy of an equal-score duplicate survives, and copies are identical
    swapped = kernels.topk_merge_dedup(packed(kernels, b_i, b_s), packed(kernels, a_i, a_s))
    assert np.array_equal(swapped.buf.cpu().numpy(), out.buf.cpu().numpy())


def test_merge_kernel_reads_and_writes_through_the_row_strides(T):
    """A and B in wider buffers with strides of their own, the result inside a PackedTopK-like row."""
    import torch
    from tensorrec_b200 import _lib, kernels
    k, n_rows = 100, 41
    a_i, a_s, b_i, b_s = list_pair(np.random.default_rng(1), n_rows, k, 0.5)
    exp_i, exp_s = merge_pair(a_i, a_s, b_i, b_s, k)
    a = torch.zeros((n_rows, 3 * k), dtype=torch.int32, device='cuda')
    a[:, :k] = torch.from_numpy(a_s).view(torch.int32).cuda()
    a[:, 2 * k:] = torch.from_numpy(a_i).cuda()
    b = torch.zeros((n_rows, 2 * k + 7), dtype=torch.int32, device='cuda')
    b[:, :k] = torch.from_numpy(b_s).view(torch.int32).cuda()
    b[:, k:2 * k] = torch.from_numpy(b_i).cuda()
    out = torch.full((n_rows, 2 * k + 3), 12345, dtype=torch.int32, device='cuda')
    p = lambda t, col: t.data_ptr() + 4 * col                                    # noqa: E731
    lib = kernels.require_cuda()
    rc = lib.trk_topk_merge_dedup_pair(p(a, 0), p(a, 2 * k), 3 * k, p(b, 0), p(b, k), 2 * k + 7, n_rows, k,
                                       p(out, 0), p(out, k), 2 * k + 3, kernels._stream())
    _lib.check(rc, 'trk_topk_merge_dedup_pair')
    got = out.cpu().numpy()
    assert np.array_equal(got[:, :k].view(np.float32), exp_s) and np.array_equal(got[:, k:2 * k], exp_i)
    assert np.all(got[:, 2 * k:] == 12345)                                        # nothing beyond the row


def test_merge_kernel_rejects_bad_arguments(T):
    from tensorrec_b200 import kernels
    with pytest.raises(ValueError, match='k=1025'):
        kernels.topk_merge_dedup(kernels.empty_topk(3, 1025, 'cuda'), kernels.empty_topk(3, 1025, 'cuda'))
    with pytest.raises(ValueError):
        kernels.topk_merge_dedup(kernels.empty_topk(3, 100, 'cuda'), kernels.empty_topk(3, 99, 'cuda'))
    empty = kernels.topk_merge_dedup(kernels.empty_topk(0, 100, 'cuda'), kernels.empty_topk(0, 100, 'cuda'))
    assert empty.n_users == 0


# ---- predict_top_k --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n_tastes', [2, 3, 5])
@pytest.mark.parametrize('d', [64, 128])
@pytest.mark.parametrize('k', [33, 100, 1024])
def test_integer_fixture_is_bit_identical_to_the_masked_oracle(wide, n_tastes, d, k):
    model, uf, itf, scores = make_model(wide, 200, 3000 + 37, d, integer=True, n_tastes=n_tastes, seed=k + n_tastes)
    exclude = exclusion(scores, k, seed=d + k)        # includes rows with fewer than k eligible items
    top = model.predict_top_k(uf, itf, k, exclude=exclude)
    assert model.last_topk_info['path'] == 'wide'
    check(top, scores, exclude, k, integer=True)
    plain = model.predict_rank(uf, itf, k=k)
    assert model.last_topk_info['path'] == 'wide'
    exp_i, exp_s = oracle.top_k_from_scores(scores, k)
    assert np.array_equal(plain.items, exp_i) and np.array_equal(plain.scores, exp_s)


def test_tie_heavy_tastes_go_through_the_fallback(wide):
    """Every item has the same features: all scores of a row tie in every taste, no row can be certified, every row is
    scored dense and ranked per taste, and the fold still returns the reference order (ties by id)."""
    T = wide
    U, I, k, n_tastes = 150, 2500, 100, 3
    uf = H.tag_features(U, 200, 20, seed=1, integer=True)
    one = H.tag_features(1, 200, 20, seed=2, integer=True)
    itf = sp.vstack([one] * I).tocsr()
    wus = [H.linear_weights(200, 64, seed=3 + t, integer=True) for t in range(n_tastes)]
    wi = H.linear_weights(200, 64, seed=9, integer=True)
    model = T.TensorRec(n_components=64, n_tastes=n_tastes, biased=False)
    model.set_weights(dict({'linear_weights_item': wi},
                           **{'linear_weights_user_%d' % t: w for t, w in enumerate(wus)}))
    scores = oracle.OracleModel(wus, wi).predict(uf, itf)
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
    model, uf, itf, _ = make_model(wide, 400, 5000, 128, integer=False, n_tastes=3, seed=7, prediction=graph)
    scores = model.predict(uf, itf)
    exclude = exclusion(scores, k, seed=8)
    top = model.predict_top_k(uf, itf, k, exclude=exclude)
    assert model.last_topk_info['path'] == 'wide'
    check(top, scores, exclude, k, integer=False)
    assert model.last_topk_info['fallback_rows'] < scores.shape[0] // 10      # summed over the three tastes
    model.predict_top_k(uf, itf, k)
    assert model.last_topk_info['fallback_rows'] < scores.shape[0] // 10


def test_user_blocks_equal_one_block(wide):
    model, uf, itf, scores = make_model(wide, 700, 4000, 128, integer=False, n_tastes=3, seed=9)
    exclude = exclusion(scores, 200, seed=10)
    whole = model.predict_top_k(uf, itf, 200, exclude=exclude)
    for size in (128, 300):
        assert_same(model.predict_top_k(uf, itf, 200, exclude=exclude, user_batch_size=size), whole)


def test_shards_merged_equal_the_whole(wide):
    import torch
    from tensorrec_b200 import kernels
    k = 150
    model, uf, itf, scores = make_model(wide, 333, 4100, 128, integer=True, n_tastes=3, seed=11)
    exclude = exclusion(scores, k, seed=12)
    whole = model.predict_top_k(uf, itf, k, exclude=exclude)
    bounds = [0, 1000, 4100]
    parts = []
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        ex = exclude if lo > 0 else sp.csr_matrix(exclude)[:, :hi]
        top = model.predict_top_k(uf, itf.tocsr()[lo:hi], k, item_id_offset=lo, to_host=False, exclude=ex)
        assert model.last_topk_info['path'] == 'wide'
        parts.append(torch.cat([top.scores.view(torch.int32), top.items], dim=1))
    merged = kernels.topk_merge_received(torch.stack(parts).contiguous(), uf.shape[0], len(parts), k)
    assert np.array_equal(merged.items.cpu().numpy(), whole.items)
    assert np.array_equal(merged.scores.cpu().numpy(), whole.scores)


def test_smaller_k_is_a_prefix_of_a_larger_one(wide):
    model, uf, itf, _ = make_model(wide, 300, 3000, 128, integer=True, n_tastes=3, seed=13)
    big = model.predict_top_k(uf, itf, 400)
    for k in (33, 100):
        small = model.predict_top_k(uf, itf, k)
        assert np.array_equal(small.items, big.items[:, :k]) and np.array_equal(small.scores, big.scores[:, :k])


def test_integer_results_equal_dense_rank(T, monkeypatch):
    model, uf, itf, scores = make_model(T, 300, 3000, 64, integer=True, n_tastes=3, seed=14)
    exclude = exclusion(scores, 100, seed=15)
    monkeypatch.setattr(T.tensorrec, 'WIDE_MIN_ITEMS', 0)
    fused = model.predict_top_k(uf, itf, 100, exclude=exclude)
    assert model.last_topk_info['path'] == 'wide'
    monkeypatch.setattr(T.tensorrec, 'WIDE_MIN_ITEMS', 10 ** 9)
    dense = model.predict_top_k(uf, itf, 100, exclude=exclude)
    assert model.last_topk_info['path'] == 'dense+rank'
    assert_same(fused, dense)


@pytest.mark.parametrize('n_tastes', [1, 4])
def test_merge_runs_once_per_extra_taste(wide, monkeypatch, n_tastes):
    from tensorrec_b200 import kernels
    calls = []
    real = kernels.topk_merge_dedup
    monkeypatch.setattr(kernels, 'topk_merge_dedup', lambda *a, **kw: calls.append(1) or real(*a, **kw))
    model, uf, itf, scores = make_model(wide, 300, 3000, 64, integer=True, n_tastes=n_tastes, seed=16)
    top = model.predict_top_k(uf, itf, 64, user_batch_size=128)          # three user blocks
    assert model.last_topk_info['path'] == 'wide'
    assert len(calls) == 3 * (n_tastes - 1)
    exp_i, exp_s = oracle.top_k_from_scores(scores, 64)
    assert np.array_equal(top.items, exp_i) and np.array_equal(top.scores, exp_s)
