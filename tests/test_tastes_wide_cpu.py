"""CPU tests of the wide route for mixtures of tastes (32 < k <= 1024): topk_route with merge_max_k, the block size of
the pairwise fold, and a numpy model of the fold R_t = R_{t-1} (+) L_t of the per-taste top-k lists (DESIGN §3.6),
which must equal the top-k of the maximum over the tastes.  merge_pair is also the model the GPU tests hold
trk_topk_merge_dedup_pair to (tests/test_tastes_wide_gpu.py)."""
import numpy as np
import pytest
import scipy.sparse as sp

import tensorrec_b200 as T
from tensorrec_b200 import kernels, tensorrec
from tests.masked_topk import SENTINEL_ID, masked_top_k

R, P = T.representation_graphs, T.prediction_graphs


def merge_pair(a_i, a_s, b_i, b_s, k):
    """Row-wise top-k of the union of two sorted lists, every real id once at its higher score (an id with equal scores
    keeps one copy), ordered by (score desc, id asc), padded with (SENTINEL_ID, -inf)."""
    n = a_i.shape[0]
    items = np.full((n, k), SENTINEL_ID, dtype=np.int32)
    scores = np.full((n, k), -np.inf, dtype=np.float32)
    for r in range(n):
        best = {}
        for ids, vals in ((a_i[r], a_s[r]), (b_i[r], b_s[r])):
            for i, s in zip(ids.tolist(), vals.tolist()):
                if i != SENTINEL_ID and (i not in best or s > best[i]):
                    best[i] = s
        order = sorted(best.items(), key=lambda e: (-e[1], e[0]))[:k]
        items[r, :len(order)] = [i for i, _ in order]
        scores[r, :len(order)] = [s for _, s in order]
    return items, scores


def fold(per_taste, exclude, k):
    """The pairwise fold of the per-taste masked top-k lists of the score matrices per_taste."""
    run_i, run_s = masked_top_k(per_taste[0], exclude, k)
    for scores in per_taste[1:]:
        ti, ts = masked_top_k(scores, exclude, k)
        run_i, run_s = merge_pair(run_i, run_s, ti, ts, k)
    return run_i, run_s


def route(k, n_items, sharded=False, single_taste=False, **kw):
    return tensorrec.topk_route(k, n_items, True, single_taste, 16, 32, sharded=sharded, **kw)


# ---- the route ------------------------------------------------------------------------------------------------------
def test_tastes_take_the_wide_route_with_the_keyword(monkeypatch):
    monkeypatch.setattr(tensorrec, 'WIDE_MIN_ITEMS', 5000)
    for k in (33, 100, 1024):
        assert route(k, 5000, merge_max_k=1024) == 'wide'
        assert route(k, 10 ** 6, merge_max_k=1024) == 'wide'
        assert route(k, 4999, merge_max_k=1024) == 'dense+rank'
    assert route(1025, 10 ** 6, merge_max_k=1024) == 'dense+rank'
    assert route(100, 0, merge_max_k=1024) == 'dense+rank'
    assert route(100, 10 ** 6, merge_max_k=64) == 'dense+rank'      # beyond what the caller can merge
    assert route(10, 10 ** 6, merge_max_k=1024) == 'filter'         # k <= 32 keeps its routes
    assert route(20, 10 ** 6, merge_max_k=1024) == 'exact3'
    monkeypatch.setattr(tensorrec, 'TOPK_PATH', 'exact')
    assert route(100, 10 ** 6, merge_max_k=1024) == 'dense+rank'


def test_sharded_tastes_take_the_wide_route_at_any_shard_size(monkeypatch):
    monkeypatch.setattr(tensorrec, 'WIDE_MIN_ITEMS', 5000)
    assert {route(100, n, sharded=True, merge_max_k=1024) for n in (0, 1, 4999, 5000, 10 ** 6)} == {'wide'}
    assert route(1025, 10 ** 6, sharded=True, merge_max_k=1024) == 'dense+rank'


def test_euclidean_and_attention_ignore_the_keyword():
    for kw in ({'euclidean': True}, {'attention': True}):
        for k, n in ((10, 10 ** 6), (100, 10 ** 6), (10, 10), (1024, 10 ** 6)):
            assert route(k, n, merge_max_k=1024, **kw) == route(k, n, **kw)
            assert route(k, n, sharded=True, merge_max_k=1024, **kw) == route(k, n, sharded=True, **kw)


def test_the_model_passes_the_wide_limit(monkeypatch):
    seen = {}
    real = tensorrec.topk_route
    monkeypatch.setattr(tensorrec, 'topk_route', lambda *a, **kw: seen.update(kw) or real(*a, **kw))
    monkeypatch.setattr(kernels, 'filter_max_k', lambda: 16)
    monkeypatch.setattr(kernels, 'topk_max_k', lambda d_pad: 32)
    model = T.TensorRec(n_components=64, n_tastes=3)
    assert model._topk_path(100, 10 ** 6, True, False) == 'wide'
    assert seen['merge_max_k'] == tensorrec.WIDE_MAX_K


# ---- block size -----------------------------------------------------------------------------------------------------
def test_wide_blocks_of_a_mixture_hold_the_fold(monkeypatch):
    monkeypatch.setattr(kernels, 'wide_list_capacity', lambda k: 2 * int(-(-(k + max(k // 2, 32)) // 32) * 32))
    one = T.TensorRec(n_components=64)
    three = T.TensorRec(n_components=64, n_tastes=3)
    for k in (33, 100, 1000, 1024):
        cap = kernels.wide_list_capacity(k)
        single = one._topk_block_rows('wide', 10 ** 7, 10 ** 6, k)
        assert single == max(2 * kernels.TILE_USERS, one.PREDICT_BLOCK_BYTES // (8 * cap) // 256 * 256)
        rows = three._topk_block_rows('wide', 10 ** 7, 10 ** 6, k, n_tastes=3)
        assert three._topk_block_rows('wide', 10 ** 7, 10 ** 6, k) == single      # similar items: one list per row
        assert rows * (8 * cap + 3 * 8 * k) <= three.PREDICT_BLOCK_BYTES
        assert rows < single and rows % 256 == 0


# ---- the fold -------------------------------------------------------------------------------------------------------
def tastes_fixture(rng, n_tastes, U, I, lo=-6, hi=7):
    """Integer scores: equal scores on different items everywhere, and the same item with the same score in two tastes
    (every taste copies a block of another's scores)."""
    per_taste = [rng.integers(lo, hi, size=(U, I)).astype(np.float32) for _ in range(n_tastes)]
    for t in range(1, n_tastes):
        cols = rng.choice(I, I // 3, replace=False)
        per_taste[t][:, cols] = per_taste[t - 1][:, cols]
    return per_taste


def heavy_exclusion(rng, U, I, k):
    """Rows cycle through: nothing excluded; fewer than k eligible items; every item; a random half."""
    rows, cols = [], []
    for u in range(U):
        kind = u % 4
        if kind == 1:
            c = rng.choice(I, I - k // 2, replace=False)
        elif kind == 2:
            c = np.arange(I)
        elif kind == 3:
            c = rng.choice(I, I // 2, replace=False)
        else:
            continue
        rows.append(np.full(len(c), u))
        cols.append(c)
    return sp.csr_matrix((np.ones(sum(map(len, cols))), (np.concatenate(rows), np.concatenate(cols))), shape=(U, I))


@pytest.mark.parametrize('n_tastes', [2, 3, 5])
@pytest.mark.parametrize('k', [33, 100])
@pytest.mark.parametrize('excluded', [False, True])
def test_fold_equals_the_topk_of_the_max(n_tastes, k, excluded):
    rng = np.random.default_rng(n_tastes * 100 + k + excluded)
    U, I = 24, 300
    per_taste = tastes_fixture(rng, n_tastes, U, I)
    exclude = heavy_exclusion(rng, U, I, k) if excluded else sp.csr_matrix((U, I))
    got_i, got_s = fold(per_taste, exclude, k)
    exp_i, exp_s = masked_top_k(np.max(per_taste, axis=0), exclude, k)
    assert np.array_equal(got_i, exp_i) and np.array_equal(got_s, exp_s)
    if excluded:
        assert (got_i[1::4] == SENTINEL_ID).any() and (got_i[2::4] == SENTINEL_ID).all()


def test_merge_pair_keeps_one_copy_at_the_higher_score():
    a_i = np.array([[5, 3, 9, SENTINEL_ID]], np.int32)
    a_s = np.array([[4, 2, 2, -np.inf]], np.float32)
    b_i = np.array([[3, 5, 7, SENTINEL_ID]], np.int32)
    b_s = np.array([[6, 4, 2, -np.inf]], np.float32)
    items, scores = merge_pair(a_i, a_s, b_i, b_s, 4)
    assert items.tolist() == [[3, 5, 7, 9]] and scores.tolist() == [[6, 4, 2, 2]]
    items, scores = merge_pair(a_i, a_s, b_i, b_s, 6)
    assert items[0, 4:].tolist() == [SENTINEL_ID] * 2 and np.all(scores[0, 4:] == -np.inf)
