"""CPU tests of predict_rank_at: its route, its user blocks, its argument checks (no device touched), a numpy model of
the exact kernel's counting mode (capture, per-row sort, passes of 32 targets, buckets) against the closed forms, the
sort order of the host layer, eval on sparse ranks, and both sides of every check of the trk_score_count* entry
points."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import oracle
from tensorrec_b200 import eval as tr_eval
from tensorrec_b200 import kernels, tensorrec
from tensorrec_b200.errors import ModelNotFitException

F32 = np.float32
NEG_INF = F32(-np.inf)


# ---- route and blocks ----------------------------------------------------------------------------------------------
def test_rank_at_route():
    m = tensorrec.RANK_AT_MIN_ITEMS
    assert tensorrec.rank_at_route(m, True) == 'exact3_count'
    assert tensorrec.rank_at_route(10 * m, True) == 'exact3_count'
    assert tensorrec.rank_at_route(m - 1, True) == 'dense+rank'
    assert tensorrec.rank_at_route(10 * m, False) == 'dense+rank'
    assert tensorrec.rank_at_route(0, False) == 'dense+rank'


@pytest.mark.parametrize('unit', [128, 6, 64])
def test_rank_at_blocks_start_at_kernel_blocks_and_bound_pairs(unit):
    rng = np.random.default_rng(unit)
    per_row = rng.integers(0, 40, 1000)
    per_row[300] = 5000                                  # one unit alone beyond max_pairs
    indptr = np.concatenate([[0], np.cumsum(per_row)])
    for max_rows, max_pairs in ((unit, 10 ** 9), (4 * unit, 10 ** 9), (10 ** 6 // unit * unit, 3000),
                                (8 * unit, 500)):
        blocks = tensorrec.rank_at_blocks(indptr, unit, max_rows, max_pairs)
        assert blocks[0][0] == 0 and blocks[-1][1] == 1000
        for (a0, a1), (b0, _) in zip(blocks, blocks[1:]):
            assert a1 == b0
        for u0, u1 in blocks:
            assert u0 % unit == 0 and u1 > u0 and u1 - u0 <= max_rows
            if u1 - u0 > unit:
                assert indptr[u1] - indptr[u0] <= max_pairs


# ---- argument checks: before any device work -----------------------------------------------------------------------
def _fitted_model(monkeypatch):
    model = tensorrec.TensorRec(n_components=8)
    model.set_weights({'linear_weights_user_0': np.ones((5, 8), F32), 'linear_weights_item': np.ones((7, 8), F32),
                       'feature_biases_user': np.zeros((5, 1), F32), 'feature_biases_item': np.zeros((7, 1), F32)})

    def no_device(*_):
        raise AssertionError('device work before the arguments were checked')
    monkeypatch.setattr(tensorrec.TensorRec, '_cuda_device', staticmethod(no_device))
    return model


def test_predict_rank_at_before_fit():
    with pytest.raises(ModelNotFitException):
        tensorrec.TensorRec(n_components=8).predict_rank_at(sp.eye(3, 5, format='csr'), sp.eye(4, 7, format='csr'),
                                                            sp.eye(3, 4, format='csr'))


@pytest.mark.parametrize('pairs,exclude,match', [
    (np.ones((3, 4)), None, 'scipy sparse'),
    (sp.eye(3, 5, format='csr'), None, 'shape'),
    (sp.eye(4, 4, format='csr'), None, 'shape'),
    (sp.eye(3, 4, format='csr'), np.ones((3, 4)), 'scipy sparse'),
    (sp.eye(3, 4, format='csr'), sp.eye(2, 4, format='csr'), 'rows'),
    (sp.eye(3, 4, format='csr'), sp.eye(3, 5, format='csr'), 'columns'),
])
def test_predict_rank_at_rejects_bad_arguments_without_device_work(monkeypatch, pairs, exclude, match):
    model = _fitted_model(monkeypatch)
    with pytest.raises(ValueError, match=match):
        model.predict_rank_at(sp.eye(3, 5, format='csr', dtype=F32), sp.eye(4, 7, format='csr', dtype=F32), pairs,
                              exclude=exclude)


def test_predict_rank_at_without_listed_pairs_needs_no_device(monkeypatch):
    model = _fitted_model(monkeypatch)
    pairs = sp.csr_matrix((np.zeros(2, F32), ([0, 2], [1, 3])), shape=(3, 4))    # explicit zeros list nothing
    r = model.predict_rank_at(sp.eye(3, 5, format='csr', dtype=F32), sp.eye(4, 7, format='csr', dtype=F32), pairs)
    assert isinstance(r, sp.csr_matrix) and r.shape == (3, 4) and r.nnz == 0 and r.dtype == np.int32


# ---- numpy model of the counting mode -----------------------------------------------------------------------------
def outranks(s, i, t, ti):
    return s > t or (s == t and i < ti)


def model_counting_mode(scores, indptr, ids, excluded=None, n_splits=1):
    """The counting mode of score_tc_kernel over one call, restated: rows of 128-item tiles, one (row, column half)
    thread over chunks of 32 columns.  Returns (ranks in the order of ids, chunks skipped)."""
    n_rows, n_items = scores.shape
    n_tiles = -(-n_items // 128)
    final = np.full((n_rows, n_tiles * 128), NEG_INF, F32)         # padding columns score -inf
    final[:, :n_items] = scores
    masked = final.copy()
    if excluded is not None:
        masked[:, :n_items][excluded] = NEG_INF
    # capture: every listed pair's unmasked score, chunk by chunk in each thread's order
    pair_score = np.full(ids.shape[0], np.nan, F32)
    for r in range(n_rows):
        row_ids = ids[indptr[r]:indptr[r + 1]]
        for half in range(2):
            for t in range(n_tiles):
                for c in range(2):
                    base = t * 128 + (half * 2 + c) * 32
                    for k in np.nonzero((row_ids >= base) & (row_ids < base + 32))[0]:
                        pair_score[indptr[r] + k] = final[r, row_ids[k]]
    assert not np.isnan(pair_score).any()
    # sort every row's pairs by (score desc, id asc), -0.0 with +0.0
    rows = np.repeat(np.arange(n_rows), np.diff(indptr))
    order = np.lexsort((ids, -(pair_score + F32(0.0)), rows))
    s_score, s_ids = pair_score[order], ids[order]
    counts = np.zeros(ids.shape[0], np.int64)
    tiles_per_split = -(-n_tiles // n_splits)
    passes = -(-int(np.diff(indptr).max(initial=0)) // 32)
    skipped = 0
    for p in range(passes):
        for sp_ in range(n_splits):
            t0, t1 = sp_ * tiles_per_split, min(n_tiles, (sp_ + 1) * tiles_per_split)
            for r in range(n_rows):
                lo = indptr[r] + 32 * p
                n = max(0, min(32, indptr[r + 1] - lo))
                ts = np.full(32, NEG_INF, F32)
                ti = np.full(32, 2 ** 31 - 1, np.int64)
                ts[:n], ti[:n] = s_score[lo:lo + n], s_ids[lo:lo + n]
                low = (ts[n - 1], ti[n - 1]) if n else (F32(np.inf), 0)
                for half in range(2):
                    h = np.zeros(32, np.int64)
                    for t in range(t0, t1):
                        for c in range(2):
                            base = t * 128 + (half * 2 + c) * 32
                            chunk = masked[r, base:base + 32]
                            if not chunk.max() >= low[0]:
                                skipped += 1
                                continue
                            for j in range(32):
                                s, i = chunk[j], base + j
                                if not outranks(s, i, *low):
                                    continue
                                lb = 0
                                for step in (16, 8, 4, 2, 1):
                                    if not outranks(s, i, ts[lb + step - 1], ti[lb + step - 1]):
                                        lb += step
                                h[lb] += 1
                    counts[lo:lo + n] += np.cumsum(h)[:n]
    ranks = np.empty(ids.shape[0], np.int64)
    ranks[order] = 1 + counts
    return ranks, skipped


def masked_closed_form(scores, excluded, r, i):
    s = scores[r]
    ok = ~excluded[r]
    ok[i] = False
    j = np.arange(s.shape[0])
    return 1 + int(np.sum(ok & ((s > s[i]) | ((s == s[i]) & (j < i)))))


def tie_heavy_fixture(seed, n_rows=12, n_items=300):
    rng = np.random.default_rng(seed)
    scores = rng.integers(-3, 4, size=(n_rows, n_items)).astype(F32)
    zeros = scores == 0
    scores[zeros & (rng.random(scores.shape) < 0.5)] = F32(-0.0)
    per_row = [0, 1, 32, 33, 120, 64, 65, 2, 31, 5, 0, 200][:n_rows]
    ids = [np.sort(rng.choice(n_items, size=k, replace=False)) for k in per_row]
    indptr = np.concatenate([[0], np.cumsum(per_row)]).astype(np.int64)
    ids = np.concatenate(ids).astype(np.int64)
    excluded = rng.random((n_rows, n_items)) < 0.2
    return scores, indptr, ids, excluded


@pytest.mark.parametrize('n_splits', [1, 2])
def test_counting_model_equals_closed_form_rank(n_splits):
    scores, indptr, ids, _ = tie_heavy_fixture(1)
    ranks, _ = model_counting_mode(scores, indptr, ids, n_splits=n_splits)
    full = oracle.rank_predictions_closed_form(scores)
    rows = np.repeat(np.arange(scores.shape[0]), np.diff(indptr))
    assert np.array_equal(ranks, full[rows, ids])


def test_counting_model_with_exclusion_equals_masked_closed_form():
    scores, indptr, ids, excluded = tie_heavy_fixture(2)
    rows = np.repeat(np.arange(scores.shape[0]), np.diff(indptr))
    assert excluded[rows, ids].any() and (~excluded[rows, ids]).any()    # excluded and eligible listed pairs
    ranks, _ = model_counting_mode(scores, indptr, ids, excluded=excluded, n_splits=2)
    expect = [masked_closed_form(scores, excluded, r, i) for r, i in zip(rows, ids)]
    assert np.array_equal(ranks, expect)


def test_counting_model_skips_chunks_below_high_targets():
    rng = np.random.default_rng(3)
    scores = rng.standard_normal((4, 1000)).astype(F32)
    top = np.argsort(-scores, axis=1, kind='stable')[:, :3]
    ids = np.sort(top, axis=1).reshape(-1)
    indptr = np.arange(0, 13, 3)
    ranks, skipped = model_counting_mode(scores, indptr, ids)
    assert np.array_equal(ranks, oracle.rank_predictions_closed_form(scores)[np.repeat(np.arange(4), 3), ids])
    assert skipped > 0.9 * 4 * 2 * 2 * 8      # rows x halves x chunks per half-tile x tiles


def test_rank_sort_order_matches_the_model_order():
    rng = np.random.default_rng(4)
    score = rng.integers(-2, 3, 500).astype(F32)
    score[(score == 0) & (rng.random(500) < 0.5)] = F32(-0.0)
    score[:5] = [np.inf, -np.inf, 1e-30, -1e-30, 3.0e38]
    rows = np.sort(rng.integers(0, 20, 500))
    order = kernels.rank_sort_order(torch.from_numpy(score), torch.from_numpy(rows)).numpy()
    assert np.array_equal(order, np.lexsort((np.arange(500), -(score + F32(0.0)), rows)))


def test_pair_block_max_and_passes():
    indptr = np.array([0, 3, 3, 40, 41, 41], np.int32)
    assert kernels.pair_block_max(indptr, 5, 2).tolist() == [3, 37, 0]
    assert kernels.pair_block_max(indptr, 5, 128).tolist() == [37]
    assert [kernels.count_passes(n) for n in (0, 1, 32, 33, 64, 1000)] == [0, 1, 1, 2, 2, 32]


# ---- eval on sparse ranks -------------------------------------------------------------------------------------------
def test_eval_sparse_ranks_equal_full_ranks():
    rng = np.random.default_rng(5)
    n_users, n_items = 30, 200
    full = oracle.rank_predictions(rng.integers(-4, 5, (n_users, n_items)).astype(F32))
    test = sp.random(n_users, n_items, density=0.05, format='csr', random_state=7)
    test.data[:] = rng.integers(1, 4, test.nnz)
    test = sp.diags((np.arange(n_users) != 3).astype(float)) @ test      # user 3 has no positives
    test.eliminate_zeros()
    listed = sp.csr_matrix(test > 0)
    ranks = sp.csr_matrix((full[listed.nonzero()].astype(np.int32), listed.nonzero()), shape=full.shape)
    extra = sp.random(n_users, n_items, density=0.05, format='csr', random_state=8)      # ranks of other pairs too
    other = sp.csr_matrix((full[extra.nonzero()], extra.nonzero()), shape=full.shape)
    ranks = ranks + other - other.multiply(listed)
    for k in (1, 5, 17, 200):
        for preserve in (False, True):
            for metric in (tr_eval.precision_at_k, tr_eval.recall_at_k, tr_eval.ndcg_at_k):
                np.testing.assert_array_equal(metric(ranks, test, k=k, preserve_rows=preserve),
                                              metric(full, test, k=k, preserve_rows=preserve))
            assert tr_eval.f1_score_at_k(ranks, test, k=k) == tr_eval.f1_score_at_k(full, test, k=k)


def test_eval_rejects_a_positive_without_rank():
    test = sp.csr_matrix(np.array([[1, 0, 2], [0, 1, 0]], F32))
    ranks = sp.csr_matrix(np.array([[1, 0, 0], [0, 3, 0]], np.int32))
    with pytest.raises(ValueError, match='no stored rank'):
        tr_eval.recall_at_k(ranks, test, k=2)
    with pytest.raises(ValueError, match='shape'):
        tr_eval.recall_at_k(sp.csr_matrix((2, 4), dtype=np.int32), test, k=2)


# ---- both sides of every check of the counting entry points ---------------------------------------------------------
A = 1 << 20          # a 16-byte aligned fake device address
MISALIGNED = A + 4
COUNT = dict(user_split=A, user_scale=A, user_bias=None, item_split=A, item_meta=A, n_users=10, n_items=300, d_pad=64,
             n_splits=1, item_id_offset=0, pair_indptr=A, pair_ids=A, pair_score=A, pair_count=A, block_pairs=A,
             pass_=0, excl_indptr=None, excl_ids=None, excl_row_map=None)
COUNT_EUCLID = dict(COUNT, user_half_sqnorm=A, item_half_sqnorm=A)
COUNT_TASTES = dict(user_split=A, user_scale=A, user_bias=None, n_tastes=2, attention=0, item_split=A, item_meta=A,
                    n_users=10, n_items=300, d_pad=64, n_splits=1, item_id_offset=0, pair_indptr=A, pair_ids=A,
                    pair_score=A, pair_count=A, block_pairs=A, pass_=0, excl_indptr=None, excl_ids=None,
                    excl_row_map=None)
ENTRY = {'trk_score_count_f16x3': COUNT, 'trk_score_count_euclid_f16x3': COUNT_EUCLID,
         'trk_score_count_tastes_f16x3': COUNT_TASTES}
VALID = [
    ('trk_score_count_f16x3', {}),
    ('trk_score_count_f16x3', dict(pass_=-1, pair_count=None, d_pad=128, n_splits=4, user_bias=A)),
    ('trk_score_count_f16x3', dict(pass_=31, excl_indptr=A, excl_ids=A, excl_row_map=A)),
    ('trk_score_count_euclid_f16x3', {}),
    ('trk_score_count_euclid_f16x3', dict(pass_=-1, excl_indptr=A, excl_ids=A)),
    ('trk_score_count_tastes_f16x3', dict(n_tastes=32, attention=1)),
    ('trk_score_count_tastes_f16x3', dict(pass_=-1, pair_count=None, excl_indptr=A, excl_ids=A)),
]
FAULTS = [
    ('trk_score_count_f16x3', dict(pair_indptr=None), 'TRK_ERR_ARG', 'null pair list'),
    ('trk_score_count_f16x3', dict(pair_ids=None), 'TRK_ERR_ARG', 'null pair list'),
    ('trk_score_count_euclid_f16x3', dict(pair_score=None), 'TRK_ERR_ARG', 'null pair list'),
    ('trk_score_count_tastes_f16x3', dict(block_pairs=None), 'TRK_ERR_ARG', 'null pair list'),
    ('trk_score_count_f16x3', dict(pair_count=None), 'TRK_ERR_ARG', 'null pair_count'),
    ('trk_score_count_f16x3', dict(pass_=-2), 'TRK_ERR_ARG', 'pass=-2'),
    ('trk_score_count_f16x3', dict(n_splits=0), 'TRK_ERR_ARG', 'n_splits'),
    ('trk_score_count_f16x3', dict(d_pad=96), 'TRK_ERR_UNSUPPORTED', 'd_pad=96'),
    ('trk_score_count_f16x3', dict(user_split=None), 'TRK_ERR_ARG', 'null operand'),
    ('trk_score_count_f16x3', dict(item_meta=MISALIGNED), 'TRK_ERR_ARG', '16-byte aligned'),
    ('trk_score_count_f16x3', dict(n_users=0), 'TRK_ERR_ARG', 'empty shape'),
    ('trk_score_count_f16x3', dict(excl_ids=A), 'TRK_ERR_ARG', 'go together'),
    ('trk_score_count_euclid_f16x3', dict(item_half_sqnorm=None), 'TRK_ERR_ARG', 'trk_score_count_euclid_f16x3: null'),
    ('trk_score_count_euclid_f16x3', dict(item_half_sqnorm=MISALIGNED), 'TRK_ERR_ARG', 'item_half_sqnorm must be'),
    ('trk_score_count_tastes_f16x3', dict(n_tastes=0), 'TRK_ERR_ARG', 'n_tastes=0'),
    ('trk_score_count_tastes_f16x3', dict(n_tastes=1), 'TRK_ERR_ARG', 'n_tastes=1'),
    ('trk_score_count_tastes_f16x3', dict(n_tastes=33, attention=1), 'TRK_ERR_UNSUPPORTED', 'exceed'),
]


@pytest.fixture(scope='module')
def lib():
    if torch.cuda.is_available():
        pytest.skip('a CUDA device is present: the fake addresses must not reach a launch')
    from tensorrec_b200 import _lib
    return _lib.load()


def call(lib, entry, fault):
    args = dict(ENTRY[entry])
    assert set(fault) <= set(args), fault
    args.update(fault)
    return getattr(lib, entry)(*args.values(), None)   # (the stream)


@pytest.mark.parametrize('entry,fault', VALID, ids=['%s-%d' % (e, i) for i, (e, _) in enumerate(VALID)])
def test_valid_count_calls_pass_every_check(lib, entry, fault):
    from tensorrec_b200 import _lib
    assert call(lib, entry, fault) == _lib.TRK_ERR_CUDA, _lib.last_error()


@pytest.mark.parametrize('entry,fault,rc,message', FAULTS,
                         ids=['%s-%s' % (e, '-'.join('%s=%s' % kv for kv in f.items())) for e, f, _, _ in FAULTS])
def test_each_count_fault_is_rejected(lib, entry, fault, rc, message):
    from tensorrec_b200 import _lib
    assert call(lib, entry, fault) == getattr(_lib, rc)
    assert message in _lib.last_error()


# ---- dense+rank with exclusion: the chunked count (torch only, runs on the CPU) -------------------------------------
@pytest.mark.parametrize('block_bytes', [0, 4 * 12 * 300 + 8 * 300 * 5, 1 << 30])
def test_dense_count_with_exclusion_equals_the_masked_closed_form(block_bytes):
    scores, indptr, ids, excluded = tie_heavy_fixture(6)
    rows = np.repeat(np.arange(scores.shape[0]), np.diff(indptr))
    ex_rows, ex_cols = np.nonzero(excluded)
    ex_indptr = np.concatenate([[0], np.cumsum(np.bincount(ex_rows, minlength=scores.shape[0]))]).astype(np.int32)
    excl = kernels.DeviceExclusion(torch.from_numpy(ex_indptr), torch.from_numpy(ex_cols.astype(np.int32)))
    got = kernels.rank_listed_from_scores(torch.from_numpy(scores.copy()), torch.from_numpy(rows),
                                          torch.from_numpy(ids), excl=excl, block_bytes=block_bytes).numpy()
    assert np.array_equal(got, [masked_closed_form(scores, excluded, r, i) for r, i in zip(rows, ids)])
