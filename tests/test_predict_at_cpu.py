"""CPU tests of predict_at: its route, its argument checks (no device touched), the host planner of the exact kernel's
pairs mode against brute force, and both sides of every check of the trk_score_pairs* entry points."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tensorrec_b200 import kernels, tensorrec
from tensorrec_b200.errors import ModelNotFitException

F32 = np.float32


# ---- route ---------------------------------------------------------------------------------------------------------
def test_predict_at_route():
    m = tensorrec.PREDICT_AT_MIN_ITEMS
    assert tensorrec.predict_at_route(m, True) == 'exact3_pairs'
    assert tensorrec.predict_at_route(10 * m, True) == 'exact3_pairs'
    assert tensorrec.predict_at_route(m - 1, True) == 'dense+gather'
    assert tensorrec.predict_at_route(10 * m, False) == 'dense+gather'
    assert tensorrec.predict_at_route(0, False) == 'dense+gather'


# ---- planner -------------------------------------------------------------------------------------------------------
def listing(seed, n_rows, n_items, per_row_max):
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(n_rows):
        k = int(rng.integers(0, per_row_max + 1))
        rows.append(np.sort(rng.choice(n_items, size=min(k, n_items), replace=False)))
    return rows


def csr_of(rows):
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    ids = np.concatenate([np.asarray(r, np.int64) for r in rows] + [np.zeros(0, np.int64)]).astype(np.int32)
    return indptr, ids


def heavy_listing(block_rows):
    """A row with more than 128 items of one residue, an item listed by every row of a block, and an empty row."""
    n_items = 200 * 128 + 7
    rows = listing(5, 3 * block_rows + block_rows // 2, n_items, 12)
    rows[1] = np.arange(3, n_items, 128)[:150]                     # 150 items of residue 3
    shared = 4097
    for r in range(block_rows, 2 * block_rows):                      # every row of block 1 lists `shared`
        rows[r] = np.union1d(rows[r], [shared])
    rows[2 * block_rows + 1] = np.zeros(0, np.int64)
    return rows, n_items


CASES = [(listing(1, 300, 1000, 20), 1000, 128), (listing(2, 77, 100000, 40), 100000, 6),
         heavy_listing(128) + (128,), heavy_listing(64) + (64,), ([np.zeros(0, np.int64)] * 5, 10, 128)]


@pytest.mark.parametrize('case', range(len(CASES)))
@pytest.mark.parametrize('max_tiles', [1, 3, 16])
def test_pairs_plan_against_brute_force(case, max_tiles):
    rows, n_items, block_rows = CASES[case]
    indptr, ids = csr_of(rows)
    n_rows = len(rows)
    plan = kernels.pairs_plan(indptr, ids, n_rows, block_rows, max_tiles=max_tiles)
    T = plan.tile_items.shape[0]
    n_blocks = -(-n_rows // block_rows)
    assert plan.tile_items.dtype == np.int32 and plan.tile_items.shape == (T, 128)
    assert plan.block_tiles.shape == (n_blocks + 1,) and plan.block_tiles[0] == 0 and plan.block_tiles[-1] == T
    # a block's tile count is its largest residue class; no slot holds two distinct items
    for b in range(n_blocks):
        items = np.unique(np.concatenate([np.asarray(rows[r], np.int64)
                                          for r in range(b * block_rows, min(n_rows, (b + 1) * block_rows))]))
        largest = np.bincount(items % 128, minlength=128).max() if items.size else 0
        t0, t1 = plan.block_tiles[b], plan.block_tiles[b + 1]
        assert t1 - t0 == largest
        held = plan.tile_items[t0:t1]
        assert np.array_equal(np.sort(held[held >= 0]), items)          # every distinct item once, nothing else
        cols = np.nonzero(held >= 0)
        assert np.array_equal(held[cols] % 128, cols[1])                # item i sits at column i % 128
    # every pair lands at its item's slot inside its block's range, virtual columns ascend within a row
    row_of = np.repeat(np.arange(n_rows), np.diff(indptr))
    listed = ids[plan.order]
    assert np.array_equal(np.sort(plan.order), np.arange(ids.size))
    assert np.array_equal(row_of[plan.order], row_of)                   # the kernel's order keeps the rows
    tile, col = plan.cols // 128, plan.cols % 128
    assert np.array_equal(plan.tile_items[tile, col], listed)
    blk = row_of // block_rows
    assert np.all((plan.block_tiles[blk] <= tile) & (tile < plan.block_tiles[blk + 1]))
    for r in range(n_rows):
        c = plan.cols[indptr[r]:indptr[r + 1]]
        assert np.all(np.diff(c) > 0)
    # the permutation restores the listing order
    restored = np.empty_like(listed)
    restored[plan.order] = listed
    assert np.array_equal(restored, ids)
    # the work list covers each tile exactly once, in chunks of at most max_tiles of one block
    w = plan.work
    assert w.dtype == np.int32 and w.shape[1] == 3
    cover = np.zeros(T, np.int64)
    for b, t0, t1 in w:
        assert plan.block_tiles[b] <= t0 < t1 <= plan.block_tiles[b + 1] and t1 - t0 <= max_tiles
        cover[t0:t1] += 1
    assert np.all(cover == 1)


# ---- argument checks: before any device work -----------------------------------------------------------------------
def _fitted_model(monkeypatch):
    model = tensorrec.TensorRec(n_components=8)
    model.set_weights({'linear_weights_user_0': np.ones((5, 8), F32), 'linear_weights_item': np.ones((7, 8), F32),
                       'feature_biases_user': np.zeros((5, 1), F32), 'feature_biases_item': np.zeros((7, 1), F32)})

    def no_device(*_):
        raise AssertionError('device work before the arguments were checked')
    monkeypatch.setattr(tensorrec.TensorRec, '_cuda_device', staticmethod(no_device))
    return model


def test_predict_at_before_fit():
    with pytest.raises(ModelNotFitException):
        tensorrec.TensorRec(n_components=8).predict_at(sp.eye(3, 5, format='csr'), sp.eye(4, 7, format='csr'),
                                                       sp.eye(3, 4, format='csr'))


@pytest.mark.parametrize('pairs,user_cols,item_cols,match', [
    (np.ones((3, 4)), 5, 7, 'scipy sparse'),
    (sp.eye(3, 5, format='csr'), 5, 7, 'shape'),
    (sp.eye(4, 4, format='csr'), 5, 7, 'shape'),
    (sp.eye(3, 4, format='csr'), 6, 7, 'user'),
    (sp.eye(3, 4, format='csr'), 5, 8, 'item'),
])
def test_predict_at_rejects_bad_arguments_without_device_work(monkeypatch, pairs, user_cols, item_cols, match):
    model = _fitted_model(monkeypatch)
    with pytest.raises(ValueError, match=match):
        model.predict_at(sp.eye(3, user_cols, format='csr', dtype=F32), sp.eye(4, item_cols, format='csr', dtype=F32),
                         pairs)


def test_predict_at_without_listed_pairs_needs_no_device(monkeypatch):
    model = _fitted_model(monkeypatch)
    pairs = sp.csr_matrix((np.zeros(2, F32), ([0, 2], [1, 3])), shape=(3, 4))    # explicit zeros list nothing
    r = model.predict_at(sp.eye(3, 5, format='csr', dtype=F32), sp.eye(4, 7, format='csr', dtype=F32), pairs)
    assert isinstance(r, sp.csr_matrix) and r.shape == (3, 4) and r.nnz == 0 and r.dtype == np.float32
    assert model.last_predict_at_info == {'path': 'dense+gather', 'tiles': 0}


# ---- both sides of every check of the pairs entry points ------------------------------------------------------------
A = 1 << 20          # a 16-byte aligned fake device address
MISALIGNED = A + 4
PAIRS = dict(user_split=A, user_scale=A, user_bias=None, item_split=A, slot_meta=A, n_users=10, n_items=300, d_pad=64,
             pair_indptr=A, pair_cols=A, pair_score=A, tile_items=A, n_tiles=3, work=A, n_work=2)
PAIRS_EUCLID = dict(PAIRS, user_half_sqnorm=A, slot_half_sqnorm=A)
PAIRS_TASTES = dict(user_split=A, user_scale=A, user_bias=None, n_tastes=2, attention=0, item_split=A, slot_meta=A,
                    n_users=10, n_items=300, d_pad=64, pair_indptr=A, pair_cols=A, pair_score=A, tile_items=A,
                    n_tiles=3, work=A, n_work=2)
PAIRS_TASTES_EUCLID = dict(PAIRS_TASTES, user_half_sqnorm=A, slot_half_sqnorm=A)
ENTRY = {'trk_score_pairs_f16x3': PAIRS, 'trk_score_pairs_euclid_f16x3': PAIRS_EUCLID,
         'trk_score_pairs_tastes_f16x3': PAIRS_TASTES, 'trk_score_pairs_tastes_euclid_f16x3': PAIRS_TASTES_EUCLID}
VALID = [
    ('trk_score_pairs_f16x3', {}),
    ('trk_score_pairs_f16x3', dict(d_pad=128, user_bias=A, n_tiles=1 << 24, n_work=1)),
    ('trk_score_pairs_euclid_f16x3', {}),
    ('trk_score_pairs_euclid_f16x3', dict(d_pad=128, user_bias=A)),
    ('trk_score_pairs_tastes_f16x3', dict(n_tastes=32, attention=1)),
    ('trk_score_pairs_tastes_f16x3', dict(n_tastes=1, attention=1, d_pad=128)),
    ('trk_score_pairs_tastes_euclid_f16x3', {}),
    ('trk_score_pairs_tastes_euclid_f16x3', dict(n_tastes=3, attention=1, user_bias=A)),
]
FAULTS = [
    ('trk_score_pairs_f16x3', dict(pair_indptr=None), 'TRK_ERR_ARG', 'null pair plan'),
    ('trk_score_pairs_f16x3', dict(pair_cols=None), 'TRK_ERR_ARG', 'null pair plan'),
    ('trk_score_pairs_euclid_f16x3', dict(pair_score=None), 'TRK_ERR_ARG', 'null pair plan'),
    ('trk_score_pairs_tastes_f16x3', dict(tile_items=None), 'TRK_ERR_ARG', 'null pair plan'),
    ('trk_score_pairs_tastes_euclid_f16x3', dict(work=None), 'TRK_ERR_ARG', 'null pair plan'),
    ('trk_score_pairs_f16x3', dict(n_tiles=0), 'TRK_ERR_ARG', 'n_tiles=0'),
    ('trk_score_pairs_f16x3', dict(n_work=0), 'TRK_ERR_ARG', 'n_work=0'),
    ('trk_score_pairs_f16x3', dict(n_tiles=(1 << 24) + 1), 'TRK_ERR_ARG', 'virtual columns'),
    ('trk_score_pairs_f16x3', dict(d_pad=96), 'TRK_ERR_UNSUPPORTED', 'd_pad=96'),
    ('trk_score_pairs_f16x3', dict(user_split=None), 'TRK_ERR_ARG', 'null operand'),
    ('trk_score_pairs_f16x3', dict(slot_meta=MISALIGNED), 'TRK_ERR_ARG', '16-byte aligned'),
    ('trk_score_pairs_f16x3', dict(n_users=0), 'TRK_ERR_ARG', 'empty shape'),
    ('trk_score_pairs_euclid_f16x3', dict(slot_half_sqnorm=None), 'TRK_ERR_ARG', 'trk_score_pairs_euclid_f16x3: null'),
    ('trk_score_pairs_euclid_f16x3', dict(slot_half_sqnorm=MISALIGNED), 'TRK_ERR_ARG', 'item_half_sqnorm must be'),
    ('trk_score_pairs_tastes_f16x3', dict(n_tastes=0), 'TRK_ERR_ARG', 'n_tastes=0'),
    ('trk_score_pairs_tastes_f16x3', dict(n_tastes=1), 'TRK_ERR_ARG', 'n_tastes=1'),
    ('trk_score_pairs_tastes_f16x3', dict(n_tastes=33, attention=1), 'TRK_ERR_UNSUPPORTED', 'exceed'),
    ('trk_score_pairs_tastes_euclid_f16x3', dict(user_half_sqnorm=None), 'TRK_ERR_ARG',
     'trk_score_pairs_tastes_euclid_f16x3: null'),
    ('trk_score_pairs_tastes_euclid_f16x3', dict(n_tastes=0), 'TRK_ERR_ARG', 'n_tastes=0'),
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
def test_valid_pairs_calls_pass_every_check(lib, entry, fault):
    from tensorrec_b200 import _lib
    assert call(lib, entry, fault) == _lib.TRK_ERR_CUDA, _lib.last_error()


@pytest.mark.parametrize('entry,fault,rc,message', FAULTS,
                         ids=['%s-%s' % (e, '-'.join('%s=%s' % kv for kv in f.items())) for e, f, _, _ in FAULTS])
def test_each_pairs_fault_is_rejected(lib, entry, fault, rc, message):
    from tensorrec_b200 import _lib
    assert call(lib, entry, fault) == getattr(_lib, rc)
    assert message in _lib.last_error()
