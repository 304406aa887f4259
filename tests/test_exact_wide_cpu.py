"""CPU tests of the exact kernel's wide mode (32 < k <= 1024 for Euclidean and attention models, DESIGN §3.8): the route
through TensorRec._topk_path, the block size, the argument checks of the three new C entry points, and a numpy model
of one list's admission (score > the k-th kept score) and exact compaction, checked against a plain sorted top-k."""
import numpy as np
import pytest

import tensorrec_b200 as T
from tensorrec_b200 import kernels, tensorrec

SENTINEL_ID = 2 ** 31 - 1


# ---- the route ------------------------------------------------------------------------------------------------------
@pytest.fixture
def limits(monkeypatch):
    monkeypatch.setattr(kernels, 'filter_max_k', lambda: 16)
    monkeypatch.setattr(kernels, 'topk_max_k', lambda d_pad: 32)


def path(k, n_items, n_tastes=1, attention=False, sharded=False):
    model = T.TensorRec(n_components=64, n_tastes=n_tastes)
    euclidean = not attention
    return model._topk_path(k, n_items, True, n_tastes == 1, sharded=sharded, euclidean=euclidean,
                            attention=attention)


@pytest.mark.parametrize('kind', [dict(), dict(n_tastes=3), dict(attention=True, n_tastes=3)])
def test_k_limits(limits, kind):
    n = 10 ** 6
    assert path(32, n, **kind) == 'exact3'
    assert path(33, n, **kind) == 'exact3_wide'
    assert path(100, n, **kind) == 'exact3_wide'
    assert path(1024, n, **kind) == 'exact3_wide'
    assert path(1025, n, **kind) == 'dense+rank'


@pytest.mark.parametrize('kind', [dict(), dict(n_tastes=3), dict(attention=True, n_tastes=3)])
def test_catalogue_floor_and_shards(limits, kind):
    floor = tensorrec.EXACT_WIDE_MIN_ITEMS
    assert path(100, floor - 1, **kind) == 'dense+rank'
    assert path(100, floor, **kind) == 'exact3_wide'
    assert path(100, 0, **kind) == 'dense+rank'
    assert {path(100, n, sharded=True, **kind) for n in (1, floor - 1, floor, 10 ** 6)} == {'exact3_wide'}
    assert path(1025, 10 ** 6, sharded=True, **kind) == 'dense+rank'


def test_floor_keeps_small_attention_catalogues_on_dense_rank():
    # the 1061-item attention catalogue of the dense+rank tests at k = 100 stays there
    assert tensorrec.EXACT_WIDE_MIN_ITEMS >= 2048


def test_last_topk_info(limits):
    model = T.TensorRec(n_components=64)
    model._topk_path(100, 10 ** 6, True, True, euclidean=True)
    assert model.last_topk_info == {'path': 'exact3_wide', 'fallback_rows': 0}


def test_the_keyword_default_leaves_every_route(limits):
    for kw in ({'euclidean': True}, {'attention': True}, {}):
        for k, n in ((10, 10 ** 6), (33, 10 ** 6), (100, 10 ** 6), (1024, 10 ** 6), (100, 10)):
            for single in (True, False):
                assert tensorrec.topk_route(k, n, True, single, 16, 32, **kw) == \
                    tensorrec.topk_route(k, n, True, single, 16, 32, exact_wide_max_k=0, **kw)
                if not kw:      # dot / cosine models do not look at the keyword
                    assert tensorrec.topk_route(k, n, True, single, 16, 32, merge_max_k=1024) == \
                        tensorrec.topk_route(k, n, True, single, 16, 32, merge_max_k=1024, exact_wide_max_k=1024)


def test_other_models_keep_their_routes(limits):
    model = T.TensorRec(n_components=64)
    assert model._topk_path(100, 10 ** 6, True, True) == 'wide'
    assert model._topk_path(100, 10 ** 6, False, True, euclidean=True) == 'dense+rank'


# ---- block size -----------------------------------------------------------------------------------------------------
def test_block_rows(monkeypatch):
    monkeypatch.setattr(kernels, 'exact_wide_list_capacity', lambda k: 2 * (-(-k // 32) * 32))
    one = T.TensorRec(n_components=64)
    three = T.TensorRec(n_components=64, n_tastes=3)
    for k in (33, 100, 1000, 1024):
        cap = kernels.exact_wide_list_capacity(k)
        per_row = 2 * (8 * cap + 4)
        rows = one._topk_block_rows('exact3_wide', 10 ** 7, 10 ** 6, k)
        assert rows * per_row <= one.PREDICT_BLOCK_BYTES and rows % 256 == 0
        assert (rows + 256) * per_row > one.PREDICT_BLOCK_BYTES
        folded = three._topk_block_rows('exact3_wide', 10 ** 7, 10 ** 6, k, n_tastes=3)
        assert folded * (per_row + 3 * 8 * k) <= three.PREDICT_BLOCK_BYTES
        assert folded < rows and folded % 256 == 0


# ---- the C entry points ---------------------------------------------------------------------------------------------
A = 1 << 20          # a 16-byte aligned fake device address
MISALIGNED = A + 4

WIDE_EUCLID = dict(user_split=A, user_scale=A, user_bias=None, item_split=A, item_meta=A, n_users=10, n_items=300,
                   d_pad=64, k=100, n_splits=1, item_id_offset=0, list_score=A, list_item=A, list_count=A,
                   n_users_live=None, excl_indptr=None, excl_ids=None, excl_row_map=None, user_half_sqnorm=A,
                   item_half_sqnorm=A)
WIDE_TASTES = dict(user_split=A, user_scale=A, user_bias=None, n_tastes=3, attention=1, item_split=A, item_meta=A,
                   n_users=10, n_items=300, d_pad=64, k=100, n_splits=1, item_id_offset=0, list_score=A, list_item=A,
                   list_count=A, excl_indptr=None, excl_ids=None, excl_row_map=None)
SELECT = dict(list_score=A, list_item=A, list_count=A, n_rows=10, n_lists=2, list_width=256, k=100, out_score=A,
              out_item=A, out_row_stride=200)

ENTRY = {
    'trk_score_topk_wide_euclid_f16x3': WIDE_EUCLID,
    'trk_score_topk_wide_tastes_f16x3': WIDE_TASTES,
    'trk_select_topk_lists': SELECT,
}

# valid calls: every check passes (TRK_ERR_CUDA from the tensor-map encode, or from the launch)
VALID = [
    ('trk_score_topk_wide_euclid_f16x3', {}),
    ('trk_score_topk_wide_euclid_f16x3', dict(k=1)),
    ('trk_score_topk_wide_euclid_f16x3', dict(k=1024, d_pad=128, n_splits=8, user_bias=A, n_users_live=A)),
    ('trk_score_topk_wide_euclid_f16x3', dict(excl_indptr=A, excl_ids=A, excl_row_map=A)),
    ('trk_score_topk_wide_tastes_f16x3', {}),
    ('trk_score_topk_wide_tastes_f16x3', dict(n_tastes=1, k=1024, d_pad=128)),
    ('trk_score_topk_wide_tastes_f16x3', dict(n_tastes=32, excl_indptr=A, excl_ids=A, excl_row_map=A)),
    ('trk_select_topk_lists', {}),
    ('trk_select_topk_lists', dict(n_lists=16, list_width=2048, k=1024, out_row_stride=1024)),
    ('trk_select_topk_lists', dict(k=1, list_width=1, out_row_stride=1)),
]

# one fault each: (entry point, fault, return code name, a substring of trk_last_error())
FAULTS = [
    ('trk_score_topk_wide_euclid_f16x3', dict(k=1025), 'TRK_ERR_UNSUPPORTED', 'k=1025'),
    ('trk_score_topk_wide_euclid_f16x3', dict(k=0), 'TRK_ERR_UNSUPPORTED', 'k=0'),
    ('trk_score_topk_wide_tastes_f16x3', dict(k=1025), 'TRK_ERR_UNSUPPORTED', 'k=1025'),
    ('trk_score_topk_wide_euclid_f16x3', dict(d_pad=96), 'TRK_ERR_UNSUPPORTED', 'd_pad=96'),
    ('trk_score_topk_wide_tastes_f16x3', dict(attention=0), 'TRK_ERR_UNSUPPORTED', 'Euclidean and attention'),
    ('trk_score_topk_wide_tastes_f16x3', dict(n_tastes=33), 'TRK_ERR_UNSUPPORTED', 'exceed'),
    ('trk_score_topk_wide_euclid_f16x3', dict(user_half_sqnorm=None), 'TRK_ERR_ARG',
     'trk_score_topk_wide_euclid_f16x3: null squared norms'),
    ('trk_score_topk_wide_euclid_f16x3', dict(item_half_sqnorm=MISALIGNED), 'TRK_ERR_ARG', 'item_half_sqnorm must be'),
    ('trk_score_topk_wide_euclid_f16x3', dict(list_count=None), 'TRK_ERR_ARG', 'null output'),
    ('trk_score_topk_wide_euclid_f16x3', dict(list_item=None), 'TRK_ERR_ARG', 'null output'),
    ('trk_score_topk_wide_tastes_f16x3', dict(list_score=None), 'TRK_ERR_ARG', 'null output'),
    ('trk_score_topk_wide_tastes_f16x3', dict(list_count=None), 'TRK_ERR_ARG', 'null output'),
    ('trk_score_topk_wide_euclid_f16x3', dict(n_splits=0), 'TRK_ERR_ARG', 'n_splits'),
    ('trk_score_topk_wide_euclid_f16x3', dict(user_split=None), 'TRK_ERR_ARG', 'null operand'),
    ('trk_score_topk_wide_euclid_f16x3', dict(user_split=MISALIGNED), 'TRK_ERR_ARG', '16-byte aligned'),
    ('trk_score_topk_wide_euclid_f16x3', dict(n_users=0), 'TRK_ERR_ARG', 'empty shape'),
    ('trk_score_topk_wide_euclid_f16x3', dict(excl_ids=A), 'TRK_ERR_ARG', 'go together'),
    ('trk_score_topk_wide_tastes_f16x3', dict(n_tastes=0), 'TRK_ERR_ARG', 'n_tastes=0'),
    ('trk_score_topk_wide_tastes_f16x3', dict(excl_row_map=A), 'TRK_ERR_ARG', 'go together'),
    ('trk_select_topk_lists', dict(list_count=None), 'TRK_ERR_ARG', 'null input'),
    ('trk_select_topk_lists', dict(out_item=None), 'TRK_ERR_ARG', 'null output'),
    ('trk_select_topk_lists', dict(k=0), 'TRK_ERR_ARG', 'bad sizes'),
    ('trk_select_topk_lists', dict(list_width=99), 'TRK_ERR_ARG', 'bad sizes'),
    ('trk_select_topk_lists', dict(n_lists=0), 'TRK_ERR_ARG', 'bad sizes'),
    ('trk_select_topk_lists', dict(n_rows=-1), 'TRK_ERR_ARG', 'bad sizes'),
    ('trk_select_topk_lists', dict(out_row_stride=99), 'TRK_ERR_ARG', 'out_row_stride'),
    ('trk_select_topk_lists', dict(n_lists=17, list_width=2048, k=1024, out_row_stride=1024), 'TRK_ERR_ARG',
     'exceed 16384'),
]


@pytest.fixture(scope='module')
def lib():
    import torch
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
def test_valid_calls_pass_every_check(lib, entry, fault):
    from tensorrec_b200 import _lib
    assert call(lib, entry, fault) == _lib.TRK_ERR_CUDA, _lib.last_error()


@pytest.mark.parametrize('entry,fault,rc,message', FAULTS,
                         ids=['%s-%s' % (e, '-'.join('%s=%s' % kv for kv in f.items())) for e, f, _, _ in FAULTS])
def test_each_fault_is_rejected(lib, entry, fault, rc, message):
    from tensorrec_b200 import _lib
    assert call(lib, entry, fault) == getattr(_lib, rc)
    assert message in _lib.last_error()


def test_every_entry_point_is_covered():
    assert {e for e, _ in VALID} == set(ENTRY) == {e for e, _, _, _ in FAULTS}


def test_select_of_no_rows_launches_nothing(lib):
    from tensorrec_b200 import _lib
    assert call(lib, 'trk_select_topk_lists', dict(n_rows=0)) == _lib.TRK_OK


def test_list_capacity(lib):
    for k, cap in ((1, 64), (32, 64), (33, 128), (100, 256), (1000, 2048), (1024, 2048)):
        assert lib.trk_score_topk_wide_list_capacity(k) == cap
    assert lib.trk_score_topk_wide_list_capacity(0) == 0 and lib.trk_score_topk_wide_list_capacity(1025) == 0


# ---- a numpy model of one list --------------------------------------------------------------------------------------
def key(s):
    """The kernel's order-preserving uint32 key of a float32 score (wide_key)."""
    u = np.float32(s).view(np.uint32)
    return int(~u & 0xffffffff) if u & 0x80000000 else int(u | 0x80000000)


def compact(ls, li, k):
    """exact_wide_compact: the k-th best key, every entry above it, then the first entries equal to it (list order)."""
    keys = [key(s) for s in ls]
    kth = sorted(keys, reverse=True)[k - 1]
    n_eq = k - sum(x > kth for x in keys)
    out_s, out_i = [], []
    for s, i, x in zip(ls, li, keys):
        if x > kth or (x == kth and n_eq > 0):
            n_eq -= x == kth
            out_s.append(s)
            out_i.append(i)
    return out_s, out_i, np.float32(ls[keys.index(kth)])


def model_list(scores, ids, k, stats=None):
    """One list over the columns `ids` (ascending) with final scores `scores`, in chunks of 32 as the kernel sees
    them.  Returns its entries at the end of the item range (at most k) and counts the compactions in stats."""
    cap = 2 * (-(-k // 32) * 32)
    ls, li, thr = [], [], np.float32(-np.inf)
    for c0 in range(0, len(ids), 32):
        chunk = [(np.float32(s), i) for s, i in zip(scores[c0:c0 + 32], ids[c0:c0 + 32])]
        if len(ls) + sum(s > thr for s, _ in chunk) > cap:
            ls, li, thr = compact(ls, li, k)
            if stats is not None:
                stats['compactions'] += 1
        for s, i in chunk:
            if s > thr:
                ls.append(s)
                li.append(i)
        assert len(ls) <= cap
    if len(ls) > k:
        ls, li, _ = compact(ls, li, k)
    return ls, li


def sorted_top(scores, ids, k):
    order = sorted(((-np.float64(s), int(i)) for s, i in zip(scores, ids) if s > -np.inf))[:k]
    items = np.full(k, SENTINEL_ID, np.int64)
    vals = np.full(k, -np.inf, np.float32)
    items[:len(order)] = [i for _, i in order]
    vals[:len(order)] = [-s for s, _ in order]
    return items, vals


def model_row(scores, k, n_splits):
    """Every list of one row -- item splits of whole 128-column tiles, each split's two column halves -- then the
    selection over their union, as the kernel and trk_select_topk_lists compute it."""
    n = len(scores)
    n_tiles = -(-n // 128)
    per_split = -(-n_tiles // n_splits)
    all_s, all_i = [], []
    for sp_ in range(n_splits):
        cols = np.arange(sp_ * per_split * 128, min(n, (sp_ + 1) * per_split * 128))
        for half in (0, 1):
            mine = cols[(cols % 128) // 64 == half]
            ls, li = model_list(scores[mine], mine, k)
            assert len(ls) <= k
            all_s += ls
            all_i += li
    return sorted_top(np.array(all_s, np.float32), np.array(all_i), k)


@pytest.mark.parametrize('k', [1, 33, 100, 256])
@pytest.mark.parametrize('kind', ['random', 'equal', 'rising', 'few_values', 'excluded'])
@pytest.mark.parametrize('n_splits', [1, 3])
def test_lists_give_the_exact_topk(k, kind, n_splits):
    rng = np.random.default_rng(k + len(kind) + n_splits)
    n = 3000 + 37
    scores = {
        'random': rng.standard_normal(n),
        'equal': np.full(n, 2.5),
        'rising': np.arange(n, dtype=np.float64),           # every item is admitted: the most compactions
        'few_values': rng.integers(-3, 4, n).astype(np.float64),
        'excluded': np.where(rng.random(n) < 0.97, -np.inf, rng.standard_normal(n)),
    }[kind].astype(np.float32)
    got = model_row(scores, k, n_splits)
    exp = sorted_top(scores, np.arange(n), k)
    assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])


def test_rising_scores_compact_as_often_as_the_capacity_allows():
    k = 100
    stats = {'compactions': 0}
    n = 128 * 40
    ls, li = model_list(np.arange(n, dtype=np.float32), np.arange(n), k, stats)
    assert sorted(li) == list(range(n - k, n))
    cap = 2 * 128
    assert stats['compactions'] >= (n - cap) // (cap - k + 32)


def test_lists_that_are_exactly_full():
    """A list that reaches the capacity exactly is not compacted until the next admission would overflow it."""
    k = 64
    cap = 2 * 64
    stats = {'compactions': 0}
    ls, li = model_list(np.arange(cap, dtype=np.float32), np.arange(cap), k, stats)
    assert stats['compactions'] == 0 and sorted(li) == list(range(cap - k, cap))
    stats = {'compactions': 0}
    ls, li = model_list(np.arange(cap + 1, dtype=np.float32), np.arange(cap + 1), k, stats)
    assert stats['compactions'] == 1 and sorted(li) == list(range(cap + 1 - k, cap + 1))


def test_equal_scores_keep_the_lowest_ids():
    k = 40
    scores = np.zeros(500, np.float32)
    scores[::7] = 1.0                                   # 72 items at 1.0, the rest at 0.0
    ls, li = model_list(scores, np.arange(500), k)
    assert sorted(li) == list(range(0, 7 * k, 7))
    scores[:] = 0.0
    ls, li = model_list(scores, np.arange(500), k)
    assert sorted(li) == list(range(k))
