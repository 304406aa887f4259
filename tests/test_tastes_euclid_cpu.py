"""CPU tests of Euclidean mixtures of tastes on the taste-collapsing tensor-core kernel (DESIGN §3.12): the predicate
_euclid_tastes_tensor_ok next to the predicates it leaves unchanged, the score form, the top-k routes of Euclidean
attention models, rank_at_route, and the argument checks of the four C entry points
trk_score_{dense,topk,topk_wide,count}_tastes_euclid_f16x3, each from both sides."""
import pytest

import tensorrec_b200 as T
from tensorrec_b200 import kernels, tensorrec

P = T.prediction_graphs
R = T.representation_graphs


def model(n_tastes=3, attention=False, prediction=P.EuclideanSimilarityPredictionGraph, d=64):
    return T.TensorRec(n_components=d, n_tastes=n_tastes, prediction_graph=prediction(),
                       attention_graph=R.LinearRepresentationGraph() if attention else None)


# (model kwargs, _euclid_tastes_tensor_ok, _tensor_score_form)
KINDS = {
    'euclid_max_t2': (dict(n_tastes=2), True, 'tastes_euclid'),
    'euclid_max_t3': (dict(n_tastes=3), True, 'tastes_euclid'),
    'euclid_max_t64': (dict(n_tastes=64), True, 'tastes_euclid'),
    'euclid_max_t65': (dict(n_tastes=65), False, None),
    'euclid_max_d128': (dict(n_tastes=3, d=128), True, 'tastes_euclid'),
    'euclid_max_d200': (dict(n_tastes=3, d=200), False, None),
    'euclid_attention_t2': (dict(n_tastes=2, attention=True), True, 'tastes_euclid'),
    'euclid_attention_t32': (dict(n_tastes=32, attention=True), True, 'tastes_euclid'),
    'euclid_attention_t33': (dict(n_tastes=33, attention=True), False, None),
    'euclid_one_taste': (dict(n_tastes=1), False, 'euclidean'),
    'dot_tastes': (dict(n_tastes=3, prediction=P.DotProductPredictionGraph), False, 'tastes'),
    'cosine_attention': (dict(n_tastes=2, attention=True, prediction=P.CosineSimilarityPredictionGraph), False,
                         'tastes'),
}


@pytest.mark.parametrize('kind', sorted(KINDS))
def test_predicate_and_score_form_by_model_kind(kind):
    kw, ok, form = KINDS[kind]
    m = model(**kw)
    assert m._euclid_tastes_tensor_ok() == ok
    assert m._tensor_score_form() == form


@pytest.mark.parametrize('attention', [False, True])
def test_existing_predicates_answer_as_before(attention):
    m = model(n_tastes=3, attention=attention)
    assert not m._tastes_tensor_ok()
    assert not m._tensor_path_ok(True)
    assert m._euclidean_tensor_ok() == (not attention)


def test_score_path_exact_turns_it_off(monkeypatch):
    monkeypatch.setattr(tensorrec, 'SCORE_PATH', 'exact')
    for kw, _, _ in KINDS.values():
        m = model(**kw)
        assert not m._euclid_tastes_tensor_ok()
        assert m._tensor_score_form() is None


def test_score_path_tensor_accepts_the_models(monkeypatch):
    monkeypatch.setattr(tensorrec, 'SCORE_PATH', 'tensor')
    for attention in (False, True):
        assert model(n_tastes=3, attention=attention)._tensor_score_form() == 'tastes_euclid'
    # a model no tensor-core form covers still raises
    with pytest.raises(RuntimeError):
        model(n_tastes=3, attention=True, d=200)._tensor_score_form()


def test_rank_at_route_for_both_variants():
    form = model(n_tastes=3)._tensor_score_form()
    assert tensorrec.rank_at_route(tensorrec.RANK_AT_MIN_ITEMS, form is not None) == 'exact3_count'
    assert tensorrec.rank_at_route(tensorrec.RANK_AT_MIN_ITEMS - 1, form is not None) == 'dense+rank'
    # with attention, from RANK_AT_EUCLID_ATTENTION_MIN_ITEMS items
    form = model(n_tastes=3, attention=True)._tensor_score_form()
    floor = tensorrec.RANK_AT_EUCLID_ATTENTION_MIN_ITEMS
    assert floor >= tensorrec.RANK_AT_MIN_ITEMS
    assert tensorrec.rank_at_route(floor, form is not None, euclid_attention=True) == 'exact3_count'
    assert tensorrec.rank_at_route(floor - 1, form is not None, euclid_attention=True) == 'dense+rank'
    assert tensorrec.rank_at_route(floor, False, euclid_attention=True) == 'dense+rank'


# ---- the top-k routes of Euclidean attention models ---------------------------------------------------------------
@pytest.fixture
def limits(monkeypatch):
    monkeypatch.setattr(kernels, 'filter_max_k', lambda: 16)
    monkeypatch.setattr(kernels, 'topk_max_k', lambda d_pad: 32)


def attention_path(k, n_items, sharded=False, d=64):
    """The route predict_top_k takes for a Euclidean attention model (model_ok and keywords as it forms them)."""
    m = model(n_tastes=3, attention=True, d=d)
    model_ok = m._tastes_tensor_ok() or m._euclid_tastes_tensor_ok()
    return m._topk_path(k, n_items, model_ok, False, sharded=sharded, euclidean=m._euclidean_tensor_ok(),
                        attention=True)


def test_attention_routes_by_k_and_catalogue(limits):
    n = 10 ** 6
    assert {attention_path(k, n) for k in (1, 10, 16, 17, 32)} == {'exact3'}
    assert {attention_path(k, n) for k in (33, 100, 1000, 1024)} == {'exact3_wide'}
    assert attention_path(1025, n) == 'dense+rank'
    assert attention_path(10, tensorrec.ATTENTION_MIN_ITEMS) == 'exact3'
    assert attention_path(10, tensorrec.ATTENTION_MIN_ITEMS - 1) == 'dense+rank'
    assert attention_path(100, tensorrec.EXACT_WIDE_MIN_ITEMS) == 'exact3_wide'
    assert attention_path(100, tensorrec.EXACT_WIDE_MIN_ITEMS - 1) == 'dense+rank'
    assert attention_path(10, 0) == 'dense+rank'
    # d_pad > 128: no tensor-core form
    assert attention_path(10, n, d=200) == 'dense+rank'


def test_attention_routes_of_sharded_calls(limits):
    for n in (1, 1000, tensorrec.EXACT_WIDE_MIN_ITEMS, 10 ** 6):
        assert attention_path(10, n, sharded=True) == 'exact3'
        assert attention_path(100, n, sharded=True) == 'exact3_wide'
    assert attention_path(1025, 10 ** 6, sharded=True) == 'dense+rank'


# ---- the C entry points ---------------------------------------------------------------------------------------------
A = 1 << 20          # a 16-byte aligned fake device address
MISALIGNED = A + 4

NORMS = dict(user_half_sqnorm=A, item_half_sqnorm=A)
DENSE = dict(user_split=A, user_scale=A, user_bias=None, n_tastes=3, attention=0, item_split=A, item_meta=A,
             n_users=10, n_items=300, d_pad=64, out=A, out_row_stride=300, **NORMS)
TOPK = dict(user_split=A, user_scale=A, user_bias=None, n_tastes=3, attention=1, item_split=A, item_meta=A,
            n_users=10, n_items=300, d_pad=64, k=5, n_splits=1, item_id_offset=0, cand_score=A, cand_item=A,
            excl_indptr=None, excl_ids=None, excl_row_map=None, **NORMS)
WIDE = dict(user_split=A, user_scale=A, user_bias=None, n_tastes=3, attention=1, item_split=A, item_meta=A,
            n_users=10, n_items=300, d_pad=64, k=100, n_splits=1, item_id_offset=0, list_score=A, list_item=A,
            list_count=A, excl_indptr=None, excl_ids=None, excl_row_map=None, **NORMS)
COUNT = dict(user_split=A, user_scale=A, user_bias=None, n_tastes=3, attention=0, item_split=A, item_meta=A,
             n_users=10, n_items=300, d_pad=64, n_splits=1, item_id_offset=0, pair_indptr=A, pair_ids=A, pair_score=A,
             pair_count=A, block_pairs=A, pass_=0, excl_indptr=None, excl_ids=None, excl_row_map=None, **NORMS)

ENTRY = {
    'trk_score_dense_tastes_euclid_f16x3': DENSE,
    'trk_score_topk_tastes_euclid_f16x3': TOPK,
    'trk_score_topk_wide_tastes_euclid_f16x3': WIDE,
    'trk_score_count_tastes_euclid_f16x3': COUNT,
}

# valid calls: every check passes (TRK_ERR_CUDA from the tensor-map encode)
VALID = [
    ('trk_score_dense_tastes_euclid_f16x3', {}),
    ('trk_score_dense_tastes_euclid_f16x3', dict(attention=1, n_tastes=32, d_pad=128, user_bias=A)),
    ('trk_score_dense_tastes_euclid_f16x3', dict(n_tastes=64, out=MISALIGNED, out_row_stride=301)),
    ('trk_score_topk_tastes_euclid_f16x3', {}),
    ('trk_score_topk_tastes_euclid_f16x3', dict(k=32, d_pad=128, excl_indptr=A, excl_ids=A, excl_row_map=A)),
    ('trk_score_topk_wide_tastes_euclid_f16x3', {}),
    ('trk_score_topk_wide_tastes_euclid_f16x3', dict(k=1024, n_splits=4, excl_indptr=A, excl_ids=A)),
    ('trk_score_count_tastes_euclid_f16x3', {}),
    ('trk_score_count_tastes_euclid_f16x3', dict(attention=1, pass_=-1, pair_count=None, excl_indptr=A, excl_ids=A)),
]

# one fault each: (entry point, fault, return code name, a substring of trk_last_error())
FAULTS = [
    ('trk_score_dense_tastes_euclid_f16x3', dict(user_half_sqnorm=None), 'TRK_ERR_ARG', 'null squared norms'),
    ('trk_score_dense_tastes_euclid_f16x3', dict(item_half_sqnorm=None), 'TRK_ERR_ARG', 'null squared norms'),
    ('trk_score_dense_tastes_euclid_f16x3', dict(item_half_sqnorm=MISALIGNED), 'TRK_ERR_ARG',
     'item_half_sqnorm must be'),
    ('trk_score_dense_tastes_euclid_f16x3', dict(n_tastes=1), 'TRK_ERR_ARG', 'n_tastes=1'),
    ('trk_score_dense_tastes_euclid_f16x3', dict(n_tastes=65), 'TRK_ERR_UNSUPPORTED', 'exceed'),
    ('trk_score_dense_tastes_euclid_f16x3', dict(d_pad=96), 'TRK_ERR_UNSUPPORTED', 'd_pad=96'),
    ('trk_score_topk_tastes_euclid_f16x3', dict(user_half_sqnorm=None), 'TRK_ERR_ARG', 'null squared norms'),
    ('trk_score_topk_tastes_euclid_f16x3', dict(item_half_sqnorm=MISALIGNED), 'TRK_ERR_ARG',
     'item_half_sqnorm must be'),
    ('trk_score_topk_tastes_euclid_f16x3', dict(attention=0), 'TRK_ERR_UNSUPPORTED', 'trk_score_topk_euclid_f16x3'),
    ('trk_score_topk_tastes_euclid_f16x3', dict(k=33), 'TRK_ERR_UNSUPPORTED', 'k=33'),
    ('trk_score_topk_tastes_euclid_f16x3', dict(n_tastes=33), 'TRK_ERR_UNSUPPORTED', 'exceed'),
    ('trk_score_topk_wide_tastes_euclid_f16x3', dict(item_half_sqnorm=None), 'TRK_ERR_ARG', 'null squared norms'),
    ('trk_score_topk_wide_tastes_euclid_f16x3', dict(item_half_sqnorm=MISALIGNED), 'TRK_ERR_ARG',
     'item_half_sqnorm must be'),
    ('trk_score_topk_wide_tastes_euclid_f16x3', dict(attention=0), 'TRK_ERR_UNSUPPORTED',
     'trk_score_topk_wide_euclid_f16x3'),
    ('trk_score_topk_wide_tastes_euclid_f16x3', dict(k=1025), 'TRK_ERR_UNSUPPORTED', 'k=1025'),
    ('trk_score_topk_wide_tastes_euclid_f16x3', dict(list_count=None), 'TRK_ERR_ARG', 'null output'),
    ('trk_score_count_tastes_euclid_f16x3', dict(user_half_sqnorm=None), 'TRK_ERR_ARG', 'null squared norms'),
    ('trk_score_count_tastes_euclid_f16x3', dict(item_half_sqnorm=MISALIGNED), 'TRK_ERR_ARG',
     'item_half_sqnorm must be'),
    ('trk_score_count_tastes_euclid_f16x3', dict(pass_=-2), 'TRK_ERR_ARG', 'pass=-2'),
    ('trk_score_count_tastes_euclid_f16x3', dict(pair_count=None), 'TRK_ERR_ARG', 'null pair_count'),
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


def test_the_twins_keep_their_return_codes(lib):
    """The norms-free twins answer as before: a dot mixture of tastes without attention has no wide mode."""
    from tensorrec_b200 import _lib
    twin = {k: v for k, v in WIDE.items() if k not in NORMS}
    twin['attention'] = 0
    assert lib.trk_score_topk_wide_tastes_f16x3(*twin.values(), None) == _lib.TRK_ERR_UNSUPPORTED
    assert 'Euclidean and attention' in _lib.last_error()
    twin = {k: v for k, v in TOPK.items() if k not in NORMS}
    twin['attention'] = 0
    assert lib.trk_score_topk_tastes_f16x3(*twin.values(), None) == _lib.TRK_ERR_CUDA
