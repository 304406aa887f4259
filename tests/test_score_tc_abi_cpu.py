"""CPU tests of the argument checks of the exact tensor-core kernel's seven C entry points (trk_score_{topk,dense}*).

Every case is a valid call with exactly one fault, made through ctypes with 16-byte aligned fake device addresses that
no check dereferences.  Without a CUDA device a valid call gets through every check and fails when the tensor maps are
encoded (TRK_ERR_CUDA), so each table covers both sides of each check.  The tests skip when a device is visible: the
fake addresses must never reach a launch."""
import pytest

A = 1 << 20          # a 16-byte aligned fake device address
MISALIGNED = A + 4

TOPK = dict(user_split=A, user_scale=A, user_bias=None, item_split=A, item_meta=A, n_users=10, n_items=300, d_pad=64,
            k=5, n_splits=1, item_id_offset=0, cand_score=A, cand_item=A, n_users_live=None)
TOPK_EXCL = dict(TOPK, excl_indptr=A, excl_ids=A, excl_row_map=None)
TOPK_EUCLID = dict(TOPK_EXCL, excl_indptr=None, excl_ids=None, user_half_sqnorm=A, item_half_sqnorm=A)
DENSE = dict(user_split=A, user_scale=A, user_bias=None, item_split=A, item_meta=A, n_users=10, n_items=300, d_pad=64,
             out=A, out_row_stride=300)
DENSE_EUCLID = dict(DENSE, user_half_sqnorm=A, item_half_sqnorm=A)
DENSE_TASTES = dict(user_split=A, user_scale=A, user_bias=None, n_tastes=2, attention=0, item_split=A, item_meta=A,
                    n_users=10, n_items=300, d_pad=64, out=A, out_row_stride=300)
TOPK_TASTES = dict(user_split=A, user_scale=A, user_bias=None, n_tastes=2, attention=0, item_split=A, item_meta=A,
                   n_users=10, n_items=300, d_pad=64, k=5, n_splits=1, item_id_offset=0, cand_score=A, cand_item=A,
                   excl_indptr=None, excl_ids=None, excl_row_map=None)

ENTRY = {
    'trk_score_topk_f16x3': TOPK,
    'trk_score_topk_f16x3_excl': TOPK_EXCL,
    'trk_score_topk_euclid_f16x3': TOPK_EUCLID,
    'trk_score_dense_f16x3': DENSE,
    'trk_score_dense_euclid_f16x3': DENSE_EUCLID,
    'trk_score_dense_tastes_f16x3': DENSE_TASTES,
    'trk_score_topk_tastes_f16x3': TOPK_TASTES,
}

# valid calls: every check passes (TRK_ERR_CUDA from the tensor-map encode)
VALID = [
    ('trk_score_topk_f16x3', {}),
    ('trk_score_topk_f16x3', dict(d_pad=128, k=32, n_splits=3, user_bias=A, n_users_live=A)),
    ('trk_score_topk_f16x3', dict(k=1)),
    ('trk_score_topk_f16x3_excl', {}),
    ('trk_score_topk_f16x3_excl', dict(excl_row_map=A, d_pad=128)),
    ('trk_score_topk_euclid_f16x3', {}),
    ('trk_score_topk_euclid_f16x3', dict(excl_indptr=A, excl_ids=A, excl_row_map=A)),
    ('trk_score_dense_f16x3', {}),
    ('trk_score_dense_f16x3', dict(out=MISALIGNED, out_row_stride=301, d_pad=128)),   # the direct-store path
    ('trk_score_dense_euclid_f16x3', {}),
    ('trk_score_dense_tastes_f16x3', {}),
    ('trk_score_dense_tastes_f16x3', dict(n_tastes=1, attention=1)),
    ('trk_score_dense_tastes_f16x3', dict(n_tastes=64)),
    ('trk_score_dense_tastes_f16x3', dict(n_tastes=32, attention=1, d_pad=128)),
    ('trk_score_topk_tastes_f16x3', dict(n_tastes=32, attention=1)),
    ('trk_score_topk_tastes_f16x3', dict(excl_indptr=A, excl_ids=A, excl_row_map=A)),
]

# one fault each: (entry point, fault, return code name, a substring of trk_last_error())
FAULTS = [
    ('trk_score_topk_f16x3', dict(k=33), 'TRK_ERR_UNSUPPORTED', 'k=33'),
    ('trk_score_topk_f16x3', dict(k=0), 'TRK_ERR_UNSUPPORTED', 'k=0'),
    ('trk_score_topk_f16x3', dict(d_pad=96), 'TRK_ERR_UNSUPPORTED', 'd_pad=96'),
    ('trk_score_dense_f16x3', dict(d_pad=96), 'TRK_ERR_UNSUPPORTED', 'd_pad=96'),
    ('trk_score_dense_tastes_f16x3', dict(n_tastes=65), 'TRK_ERR_UNSUPPORTED', 'exceed'),
    ('trk_score_topk_tastes_f16x3', dict(n_tastes=33, attention=1), 'TRK_ERR_UNSUPPORTED', 'exceed'),
    ('trk_score_topk_tastes_f16x3', dict(k=33), 'TRK_ERR_UNSUPPORTED', 'k=33'),
    ('trk_score_topk_f16x3', dict(user_split=None), 'TRK_ERR_ARG', 'null operand'),
    ('trk_score_topk_f16x3', dict(user_scale=None), 'TRK_ERR_ARG', 'null operand'),
    ('trk_score_dense_f16x3', dict(item_meta=None), 'TRK_ERR_ARG', 'null operand'),
    ('trk_score_topk_tastes_f16x3', dict(item_split=None), 'TRK_ERR_ARG', 'null operand'),
    ('trk_score_topk_f16x3', dict(user_split=MISALIGNED), 'TRK_ERR_ARG', '16-byte aligned'),
    ('trk_score_dense_f16x3', dict(item_meta=MISALIGNED), 'TRK_ERR_ARG', '16-byte aligned'),
    ('trk_score_topk_f16x3', dict(n_users=0), 'TRK_ERR_ARG', 'empty shape'),
    ('trk_score_dense_f16x3', dict(n_items=0, out_row_stride=0), 'TRK_ERR_ARG', 'empty shape'),
    ('trk_score_topk_f16x3', dict(n_items=(1 << 31) - 512), 'TRK_ERR_ARG', 'int32 indexing'),
    ('trk_score_topk_f16x3', dict(cand_item=None), 'TRK_ERR_ARG', 'null output'),
    ('trk_score_topk_f16x3', dict(n_splits=0), 'TRK_ERR_ARG', 'n_splits'),
    ('trk_score_topk_f16x3_excl', dict(excl_ids=None), 'TRK_ERR_ARG', 'trk_score_topk_f16x3_excl: null exclusion list'),
    ('trk_score_topk_f16x3_excl', dict(excl_indptr=None), 'TRK_ERR_ARG', 'trk_score_topk_f16x3_excl: null exclusion list'),
    ('trk_score_topk_euclid_f16x3', dict(excl_ids=A), 'TRK_ERR_ARG', 'go together'),
    ('trk_score_topk_euclid_f16x3', dict(excl_row_map=A), 'TRK_ERR_ARG', 'go together'),
    ('trk_score_topk_euclid_f16x3', dict(item_half_sqnorm=None), 'TRK_ERR_ARG', 'trk_score_topk_euclid_f16x3: null'),
    ('trk_score_topk_euclid_f16x3', dict(item_half_sqnorm=MISALIGNED), 'TRK_ERR_ARG', 'item_half_sqnorm must be'),
    ('trk_score_dense_euclid_f16x3', dict(user_half_sqnorm=None), 'TRK_ERR_ARG', 'trk_score_dense_euclid_f16x3: null'),
    ('trk_score_dense_f16x3', dict(out_row_stride=299), 'TRK_ERR_ARG', 'bad output'),
    ('trk_score_dense_f16x3', dict(out=None), 'TRK_ERR_ARG', 'bad output'),
    ('trk_score_dense_tastes_f16x3', dict(n_tastes=0), 'TRK_ERR_ARG', 'n_tastes=0'),
    ('trk_score_topk_tastes_f16x3', dict(n_tastes=-1), 'TRK_ERR_ARG', 'n_tastes=-1'),
    ('trk_score_dense_tastes_f16x3', dict(n_tastes=1), 'TRK_ERR_ARG', 'n_tastes=1'),
    ('trk_score_topk_tastes_f16x3', dict(n_tastes=1), 'TRK_ERR_ARG', 'n_tastes=1'),
    ('trk_score_dense_tastes_f16x3', dict(out_row_stride=299), 'TRK_ERR_ARG', 'bad output'),
    ('trk_score_topk_tastes_f16x3', dict(excl_row_map=A), 'TRK_ERR_ARG', 'go together'),
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
