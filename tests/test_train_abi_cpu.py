"""CPU tests of the argument checks of the training step's three C entry points (trk_wmrb_step, trk_wmrb_step_tastes,
trk_serial_loss_step).

Every case is an otherwise valid call with one fault, made through ctypes on small 16-byte aligned host buffers that
no check dereferences.  Each call is either rejected by a check or, for the two WMRB entry points, returns at
n_users = 0 before any CUDA call, so the tests run with or without a device and never reach a kernel.  The accepted
side of a bound is shown by n_users = 0 (WMRB: TRK_OK) or by a misaligned row that only the last check rejects
(serial: the alignment message instead of the bound's)."""
import numpy as np
import pytest

_BLOCK = np.zeros(64, np.float32)
A = (_BLOCK.ctypes.data + 15) // 16 * 16     # a 16-byte aligned host address inside _BLOCK
MISALIGNED = A + 4

WMRB = dict(user_repr=A, item_repr=A, repr_is_bf16=0, user_bias=None, item_bias=None, inter_indptr=A, inter_item=A,
            inter_val=A, item_weight_sum=None, samples=A, n_users=10, n_items=300, d=64, n_sampled=16, loss=A,
            pred_serial=A, coef=A, d_user_repr=A, d_user_bias=None, d_item_repr=A, d_item_bias=None)
TASTES = dict(user_rows=A, item_repr=A, repr_is_bf16=0, n_tastes=2, attention=0, euclidean=0, user_bias=None,
              item_bias=None, inter_indptr=A, inter_item=A, inter_val=A, item_weight_sum=None, samples=A, n_users=10,
              n_items=300, d=64, n_sampled=16, loss=A, pred_serial=A, coef=A, d_user_rows=A, d_user_bias=None,
              d_item_repr=A, d_item_bias=None)
SERIAL = dict(loss_kind=0, user_rows=A, item_repr=A, repr_is_bf16=0, n_tastes=2, attention=0, euclidean=0,
              user_bias=None, item_bias=None, inter_indptr=A, inter_item=A, inter_val=A, n_users=10, n_items=300, d=64,
              nnz=20, loss=A, pred_serial=A, d_user_rows=A, d_user_bias=None, d_item_repr=A, d_item_bias=None,
              workspace=A, workspace_bytes=1 << 20)

ENTRY = {'trk_wmrb_step': WMRB, 'trk_wmrb_step_tastes': TASTES, 'trk_serial_loss_step': SERIAL}
PREFIX = {'trk_wmrb_step': 'wmrb_step:', 'trk_wmrb_step_tastes': 'wmrb_step_tastes:',
          'trk_serial_loss_step': 'serial_loss_step:'}
BIASED = dict(user_bias=A, item_bias=A, d_user_bias=A, d_item_bias=A)
EMPTY = dict(n_users=0)                   # WMRB: every check passed, nothing to do
LATE = dict(item_repr=MISALIGNED)         # serial: every check passed up to the alignment of the rows

# accepted: (entry point, arguments); the WMRB calls return TRK_OK at n_users = 0
ACCEPTED = [
    ('trk_wmrb_step', {}),
    ('trk_wmrb_step', BIASED),
    ('trk_wmrb_step', dict(d=512, n_sampled=2048, repr_is_bf16=1)),
    ('trk_wmrb_step', dict(d=4, n_sampled=1, n_items=(1 << 31) - 1)),
    ('trk_wmrb_step_tastes', {}),
    ('trk_wmrb_step_tastes', BIASED),
    ('trk_wmrb_step_tastes', dict(n_tastes=1, d=512, n_sampled=2048, euclidean=1)),
    ('trk_wmrb_step_tastes', dict(n_tastes=8, d=128)),
    ('trk_wmrb_step_tastes', dict(n_tastes=2, attention=1)),
    ('trk_wmrb_step_tastes', dict(n_tastes=4, attention=1, d=128, euclidean=1, repr_is_bf16=1)),
]

# one fault each: (entry point, fault, return code name, a substring of trk_last_error())
FAULTS = [
    # nulls
    ('trk_wmrb_step', dict(user_repr=None), 'TRK_ERR_ARG', 'null input'),
    ('trk_wmrb_step', dict(samples=None), 'TRK_ERR_ARG', 'null input'),
    ('trk_wmrb_step', dict(inter_indptr=None), 'TRK_ERR_ARG', 'null input'),
    ('trk_wmrb_step', dict(coef=None), 'TRK_ERR_ARG', 'null output'),
    ('trk_wmrb_step', dict(d_item_repr=None), 'TRK_ERR_ARG', 'null output'),
    ('trk_wmrb_step_tastes', dict(item_repr=None), 'TRK_ERR_ARG', 'null input'),
    ('trk_wmrb_step_tastes', dict(samples=None), 'TRK_ERR_ARG', 'null input'),
    ('trk_wmrb_step_tastes', dict(loss=None), 'TRK_ERR_ARG', 'null output'),
    ('trk_wmrb_step_tastes', dict(d_user_rows=None), 'TRK_ERR_ARG', 'null output'),
    ('trk_serial_loss_step', dict(item_repr=None), 'TRK_ERR_ARG', 'null item operand'),
    ('trk_serial_loss_step', dict(loss=None), 'TRK_ERR_ARG', 'null item operand'),
    ('trk_serial_loss_step', dict(user_rows=None), 'TRK_ERR_ARG', 'null user operand'),
    ('trk_serial_loss_step', dict(inter_val=None), 'TRK_ERR_ARG', 'null interaction'),
    ('trk_serial_loss_step', dict(pred_serial=None), 'TRK_ERR_ARG', 'null interaction'),
    ('trk_serial_loss_step', dict(workspace=None), 'TRK_ERR_ARG', 'null interaction'),
    # unpaired biases and bias gradients
    ('trk_wmrb_step', dict(user_bias=A, d_user_bias=A), 'TRK_ERR_ARG', 'given together'),
    ('trk_wmrb_step', dict(BIASED, d_item_bias=None), 'TRK_ERR_ARG', 'bias gradients'),
    ('trk_wmrb_step_tastes', dict(item_bias=A, d_item_bias=A), 'TRK_ERR_ARG', 'given together'),
    ('trk_wmrb_step_tastes', dict(BIASED, d_user_bias=None), 'TRK_ERR_ARG', 'bias gradients'),
    ('trk_wmrb_step_tastes', dict(d_user_bias=A), 'TRK_ERR_ARG', 'bias gradients'),
    ('trk_serial_loss_step', dict(user_bias=A, d_user_bias=A), 'TRK_ERR_ARG', 'given together'),
    ('trk_serial_loss_step', dict(BIASED, d_item_bias=None), 'TRK_ERR_ARG', 'bias gradients'),
    # misaligned rows
    ('trk_wmrb_step', dict(user_repr=MISALIGNED), 'TRK_ERR_ARG', '16-byte aligned'),
    ('trk_wmrb_step', dict(d_item_repr=MISALIGNED), 'TRK_ERR_ARG', '16-byte aligned'),
    ('trk_wmrb_step_tastes', dict(item_repr=MISALIGNED), 'TRK_ERR_ARG', '16-byte aligned'),
    ('trk_wmrb_step_tastes', dict(d_user_rows=MISALIGNED), 'TRK_ERR_ARG', '16-byte aligned'),
    ('trk_serial_loss_step', dict(user_rows=MISALIGNED), 'TRK_ERR_ARG', '16-byte aligned'),
    ('trk_serial_loss_step', dict(d_item_repr=MISALIGNED), 'TRK_ERR_ARG', '16-byte aligned'),
    # flags
    ('trk_wmrb_step_tastes', dict(attention=2), 'TRK_ERR_ARG', 'flags'),
    ('trk_wmrb_step_tastes', dict(euclidean=-1), 'TRK_ERR_ARG', 'flags'),
    ('trk_serial_loss_step', dict(attention=-1), 'TRK_ERR_ARG', 'flags'),
    ('trk_serial_loss_step', dict(euclidean=2), 'TRK_ERR_ARG', 'flags'),
    # sizes
    ('trk_wmrb_step', dict(n_items=0), 'TRK_ERR_ARG', 'bad sizes'),
    ('trk_wmrb_step', dict(n_items=1 << 31), 'TRK_ERR_ARG', 'bad sizes'),
    ('trk_wmrb_step', dict(n_users=-1), 'TRK_ERR_ARG', 'bad sizes'),
    ('trk_wmrb_step', dict(n_sampled=0), 'TRK_ERR_ARG', 'bad sizes'),
    ('trk_wmrb_step_tastes', dict(n_tastes=0), 'TRK_ERR_ARG', 'bad sizes'),
    ('trk_wmrb_step_tastes', dict(n_items=1 << 31), 'TRK_ERR_ARG', 'bad sizes'),
    ('trk_wmrb_step_tastes', dict(n_sampled=0), 'TRK_ERR_ARG', 'bad sizes'),
    ('trk_serial_loss_step', dict(n_tastes=0), 'TRK_ERR_ARG', 'bad sizes'),
    ('trk_serial_loss_step', dict(n_items=0), 'TRK_ERR_ARG', 'bad sizes'),
    ('trk_serial_loss_step', dict(nnz=-1), 'TRK_ERR_ARG', 'bad sizes'),
    ('trk_serial_loss_step', dict(nnz=1 << 31), 'TRK_ERR_ARG', 'bad sizes'),
    ('trk_serial_loss_step', dict(n_users=0), 'TRK_ERR_ARG', 'bad sizes'),      # interactions without users
    # the serial step's own arguments
    ('trk_serial_loss_step', dict(loss_kind=2), 'TRK_ERR_ARG', 'unknown loss'),
    ('trk_serial_loss_step', dict(loss_kind=-1), 'TRK_ERR_ARG', 'unknown loss'),
    ('trk_serial_loss_step', dict(workspace_bytes=16), 'TRK_ERR_ARG', 'workspace'),
    ('trk_serial_loss_step', dict(workspace=A + 4), 'TRK_ERR_ARG', 'workspace'),
    # form limits, the rejected side (the accepted side: ACCEPTED and SERIAL_ACCEPTED)
    ('trk_wmrb_step', dict(d=516), 'TRK_ERR_UNSUPPORTED', 'n_components=516'),
    ('trk_wmrb_step', dict(d=0), 'TRK_ERR_UNSUPPORTED', 'n_components=0'),
    ('trk_wmrb_step', dict(d=6), 'TRK_ERR_UNSUPPORTED', 'n_components=6'),
    ('trk_wmrb_step', dict(n_sampled=2049), 'TRK_ERR_UNSUPPORTED', 'n_sampled=2049'),
    ('trk_wmrb_step_tastes', dict(n_tastes=1, d=516), 'TRK_ERR_UNSUPPORTED', 'n_components=516'),
    ('trk_wmrb_step_tastes', dict(n_tastes=2, d=132), 'TRK_ERR_UNSUPPORTED', 'n_components=132'),
    ('trk_wmrb_step_tastes', dict(d=10), 'TRK_ERR_UNSUPPORTED', 'n_components=10'),
    ('trk_wmrb_step_tastes', dict(n_tastes=9), 'TRK_ERR_UNSUPPORTED', 'n_tastes=9'),
    ('trk_wmrb_step_tastes', dict(n_tastes=5, attention=1), 'TRK_ERR_UNSUPPORTED', 'n_tastes=5'),
    ('trk_wmrb_step_tastes', dict(n_tastes=1, attention=1), 'TRK_ERR_UNSUPPORTED', 'n_tastes=1'),
    ('trk_wmrb_step_tastes', dict(n_sampled=2049), 'TRK_ERR_UNSUPPORTED', 'n_sampled=2049'),
    ('trk_serial_loss_step', dict(n_tastes=1, d=516), 'TRK_ERR_UNSUPPORTED', 'n_components=516'),
    ('trk_serial_loss_step', dict(n_tastes=2, d=132), 'TRK_ERR_UNSUPPORTED', 'n_components=132'),
    ('trk_serial_loss_step', dict(d=2), 'TRK_ERR_UNSUPPORTED', 'n_components=2'),
    ('trk_serial_loss_step', dict(n_tastes=9), 'TRK_ERR_UNSUPPORTED', 'n_tastes=9'),
    ('trk_serial_loss_step', dict(n_tastes=5, attention=1), 'TRK_ERR_UNSUPPORTED', 'n_tastes=5'),
    ('trk_serial_loss_step', dict(n_tastes=1, attention=1), 'TRK_ERR_UNSUPPORTED', 'n_tastes=1'),
]

# the serial step's accepted side of each bound: the form check passes and the rows' alignment is what rejects
SERIAL_ACCEPTED = [
    dict(n_tastes=1, d=512),
    dict(n_tastes=8, d=128),
    dict(n_tastes=4, attention=1, d=128, euclidean=1),
    dict(n_tastes=2, attention=1, d=4, loss_kind=1, repr_is_bf16=1),
    dict(BIASED, nnz=(1 << 31) - 1, n_items=(1 << 31) - 1, workspace_bytes=1 << 20),
]


@pytest.fixture(scope='module')
def lib():
    from tensorrec_b200 import _lib
    return _lib.load()


def call(lib, entry, fault):
    args = dict(ENTRY[entry])
    assert set(fault) <= set(args), fault
    args.update(fault)
    return getattr(lib, entry)(*args.values(), None)   # (the stream)


@pytest.mark.parametrize('entry,args', ACCEPTED, ids=['%s-%d' % (e, i) for i, (e, _) in enumerate(ACCEPTED)])
def test_valid_wmrb_calls_without_users_return_ok(lib, entry, args):
    from tensorrec_b200 import _lib
    assert call(lib, entry, dict(args, **EMPTY)) == _lib.TRK_OK, _lib.last_error()


@pytest.mark.parametrize('args', SERIAL_ACCEPTED, ids=[str(i) for i in range(len(SERIAL_ACCEPTED))])
def test_valid_serial_calls_pass_every_check_up_to_the_row_alignment(lib, args):
    from tensorrec_b200 import _lib
    assert call(lib, 'trk_serial_loss_step', dict(args, **LATE)) == _lib.TRK_ERR_ARG
    assert 'serial_loss_step: rows must be 16-byte aligned' in _lib.last_error()


@pytest.mark.parametrize('entry,fault,rc,message', FAULTS,
                         ids=['%s-%s' % (e, '-'.join('%s=%s' % kv for kv in f.items())) for e, f, _, _ in FAULTS])
def test_each_fault_is_rejected_with_the_entry_points_name(lib, entry, fault, rc, message):
    from tensorrec_b200 import _lib
    assert call(lib, entry, fault) == getattr(_lib, rc)
    err = _lib.last_error()
    assert err.startswith(PREFIX[entry]) and message in err, err


def test_every_entry_point_is_covered():
    assert {e for e, _ in ACCEPTED} | {'trk_serial_loss_step'} == set(ENTRY) == {e for e, _, _, _ in FAULTS}
