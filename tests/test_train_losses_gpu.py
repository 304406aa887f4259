"""GPU tests of the serial-loss training step (RMSELossGraph, SeparationLossGraph; DESIGN §3.11) against the step
oracle (tests/train_step_oracle.serial_loss_step_reference, pinned on the CPU against torch autograd over the host
mirror: tests/test_train_losses_cpu.py): every prediction, representation and taste form, bf16 representations, Adam
over every weight, fit() on TensorRec()'s default model and the reference's examples, and degenerate batches
(interaction-free, one-sided, empty) with the torch path's finite / NaN pattern."""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import loss_ops
from tests.helpers import csr_order, kernel_step, make_serial_model, make_weights, rough_interactions
from tests.train_step_oracle import serial_loss_step_reference

pytestmark = pytest.mark.gpu
F32 = np.float32


@pytest.fixture(scope='module')
def T():
    import torch
    import tensorrec_b200
    from tensorrec_b200 import kernels, session_management as sm
    kernels.require_cuda()
    torch.cuda.set_device(0)
    sm.set_session(None)
    return tensorrec_b200


CASES = [  # loss, prediction, user_norm, item_norm, n_tastes, attention, biased, d
    ('rmse', 'dot', False, False, 1, False, True, 5),
    ('separation', 'dot', True, False, 1, False, True, 10),
    ('rmse', 'cosine', False, False, 1, False, False, 10),
    ('separation', 'cosine', True, True, 1, False, True, 128),
    ('rmse', 'euclidean', False, False, 1, False, True, 10),
    ('separation', 'euclidean', True, False, 1, False, False, 200),
    ('rmse', 'cosine', False, False, 1, False, True, 300),
    ('separation', 'dot', False, False, 1, False, True, 512),
    ('rmse', 'dot', True, False, 3, False, True, 10),
    ('separation', 'cosine', True, True, 3, False, True, 128),
    ('rmse', 'euclidean', False, True, 3, False, True, 5),
    ('separation', 'dot', True, False, 3, True, True, 10),
    ('rmse', 'cosine', False, False, 3, True, False, 128),
    ('separation', 'euclidean', True, False, 3, True, True, 10),
    ('rmse', 'dot', False, False, 8, False, True, 128),
    ('separation', 'euclidean', False, False, 4, True, True, 128),
]


@pytest.mark.parametrize('loss,prediction,user_norm,item_norm,n_tastes,attention,biased,d', CASES)
def test_kernel_step_matches_the_oracle_fp32(T, loss, prediction, user_norm, item_norm, n_tastes, attention, biased, d):
    interactions, uf, itf = rough_interactions(260, 230, seed=d + n_tastes, density=0.05)
    weights = make_weights(uf, itf, d, n_tastes, attention, biased, seed=d + 100)
    normalize = [side for side, on in (('user', user_norm), ('item', item_norm)) if on]
    ref = serial_loss_step_reference(uf, itf, interactions, weights, loss=loss, prediction=prediction,
                                     normalize=normalize, n_tastes=n_tastes, attention=attention)
    model = make_serial_model(loss, prediction, user_norm, item_norm, n_tastes, attention, biased, d)
    stepper, out, pred = kernel_step(model, weights, interactions, uf, itf)
    assert out.shape == (1,)
    value = float(out[0])
    order = csr_order(interactions)
    assert np.allclose(pred, ref['pred_serial'][order], rtol=2e-5, atol=2e-6)
    assert np.isfinite(value) and np.isclose(value, ref['loss'], rtol=1e-4, atol=1e-6)
    g = {k: v.cpu().numpy().reshape(ref['grads'][k].shape) for k, v in stepper.last['grads'].items()}
    assert set(g) == set(ref['grads'])
    for name, exp in ref['grads'].items():
        scale = float(np.abs(exp).max())
        assert np.allclose(g[name], exp, rtol=1e-3, atol=1e-4 * scale), name


@pytest.mark.parametrize('loss,prediction,n_tastes,attention', [('rmse', 'dot', 1, False),
                                                                ('separation', 'euclidean', 3, True)])
def test_kernel_step_bf16_representations(T, loss, prediction, n_tastes, attention):
    interactions, uf, itf = rough_interactions(260, 230, seed=3, density=0.05)
    weights = make_weights(uf, itf, 128, n_tastes, attention, True, seed=9)
    kw = dict(loss=loss, prediction=prediction, normalize=['user'], n_tastes=n_tastes, attention=attention)
    ref = serial_loss_step_reference(uf, itf, interactions, weights, round_repr=loss_ops.round_to_bfloat16, **kw)
    model = make_serial_model(loss, prediction, True, False, n_tastes, attention, True, 128)
    stepper, out, pred = kernel_step(model, weights, interactions, uf, itf, bf16=True)
    assert out.shape == (1,)
    value = float(out[0])
    order = csr_order(interactions)
    err = np.abs(pred - ref['pred_serial'][order])
    assert np.mean(err <= 2e-5 * np.abs(pred) + 2e-6) > 0.9 and err.max() < 0.02
    assert np.isclose(value, ref['loss'], rtol=1e-3)
    for name in ('linear_weights_item', 'linear_weights_user_0'):
        g = stepper.last['grads'][name].cpu().numpy()
        exp = ref['grads'][name]
        scale = float(np.abs(exp).max())
        assert np.abs(g - exp).max() < 5e-3 * scale, name
        assert np.mean(np.abs(g - exp) <= 1e-3 * np.abs(exp) + 1e-4 * scale) > 0.9, name


@pytest.mark.parametrize('loss', ['rmse', 'separation'])
def test_two_adam_steps_over_every_weight_match_the_oracle(T, loss):
    from tensorrec_b200.input_utils import SparseInput
    interactions, uf, itf = rough_interactions(120, 90, seed=9)
    weights = make_weights(uf, itf, 10, 3, True, True, seed=5)
    lr, l2 = 0.1, 0.3
    model = make_serial_model(loss, 'cosine', True, False, 3, True, True, 10)
    stepper, out, _ = kernel_step(model, weights, interactions, uf, itf, lr=lr, l2=l2)
    assert out.shape == (1,)
    w1 = model.get_weights()
    g1 = {k: v.cpu().numpy().reshape(weights[k].shape) for k, v in stepper.last['grads'].items()}
    assert set(w1) == set(weights)
    moments = {}
    for name, w0 in weights.items():
        exp, m, v = loss_ops.adam_reference(w0, g1[name], np.zeros_like(w0), np.zeros_like(w0), 1, lr, l2=l2)
        assert np.allclose(w1[name], exp, rtol=1e-6, atol=1e-7), name
        moments[name] = (m, v)
    stepper.step(SparseInput(interactions), SparseInput(uf), SparseInput(itf), None, lr, l2)
    w2 = model.get_weights()
    for name in weights:
        g2 = stepper.last['grads'][name].cpu().numpy().reshape(weights[name].shape)
        exp, _, _ = loss_ops.adam_reference(w1[name], g2, *moments[name], 2, lr, l2=l2)
        assert np.allclose(w2[name], exp, rtol=1e-5, atol=1e-6), name


def test_fit_on_the_default_and_example_models_takes_the_kernel_path_and_learns(T):
    from tensorrec_b200 import util
    from tensorrec_b200.loss_graphs import SeparationLossGraph
    interactions, uf, itf = util.generate_dummy_data(num_users=200, num_items=300, interaction_density=.05, seed=4)
    models = [T.TensorRec(), T.TensorRec(n_components=5), T.TensorRec(n_components=5, loss_graph=SeparationLossGraph())]
    for model in models:
        model.fit(interactions, uf, itf, epochs=1, learning_rate=0.01)
        assert model._wmrb_step is not None and model._wmrb_step.t == 1, 'the kernel training path was not taken'
        first = float(model._wmrb_step.last['loss'][0])
        model.fit_partial(interactions, uf, itf, epochs=30, learning_rate=0.01)
        assert model._wmrb_step.t == 31
        assert float(model._wmrb_step.last['loss'][0]) < first


def fit_both(T, monkeypatch, make, weights, interactions, uf, itf, **kw):
    """The weights after fit_partial from the same starting weights on the kernel path and on the torch path."""
    from tensorrec_b200 import train_kernels
    out = []
    for path in ('auto', 'torch'):
        monkeypatch.setattr(train_kernels, 'TRAIN_PATH', path)
        model = make()
        model.set_weights(weights)
        model.fit_partial(interactions, uf, itf, **kw)
        assert (getattr(model, '_wmrb_step', None) is not None) == (path == 'auto')
        out.append(model.get_weights())
    return out


def assert_same_pattern(kernel, torch_path, lr, n_steps):
    """The same NaN entries per weight, and the same finite values: almost everywhere within 0.2 % of the distance the
    Adam steps can move a weight (Adam divides the float rounding of a gradient by the gradient's own size, and torch's
    Adam places epsilon differently from TensorFlow's), and everywhere within that distance (an entry whose gradient
    is near 0 moves by about +-lr on either path, with the sign of its rounding)."""
    assert set(kernel) == set(torch_path)
    for name in kernel:
        a, b = kernel[name], torch_path[name]
        assert np.array_equal(np.isnan(a), np.isnan(b)), name
        finite = ~np.isnan(a)
        err = np.abs(a[finite] - b[finite])
        if err.size:
            assert np.mean(err <= 2e-3 * lr * n_steps + 1e-5 * np.abs(b[finite])) > 0.99, name
            assert err.max() <= lr * n_steps, name


def test_one_fit_from_identical_weights_agrees_on_both_paths(T, monkeypatch):
    from tensorrec_b200.loss_graphs import RMSELossGraph, SeparationLossGraph
    interactions, uf, itf = rough_interactions(80, 60, seed=12)
    for lg in (RMSELossGraph, SeparationLossGraph):
        weights = make_weights(uf, itf, 8, 2, False, True, seed=1)
        make = lambda: T.TensorRec(n_components=8, n_tastes=2, loss_graph=lg())  # noqa: E731
        k, t = fit_both(T, monkeypatch, make, weights, interactions, uf, itf, epochs=2, learning_rate=0.01,
                        alpha=0.1, user_batch_size=40)
        assert all(np.all(np.isfinite(v)) for v in k.values())
        assert_same_pattern(k, t, 0.01, 4)


def test_degenerate_batches_match_the_torch_path_without_a_fault(T, monkeypatch):
    import torch
    from tensorrec_b200.loss_graphs import RMSELossGraph, SeparationLossGraph
    interactions, uf, itf = rough_interactions(60, 50, seed=6)
    coo = sp.coo_matrix(interactions)
    weights = make_weights(uf, itf, 8, 1, False, True, seed=2)
    kw = dict(epochs=1, learning_rate=0.01, alpha=0.1)
    for lg in (RMSELossGraph, SeparationLossGraph):
        make = lambda: T.TensorRec(n_components=8, loss_graph=lg())  # noqa: E731
        # a user batch without interactions: users [0, 20) have none
        keep = coo.row >= 20
        sparse_head = sp.coo_matrix((coo.data[keep], (coo.row[keep], coo.col[keep])), shape=coo.shape)
        k, t = fit_both(T, monkeypatch, make, weights, sparse_head, uf, itf, user_batch_size=20, **kw)
        assert all(np.all(np.isfinite(v)) for v in k.values())
        assert_same_pattern(k, t, 0.01, 3)
        # no interaction at all: NaN loss, an Adam step on the L2 term alone
        empty = sp.coo_matrix(coo.shape, dtype=np.float32)
        k, t = fit_both(T, monkeypatch, make, weights, empty, uf, itf, **kw)
        assert all(np.all(np.isfinite(v)) for v in k.values())
        assert_same_pattern(k, t, 0.01, 1)
    # a Separation batch whose interactions are all positive: NaN on the rows they touch
    positive = sp.coo_matrix((np.abs(coo.data) + 1.0, (coo.row, coo.col)), shape=coo.shape)
    keep = positive.row < 30
    positive = sp.coo_matrix((positive.data[keep], (positive.row[keep], positive.col[keep])), shape=coo.shape)
    make = lambda: T.TensorRec(n_components=8, loss_graph=SeparationLossGraph())  # noqa: E731
    k, t = fit_both(T, monkeypatch, make, weights, positive, uf, itf, **kw)
    assert np.any(np.isnan(k['linear_weights_user_0'])) and np.any(np.isnan(k['linear_weights_item']))
    assert_same_pattern(k, t, 0.01, 1)
    torch.cuda.synchronize()
