"""CPU tests of the serial-loss training step (RMSELossGraph, SeparationLossGraph; DESIGN §3.11): the step oracle
(tests/train_step_oracle.serial_loss_step_reference) equals torch autograd over the host mirror of the reference's
graph functions for every form the step covers, on interactions with explicit zeros, duplicates and negative values;
step_plan gives exactly the stated models a serial loss and the WMRB models the answers they had; the L2 coefficient
of a scalar loss is batched_alpha."""
import itertools

import numpy as np
import pytest
import torch

import tensorrec_b200 as T
from tensorrec_b200 import train_kernels, util
from tensorrec_b200.loss_graphs import (BalancedWMRBLossGraph, RMSEDenseLossGraph, RMSELossGraph,
                                        SeparationDenseLossGraph, SeparationLossGraph, WMRBLossGraph)
from tensorrec_b200.prediction_graphs import (CosineSimilarityPredictionGraph, DotProductPredictionGraph,
                                              EuclideanSimilarityPredictionGraph)
from tensorrec_b200.representation_graphs import (LinearRepresentationGraph, NormalizedLinearRepresentationGraph,
                                                  ReLURepresentationGraph)
from tests.helpers import make_serial_model, make_weights, rough_interactions
from tests.train_step_oracle import serial_loss_coefficients, serial_loss_step_reference

PREDICTIONS = {'dot': DotProductPredictionGraph, 'cosine': CosineSimilarityPredictionGraph,
               'euclidean': EuclideanSimilarityPredictionGraph}
LOSSES = {'rmse': RMSELossGraph, 'separation': SeparationLossGraph}


@pytest.fixture
def cpu_session():
    from tensorrec_b200 import session_management as sm
    sm.set_session(sm.Session('cpu'))
    yield
    sm.set_session(None)


def autograd_of_the_mirror(model, weights, interactions, uf, itf):
    """The torch path's loss, serial predictions and weight gradients (no L2 term)."""
    from tensorrec_b200.input_utils import SparseInput
    from tensorrec_b200.session_management import variable_scope
    model.set_weights(weights)
    with variable_scope(model._variables):
        basic_loss, _, pred_serial, _ = model._training_losses(SparseInput(interactions), SparseInput(uf),
                                                               SparseInput(itf), None, torch.device('cpu'))
    basic_loss.backward()
    return (float(basic_loss.detach()), pred_serial.detach().numpy(),
            {k: v.grad.detach().numpy() for k, v in model._variables.items()})


# every factor at both levels, trimmed to combinations that exercise each one
GRID = [(loss, p, un, inn, nt, att, bia)
        for loss, p, un, inn, nt, att, bia in itertools.product(LOSSES, PREDICTIONS, (False, True), (False, True),
                                                                (1, 3), (False, True), (True, False))
        if not (att and nt == 1) and (un == inn or nt == 1) and (bia or p != 'dot')]


@pytest.mark.parametrize('loss,prediction,user_norm,item_norm,n_tastes,attention,biased', GRID)
def test_serial_oracle_equals_autograd_of_the_host_mirror(cpu_session, loss, prediction, user_norm, item_norm,
                                                          n_tastes, attention, biased):
    d = 6
    interactions, uf, itf = rough_interactions(30, 40, seed=2)
    weights = make_weights(uf, itf, d, n_tastes, attention, biased, seed=11)
    normalize = [side for side, on in (('user', user_norm), ('item', item_norm)) if on]
    ref = serial_loss_step_reference(uf, itf, interactions, weights, loss=loss, prediction=prediction,
                                     normalize=normalize, n_tastes=n_tastes, attention=attention)
    model = make_serial_model(loss, prediction, user_norm, item_norm, n_tastes, attention, biased, d)
    value, pred, grads = autograd_of_the_mirror(model, weights, interactions, uf, itf)
    assert np.isfinite(ref['loss']) and np.isclose(value, ref['loss'], rtol=2e-5, atol=2e-6)
    assert np.allclose(pred, ref['pred_serial'], rtol=2e-5, atol=2e-6)
    assert set(grads) == set(ref['grads'])
    for name, g in grads.items():
        scale = max(1e-3, float(np.abs(ref['grads'][name]).max()))
        assert np.allclose(g, ref['grads'][name], rtol=2e-3, atol=2e-4 * scale), name


@pytest.mark.parametrize('loss', list(LOSSES))
def test_loss_coefficients_equal_autograd_of_the_loss_graph(loss):
    rng = np.random.default_rng(4)
    pred = rng.standard_normal(200).astype(np.float32)
    val = np.where(rng.random(200) < 0.5, rng.random(200) + 0.1, -rng.random(200)).astype(np.float32)
    val[::7] = 0.0
    p = torch.from_numpy(pred.copy()).requires_grad_(True)
    out = LOSSES[loss]().connect_loss_graph(tf_prediction_serial=p, tf_interactions_serial=torch.from_numpy(val))
    out.backward()
    value, g = serial_loss_coefficients(pred, val, loss)
    assert np.isclose(float(out.detach()), value, rtol=1e-5)
    assert np.allclose(p.grad.numpy(), g, rtol=1e-4, atol=1e-7)


def test_degenerate_coefficients_are_nan_as_the_loss_graphs_give():
    empty = np.zeros(0, np.float32)
    for loss in LOSSES:
        value, g = serial_loss_coefficients(empty, empty, loss)
        assert np.isnan(value) and g.shape == (0,)
    pred = np.array([0.5, 1.0, -0.25], np.float32)
    value, g = serial_loss_coefficients(pred, np.ones(3, np.float32), 'separation')      # no y <= 0 group
    assert np.isnan(value) and np.all(np.isnan(g))
    value, g = serial_loss_coefficients(pred, pred, 'rmse')                               # L = 0
    assert value == 0.0 and np.all(np.isnan(g))
    for loss, val in (('separation', np.ones(3, np.float32)), ('rmse', pred)):
        p = torch.from_numpy(pred.copy()).requires_grad_(True)
        out = LOSSES[loss]().connect_loss_graph(tf_prediction_serial=p, tf_interactions_serial=torch.from_numpy(val))
        out.backward()
        assert np.all(np.isnan(p.grad.numpy()))


# ---- routing -------------------------------------------------------------------------------------------------
def getting_started_models():
    """TensorRec()'s default loss and the serial-loss models of the reference's examples (getting_started.py:45,
    check_movielens_losses.py)."""
    yield T.TensorRec()
    yield T.TensorRec(n_components=5)
    yield T.TensorRec(n_components=5, loss_graph=SeparationLossGraph())
    yield T.TensorRec(n_components=10, n_tastes=3, user_repr_graph=NormalizedLinearRepresentationGraph(),
                      prediction_graph=CosineSimilarityPredictionGraph(), loss_graph=SeparationLossGraph())


def test_step_plan_gives_exactly_the_serial_loss_models_a_serial_form(monkeypatch):
    monkeypatch.setattr(train_kernels, 'TRAIN_PATH', 'auto')
    for model in getting_started_models():
        form = train_kernels.step_plan(model)
        assert form is not None and form.loss in ('rmse', 'separation')
        assert form.d_pad == (model.n_components + 3) // 4 * 4
        # nothing is sampled: n_sampled_items, even beyond the WMRB step's limit, changes nothing
        assert train_kernels.step_plan(model, 10) == form and train_kernels.step_plan(model, 4096) == form
    assert train_kernels.step_plan(T.TensorRec()).loss == 'rmse'
    nl, lin = NormalizedLinearRepresentationGraph, LinearRepresentationGraph
    for loss, pred, un, inn, att, nt, d in itertools.product(LOSSES, PREDICTIONS.values(), (lin, nl), (lin, nl),
                                                             (None, lin, nl), (1, 2, 4), (1, 7, 128)):
        if att is not None and nt == 1:
            continue
        model = T.TensorRec(n_components=d, n_tastes=nt, user_repr_graph=un(), item_repr_graph=inn(),
                            attention_graph=att() if att else None, prediction_graph=pred(), loss_graph=LOSSES[loss]())
        form = train_kernels.step_plan(model)
        assert form is not None and form.loss == loss
        wmrb = train_kernels.step_plan(T.TensorRec(n_components=d, n_tastes=nt, user_repr_graph=un(),
                                                   item_repr_graph=inn(), attention_graph=att() if att else None,
                                                   prediction_graph=pred(), loss_graph=WMRBLossGraph()))
        assert form == wmrb._replace(loss=loss)            # the same operand layout as the WMRB step's
    for lg in (RMSELossGraph, SeparationLossGraph):
        ok = lambda **kw: train_kernels.step_plan(T.TensorRec(loss_graph=lg(), **kw)) is not None  # noqa
        assert ok(n_components=512) and not ok(n_components=513)
        assert ok(n_components=128, n_tastes=8) and not ok(n_components=129, n_tastes=2)
        assert not ok(n_components=8, n_tastes=9)
        assert ok(n_components=128, n_tastes=4, attention_graph=lin())
        assert not ok(n_components=8, n_tastes=5, attention_graph=lin())
        assert not ok(n_components=8, user_repr_graph=ReLURepresentationGraph())
        assert not ok(n_components=8, attention_graph=ReLURepresentationGraph(), n_tastes=2)
    for lg in (WMRBLossGraph, BalancedWMRBLossGraph):
        assert train_kernels.step_plan(T.TensorRec(n_components=8, loss_graph=lg())).loss == 'wmrb'
    for lg in (RMSEDenseLossGraph, SeparationDenseLossGraph):
        assert train_kernels.step_plan(T.TensorRec(n_components=8, loss_graph=lg())) is None
    # the sampled-rank routing keeps every answer: the serial losses never reach the WMRB step
    assert train_kernels.step_plan(T.TensorRec(n_components=8, loss_graph=RMSELossGraph())).loss == 'rmse'
    assert train_kernels.step_plan(T.TensorRec(n_components=8, loss_graph=SeparationLossGraph())).loss == 'separation'
    assert train_kernels.step_plan(T.TensorRec(n_components=8, loss_graph=WMRBLossGraph()), 64).loss == 'wmrb'
    assert train_kernels.step_plan(T.TensorRec(n_components=8, loss_graph=WMRBLossGraph()), 2049) is None
    monkeypatch.setattr(train_kernels, 'TRAIN_PATH', 'torch')
    for model in getting_started_models():
        assert train_kernels.step_plan(model) is None


def test_the_serial_step_adds_the_l2_term_once(monkeypatch, cpu_session):
    """A scalar loss: Adam's L2 coefficient is batched_alpha (the reference adds alpha * reg once), where WMRB's is
    n_positive * batched_alpha."""
    calls = []

    class Recorder(object):
        def __init__(self, model, device):
            self.device, self.t = device, 0

        def step(self, int_in, uf_in, if_in, n_sampled_items, learning_rate, l2, samples=None):
            calls.append((n_sampled_items, l2))
            self.t += 1
            return torch.zeros(1), torch.zeros(int_in.matrix.nnz)

    monkeypatch.setattr(train_kernels, 'WmrbStep', Recorder)
    monkeypatch.setattr(train_kernels, 'TRAIN_PATH', 'auto')
    interactions, uf, itf = util.generate_dummy_data(num_users=40, num_items=30, interaction_density=.2, seed=1)
    model = T.TensorRec(n_components=4)
    model.n_user_features, model.n_item_features = uf.shape[1], itf.shape[1]
    batches = model._create_batched_inputs(interactions=interactions, user_features=uf, item_features=itf,
                                           user_batch_size=10)
    alpha = 0.01
    batched_alpha = T.tensorrec.calculate_batched_alpha(num_batches=len(batches), alpha=alpha)
    model._fit_epochs(batches, 1, 0.1, alpha, batched_alpha, False, None, torch.device('cuda', 0))
    assert calls == [(None, batched_alpha)] * len(batches) and len(batches) == 4
