"""CPU tests of the fused training step's forms (DESIGN §3.10): the general step oracle
(tests/train_step_oracle.sampled_rank_step_reference) equals torch autograd over the host mirror of the reference's
graph functions for every factor the step covers, splits tied tastes evenly, the routing predicate covers exactly the
stated models, and the step's input check rejects malformed inputs before any launch."""
import itertools

import numpy as np
import pytest
import torch

from oracle import loss_ops
from tests.helpers import make_model, make_weights, reference_example_models
from tests.train_step_oracle import sampled_rank_step_reference
import tensorrec_b200 as T
from tensorrec_b200 import train_kernels, util
from tensorrec_b200.loss_graphs import RMSELossGraph, WMRBLossGraph
from tensorrec_b200.prediction_graphs import (CosineSimilarityPredictionGraph, DotProductPredictionGraph,
                                              EuclideanSimilarityPredictionGraph)
from tensorrec_b200.representation_graphs import (LinearRepresentationGraph, NormalizedLinearRepresentationGraph,
                                                  ReLURepresentationGraph)

PREDICTIONS = {'dot': DotProductPredictionGraph, 'cosine': CosineSimilarityPredictionGraph,
               'euclidean': EuclideanSimilarityPredictionGraph}


@pytest.fixture
def cpu_session():
    from tensorrec_b200 import session_management as sm
    sm.set_session(sm.Session('cpu'))
    yield
    sm.set_session(None)


def autograd_of_the_mirror(monkeypatch, model, weights, interactions, uf, itf, samples):
    from tensorrec_b200.input_utils import SparseInput
    from tensorrec_b200.session_management import variable_scope
    n_users, n_sampled = samples.shape
    model.set_weights(weights)
    pairs = np.stack([np.repeat(np.arange(n_users), n_sampled), samples.reshape(-1)], axis=1).astype(np.int64)
    monkeypatch.setattr(T.tensorrec, 'sample_items', lambda *a, **k: pairs)
    with variable_scope(model._variables):
        basic_loss, _, pred_serial, _ = model._training_losses(SparseInput(interactions), SparseInput(uf),
                                                               SparseInput(itf), n_sampled, torch.device('cpu'))
    basic_loss.sum().backward()
    return (basic_loss.detach().numpy(), pred_serial.detach().numpy(),
            {k: v.grad.detach().numpy() for k, v in model._variables.items()})


# every factor at both levels, in a grid trimmed to the combinations that exercise each one
GRID = [(p, un, inn, nt, att, bal, bia)
        for p, un, inn, nt, att, bal, bia in itertools.product(PREDICTIONS, (False, True), (False, True), (1, 3),
                                                               (False, True), (False, True), (True, False))
        if not (att and nt == 1) and (bal == bia or p == 'dot') and (un == inn or nt == 1)]


@pytest.mark.parametrize('prediction,user_norm,item_norm,n_tastes,attention,balanced,biased', GRID)
def test_step_oracle_equals_autograd_of_the_host_mirror(monkeypatch, cpu_session, prediction, user_norm, item_norm,
                                                        n_tastes, attention, balanced, biased):
    d = 6
    interactions, uf, itf = util.generate_dummy_data(num_users=30, num_items=40, interaction_density=.15,
                                                     num_user_features=20, num_item_features=18,
                                                     n_features_per_user=5, n_features_per_item=4, seed=2)
    weights = make_weights(uf, itf, d, n_tastes, attention, biased, seed=11)
    samples = np.stack([np.random.default_rng(u).choice(itf.shape[0], 7, replace=False) for u in range(uf.shape[0])])
    normalize = [side for side, on in (('user', user_norm), ('item', item_norm)) if on]
    ref = sampled_rank_step_reference(uf, itf, interactions, weights, samples, prediction=prediction,
                                      normalize=normalize, n_tastes=n_tastes, attention=attention, balanced=balanced)
    model = make_model(prediction, user_norm, item_norm, n_tastes, attention, balanced, biased, d)
    loss, pred, grads = autograd_of_the_mirror(monkeypatch, model, weights, interactions, uf, itf, samples)
    assert np.allclose(loss, ref['loss'], rtol=2e-5, atol=2e-6)
    assert np.allclose(pred, ref['pred_serial'], rtol=2e-5, atol=2e-6)
    assert set(grads) == set(ref['grads'])
    for name, g in grads.items():
        scale = max(1.0, float(np.abs(ref['grads'][name]).max()))
        assert np.allclose(g, ref['grads'][name], rtol=1e-4, atol=2e-5 * scale), name


def test_the_general_oracle_restates_the_dot_step_oracle():
    interactions, uf, itf = util.generate_dummy_data(num_users=25, num_items=30, interaction_density=.2,
                                                     num_user_features=15, num_item_features=12,
                                                     n_features_per_user=4, n_features_per_item=4, seed=5)
    w = make_weights(uf, itf, 8, 1, False, True, seed=3)
    samples = np.stack([np.random.default_rng(u).choice(30, 6, replace=False) for u in range(25)])
    new = sampled_rank_step_reference(uf, itf, interactions, w, samples, balanced=True)
    old = loss_ops.wmrb_step_reference(uf, itf, interactions, w['linear_weights_user_0'], w['linear_weights_item'],
                                       w['feature_biases_user'][:, 0], w['feature_biases_item'][:, 0], samples,
                                       balanced=True)
    assert np.allclose(new['loss'], old['loss'], rtol=1e-6, atol=1e-7)
    for name, key in (('linear_weights_user_0', 'd_w_user'), ('linear_weights_item', 'd_w_item')):
        assert np.allclose(new['grads'][name], old[key], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize('prediction', ['dot', 'euclidean'])
def test_identical_tastes_share_the_gradient_equally(prediction):
    interactions, uf, itf = util.generate_dummy_data(num_users=20, num_items=25, interaction_density=.2,
                                                     num_user_features=10, num_item_features=10,
                                                     n_features_per_user=4, n_features_per_item=4, seed=8)
    one = make_weights(uf, itf, 8, 1, False, True, seed=4)
    two = dict(one, linear_weights_user_1=one['linear_weights_user_0'].copy())
    samples = np.stack([np.random.default_rng(u).choice(25, 5, replace=False) for u in range(20)])
    r1 = sampled_rank_step_reference(uf, itf, interactions, one, samples, prediction=prediction)
    r2 = sampled_rank_step_reference(uf, itf, interactions, two, samples, prediction=prediction, n_tastes=2)
    assert np.array_equal(r1['loss'], r2['loss'])
    assert np.array_equal(r2['grads']['linear_weights_user_0'], r2['grads']['linear_weights_user_1'])
    assert np.allclose(r2['grads']['linear_weights_user_0'], 0.5 * r1['grads']['linear_weights_user_0'],
                       rtol=1e-5, atol=1e-6)
    assert np.allclose(r2['grads']['linear_weights_item'], r1['grads']['linear_weights_item'], rtol=1e-5, atol=1e-6)


# ---- routing -------------------------------------------------------------------------------------------------
def test_step_plan_gives_the_wmrb_models_their_form_within_the_stated_limits(monkeypatch):
    monkeypatch.setattr(train_kernels, 'TRAIN_PATH', 'auto')
    for model in reference_example_models():
        form = train_kernels.step_plan(model, n_sampled_items=100)
        assert form is not None and form.d_pad == (model.n_components + 3) // 4 * 4
    nl, lin = NormalizedLinearRepresentationGraph, LinearRepresentationGraph
    for pred, un, inn, att, nt, d in itertools.product(PREDICTIONS.values(), (lin, nl), (lin, nl), (None, lin, nl),
                                                       (1, 2, 4), (1, 7, 128)):
        if att is not None and nt == 1:
            continue
        model = T.TensorRec(n_components=d, n_tastes=nt, user_repr_graph=un(), item_repr_graph=inn(),
                            attention_graph=att() if att else None, prediction_graph=pred(), loss_graph=WMRBLossGraph())
        form = train_kernels.step_plan(model, 2048)
        assert form is not None
        assert form.pair == ('euclidean' if pred is EuclideanSimilarityPredictionGraph else 'dot')
        cos = int(pred is CosineSimilarityPredictionGraph)
        assert form.normalize_user == int(un is nl) + cos and form.normalize_item == int(inn is nl) + cos
        assert form.n_tastes == nt and form.attention == (att is not None)
    ok = lambda **kw: train_kernels.step_plan(T.TensorRec(loss_graph=WMRBLossGraph(), **kw), 64) is not None  # noqa
    assert ok(n_components=512) and not ok(n_components=513)
    assert ok(n_components=128, n_tastes=8) and not ok(n_components=129, n_tastes=2)
    assert not ok(n_components=8, n_tastes=9)
    assert ok(n_components=128, n_tastes=4, attention_graph=lin())
    assert not ok(n_components=8, n_tastes=5, attention_graph=lin())
    assert not ok(n_components=8, item_repr_graph=ReLURepresentationGraph())
    assert not ok(n_components=8, attention_graph=ReLURepresentationGraph(), n_tastes=2)
    assert train_kernels.step_plan(T.TensorRec(n_components=8, loss_graph=RMSELossGraph())).loss == 'rmse'
    assert train_kernels.step_plan(T.TensorRec(n_components=8, loss_graph=WMRBLossGraph()), 2049) is None
    monkeypatch.setattr(train_kernels, 'TRAIN_PATH', 'torch')
    for model in reference_example_models():
        assert train_kernels.step_plan(model, 100) is None


# ---- input validation ----------------------------------------------------------------------------------------
def test_step_inputs_are_checked_before_any_launch():
    check = train_kernels.check_step_inputs
    good = np.zeros((4, 3), np.int32)
    check((4, 10), 4, 10, 3, None)
    check((4, 10), 4, 10, 3, good)
    check((4, 10), 4, 10, 3, torch.from_numpy(good + 9))
    with pytest.raises(ValueError, match='interactions'):
        check((4, 11), 4, 10, 3, None)
    with pytest.raises(ValueError, match='interactions'):
        check((5, 10), 4, 10, 3, None)
    with pytest.raises(ValueError, match='int32'):
        check((4, 10), 4, 10, 3, good.astype(np.int64))
    with pytest.raises(ValueError, match='int32'):
        check((4, 10), 4, 10, 3, torch.zeros((4, 3), dtype=torch.int64))
    with pytest.raises(ValueError, match='shape'):
        check((4, 10), 4, 10, 3, np.zeros((4, 2), np.int32))
    with pytest.raises(ValueError, match='shape'):
        check((4, 10), 4, 10, 3, np.zeros((3, 3), np.int32))
    with pytest.raises(ValueError, match='outside'):
        check((4, 10), 4, 10, 3, good + 10)
    with pytest.raises(ValueError, match='outside'):
        check((4, 10), 4, 10, 3, torch.from_numpy(good - 1))
