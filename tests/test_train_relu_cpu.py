"""CPU tests of the fused training step of ReLURepresentationGraph models (DESIGN §3.14): the ReLU step oracle
(tests/relu_step_oracle.py) equals torch autograd over the host mirror, relu_step_plan covers exactly the stated models
while step_plan's answers stay as they were, the kernel path creates the mirror's weights in the mirror's order, and the
layer's two C entry points reject every malformed argument before any launch."""
import itertools

import numpy as np
import pytest
import torch

from tests.helpers import reference_example_models
from tests.relu_step_oracle import relu_model, relu_step_reference, relu_weights
import tensorrec_b200 as T
from tensorrec_b200 import train_kernels, util
from tensorrec_b200.loss_graphs import BalancedWMRBLossGraph, RMSELossGraph, SeparationLossGraph, WMRBLossGraph
from tensorrec_b200.prediction_graphs import (CosineSimilarityPredictionGraph, DotProductPredictionGraph,
                                              EuclideanSimilarityPredictionGraph)
from tensorrec_b200.representation_graphs import (FeaturePassThroughRepresentationGraph, LinearRepresentationGraph,
                                                  NormalizedLinearRepresentationGraph, ReLURepresentationGraph)


@pytest.fixture
def cpu_session():
    from tensorrec_b200 import session_management as sm
    sm.set_session(sm.Session('cpu'))
    yield
    sm.set_session(None)


def mirror_step(monkeypatch, model, weights, interactions, uf, itf, samples):
    """Loss, pred_serial and weight gradients of torch autograd over the host mirror (TensorRec._training_losses)."""
    from tensorrec_b200.input_utils import SparseInput
    from tensorrec_b200.session_management import variable_scope
    model.set_weights(weights, n_user_features=uf.shape[1], n_item_features=itf.shape[1])
    n_sampled = None
    if samples is not None:
        n_users, n_sampled = samples.shape
        pairs = np.stack([np.repeat(np.arange(n_users), n_sampled), samples.reshape(-1)], axis=1).astype(np.int64)
        monkeypatch.setattr(T.tensorrec, 'sample_items', lambda *a, **k: pairs)
    with variable_scope(model._variables):
        basic_loss, _, pred_serial, _ = model._training_losses(SparseInput(interactions), SparseInput(uf),
                                                               SparseInput(itf), n_sampled, torch.device('cpu'))
    basic_loss.sum().backward()
    return (basic_loss.detach().numpy(), pred_serial.detach().numpy(),
            {k: v.grad.detach().numpy() for k, v in model._variables.items()})


ORACLE_CASES = [  # loss, prediction, relu sides, user_norm, n_tastes, attention, biased, hidden
    ('wmrb', 'dot', ('item',), True, 1, False, True, 12),
    ('balanced', 'cosine', ('item',), True, 1, False, False, 12),
    ('wmrb', 'euclidean', ('item',), True, 3, False, True, 9),
    ('wmrb', 'dot', ('user',), False, 1, False, False, 16),
    ('balanced', 'dot', ('attn',), True, 3, True, True, 8),
    ('rmse', 'dot', ('item',), False, 1, False, True, 12),
    ('separation', 'cosine', ('user', 'item'), False, 1, False, False, 10),
]


@pytest.mark.parametrize('loss,prediction,relu_sides,user_norm,n_tastes,attention,biased,hidden', ORACLE_CASES)
def test_relu_step_oracle_equals_autograd_of_the_host_mirror(monkeypatch, cpu_session, loss, prediction, relu_sides,
                                                             user_norm, n_tastes, attention, biased, hidden):
    d = 6
    interactions, uf, itf = util.generate_dummy_data(num_users=30, num_items=40, interaction_density=.15,
                                                     num_user_features=20, num_item_features=18,
                                                     n_features_per_user=5, n_features_per_item=4, seed=2)
    weights = relu_weights(uf, itf, d, hidden, relu_sides, n_tastes, attention, biased, seed=11)
    samples = None
    if loss in ('wmrb', 'balanced'):
        samples = np.stack([np.random.default_rng(u).choice(itf.shape[0], 7, replace=False)
                            for u in range(uf.shape[0])])
    ref = relu_step_reference(uf, itf, interactions, weights, relu_sides, samples=samples,
                              loss='wmrb' if samples is not None else loss, prediction=prediction,
                              normalize=['user'] if user_norm else [], n_tastes=n_tastes, attention=attention,
                              balanced=loss == 'balanced')
    model = relu_model(loss, prediction, relu_sides, user_norm, n_tastes, attention, biased, d, relu_size=hidden)
    got_loss, pred, grads = mirror_step(monkeypatch, model, weights, interactions, uf, itf, samples)
    assert np.allclose(got_loss, ref['loss'], rtol=2e-5, atol=2e-6)
    assert np.allclose(pred, ref['pred_serial'], rtol=2e-5, atol=2e-6)
    assert set(grads) == set(ref['grads'])
    assert any(name.startswith('relu_biases_') for name in grads)
    for name, g in grads.items():
        scale = max(1.0, float(np.abs(ref['grads'][name]).max()))
        assert np.allclose(g, ref['grads'][name], rtol=1e-4, atol=2e-5 * scale), name


def test_the_relu_gradient_passes_only_where_the_pre_activation_is_positive():
    from tests.relu_step_oracle import relu_layer_backward_reference, relu_layer_reference
    x = np.array([[1.0, 0.0], [0.0, 1.0], [1.0, 1.0]])
    w1 = np.array([[1.0, -2.0], [-1.0, 3.0]])
    b = np.array([-1.0, 2.0])             # Z = [[0, 0], [-2, 5], [-1, 3]]: two exact zeros
    w2 = np.array([[1.0], [2.0]])
    z, h, out = relu_layer_reference(x, w1, b, w2)
    dz, db, dw2 = relu_layer_backward_reference(z, h, w2, np.ones((3, 1)))
    assert np.array_equal(z, [[0.0, 0.0], [-2.0, 5.0], [-1.0, 3.0]])
    assert np.array_equal(dz, [[0.0, 0.0], [0.0, 2.0], [0.0, 2.0]])
    assert np.array_equal(db, [0.0, 4.0]) and np.array_equal(dw2, [[0.0], [8.0]])
    zt = torch.tensor(z, requires_grad=True)          # torch's rule is the same
    torch.relu(zt).sum().backward()
    assert np.array_equal(zt.grad.numpy(), (z > 0).astype(np.float64))


# ---- routing -------------------------------------------------------------------------------------------------
PREDICTIONS = (DotProductPredictionGraph, CosineSimilarityPredictionGraph, EuclideanSimilarityPredictionGraph)


def movielens_relu_models():
    """The 12 ReLU-item configurations of the reference's check_movielens_losses.py: NormalizedLinear users, ReLU items,
    WMRB / BalancedWMRB x dot / cosine / Euclidean x 1 / 3 tastes."""
    for lg, pred, nt in itertools.product((WMRBLossGraph, BalancedWMRBLossGraph), PREDICTIONS, (1, 3)):
        yield T.TensorRec(n_components=10, n_tastes=nt, user_repr_graph=NormalizedLinearRepresentationGraph(),
                          item_repr_graph=ReLURepresentationGraph(), prediction_graph=pred(), loss_graph=lg())


def test_relu_step_plan_covers_the_reference_examples_relu_half(monkeypatch):
    monkeypatch.setattr(train_kernels, 'TRAIN_PATH', 'auto')
    models = list(movielens_relu_models())
    assert len(models) == 12
    for model in models:
        assert train_kernels.step_plan(model, 100) is None
        form = train_kernels.relu_step_plan(model, 100)
        assert form is not None and form.loss == 'wmrb' and form.d_pad == 12
        cos = int(type(model.prediction_graph_factory) is CosineSimilarityPredictionGraph)
        assert form.normalize_user == 1 + cos and form.normalize_item == cos
        assert form.hidden == (0, 0, 40)
    monkeypatch.setattr(train_kernels, 'TRAIN_PATH', 'torch')
    for model in movielens_relu_models():
        assert train_kernels.relu_step_plan(model, 100) is None


def test_relu_step_plan_gives_each_side_its_padded_hidden_width_within_the_stated_limits(monkeypatch):
    monkeypatch.setattr(train_kernels, 'TRAIN_PATH', 'auto')
    relu, nl, lin = ReLURepresentationGraph, NormalizedLinearRepresentationGraph, LinearRepresentationGraph

    def plan(loss=WMRBLossGraph, n_sampled=64, **kw):
        return train_kernels.relu_step_plan(T.TensorRec(loss_graph=loss(), **kw), n_sampled)

    assert plan(n_components=8, user_repr_graph=relu(37)).hidden == (40, 0, 0)
    assert plan(n_components=8, user_repr_graph=relu(37), item_repr_graph=relu()).hidden == (40, 0, 32)
    assert plan(n_components=8, n_tastes=3, attention_graph=relu(16)).hidden == (0, 16, 0)
    assert plan(n_components=8, n_tastes=2, user_repr_graph=nl(), attention_graph=relu(5)).normalize_user == 1
    assert plan(n_components=8, item_repr_graph=relu(), prediction_graph=CosineSimilarityPredictionGraph()) \
        .normalize_item == 1
    assert plan(n_components=512, item_repr_graph=relu(2048)).hidden == (0, 0, 2048)
    assert plan(n_components=512, item_repr_graph=relu(2048), n_sampled=2048).d_pad == 512
    assert plan(n_components=13, item_repr_graph=relu(8)).d_pad == 16
    assert plan(n_components=8, loss=RMSELossGraph, n_sampled=None, item_repr_graph=relu()).loss == 'rmse'
    assert plan(n_components=8, loss=SeparationLossGraph, n_sampled=None, item_repr_graph=relu()).loss == 'separation'
    assert plan(n_components=128, n_tastes=4, attention_graph=relu(), item_repr_graph=relu()).hidden == (0, 512, 512)
    # the limits
    assert plan(n_components=8, item_repr_graph=relu(2049)) is None
    assert plan(n_components=8, item_repr_graph=relu(0)) is None
    assert plan(n_components=513, item_repr_graph=relu(16)) is None
    assert plan(n_components=129, n_tastes=2, item_repr_graph=relu(16)) is None
    assert plan(n_components=8, n_tastes=9, item_repr_graph=relu()) is None
    assert plan(n_components=8, n_tastes=5, attention_graph=relu()) is None
    assert plan(n_components=8, item_repr_graph=relu(), n_sampled=2049) is None
    # only Linear, NormalizedLinear and ReLU graphs, at least one ReLU
    assert plan(n_components=8) is None
    assert plan(n_components=8, user_repr_graph=nl(), attention_graph=lin(), n_tastes=2) is None
    assert plan(n_components=8, item_repr_graph=relu(), user_repr_graph=FeaturePassThroughRepresentationGraph()) \
        is None
    assert train_kernels.relu_step_plan(T.TensorRec(n_components=8, item_repr_graph=relu(),
                                                    loss_graph=T.loss_graphs.RMSEDenseLossGraph())) is None


def test_step_plan_answers_as_before_for_every_relu_model(monkeypatch):
    monkeypatch.setattr(train_kernels, 'TRAIN_PATH', 'auto')
    relu = ReLURepresentationGraph
    for kw in (dict(item_repr_graph=relu()), dict(user_repr_graph=relu()), dict(attention_graph=relu(), n_tastes=2),
               dict(item_repr_graph=relu(), user_repr_graph=relu())):
        for loss in (WMRBLossGraph, RMSELossGraph):
            model = T.TensorRec(n_components=8, loss_graph=loss(), **kw)
            assert train_kernels.step_plan(model, 64) is None
            assert train_kernels.relu_step_plan(model, 64) is not None
    for model in reference_example_models():          # and relu_step_plan leaves the models step_plan covers alone
        assert train_kernels.step_plan(model, 100) is not None
        assert train_kernels.relu_step_plan(model, 100) is None
        assert train_kernels.step_plan(model, 100).hidden == (0, 0, 0)


# ---- weights -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('relu_sides,n_tastes,attention,biased', [(('item',), 1, False, True),
                                                                   (('user',), 3, False, False),
                                                                   (('attn', 'item'), 2, True, True)])
def test_the_kernel_path_creates_the_mirrors_weights_in_the_mirrors_order(cpu_session, relu_sides, n_tastes,
                                                                          attention, biased):
    from tensorrec_b200.input_utils import SparseInput
    from tensorrec_b200.session_management import variable_scope
    interactions, uf, itf = util.generate_dummy_data(num_users=12, num_items=15, interaction_density=.2,
                                                     num_user_features=9, num_item_features=7,
                                                     n_features_per_user=3, n_features_per_item=3, seed=1)
    mirror = relu_model('wmrb', 'dot', relu_sides, False, n_tastes, attention, biased, 6, relu_size=11)
    mirror.n_user_features, mirror.n_item_features = uf.shape[1], itf.shape[1]
    with variable_scope(mirror._variables):
        mirror._training_losses(SparseInput(interactions), SparseInput(uf), SparseInput(itf), 3, torch.device('cpu'))
    expected = [(k, tuple(v.shape)) for k, v in mirror._variables.items()]

    model = relu_model('wmrb', 'dot', relu_sides, False, n_tastes, attention, biased, 6, relu_size=11)
    stepper = train_kernels.WmrbStep(model, torch.device('cpu'), seed=1)
    names, ws = stepper._weights(uf.shape[1], itf.shape[1], train_kernels.relu_step_plan(model, 3))
    assert names == [k for k, _ in expected]
    assert list(model._variables) == names
    assert [(k, tuple(ws[k].shape)) for k in names] == expected
    for end in ('item', 'user_0', 'attn_0'):
        if 'relu_biases_' + end in ws:
            assert not ws['relu_biases_' + end].any()
            w1 = ws['relu_weights_' + end].detach()
            assert 0.3 < float(w1.std()) < 0.7          # normal, stddev .5
    assert set(model._variables) == set(mirror._variables)


# ---- the C entry points' argument checks ---------------------------------------------------------------------
_BLOCK = np.zeros(64, np.float32)
A = (_BLOCK.ctypes.data + 15) // 16 * 16
MISALIGNED = A + 4
FORWARD = dict(pre=A, bias=A, w2=A, rows=10, hidden=64, d=32, out=A)
BACKWARD = dict(pre=A, bias=A, w2=A, d_out=A, rows=10, hidden=64, d=32, d_bias=A, d_w2=A, workspace=A,
                workspace_bytes=1 << 30)
ENTRY = {'trk_relu_layer_forward_f32': FORWARD, 'trk_relu_layer_backward_f32': BACKWARD}
PREFIX = {'trk_relu_layer_forward_f32': 'relu_layer_forward:', 'trk_relu_layer_backward_f32': 'relu_layer_backward:'}

FAULTS = [  # (entry point, fault, substring of trk_last_error())
    ('trk_relu_layer_forward_f32', dict(pre=None), 'null input'),
    ('trk_relu_layer_forward_f32', dict(bias=None), 'null input'),
    ('trk_relu_layer_forward_f32', dict(w2=None), 'null input'),
    ('trk_relu_layer_forward_f32', dict(out=None), 'null output'),
    ('trk_relu_layer_forward_f32', dict(rows=-1), 'rows=-1'),
    ('trk_relu_layer_forward_f32', dict(rows=1 << 31), 'rows='),
    ('trk_relu_layer_forward_f32', dict(hidden=0), 'hidden=0'),
    ('trk_relu_layer_forward_f32', dict(hidden=36), 'hidden=36'),
    ('trk_relu_layer_forward_f32', dict(hidden=2056), 'hidden=2056'),
    ('trk_relu_layer_forward_f32', dict(d=0), 'd=0'),
    ('trk_relu_layer_forward_f32', dict(d=10), 'd=10'),
    ('trk_relu_layer_forward_f32', dict(d=516), 'd=516'),
    ('trk_relu_layer_forward_f32', dict(pre=MISALIGNED), '16-byte aligned'),
    ('trk_relu_layer_forward_f32', dict(bias=MISALIGNED), '16-byte aligned'),
    ('trk_relu_layer_forward_f32', dict(w2=MISALIGNED), '16-byte aligned'),
    ('trk_relu_layer_forward_f32', dict(out=MISALIGNED), '16-byte aligned'),
    ('trk_relu_layer_backward_f32', dict(pre=None), 'null input'),
    ('trk_relu_layer_backward_f32', dict(bias=None), 'null input'),
    ('trk_relu_layer_backward_f32', dict(w2=None), 'null input'),
    ('trk_relu_layer_backward_f32', dict(d_out=None), 'null d_out'),
    ('trk_relu_layer_backward_f32', dict(d_bias=None), 'null output'),
    ('trk_relu_layer_backward_f32', dict(d_w2=None), 'null output'),
    ('trk_relu_layer_backward_f32', dict(workspace=None), 'null workspace'),
    ('trk_relu_layer_backward_f32', dict(rows=-1), 'rows=-1'),
    ('trk_relu_layer_backward_f32', dict(hidden=12), 'hidden=12'),
    ('trk_relu_layer_backward_f32', dict(hidden=4096), 'hidden=4096'),
    ('trk_relu_layer_backward_f32', dict(d=6), 'd=6'),
    ('trk_relu_layer_backward_f32', dict(d=1024), 'd=1024'),
    ('trk_relu_layer_backward_f32', dict(pre=MISALIGNED), '16-byte aligned'),
    ('trk_relu_layer_backward_f32', dict(d_out=MISALIGNED), 'aligned'),
    ('trk_relu_layer_backward_f32', dict(workspace=MISALIGNED), 'aligned'),
    ('trk_relu_layer_backward_f32', dict(d_w2=A + 4), 'aligned'),
    ('trk_relu_layer_backward_f32', dict(workspace_bytes=0), 'workspace of 0 bytes'),
]


def call(lib, entry, fault):
    args = dict(ENTRY[entry], **fault)
    return getattr(lib, entry)(*args.values(), None)


@pytest.mark.parametrize('entry,fault,message', FAULTS, ids=['{}-{}'.format(e.split('_')[3], '-'.join(f))
                                                             + str(i) for i, (e, f, _) in enumerate(FAULTS)])
def test_each_fault_is_rejected_with_the_entry_points_name(entry, fault, message):
    from tensorrec_b200 import _lib
    lib = _lib.load()
    assert call(lib, entry, fault) == _lib.TRK_ERR_ARG
    err = _lib.last_error()
    assert err.startswith(PREFIX[entry]) and message in err, err


def test_the_accepted_sides_of_the_bounds_pass_every_check():
    """rows = 0 has nothing to compute: the forward returns TRK_OK at the widest and narrowest accepted shapes, without
    a launch.  The backward's checks pass on the same shapes up to its workspace size, whose query gives the need."""
    from tensorrec_b200 import _lib
    lib = _lib.load()
    for hidden, d in ((8, 4), (2048, 512), (40, 36)):
        assert call(lib, 'trk_relu_layer_forward_f32', dict(rows=0, hidden=hidden, d=d)) == _lib.TRK_OK
        need = int(lib.trk_relu_layer_workspace_bytes(1000, hidden, d))
        assert need > 0 and need % 16 == 0 and need >= hidden * (d + 1) * 4
        assert call(lib, 'trk_relu_layer_backward_f32', dict(rows=1000, hidden=hidden, d=d,
                                                             workspace_bytes=need - 1)) == _lib.TRK_ERR_ARG
        assert 'workspace of {} bytes, {} needed'.format(need - 1, need) in _lib.last_error()
    # the partition depends on the shape only: the same shape always needs the same workspace
    assert lib.trk_relu_layer_workspace_bytes(1 << 20, 512, 128) == lib.trk_relu_layer_workspace_bytes(1 << 20, 512,
                                                                                                        128)
