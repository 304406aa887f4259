"""GPU tests of the fused training step of ReLURepresentationGraph models (DESIGN §3.14): the hidden layer's kernels
against float64 within the 3xTF32 bound, one step against the ReLU step oracle (tests/relu_step_oracle.py, pinned on
the CPU against torch autograd over the host mirror), run-to-run determinism, Adam over every weight, bf16
representations, and fit() on the ReLU configurations of the reference's check_movielens_losses.py."""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import loss_ops
from tests.helpers import csr_order
from tests.relu_step_oracle import (relu_layer_backward_reference, relu_layer_reference, relu_model,
                                    relu_step_reference, relu_weights)

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


# ---- the layer kernels alone ---------------------------------------------------------------------------------
def run_layer(pre, bias, w2, d_out):
    """trk_relu_layer_forward_f32 and _backward_f32 on the device: (out, dP, d_bias, d_w2) on the host."""
    import torch
    from tensorrec_b200 import _lib
    from tensorrec_b200.kernels import _p, _stream
    lib = _lib.load()
    rows, hidden = pre.shape
    d = w2.shape[1]
    dev = torch.device('cuda', 0)
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=F32)).to(dev)   # noqa: E731
    p, b, w, g = up(pre), up(bias.reshape(-1)), up(w2), up(d_out)
    out = torch.full((rows, d), float('nan'), dtype=torch.float32, device=dev)
    _lib.check(lib.trk_relu_layer_forward_f32(_p(p), _p(b), _p(w), rows, hidden, d, _p(out), _stream()), 'forward')
    n = int(lib.trk_relu_layer_workspace_bytes(rows, hidden, d))
    ws = torch.empty((n,), dtype=torch.uint8, device=dev)
    db = torch.full((hidden,), float('nan'), dtype=torch.float32, device=dev)
    dw2 = torch.full((hidden, d), float('nan'), dtype=torch.float32, device=dev)
    _lib.check(lib.trk_relu_layer_backward_f32(_p(p), _p(b), _p(w), _p(g), rows, hidden, d, _p(db), _p(dw2), _p(ws), n,
                                               _stream()), 'backward')
    return out.cpu().numpy(), p.cpu().numpy(), db.cpu().numpy(), dw2.cpu().numpy()


def bound(abs_a, abs_b, k):
    """|3xTF32 - exact| <= (3 2^-22 + (k + 2) 2^-23) sum_k |a||b| (DESIGN §3.14): per product the dropped small.small
    term and the two splits' residuals, then fp32 accumulation over k terms."""
    return (3 * 2.0 ** -22 + (k + 2) * 2.0 ** -23) * (abs_a @ abs_b) + 1e-30


LAYER_SHAPES = [(1, 8, 4), (257, 40, 36), (1000, 512, 128), (300, 2048, 512), (130, 96, 20), (64, 8, 512)]


@pytest.mark.parametrize('rows,hidden,d', LAYER_SHAPES)
def test_the_layer_kernels_match_float64_within_the_3xtf32_bound(T, rows, hidden, d):
    rng = np.random.default_rng(rows + hidden + d)
    pre = rng.standard_normal((rows, hidden)).astype(F32)
    pre[::7] = -np.abs(pre[::7]) - 3.0              # rows whose pre-activations are all negative
    bias = (0.3 * rng.standard_normal(hidden)).astype(F32)
    bias[::7] = -10.0                               # (and so, for every row, these units)
    w2 = (rng.standard_normal((hidden, d)) / np.sqrt(hidden)).astype(F32)
    d_out = rng.standard_normal((rows, d)).astype(F32)
    out, dp, db, dw2 = run_layer(pre, bias, w2, d_out)

    z, h, exp_out = relu_layer_reference(pre.astype(np.float64), w2=w2, w1=np.eye(hidden), b=bias)
    exp_dz, exp_db, exp_dw2 = relu_layer_backward_reference(z, h, w2, d_out)
    assert np.all(np.abs(out - exp_out) <= bound(h, np.abs(w2), hidden))
    assert np.all(out[::7] == 0.0)
    dz_bound = bound(np.abs(d_out), np.abs(w2).T, d)
    assert np.all(np.abs(dp - exp_dz) <= dz_bound)
    assert np.all(dp[z <= 0] == 0.0) and np.all(dp[::7] == 0.0)
    # db and dW2: each chunk's partial within the bound, then fp32 sums of the chunks
    assert np.all(np.abs(db - exp_db) <= dz_bound.sum(axis=0) + (rows + 2) * 2.0 ** -23 * np.abs(exp_dz).sum(axis=0)
                  + 1e-30)
    assert np.all(np.abs(dw2 - exp_dw2) <= 2 * bound(h.T, np.abs(d_out), rows))
    assert np.all(db[::7] == 0.0) and np.all(dw2[::7] == 0.0)


def test_an_exact_zero_pre_activation_gets_no_gradient(T):
    """Integer-valued inputs make every product exact: P + b == 0 exactly for a third of the entries."""
    rng = np.random.default_rng(3)
    rows, hidden, d = 200, 24, 8
    pre = rng.integers(-3, 4, (rows, hidden)).astype(F32)
    bias = rng.integers(-2, 3, hidden).astype(F32)
    w2 = rng.integers(-2, 3, (hidden, d)).astype(F32)
    d_out = rng.integers(-2, 3, (rows, d)).astype(F32)
    out, dp, db, dw2 = run_layer(pre, bias, w2, d_out)
    z, h, exp_out = relu_layer_reference(pre.astype(np.float64), np.eye(hidden), bias, w2)
    exp_dz, exp_db, exp_dw2 = relu_layer_backward_reference(z, h, w2, d_out)
    assert (z == 0.0).sum() > rows * hidden // 10
    assert np.array_equal(out, exp_out) and np.array_equal(dp, exp_dz)
    assert np.all(dp[z == 0.0] == 0.0)
    assert np.array_equal(db, exp_db) and np.array_equal(dw2, exp_dw2)


# ---- one step against the oracle -----------------------------------------------------------------------------
def make_case(seed, d, hidden, relu_sides, n_tastes, attention, biased, n_users=260, n_items=230):
    from tensorrec_b200 import util
    interactions, uf, itf = util.generate_dummy_data(num_users=n_users, num_items=n_items, interaction_density=0.05,
                                                     num_user_features=40, num_item_features=30,
                                                     n_features_per_user=6, n_features_per_item=5, seed=seed)
    weights = relu_weights(uf, itf, d, hidden, relu_sides, n_tastes, attention, biased, seed + 100)
    return sp.csr_matrix(interactions), uf, itf, weights


def relu_step(model, weights, interactions, uf, itf, samples=None, bf16=False, lr=0.05, l2=0.0):
    """One WmrbStep.step from `weights` on device 0: the stepper, and the loss and pred_serial on the host."""
    import torch
    from tensorrec_b200 import train_kernels as TK
    from tensorrec_b200.input_utils import SparseInput
    model.set_weights(weights, n_user_features=uf.shape[1], n_item_features=itf.shape[1])
    stepper = TK.WmrbStep(model, torch.device('cuda', 0), seed=3, bf16=bf16)
    st = None if samples is None else torch.from_numpy(np.ascontiguousarray(samples, dtype=np.int32)).cuda()
    loss, pred = stepper.step(SparseInput(interactions), SparseInput(uf), SparseInput(itf),
                              None if samples is None else samples.shape[1], lr, l2, samples=st)
    return stepper, loss.cpu().numpy(), pred.cpu().numpy()


STEP_CASES = [  # loss, prediction, relu sides, user_norm, n_tastes, attention, biased, d, hidden
    ('wmrb', 'dot', ('item',), True, 1, False, True, 10, 40),
    ('balanced', 'dot', ('item',), True, 1, False, False, 10, 40),
    ('wmrb', 'cosine', ('item',), True, 1, False, False, 10, 40),
    ('balanced', 'cosine', ('item',), True, 3, False, True, 10, 40),
    ('wmrb', 'euclidean', ('item',), True, 1, False, True, 10, 40),
    ('balanced', 'euclidean', ('item',), True, 3, False, False, 10, 40),
    ('wmrb', 'dot', ('user',), False, 1, False, True, 8, 37),
    ('balanced', 'cosine', ('attn',), True, 3, True, True, 10, 40),
    ('wmrb', 'euclidean', ('user', 'item', 'attn'), False, 3, True, False, 6, 16),
    ('rmse', 'dot', ('item',), False, 1, False, True, 10, 40),
    ('rmse', 'cosine', ('user', 'item'), False, 1, False, False, 7, 37),
    ('separation', 'euclidean', ('item',), True, 1, False, True, 12, 48),
    ('separation', 'dot', ('user',), False, 3, False, False, 10, 24),
    ('wmrb', 'dot', ('item',), True, 1, False, True, 512, 2048),
    ('rmse', 'dot', ('user',), False, 1, False, True, 130, 520),
]


@pytest.mark.parametrize('loss,prediction,relu_sides,user_norm,n_tastes,attention,biased,d,hidden', STEP_CASES)
def test_kernel_step_matches_the_relu_oracle(T, loss, prediction, relu_sides, user_norm, n_tastes, attention, biased,
                                             d, hidden):
    interactions, uf, itf, weights = make_case(d + hidden, d, hidden, relu_sides, n_tastes, attention, biased)
    samples = None
    if loss in ('wmrb', 'balanced'):
        rng = np.random.default_rng(5)
        samples = np.stack([rng.choice(itf.shape[0], 17, replace=False) for _ in range(uf.shape[0])])
    ref = relu_step_reference(uf, itf, interactions, weights, relu_sides, samples=samples,
                              loss='wmrb' if samples is not None else loss, prediction=prediction,
                              normalize=['user'] if user_norm else [], n_tastes=n_tastes, attention=attention,
                              balanced=loss == 'balanced')
    model = relu_model(loss, prediction, relu_sides, user_norm, n_tastes, attention, biased, d, relu_size=hidden)
    stepper, got_loss, pred = relu_step(model, weights, interactions, uf, itf, samples)
    order = csr_order(interactions)
    pscale = float(np.abs(ref['pred_serial']).max())
    assert np.allclose(pred, ref['pred_serial'][order], rtol=1e-4, atol=1e-5 * max(1.0, pscale))
    if samples is not None:
        full = np.zeros(len(order), F32)
        full[ref['positive_mask']] = ref['loss']
        assert np.allclose(got_loss, full[order], rtol=1e-4, atol=1e-5 + 1e-4 * pscale)
    else:
        assert np.allclose(got_loss[0], ref['loss'], rtol=1e-4, atol=1e-6)
    g = {k: v.cpu().numpy().reshape(ref['grads'][k].shape) for k, v in stepper.last['grads'].items()}
    assert set(g) == set(ref['grads'])
    assert {k for k in g if k.startswith('relu_biases_')} == {'relu_biases_' + e for e in ref['d_rows']
                                                              if e.split('_')[0] in relu_sides}
    for name, exp in ref['grads'].items():
        # (a WMRB user bias gradient cancels to rounding noise: the absolute floor covers it)
        scale = max(1.0, float(np.abs(exp).max()))
        assert np.allclose(g[name], exp, rtol=1e-3, atol=2e-4 * scale), name
    w = model.get_weights()
    assert [(k, v.shape) for k, v in w.items()] == [(k, weights[k].shape) for k in w]


def test_two_identical_steps_give_bit_identical_gradients(T):
    """The layer adds no unordered sum: a ReLU user side, whose d_rows the loss kernels write without atomics, gets the
    same bits in every weight gradient; the layer alone gives the same bits for the same inputs.  (The loss kernels add
    the item rows' gradients with red.global.add, in no fixed order: DESIGN §3.10.)"""
    for loss in ('wmrb', 'rmse'):
        interactions, uf, itf, weights = make_case(21, 16, 64, ('user',), 1, False, True, n_users=3000, n_items=2000)
        samples = None if loss == 'rmse' else np.random.default_rng(1).integers(0, itf.shape[0], (uf.shape[0], 20))
        runs = []
        for _ in range(2):
            model = relu_model(loss, 'dot', ('user',), False, 1, False, True, 16, relu_size=64)
            stepper, _, _ = relu_step(model, weights, interactions, uf, itf, samples)
            runs.append({k: v.cpu().numpy() for k, v in stepper.last['grads'].items()})
        for name in ('relu_weights_user_0', 'relu_biases_user_0', 'linear_weights_user_0'):
            assert np.array_equal(runs[0][name], runs[1][name]), (loss, name)
    rng = np.random.default_rng(8)
    pre = rng.standard_normal((20000, 512)).astype(F32)
    bias = rng.standard_normal(512).astype(F32)
    w2 = rng.standard_normal((512, 128)).astype(F32)
    d_out = rng.standard_normal((20000, 128)).astype(F32)
    first, second = run_layer(pre, bias, w2, d_out), run_layer(pre, bias, w2, d_out)
    for a, b in zip(first, second):
        assert np.array_equal(a, b)


def test_two_adam_steps_over_every_weight_match_the_adam_reference(T):
    import torch
    from tensorrec_b200.input_utils import SparseInput
    interactions, uf, itf, weights = make_case(9, 10, 40, ('item',), 3, False, True)
    samples = np.stack([np.random.default_rng(u).choice(itf.shape[0], 8, replace=False) for u in range(uf.shape[0])])
    model = relu_model('balanced', 'cosine', ('item',), True, 3, False, True, 10, relu_size=40)
    lr, l2 = 0.05, 0.01
    stepper, _, _ = relu_step(model, weights, interactions, uf, itf, samples, lr=lr, l2=l2)
    w1 = model.get_weights()
    g1 = {k: v.cpu().numpy().reshape(weights[k].shape) for k, v in stepper.last['grads'].items()}
    assert set(w1) == set(weights) and {'relu_weights_item', 'relu_biases_item', 'linear_weights_item'} <= set(w1)
    moments = {}
    for name, w0 in weights.items():
        exp, m, v = loss_ops.adam_reference(w0, g1[name], np.zeros_like(w0), np.zeros_like(w0), 1, lr, l2=l2)
        assert np.allclose(w1[name], exp, rtol=1e-6, atol=1e-7), name
        moments[name] = (m, v)
    st = torch.from_numpy(samples.astype(np.int32)).cuda()
    stepper.step(SparseInput(interactions), SparseInput(uf), SparseInput(itf), 8, lr, l2, samples=st)
    w2 = model.get_weights()
    for name in weights:
        g2 = stepper.last['grads'][name].cpu().numpy().reshape(weights[name].shape)
        exp, _, _ = loss_ops.adam_reference(w1[name], g2, *moments[name], 2, lr, l2=l2)
        assert np.allclose(w2[name], exp, rtol=1e-5, atol=1e-6), name


@pytest.mark.parametrize('loss,prediction', [('wmrb', 'dot'), ('rmse', 'euclidean')])
def test_bf16_rounds_the_representation_after_the_layer(T, loss, prediction):
    import torch
    interactions, uf, itf, weights = make_case(13, 12, 48, ('item',), 1, False, True)
    samples = None
    if loss == 'wmrb':
        samples = np.stack([np.random.default_rng(u).choice(itf.shape[0], 9, replace=False)
                            for u in range(uf.shape[0])])

    def bf16(x):
        return torch.from_numpy(np.ascontiguousarray(x, F32)).to(torch.bfloat16).to(torch.float32).numpy()

    ref = relu_step_reference(uf, itf, interactions, weights, ('item',), samples=samples, loss=loss,
                              prediction=prediction, normalize=['user'], round_repr=bf16)
    model = relu_model(loss, prediction, ('item',), True, 1, False, True, 12, relu_size=48)
    stepper, got_loss, pred = relu_step(model, weights, interactions, uf, itf, samples, bf16=True)
    order = csr_order(interactions)
    # the layer's last-bit differences can move a representation across a bf16 rounding boundary (2^-8 relative)
    pscale = float(np.abs(ref['pred_serial']).max())
    assert np.allclose(pred, ref['pred_serial'][order], rtol=1e-2, atol=1e-2 * pscale)
    g = {k: v.cpu().numpy().reshape(ref['grads'][k].shape) for k, v in stepper.last['grads'].items()}
    for name, exp in ref['grads'].items():
        scale = max(1e-3, float(np.abs(exp).max()))
        assert np.allclose(g[name], exp, rtol=3e-2, atol=3e-2 * scale), name


# ---- fit -----------------------------------------------------------------------------------------------------
def movielens_relu_models(T):
    """The 12 ReLU-item configurations of the reference's check_movielens_losses.py."""
    import itertools
    from tensorrec_b200.loss_graphs import BalancedWMRBLossGraph, WMRBLossGraph
    from tensorrec_b200.prediction_graphs import (CosineSimilarityPredictionGraph, DotProductPredictionGraph,
                                                  EuclideanSimilarityPredictionGraph)
    from tensorrec_b200.representation_graphs import NormalizedLinearRepresentationGraph, ReLURepresentationGraph
    for lg, pred, nt in itertools.product((WMRBLossGraph, BalancedWMRBLossGraph),
                                          (DotProductPredictionGraph, CosineSimilarityPredictionGraph,
                                           EuclideanSimilarityPredictionGraph), (1, 3)):
        yield T.TensorRec(n_components=10, n_tastes=nt, user_repr_graph=NormalizedLinearRepresentationGraph(),
                          item_repr_graph=ReLURepresentationGraph(), prediction_graph=pred(), loss_graph=lg())


def test_fit_on_the_relu_configurations_of_the_movielens_comparison_takes_the_kernel_path_and_learns(T):
    from tensorrec_b200 import util
    # MovieLens-100k's shape: 943 users x 1682 items
    interactions, uf, itf = util.generate_dummy_data(num_users=943, num_items=1682, interaction_density=.03,
                                                     num_user_features=100, num_item_features=150,
                                                     n_features_per_user=8, n_features_per_item=8, seed=4)
    pos = sp.coo_matrix(interactions)
    keep = pos.data > 0
    models = list(movielens_relu_models(T))
    assert len(models) == 12
    for model in models:
        model.fit(interactions, uf, itf, epochs=1, n_sampled_items=50, learning_rate=0.05)
        assert model._wmrb_step is not None and model._wmrb_step.t == 1, 'the kernel training path was not taken'
        first = float(model._wmrb_step.last['loss'].sum())
        model.fit_partial(interactions, uf, itf, epochs=40, n_sampled_items=50, learning_rate=0.05)
        assert model._wmrb_step.t == 41
        assert float(model._wmrb_step.last['loss'].sum()) < first
        assert set(model.get_weights()) >= {'relu_weights_item', 'relu_biases_item', 'linear_weights_item'}
        ranks = model.predict_rank(uf, itf)
        assert ranks[pos.row[keep], pos.col[keep]].mean() < 0.5 * 1682       # better than chance


def test_fit_under_train_path_torch_keeps_the_torch_path_for_relu_models(T, monkeypatch):
    from tensorrec_b200 import train_kernels, util
    monkeypatch.setattr(train_kernels, 'TRAIN_PATH', 'torch')
    interactions, uf, itf = util.generate_dummy_data(num_users=50, num_items=60, interaction_density=.1, seed=4)
    for model in list(movielens_relu_models(T))[:3]:
        model.fit(interactions, uf, itf, epochs=2, n_sampled_items=10)
        assert getattr(model, '_wmrb_step', None) is None and model._optimizer is not None
