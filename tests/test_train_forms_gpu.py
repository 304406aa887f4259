"""GPU tests of the fused training step's forms (DESIGN §3.10) against the general step oracle
(tests/train_step_oracle.sampled_rank_step_reference, pinned on the CPU against torch autograd over the host mirror:
tests/test_train_forms_cpu.py): cosine / Euclidean prediction, NormalizedLinear sides, mixtures of tastes with max or
attention collapse, padded n_components, bf16 representations, Adam over every weight, and fit() on the WMRB
configurations of the reference's examples."""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import loss_ops
from tests.helpers import csr_order, kernel_step, make_model, make_weights, reference_example_models
from tests.train_step_oracle import sampled_rank_step_reference

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


def make_case(seed, d, n_tastes, attention, biased, n_users=260, n_items=230):
    from tensorrec_b200 import util
    interactions, uf, itf = util.generate_dummy_data(num_users=n_users, num_items=n_items, interaction_density=0.05,
                                                     num_user_features=40, num_item_features=30,
                                                     n_features_per_user=6, n_features_per_item=5, seed=seed)
    return sp.csr_matrix(interactions), uf, itf, make_weights(uf, itf, d, n_tastes, attention, biased, seed + 100)


CASES = [  # prediction, user_norm, item_norm, n_tastes, attention, balanced, biased, d, n_sampled
    ('dot', False, False, 1, False, False, True, 5, 9),
    ('dot', True, False, 1, False, True, True, 10, 17),
    ('cosine', False, False, 1, False, False, False, 10, 9),
    ('cosine', True, True, 1, False, True, True, 128, 33),
    ('euclidean', False, False, 1, False, False, True, 10, 9),
    ('euclidean', True, False, 1, False, True, False, 200, 64),
    ('cosine', False, False, 1, False, False, True, 300, 20),
    ('dot', True, False, 3, False, False, True, 10, 9),
    ('cosine', True, True, 3, False, True, True, 128, 33),
    ('euclidean', False, True, 3, False, False, True, 5, 9),
    ('dot', True, False, 3, True, True, True, 10, 17),
    ('cosine', False, False, 3, True, False, False, 128, 20),
    ('euclidean', True, False, 3, True, False, True, 10, 9),
    ('dot', False, False, 8, False, False, True, 128, 16),
    ('euclidean', False, False, 4, True, True, True, 128, 16),
]


@pytest.mark.parametrize('prediction,user_norm,item_norm,n_tastes,attention,balanced,biased,d,n_sampled', CASES)
def test_kernel_step_matches_the_oracle_fp32(T, prediction, user_norm, item_norm, n_tastes, attention, balanced, biased,
                                             d, n_sampled):
    interactions, uf, itf, weights = make_case(d + n_tastes, d, n_tastes, attention, biased)
    rng = np.random.default_rng(5)
    samples = np.stack([rng.choice(itf.shape[0], n_sampled, replace=False) for _ in range(uf.shape[0])])
    normalize = [side for side, on in (('user', user_norm), ('item', item_norm)) if on]
    ref = sampled_rank_step_reference(uf, itf, interactions, weights, samples, prediction=prediction,
                                      normalize=normalize, n_tastes=n_tastes, attention=attention, balanced=balanced)
    model = make_model(prediction, user_norm, item_norm, n_tastes, attention, balanced, biased, d)
    stepper, loss, pred = kernel_step(model, weights, interactions, uf, itf, samples)
    order = csr_order(interactions)
    assert np.allclose(pred, ref['pred_serial'][order], rtol=2e-5, atol=2e-6)
    full = np.zeros(len(order), F32)
    full[ref['positive_mask']] = ref['loss']
    # a hinge term carries its scores' rounding (2e-5 relative of scores far larger than the loss with many tastes)
    assert np.allclose(loss, full[order], rtol=2e-5, atol=2e-6 + 2e-5 * float(np.abs(pred).max()))
    g = {k: v.cpu().numpy().reshape(ref['grads'][k].shape) for k, v in stepper.last['grads'].items()}
    assert set(g) == set(ref['grads'])
    for name, exp in ref['grads'].items():
        scale = max(1.0, float(np.abs(exp).max()))
        assert np.allclose(g[name], exp, rtol=2e-4, atol=2e-5 * scale), name


@pytest.mark.parametrize('prediction,n_tastes,attention', [('cosine', 1, False), ('euclidean', 3, True)])
def test_kernel_step_bf16_representations(T, prediction, n_tastes, attention):
    interactions, uf, itf, weights = make_case(3, 128, n_tastes, attention, True)
    rng = np.random.default_rng(6)
    samples = np.stack([rng.choice(itf.shape[0], 20, replace=False) for _ in range(uf.shape[0])])
    kw = dict(prediction=prediction, normalize=['user'], n_tastes=n_tastes, attention=attention)
    ref = sampled_rank_step_reference(uf, itf, interactions, weights, samples, round_repr=loss_ops.round_to_bfloat16,
                                      **kw)
    model = make_model(prediction, True, False, n_tastes, attention, False, True, 128)
    stepper, loss, pred = kernel_step(model, weights, interactions, uf, itf, samples, bf16=True)
    order = csr_order(interactions)
    err = np.abs(pred - ref['pred_serial'][order])
    assert np.mean(err <= 2e-5 * np.abs(pred) + 2e-6) > 0.9
    assert err.max() < 0.02
    g = stepper.last['grads']['linear_weights_item'].cpu().numpy()
    exp = ref['grads']['linear_weights_item']
    scale = max(1.0, float(np.abs(exp).max()))
    assert np.abs(g - exp).max() < 5e-3 * scale
    assert np.mean(np.abs(g - exp) <= 2e-4 * np.abs(exp) + 2e-5 * scale) > 0.9
    exact = sampled_rank_step_reference(uf, itf, interactions, weights, samples, **kw)
    diff = np.abs(pred - exact['pred_serial'][order])
    assert diff.max() < 0.25 and diff.mean() > 1e-5


def test_two_adam_steps_over_every_weight_match_the_oracle(T):
    import torch
    from tensorrec_b200.input_utils import SparseInput
    interactions, uf, itf, weights = make_case(9, 10, 3, True, True, n_users=120, n_items=90)
    rng = np.random.default_rng(2)
    samples = np.stack([rng.choice(itf.shape[0], 8, replace=False) for _ in range(uf.shape[0])])
    lr, l2 = 0.1, 0.3
    model = make_model('cosine', True, False, 3, True, False, True, 10)
    stepper, _, _ = kernel_step(model, weights, interactions, uf, itf, samples, lr=lr, l2=l2)
    w1 = model.get_weights()
    g1 = {k: v.cpu().numpy().reshape(weights[k].shape) for k, v in stepper.last['grads'].items()}
    assert set(w1) == set(weights)
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


def test_fit_on_every_reference_example_configuration_takes_the_kernel_path_and_learns(T):
    from tensorrec_b200 import util
    interactions, uf, itf = util.generate_dummy_data(num_users=200, num_items=300, interaction_density=.05, seed=4)
    pos = sp.coo_matrix(interactions)
    keep = pos.data > 0
    for model in reference_example_models():
        model.fit(interactions, uf, itf, epochs=1, n_sampled_items=20, learning_rate=0.05)
        assert model._wmrb_step is not None and model._wmrb_step.t == 1, 'the kernel training path was not taken'
        first = float(model._wmrb_step.last['loss'].sum())
        model.fit_partial(interactions, uf, itf, epochs=30, n_sampled_items=20, learning_rate=0.05)
        assert model._wmrb_step.t == 31
        assert float(model._wmrb_step.last['loss'].sum()) < first
        ranks = model.predict_rank(uf, itf)
        assert ranks[pos.row[keep], pos.col[keep]].mean() < 0.5 * 300       # better than chance


def test_fit_under_train_path_torch_keeps_the_torch_path(T, monkeypatch):
    from tensorrec_b200 import train_kernels, util
    monkeypatch.setattr(train_kernels, 'TRAIN_PATH', 'torch')
    interactions, uf, itf = util.generate_dummy_data(num_users=50, num_items=60, interaction_density=.1, seed=4)
    for model in list(reference_example_models())[:3]:
        model.fit(interactions, uf, itf, epochs=2, n_sampled_items=10)
        assert getattr(model, '_wmrb_step', None) is None and model._optimizer is not None


def test_identical_tastes_stay_identical_after_a_kernel_step(T):
    for prediction in ('dot', 'euclidean'):
        interactions, uf, itf, weights = make_case(7, 10, 2, False, True)
        weights['linear_weights_user_1'] = weights['linear_weights_user_0'].copy()
        samples = np.stack([np.random.default_rng(u).choice(itf.shape[0], 9, replace=False)
                            for u in range(uf.shape[0])])
        model = make_model(prediction, True, False, 2, False, False, True, 10)
        stepper, _, _ = kernel_step(model, weights, interactions, uf, itf, samples)
        g = stepper.last['grads']
        assert np.array_equal(g['linear_weights_user_0'].cpu().numpy(), g['linear_weights_user_1'].cpu().numpy())
        w = model.get_weights()
        assert np.array_equal(w['linear_weights_user_0'], w['linear_weights_user_1'])
        assert not np.array_equal(w['linear_weights_user_0'], weights['linear_weights_user_0'])
