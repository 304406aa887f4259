"""Seeded synthetic inputs shared by the tests, the golden-fixture generator and bench.py; the models, weights,
interactions and one kernel step of the fused training step's tests.

Generators follow the reference's tensorrec/util.py:61-85 (tag regime: sp.rand features) and :88-117 (indicator
regime: identity + random tag columns), but are seeded (the reference is unseeded) -- SURVEY.md 8(d)."""
import numpy as np
import scipy.sparse as sp

F32 = np.float32


def tag_features(rows, n_features=200, per_row=20, seed=0, integer=False):
    """util.py:75-78: sp.rand(rows, n_features, density=per_row/n_features), values U[0,1) (or {1} if integer)."""
    rng = np.random.default_rng(seed)
    m = sp.random(rows, n_features, density=float(per_row) / n_features, format='csr', dtype=np.float64,
                  random_state=rng)
    if integer:
        m.data[:] = 1.0
    return m.astype(F32)


def indicator_features(rows, seed=0, tags_per_row=3):
    """util.py:90-108: identity block + tags_per_row*rows random 1.0 entries in columns [rows, 1.2*rows)."""
    rng = np.random.default_rng(seed)
    n_features = int(rows * 1.2)
    n_tag_cols = max(n_features - rows, 1)
    n_features = rows + n_tag_cols
    n_tags = rows * tags_per_row
    r = np.concatenate([np.arange(rows), rng.integers(0, rows, n_tags)])
    c = np.concatenate([np.arange(rows), rows + rng.integers(0, n_tag_cols, n_tags)])
    m = sp.csr_matrix((np.ones(r.shape[0], dtype=F32), (r, c)), shape=(rows, n_features))
    m.sum_duplicates()            # the reference writes `= 1` into a lil_matrix: duplicates collapse
    m.data[:] = 1.0
    return m.astype(F32)


def linear_weights(n_features, d, seed=2, integer=False):
    """representation_graphs.py:35-36: random_normal rows, L2-normalised (or small integers for exact fixtures)."""
    rng = np.random.default_rng(seed)
    if integer:
        return rng.integers(-2, 3, size=(n_features, d)).astype(F32)
    w = rng.standard_normal((n_features, d)).astype(F32)
    w /= np.maximum(np.linalg.norm(w, axis=1, keepdims=True), 1e-6).astype(F32)
    return w.astype(F32)


def feature_biases(n_features, seed=4, integer=False):
    rng = np.random.default_rng(seed)
    if integer:
        return rng.integers(-3, 4, size=(n_features,)).astype(F32)
    return (0.1 * rng.standard_normal(n_features)).astype(F32)


def messy_coo(rows, n_features, nnz, seed=5):
    """Unsorted COO with duplicates and empty rows -- the SpMM edge cases the reference never pins."""
    rng = np.random.default_rng(seed)
    r = rng.integers(0, rows, nnz)
    r[r % 7 == 3] = 0                       # leaves several rows empty, piles duplicates on row 0
    c = rng.integers(0, max(n_features // 3, 1), nnz)    # few columns -> many (row, col) duplicates
    v = rng.standard_normal(nnz).astype(F32)
    return sp.coo_matrix((v, (r, c)), shape=(rows, n_features))


def norm_tolerance(user_repr, item_repr, rel=1e-5):
    """|score error| bound: rel * |u| * |i| (scores cancel to ~0, so per-element relative error is meaningless)."""
    nu = np.linalg.norm(np.asarray(user_repr, dtype=np.float64), axis=-1)
    ni = np.linalg.norm(np.asarray(item_repr, dtype=np.float64), axis=-1)
    return rel * nu[..., :, None] * ni[None, :]


# ---- the fused training step (tests/test_train_{forms,losses}_*) --------------------------------------------------
def make_weights(uf, itf, d, n_tastes, attention, biased, seed):
    """Every weight of a model with these features, tastes, attention and biases (names as the model's)."""
    rng = np.random.default_rng(seed)
    w = {'linear_weights_item': (0.3 * rng.standard_normal((itf.shape[1], d))).astype(F32)}
    for t in range(n_tastes):
        w['linear_weights_user_{}'.format(t)] = (0.3 * rng.standard_normal((uf.shape[1], d))).astype(F32)
        if attention:
            w['linear_weights_attn_{}'.format(t)] = (0.3 * rng.standard_normal((uf.shape[1], d))).astype(F32)
    if biased:
        w['feature_biases_user'] = (0.2 * rng.standard_normal((uf.shape[1], 1))).astype(F32)
        w['feature_biases_item'] = (0.2 * rng.standard_normal((itf.shape[1], 1))).astype(F32)
    return w


def step_model(loss, prediction, user_norm, item_norm, n_tastes, attention, biased, d):
    """A TensorRec of one form of the fused step: loss 'wmrb' | 'balanced' | 'rmse' | 'separation', prediction 'dot' |
    'cosine' | 'euclidean', NormalizedLinear user / item graphs where *_norm, a Linear attention graph if attention."""
    import tensorrec_b200 as T
    from tensorrec_b200 import loss_graphs as L, prediction_graphs as P
    from tensorrec_b200.representation_graphs import LinearRepresentationGraph, NormalizedLinearRepresentationGraph
    losses = {'wmrb': L.WMRBLossGraph, 'balanced': L.BalancedWMRBLossGraph, 'rmse': L.RMSELossGraph,
              'separation': L.SeparationLossGraph}
    predictions = {'dot': P.DotProductPredictionGraph, 'cosine': P.CosineSimilarityPredictionGraph,
                   'euclidean': P.EuclideanSimilarityPredictionGraph}
    repr_graph = lambda norm: NormalizedLinearRepresentationGraph() if norm else LinearRepresentationGraph()  # noqa
    return T.TensorRec(n_components=d, n_tastes=n_tastes, user_repr_graph=repr_graph(user_norm),
                       item_repr_graph=repr_graph(item_norm),
                       attention_graph=LinearRepresentationGraph() if attention else None,
                       prediction_graph=predictions[prediction](), loss_graph=losses[loss](), biased=biased)


def make_model(prediction, user_norm, item_norm, n_tastes, attention, balanced, biased, d):
    """A WMRB (or BalancedWMRB) model of one form."""
    return step_model('balanced' if balanced else 'wmrb', prediction, user_norm, item_norm, n_tastes, attention, biased,
                      d)


def make_serial_model(loss, prediction, user_norm, item_norm, n_tastes, attention, biased, d):
    """An RMSE or Separation model of one form."""
    return step_model(loss, prediction, user_norm, item_norm, n_tastes, attention, biased, d)


def reference_example_models():
    """The WMRB configurations of the reference's examples (getting_started.py:98, check_movielens_losses.py:45-58,
    attention_example.py:27-41)."""
    import tensorrec_b200 as T
    from tensorrec_b200.loss_graphs import BalancedWMRBLossGraph, WMRBLossGraph
    from tensorrec_b200.prediction_graphs import (CosineSimilarityPredictionGraph, DotProductPredictionGraph,
                                                  EuclideanSimilarityPredictionGraph)
    from tensorrec_b200.representation_graphs import LinearRepresentationGraph, NormalizedLinearRepresentationGraph
    yield T.TensorRec(n_components=5, loss_graph=WMRBLossGraph())
    nl = NormalizedLinearRepresentationGraph
    for pred in (DotProductPredictionGraph, CosineSimilarityPredictionGraph, EuclideanSimilarityPredictionGraph):
        for nt in (1, 3):
            for lg in (WMRBLossGraph, BalancedWMRBLossGraph):
                yield T.TensorRec(n_components=10, n_tastes=nt, user_repr_graph=nl(), prediction_graph=pred(),
                                  loss_graph=lg())
    for att in (None, LinearRepresentationGraph()):
        yield T.TensorRec(n_components=10, n_tastes=3, user_repr_graph=nl(), attention_graph=att,
                          loss_graph=BalancedWMRBLossGraph())


def rough_interactions(n_users, n_items, seed, density=0.15):
    """Dummy interactions with explicit zeros, negative values and duplicate (user, item) entries, as COO in a mixed
    order: every stored entry is one interaction of the serial losses."""
    from tensorrec_b200 import util
    interactions, uf, itf = util.generate_dummy_data(num_users=n_users, num_items=n_items, interaction_density=density,
                                                     num_user_features=20, num_item_features=18,
                                                     n_features_per_user=5, n_features_per_item=4, seed=seed)
    coo = sp.coo_matrix(interactions)
    rng = np.random.default_rng(seed)
    val = coo.data.astype(F32).copy()
    val[rng.random(val.shape[0]) < 0.15] = 0.0
    neg = rng.random(val.shape[0]) < 0.15
    val[neg] = -np.abs(val[neg]) - 0.5
    dup = rng.choice(val.shape[0], max(1, val.shape[0] // 10), replace=False)
    row = np.concatenate([coo.row, coo.row[dup]])
    col = np.concatenate([coo.col, coo.col[dup]])
    val = np.concatenate([val, 2.0 * val[dup] + 0.25]).astype(F32)
    order = rng.permutation(row.shape[0])
    return sp.coo_matrix((val[order], (row[order], col[order])), shape=coo.shape), uf, itf


def kernel_step(model, weights, interactions, uf, itf, samples=None, bf16=False, lr=0.05, l2=0.0):
    """One WmrbStep.step of `model` from `weights` on device 0, with the caller's samples (int [n_users, n_sampled]
    item ids; a serial-loss model takes none): the stepper, and the loss and pred_serial on the host."""
    import torch
    from tensorrec_b200 import train_kernels as TK
    from tensorrec_b200.input_utils import SparseInput
    model.set_weights(weights)
    stepper = TK.WmrbStep(model, torch.device('cuda', 0), seed=3, bf16=bf16)
    st = None if samples is None else torch.from_numpy(np.ascontiguousarray(samples, dtype=np.int32)).cuda()
    loss, pred = stepper.step(SparseInput(interactions), SparseInput(uf), SparseInput(itf),
                              None if samples is None else samples.shape[1], lr, l2, samples=st)
    return stepper, loss.cpu().numpy(), pred.cpu().numpy()


def csr_order(interactions):
    """The step's (CSR) order of the interactions' COO entries."""
    return np.argsort(sp.coo_matrix(interactions).row, kind='stable')
