"""TEST INFRASTRUCTURE: the fused training step of models with ReLURepresentationGraph sides (DESIGN §3.14), the
checker of tests/test_train_relu_gpu.py, pinned on the CPU against torch autograd over the host mirror
(tests/test_train_relu_cpu.py).

It reuses tests/train_step_oracle.py unchanged.  Every side's representation rows are formed first -- a ReLU side as
relu(X W1 + b) W2 in float64, a Linear side as X W -- and handed to that oracle as the "linear weights" of identity
features (projected biases likewise), so its gradients with respect to those weights are d loss / d rows (through the
normalisations).  The chain back through each side's layer is then taken by hand in float64:

    dZ = (d_rows W2^T) * [Z > 0],  Z = X W1 + b     (an exact 0 passes no gradient, as tf.nn.relu / torch.relu)
    d relu_weights = X^T dZ,  d relu_biases = sum_rows dZ,  d linear_weights = relu(Z)^T d_rows."""
import numpy as np
import scipy.sparse as sp

from tests.train_step_oracle import sampled_rank_step_reference, serial_loss_step_reference

F32 = np.float32


def side_ends(n_tastes, attention):
    """The sides in the creation order of the reference's graph: item, then user_<t> (and attn_<t>) per taste."""
    ends = ['item']
    for t in range(n_tastes):
        ends.append('user_{}'.format(t))
        if attention:
            ends.append('attn_{}'.format(t))
    return ends


def relu_layer_reference(x, w1, b, w2):
    """float64 (Z = x W1 + b, relu(Z), relu(Z) W2) of one ReLU side; x a scipy matrix or an array."""
    z = np.asarray(x @ np.asarray(w1, np.float64), np.float64) + np.asarray(b, np.float64).reshape(1, -1)
    h = np.maximum(z, 0.0)
    return z, h, h @ np.asarray(w2, np.float64)


def relu_layer_backward_reference(z, h, w2, d_out):
    """float64 (dZ, d relu_biases [H], d linear_weights [H, d]) of relu_layer_reference for d_out = d loss / d out."""
    d_out = np.asarray(d_out, np.float64)
    dz = (d_out @ np.asarray(w2, np.float64).T) * (z > 0.0)
    return dz, dz.sum(axis=0), h.T @ d_out


def relu_step_reference(user_features, item_features, interactions, weights, relu_sides, samples=None, loss='wmrb',
                        prediction='dot', normalize=(), n_tastes=1, attention=False, balanced=False, round_repr=None):
    """One step of a model whose `relu_sides` ('user', 'item', 'attn') are ReLURepresentationGraph and whose other
    sides are Linear (NormalizedLinear where listed in `normalize`).  loss 'wmrb' (BalancedWMRB with balanced=True;
    samples int [n_users, n_sampled]) or 'rmse' / 'separation'.  weights: name -> array as the model names them.

    Returns the inner oracle's dict (loss, pred_serial, ...) with grads = name -> float64 gradient of every weight and
    d_rows = end -> d loss / d (pre-normalisation) representation rows of each side."""
    uf = sp.csr_matrix(user_features, dtype=np.float64)
    itf = sp.csr_matrix(item_features, dtype=np.float64)
    ends = side_ends(n_tastes, attention)
    rows, layers, lin = {}, {}, {}
    for end in ends:
        x = itf if end == 'item' else uf
        if end.split('_')[0] in relu_sides:
            z, h, r = relu_layer_reference(x, weights['relu_weights_' + end], weights['relu_biases_' + end],
                                           weights['linear_weights_' + end])
            layers[end] = (z, h)
        else:
            r = np.asarray(x @ np.asarray(weights['linear_weights_' + end], np.float64), np.float64)
        rows[end] = r
        lin['linear_weights_' + end] = r.astype(F32)
    biased = 'feature_biases_user' in weights
    if biased:
        lin['feature_biases_user'] = np.asarray(uf @ np.asarray(weights['feature_biases_user'], np.float64), F32)
        lin['feature_biases_item'] = np.asarray(itf @ np.asarray(weights['feature_biases_item'], np.float64), F32)
    eye_u = sp.identity(uf.shape[0], dtype=F32, format='csr')
    eye_i = sp.identity(itf.shape[0], dtype=F32, format='csr')
    kw = dict(prediction=prediction, normalize=normalize, n_tastes=n_tastes, attention=attention, round_repr=round_repr)
    if loss == 'wmrb':
        ref = sampled_rank_step_reference(eye_u, eye_i, interactions, lin, samples, balanced=balanced, **kw)
    else:
        ref = serial_loss_step_reference(eye_u, eye_i, interactions, lin, loss=loss, **kw)

    grads, d_rows = {}, {}
    for end in ends:
        x = itf if end == 'item' else uf
        g = np.asarray(ref['grads']['linear_weights_' + end], np.float64)
        d_rows[end] = g
        if end in layers:
            z, h = layers[end]
            dz, db, dw2 = relu_layer_backward_reference(z, h, weights['linear_weights_' + end], g)
            grads['relu_weights_' + end] = np.asarray(x.T @ dz)
            grads['relu_biases_' + end] = db.reshape(1, -1)
            grads['linear_weights_' + end] = dw2
        else:
            grads['linear_weights_' + end] = np.asarray(x.T @ g)
    if biased:
        grads['feature_biases_user'] = np.asarray(uf.T @ np.asarray(ref['grads']['feature_biases_user'], np.float64))
        grads['feature_biases_item'] = np.asarray(itf.T @ np.asarray(ref['grads']['feature_biases_item'], np.float64))
    return dict(ref, grads=grads, d_rows=d_rows, rows=rows)


def relu_weights(uf, itf, d, hidden, relu_sides, n_tastes, attention, biased, seed):
    """Every weight of such a model (names as the model's): ReLU sides with W1 and W2 of the scale of the reference's
    initialiser and small non-zero hidden biases, Linear sides as tests/helpers.make_weights."""
    rng = np.random.default_rng(seed)
    w = {}
    for end in side_ends(n_tastes, attention):
        n_features = itf.shape[1] if end == 'item' else uf.shape[1]
        if end.split('_')[0] in relu_sides:
            w['relu_weights_' + end] = (0.5 * rng.standard_normal((n_features, hidden))).astype(F32)
            w['relu_biases_' + end] = (0.1 * rng.standard_normal((1, hidden))).astype(F32)
            w['linear_weights_' + end] = ((0.5 / np.sqrt(hidden)) * rng.standard_normal((hidden, d))).astype(F32)
        else:
            w['linear_weights_' + end] = (0.3 * rng.standard_normal((n_features, d))).astype(F32)
    if biased:
        w['feature_biases_user'] = (0.2 * rng.standard_normal((uf.shape[1], 1))).astype(F32)
        w['feature_biases_item'] = (0.2 * rng.standard_normal((itf.shape[1], 1))).astype(F32)
    return w


def relu_model(loss, prediction, relu_sides, user_norm, n_tastes, attention, biased, d, relu_size=None):
    """A TensorRec whose `relu_sides` are ReLURepresentationGraph(relu_size), the others Linear (the user graph
    NormalizedLinear if user_norm); loss 'wmrb' | 'balanced' | 'rmse' | 'separation'."""
    import tensorrec_b200 as T
    from tensorrec_b200 import loss_graphs as L, prediction_graphs as P
    from tensorrec_b200.representation_graphs import (LinearRepresentationGraph, NormalizedLinearRepresentationGraph,
                                                      ReLURepresentationGraph)
    losses = {'wmrb': L.WMRBLossGraph, 'balanced': L.BalancedWMRBLossGraph, 'rmse': L.RMSELossGraph,
              'separation': L.SeparationLossGraph}
    predictions = {'dot': P.DotProductPredictionGraph, 'cosine': P.CosineSimilarityPredictionGraph,
                   'euclidean': P.EuclideanSimilarityPredictionGraph}

    def graph(side, norm=False):
        if side in relu_sides:
            return ReLURepresentationGraph(relu_size=relu_size)
        return NormalizedLinearRepresentationGraph() if norm else LinearRepresentationGraph()

    return T.TensorRec(n_components=d, n_tastes=n_tastes, user_repr_graph=graph('user', user_norm),
                       item_repr_graph=graph('item'), attention_graph=graph('attn') if attention else None,
                       prediction_graph=predictions[prediction](), loss_graph=losses[loss](), biased=biased)
