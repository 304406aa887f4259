"""TEST INFRASTRUCTURE: numpy forward + analytic backward of the serial-loss training step (RMSELossGraph,
SeparationLossGraph; DESIGN §3.11) for every form the fused step trains, the checker of tests/test_train_losses_gpu.py.
It is pinned against torch autograd over the host mirror of the reference's graph functions in
tests/test_train_losses_cpu.py.  Predictions are float32 like the reference's graph; the loss statistics are taken in
float64, as the device's statistics kernels take them."""
import numpy as np
import scipy.sparse as sp

from tests.train_forms_oracle import _l2n_backward, _l2n_forward

F32 = np.float32


def serial_loss_coefficients(pred, val, loss):
    """The scalar loss and g = d loss / d pred of every interaction (float64 statistics, float32 g):
    RMSE        L = sqrt(mean (y - p)^2), g = (p - y) / (N L);
    Separation  L = 1 - Phi(-loc / sigma) over P = {y > 0} and Q = {y <= 0}, loc = mu_Q - mu_P,
                sigma = sqrt(v_Q + v_P) (biased variances), phi the normal density at -loc / sigma,
                g = -(phi / (sigma |P|)) (1 + loc (p - mu_P) / sigma^2) on P,
                g =  (phi / (sigma |Q|)) (1 - loc (p - mu_Q) / sigma^2) on Q.
    Empty inputs and groups give NaN, as the means of nothing do."""
    from math import erf
    p, y = np.asarray(pred, np.float64), np.asarray(val, np.float64)
    with np.errstate(invalid='ignore', divide='ignore'):
        if loss == 'rmse':
            n = p.shape[0]
            value = np.sqrt(np.sum((y - p) ** 2) / n) if n else np.nan
            return F32(value), ((p - y) / (n * value)).astype(F32)
        pos = y > 0
        groups = []
        for mask in (pos, ~pos):
            n = int(mask.sum())
            mu = p[mask].mean() if n else np.nan
            var = np.mean((p[mask] - mu) ** 2) if n else np.nan
            groups.append((n, mu, var))
        (n_p, mu_p, v_p), (n_q, mu_q, v_q) = groups
        loc = mu_q - mu_p
        var = v_q + v_p
        sigma = np.sqrt(var)
        z = -loc / sigma
        value = 1.0 - 0.5 * (1.0 + erf(z / np.sqrt(2.0))) if np.isfinite(z) else np.nan
        phi = np.exp(-0.5 * z * z) / np.sqrt(2.0 * np.pi)
        g = np.where(pos, -(phi / (sigma * n_p)) * (1.0 + loc * (p - mu_p) / var),
                     (phi / (sigma * n_q)) * (1.0 - loc * (p - mu_q) / var))
        return F32(value), g.astype(F32)


def serial_loss_step_reference(user_features, item_features, interactions, weights, loss='rmse', prediction='dot',
                               normalize=(), n_tastes=1, attention=False, round_repr=None):
    """weights: name -> array as the model names them (as train_forms_oracle.sampled_rank_step_reference);
    loss: 'rmse' | 'separation'; prediction: 'dot' | 'cosine' | 'euclidean'; normalize: the sides ('user', 'item',
    'attn') whose representation graph is NormalizedLinearRepresentationGraph; round_repr: applied to every operand
    row (the gradient passes straight through it).  Every stored interaction counts, explicit zeros and duplicates
    included, in COO order.

    Returns dict(loss (scalar), pred_serial [nnz] (COO order), g [nnz] (d loss / d prediction), grads = name ->
    gradient of the loss with the weight's shape)."""
    uf, itf = sp.csr_matrix(user_features, dtype=F32), sp.csr_matrix(item_features, dtype=F32)
    coo = sp.coo_matrix(interactions)
    pu, pi, val = coo.row.astype(np.int64), coo.col.astype(np.int64), coo.data.astype(F32)
    n_users, n_items = uf.shape[0], itf.shape[0]
    biased = 'feature_biases_user' in weights
    cos = 1 if prediction == 'cosine' else 0
    euclid = prediction == 'euclidean'

    def operand(features, name, side):
        raw = np.asarray(features @ np.asarray(weights[name], dtype=F32), dtype=F32)
        y, levels = _l2n_forward(raw, (1 if side in normalize else 0) + cos)
        return (round_repr(y) if round_repr is not None else y), levels

    item, item_levels = operand(itf, 'linear_weights_item', 'item')
    users = [operand(uf, 'linear_weights_user_{}'.format(t), 'user') for t in range(n_tastes)]
    attns = [operand(uf, 'linear_weights_attn_{}'.format(t), 'attn') for t in range(n_tastes)] if attention else []
    ub = np.asarray(uf @ np.asarray(weights['feature_biases_user'], F32).reshape(-1), F32) if biased else None
    ib = np.asarray(itf @ np.asarray(weights['feature_biases_item'], F32).reshape(-1), F32) if biased else None

    def forms(rows):                         # the pair's row form: u.i, or sum (u - i)^2
        if euclid:
            return np.sum(np.square(rows[pu] - item[pi]), axis=1, dtype=F32)
        return np.einsum('nk,nk->n', rows[pu], item[pi]).astype(F32)

    def score(f):
        return (-np.sqrt(np.maximum(f, F32(1e-16)))).astype(F32) if euclid else f

    f = np.stack([forms(users[t][0]) for t in range(n_tastes)]).reshape(n_tastes, -1)       # [T, nnz]
    s = score(f)
    if attention:
        fa = np.stack([forms(attns[t][0]) for t in range(n_tastes)]).reshape(n_tastes, -1)
        a = score(fa)
        e = np.exp(a - a.max(axis=0, keepdims=True)).astype(F32)
        w = (e / e.sum(axis=0, keepdims=True, dtype=F32)).astype(F32)
        pred = np.sum(w * s, axis=0, dtype=F32)
    elif n_tastes > 1:
        pred = s.max(axis=0)
    else:
        pred = s[0]
    if biased:
        pred = ((pred + ub[pu]) + ib[pi]).astype(F32)

    value, g = serial_loss_coefficients(pred, val, loss)

    if attention:
        ds = (g[None, :] * w).astype(F32)
        da = (ds * (s - np.sum(w * s, axis=0, dtype=F32)[None, :])).astype(F32)
    elif n_tastes > 1:
        ties = (s == s.max(axis=0, keepdims=True)).astype(F32)       # tf.reduce_max: split among the maxima
        ds = (g[None, :] * ties / ties.sum(axis=0, keepdims=True)).astype(F32)
    else:
        ds = g[None, :]

    d_item = np.zeros_like(item)

    def back(rows, f_rows, ds_rows):
        c = np.where(f_rows >= F32(1e-16), ds_rows / np.sqrt(np.maximum(f_rows, F32(1e-16))), F32(0.0)).astype(F32) \
            if euclid else ds_rows
        d_rows = np.zeros_like(rows)
        if euclid:
            diff = (item[pi] - rows[pu]).astype(F32)
            np.add.at(d_rows, pu, c[:, None] * diff)
            np.add.at(d_item, pi, -c[:, None] * diff)
        else:
            np.add.at(d_rows, pu, c[:, None] * item[pi])
            np.add.at(d_item, pi, c[:, None] * rows[pu])
        return d_rows

    grads = {}
    for t in range(n_tastes):
        d_rows = back(users[t][0], f[t], ds[t])
        grads['linear_weights_user_{}'.format(t)] = np.asarray(uf.T @ _l2n_backward(users[t][1], d_rows), F32)
        if attention:
            d_rows = back(attns[t][0], fa[t], da[t])
            grads['linear_weights_attn_{}'.format(t)] = np.asarray(uf.T @ _l2n_backward(attns[t][1], d_rows), F32)
    grads['linear_weights_item'] = np.asarray(itf.T @ _l2n_backward(item_levels, d_item), F32)
    if biased:
        d_ub, d_ib = np.zeros(n_users, F32), np.zeros(n_items, F32)
        np.add.at(d_ub, pu, g)
        np.add.at(d_ib, pi, g)
        grads['feature_biases_user'] = np.asarray(uf.T @ d_ub, F32)[:, None]
        grads['feature_biases_item'] = np.asarray(itf.T @ d_ib, F32)[:, None]
    return {'loss': value, 'pred_serial': pred, 'g': g, 'grads': grads}
