"""TEST INFRASTRUCTURE: numpy forward + analytic backward of the fused training step for every form it trains, the
checker of tests/test_train_forms_gpu.py and tests/test_train_losses_gpu.py.  The sampled-rank step (WMRB /
BalancedWMRB; DESIGN §3.10) and the serial-loss step (RMSE / Separation; DESIGN §3.11) share one forward of the pairs'
predictions and one backward from g = d loss / d prediction to the weight gradients; only the loss in between differs.
It extends oracle/loss_ops.wmrb_step_reference (dot, one taste, Linear) to the other forms and losses, and is pinned
against torch autograd over the host mirror of the reference's graph functions in tests/test_train_forms_cpu.py and
tests/test_train_losses_cpu.py.  Predictions are float32 like the reference's graph; the serial losses' statistics are
taken in float64, as the device's statistics kernels take them."""
import numpy as np
import scipy.sparse as sp

F32 = np.float32


# ---------------------------------------------------------------------------------------------------
# The forms the fused step trains (DESIGN §3.10): dot / cosine / Euclidean prediction (prediction_graphs.py:52-55,
# 67-72, 102-117), Linear or NormalizedLinear user, item and attention representations (representation_graphs.py:32-58),
# n_tastes with max or attention collapse (recommendation_graphs.py:85-109, with the sampled items' attention taken
# from the user representation as tensorrec.py:367-372 does) and biases.  Backward with TensorFlow's gradients:
# tf.maximum passes the gradient to its first argument where it is >= the second (the L2-normalisation clamp, the
# Euclidean clamp, the hinge), tf.reduce_max splits it evenly among tied maxima.
# ---------------------------------------------------------------------------------------------------
def _l2n_forward(x, n):
    """n row L2-normalisations x * rsqrt(max(sum x^2, 1e-12)); returns the output and, per normalisation, its input,
    rsqrt and whether the clamp was active."""
    levels = []
    for _ in range(n):
        ss = np.sum(x * x, axis=1, dtype=F32)
        scale = (F32(1.0) / np.sqrt(np.maximum(ss, F32(1e-12)))).astype(F32)
        levels.append((x, scale, ss < F32(1e-12)))
        x = (x * scale[:, None]).astype(F32)
    return x, levels


def _l2n_backward(levels, g):
    for x, scale, clamped in reversed(levels):
        xg = np.sum(x * g, axis=1, dtype=F32)
        t = np.where(clamped, F32(0.0), scale * scale * scale * xg).astype(F32)
        g = (scale[:, None] * g - t[:, None] * x).astype(F32)
    return g


class _Pairs(object):
    """The forward of the predictions of the pairs (pu[n], pi[n]) -- the interactions, then (sampled-rank step) the
    samples, the last n_samples pairs -- into .pred, and backward(g): the weight gradients of a loss whose gradient
    with respect to .pred is g.  Arguments as sampled_rank_step_reference."""

    def __init__(self, user_features, item_features, weights, pu, pi, n_samples, prediction, normalize, n_tastes,
                 attention, round_repr):
        self.uf, self.itf = sp.csr_matrix(user_features, dtype=F32), sp.csr_matrix(item_features, dtype=F32)
        self.pu, self.pi, self.n_tastes, self.attention = pu, pi, n_tastes, attention
        self.biased = 'feature_biases_user' in weights
        self.euclid = prediction == 'euclidean'
        cos = 1 if prediction == 'cosine' else 0

        def operand(features, name, side):
            raw = np.asarray(features @ np.asarray(weights[name], dtype=F32), dtype=F32)
            y, levels = _l2n_forward(raw, (1 if side in normalize else 0) + cos)
            return (round_repr(y) if round_repr is not None else y), levels

        uf, itf = self.uf, self.itf
        self.item, self.item_levels = operand(itf, 'linear_weights_item', 'item')
        self.users = [operand(uf, 'linear_weights_user_{}'.format(t), 'user') for t in range(n_tastes)]
        self.attns = [operand(uf, 'linear_weights_attn_{}'.format(t), 'attn') for t in range(n_tastes)] \
            if attention else []
        ub = np.asarray(uf @ np.asarray(weights['feature_biases_user'], F32).reshape(-1), F32) if self.biased else None
        ib = np.asarray(itf @ np.asarray(weights['feature_biases_item'], F32).reshape(-1), F32) if self.biased else None

        self.is_sample = np.arange(pu.shape[0]) >= pu.shape[0] - n_samples
        self.f = np.stack([self.forms(self.users[t][0]) for t in range(n_tastes)])          # [T, pairs]
        self.s = s = self.score(self.f)
        if attention:
            self.fa = np.stack([self.forms(self.attns[t][0]) for t in range(n_tastes)])
            a = np.where(self.is_sample[None, :], s, self.score(self.fa))   # samples attend with the user rows
            e = np.exp(a - a.max(axis=0, keepdims=True)).astype(F32)
            self.w = (e / e.sum(axis=0, keepdims=True, dtype=F32)).astype(F32)
            pred = np.sum(self.w * s, axis=0, dtype=F32)
        elif n_tastes > 1:
            pred = s.max(axis=0)
        else:
            pred = s[0]
        if self.biased:
            pred = ((pred + ub[pu]) + ib[pi]).astype(F32)
        self.pred = pred

    def forms(self, rows):
        """The pairs' row form of one operand plane: u.i, or sum (u - i)^2."""
        if self.euclid:
            return np.sum(np.square(rows[self.pu] - self.item[self.pi]), axis=1, dtype=F32)
        return np.einsum('nk,nk->n', rows[self.pu], self.item[self.pi]).astype(F32)

    def score(self, f):
        return (-np.sqrt(np.maximum(f, F32(1e-16)))).astype(F32) if self.euclid else f

    def backward(self, g):
        """name -> the gradient (the weight's shape) of the loss whose gradient with respect to every pair's
        prediction is g."""
        pu, pi, s, n_tastes, uf, itf = self.pu, self.pi, self.s, self.n_tastes, self.uf, self.itf
        da = None
        if self.attention:
            w = self.w
            ds = (g[None, :] * w).astype(F32)
            da = (ds * (s - np.sum(w * s, axis=0, dtype=F32)[None, :])).astype(F32)
            ds = np.where(self.is_sample[None, :], ds + da, ds).astype(F32)
            da = np.where(self.is_sample[None, :], F32(0.0), da).astype(F32)
        elif n_tastes > 1:
            ties = (s == s.max(axis=0, keepdims=True)).astype(F32)       # tf.reduce_max: split among the maxima
            ds = (g[None, :] * ties / ties.sum(axis=0, keepdims=True)).astype(F32)
        else:
            ds = g[None, :]

        item = self.item
        d_item = np.zeros_like(item)

        def back(rows, f_rows, ds_rows):
            """d rows of one operand plane, and its share of d item."""
            c = np.where(f_rows >= F32(1e-16), ds_rows / np.sqrt(np.maximum(f_rows, F32(1e-16))), F32(0.0)) \
                .astype(F32) if self.euclid else ds_rows
            d_rows = np.zeros_like(rows)
            if self.euclid:
                diff = (item[pi] - rows[pu]).astype(F32)                  # d score / d u = (i - u) / sqrt(f)
                np.add.at(d_rows, pu, c[:, None] * diff)
                np.add.at(d_item, pi, -c[:, None] * diff)
            else:
                np.add.at(d_rows, pu, c[:, None] * item[pi])
                np.add.at(d_item, pi, c[:, None] * rows[pu])
            return d_rows

        grads = {}
        for t in range(n_tastes):
            d_rows = back(self.users[t][0], self.f[t], ds[t])
            grads['linear_weights_user_{}'.format(t)] = np.asarray(uf.T @ _l2n_backward(self.users[t][1], d_rows), F32)
            if self.attention:
                d_rows = back(self.attns[t][0], self.fa[t], da[t])
                grads['linear_weights_attn_{}'.format(t)] = np.asarray(uf.T @ _l2n_backward(self.attns[t][1], d_rows),
                                                                       F32)
        grads['linear_weights_item'] = np.asarray(itf.T @ _l2n_backward(self.item_levels, d_item), F32)
        if self.biased:
            d_ub, d_ib = np.zeros(uf.shape[0], F32), np.zeros(itf.shape[0], F32)
            np.add.at(d_ub, pu, g)
            np.add.at(d_ib, pi, g)
            grads['feature_biases_user'] = np.asarray(uf.T @ d_ub, F32)[:, None]
            grads['feature_biases_item'] = np.asarray(itf.T @ d_ib, F32)[:, None]
        return grads


def sampled_rank_step_reference(user_features, item_features, interactions, weights, samples, prediction='dot',
                                normalize=(), n_tastes=1, attention=False, balanced=False, round_repr=None):
    """The sampled-rank step, WMRB / BalancedWMRB as wmrb_step_reference.  weights: name -> array as the model names
    them (linear_weights_user_<t>, linear_weights_attn_<t>, linear_weights_item, and feature_biases_user /
    feature_biases_item [n, 1] when the model is biased); prediction: 'dot' | 'cosine' | 'euclidean'; normalize: the
    sides ('user', 'item', 'attn') whose representation graph is NormalizedLinearRepresentationGraph; samples: int
    [n_users, n_sampled] item ids; round_repr as in wmrb_step_reference (applied to every operand row the pairs use;
    the gradient passes straight through it).

    Returns dict(loss [n_pos] (COO order of the positive interactions), pred_serial [nnz] (COO order), sample_pred
    [n_users, n_sampled], grads = name -> gradient of sum(loss) with the weight's shape, positive_mask)."""
    coo = sp.coo_matrix(interactions)
    row, col, val = coo.row.astype(np.int64), coo.col.astype(np.int64), coo.data.astype(F32)
    n_items = item_features.shape[0]
    samples = np.asarray(samples, dtype=np.int64)
    n_users, n_sampled = samples.shape
    pairs = _Pairs(user_features, item_features, weights, np.concatenate([row, np.repeat(np.arange(n_users), n_sampled)]),
                   np.concatenate([col, samples.reshape(-1)]), n_users * n_sampled, prediction, normalize, n_tastes,
                   attention, round_repr)
    pred_serial = pairs.pred[:row.shape[0]]
    sample_pred = pairs.pred[row.shape[0]:].reshape(n_users, n_sampled)

    mask = val > 0.0
    prow, pcol, pval = row[mask], col[mask], val[mask]
    term = (F32(1.0) - pred_serial[mask][:, None]) + sample_pred[prow]
    summed = np.sum(np.maximum(term, F32(0.0)), axis=1, dtype=F32)
    scale = F32(n_items) / F32(n_sampled)
    weight = np.full(prow.shape[0], scale, dtype=F32)
    smr = scale * summed
    if balanced:
        item_sum = np.zeros(n_items, dtype=F32)
        np.add.at(item_sum, pcol, pval)
        smr = smr * pval / item_sum[pcol]
        weight = weight * pval / item_sum[pcol]
    loss = np.log(smr + F32(1.0)).astype(F32)

    # g = d sum(loss) / d prediction of every pair
    dsum = (weight / (smr + F32(1.0))).astype(F32)
    active = term >= 0.0
    g_int = np.zeros(row.shape[0], F32)
    g_int[mask] = -dsum * active.sum(axis=1).astype(F32)
    d_samp = np.zeros((n_users, n_sampled), dtype=F32)
    np.add.at(d_samp, prow, dsum[:, None] * active.astype(F32))
    g = np.concatenate([g_int, d_samp.reshape(-1)]).astype(F32)
    return {'loss': loss, 'pred_serial': pred_serial, 'sample_pred': sample_pred, 'grads': pairs.backward(g),
            'positive_mask': mask}


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
    """The serial-loss step.  weights, prediction, normalize and round_repr as sampled_rank_step_reference; loss:
    'rmse' | 'separation'.  Every stored interaction counts, explicit zeros and duplicates included, in COO order.

    Returns dict(loss (scalar), pred_serial [nnz] (COO order), g [nnz] (d loss / d prediction), grads = name ->
    gradient of the loss with the weight's shape)."""
    coo = sp.coo_matrix(interactions)
    pairs = _Pairs(user_features, item_features, weights, coo.row.astype(np.int64), coo.col.astype(np.int64), 0,
                   prediction, normalize, n_tastes, attention, round_repr)
    value, g = serial_loss_coefficients(pairs.pred, coo.data.astype(F32), loss)
    return {'loss': value, 'pred_serial': pairs.pred, 'g': g, 'grads': pairs.backward(g)}
