"""TEST INFRASTRUCTURE: numpy forward + analytic backward of the sampled-rank training step for every form the fused
step trains (DESIGN §3.10), the checker of tests/test_train_forms_gpu.py. It extends
oracle/loss_ops.wmrb_step_reference (dot, one taste, Linear) to the other forms and is pinned against torch autograd
over the host mirror of the reference's graph functions in tests/test_train_forms_cpu.py. float32 like the
reference's graph."""
import numpy as np

F32 = np.float32


# ---------------------------------------------------------------------------------------------------
# The sampled-rank training step for every form the fused step trains (DESIGN §3.10): dot / cosine / Euclidean
# prediction (prediction_graphs.py:52-55, 67-72, 102-117), Linear or NormalizedLinear user, item and attention
# representations (representation_graphs.py:32-58), n_tastes with max or attention collapse
# (recommendation_graphs.py:85-109, with the sampled items' attention taken from the user representation as
# tensorrec.py:367-372 does), biases and WMRB / BalancedWMRB as wmrb_step_reference.  Backward with TensorFlow's
# gradients: tf.maximum passes the gradient to its first argument where it is >= the second (the L2-normalisation
# clamp, the Euclidean clamp, the hinge), tf.reduce_max splits it evenly among tied maxima.
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


def sampled_rank_step_reference(user_features, item_features, interactions, weights, samples, prediction='dot',
                                normalize=(), n_tastes=1, attention=False, balanced=False, round_repr=None):
    """weights: name -> array as the model names them (linear_weights_user_<t>, linear_weights_attn_<t>,
    linear_weights_item, and feature_biases_user / feature_biases_item [n, 1] when the model is biased);
    prediction: 'dot' | 'cosine' | 'euclidean'; normalize: the sides ('user', 'item', 'attn') whose representation graph
    is NormalizedLinearRepresentationGraph; samples: int [n_users, n_sampled] item ids; round_repr as in
    wmrb_step_reference (applied to every operand row the pairs use; the gradient passes straight through it).

    Returns dict(loss [n_pos] (COO order of the positive interactions), pred_serial [nnz] (COO order), sample_pred
    [n_users, n_sampled], grads = name -> gradient of sum(loss) with the weight's shape, positive_mask)."""
    import scipy.sparse as sp
    uf, itf = sp.csr_matrix(user_features, dtype=F32), sp.csr_matrix(item_features, dtype=F32)
    coo = sp.coo_matrix(interactions)
    row, col, val = coo.row.astype(np.int64), coo.col.astype(np.int64), coo.data.astype(F32)
    n_users, n_items = uf.shape[0], itf.shape[0]
    samples = np.asarray(samples, dtype=np.int64)
    n_sampled = samples.shape[1]
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

    def forms(rows, pu, pi):                 # the pair's row form: u.i, or sum (u - i)^2
        if euclid:
            return np.sum(np.square(rows[pu] - item[pi]), axis=1, dtype=F32)
        return np.einsum('nk,nk->n', rows[pu], item[pi]).astype(F32)

    def score(f):
        return (-np.sqrt(np.maximum(f, F32(1e-16)))).astype(F32) if euclid else f

    su = np.repeat(np.arange(n_users), n_sampled)
    si = samples.reshape(-1)
    pu = np.concatenate([row, su])           # every pair: the interactions, then the samples
    pi = np.concatenate([col, si])
    is_sample = np.arange(pu.shape[0]) >= row.shape[0]
    f = np.stack([forms(users[t][0], pu, pi) for t in range(n_tastes)])               # [T, pairs]
    s = score(f)
    if attention:
        fa = np.stack([forms(attns[t][0], pu, pi) for t in range(n_tastes)])
        a = np.where(is_sample[None, :], s, score(fa))     # tensorrec.py:367-372: samples attend with the user rows
        e = np.exp(a - a.max(axis=0, keepdims=True)).astype(F32)
        w = (e / e.sum(axis=0, keepdims=True, dtype=F32)).astype(F32)
        pred = np.sum(w * s, axis=0, dtype=F32)
    elif n_tastes > 1:
        pred = s.max(axis=0)
    else:
        pred = s[0]
    if biased:
        pred = ((pred + ub[pu]) + ib[pi]).astype(F32)
    pred_serial = pred[:row.shape[0]]
    sample_pred = pred[row.shape[0]:].reshape(n_users, n_sampled)

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

    # backward of sum(loss): g = d / d prediction of every pair
    dsum = (weight / (smr + F32(1.0))).astype(F32)
    active = term >= 0.0
    g_int = np.zeros(row.shape[0], F32)
    g_int[mask] = -dsum * active.sum(axis=1).astype(F32)
    d_samp = np.zeros((n_users, n_sampled), dtype=F32)
    np.add.at(d_samp, prow, dsum[:, None] * active.astype(F32))
    g = np.concatenate([g_int, d_samp.reshape(-1)]).astype(F32)

    da = None
    if attention:
        ds = (g[None, :] * w).astype(F32)
        da = (ds * (s - np.sum(w * s, axis=0, dtype=F32)[None, :])).astype(F32)
        ds = np.where(is_sample[None, :], ds + da, ds).astype(F32)
        da = np.where(is_sample[None, :], F32(0.0), da).astype(F32)
    elif n_tastes > 1:
        ties = (s == s.max(axis=0, keepdims=True)).astype(F32)       # tf.reduce_max: split among the maxima
        ds = (g[None, :] * ties / ties.sum(axis=0, keepdims=True)).astype(F32)
    else:
        ds = g[None, :]

    d_item = np.zeros_like(item)

    def back(rows, f_rows, ds_rows):
        """d rows of one operand plane, and its share of d item."""
        c = np.where(f_rows >= F32(1e-16), ds_rows / np.sqrt(np.maximum(f_rows, F32(1e-16))), F32(0.0)).astype(F32) \
            if euclid else ds_rows
        d_rows = np.zeros_like(rows)
        if euclid:
            diff = (item[pi] - rows[pu]).astype(F32)                  # d score / d u = (i - u) / sqrt(f)
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
    return {'loss': loss, 'pred_serial': pred_serial, 'sample_pred': sample_pred, 'grads': grads,
            'positive_mask': mask}
