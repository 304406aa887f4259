"""
TEST INFRASTRUCTURE (see oracle/__init__.py).  numpy/scipy restatement of the reference ops on the
predict / predict_rank path.  Every function cites the reference lines it follows
(paths relative to the root of jfkirk/tensorrec @ 80690737).  All arithmetic is float32, like the reference's TF graph
(tensorrec/input_utils.py:34 casts values to float32; every tf.Variable is float32).

TensorFlow op semantics encoded here (TF is a third-party dependency of the reference, not vendored;
constraint tensorflow>=1.7.0, setup.py:21):
  * tf.sparse_tensor_dense_matmul: out[row] += val * W[col] for every COO entry, duplicates summed,
    float32 accumulation in index order.
  * tf.nn.l2_normalize(x, 1): x * rsqrt(max(sum(x**2, axis=1), 1e-12)).
  * tf.nn.top_k: descending values, equal values ordered by LOWER index first, int32 indices.
"""
import numpy as np
import scipy.sparse as sp

F32 = np.float32
L2_EPSILON = F32(1e-12)  # tf.nn.l2_normalize default epsilon


# ---------------------------------------------------------------------------------------------------
# a1: input coercion -- tensorrec/input_utils.py:22-40, tensorrec/tensorrec.py:285-293
# ---------------------------------------------------------------------------------------------------
def coo_from_sparse(matrix):
    """Any scipy sparse matrix -> (row i64[nnz], col i64[nnz], val f32[nnz], d0, d1) in COO order as given.

    tensorrec/input_utils.py:29-36: non-COO inputs go through sp.coo_matrix(); order is whatever that
    conversion yields (row-major for CSR); duplicates are kept."""
    if not isinstance(matrix, sp.coo_matrix):
        matrix = sp.coo_matrix(matrix)
    return (np.asarray(matrix.row, dtype=np.int64), np.asarray(matrix.col, dtype=np.int64),
            np.asarray(matrix.data, dtype=F32), int(matrix.shape[0]), int(matrix.shape[1]))


# ---------------------------------------------------------------------------------------------------
# a2 / a3: representation graphs -- tensorrec/representation_graphs.py:32-58
# ---------------------------------------------------------------------------------------------------
def sparse_dense_matmul(coo, weights):
    """tf.sparse_tensor_dense_matmul(SparseTensor(coo), weights) (representation_graphs.py:40).

    Sequential float32 multiply-then-add in COO order; duplicates are summed."""
    row, col, val, d0, _ = coo
    weights = np.ascontiguousarray(weights, dtype=F32)
    out = np.zeros((d0, weights.shape[1]), dtype=F32)
    # ufunc.at is unbuffered and applies the entries one after another, in the order given
    np.add.at(out, row, (val[:, None] * weights[col]).astype(F32))
    return out


def sparse_dense_matmul_fast(csr, weights):
    """Same contraction through scipy's CSR kernel (row-major order, sequential per row).  Used only
    where the oracle is TIMED (bench cpu_baseline); tests check it against sparse_dense_matmul."""
    return np.asarray(csr.astype(F32) @ np.ascontiguousarray(weights, dtype=F32), dtype=F32)


def l2_normalize(x, eps=L2_EPSILON):
    """tf.nn.l2_normalize(x, 1) (representation_graphs.py:36,57; recommendation_graphs.py:119-120)."""
    x = np.asarray(x, dtype=F32)
    square_sum = np.sum(np.square(x), axis=1, keepdims=True, dtype=F32)
    inv_norm = (F32(1.0) / np.sqrt(np.maximum(square_sum, eps))).astype(F32)
    return (x * inv_norm).astype(F32)


def linear_representation(coo, weights):
    """LinearRepresentationGraph.connect_representation_graph (representation_graphs.py:32-43)."""
    return sparse_dense_matmul(coo, weights)


def normalized_linear_representation(coo, weights):
    """NormalizedLinearRepresentationGraph (representation_graphs.py:53-58)."""
    return l2_normalize(sparse_dense_matmul(coo, weights))


# ---------------------------------------------------------------------------------------------------
# a4 / a5: dense prediction graphs -- tensorrec/prediction_graphs.py:49-50, 64-65, 84-100
# ---------------------------------------------------------------------------------------------------
def dot_product_dense(user_repr, item_repr):
    """DotProductPredictionGraph.connect_dense_prediction_graph (prediction_graphs.py:49-50)."""
    return np.matmul(np.asarray(user_repr, dtype=F32), np.asarray(item_repr, dtype=F32).T).astype(F32)


def cosine_dense(user_repr, item_repr):
    """CosineSimilarityPredictionGraph dense (prediction_graphs.py:64-65) -> relative_cosine
    (recommendation_graphs.py:112-121)."""
    return dot_product_dense(l2_normalize(user_repr), l2_normalize(item_repr))


def euclidean_dense(user_repr, item_repr, epsilon=1e-16):
    """EuclideanSimilarityPredictionGraph dense (prediction_graphs.py:84-100)."""
    u = np.asarray(user_repr, dtype=F32)
    i = np.asarray(item_repr, dtype=F32)
    r_user = np.sum(u ** 2, axis=1, keepdims=True, dtype=F32)
    r_item = np.sum(i ** 2, axis=1, keepdims=True, dtype=F32)
    distance = (r_user - F32(2.0) * np.matmul(u, i.T) + r_item.T).astype(F32)
    distance = np.maximum(distance, F32(epsilon))
    return (F32(-1.0) * np.sqrt(distance)).astype(F32)


# ---------------------------------------------------------------------------------------------------
# f1 (training step, SURVEY 8f): the serial forms -- one prediction per (user, item) index pair
# ---------------------------------------------------------------------------------------------------
def dot_product_serial(user_repr, item_repr, x_user, x_item):
    """DotProductPredictionGraph.connect_serial_prediction_graph (prediction_graphs.py:52-55): gather both rows,
    multiply elementwise, reduce_sum over the components."""
    u = np.asarray(user_repr, dtype=F32)[np.asarray(x_user)]
    i = np.asarray(item_repr, dtype=F32)[np.asarray(x_item)]
    return np.sum(u * i, axis=1, dtype=F32)


def cosine_serial(user_repr, item_repr, x_user, x_item):
    """CosineSimilarityPredictionGraph serial (prediction_graphs.py:67-72): l2_normalize rows, then the dot form."""
    return dot_product_serial(l2_normalize(user_repr), l2_normalize(item_repr), x_user, x_item)


def euclidean_serial(user_repr, item_repr, x_user, x_item, epsilon=1e-16):
    """EuclideanSimilarityPredictionGraph serial (prediction_graphs.py:102-117): -sqrt(max(sum((u - i)^2), eps))."""
    u = np.asarray(user_repr, dtype=F32)[np.asarray(x_user)]
    i = np.asarray(item_repr, dtype=F32)[np.asarray(x_item)]
    distance = np.maximum(np.sum((u - i) ** 2, axis=1, dtype=F32), F32(epsilon))
    return (F32(-1.0) * np.sqrt(distance)).astype(F32)


def split_sparse_tensor_indices(matrix):
    """split_sparse_tensor_indices (recommendation_graphs.py:22-30) of the SparseTensor built from a scipy matrix
    (tensorrec.py:285-293): the row and the column index of every stored entry, in COO order."""
    row, col = coo_from_sparse(matrix)[:2]
    return row, col


def bias_prediction_serial(prediction_serial, projected_user_biases, projected_item_biases, x_user, x_item):
    """pred + gather(ub, x_user) + gather(ib, x_item), left to right (recommendation_graphs.py:44-57)."""
    p = np.asarray(prediction_serial, dtype=F32)
    ub = np.asarray(projected_user_biases, dtype=F32)[np.asarray(x_user)]
    ib = np.asarray(projected_item_biases, dtype=F32)[np.asarray(x_item)]
    return ((p + ub).astype(F32) + ib).astype(F32)


def densify_sampled_item_predictions(sample_predictions_serial, n_sampled_items, n_users):
    """reshape to [n_users, n_sampled_items] (recommendation_graphs.py:60-70)."""
    return np.asarray(sample_predictions_serial).reshape(int(n_users), int(n_sampled_items))


# ---------------------------------------------------------------------------------------------------
# a6: taste collapse -- tensorrec/recommendation_graphs.py:85-109
# ---------------------------------------------------------------------------------------------------
def collapse_mixture_of_tastes(tastes_predictions, tastes_attentions=None):
    stacked = np.stack([np.asarray(p, dtype=F32) for p in tastes_predictions])
    if tastes_attentions is not None:
        att = np.stack([np.asarray(a, dtype=F32) for a in tastes_attentions])
        att = att - np.max(att, axis=0, keepdims=True)        # tf.nn.softmax is max-shifted
        e = np.exp(att).astype(F32)
        soft = (e / np.sum(e, axis=0, keepdims=True, dtype=F32)).astype(F32)
        return np.sum(stacked * soft, axis=0, dtype=F32)      # recommendation_graphs.py:102-103
    return np.max(stacked, axis=0)                            # recommendation_graphs.py:107


# ---------------------------------------------------------------------------------------------------
# a7 / a8: biases -- tensorrec/recommendation_graphs.py:4-19, 33-41
# ---------------------------------------------------------------------------------------------------
def project_biases(coo, feature_biases):
    """reduce_sum(SparseTensor @ b[F,1], axis=1) (recommendation_graphs.py:13-17)."""
    b = np.asarray(feature_biases, dtype=F32).reshape(-1, 1)
    return sparse_dense_matmul(coo, b)[:, 0]


def bias_prediction_dense(prediction, projected_user_biases, projected_item_biases):
    """pred + ub[:, None] + ib[None, :], left to right (recommendation_graphs.py:41)."""
    p = np.asarray(prediction, dtype=F32)
    ub = np.asarray(projected_user_biases, dtype=F32)
    ib = np.asarray(projected_item_biases, dtype=F32)
    return ((p + ub[:, None]).astype(F32) + ib[None, :]).astype(F32)


# ---------------------------------------------------------------------------------------------------
# a9: ranking -- tensorrec/recommendation_graphs.py:73-82
# ---------------------------------------------------------------------------------------------------
def rank_predictions(prediction):
    """The literal double sort.  tf.nn.top_k(x, k=n).indices == stable argsort of -x (equal values keep
    ascending index order); the second top_k of the negated int32 indices is the inverse permutation."""
    p = np.asarray(prediction, dtype=F32)
    indices_of_ranks = np.argsort(-p, axis=1, kind='stable').astype(np.int32)           # :81
    return (np.argsort(indices_of_ranks, axis=1, kind='stable') + 1).astype(np.int32)   # :82  (-(-x))


def rank_predictions_closed_form(prediction):
    """rank[u,i] = 1 + #{j: s_j > s_i} + #{j < i: s_j == s_i}.  O(I^2) per row: small cases only."""
    p = np.asarray(prediction, dtype=F32)
    n = p.shape[1]
    greater = (p[:, None, :] > p[:, :, None]).sum(axis=2)
    lower_index = np.tril(np.ones((n, n), dtype=bool), k=-1)      # [i, j] true when j < i
    equal_before = ((p[:, None, :] == p[:, :, None]) & lower_index[None]).sum(axis=2)
    return (1 + greater + equal_before).astype(np.int32)


def top_k_from_scores(prediction, k):
    """The items whose reference rank is 1..k, in rank order, with their scores.
    Equivalent to selecting rank_predictions(prediction) <= k (eval.py:23,49 only ever test that)."""
    p = np.asarray(prediction, dtype=F32)
    order = np.argsort(-p, axis=1, kind='stable')[:, :k].astype(np.int32)
    return order, np.take_along_axis(p, order, axis=1)


def top_k_from_scores_fast(prediction, k):
    """Same result as top_k_from_scores without sorting whole rows: an argpartition finds the k-th best score, every
    entry >= it is kept and those few are ordered by (score descending, index ascending) -- the order the reference's
    double tf.nn.top_k (recommendation_graphs.py:81-82) gives the entries with rank <= k.  Checked against
    top_k_from_scores in tests/test_oracle.py; used where the oracle ranks thousands of users against 1M items."""
    p = np.asarray(prediction, dtype=F32)
    n_rows, n_cols = p.shape
    k = min(int(k), n_cols)
    ids = np.empty((n_rows, k), dtype=np.int32)
    vals = np.empty((n_rows, k), dtype=F32)
    for r in range(n_rows):
        row = p[r]
        kth = np.partition(row, n_cols - k)[n_cols - k]           # the k-th largest value
        cand = np.nonzero(row >= kth)[0]                          # ascending indices, >= k of them (ties at the k-th)
        order = np.lexsort((cand, -row[cand].astype(np.float64)))[:k]
        ids[r] = cand[order]
        vals[r] = row[cand[order]]
    return ids, vals


# ---------------------------------------------------------------------------------------------------
# a10: composition -- tensorrec/tensorrec.py:307-313, 339-346, 380-383, 406-410, 421-435, 454
# ---------------------------------------------------------------------------------------------------
class OracleModel(object):
    """Holds injected weights and evaluates the reference's predict graph in the reference's order.

    user_weights: list (one per taste) of f32[F_user, d]; item_weights f32[F_item, d];
    user_bias / item_bias: f32[F] or None (biased=False); attention_weights: list per taste or None.
    user_repr / item_repr / attention_repr: 'linear' | 'normalized_linear'; prediction: 'dot' | 'cosine'
    | 'euclidean'."""

    def __init__(self, user_weights, item_weights, user_bias=None, item_bias=None, attention_weights=None,
                 user_repr='linear', item_repr='linear', attention_repr='linear', prediction='dot'):
        self.user_weights = [np.asarray(w, dtype=F32) for w in user_weights]
        self.item_weights = np.asarray(item_weights, dtype=F32)
        self.user_bias = None if user_bias is None else np.asarray(user_bias, dtype=F32)
        self.item_bias = None if item_bias is None else np.asarray(item_bias, dtype=F32)
        self.attention_weights = None if attention_weights is None else \
            [np.asarray(w, dtype=F32) for w in attention_weights]
        self.user_repr, self.item_repr, self.attention_repr = user_repr, item_repr, attention_repr
        self.prediction = prediction

    @staticmethod
    def _repr(kind, coo, w):
        if kind == 'linear':
            return linear_representation(coo, w)
        if kind == 'normalized_linear':
            return normalized_linear_representation(coo, w)
        raise ValueError(kind)

    def _pred(self, u, i):
        return {'dot': dot_product_dense, 'cosine': cosine_dense, 'euclidean': euclidean_dense}[self.prediction](u, i)

    def item_representation(self, item_features):
        return self._repr(self.item_repr, coo_from_sparse(item_features), self.item_weights)

    def user_representation(self, user_features):
        coo = coo_from_sparse(user_features)
        return np.stack([self._repr(self.user_repr, coo, w) for w in self.user_weights])

    def predict(self, user_features, item_features):
        ucoo, icoo = coo_from_sparse(user_features), coo_from_sparse(item_features)
        item_repr = self._repr(self.item_repr, icoo, self.item_weights)                 # tensorrec.py:308-312
        preds, atts = [], (None if self.attention_weights is None else [])
        for t, w in enumerate(self.user_weights):                                       # :339-346
            user_repr = self._repr(self.user_repr, ucoo, w)
            if atts is not None:                                                        # :349-360
                att_repr = self._repr(self.attention_repr, ucoo, self.attention_weights[t])
                atts.append(self._pred(att_repr, item_repr))
            preds.append(self._pred(user_repr, item_repr))                              # :380-383
        pred = collapse_mixture_of_tastes(preds, atts)                                  # :407-410
        if self.user_bias is not None:                                                  # :421-435
            pred = bias_prediction_dense(pred, project_biases(ucoo, self.user_bias),
                                         project_biases(icoo, self.item_bias))
        return pred

    def predict_rank(self, user_features, item_features):
        return rank_predictions(self.predict(user_features, item_features))             # :454


def predict(model, user_features, item_features):
    return model.predict(user_features, item_features)


def predict_rank(model, user_features, item_features):
    return model.predict_rank(user_features, item_features)


def predict_similar_items(prediction, item_repr, item_ids):
    """recommendation_graphs.py:124-137: gather rows, then the dense prediction graph."""
    item_repr = np.asarray(item_repr, dtype=F32)
    gathered = item_repr[np.asarray(item_ids, dtype=np.int64)]
    return {'dot': dot_product_dense, 'cosine': cosine_dense, 'euclidean': euclidean_dense}[prediction](
        gathered, item_repr)
