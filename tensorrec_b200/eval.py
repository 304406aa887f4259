"""Ranking metrics over predict_rank output (API of tensorrec/eval.py).

Consumers of the hot path, host-side numpy/scipy.  The reference builds `predicted_ranks * positive.A` dense
(eval.py:22,48) and only ever tests `rank <= k` (eval.py:23,49,68-69); that is what makes the top-k output of
predict_rank(k=...) sufficient: every function here accepts the full int32 rank matrix, a TopK result, or a scipy
sparse rank matrix such as predict_rank_at returns -- the ranks of the test positives only, exact at any k (a positive
without a stored rank raises ValueError).  fit_and_eval keeps the reference's full predict_rank."""
import numpy as np
import scipy.sparse as sp


def _ranks_of_positives(predicted_ranks, positive):
    """csr matrix with the predicted rank of every positive test interaction (0 entries are not stored).

    For a TopK input, positives outside the top-k get rank n_items + 1 (any value > k would do).  A scipy sparse input
    (predict_rank_at) must hold a rank for every positive: a missing entry would read as rank 0, a hit at every k."""
    positive = sp.csr_matrix(positive)
    if sp.issparse(predicted_ranks):
        ranks = sp.csr_matrix(predicted_ranks)
        if ranks.shape != positive.shape:
            raise ValueError('the rank matrix has shape %s but the interactions have %s' % (ranks.shape, positive.shape))
        stored = sp.csr_matrix(positive != 0).multiply(ranks != 0)
        if stored.nnz != sp.csr_matrix(positive != 0).nnz:
            raise ValueError('%d positive interactions have no stored rank (list them in the pairs of predict_rank_at)'
                             % (sp.csr_matrix(positive != 0).nnz - stored.nnz))
        return sp.csr_matrix(positive.multiply(ranks))
    if hasattr(predicted_ranks, 'items') and hasattr(predicted_ranks, 'scores'):       # TopK
        items = np.asarray(predicted_ranks.items)
        n_users, n_items = positive.shape
        k = items.shape[1]
        rows = np.repeat(np.arange(n_users), k)
        valid = (items.reshape(-1) >= 0) & (items.reshape(-1) < n_items)
        rank_of = sp.csr_matrix((np.tile(np.arange(1, k + 1), n_users)[valid],
                                 (rows[valid], items.reshape(-1)[valid])), shape=positive.shape)
        inside = positive.multiply(rank_of)                    # rank where the positive is in the top-k
        outside = positive - positive.multiply(rank_of > 0)    # positives not in the top-k
        return sp.csr_matrix(inside + outside * (n_items + 1))
    return sp.csr_matrix(np.asarray(predicted_ranks) * positive.toarray())


def _hits_within_k(predicted_ranks, test_interactions, k):
    """(positives per user, positives ranked <= k per user): the two counts precision and recall are made of."""
    positives = sp.csr_matrix(sp.csr_matrix(test_interactions) > 0)
    ranks = _ranks_of_positives(predicted_ranks, positives)
    n_positive = np.asarray(positives.getnnz(axis=1)).reshape(-1)
    inside = sp.csr_matrix((ranks.data <= k, ranks.indices, ranks.indptr), shape=ranks.shape)
    n_hit = np.asarray(inside.sum(axis=1)).reshape(-1)
    return n_positive, n_hit


def precision_at_k(predicted_ranks, test_interactions, k=10, preserve_rows=False):
    """Share of the k recommended items that are positives (eval.py:7-30).  preserve_rows keeps users without test
    interactions (value 0)."""
    n_positive, n_hit = _hits_within_k(predicted_ranks, test_interactions, k)
    precision = n_hit.astype(float) / k
    return precision if preserve_rows else precision[n_positive > 0]


def recall_at_k(predicted_ranks, test_interactions, k=10, preserve_rows=False):
    """Share of a user's positives found in the first k ranks (eval.py:33-58; users without positives: 0/0 = nan when
    preserve_rows, dropped otherwise)."""
    n_positive, n_hit = _hits_within_k(predicted_ranks, test_interactions, k)
    if not preserve_rows:
        keep = n_positive > 0
        n_positive, n_hit = n_positive[keep], n_hit[keep]
    with np.errstate(divide='ignore', invalid='ignore'):
        return n_hit.astype(float) / n_positive.astype(float)


def _setup_ndcg(predicted_ranks, test_interactions, k=10):
    """The pieces ndcg is computed from (eval.py:61-72): relevance = the positive interaction values, ror = the
    predicted rank of each of them, k_mask = rank <= k, ror_at_k = rank inside k else 1.  All aligned entry by entry."""
    interactions = sp.csr_matrix(test_interactions)
    positives = sp.csr_matrix(interactions > 0)
    ror = _ranks_of_positives(predicted_ranks, positives).astype(np.float64)
    relevance = sp.csr_matrix(interactions.multiply(positives)).astype(np.float64)
    for m in (ror, relevance):
        m.sort_indices()
    k_mask = ror.data < k + 1
    ror_at_k = np.where(k_mask, ror.data, 1.0)
    return relevance, k_mask, ror, ror_at_k


def _idcg(hits, k=10):
    """Ideal DCG of one user's relevance row (eval.py:75-78): the k largest gains at ranks 1..k."""
    best = np.sort(np.asarray(hits))[::-1][:k]
    return float(np.sum((np.exp2(best) - 1.0) / np.log2(np.arange(2, best.shape[0] + 2))))


def _dcg(relevance, k_mask, ror_at_k, ror):
    """DCG per user (eval.py:81-87): sum over the positives ranked inside k of (2^relevance - 1) / log2(rank + 1);
    returned as the reference does, a 1 x n_users matrix."""
    gain = (np.exp2(np.where(k_mask, relevance.data, 0.0)) - 1.0) / np.log2(ror_at_k + 1.0)
    per_entry = sp.csr_matrix((gain, ror.indices, ror.indptr), shape=ror.shape)
    return per_entry.sum(axis=1).flatten()


def ndcg_at_k(predicted_ranks, test_interactions, k=10, preserve_rows=False):
    """Normalised discounted cumulative gain at k (eval.py:89-117)."""
    relevance, k_mask, ror, ror_at_k = _setup_ndcg(predicted_ranks, test_interactions, k)
    dcg = np.asarray(_dcg(relevance, k_mask, ror_at_k, ror)).reshape(-1)
    ideal = np.array([_idcg(row) for row in relevance.toarray()])
    with np.errstate(divide='ignore', invalid='ignore'):
        ndcg = dcg / ideal
    if preserve_rows:
        return ndcg
    return ndcg[np.asarray(relevance.getnnz(axis=1)).reshape(-1) > 0]


def f1_score_at_k(predicted_ranks, test_interactions, k=10, preserve_rows=False):
    """Harmonic mean of the mean precision and the mean recall at k (eval.py:120-148)."""
    mean_p = np.mean(precision_at_k(predicted_ranks, test_interactions, k=k, preserve_rows=preserve_rows))
    mean_r = np.mean(recall_at_k(predicted_ranks, test_interactions, k=k, preserve_rows=preserve_rows))
    return 2.0 * mean_p * mean_r / (mean_p + mean_r)


def _mean_metrics(predicted_ranks, interactions, recall_k, precision_k, ndcg_k):
    return (np.mean(recall_at_k(predicted_ranks, interactions, k=recall_k)),
            np.mean(precision_at_k(predicted_ranks, interactions, k=precision_k)),
            np.mean(ndcg_at_k(predicted_ranks, interactions, k=ndcg_k)))


def fit_and_eval(model, user_features, item_features, train_interactions, test_interactions, fit_kwargs, recall_k=30,
                 precision_k=5, ndcg_k=30):
    """Fit, rank, and report (recall, precision, ndcg) out of sample followed by the same three in sample
    (eval.py:151-166)."""
    model.fit(user_features=user_features, item_features=item_features, interactions=train_interactions, **fit_kwargs)
    predicted_ranks = model.predict_rank(user_features=user_features, item_features=item_features)
    return (_mean_metrics(predicted_ranks, test_interactions, recall_k, precision_k, ndcg_k)
            + _mean_metrics(predicted_ranks, train_interactions, recall_k, precision_k, ndcg_k))


def eval_random_ranks_on_dataset(interactions, recall_k=30, precision_k=5, ndcg_k=30):
    """The metrics of uniformly random rankings, a floor to compare a model with (eval.py:181-192)."""
    n_users, n_items = interactions.shape
    random_ranks = np.stack([np.random.permutation(n_items) + 1 for _ in range(n_users)])
    return _mean_metrics(random_ranks, interactions, recall_k, precision_k, ndcg_k)
