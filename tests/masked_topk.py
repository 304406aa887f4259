"""Oracle of the top-k with exclusion: the k best NON-excluded items per row in reference rank order (score descending,
lower item id on ties -- tf.nn.top_k), i.e. the top-k of the scores with the excluded pairs at -inf, where excluded items
never appear and missing slots hold the sentinel (id 2**31 - 1, score -inf)."""
import numpy as np
import scipy.sparse as sp

SENTINEL_ID = 2 ** 31 - 1


def excluded_mask(exclude, shape):
    """Dense bool [n_users, n_items]: exclude[u, i] != 0 after duplicates are summed (explicit zeros exclude nothing)."""
    m = sp.csr_matrix(exclude, copy=True)
    m.sum_duplicates()
    dense = np.asarray(m.toarray() != 0)
    assert dense.shape[0] == shape[0] and dense.shape[1] >= shape[1]
    return dense[:, :shape[1]]


def masked_top_k(scores, exclude, k):
    """(items int32 [n_users, k], scores float32 [n_users, k])."""
    p = np.asarray(scores, dtype=np.float32)
    mask = excluded_mask(exclude, p.shape)
    items = np.full((p.shape[0], k), SENTINEL_ID, dtype=np.int32)
    vals = np.full((p.shape[0], k), -np.inf, dtype=np.float32)
    for r in range(p.shape[0]):
        eligible = np.nonzero(~mask[r])[0]
        order = eligible[np.lexsort((eligible, -p[r, eligible].astype(np.float64)))][:k]
        items[r, :len(order)] = order
        vals[r, :len(order)] = p[r, order]
    return items, vals


def masked_top_k_rows(score_row_fn, exclude_csr, rows, k):
    """The oracle for a sample of rows: score_row_fn(r) -> float32 [n_items] scores of row r."""
    exclude_csr = sp.csr_matrix(exclude_csr)
    items = np.full((len(rows), k), SENTINEL_ID, dtype=np.int32)
    vals = np.full((len(rows), k), -np.inf, dtype=np.float32)
    for j, r in enumerate(rows):
        s = np.asarray(score_row_fn(r), dtype=np.float32)
        row = exclude_csr[r]
        row.sum_duplicates()
        excl = row.indices[row.data != 0]
        eligible = np.setdiff1d(np.arange(s.shape[0]), excl)
        order = eligible[np.lexsort((eligible, -s[eligible].astype(np.float64)))][:k]
        items[j, :len(order)] = order
        vals[j, :len(order)] = s[order]
    return items, vals
