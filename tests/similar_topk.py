"""Oracle of TensorRec.predict_similar_items_top_k: the reference's similar-items scores (oracle.predict_similar_items:
the prediction graph between the query rows and every item, no biases) followed by the masked top-k
(tests/masked_topk.py), where the excluded pairs are the non-zero entries of `exclude` united with every query's own id
when exclude_self."""
import numpy as np
import scipy.sparse as sp

import oracle
from tests.masked_topk import excluded_mask, masked_top_k


def similar_items_top_k(prediction, item_repr, item_ids, n, exclude=None, exclude_self=False):
    """prediction: 'dot' | 'cosine' | 'euclidean'; item_ids None = every item.  -> (items int32, scores float32)."""
    ids = np.arange(np.asarray(item_repr).shape[0]) if item_ids is None else np.asarray(item_ids, dtype=np.int64)
    scores = oracle.predict_similar_items(prediction, item_repr, ids)
    mask = np.zeros(scores.shape, dtype=bool)
    if exclude is not None:
        mask |= excluded_mask(exclude, scores.shape)
    if exclude_self:
        mask[np.arange(len(ids)), ids] = True
    return masked_top_k(scores, sp.csr_matrix(mask.astype(np.float32)), n)
