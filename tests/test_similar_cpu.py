"""CPU tests of predict_similar_items_top_k: its oracle (tests/similar_topk.py) against the reference's literal double
sort on a tie-heavy integer fixture, the union of `exclude` and `exclude_self` as masks, and the argument checks, which
run before any device work."""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from tensorrec_b200 import TensorRec
from tensorrec_b200.errors import ModelNotFitException
from tensorrec_b200.tensorrec import _similar_exclusion_mask
from tests import helpers as H
from tests.masked_topk import SENTINEL_ID
from tests.similar_topk import similar_items_top_k


def tie_heavy_items(n_items=40, d=6, seed=3):
    """Integer representations in {-1, 0, 1}: scores repeat everywhere; items 5, 9 and 30 are one vector no other item
    has."""
    rng = np.random.default_rng(seed)
    repr_ = rng.integers(-1, 2, size=(n_items, d)).astype(np.float32)
    if n_items > 30:
        repr_[[5, 9, 30]] = 2.0
    return repr_


def brute_force(scores, excluded, n):
    """Ranks by the reference's double sort (oracle.rank_predictions) with the excluded pairs at -inf, then the
    non-excluded entries of rank <= n, in rank order."""
    s = np.where(excluded, -np.inf, scores).astype(np.float32)
    ranks = oracle.rank_predictions(s)
    items = np.full((s.shape[0], n), SENTINEL_ID, np.int32)
    vals = np.full((s.shape[0], n), -np.inf, np.float32)
    for q in range(s.shape[0]):
        for i in np.nonzero((ranks[q] <= n) & ~excluded[q])[0]:
            items[q, ranks[q, i] - 1] = i
            vals[q, ranks[q, i] - 1] = scores[q, i]
    return items, vals


@pytest.mark.parametrize('prediction', ['dot', 'cosine', 'euclidean'])
@pytest.mark.parametrize('n', [1, 5, 12, 45])
def test_oracle_matches_the_double_sort_on_ties(prediction, n):
    repr_ = tie_heavy_items()
    ids = np.array([0, 5, 9, 30, 17, 17, 39])
    scores = oracle.predict_similar_items(prediction, repr_, ids)
    none = np.zeros(scores.shape, bool)
    items, vals = similar_items_top_k(prediction, repr_, ids, n)
    exp_i, exp_s = brute_force(scores, none, n)
    assert np.array_equal(items, exp_i) and np.array_equal(vals, exp_s)
    # every query's own id excluded, plus a random pattern
    rng = np.random.default_rng(n)
    pattern = rng.random(scores.shape) < 0.3
    items, vals = similar_items_top_k(prediction, repr_, ids, n, exclude=sp.csr_matrix(pattern.astype(np.float32)),
                                      exclude_self=True)
    excluded = pattern.copy()
    excluded[np.arange(len(ids)), ids] = True
    exp_i, exp_s = brute_force(scores, excluded, n)
    assert np.array_equal(items, exp_i) and np.array_equal(vals, exp_s)


def test_oracle_whole_catalogue_and_the_self_match():
    repr_ = tie_heavy_items()
    items, vals = similar_items_top_k('euclidean', repr_, None, 3)
    assert items.shape == (40, 3)
    # distance 0 clamps to -sqrt(1e-16); equal vectors 5, 9, 30 share it and come in id order
    assert items[5].tolist() == [5, 9, 30] and items[30].tolist() == [5, 9, 30]
    assert np.all(vals[5] == np.float32(-np.sqrt(np.float32(1e-16))))
    items, _ = similar_items_top_k('euclidean', repr_, None, 3, exclude_self=True)
    assert items[5].tolist()[:2] == [9, 30] and 5 not in items[5]


def test_exclusion_mask_is_a_union_not_a_sum():
    ids = np.array([2, 0, 2])
    # row 0: -1 on its own id (a sum with the self entry would be 0 and re-admit it), row 1: duplicates 1 - 1 = 0 on
    # item 3 (not excluded) and an explicit zero on item 1, row 2: -2 on item 4
    exclude = sp.coo_matrix((np.array([-1., 1., -1., 0., -2.]), (np.array([0, 1, 1, 1, 2]), np.array([2, 3, 3, 1, 4]))),
                            shape=(3, 5)).tocsr()
    before = exclude.copy()
    union = _similar_exclusion_mask(exclude, True, ids, 3, 5).toarray()
    assert union.tolist() == [[0, 0, 1, 0, 0], [1, 0, 0, 0, 0], [0, 0, 1, 0, 1]]
    assert (exclude != before).nnz == 0                                # the caller's matrix is unchanged
    mask = _similar_exclusion_mask(exclude, False, ids, 3, 5).toarray()
    assert mask.tolist() == [[0, 0, 1, 0, 0], [0, 0, 0, 0, 0], [0, 0, 0, 0, 1]]
    assert _similar_exclusion_mask(None, False, ids, 3, 5) is None
    assert _similar_exclusion_mask(None, True, None, 3, 5).toarray().tolist() == np.eye(3, 5).tolist()
    # the oracle applies the same union
    repr_ = tie_heavy_items(n_items=5, d=3)
    items, _ = similar_items_top_k('dot', repr_, ids, 5, exclude=exclude, exclude_self=True)
    for q in range(3):
        got = items[q][items[q] != SENTINEL_ID]
        assert sorted(got) == np.nonzero(union[q] == 0)[0].tolist()     # exactly the items outside the union


# ---- argument checks, before any device work ---------------------------------------------------------------------
@pytest.fixture(scope='module')
def fitted():
    itf = H.tag_features(9, 20, 4, seed=2)
    model = TensorRec(n_components=4)
    model.set_weights({'linear_weights_user_0': np.zeros((20, 4)), 'linear_weights_item': np.zeros((20, 4)),
                       'feature_biases_user': np.zeros((20, 1)), 'feature_biases_item': np.zeros((20, 1))})
    return model, itf


def test_unfitted_model_raises_model_not_fit():
    with pytest.raises(ModelNotFitException):
        TensorRec(n_components=4).predict_similar_items_top_k(H.tag_features(9, 20, 4, seed=2), 3)


def test_argument_errors_are_value_errors(fitted):
    model, itf = fitted
    with pytest.raises(ValueError, match='lie in'):
        model.predict_similar_items_top_k(itf, 3, item_ids=[0, 9])
    with pytest.raises(ValueError, match='lie in'):
        model.predict_similar_items_top_k(itf, 3, item_ids=[-1])
    with pytest.raises(ValueError, match='1-D'):
        model.predict_similar_items_top_k(itf, 3, item_ids=[[0, 1]])
    with pytest.raises(ValueError, match='1-D'):
        model.predict_similar_items_top_k(itf, 3, item_ids=4)
    with pytest.raises(ValueError, match='integers'):
        model.predict_similar_items_top_k(itf, 3, item_ids=[0.5, 1.0])
    with pytest.raises(ValueError, match='n_similar'):
        model.predict_similar_items_top_k(itf, 0)
    with pytest.raises(ValueError, match='rows'):
        model.predict_similar_items_top_k(itf, 3, item_ids=[1, 2], exclude=sp.csr_matrix((3, 9)))
    with pytest.raises(ValueError, match='rows'):
        model.predict_similar_items_top_k(itf, 3, exclude=sp.csr_matrix((8, 9)))    # None = all 9 items
    with pytest.raises(ValueError, match='columns'):
        model.predict_similar_items_top_k(itf, 3, item_ids=[1, 2], exclude=sp.csr_matrix((2, 10)))
    with pytest.raises(ValueError, match='sparse'):
        model.predict_similar_items_top_k(itf, 3, item_ids=[1, 2], exclude=np.zeros((2, 9)))
    with pytest.raises(ValueError, match='columns but the model'):
        model.predict_similar_items_top_k(H.tag_features(9, 21, 4, seed=2), 3)
