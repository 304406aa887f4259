"""CPU tests of the top-k with exclusion (predict_top_k(..., exclude=...)): the masked oracle on hand-computed answers,
a model of the filter kernel's algorithm with masked columns (warm start included), the host preparation of the
exclusion lists, and the argument checks, which run before any device work."""
import numpy as np
import pytest
import scipy.sparse as sp

from tensorrec_b200 import TensorRec, kernels
from tests import helpers as H
from tests.masked_topk import SENTINEL_ID, masked_top_k

NEG = -np.inf
RANK_FIXTURE = np.array([[1, 2, 3, 4], [4, 3, 2, 1], [3, 4, 1, 2]], dtype=np.float32)   # the reference's rank fixture


# ---- the masked oracle --------------------------------------------------------------------------------------------
def test_masked_oracle_hand_computed():
    # row 0 excludes its best item (3), row 1 excludes everything, row 2 excludes 1 and 3 (2 eligible < k = 3)
    exclude = sp.csr_matrix((np.ones(7), ([0, 1, 1, 1, 1, 2, 2], [3, 0, 1, 2, 3, 1, 3])), shape=(3, 4))
    items, scores = masked_top_k(RANK_FIXTURE, exclude, 3)
    assert items.tolist() == [[2, 1, 0], [SENTINEL_ID] * 3, [0, 2, SENTINEL_ID]]
    assert scores.tolist() == [[3, 2, 1], [NEG] * 3, [3, 1, NEG]]


def test_masked_oracle_ties_go_to_the_lower_id():
    scores = np.array([[5, 7, 7, 7, 5]], dtype=np.float32)
    exclude = sp.csr_matrix((np.ones(1), ([0], [2])), shape=(1, 5))
    items, vals = masked_top_k(scores, exclude, 4)
    assert items.tolist() == [[1, 3, 0, 4]] and vals.tolist() == [[7, 7, 5, 5]]


def test_masked_oracle_duplicates_unsorted_and_explicit_zeros():
    # COO, unsorted, with duplicates: (0, 3) twice (1 + 1 -> excluded), (0, 1) = 1 - 1 = 0 (sums to zero: not excluded),
    # (1, 0) an explicit zero (not excluded), (2, 2) negative (excluded: "disliked" counts as seen)
    exclude = sp.coo_matrix((np.array([1., 1., 1., -1., 0., -2.]),
                             (np.array([0, 0, 0, 0, 1, 2]), np.array([3, 3, 1, 1, 0, 2]))), shape=(3, 4))
    items, _ = masked_top_k(RANK_FIXTURE, exclude, 2)
    assert items.tolist() == [[2, 1], [0, 1], [1, 0]]


# ---- the filter kernel's algorithm with masked columns -------------------------------------------------------------
BUF, KEEP, MARGINS = 32, 16, 2.25


def run_masked_row(exact, approx, masked, order, m, k, block=128, step=16, warm_start=True):
    """One row of score_filter_kernel<..., kExclude> + rescore_topk_kernel: masked columns carry -inf (never admitted,
    neutral in the warm start's group maxima); the warm start takes the k-th largest of the 8-column group maxima of the
    first tile.  Returns (reported top-k ids, certified) with the kernel's certificate rule."""
    n = len(exact)
    a = np.where(masked, -np.inf, approx)
    theta, drop_max = -np.inf, -np.inf
    if warm_start:
        first = a[order[:block]]
        g = sorted((first[i:i + 8].max() for i in range(0, len(first), 8)), reverse=True)
        if len(g) >= k and np.isfinite(g[k - 1]):        # (k-th group maximum -inf: start from -inf as before)
            theta = g[k - 1] - MARGINS * m
    tau = theta
    buf = []

    def compact():
        nonlocal buf, theta, tau, drop_max
        buf.sort(key=lambda e: (-e[0], e[1]))
        if len(buf) >= k:
            floor = buf[k - 1][0] - MARGINS * m
            kept = [e for e in buf if e[0] >= floor]
            if len(kept) > KEEP:
                drop_max = max(drop_max, kept[KEEP][0])
                kept = kept[:KEEP]
            buf, theta, tau = kept, floor, floor

    for p0 in range(0, n, step):
        passing = [p for p in range(p0, min(p0 + step, n)) if a[order[p]] > tau]
        if len(buf) + len(passing) > BUF:
            compact()
        buf.extend((a[order[p]], int(order[p])) for p in passing)
    compact()
    row_theta = max(theta, drop_max)
    surv = sorted(((exact[i], i) for _, i in buf), key=lambda e: (-e[0], e[1]))
    top = surv[:k]
    certified = row_theta == -np.inf or (len(surv) >= k and row_theta + m < top[k - 1][0])
    return [i for _, i in top], certified


def masked_exact(exact, masked, k):
    ids = np.nonzero(~masked)[0]
    return [int(i) for i in ids[np.lexsort((ids, -exact[ids]))][:k]]


@pytest.mark.parametrize('seed', range(40))
def test_certified_masked_rows_equal_the_masked_exact_topk(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(40, 900))
    k = int(rng.integers(1, 13))
    kind = seed % 4
    exact = [rng.standard_normal(n), rng.integers(-2, 3, n).astype(np.float64),
             np.concatenate([rng.standard_normal(n - 30) - 5.0, np.full(30, 1.0)]),
             1.0 + 1e-4 * rng.standard_normal(n)][kind]
    m = 1e-3 if kind != 1 else 0.0
    approx = exact + (np.where(rng.random(n) < 0.5, m, -m) if kind == 3 else rng.uniform(-m, m, n) if m else 0.0)
    pattern = (seed // 4) % 5
    if pattern == 0:                                        # the row's own unmasked top-k: theta has to go deeper
        masked = np.zeros(n, bool)
        masked[masked_exact(exact, masked, k)] = True
    elif pattern == 1:                                      # heavy: more than half of the catalogue
        masked = rng.random(n) < 0.7
    elif pattern == 2:                                      # fewer than k eligible items
        masked = np.ones(n, bool)
        masked[rng.choice(n, int(rng.integers(0, k)), replace=False)] = False
    elif pattern == 3:                                      # everything
        masked = np.ones(n, bool)
    else:                                                   # the best items of the first tile (the warm start's)
        order0 = rng.permutation(n)
        masked = np.zeros(n, bool)
        first = order0[:128]
        masked[first[np.argsort(-approx[first])[:2 * k]]] = True
    order = rng.permutation(n) if pattern != 4 else order0
    expect = masked_exact(exact, masked, k)
    for warm in (True, False):
        top, certified = run_masked_row(exact, approx, masked, order, m, k, warm_start=warm)
        if certified:
            assert top == expect
        assert not (set(top) & set(np.nonzero(masked)[0].tolist()))      # excluded items never reported
    if pattern in (2, 3):                                   # too few eligible items: certified, with sentinel slots
        top, certified = run_masked_row(exact, approx, masked, order, m, k)
        assert len(expect) < k and certified and top == expect


def test_clear_cut_masked_rows_are_certified():
    rng = np.random.default_rng(7)
    n, k, m = 3000, 10, 1e-4
    exact = rng.standard_normal(n)
    approx = exact + rng.uniform(-m, m, n)
    masked = np.zeros(n, bool)
    masked[masked_exact(exact, masked, k)] = True            # the unmasked top-k is excluded
    masked |= rng.random(n) < 0.3
    accepted = 0
    for _ in range(10):
        top, certified = run_masked_row(exact, approx, masked, rng.permutation(n), m, k)
        accepted += int(certified)
        assert not certified or top == masked_exact(exact, masked, k)
    assert accepted >= 9


# ---- host preparation --------------------------------------------------------------------------------------------
def test_host_lists_sum_duplicates_drop_zeros_and_sort():
    exclude = sp.coo_matrix((np.array([1., 1., 2., -1., 0., 3., 1.]),
                             (np.array([0, 0, 0, 0, 1, 2, 2]), np.array([5, 5, 1, 1, 0, 4, 2]))), shape=(3, 6))
    indptr, ids = kernels.exclusion_host_csr(exclude, 0, 6)
    assert indptr.dtype == np.int32 and ids.dtype == np.int32
    assert indptr.tolist() == [0, 2, 2, 4] and ids.tolist() == [1, 5, 2, 4]   # (0,1) = 2 - 1 = 1 stays excluded


def test_host_lists_slice_shards_and_user_blocks():
    rng = np.random.default_rng(3)
    exclude = sp.random(50, 300, density=0.1, format='csr', random_state=rng)
    exclude.data[::7] = 0.0                                  # explicit zeros
    dense = exclude.toarray() != 0
    full = sp.csr_matrix(exclude)
    for (lo, hi) in ((0, 300), (0, 120), (120, 250), (250, 300)):
        for (u0, u1) in ((0, 50), (0, 17), (17, 34), (34, 50)):
            indptr, ids = kernels.exclusion_host_csr(exclude, lo, hi - lo, u0, u1)
            assert len(indptr) == u1 - u0 + 1
            for r in range(u1 - u0):
                row = ids[indptr[r]:indptr[r + 1]]
                assert np.all(np.diff(row) > 0)
                assert row.tolist() == (np.nonzero(dense[u0 + r, lo:hi])[0]).tolist()
    assert (full != exclude).nnz == 0                        # the caller's matrix is unchanged


# ---- argument checks, before any device work ---------------------------------------------------------------------
@pytest.fixture(scope='module')
def fitted():
    uf, itf = H.tag_features(6, 20, 4, seed=1), H.tag_features(9, 20, 4, seed=2)
    model = TensorRec(n_components=4)
    model.set_weights({'linear_weights_user_0': np.zeros((20, 4)), 'linear_weights_item': np.zeros((20, 4)),
                       'feature_biases_user': np.zeros((20, 1)), 'feature_biases_item': np.zeros((20, 1))})
    return model, uf, itf


def test_exclude_shape_errors_are_value_errors(fitted):
    model, uf, itf = fitted
    with pytest.raises(ValueError, match='rows'):
        model.predict_top_k(uf, itf, 3, exclude=sp.csr_matrix((5, 9)))
    with pytest.raises(ValueError, match='columns'):
        model.predict_top_k(uf, itf, 3, exclude=sp.csr_matrix((6, 10)))
    with pytest.raises(ValueError, match='columns'):
        model.predict_rank(uf, itf, k=3, exclude=sp.csr_matrix((6, 8)))
    with pytest.raises(ValueError, match='columns'):                 # a shard needs >= item_id_offset + n_items
        model.predict_top_k(uf, itf, 3, item_id_offset=5, exclude=sp.csr_matrix((6, 13)))
    with pytest.raises(ValueError, match='sparse'):
        model.predict_top_k(uf, itf, 3, exclude=np.zeros((6, 9)))


def test_exclude_with_full_ranks_is_a_value_error(fitted):
    model, uf, itf = fitted
    with pytest.raises(ValueError, match='k'):
        model.predict_rank(uf, itf, exclude=sp.csr_matrix((6, 9)))
