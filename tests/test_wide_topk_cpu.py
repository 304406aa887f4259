"""CPU checks of the wide filter route (32 < k <= 1024) without a GPU: a numpy model of the ALGORITHM of
score_wide_tc.cu + rescore_wide.cu (lists of capacity C = 2 K_keep, compaction by selection of the k-th best to at most
K_keep entries >= k-th best - 2.25 m, drop_max, give-up, no warm start, exclusion as a mask), the route helper
tensorrec.topk_route and the default row blocks of the wide and dense+rank routes."""
import numpy as np
import pytest

MARGINS, GIVE_UP = 2.25, 8


def keep_for(k):
    """K_keep of the kernel: k + max(k / 2, 32) rounded up to 32 (score_wide_tc.cu: wide_keep)."""
    return -(-(k + max(k // 2, 32)) // 32) * 32


def run_row(exact, approx, order, slack_of, m, k, excluded=(), chunk=32, block=128):
    """One user row of the wide form.  exact / approx: per-item scores (approx within m of exact), processed in `order`;
    slack_of(block) >= 0 widens the admission test (the block-bias bound); excluded items are never admitted.
    Returns (reported ids, certified, statistics)."""
    keep = keep_for(k)
    cap = 2 * keep
    excluded = set(int(i) for i in excluded)
    theta, tau, drop_max, n_ovf = -np.inf, -np.inf, -np.inf, 0
    lst = []                                           # [(approx score, item id)], unsorted
    stats = {'compactions': 0, 'overflows': 0, 'max_len': 0}

    def compact():
        nonlocal lst, theta, tau, drop_max, n_ovf
        stats['compactions'] += 1
        if len(lst) < k:
            return
        scores = np.array([s for s, _ in lst])
        kth = np.sort(scores)[::-1][k - 1]                 # the radix select: the k-th best value
        floor = kth - MARGINS * m
        kept = [e for e in lst if e[0] >= floor]
        if len(kept) > keep:                               # overflow: keep only what beats the (keep + 1)-th best
            cut = np.sort(np.array([s for s, _ in kept]))[::-1][keep]
            kept = [e for e in kept if e[0] > cut]
            drop_max = max(drop_max, cut)
            n_ovf += 1
            stats['overflows'] += 1
        assert len(kept) <= keep
        lst = kept
        theta = max(theta, floor)
        tau = theta
        if n_ovf >= GIVE_UP:
            tau, drop_max = np.inf, np.inf

    for p0 in range(0, len(order), chunk):
        ids = [int(i) for i in order[p0:p0 + chunk]]
        slack = slack_of(p0 // block)
        passing = [i for i in ids if i not in excluded and approx[i] + slack > tau]
        if len(lst) + len(passing) > cap:
            compact()
        if n_ovf < GIVE_UP:
            lst.extend((approx[i], i) for i in passing)
        assert len(lst) <= cap
        stats['max_len'] = max(stats['max_len'], len(lst))
    compact()                                          # the kernel's final compaction
    row_theta = max(theta, drop_max)
    # select_wide_kernel: exact scores, (score desc, id asc), certificate
    surv = sorted(((exact[i], i) for _, i in lst), key=lambda e: (-e[0], e[1]))
    top = surv[:k]
    certified = (row_theta == -np.inf) or (len(surv) >= k and row_theta + m < top[k - 1][0])
    return [i for _, i in top], certified, stats


def exact_topk(exact, k, excluded=()):
    eligible = np.setdiff1d(np.arange(len(exact)), np.asarray(list(excluded), dtype=np.int64))
    order = eligible[np.lexsort((eligible, -np.asarray(exact, dtype=np.float64)[eligible]))]
    return list(order[:k])


def fixture(rng, kind, n):
    if kind == 0:                                       # continuous scores
        return rng.standard_normal(n), 1e-3
    if kind == 1:                                       # massive ties
        return rng.integers(-2, 3, n).astype(np.float64), 0.0
    if kind == 2:                                       # a plateau across the k-th place
        return np.concatenate([rng.standard_normal(n - 400) - 5.0, np.full(400, 1.0)]), 1e-3
    return 1.0 + 1e-4 * rng.standard_normal(n), 1e-3   # near-ties inside the error bound


@pytest.mark.parametrize('seed', range(24))
def test_certified_rows_equal_the_exact_topk(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1500, 6000))
    k = int(rng.choice([33, 64, 100, 257, 1024]))
    kind = seed % 4
    exact, m = fixture(rng, kind, n)
    approx = exact + (np.where(rng.random(n) < 0.5, m, -m) if kind == 3 else rng.uniform(-m, m, n) if m else 0.0)
    excluded = rng.choice(n, int(rng.integers(0, n // 2)), replace=False) if seed % 3 else ()
    slack = rng.uniform(0.0, 0.01, n // 128 + 1)
    top, certified, stats = run_row(exact, approx, rng.permutation(n), lambda b: slack[b], m, k, excluded)
    assert stats['max_len'] <= 2 * keep_for(k)
    if certified:
        expected = exact_topk(exact, k, excluded)
        assert top == expected
        if len(expected) < k:                           # fewer eligible items than k: certified with sentinel slots
            assert len(top) < k


@pytest.mark.parametrize('seed', range(6))
def test_plateaus_and_ties_are_flagged_never_wrong(seed):
    rng = np.random.default_rng(100 + seed)
    n, k, m = 3000, 100, 1e-3
    exact = np.concatenate([rng.standard_normal(n - 600) - 10.0, np.full(600, 1.0)])    # 600 ties for 100 places
    approx = exact + rng.uniform(-m, m, n)
    top, certified, stats = run_row(exact, approx, rng.permutation(n), lambda b: 0.0, m, k)
    assert stats['overflows'] > 0                      # more than K_keep within the bound: entries were dropped
    assert not certified


def test_give_up_stops_admissions():
    """All-equal scores: every chunk passes, compactions overflow until the row gives up and stops admitting."""
    n, k = 20000, 40
    exact = np.zeros(n)
    top, certified, stats = run_row(exact, exact, np.arange(n), lambda b: 0.0, 1e-3, k)
    assert stats['overflows'] == GIVE_UP and not certified
    assert stats['compactions'] < n // (2 * keep_for(k) - keep_for(k))   # the sweep did not keep compacting


def test_clear_cut_rows_are_certified_from_a_cold_start():
    """No warm start: theta starts at -inf and the first compaction sets it; clear rows still certify."""
    rng = np.random.default_rng(7)
    n, k, m = 20000, 100, 1e-5
    exact = rng.standard_normal(n)
    approx = exact + rng.uniform(-m, m, n)
    accepted = 0
    for _ in range(6):
        top, certified, stats = run_row(exact, approx, rng.permutation(n), lambda b: 0.0, m, k)
        accepted += int(certified)
        assert not certified or top == exact_topk(exact, k)
        assert stats['compactions'] < n // 64
    assert accepted == 6


def test_list_capacity_and_keep():
    for k in (33, 64, 100, 500, 1000, 1024):
        keep = keep_for(k)
        assert keep % 32 == 0 and keep >= k + 32 and 2 * keep - keep >= 32    # a chunk always fits after compaction
    assert 2 * keep_for(1024) * 5 <= 16384            # k = 1024 still runs with several item splits


# ---- the route helper ---------------------------------------------------------------------------------------------
@pytest.fixture
def TR():
    from tensorrec_b200 import tensorrec
    return tensorrec


def route(TR, k, n_items=10 ** 6, model_ok=True, single_taste=True, sharded=False):
    return TR.topk_route(k, n_items, model_ok, single_taste, 12, 32, sharded=sharded)


def test_route_boundaries(TR, monkeypatch):
    monkeypatch.setattr(TR, 'WIDE_MIN_ITEMS', 5000)
    assert route(TR, 12) == 'filter' and route(TR, 13) == 'exact3' and route(TR, 32) == 'exact3'
    assert route(TR, 33) == 'wide' and route(TR, 1024) == 'wide' and route(TR, 1025) == 'dense+rank'
    assert route(TR, 100, n_items=4999) == 'dense+rank' and route(TR, 100, n_items=5000) == 'wide'
    assert route(TR, 10, n_items=0) == 'dense+rank'


def test_route_by_model_kind(TR, monkeypatch):
    monkeypatch.setattr(TR, 'WIDE_MIN_ITEMS', 5000)
    # tastes > 1: the fused k <= 32 routes merge per-taste lists; k > 32 has no de-duplicating merge
    assert route(TR, 10, single_taste=False) == 'filter' and route(TR, 100, single_taste=False) == 'dense+rank'
    # attention, custom graphs, d > 128, Euclidean user x item (model_ok False): always dense+rank
    for k in (10, 100, 2000):
        assert route(TR, k, model_ok=False) == 'dense+rank'
    monkeypatch.setattr(TR, 'TOPK_PATH', 'exact')     # "no filter": k > 32 goes to dense+rank
    assert route(TR, 10) == 'exact3' and route(TR, 100) == 'dense+rank'


def test_sharded_route_does_not_depend_on_the_shard_size(TR, monkeypatch):
    monkeypatch.setattr(TR, 'WIDE_MIN_ITEMS', 5000)
    routes = {route(TR, 100, n_items=n, sharded=True) for n in (0, 1, 4999, 5000, 10 ** 6)}
    assert routes == {'wide'}
    assert {route(TR, 2000, n_items=n, sharded=True) for n in (0, 10 ** 6)} == {'dense+rank'}


def test_wide_min_items_keeps_small_catalogues_on_dense_rank(TR):
    assert TR.WIDE_MIN_ITEMS > 911 and TR.WIDE_MAX_K == 1024


def test_route_of_model_kinds_through_the_model(TR):
    """_tensor_path_ok decides model_ok for user x item top-k: dot and cosine only, one taste or several, no attention."""
    import tensorrec_b200 as T
    P = T.prediction_graphs
    assert T.TensorRec(n_components=64)._tensor_path_ok(allow_tastes=True)
    assert T.TensorRec(n_components=64, prediction_graph=P.CosineSimilarityPredictionGraph())._tensor_path_ok(True)
    assert not T.TensorRec(n_components=64, prediction_graph=P.EuclideanSimilarityPredictionGraph())._tensor_path_ok(True)
    assert not T.TensorRec(n_components=200)._tensor_path_ok(allow_tastes=True)
    assert not T.TensorRec(n_components=64, n_tastes=2, attention_graph=T.representation_graphs.LinearRepresentationGraph()
                           )._tensor_path_ok(allow_tastes=True)


# ---- block sizing ---------------------------------------------------------------------------------------------------
def test_dense_route_blocks_bound_the_memory(TR, monkeypatch):
    from tensorrec_b200 import kernels
    model = TR.TensorRec(n_components=64)
    n_items = 1000000
    rows = model._topk_block_rows('dense+rank', 100000, n_items, 100)
    assert rows * n_items * kernels.DENSE_RANK_BYTES_PER_PAIR <= model.PREDICT_BLOCK_BYTES
    assert (rows + 1) * n_items * kernels.DENSE_RANK_BYTES_PER_PAIR > model.PREDICT_BLOCK_BYTES
    assert model._topk_block_rows('dense+rank', 10, 10 ** 12, 100) == 1     # at least one row
    monkeypatch.setattr(TR.TensorRec, 'PREDICT_BLOCK_BYTES', 35 * 1000 * 40)
    assert model._topk_block_rows('dense+rank', 500, 1000, 100) == 40
    assert model._topk_block_rows('filter', 500, 1000, 10) == 500           # the k <= 32 routes: one block


# ---- sharded calls: every rank cuts the users into the same blocks --------------------------------------------------
def _block_worker(rank, world, port, n_items, out_dir):
    import os
    import sys
    import torch.distributed as dist
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import tensorrec_b200 as T
    from tensorrec_b200.distributed import shard_bounds
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        lo, hi = shard_bounds(n_items, world, rank)
        model = T.TensorRec(n_components=64)
        local = model._topk_block_rows('dense+rank', 10 ** 6, hi - lo, 100)
        shared = model._topk_block_rows('dense+rank', 10 ** 6, hi - lo, 100, dist.group.WORLD, 'cpu')
        mine = [(u0, min(10 ** 6, u0 + shared)) for u0 in range(0, 10 ** 6, shared)]
        every = [None] * world
        dist.all_gather_object(every, (local, mine))
        with open(os.path.join(out_dir, 'rank_%d' % rank), 'w') as f:
            f.write(repr([(loc, len(part), part == every[0][1]) for loc, part in every]))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('world, n_items', [(2, 20001), (4, 20005), (4, 3)])
def test_sharded_dense_blocks_are_the_same_on_every_rank(tmp_path, world, n_items):
    """Shards of n and n + 1 items (and an empty shard: 3 items over 4 ranks) choose different block sizes on their
    own; the shared choice gives every rank the same partition of the users."""
    import os
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    mp.spawn(_block_worker, args=(world, port, n_items, str(tmp_path)), nprocs=world, join=True)
    views = [eval(open(os.path.join(str(tmp_path), 'rank_%d' % r)).read()) for r in range(world)]
    assert all(v == views[0] for v in views)
    local_sizes = [loc for loc, _, _ in views[0]]
    assert len(set(local_sizes)) > 1                   # the ranks would disagree on their own
    assert all(same for _, _, same in views[0])          # ... and agree on the shared partition
