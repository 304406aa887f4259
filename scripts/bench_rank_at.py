"""Full ranks of listed (user, item) pairs with predict_rank_at, on one GPU.

    python scripts/bench_rank_at.py --out DIR [--parts flagship,dense,crossover --cases a,b,c,euclidean,attention
                                               --reps R --oracle-rows R]

Inputs are bench.py's flagship problem (1M users x 1M items x d128, biased dot), bench_euclidean.py's biased Euclidean
model and bench_tastes.py's biased three-taste attention model.  Every timing is one warm-up pass, then R timed passes
(median and range); a pass is one predict_rank_at call ended by a device synchronisation.
  flagship   'exact3_count' on the cases
               a  leave-one-out, friendly: one pair per user drawn from the user's own top 100 (most chunks skipped);
               b  leave-one-out, hostile: one uniformly random item per user (few chunks skipped);
               c  heavy tail: Pareto-distributed pairs per user (alpha 1.2, mean about 10, capped at 1000: many passes);
               euclidean, attention: case a for the other two models;
             with the peak device memory of a pass.  Every case is checked on 32 whole 128-user blocks against
             trk_rank_full of those blocks' dense tensor-core scores (must be equal), and cases a / b of the dot model on
             --oracle-rows users against float64 ranks from the CPU oracle's fp32 representations (rank differences
             there are near-ties: the pair's score and the ones that moved differ by about 1e-7 relative).
  dense      'dense+rank' on case a's pairs of the first 4096 users, extrapolated to 1M users.
  crossover  65536 users, d128, 10 random pairs per user, items in {1K, 2K, 4K, 16K, 64K}, both routes forced.
Results, with the card's name and power limit, go to DIR/bench_rank_at.json."""
import argparse
import json
import os
import sys

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts import bench_euclidean as BE  # noqa: E402
from scripts import bench_tastes as BT  # noqa: E402
from scripts.bench_euclidean import problem, timed  # noqa: E402
from scripts.bench_similar import card  # noqa: E402

BLOCK = 128
CHECK_BLOCKS = 32


def model_of(kind, d, wu, wi, bu, bi):
    if kind == 'attention':
        return BT.model_of(True, d, wu, wi, bu, bi)
    return BE.model_of(kind, d, wu, wi, bu, bi)


def with_floor(T, floor, fn):
    old = T.tensorrec.RANK_AT_MIN_ITEMS
    T.tensorrec.RANK_AT_MIN_ITEMS = floor
    try:
        return fn()
    finally:
        T.tensorrec.RANK_AT_MIN_ITEMS = old


def friendly_pairs(model, uf, itf, seed):
    """One pair per user from the user's own top 100."""
    top = model.predict_top_k(uf, itf, 100, to_host=False).items.cpu().numpy()
    n = uf.shape[0]
    pick = top[np.arange(n), np.random.default_rng(seed).integers(0, 100, n)]
    return sp.csr_matrix((np.ones(n, np.float32), pick, np.arange(n + 1)), shape=(n, itf.shape[0]))


def random_pairs(n_users, n_items, per_row, seed):
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(n_users), per_row)
    m = sp.csr_matrix((np.ones(rows.size, np.float32), (rows, rng.integers(0, n_items, rows.size))),
                      shape=(n_users, n_items))
    m.sum_duplicates()
    return m


def pareto_counts(n_users, seed, alpha=1.2, mean=10.0, cap=1000):
    x_m = mean * (alpha - 1) / alpha
    return np.minimum(cap, np.ceil(x_m * (1 + np.random.default_rng(seed).pareto(alpha, n_users)))).astype(np.int64)


def block_check(model, uf, itf, pairs, ranks):
    """Ranks of the first CHECK_BLOCKS whole user blocks against trk_rank_full of their dense tensor-core scores."""
    import torch
    from tensorrec_b200 import kernels
    from tensorrec_b200.input_utils import SparseInput
    device = torch.device('cuda')
    n = CHECK_BLOCKS * BLOCK
    item_in = SparseInput(sp.csr_matrix(itf))
    score = model._score_plan(item_in, device)
    diff = checked = 0
    step = 8 * BLOCK
    for u0 in range(0, n, step):
        full = kernels.rank_full(score(SparseInput(sp.csr_matrix(uf[u0:u0 + step]))))
        sub = ranks[u0:u0 + step].tocoo()
        want = full[torch.from_numpy(sub.row).long().cuda(), torch.from_numpy(sub.col).long().cuda()].cpu().numpy()
        diff += int(np.sum(want != sub.data))
        checked += int(sub.nnz)
        del full
    return {'users': n, 'pairs': checked, 'pairs_differing': diff}


def oracle_check(uf, itf, wu, wi, bu, bi, ranks, n_rows):
    """float64 ranks of the pairs of n_rows users from the oracle's fp32 representations (dot model)."""
    from oracle import reference_ops as R
    item = R.sparse_dense_matmul_fast(itf, wi).astype(np.float64)
    ib = np.asarray(itf @ bi, dtype=np.float64)
    rows = np.sort(np.random.default_rng(13).choice(uf.shape[0], n_rows, replace=False))
    diff, gaps, n = 0, [], 0
    for r in rows:
        user = R.sparse_dense_matmul_fast(uf[r], wu).astype(np.float64)
        s = item @ user[0] + float(np.asarray(uf[r] @ bu).reshape(-1)[0]) + ib
        got = ranks[r].tocoo()
        for c, rank in zip(got.col, got.data):
            want = 1 + int(np.sum(s > s[c])) + int(np.sum(s[:c] == s[c]))
            n += 1
            if want != rank:
                diff += 1
                gaps.append(abs(int(want) - int(rank)))
    return {'rows': int(n_rows), 'pairs': n, 'pairs_differing': diff, 'max_rank_gap': max(gaps) if gaps else 0}


def run_flagship(args, T, out):
    import torch
    n, d = args.flagship_size, 128
    uf, itf, wu, wi, bu, bi = out['_problem'] = problem(n, n, d)
    res = {'workload': '%d users x %d items x d%d, biased' % (n, n, d)}
    for case in args.cases.split(','):
        kind = case if case in ('euclidean', 'attention') else 'dot'
        model = model_of(kind, d, wu, wi, bu, bi)
        if case in ('a', 'euclidean', 'attention'):
            pairs = friendly_pairs(model, uf, itf, seed=1)
        elif case == 'b':
            pairs = random_pairs(n, n, 1, seed=2)
        else:
            pairs = random_pairs(n, n, pareto_counts(n, seed=3), seed=4)
        box = {}

        def run():
            box['ranks'] = model.predict_rank_at(uf, itf, pairs)
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        r = timed(run, args.reps)
        r['peak_device_bytes'] = int(torch.cuda.max_memory_allocated())
        r.update(model.last_rank_info)
        r['pairs'] = int(box['ranks'].nnz)
        r['median_rank'] = float(np.median(box['ranks'].data))
        r['block_check'] = block_check(model, uf, itf, pairs, box['ranks'])
        if kind == 'dot' and case in ('a', 'b') and args.oracle_rows:
            r['oracle_check'] = oracle_check(uf, itf, wu, wi, bu, bi, box['ranks'], args.oracle_rows)
        res[case] = r
        print('flagship', case, json.dumps(r), file=sys.stderr, flush=True)
        if case == 'a':
            out['_pairs_a'] = pairs
        del model, box
        torch.cuda.empty_cache()
        out['flagship'] = res
        yield


def run_dense(args, T, out):
    n, d, rows = args.flagship_size, 128, 4096
    uf, itf, wu, wi, bu, bi = out['_problem'] if '_problem' in out else problem(n, n, d)
    model = model_of('dot', d, wu, wi, bu, bi)
    pairs = out.pop('_pairs_a', None)
    pairs = friendly_pairs(model, uf, itf, seed=1) if pairs is None else pairs
    sub_u, sub_p = uf[:rows], pairs[:rows]
    r = with_floor(T, 10 ** 12, lambda: timed(lambda: model.predict_rank_at(sub_u, itf, sub_p), args.reps))
    assert model.last_rank_info['path'] == 'dense+rank'
    r['users'] = rows
    r['extrapolated_s_1M_users'] = r['ms_median'] * n / rows / 1e3
    out['dense'] = r
    print('dense', json.dumps(r), file=sys.stderr, flush=True)
    yield


def run_crossover(args, T, out):
    import torch
    U, d = 65536, 128
    table = []
    for I in (1024, 2048, 4096, 16384, 65536):
        uf, itf, wu, wi, bu, bi = problem(U, I, d)
        model = model_of('dot', d, wu, wi, bu, bi)
        pairs = random_pairs(U, I, 10, seed=5)
        row = {'items': I}
        for route, floor in (('exact3_count', 0), ('dense+rank', 10 ** 12)):
            row[route] = with_floor(T, floor, lambda: timed(lambda: model.predict_rank_at(uf, itf, pairs), args.reps))
            assert model.last_rank_info['path'] == route
        del model
        torch.cuda.empty_cache()
        table.append(row)
        print('crossover', json.dumps(row), file=sys.stderr, flush=True)
        out['crossover'] = {'workload': '%d users, d%d, 10 random pairs per user, biased dot' % (U, d), 'table': table}
        yield


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--parts', default='flagship,dense,crossover')
    ap.add_argument('--cases', default='a,b,c,euclidean,attention')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--oracle-rows', type=int, default=64)
    ap.add_argument('--flagship-size', type=int, default=1000000)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    import tensorrec_b200 as T
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    out = {'card': card(), 'RANK_AT_MIN_ITEMS': T.tensorrec.RANK_AT_MIN_ITEMS}
    parts = {'flagship': run_flagship, 'dense': run_dense, 'crossover': run_crossover}
    for part in args.parts.split(','):
        for _ in parts[part](args, T, out):
            with open(os.path.join(args.out, 'bench_rank_at.json'), 'w') as f:   # after every step: partial results
                json.dump({k: v for k, v in out.items() if not k.startswith('_')}, f, indent=1)
    print(json.dumps({k: v for k, v in out.items() if not k.startswith('_')}))


if __name__ == '__main__':
    main()
