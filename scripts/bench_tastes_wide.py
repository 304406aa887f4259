"""Mixture-of-tastes top-k lists with 32 < k <= 1024 on the wide route, on one GPU.

    python scripts/bench_tastes_wide.py --out DIR [--parts merge,crossover,flagship --reps R --check-rows R]

Inputs are bench.py's flagship problem with bench_tastes.py's biased dot-product model of three tastes without
attention (the user weights of taste t are bench.py's user weights rolled by t rows).  Every timing is one warm-up pass,
then R timed passes (median and range); a pass is one call ended by a device synchronisation.
  flagship   1M users x 1M items x d128, k = 100 and k = 1000: predict_top_k(..., to_host=False) on 'wide', with the
             fallback rows and peak device memory of a pass, and --check-rows sampled rows against the CPU oracle
             (max over the tastes, then the biases) with the float64 gap of every differing slot over |u_t*||i| (t* the
             taste that gives the item its score); 'dense+rank' over 4096 users (WIDE_MIN_ITEMS forced above n_items),
             extrapolated to 1M users.
  merge      trk_topk_merge_dedup_pair alone (CUDA events) over 1M rows for k = 100 and k = 1000: two sorted lists per
             row whose ids partly overlap (A: (7919 u + 13 j) mod 1M, B: (7919 u + 17 j) mod 1M).
  crossover  65536 users, k = 100, items in {1K, 2K, 4K, 16K, 64K}: 'wide' and 'dense+rank' forced in turn.
Results, with the card's name and power limit, go to DIR/bench_tastes_wide.json."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.bench_euclidean import problem, timed  # noqa: E402
from scripts.bench_similar import card  # noqa: E402
from scripts.bench_tastes import N_TASTES, model_of, weights_of  # noqa: E402


def with_floor(T, floor, fn):
    old = T.tensorrec.WIDE_MIN_ITEMS
    T.tensorrec.WIDE_MIN_ITEMS = floor
    try:
        return fn()
    finally:
        T.tensorrec.WIDE_MIN_ITEMS = old


def oracle_rows(uf, itf, wu, wi, bu, bi, rows, k, chunk=64):
    """The reference's top-k (max over the tastes, bias_prediction_dense) of the user rows `rows`, and the float64
    inputs of the gap check: per-taste user representations, user biases, item representations and biases."""
    from oracle import reference_ops as R
    wus, _ = weights_of(wu)
    item_repr = R.sparse_dense_matmul_fast(itf, wi)
    ib = np.asarray(itf.astype(np.float32) @ bi, dtype=np.float32)
    ids = []
    for c0 in range(0, len(rows), chunk):
        sub = uf[rows[c0:c0 + chunk]]
        preds = [R.sparse_dense_matmul_fast(sub, w) @ item_repr.T for w in wus]
        s = R.bias_prediction_dense(R.collapse_mixture_of_tastes(preds, None),
                                    np.asarray(sub.astype(np.float32) @ bu, dtype=np.float32), ib)
        ids.append(R.top_k_from_scores_fast(s, k)[0])
    users = np.stack([R.sparse_dense_matmul_fast(uf[rows], w).astype(np.float64) for w in wus])   # [T, n, d]
    ub = np.asarray(uf[rows] @ bu, dtype=np.float64)
    return np.concatenate(ids), users, ub, item_repr.astype(np.float64), ib.astype(np.float64)


def gaps(got, exp, users, ub, item_repr, ib):
    """float64 |score(kernel's item) - score(oracle's item)| / |u_t*||i| of every differing slot."""
    rows, slots = np.nonzero(got != exp)
    out = []
    for r, j in zip(rows, slots):
        vals = []
        for i in (got[r, j], exp[r, j]):
            if i == 2 ** 31 - 1:
                vals.append((-np.inf, 1.0))
                continue
            per = users[:, r] @ item_repr[i]
            t = int(np.argmax(per))
            vals.append((per[t] + ub[r] + ib[i], np.linalg.norm(users[t, r]) * np.linalg.norm(item_repr[i])))
        out.append(abs(vals[0][0] - vals[1][0]) / max(vals[0][1], vals[1][1]))
    return out


def run_flagship(args, T, out):
    import torch
    n, d = args.flagship_size, 128
    uf, itf, wu, wi, bu, bi = problem(n, n, d)
    model = model_of(False, d, wu, wi, bu, bi)
    res = {'workload': '%d users x %d items x d%d, %d tastes without attention, biased' % (n, n, d, N_TASTES)}
    ks = [int(k) for k in args.ks.split(',')]
    sample = np.sort(np.random.default_rng(11).choice(n, min(args.check_rows, n), replace=False))
    exp, users, ub, item_repr, ib = oracle_rows(uf, itf, wu, wi, bu, bi, sample, max(ks))
    for k in ks:
        box, infos = {}, []

        def fused():
            box['top'] = None
            box['top'] = model.predict_top_k(uf, itf, k, to_host=False)
            infos.append(dict(model.last_topk_info))
        box['top'] = None
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        r = timed(fused, args.reps)
        r['peak_device_bytes'] = int(torch.cuda.max_memory_allocated() - base)
        r['path'] = infos[-1]['path']
        r['fallback_rows'] = [int(i['fallback_rows']) for i in infos]
        got = box['top'].items.cpu().numpy()[sample]
        box['top'] = None
        torch.cuda.empty_cache()
        g = gaps(got, exp[:, :k], users, ub, item_repr, ib)
        r['oracle_check'] = {'rows': int(len(sample)), 'rows_differing': int((got != exp[:, :k]).any(axis=1).sum()),
                             'slots_differing': int((got != exp[:, :k]).sum()),
                             'max_float64_gap_over_norms': float(max(g)) if g else None,
                             'gaps_over_norms': [float(x) for x in sorted(g, reverse=True)[:100]]}
        res['wide_k%d' % k] = r
        print('flagship k=%d' % k, json.dumps(r), file=sys.stderr, flush=True)

    few = uf[:4096]
    dr = with_floor(T, 10 ** 12, lambda: timed(lambda: model.predict_top_k(few, itf, 100, to_host=False), args.reps))
    dr['path'] = model.last_topk_info['path']
    dr['users'] = 4096
    dr['extrapolated_s_for_all_users'] = dr['ms_median'] * n / 4096 / 1e3
    res['dense_rank_k100_4096_users'] = dr
    print('flagship dense+rank', json.dumps(dr), file=sys.stderr, flush=True)
    out['flagship'] = res
    del model
    torch.cuda.empty_cache()


def run_merge(args, T, out):
    import torch
    from tensorrec_b200 import kernels
    n = args.merge_rows
    res = {}
    for k in (100, 1000):
        u = torch.arange(n, dtype=torch.int64, device='cuda')[:, None]
        j = torch.arange(k, dtype=torch.int64, device='cuda')[None, :]
        scores = torch.sort(torch.rand((n, k), device='cuda'), dim=1, descending=True).values
        a, b = kernels.PackedTopK(n, k, 'cuda'), kernels.PackedTopK(n, k, 'cuda')
        a.items.copy_((7919 * u + 13 * j) % 1000000)
        b.items.copy_((7919 * u + 17 * j) % 1000000)
        a.scores.copy_(scores)
        b.scores.copy_(torch.sort(torch.rand((n, k), device='cuda'), dim=1, descending=True).values)
        del scores, u, j
        merged = kernels.topk_merge_dedup(a, b)
        ms = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            kernels.topk_merge_dedup(a, b, out=merged)
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        moved = 3 * n * 8 * k
        med = float(np.median(ms))
        res['k%d' % k] = {'rows': n, 'ms': ms, 'ms_median': med, 'ms_range': [min(ms), max(ms)],
                          'bytes_read_and_written': moved, 'gb_per_s': moved / med / 1e6}
        print('merge k=%d' % k, json.dumps(res['k%d' % k]), file=sys.stderr, flush=True)
        del a, b, merged
        torch.cuda.empty_cache()
    out['merge'] = res


def run_crossover(args, T, out):
    import torch
    U, d, k = 65536, 128, 100
    table = []
    for I in (1024, 2048, 4096, 16384, 65536):
        uf, itf, wu, wi, bu, bi = problem(U, I, d)
        model = model_of(False, d, wu, wi, bu, bi)
        row = {'items': I}
        tops = {}
        for route, floor in (('wide', 0), ('dense+rank', 10 ** 12)):
            def run():
                tops[route] = model.predict_top_k(uf, itf, k, to_host=False)
            r = with_floor(T, floor, lambda: timed(run, args.reps))
            assert model.last_topk_info['path'] == route
            r['fallback_rows'] = int(model.last_topk_info['fallback_rows'])
            row[route] = r
        row['routes_agree_rows'] = int((tops['wide'].items == tops['dense+rank'].items).all(dim=1).sum())
        table.append(row)
        print('crossover', json.dumps(row), file=sys.stderr, flush=True)
        del model, tops
        torch.cuda.empty_cache()
    out['crossover'] = {'workload': '%d users, d%d, %d tastes without attention, k=%d, biased' % (U, d, N_TASTES, k),
                        'table': table}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--parts', default='merge,crossover,flagship')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--ks', default='100,1000')
    ap.add_argument('--check-rows', type=int, default=4096)
    ap.add_argument('--flagship-size', type=int, default=1000000)
    ap.add_argument('--merge-rows', type=int, default=1000000)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    import tensorrec_b200 as T
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    out = {'card': card(), 'WIDE_MIN_ITEMS': T.tensorrec.WIDE_MIN_ITEMS}
    parts = {'flagship': run_flagship, 'merge': run_merge, 'crossover': run_crossover}
    for part in args.parts.split(','):
        parts[part](args, T, out)
        with open(os.path.join(args.out, 'bench_tastes_wide.json'), 'w') as f:   # after every part: partial results
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
