"""Top-k lists with 32 < k <= 1024 for Euclidean and attention models on the exact kernel's wide mode, on one GPU.

    python scripts/bench_exact_wide.py --out DIR [--parts crossover,flagship --reps R --check-rows R]

Inputs are bench.py's flagship problem with bench_euclidean.py's biased Euclidean model and bench_tastes.py's biased
three-taste attention model.  Every timing is one warm-up pass, then R timed passes (median and range); a pass is one
predict_top_k(..., to_host=False) call ended by a device synchronisation.
  flagship   1M users x 1M items x d128: Euclidean at k = 100 and k = 1000, attention at k = 100, on 'exact3_wide',
             with the peak device memory of a pass and --check-rows sampled rows against the CPU oracle; every slot
             whose id differs from the oracle's is reported with the float64 scores of both ids (a near-tie when they
             differ by at most 1e-5 (1 + |score|)).  --cases picks some of them, e.g. euclidean:1000,attention:100.
  crossover  65536 users, d128, k = 100, items in {1K, 2K, 4K, 16K, 64K}, both models: 'exact3_wide' and 'dense+rank'
             forced in turn.
Results, with the card's name and power limit, go to DIR/bench_exact_wide.json."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts import bench_euclidean as BE  # noqa: E402
from scripts import bench_tastes as BT  # noqa: E402
from scripts.bench_euclidean import problem, timed  # noqa: E402
from scripts.bench_similar import card  # noqa: E402


def model_of(kind, d, wu, wi, bu, bi):
    return BE.model_of('euclidean', d, wu, wi, bu, bi) if kind == 'euclidean' else BT.model_of(True, d, wu, wi, bu, bi)


def with_floor(T, floor, fn):
    old = T.tensorrec.EXACT_WIDE_MIN_ITEMS
    T.tensorrec.EXACT_WIDE_MIN_ITEMS = floor
    try:
        return fn()
    finally:
        T.tensorrec.EXACT_WIDE_MIN_ITEMS = old


def float64_scores(kind, uf, itf, wu, wi, bu, bi, rows, cols):
    """float64 scores of the (rows[j], cols[j]) pairs from the oracle's fp32 representations."""
    from oracle import reference_ops as R
    sub = uf[rows]
    it = itf[cols]
    item = R.sparse_dense_matmul_fast(it, wi).astype(np.float64)
    ub = np.asarray(sub @ bu, dtype=np.float64)
    ib = np.asarray(it @ bi, dtype=np.float64)
    if kind == 'euclidean':
        user = R.sparse_dense_matmul_fast(sub, wu).astype(np.float64)
        pred = -np.sqrt(np.maximum(((user - item) ** 2).sum(1), 1e-16))
    else:
        wus, was = BT.weights_of(wu)
        p = np.stack([(R.sparse_dense_matmul_fast(sub, w).astype(np.float64) * item).sum(1) for w in wus])
        a = np.stack([(R.sparse_dense_matmul_fast(sub, w).astype(np.float64) * item).sum(1) for w in was])
        w = np.exp(a - a.max(0))
        pred = (w / w.sum(0) * p).sum(0)
    return pred + ub + ib


def oracle_check(kind, top, uf, itf, wu, wi, bu, bi, n_rows, k):
    n = uf.shape[0]
    sample = np.sort(np.random.default_rng(11).choice(n, min(n_rows, n), replace=False))
    got_i = top.items.cpu().numpy()[sample]
    oracle_rows = BE.oracle_rows if kind == 'euclidean' else BT.oracle_rows
    parts = []
    for r0 in range(0, len(sample), 256):          # progress on stderr: the CPU oracle takes minutes
        parts.append(oracle_rows(uf, itf, wu, wi, bu, bi, sample[r0:r0 + 256], k)[0])
        print('oracle rows %d / %d' % (r0 + len(parts[-1]), len(sample)), file=sys.stderr, flush=True)
    exp_i = np.concatenate(parts)
    r, c = np.nonzero(got_i != exp_i)
    res = {'rows': int(len(sample)), 'rows_differing': int(len(np.unique(r))), 'slots_differing': int(len(r))}
    if len(r):
        rows = sample[r]
        s_got = float64_scores(kind, uf, itf, wu, wi, bu, bi, rows, got_i[r, c])
        s_exp = float64_scores(kind, uf, itf, wu, wi, bu, bi, rows, exp_i[r, c])
        gap = np.abs(s_got - s_exp)
        res['max_float64_gap'] = float(gap.max())
        res['all_near_ties'] = bool(np.all(gap <= 1e-5 * (1 + np.abs(s_exp))))
    return res


def run_flagship(args, T, out):
    import torch
    n, d = args.flagship_size, 128
    uf, itf, wu, wi, bu, bi = problem(n, n, d)
    res = {'workload': '%d users x %d items x d%d, biased' % (n, n, d)}
    for kind, k in [c for c in (('euclidean', 100), ('euclidean', 1000), ('attention', 100))
                    if args.cases is None or '%s:%d' % c in args.cases.split(',')]:
        model = model_of(kind, d, wu, wi, bu, bi)
        box = {}

        def run():
            box['top'] = model.predict_top_k(uf, itf, k, to_host=False)
        torch.cuda.reset_peak_memory_stats()
        r = timed(run, args.reps)
        r['peak_device_bytes'] = int(torch.cuda.max_memory_allocated())
        r['path'] = model.last_topk_info['path']
        r['oracle_check'] = oracle_check(kind, box.pop('top'), uf, itf, wu, wi, bu, bi, args.check_rows, k)
        res['%s_k%d' % (kind, k)] = r
        print('flagship', kind, k, json.dumps(r), file=sys.stderr, flush=True)
        del model
        torch.cuda.empty_cache()
    out['flagship'] = res


def run_crossover(args, T, out):
    import torch
    U, d, k = 65536, 128, 100
    table = []
    for I in (1024, 2048, 4096, 16384, 65536):
        uf, itf, wu, wi, bu, bi = problem(U, I, d)
        row = {'items': I}
        for kind in ('euclidean', 'attention'):
            model = model_of(kind, d, wu, wi, bu, bi)
            for route, floor in (('exact3_wide', 0), ('dense+rank', 10 ** 12)):
                r = with_floor(T, floor, lambda: timed(lambda: model.predict_top_k(uf, itf, k, to_host=False),
                                                       args.reps))
                assert model.last_topk_info['path'] == route
                row['%s %s' % (kind, route)] = r
            del model
            torch.cuda.empty_cache()
        table.append(row)
        print('crossover', json.dumps(row), file=sys.stderr, flush=True)
    out['crossover'] = {'workload': '%d users, d%d, k=%d, biased' % (U, d, k), 'table': table}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--parts', default='crossover,flagship')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--check-rows', type=int, default=4096)
    ap.add_argument('--flagship-size', type=int, default=1000000)
    ap.add_argument('--cases', default=None, help="flagship cases to run, e.g. 'attention:100' (default: all)")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    import tensorrec_b200 as T
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    out = {'card': card(), 'EXACT_WIDE_MIN_ITEMS': T.tensorrec.EXACT_WIDE_MIN_ITEMS}
    parts = {'flagship': run_flagship, 'crossover': run_crossover}
    for part in args.parts.split(','):
        parts[part](args, T, out)
        with open(os.path.join(args.out, 'bench_exact_wide.json'), 'w') as f:   # after every part: partial results
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
