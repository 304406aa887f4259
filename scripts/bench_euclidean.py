"""Euclidean user x item models on the tensor-core kernels, on one GPU.

    python scripts/bench_euclidean.py --out DIR [--parts flagship,dense,crossover --reps R --check-rows R]

Inputs are bench.py's flagship problem (indicator features, normal L2-normalised weights, 0.1-normal biases) with a
biased EuclideanSimilarityPredictionGraph model.  Every timing is one warm-up pass, then R timed passes (median and
range); a pass is one call ended by a device synchronisation.
  flagship   1M users x 1M items x d128, k = 10: predict_top_k(..., to_host=False) on its route, sampled rows against
             the CPU oracle; in the same session the dot model on 'exact3' (TOPK_PATH=exact) and the Euclidean model on
             'dense+rank' over 4096 users (EUCLIDEAN_MIN_ITEMS forced above n_items), extrapolated to 1M users.
  dense      predict()'s scoring into a resident [65536, 100000] matrix at d64: Euclidean on tensor cores, dot on tensor
             cores and Euclidean on the CUDA-core kernel (SCORE_PATH=exact), alternated.
  crossover  65536 users, k = 10, items in {1K, 2K, 4K, 16K, 64K}: 'exact3' and 'dense+rank' forced in turn.
Results, with the card's name and power limit, go to DIR/bench_euclidean.json."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from scripts.bench_similar import card  # noqa: E402


def timed(fn, reps):
    import torch
    fn()                                                       # warm-up
    ms = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ms.append(1e3 * (time.perf_counter() - t0))
    return {'ms': ms, 'ms_median': float(np.median(ms)), 'ms_range': [min(ms), max(ms)]}


def problem(users, items, d):
    ns = argparse.Namespace(users=users, items=items, d=d)
    return bench.make_problem(ns)


def model_of(kind, d, wu, wi, bu, bi):
    from tensorrec_b200 import TensorRec, prediction_graphs as P
    graph = P.EuclideanSimilarityPredictionGraph() if kind == 'euclidean' else P.DotProductPredictionGraph()
    model = TensorRec(n_components=d, prediction_graph=graph)
    model.set_weights({'linear_weights_user_0': wu, 'linear_weights_item': wi, 'feature_biases_user': bu[:, None],
                       'feature_biases_item': bi[:, None]})
    return model


def oracle_rows(uf, itf, wu, wi, bu, bi, rows, k, chunk=128):
    """The reference's Euclidean top-k (scores, then bias_prediction_dense) of the user rows `rows`."""
    from oracle import reference_ops as R
    item_repr = R.sparse_dense_matmul_fast(itf, wi)
    ib = np.asarray(itf.astype(np.float32) @ bi, dtype=np.float32)
    ids, vals = [], []
    for c0 in range(0, len(rows), chunk):
        sub = uf[rows[c0:c0 + chunk]]
        s = R.bias_prediction_dense(R.euclidean_dense(R.sparse_dense_matmul_fast(sub, wu), item_repr),
                                    np.asarray(sub.astype(np.float32) @ bu, dtype=np.float32), ib)
        i, v = R.top_k_from_scores_fast(s, k)
        ids.append(i)
        vals.append(v)
    return np.concatenate(ids), np.concatenate(vals)


def run_flagship(args, T, out):
    import torch
    n, d, k = args.flagship_size, 128, 10
    uf, itf, wu, wi, bu, bi = problem(n, n, d)
    res = {'workload': '%d users x %d items x d%d, k=%d, biased' % (n, n, d, k)}
    model = model_of('euclidean', d, wu, wi, bu, bi)
    box = {}

    def euclid():
        box['top'] = model.predict_top_k(uf, itf, k, to_host=False)
    res['euclidean'] = timed(euclid, args.reps)
    res['euclidean']['path'] = model.last_topk_info['path']
    sample = np.sort(np.random.default_rng(11).choice(n, min(args.check_rows, n), replace=False))
    got_i = box['top'].items.cpu().numpy()[sample]
    got_s = box['top'].scores.cpu().numpy()[sample]
    del box['top']
    torch.cuda.empty_cache()
    exp_i, exp_s = oracle_rows(uf, itf, wu, wi, bu, bi, sample, k)
    res['euclidean']['oracle_check'] = {'rows': int(len(sample)),
                                        'rows_differing': int((got_i != exp_i).any(axis=1).sum()),
                                        'slots_differing': int((got_i != exp_i).sum()),
                                        'scores_equal_where_ids_equal': bool(np.array_equal(got_s[got_i == exp_i],
                                                                                            exp_s[got_i == exp_i]))}
    print('flagship euclidean', json.dumps(res['euclidean']), file=sys.stderr, flush=True)

    dot = model_of('dot', d, wu, wi, bu, bi)
    old = T.tensorrec.TOPK_PATH
    T.tensorrec.TOPK_PATH = 'exact'
    res['dot_exact3'] = timed(lambda: dot.predict_top_k(uf, itf, k, to_host=False), args.reps)
    res['dot_exact3']['path'] = dot.last_topk_info['path']
    T.tensorrec.TOPK_PATH = old
    print('flagship dot', json.dumps(res['dot_exact3']), file=sys.stderr, flush=True)

    few = uf[:4096]
    floor = T.tensorrec.EUCLIDEAN_MIN_ITEMS
    T.tensorrec.EUCLIDEAN_MIN_ITEMS = 10 ** 12
    dr = timed(lambda: model.predict_top_k(few, itf, k, to_host=False), args.reps)
    dr['path'] = model.last_topk_info['path']
    T.tensorrec.EUCLIDEAN_MIN_ITEMS = floor
    dr['users'] = 4096
    dr['extrapolated_s_for_all_users'] = dr['ms_median'] * n / 4096 / 1e3
    res['euclidean_dense_rank_4096_users'] = dr
    print('flagship dense+rank', json.dumps(dr), file=sys.stderr, flush=True)
    out['flagship'] = res
    del model, dot
    torch.cuda.empty_cache()


def run_dense(args, T, out):
    import torch
    from tensorrec_b200.input_utils import SparseInput
    U, I, d = 65536, 100000, 64
    uf, itf, wu, wi, bu, bi = problem(U, I, d)
    user_in, item_in = SparseInput(uf), SparseInput(itf)
    dev = torch.device('cuda', torch.cuda.current_device())
    buf = torch.empty((U, I), dtype=torch.float32, device=dev)
    models = {'euclidean_tensor': model_of('euclidean', d, wu, wi, bu, bi), 'dot_tensor': model_of('dot', d, wu, wi, bu, bi),
              'euclidean_exact': model_of('euclidean', d, wu, wi, bu, bi)}

    def run(name):
        old = T.tensorrec.SCORE_PATH
        T.tensorrec.SCORE_PATH = 'exact' if name == 'euclidean_exact' else 'auto'
        try:
            models[name]._score_plan(item_in, dev)(user_in, out=buf)
        finally:
            T.tensorrec.SCORE_PATH = old
    for name in models:
        run(name)                                              # warm-up of every form
    ms = {name: [] for name in models}
    for _ in range(args.reps):                                 # alternated
        for name in models:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(name)
            torch.cuda.synchronize()
            ms[name].append(1e3 * (time.perf_counter() - t0))
    out['dense'] = {'workload': 'scores of %d users x %d items x d%d into a resident device matrix, biased' % (U, I, d),
                    'results': {name: {'ms': v, 'ms_median': float(np.median(v)), 'ms_range': [min(v), max(v)]}
                                for name, v in ms.items()}}
    print('dense', json.dumps(out['dense']), file=sys.stderr, flush=True)
    del buf
    torch.cuda.empty_cache()


def run_crossover(args, T, out):
    import torch
    U, d, k = 65536, 128, 10
    table = []
    for I in (1024, 2048, 4096, 16384, 65536):
        uf, itf, wu, wi, bu, bi = problem(U, I, d)
        model = model_of('euclidean', d, wu, wi, bu, bi)
        row = {'items': I}
        floor = T.tensorrec.EUCLIDEAN_MIN_ITEMS
        for route, f in (('exact3', 0), ('dense+rank', 10 ** 12)):
            T.tensorrec.EUCLIDEAN_MIN_ITEMS = f
            r = timed(lambda: model.predict_top_k(uf, itf, k, to_host=False), args.reps)
            assert model.last_topk_info['path'] == route
            row[route] = r
        T.tensorrec.EUCLIDEAN_MIN_ITEMS = floor
        table.append(row)
        print('crossover', json.dumps(row), file=sys.stderr, flush=True)
        del model
        torch.cuda.empty_cache()
    out['crossover'] = {'workload': '%d users, d%d, k=%d, biased' % (U, d, k), 'table': table}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--parts', default='crossover,dense,flagship')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--check-rows', type=int, default=4096)
    ap.add_argument('--flagship-size', type=int, default=1000000)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    import tensorrec_b200 as T
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    out = {'card': card(), 'EUCLIDEAN_MIN_ITEMS': T.tensorrec.EUCLIDEAN_MIN_ITEMS}
    parts = {'flagship': run_flagship, 'dense': run_dense, 'crossover': run_crossover}
    for part in args.parts.split(','):
        parts[part](args, T, out)
        with open(os.path.join(args.out, 'bench_euclidean.json'), 'w') as f:   # after every part: partial results
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
