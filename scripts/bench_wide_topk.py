"""Top-k lists with 32 < k <= 1024: the wide filter route against dense+rank, on one GPU.

    python scripts/bench_wide_topk.py --out DIR [--sections flagship,dense,crossover,similar] [--users N --items N]

Sections (each writes its part of DIR/bench_wide_topk.json, with the card's name and power limit read in the same run):
  flagship   bench.py's flagship inputs (indicator features, normal L2-normalised weights, N(0, 0.1) biases; 1M users x
             1M items x d128 by default), predict_top_k(..., to_host=False) for every k of --ks: one warm-up pass, then
             --reps timed passes ended by a device synchronisation (median and range), the route, the rows sent to the
             dense fallback, the peak device memory of a pass, and --check-rows sampled rows against the CPU oracle.
  dense      today's route for k = 100 on the same catalogue: dense+rank with an explicit user_batch_size over
             --dense-users users; the per-user cost times the flagship's users is reported as an extrapolation.
  crossover  k = 100, --cross-users users, n_items in --cross-items, both routes (WIDE_MIN_ITEMS forced either way):
             the measurement that sets tensorrec.WIDE_MIN_ITEMS.  The items on each side of it are the workloads that
             keep both routes measured.
  similar    the related-items table predict_similar_items_top_k(n_similar=100, exclude_self=True) over every item of
             the flagship catalogue, dot and Euclidean."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import bench  # noqa: E402
from bench_similar import card, oracle_rows  # noqa: E402


def timed(fn, reps):
    """One warm-up call, then `reps` timed calls: (ms list, last result, peak device bytes of a call)."""
    import torch
    fn()
    ms, out = [], None
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    for _ in range(reps):
        out = None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ms.append(1e3 * (time.perf_counter() - t0))
    return ms, out, int(torch.cuda.max_memory_allocated() - base)


def summary(ms):
    return {'ms': ms, 'ms_median': float(np.median(ms)), 'ms_range': [float(min(ms)), float(max(ms))]}


def flagship(args, model, uf, itf, wu, wi, bu, bi):
    import torch
    from tensorrec_b200 import tensorrec as TR
    res = {}
    ks = [int(k) for k in args.ks.split(',')]
    sample = np.sort(np.random.default_rng(11).choice(args.users, min(args.check_rows, args.users), replace=False))
    exp, item_repr, item_bias = bench.oracle_topk_rows(uf, itf, wu, wi, bu, bi, sample, max(ks))
    from oracle import reference_ops as R
    user_repr = R.sparse_dense_matmul_fast(uf[sample], wu).astype(np.float64)
    user_bias = np.asarray(uf[sample] @ bu, dtype=np.float64)

    def exact64(rows, ids):
        """float64 scores of (sampled row j, item ids[j]) pairs, and |u||i| of each pair"""
        ir = item_repr[ids].astype(np.float64)
        dot = np.einsum('jd,jkd->jk', user_repr[rows], ir)
        norm = np.linalg.norm(user_repr[rows], axis=1)[:, None] * np.linalg.norm(ir, axis=2)
        return dot + user_bias[rows, None] + item_bias[ids].astype(np.float64), norm
    for k in ks:
        infos = []

        def run():
            top = model.predict_top_k(uf, itf, k, to_host=False)
            infos.append(dict(model.last_topk_info))
            return top
        ms, top, peak = timed(run, args.reps)
        got = top.items.cpu().numpy()[sample]
        del top
        torch.cuda.empty_cache()
        differ = (got != exp[:, :k]).any(axis=1)
        # a differing slot is a near-tie when the float64 scores of the kernel's item and the oracle's item in that slot
        # differ by less than the fp32 arithmetic of either side can resolve
        rows = np.nonzero(differ)[0]
        gap = None
        if len(rows):
            s_got, norm = exact64(rows, got[rows])
            s_exp, _ = exact64(rows, exp[rows, :k])
            slot = got[rows] != exp[rows, :k]
            gap = float(np.max(np.abs(s_got - s_exp)[slot] / norm[slot]))
        res[k] = dict(summary(ms), path=infos[-1]['path'], fallback_rows=[int(i['fallback_rows']) for i in infos[1:]],
                      peak_device_bytes=peak, default_user_block=int(model._topk_block_rows(infos[-1]['path'],
                                                                                           args.users, args.items, k)),
                      oracle_check={'rows': int(len(sample)), 'rows_differing': int(differ.sum()),
                                    'slots_differing': int((got != exp[:, :k]).sum()),
                                    'max_float64_score_gap_of_differing_slots_over_norms': gap})
        print('flagship k=%d' % k, json.dumps(res[k]), file=sys.stderr, flush=True)
    res['wide_min_items'] = TR.WIDE_MIN_ITEMS
    return res


def dense_baseline(args, model, uf, itf):
    import torch
    from tensorrec_b200 import tensorrec as TR
    rows = uf[:args.dense_users]
    old = TR.WIDE_MIN_ITEMS
    TR.WIDE_MIN_ITEMS = 10 ** 12
    try:
        infos = []

        def run():
            top = model.predict_top_k(rows, itf, 100, to_host=False, user_batch_size=args.dense_block)
            infos.append(model.last_topk_info['path'])
            return top
        ms, _, peak = timed(run, args.reps)
    finally:
        TR.WIDE_MIN_ITEMS = old
    torch.cuda.empty_cache()
    per_user = float(np.median(ms)) / args.dense_users
    return dict(summary(ms), path=infos[-1], users=args.dense_users, user_batch_size=args.dense_block,
                peak_device_bytes=peak, ms_per_user=per_user,
                extrapolated_ms_for_flagship_users=per_user * args.users)


def crossover(args):
    import torch
    from tensorrec_b200 import TensorRec, tensorrec as TR
    uf = bench.indicator_csr(args.cross_users, seed=0)
    rng = np.random.default_rng(4)
    res = {}
    for n_items in [int(i) for i in args.cross_items.split(',')]:
        itf = bench.indicator_csr(n_items, seed=1)
        model = TensorRec(n_components=args.d)
        model.set_weights({'linear_weights_user_0': bench.make_weights(uf.shape[1], args.d, seed=2),
                           'linear_weights_item': bench.make_weights(itf.shape[1], args.d, seed=3),
                           'feature_biases_user': (0.1 * rng.standard_normal((uf.shape[1], 1))).astype(np.float32),
                           'feature_biases_item': (0.1 * rng.standard_normal((itf.shape[1], 1))).astype(np.float32)})
        row = {}
        old = TR.WIDE_MIN_ITEMS
        for route, threshold in (('wide', 0), ('dense+rank', 10 ** 12)):
            TR.WIDE_MIN_ITEMS = threshold
            try:
                ms, top, peak = timed(lambda: model.predict_top_k(uf, itf, 100, to_host=False), args.reps)
                row[route] = dict(summary(ms), path=model.last_topk_info['path'], peak_device_bytes=peak,
                                  fallback_rows=int(model.last_topk_info['fallback_rows']))
                row[route]['items'] = top.items.cpu().numpy()
            finally:
                TR.WIDE_MIN_ITEMS = old
            del top
            torch.cuda.empty_cache()
        row['routes_agree_rows'] = int((row['wide'].pop('items') == row['dense+rank'].pop('items')).all(axis=1).sum())
        res[n_items] = row
        print('crossover items=%d' % n_items, json.dumps(row), file=sys.stderr, flush=True)
    return res


def similar(args, itf, wi):
    import torch
    from tensorrec_b200 import TensorRec, prediction_graphs as P
    from oracle import reference_ops as R
    item_repr = R.sparse_dense_matmul_fast(itf, wi)
    sample = np.sort(np.random.default_rng(11).choice(args.items, min(args.check_rows, args.items), replace=False))
    res = {}
    graphs = {'dot': P.DotProductPredictionGraph, 'euclidean': P.EuclideanSimilarityPredictionGraph}
    for name in args.similar_graphs.split(','):
        graph = graphs[name]
        model = TensorRec(n_components=args.d, prediction_graph=graph())
        model.set_weights({'linear_weights_item': wi})
        infos = []

        def run():
            top = model.predict_similar_items_top_k(itf, 100, exclude_self=True, to_host=False)
            infos.append(dict(model.last_topk_info))
            return top
        ms, top, peak = timed(run, args.reps)
        got = top.items.cpu().numpy()[sample]
        del top
        torch.cuda.empty_cache()
        exp, _ = oracle_rows(name, item_repr, None, sample, 100)
        # differing slots: the float64 gap between the kernel's and the oracle's item, on the scale the kernels rank by
        # (dot: q.i over |q||i|; Euclidean: d^2 over |q|^2 + |i|^2)
        rows = np.nonzero((got != exp).any(axis=1))[0]
        gap = None
        if len(rows):
            q = item_repr[sample[rows]].astype(np.float64)
            slot = got[rows] != exp[rows]

            def score(ids):
                it = item_repr[ids].astype(np.float64)
                if name == 'dot':
                    return (np.einsum('jd,jkd->jk', q, it),
                            np.linalg.norm(q, axis=1)[:, None] * np.linalg.norm(it, axis=2))
                return (np.sum((q[:, None, :] - it) ** 2, axis=2),
                        np.sum(q * q, axis=1)[:, None] + np.sum(it * it, axis=2))
            s_got, scale = score(got[rows])
            s_exp, _ = score(exp[rows])
            gap = float(np.max(np.abs(s_got - s_exp)[slot] / scale[slot]))
        res[name] = dict(summary(ms), path=infos[-1]['path'], fallback_rows=[int(i['fallback_rows']) for i in infos[1:]],
                         peak_device_bytes=peak, oracle_check={'rows': int(len(sample)), 'rows_differing': int(len(rows)),
                                                               'slots_differing': int((got != exp).sum()),
                                                               'max_float64_gap_of_differing_slots': gap})
        print('similar', name, json.dumps(res[name]), file=sys.stderr, flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--sections', default='flagship,dense,crossover,similar')
    ap.add_argument('--users', type=int, default=1000000)
    ap.add_argument('--items', type=int, default=1000000)
    ap.add_argument('--d', type=int, default=128)
    ap.add_argument('--ks', default='10,32,100,1000')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--check-rows', type=int, default=4096)
    ap.add_argument('--dense-users', type=int, default=4096)
    ap.add_argument('--dense-block', type=int, default=1024)
    ap.add_argument('--cross-users', type=int, default=65536)
    ap.add_argument('--cross-items', default='1024,4096,16384,65536')
    ap.add_argument('--similar-graphs', default='dot,euclidean')
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, 'bench_wide_topk.json')
    info = json.load(open(path)) if os.path.exists(path) else {}
    info['card'] = card()
    info.setdefault('config', {}).update(vars(args))

    from tensorrec_b200 import TensorRec, kernels
    kernels.require_cuda()

    def save():
        with open(path, 'w') as f:
            json.dump(info, f, indent=1)
    sections = args.sections.split(',')
    if 'crossover' in sections:
        info['crossover_k100'] = crossover(args)
        save()
    if sections == ['crossover']:
        sections = []
    else:
        problem = argparse.Namespace(users=args.users, items=args.items, d=args.d, scores='iid')
        uf, itf, wu, wi, bu, bi = bench.make_problem(problem)
        model = TensorRec(n_components=args.d)
        model.set_weights({'linear_weights_user_0': wu, 'linear_weights_item': wi,
                           'feature_biases_user': bu[:, None], 'feature_biases_item': bi[:, None]})
    if 'flagship' in sections:
        info['flagship'] = flagship(args, model, uf, itf, wu, wi, bu, bi)
        save()
    if 'dense' in sections:
        info['dense_k100'] = dense_baseline(args, model, uf, itf)
        save()
    if 'similar' in sections:
        info['similar_n100'] = similar(args, itf, wi)
        save()
    print(json.dumps(info))


if __name__ == '__main__':
    main()
