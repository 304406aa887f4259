"""Measures predict_at: the exact kernel's pairs mode ('exact3_pairs') against the capture launch of the counting mode
over the same pairs and against 'dense+gather'.

    python scripts/bench_predict_at.py [--users N] [--items N] [--d 128] [--reps 3] [--out FILE]

Reports the card name and power limit of the run, then per case the milliseconds per predict_at call (median of
--reps after one warm-up, with the range), the host planner's share, the gathered tiles, and a bit-for-bit check of
32 whole user blocks against predict_batches."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tensorrec_b200 import kernels, prediction_graphs as P, representation_graphs as R, tensorrec  # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        q = 'unknown (%s)' % e
    return q


def features(n, n_features, seed):
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(n), 4)
    cols = rng.integers(0, n_features, rows.size)
    return sp.csr_matrix((np.ones(rows.size, np.float32), (rows, cols)), shape=(n, n_features))


def model_for(form, d, n_features, seed=0):
    rng = np.random.default_rng(seed)
    n_tastes = 3 if form == 'attention' else 1
    pred = P.EuclideanSimilarityPredictionGraph() if form == 'euclidean' else P.DotProductPredictionGraph()
    m = tensorrec.TensorRec(n_components=d, n_tastes=n_tastes, prediction_graph=pred,
                            attention_graph=R.LinearRepresentationGraph() if form == 'attention' else None)
    w = {'linear_weights_item': rng.standard_normal((n_features, d)).astype(np.float32) * 0.1,
         'feature_biases_user': rng.standard_normal((n_features, 1)).astype(np.float32),
         'feature_biases_item': rng.standard_normal((n_features, 1)).astype(np.float32)}
    for t in range(n_tastes):
        w['linear_weights_user_%d' % t] = rng.standard_normal((n_features, d)).astype(np.float32) * 0.1
        if form == 'attention':
            w['linear_weights_attn_%d' % t] = rng.standard_normal((n_features, d)).astype(np.float32) * 0.1
    m.set_weights(w)
    return m


def listing(kind, n_users, n_items, seed):
    rng = np.random.default_rng(seed)
    if kind == 'pareto':
        per_row = np.minimum(1000, np.ceil(rng.pareto(1.5, n_users) * 5)).astype(np.int64)
    else:
        per_row = np.full(n_users, int(kind), np.int64)
    rows = np.repeat(np.arange(n_users), per_row)
    cols = rng.integers(0, n_items, rows.size)
    m = sp.csr_matrix((np.ones(rows.size, np.float32), (rows, cols)), shape=(n_users, n_items))
    m.sum_duplicates()
    return m


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, 1e3 * (time.perf_counter() - t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--users', type=int, default=1 << 20)
    ap.add_argument('--items', type=int, default=1 << 20)
    ap.add_argument('--d', type=int, default=128)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--cases', default='dot:1,dot:10,dot:pareto,euclidean:10,attention:10')
    ap.add_argument('--crossover', action='store_true')
    ap.add_argument('--crossover-items', default='1024,4096,16384,65536,131072,262144,524288,1048576')
    ap.add_argument('--crossover-users', type=int, default=16384)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    report = {'card': card(), 'users': a.users, 'items': a.items, 'd': a.d, 'cases': []}
    print(json.dumps({'card': report['card']}), flush=True)
    nf = 4096
    if a.cases:
        uf, itf = features(a.users, nf, 1), features(a.items, nf, 2)
    plan_ms = []
    real_plan = kernels.pairs_plan

    def clocked_plan(*args, **kw):
        t = time.perf_counter()
        out = real_plan(*args, **kw)
        plan_ms.append(1e3 * (time.perf_counter() - t))
        return out
    kernels.pairs_plan = clocked_plan
    for case in [c for c in a.cases.split(',') if c]:
        form, kind = case.split(':')
        model = model_for(form, a.d, nf)
        pairs = listing(kind, a.users, a.items, 3)
        model.predict_at(uf, itf, pairs)                        # warm-up
        times, plans = [], []
        for _ in range(a.reps):
            plan_ms.clear()
            out, ms = timed(lambda: model.predict_at(uf, itf, pairs))
            times.append(ms)
            plans.append(sum(plan_ms))
        info = dict(model.last_predict_at_info)
        # the capture launch of the counting mode over the same pairs (one full exact sweep)
        rank_ms = None
        if form == 'dot':
            _, rank_ms = timed(lambda: model.predict_rank_at(uf, itf, pairs))
        # dense+gather on 4096 users, extrapolated
        sub = 4096
        tensorrec_route = tensorrec.predict_at_route
        tensorrec.predict_at_route = lambda _n, _ok: 'dense+gather'
        try:
            model.predict_at(uf[:sub], itf, pairs[:sub])
            _, dg = timed(lambda: model.predict_at(uf[:sub], itf, pairs[:sub]))
        finally:
            tensorrec.predict_at_route = tensorrec_route
        # 32 whole user blocks bit for bit against predict_batches
        n_check = min(a.users, 32 * 128)
        got = out[:n_check].tocsr()
        ok = True
        for u0, u1, block in model.predict_batches(uf[:n_check], itf, user_batch_size=1024):
            g = got[u0:u1]
            r, c = g.nonzero()
            want = np.ascontiguousarray(block[r, c])
            gv = np.asarray(g[r, c]).reshape(-1).astype(np.float32)
            ok = ok and np.array_equal(gv.view(np.int32), want.view(np.int32))
        row = {'case': case, 'pairs': int(pairs.nnz), 'ms_median': float(np.median(times)), 'ms_min': min(times),
               'ms_max': max(times), 'planner_ms_median': float(np.median(plans)), 'tiles': info['tiles'],
               'path': info['path'], 'rank_at_ms': rank_ms, 'dense_gather_4096_ms': dg,
               'dense_gather_extrapolated_ms': dg * a.users / sub, 'bits_equal_32_blocks': bool(ok)}
        report['cases'].append(row)
        print(json.dumps(row), flush=True)
    if a.crossover:
        model = model_for('dot', a.d, nf)
        for n_items in [int(n) for n in a.crossover_items.split(',')]:
            it = features(n_items, nf, 5)
            users = features(a.crossover_users, nf, 6)
            pairs = listing('10', a.crossover_users, n_items, 7)
            row = {'crossover_items': n_items}
            for route in ('exact3_pairs', 'dense+gather'):
                saved = tensorrec.predict_at_route
                tensorrec.predict_at_route = lambda _n, _ok, r=route: r
                try:
                    model.predict_at(users, it, pairs)
                    ts = [timed(lambda: model.predict_at(users, it, pairs))[1] for _ in range(a.reps)]
                finally:
                    tensorrec.predict_at_route = saved
                row[route] = float(np.median(ts))
            report.setdefault('crossover', []).append(row)
            print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(report, f, indent=1)


if __name__ == '__main__':
    main()
