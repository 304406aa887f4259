"""Euclidean mixtures of tastes (max and attention) on the taste-collapsing tensor-core kernel, on one GPU.

    python scripts/bench_tastes_euclid.py --out DIR [--parts dense,flagship,rank_at,crossover --reps R]

Inputs are bench.py's flagship problem (indicator features, normal L2-normalised weights, 0.1-normal biases) with a
biased Euclidean model of three tastes; the user weights of taste t are bench.py's user weights rolled by t rows, the
attention weights of taste t are rolled by 7 + t rows (scripts/bench_tastes.py).  Every timing is one warm-up pass,
then R timed passes (median and range); a pass is one call ended by a device synchronisation.
  dense      predict()'s scoring of 65536 users x 100000 items x d64 into a resident device matrix, max and attention:
             the tensor-core form against SCORE_PATH=exact (the fp32 CUDA-core kernel for max; for attention the torch
             collapse, which holds six [rows, items] matrices, timed on 4096-user blocks and summed over the 16 blocks).
  flagship   the attention model at 1M users x 1M items x d128: top-10 on 'exact3' and top-100 on 'exact3_wide';
             'dense+rank' over 4096 users (the floors forced above n_items), extrapolated to 1M users; --check-rows
             sampled rows of the top-10 against the CPU oracle.
  rank_at    predict_rank_at leave-one-out at 1M x 1M x d128 (one uniformly random item per user), max and attention,
             on 'exact3_count'; the first eight whole user blocks checked against trk_rank_full of their dense
             scores.
  crossover  65536 users x d128, items in {1K, 2K, 4K, 16K, 64K}: attention top-10 ('exact3') and top-100
             ('exact3_wide'), and predict_rank_at of max and attention ('exact3_count'), each against 'dense+rank'.
Results, with the card's name and power limit, go to DIR/bench_tastes_euclid.json."""
import argparse
import json
import os
import sys
import time

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.bench_euclidean import problem, timed  # noqa: E402
from scripts.bench_similar import card  # noqa: E402
from scripts.bench_tastes import weights_of  # noqa: E402

N_TASTES = 3
FLOORS = ('ATTENTION_MIN_ITEMS', 'EXACT_WIDE_MIN_ITEMS', 'RANK_AT_MIN_ITEMS', 'RANK_AT_EUCLID_ATTENTION_MIN_ITEMS')


def model_of(attention, d, wu, wi, bu, bi):
    from tensorrec_b200 import TensorRec, prediction_graphs as P, representation_graphs as R
    wus, was = weights_of(wu)
    model = TensorRec(n_components=d, n_tastes=N_TASTES, prediction_graph=P.EuclideanSimilarityPredictionGraph(),
                      attention_graph=R.LinearRepresentationGraph() if attention else None)
    w = {'linear_weights_item': wi, 'feature_biases_user': bu[:, None], 'feature_biases_item': bi[:, None]}
    for t in range(N_TASTES):
        w['linear_weights_user_%d' % t] = wus[t]
        if attention:
            w['linear_weights_attn_%d' % t] = was[t]
    model.set_weights(w)
    return model


def forced(T, floor, fn):
    """fn() with every route floor set to `floor` (0: the fused routes, 10**12: dense+rank)."""
    old = {name: getattr(T.tensorrec, name) for name in FLOORS}
    for name in FLOORS:
        setattr(T.tensorrec, name, floor)
    try:
        return fn()
    finally:
        for name, v in old.items():
            setattr(T.tensorrec, name, v)


def oracle_rows(uf, itf, wu, wi, bu, bi, rows, k, chunk=64):
    """The reference's top-k (Euclidean prediction per taste and attention row, the attention collapse,
    bias_prediction_dense) of the user rows `rows`."""
    from oracle import reference_ops as R
    F32 = np.float32
    wus, was = weights_of(wu)
    item_repr = R.sparse_dense_matmul_fast(itf, wi)
    r_item = np.sum(item_repr ** 2, axis=1, keepdims=True, dtype=F32).T     # (R.euclidean_dense's, formed once)
    ib = np.asarray(itf.astype(np.float32) @ bi, dtype=np.float32)

    def euclidean_dense(u):   # R.euclidean_dense(u, item_repr), operation for operation
        r_user = np.sum(u ** 2, axis=1, keepdims=True, dtype=F32)
        distance = np.maximum((r_user - F32(2.0) * np.matmul(u, item_repr.T) + r_item).astype(F32), F32(1e-16))
        return (F32(-1.0) * np.sqrt(distance)).astype(F32)

    ids, vals = [], []
    for c0 in range(0, len(rows), chunk):
        sub = uf[rows[c0:c0 + chunk]]
        preds = [euclidean_dense(R.sparse_dense_matmul_fast(sub, w)) for w in wus]
        atts = [euclidean_dense(R.sparse_dense_matmul_fast(sub, w)) for w in was]
        s = R.bias_prediction_dense(R.collapse_mixture_of_tastes(preds, atts),
                                    np.asarray(sub.astype(np.float32) @ bu, dtype=np.float32), ib)
        i, v = R.top_k_from_scores_fast(s, k)
        ids.append(i)
        vals.append(v)
    return np.concatenate(ids), np.concatenate(vals)


def run_dense(args, T, out):
    import torch
    from tensorrec_b200.input_utils import SparseInput
    U, I, d, block = 65536, 100000, 64, 4096
    uf, itf, wu, wi, bu, bi = problem(U, I, d)
    user_in, item_in = SparseInput(uf), SparseInput(itf)
    blocks = [SparseInput(sp.csr_matrix(uf[u0:u0 + block])) for u0 in range(0, U, block)]
    dev = torch.device('cuda', torch.cuda.current_device())
    buf = torch.empty((U, I), dtype=torch.float32, device=dev)
    res = {}
    for kind in ('max', 'attention'):
        model = model_of(kind == 'attention', d, wu, wi, bu, bi)
        assert model._tensor_score_form() == 'tastes_euclid'
        res[kind + '_tensor'] = timed(lambda: model._score_plan(item_in, dev)(user_in, out=buf), args.reps)
        T.tensorrec.SCORE_PATH = 'exact'
        try:
            if kind == 'max':        # the fp32 CUDA-core kernel takes all users at once
                r = timed(lambda: model._score_plan(item_in, dev)(user_in, out=buf), args.reps)
            else:                    # the torch collapse, in blocks of 4096 users
                def run():
                    score = model._score_plan(item_in, dev)
                    for b, blk in enumerate(blocks):
                        score(blk, out=buf[b * block:(b + 1) * block])
                r = timed(run, args.reps)
                r['blocks_of_users'] = block
        finally:
            T.tensorrec.SCORE_PATH = 'auto'
        res[kind + '_exact'] = r
        res[kind + '_speedup'] = r['ms_median'] / res[kind + '_tensor']['ms_median']
        print('dense', kind, json.dumps({k: v for k, v in res.items() if k.startswith(kind)}), file=sys.stderr,
              flush=True)
        del model
    out['dense'] = {'workload': 'scores of %d users x %d items x d%d, %d Euclidean tastes, into a resident device '
                                'matrix, biased' % (U, I, d, N_TASTES), 'results': res}
    del buf
    torch.cuda.empty_cache()


def run_flagship(args, T, out):
    import torch
    n, d = args.flagship_size, 128
    uf, itf, wu, wi, bu, bi = out['_problem'] = problem(n, n, d)
    res = {'workload': '%d users x %d items x d%d, %d Euclidean tastes with attention, biased' % (n, n, d, N_TASTES)}
    model = model_of(True, d, wu, wi, bu, bi)
    box = {}
    for k in args.flagship_k:
        route = 'exact3' if k <= 32 else 'exact3_wide'

        def fused():
            box[k] = model.predict_top_k(uf, itf, k, to_host=False)
        r = timed(fused, args.reps)
        r['path'] = model.last_topk_info['path']
        assert r['path'] == route
        res['%s_k%d' % (route, k)] = r
        print('flagship', route, k, json.dumps(r), file=sys.stderr, flush=True)
        if k == 10:
            sample = np.sort(np.random.default_rng(11).choice(n, min(args.check_rows, n), replace=False))
            got_i = box[k].items.cpu().numpy()[sample]
            got_s = box[k].scores.cpu().numpy()[sample]
        del box[k]
        torch.cuda.empty_cache()
        few = uf[:4096]
        dr = forced(T, 10 ** 12, lambda: timed(lambda: model.predict_top_k(few, itf, k, to_host=False), args.reps))
        dr['path'] = model.last_topk_info['path']
        dr['users'] = 4096
        dr['extrapolated_s_for_all_users'] = dr['ms_median'] * n / 4096 / 1e3
        res['dense_rank_k%d_4096_users' % k] = dr
        print('flagship dense+rank', k, json.dumps(dr), file=sys.stderr, flush=True)
    if 10 not in args.flagship_k:
        out['flagship'] = res
        return
    exp_i, exp_s = oracle_rows(uf, itf, wu, wi, bu, bi, sample, 10)
    same = got_i == exp_i
    res['exact3_k10']['oracle_check'] = {
        'rows': int(len(sample)), 'rows_differing': int((~same).any(axis=1).sum()),
        'slots_differing': int((~same).sum()),
        'max_abs_score_diff_where_ids_equal': float(np.max(np.abs(got_s - exp_s)[same])),
        # a differing slot where the two lists' scores there differ by a few ulps is a near-tie, not an error
        'max_abs_score_diff_where_ids_differ': float(np.max(np.abs(got_s - exp_s)[~same])) if (~same).any() else 0.0}
    print('flagship oracle', json.dumps(res['exact3_k10']['oracle_check']), file=sys.stderr, flush=True)
    out['flagship'] = res
    del model
    torch.cuda.empty_cache()


def block_check(model, uf, itf, ranks, n_users):
    """Ranks of the first n_users users (whole user blocks) against trk_rank_full of their dense scores."""
    import torch
    from tensorrec_b200 import kernels
    from tensorrec_b200.input_utils import SparseInput
    score = model._score_plan(SparseInput(sp.csr_matrix(itf)), torch.device('cuda'))
    full = kernels.rank_full(score(SparseInput(sp.csr_matrix(uf[:n_users]))))
    sub = ranks[:n_users].tocoo()
    want = full[torch.from_numpy(sub.row).long().cuda(), torch.from_numpy(sub.col).long().cuda()].cpu().numpy()
    return {'users': n_users, 'pairs': int(sub.nnz), 'pairs_differing': int(np.sum(want != sub.data))}


def run_rank_at(args, T, out):
    import torch
    from tensorrec_b200 import kernels
    n, d = args.flagship_size, 128
    uf, itf, wu, wi, bu, bi = out['_problem'] if '_problem' in out else problem(n, n, d)
    res = {'workload': '%d users x %d items x d%d, %d Euclidean tastes, leave-one-out (one uniformly random item per '
                       'user), biased' % (n, n, d, N_TASTES)}
    for kind in args.rank_at_forms.split(','):
        model = model_of(kind == 'attention', d, wu, wi, bu, bi)
        pairs = random_pairs(n, n)
        box = {}

        def run():
            box['ranks'] = model.predict_rank_at(uf, itf, pairs)
        r = timed(run, args.reps)
        r.update(model.last_rank_info)
        r['block_check'] = block_check(model, uf, itf, box['ranks'], 8 * kernels.tastes_plan(N_TASTES, kind != 'max')[1])
        res[kind] = r
        print('rank_at', kind, json.dumps(r), file=sys.stderr, flush=True)
        del model, box
        torch.cuda.empty_cache()
    out['rank_at'] = res


def run_crossover(args, T, out):
    import torch
    U, d = 65536, 128
    table = []
    for I in (1024, 2048, 4096, 16384, 65536):
        uf, itf, wu, wi, bu, bi = problem(U, I, d)
        row = {'items': I}
        attention = model_of(True, d, wu, wi, bu, bi)
        for k, route in ((10, 'exact3'), (100, 'exact3_wide')):
            for r_name, floor in ((route, 0), ('dense+rank', 10 ** 12)):
                t = forced(T, floor, lambda: timed(lambda: attention.predict_top_k(uf, itf, k, to_host=False),
                                                   args.reps))
                assert attention.last_topk_info['path'] == r_name
                row['attention_k%d_%s' % (k, r_name)] = t['ms_median']
        pairs = random_pairs(U, I)
        for kind, model in (('max', model_of(False, d, wu, wi, bu, bi)), ('attention', attention)):
            for r_name, floor in (('exact3_count', 0), ('dense+rank', 10 ** 12)):
                t = forced(T, floor, lambda: timed(lambda: model.predict_rank_at(uf, itf, pairs), args.reps))
                assert model.last_rank_info['path'] == r_name
                row['rank_at_%s_%s' % (kind, r_name)] = t['ms_median']
        table.append(row)
        print('crossover', json.dumps(row), file=sys.stderr, flush=True)
        del attention, model
        torch.cuda.empty_cache()
    out['crossover'] = {'workload': '%d users, d%d, %d Euclidean tastes, biased; median ms' % (U, d, N_TASTES),
                        'table': table}


def random_pairs(n_users, n_items, seed=2):
    """One uniformly random pair per user."""
    cols = np.random.default_rng(seed).integers(0, n_items, n_users)
    return sp.csr_matrix((np.ones(n_users, np.float32), cols, np.arange(n_users + 1)), shape=(n_users, n_items))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--parts', default='dense,flagship,rank_at,crossover')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--check-rows', type=int, default=4096)
    ap.add_argument('--flagship-size', type=int, default=1000000)
    ap.add_argument('--rank-at-forms', default='max,attention')
    ap.add_argument('--flagship-k', type=lambda v: [int(x) for x in v.split(',')], default=[10, 100])
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    import tensorrec_b200 as T
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    out = {'card': card(), 'floors': {name: getattr(T.tensorrec, name) for name in FLOORS}}
    parts = {'dense': run_dense, 'flagship': run_flagship, 'rank_at': run_rank_at, 'crossover': run_crossover}
    for part in args.parts.split(','):
        parts[part](args, T, out)
        with open(os.path.join(args.out, 'bench_tastes_euclid.json'), 'w') as f:   # after every part
            json.dump({k: v for k, v in out.items() if not k.startswith('_')}, f, indent=1)
    print(json.dumps({k: v for k, v in out.items() if not k.startswith('_')}))


if __name__ == '__main__':
    main()
