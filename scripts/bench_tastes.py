"""Mixture-of-tastes and attention models on the tensor-core kernels, on one GPU.

    python scripts/bench_tastes.py --out DIR [--parts crossover,dense,flagship --reps R --check-rows R]

Inputs are bench.py's flagship problem (indicator features, normal L2-normalised weights, 0.1-normal biases) with a
biased dot-product model of three tastes; the user weights of taste t are bench.py's user weights rolled by t rows, the
attention weights of taste t are rolled by 7 + t rows.  Every timing is one warm-up pass, then R timed passes (median
and range); a pass is one call ended by a device synchronisation.
  dense      predict()'s scoring into a resident [65536, 100000] matrix at d64, with and without attention: tensor
             cores against the CUDA-core kernel (SCORE_PATH=exact), alternated.  Also the taste-collapsing kernel alone
             (CUDA events, operands prepared) with its algorithmic rate 2 U I d n_ops and its issued rate (x3 passes).
  flagship   the attention model at 1M users x 1M items x d128, k = 10: predict_top_k(..., to_host=False) on 'exact3',
             sampled rows against the CPU oracle; 'dense+rank' over 4096 users (ATTENTION_MIN_ITEMS forced above
             n_items), extrapolated to 1M users.
  crossover  the attention model, 65536 users, k = 10, items in {1K, 2K, 4K, 16K, 64K}: 'exact3' and 'dense+rank'
             forced in turn.
Results, with the card's name and power limit, go to DIR/bench_tastes.json."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.bench_euclidean import problem, timed  # noqa: E402
from scripts.bench_similar import card  # noqa: E402

N_TASTES = 3


def weights_of(wu):
    return [np.roll(wu, t, axis=0) for t in range(N_TASTES)], [np.roll(wu, 7 + t, axis=0) for t in range(N_TASTES)]


def model_of(attention, d, wu, wi, bu, bi):
    from tensorrec_b200 import TensorRec, representation_graphs as R
    wus, was = weights_of(wu)
    model = TensorRec(n_components=d, n_tastes=N_TASTES,
                      attention_graph=R.LinearRepresentationGraph() if attention else None)
    w = {'linear_weights_item': wi, 'feature_biases_user': bu[:, None], 'feature_biases_item': bi[:, None]}
    for t in range(N_TASTES):
        w['linear_weights_user_%d' % t] = wus[t]
        if attention:
            w['linear_weights_attn_%d' % t] = was[t]
    model.set_weights(w)
    return model


def oracle_rows(uf, itf, wu, wi, bu, bi, rows, k, chunk=64):
    """The reference's top-k (tastes, attention collapse, bias_prediction_dense) of the user rows `rows`."""
    from oracle import reference_ops as R
    wus, was = weights_of(wu)
    item_repr = R.sparse_dense_matmul_fast(itf, wi)
    ib = np.asarray(itf.astype(np.float32) @ bi, dtype=np.float32)
    ids, vals = [], []
    for c0 in range(0, len(rows), chunk):
        sub = uf[rows[c0:c0 + chunk]]
        preds = [R.sparse_dense_matmul_fast(sub, w) @ item_repr.T for w in wus]
        atts = [R.sparse_dense_matmul_fast(sub, w) @ item_repr.T for w in was]
        s = R.bias_prediction_dense(R.collapse_mixture_of_tastes(preds, atts),
                                    np.asarray(sub.astype(np.float32) @ bu, dtype=np.float32), ib)
        i, v = R.top_k_from_scores_fast(s, k)
        ids.append(i)
        vals.append(v)
    return np.concatenate(ids), np.concatenate(vals)


def run_dense(args, T, out):
    import torch
    from tensorrec_b200 import kernels
    from tensorrec_b200.input_utils import SparseInput
    U, I, d = 65536, 100000, 64
    uf, itf, wu, wi, bu, bi = problem(U, I, d)
    user_in, item_in = SparseInput(uf), SparseInput(itf)
    dev = torch.device('cuda', torch.cuda.current_device())
    buf = torch.empty((U, I), dtype=torch.float32, device=dev)
    models = {'%s_%s' % (kind, path): (model_of(kind == 'attention', d, wu, wi, bu, bi), path)
              for kind in ('max', 'attention') for path in ('tensor', 'exact')}

    def run(name):
        model, path = models[name]
        old = T.tensorrec.SCORE_PATH
        T.tensorrec.SCORE_PATH = 'exact' if path == 'exact' else 'auto'
        try:
            model._score_plan(item_in, dev)(user_in, out=buf)
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
    res = {name: {'ms': v, 'ms_median': float(np.median(v)), 'ms_range': [min(v), max(v)]} for name, v in ms.items()}
    # the kernel alone: CUDA events around trk_score_dense_tastes_f16x3 with the operands prepared
    for kind in ('max', 'attention'):
        model = models[kind + '_tensor'][0]
        attention = kind == 'attention'
        users = model._taste_operands(user_in, dev)
        items = model._side_operands('item', item_in, dev)
        meta = kernels.pack_item_meta(items.scale, items.bias, I)
        launch = lambda: kernels.score_dense_tastes(users, items.split, meta, I, N_TASTES, attention, out=buf)  # noqa
        launch()
        kms = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            launch()
            e1.record()
            e1.synchronize()
            kms.append(e0.elapsed_time(e1))
        n_ops = kernels.tastes_n_ops(N_TASTES, attention)
        kmed = float(np.median(kms))
        flops = 2.0 * U * I * d * n_ops
        res[kind + '_kernel'] = {'ms': kms, 'ms_median': kmed, 'ms_range': [min(kms), max(kms)], 'n_ops': n_ops,
                                 'algorithmic_tflops': flops / kmed / 1e9, 'issued_tflops': 3 * flops / kmed / 1e9}
        del users
    out['dense'] = {'workload': 'scores of %d users x %d items x d%d, %d tastes, into a resident device matrix, biased'
                    % (U, I, d, N_TASTES), 'results': res}
    print('dense', json.dumps(out['dense']), file=sys.stderr, flush=True)
    del buf
    torch.cuda.empty_cache()


def run_flagship(args, T, out):
    import torch
    n, d, k = args.flagship_size, 128, 10
    uf, itf, wu, wi, bu, bi = problem(n, n, d)
    res = {'workload': '%d users x %d items x d%d, %d tastes with attention, k=%d, biased' % (n, n, d, N_TASTES, k)}
    model = model_of(True, d, wu, wi, bu, bi)
    box = {}

    def fused():
        box['top'] = model.predict_top_k(uf, itf, k, to_host=False)
    res['exact3'] = timed(fused, args.reps)
    res['exact3']['path'] = model.last_topk_info['path']
    sample = np.sort(np.random.default_rng(11).choice(n, min(args.check_rows, n), replace=False))
    got_i = box['top'].items.cpu().numpy()[sample]
    got_s = box['top'].scores.cpu().numpy()[sample]
    del box['top']
    torch.cuda.empty_cache()
    print('flagship exact3', json.dumps(res['exact3']), file=sys.stderr, flush=True)
    exp_i, exp_s = oracle_rows(uf, itf, wu, wi, bu, bi, sample, k)
    same = got_i == exp_i
    res['exact3']['oracle_check'] = {'rows': int(len(sample)), 'rows_differing': int((~same).any(axis=1).sum()),
                                     'slots_differing': int((~same).sum()),
                                     'max_abs_score_diff_where_ids_equal': float(np.max(np.abs(got_s - exp_s)[same]))}
    print('flagship oracle', json.dumps(res['exact3']['oracle_check']), file=sys.stderr, flush=True)

    few = uf[:4096]
    floor = T.tensorrec.ATTENTION_MIN_ITEMS
    T.tensorrec.ATTENTION_MIN_ITEMS = 10 ** 12
    dr = timed(lambda: model.predict_top_k(few, itf, k, to_host=False), args.reps)
    dr['path'] = model.last_topk_info['path']
    T.tensorrec.ATTENTION_MIN_ITEMS = floor
    dr['users'] = 4096
    dr['extrapolated_s_for_all_users'] = dr['ms_median'] * n / 4096 / 1e3
    res['dense_rank_4096_users'] = dr
    print('flagship dense+rank', json.dumps(dr), file=sys.stderr, flush=True)
    out['flagship'] = res
    del model
    torch.cuda.empty_cache()


def run_crossover(args, T, out):
    import torch
    U, d, k = 65536, 128, 10
    table = []
    for I in (1024, 2048, 4096, 16384, 65536):
        uf, itf, wu, wi, bu, bi = problem(U, I, d)
        model = model_of(True, d, wu, wi, bu, bi)
        row = {'items': I}
        floor = T.tensorrec.ATTENTION_MIN_ITEMS
        for route, f in (('exact3', 0), ('dense+rank', 10 ** 12)):
            T.tensorrec.ATTENTION_MIN_ITEMS = f
            r = timed(lambda: model.predict_top_k(uf, itf, k, to_host=False), args.reps)
            assert model.last_topk_info['path'] == route
            row[route] = r
        T.tensorrec.ATTENTION_MIN_ITEMS = floor
        table.append(row)
        print('crossover', json.dumps(row), file=sys.stderr, flush=True)
        del model
        torch.cuda.empty_cache()
    out['crossover'] = {'workload': '%d users, d%d, %d tastes with attention, k=%d, biased' % (U, d, N_TASTES, k),
                        'table': table}


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
    out = {'card': card(), 'ATTENTION_MIN_ITEMS': T.tensorrec.ATTENTION_MIN_ITEMS}
    parts = {'flagship': run_flagship, 'dense': run_dense, 'crossover': run_crossover}
    for part in args.parts.split(','):
        parts[part](args, T, out)
        with open(os.path.join(args.out, 'bench_tastes.json'), 'w') as f:   # after every part: partial results
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
