"""The catalogue-wide "related items" table: predict_similar_items_top_k over every item (1M items x d128, n_similar = 10,
exclude_self=True) on one GPU, for dot, cosine and Euclidean similarity.

    python scripts/bench_similar.py --out DIR [--items N --d D --n N --reps R --check-rows R]

Items are the flagship item side of bench.py (indicator features, normal L2-normalised weights).  Per similarity: one
warm-up pass, then R timed passes; a pass is one predict_similar_items_top_k(..., to_host=False) call ended by a device
synchronisation.  The route, the rows the certificate sent to the device-side fallback and sampled rows checked against
the CPU oracle (no biases, own id excluded) are recorded.  Results, with the card's name and power limit, go to
DIR/bench_similar.json."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [f.strip() for f in out.split(',')]
        return {'name': name, 'power_limit': power}
    except Exception as e:   # noqa: BLE001
        return {'name': None, 'power_limit': None, 'error': str(e)}


def oracle_scores(prediction, item_repr, item_repr_unit, q):
    """The reference's similar-items scores of the query ids q against every item."""
    from oracle import reference_ops as R
    if prediction == 'euclidean':
        return R.euclidean_dense(item_repr[q], item_repr)
    r = item_repr_unit if prediction == 'cosine' else item_repr    # cosine: R.cosine_dense, normalisation done once
    return R.dot_product_dense(r[q], r)


def oracle_rows(prediction, item_repr, item_repr_unit, rows, n, chunk=128):
    """The reference's similar-items top-n of the query ids `rows` with their own id excluded (ids, scores)."""
    from oracle import reference_ops as R
    ids, vals = [], []
    for c0 in range(0, len(rows), chunk):
        q = rows[c0:c0 + chunk]
        s = oracle_scores(prediction, item_repr, item_repr_unit, q)
        s[np.arange(len(q)), q] = -np.inf
        i, v = R.top_k_from_scores_fast(s, n)
        ids.append(i)
        vals.append(v)
    return np.concatenate(ids), np.concatenate(vals)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--items', type=int, default=1000000)
    ap.add_argument('--d', type=int, default=128)
    ap.add_argument('--n', type=int, default=10)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--check-rows', type=int, default=4096)
    ap.add_argument('--predictions', default='dot,cosine,euclidean')
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    info = {'workload': '%d items x d%d, item_ids=None, n_similar=%d, exclude_self=True'
                        % (args.items, args.d, args.n), 'card': card()}

    import torch
    from tensorrec_b200 import TensorRec, kernels, prediction_graphs as P
    from oracle import reference_ops as R
    kernels.require_cuda()
    itf = bench.indicator_csr(args.items, seed=1)
    wi = bench.make_weights(itf.shape[1], args.d, seed=3)
    item_repr = R.sparse_dense_matmul_fast(itf, wi)
    item_repr_unit = R.l2_normalize(item_repr)
    sample = np.sort(np.random.default_rng(11).choice(args.items, min(args.check_rows, args.items), replace=False))
    graphs = {'dot': P.DotProductPredictionGraph, 'cosine': P.CosineSimilarityPredictionGraph,
              'euclidean': P.EuclideanSimilarityPredictionGraph}
    results = {}
    for prediction in args.predictions.split(','):
        model = TensorRec(n_components=args.d, prediction_graph=graphs[prediction]())
        model.set_weights({'linear_weights_item': wi})

        def run():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            top = model.predict_similar_items_top_k(itf, args.n, exclude_self=True, to_host=False)
            torch.cuda.synchronize()
            return top, 1e3 * (time.perf_counter() - t0), dict(model.last_topk_info)

        run()                                                    # warm-up
        ms, fallback, top, tinfo = [], [], None, None
        for _ in range(args.reps):
            top, t, tinfo = run()
            ms.append(t)
            fallback.append(int(tinfo['fallback_rows']))
        got_i = top.items.cpu().numpy()[sample]
        got_s = top.scores.cpu().numpy()[sample]
        del top
        torch.cuda.empty_cache()
        exp_i, exp_s = oracle_rows(prediction, item_repr, item_repr_unit, sample, args.n)
        differ = (got_i != exp_i).any(axis=1)
        detail = []
        for j in np.nonzero(differ)[0][:8]:     # what differs: the oracle's scores of the kernel's items, and its own
            s = oracle_scores(prediction, item_repr, item_repr_unit, sample[j:j + 1])[0]
            detail.append({'row': int(sample[j]), 'items': got_i[j].tolist(), 'scores': got_s[j].tolist(),
                           'oracle_scores_of_items': [float(s[i]) for i in got_i[j]],
                           'oracle_items': exp_i[j].tolist(), 'oracle_scores': exp_s[j].tolist()})
        results[prediction] = {
            'path': tinfo['path'], 'ms': ms, 'ms_median': float(np.median(ms)), 'ms_range': [min(ms), max(ms)],
            'fallback_rows': fallback, 'overflow_blocks': int(tinfo.get('overflow_blocks', 0)),
            'oracle_check': {'rows': int(len(sample)), 'rows_differing': int(differ.sum()),
                             'slots_differing': int((got_i != exp_i).sum()),
                             'self_reported': int((got_i == sample[:, None]).sum()), 'differing': detail,
                             'max_abs_score_diff_same_ids': float(np.max(np.abs(got_s - exp_s)[got_i == exp_i]))
                             if (got_i == exp_i).any() else None}}
        print(prediction, json.dumps(results[prediction]), file=sys.stderr, flush=True)
        del model
        torch.cuda.empty_cache()
    info['results'] = results
    with open(os.path.join(args.out, 'bench_similar.json'), 'w') as f:
        json.dump(info, f, indent=1)
    print(json.dumps(info))


if __name__ == '__main__':
    main()
