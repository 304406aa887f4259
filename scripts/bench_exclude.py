"""Cost of exclude= on the flagship top-k workload (1M users x 1M items x d128, k = 10, one GPU).

    python scripts/bench_exclude.py --out DIR [--users N --items N --d D --k K --reps R]

Four configurations, alternated in one process (R timed passes each after one warm-up pass):
  none         exclude=None (the code path without exclusion);
  empty        an exclude matrix without entries (must be bit-identical to none);
  history      heavy-tailed per-user counts (Pareto, mean ~30, cap 10 000), skewed toward high-bias items;
  adversarial  every user's own unmasked top-k (the threshold has to go deeper than without exclusion).
A pass is one predict_top_k(..., to_host=False) call ended by a device synchronisation.  The preparation of the lists
(host CSR + upload + the position sort of the filter) is timed on its own as well.  Sampled rows are checked against
the masked oracle on the CPU.  Results, with the card's name and power limit, go to DIR/bench_exclude.json."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp

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


def history_exclusion(n_users, item_bias, rng, mean=30.0, cap=10000):
    """Per-user counts (Pareto(1.5) + 1) * 10 (mean 30) capped at `cap`; items drawn from the bias-descending order at
    position floor(n_items * u^3): heavily skewed toward high-bias items.  Duplicates are summed by the API."""
    n_items = item_bias.shape[0]
    counts = np.minimum(cap, ((rng.pareto(1.5, n_users) + 1.0) * (mean / 3.0)).astype(np.int64))
    order = np.argsort(-item_bias, kind='stable')
    rows = np.repeat(np.arange(n_users, dtype=np.int64), counts)
    cols = order[np.minimum(n_items - 1, (n_items * rng.random(rows.shape[0]) ** 3).astype(np.int64))]
    m = sp.csr_matrix((np.ones(rows.shape[0], np.float32), (rows, cols)), shape=(n_users, n_items))
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--users', type=int, default=1000000)
    ap.add_argument('--items', type=int, default=1000000)
    ap.add_argument('--d', type=int, default=128)
    ap.add_argument('--k', type=int, default=10)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--check-rows', type=int, default=4096)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    info = {'workload': '%d users x %d items x d%d, k=%d' % (args.users, args.items, args.d, args.k), 'card': card()}

    import torch
    from tensorrec_b200 import TensorRec, kernels
    kernels.require_cuda()
    uf, itf, wu, wi, bu, bi = bench.make_problem(argparse.Namespace(users=args.users, items=args.items, d=args.d,
                                                                    scores='iid'))
    model = TensorRec(n_components=args.d)
    model.set_weights({'linear_weights_user_0': wu, 'linear_weights_item': wi, 'feature_biases_user': bu[:, None],
                       'feature_biases_item': bi[:, None]})
    rng = np.random.default_rng(7)
    item_bias = np.asarray(itf @ bi, dtype=np.float32)

    def run(exclude):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        top = model.predict_top_k(uf, itf, args.k, to_host=False,
                                  **({} if exclude is None else {'exclude': exclude}))
        torch.cuda.synchronize()
        return top, 1e3 * (time.perf_counter() - t0), dict(model.last_topk_info)

    base, _, _ = run(None)                                       # warm-up, and the rows the adversary excludes
    base_items = base.items.cpu().numpy()
    rows = np.repeat(np.arange(args.users), args.k)
    configs = {
        'none': None,
        'empty': sp.csr_matrix((args.users, args.items), dtype=np.float32),
        'history': history_exclusion(args.users, item_bias, rng),
        'adversarial': sp.csr_matrix((np.ones(rows.shape[0], np.float32), (rows, base_items.reshape(-1))),
                                     shape=(args.users, args.items)),
    }
    info['nnz'] = {name: (0 if m is None else int(m.nnz)) for name, m in configs.items()}
    results = {name: {'ms': [], 'prep_ms': [], 'fallback_rows': []} for name in configs}
    outputs = {}
    for name, m in configs.items():                              # warm-up of every configuration
        run(m)
    for rep in range(args.reps):
        for name, m in configs.items():
            top, ms, tinfo = run(m)
            results[name]['ms'].append(ms)
            results[name]['fallback_rows'].append(int(tinfo['fallback_rows']))
            outputs[name] = top
            if m is not None:                                    # the list preparation on its own
                fitems = kernels.FilterItems(model._side_operands('item', model._single_input(itf, 'item'),
                                                                  torch.device('cuda'), for_filter=True))
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                host = kernels.exclusion_host_csr(m, 0, args.items)
                excl = kernels.DeviceExclusion.upload(*host, device=torch.device('cuda'))
                kernels.exclusion_positions(excl, fitems.perm, args.items)
                torch.cuda.synchronize()
                results[name]['prep_ms'].append(1e3 * (time.perf_counter() - t0))
                del fitems, excl
    for name, r in results.items():
        for key in ('ms', 'prep_ms'):
            v = r[key]
            if v:
                r[key + '_median'] = float(np.median(v))
                r[key + '_spread'] = [float(min(v)), float(max(v))]
    none_i, none_s = outputs['none'].items.cpu().numpy(), outputs['none'].scores.cpu().numpy()
    emp_i, emp_s = outputs['empty'].items.cpu().numpy(), outputs['empty'].scores.cpu().numpy()
    info['empty_bit_identical_to_none'] = bool(np.array_equal(none_i, emp_i) and np.array_equal(none_s, emp_s))

    # masked oracle on sampled rows (continuous scores: the ids must agree, the scores to the fp32 tolerance)
    from oracle import reference_ops as R
    sample = np.sort(np.random.default_rng(11).choice(args.users, min(args.check_rows, args.users), replace=False))
    item_repr = R.sparse_dense_matmul_fast(itf, wi)
    checks = {}
    for name in ('history', 'adversarial'):
        got_i = outputs[name].items.cpu().numpy()[sample]
        got_s = outputs[name].scores.cpu().numpy()[sample]
        mism, detail = 0, []
        for c0 in range(0, len(sample), 512):
            sub_rows = sample[c0:c0 + 512]
            sub = uf[sub_rows]
            scores = R.bias_prediction_dense(R.dot_product_dense(R.sparse_dense_matmul_fast(sub, wu), item_repr),
                                             np.asarray(sub @ bu, dtype=np.float32), item_bias)
            ex = configs[name][sub_rows].tocoo()
            scores[ex.row[ex.data != 0], ex.col[ex.data != 0]] = -np.inf     # every row keeps >= k eligible items
            exp_i, exp_s = R.top_k_from_scores_fast(scores, args.k)
            differ = np.nonzero((got_i[c0:c0 + 512] != exp_i).any(axis=1))[0]
            mism += int(differ.shape[0])
            for j in differ[:8]:     # what differs: the kernel's items with its and the oracle's scores, and the oracle's
                g = got_i[c0 + j]
                detail.append({'row': int(sub_rows[j]), 'items': g.tolist(), 'scores': got_s[c0 + j].tolist(),
                               'oracle_scores_of_items': [float(scores[j, i]) if 0 <= i < scores.shape[1] else None
                                                          for i in g],
                               'oracle_items': exp_i[j].tolist(), 'oracle_scores': exp_s[j].tolist()})
        checks[name] = {'rows': int(len(sample)), 'rows_differing': mism, 'differing': detail}
    info['oracle_check'] = checks
    info['results'] = results
    with open(os.path.join(args.out, 'bench_exclude.json'), 'w') as f:
        json.dump(info, f, indent=1)
    print(json.dumps(info))


if __name__ == '__main__':
    main()
