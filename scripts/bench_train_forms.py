"""Times the fused training step (tensorrec_b200/train_kernels.py) for each model form it trains, on bench.py's training
workload (LinearRepr features, 1M users x 1M items, d = 128, n_sampled_items = 64, 4 positives per user and one negative
in four users), with WmrbStep's phase split and the ratio to the dot step of the same run; then, at a size the torch
path finishes, the kernel path against the torch-autograd path (fit_partial, one epoch) for the same forms.

    python scripts/bench_train_forms.py [--users N] [--items N] [--steps K] [--warmup W] [--small-users N]

Prints one JSON line per measurement and records the card name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import bench  # noqa: E402

PHASES = ['representations', 'sampler', 'wmrb_step', 'weight_gradients', 'adam']


def forms():
    from tensorrec_b200.prediction_graphs import CosineSimilarityPredictionGraph, EuclideanSimilarityPredictionGraph
    from tensorrec_b200.representation_graphs import LinearRepresentationGraph, NormalizedLinearRepresentationGraph
    return [('dot', {}),
            ('cosine', {'prediction_graph': CosineSimilarityPredictionGraph()}),
            ('euclidean', {'prediction_graph': EuclideanSimilarityPredictionGraph()}),
            ('normalized_linear_users', {'user_repr_graph': NormalizedLinearRepresentationGraph()}),
            ('3_tastes', {'n_tastes': 3}),
            ('3_tastes_attention', {'n_tastes': 3, 'attention_graph': LinearRepresentationGraph()})]


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def interactions_for(n_users, n_items, seed=5):
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(n_users, dtype=np.int64), 4)
    neg = np.arange(0, n_users, 4, dtype=np.int64)
    data = np.concatenate([np.ones(rows.shape[0], np.float32), -np.ones(neg.shape[0], np.float32)])
    return sp.csr_matrix((data, (np.concatenate([rows, neg]),
                                 np.concatenate([rng.integers(0, n_items, rows.shape[0]),
                                                 rng.integers(0, n_items, neg.shape[0])]))), shape=(n_users, n_items))


def weights_for(kw, uf, itf, d, wu, wi, bu, bi):
    rng = np.random.default_rng(9)
    w = {'linear_weights_item': wi, 'feature_biases_user': bu[:, None], 'feature_biases_item': bi[:, None]}
    for t in range(kw.get('n_tastes', 1)):
        w['linear_weights_user_%d' % t] = wu if t == 0 else bench.make_weights(uf.shape[1], d, seed=20 + t)
        if kw.get('attention_graph') is not None:
            w['linear_weights_attn_%d' % t] = (0.1 * rng.standard_normal((uf.shape[1], d))).astype(np.float32)
    return w


def kernel_path(args, dtype):
    import torch
    import tensorrec_b200
    from tensorrec_b200 import train_kernels
    from tensorrec_b200.input_utils import SparseInput
    ns = argparse.Namespace(users=args.users, items=args.items, d=args.d, scores='iid')
    uf, itf, wu, wi, bu, bi = bench.make_problem(ns)
    inter = interactions_for(args.users, args.items)
    int_in, uf_in, if_in = SparseInput(inter), SparseInput(uf), SparseInput(itf)
    dev = torch.device('cuda', 0)
    results, dot_ms = [], None
    for name, kw in forms():
        model = tensorrec_b200.TensorRec(n_components=args.d, loss_graph=tensorrec_b200.loss_graphs.WMRBLossGraph(), **kw)
        model.set_weights(weights_for(kw, uf, itf, args.d, wu, wi, bu, bi))
        stepper = train_kernels.WmrbStep(model, dev, seed=0, bf16=dtype == 'bf16')
        l2 = int_in.n_positive * 1e-5
        for _ in range(args.warmup):
            stepper.step(int_in, uf_in, if_in, args.n_sampled, 0.01, l2)
        torch.cuda.synchronize()
        stepper.marks = []
        for _ in range(args.steps):
            stepper.step(int_in, uf_in, if_in, args.n_sampled, 0.01, l2)
        torch.cuda.synchronize()
        marks, per = stepper.marks, len(PHASES) + 1
        phase = {p: sum(marks[s * per + j][1].elapsed_time(marks[s * per + j + 1][1]) for s in range(args.steps))
                 / args.steps for j, p in enumerate(PHASES)}
        ms = sum(marks[s * per][1].elapsed_time(marks[s * per + per - 1][1]) for s in range(args.steps)) / args.steps
        dot_ms = ms if name == 'dot' else dot_ms
        r = {'path': 'kernel', 'form': name, 'dtype': dtype, 'ms_per_step': round(ms, 3),
             'ratio_to_dot': round(ms / dot_ms, 3), 'phases_ms': {k: round(v, 3) for k, v in phase.items()},
             'workload': '%d users x %d items, d=%d, n_sampled=%d, %d interactions' % (
                 args.users, args.items, args.d, args.n_sampled, inter.nnz)}
        print(json.dumps(r), flush=True)
        results.append(r)
        del model, stepper
        torch.cuda.empty_cache()
    return results


def against_torch(args):
    import torch
    import tensorrec_b200
    from tensorrec_b200 import session_management as sm, train_kernels
    sm.set_session(None)
    ns = argparse.Namespace(users=args.small_users, items=args.small_items, d=args.d, scores='iid')
    uf, itf, wu, wi, bu, bi = bench.make_problem(ns)
    inter = interactions_for(args.small_users, args.small_items)
    results = []
    for name, kw in forms():
        times = {}
        for path in ('kernel', 'torch'):
            train_kernels.TRAIN_PATH = 'torch' if path == 'torch' else 'auto'
            model = tensorrec_b200.TensorRec(n_components=args.d, loss_graph=tensorrec_b200.loss_graphs.WMRBLossGraph(),
                                             **kw)
            model.set_weights(weights_for(kw, uf, itf, args.d, wu, wi, bu, bi))
            model.fit_partial(inter, uf, itf, epochs=1, n_sampled_items=args.n_sampled)       # warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model.fit_partial(inter, uf, itf, epochs=args.small_epochs, n_sampled_items=args.n_sampled)
            torch.cuda.synchronize()
            times[path] = (time.perf_counter() - t0) * 1e3 / args.small_epochs
            assert (getattr(model, '_wmrb_step', None) is not None) == (path == 'kernel'), (name, path)
        train_kernels.TRAIN_PATH = 'auto'
        r = {'path': 'kernel_vs_torch', 'form': name, 'kernel_ms_per_step': round(times['kernel'], 2),
             'torch_ms_per_step': round(times['torch'], 2), 'speedup': round(times['torch'] / times['kernel'], 1),
             'workload': '%d users x %d items, d=%d, n_sampled=%d, f32' % (args.small_users, args.small_items, args.d,
                                                                            args.n_sampled)}
        print(json.dumps(r), flush=True)
        results.append(r)
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--users', type=int, default=1000000)
    ap.add_argument('--items', type=int, default=1000000)
    ap.add_argument('--d', type=int, default=128)
    ap.add_argument('--n-sampled', type=int, default=64)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--small-users', type=int, default=4096)
    ap.add_argument('--small-items', type=int, default=8192)
    ap.add_argument('--small-epochs', type=int, default=3)
    ap.add_argument('--dtypes', default='bf16,f32', help='representation dtypes of the kernel-path table')
    ap.add_argument('--no-torch', action='store_true', help='skip the kernel path against torch path table')
    ap.add_argument('--out', default=None, help='also write every result line to this JSON file')
    args = ap.parse_args()
    import torch
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    torch.cuda.set_device(0)
    info = {'card': card()}
    print(json.dumps(info), flush=True)
    results = [info]
    for dtype in [t for t in args.dtypes.split(',') if t]:
        results += kernel_path(args, dtype)
    if not args.no_torch:
        results += against_torch(args)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(results, f, indent=1)


if __name__ == '__main__':
    main()
