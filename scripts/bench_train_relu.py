"""Times the fused training step of ReLURepresentationGraph models (DESIGN §3.14) on bench_train_forms.py's workload
(1M users x 1M items, d = 128): NormalizedLinear users x ReLU items (relu_size 512), dot / cosine / Euclidean, WMRB and
RMSE, one and three tastes, with WmrbStep's phase split, beside the Linear-item step of the same run; then the hidden
layer's kernels alone against an unfused torch version of the same layer (cuBLAS fp32, TF32 off), with achieved
TFLOP/s and bytes/s; then, at a size the torch path finishes, the kernel path against the torch-autograd path.

    python scripts/bench_train_relu.py [--users N] [--items N] [--steps K] [--warmup W] [--no-torch]

Prints one JSON line per measurement and records the card name and power limit read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bench  # noqa: E402
import bench_train_forms as forms_bench  # noqa: E402


def make_model(args, loss, prediction, n_tastes, relu):
    import tensorrec_b200
    from tensorrec_b200 import loss_graphs as L, prediction_graphs as P
    from tensorrec_b200.representation_graphs import (LinearRepresentationGraph, NormalizedLinearRepresentationGraph,
                                                      ReLURepresentationGraph)
    return tensorrec_b200.TensorRec(
        n_components=args.d, n_tastes=n_tastes, user_repr_graph=NormalizedLinearRepresentationGraph(),
        item_repr_graph=ReLURepresentationGraph(relu_size=args.hidden) if relu else LinearRepresentationGraph(),
        prediction_graph={'dot': P.DotProductPredictionGraph, 'cosine': P.CosineSimilarityPredictionGraph,
                          'euclidean': P.EuclideanSimilarityPredictionGraph}[prediction](),
        loss_graph={'wmrb': L.WMRBLossGraph, 'rmse': L.RMSELossGraph}[loss]())


def phase_split(marks):
    """ms per step of each phase (named by the mark that ends it) and of the whole step."""
    phases, steps, total = {}, 0, 0.0
    start = None
    for i, (name, ev) in enumerate(marks):
        if name == 'start':
            steps += 1
            start = ev
            continue
        phases[name] = phases.get(name, 0.0) + marks[i - 1][1].elapsed_time(ev)
        if i + 1 == len(marks) or marks[i + 1][0] == 'start':
            total += start.elapsed_time(ev)
    return {k: round(v / steps, 3) for k, v in phases.items()}, total / steps


def kernel_path(args):
    import torch
    from tensorrec_b200 import train_kernels
    from tensorrec_b200.input_utils import SparseInput
    ns = argparse.Namespace(users=args.users, items=args.items, d=args.d, scores='iid')
    uf, itf, wu, wi, bu, bi = bench.make_problem(ns)
    inter = forms_bench.interactions_for(args.users, args.items)
    int_in, uf_in, if_in = SparseInput(inter), SparseInput(uf), SparseInput(itf)
    dev = torch.device('cuda', 0)
    rng = np.random.default_rng(3)
    results = []
    runs = [(loss, pred, nt, relu) for loss in ('wmrb', 'rmse') for nt in (1, 3) for relu in (False, True)
            for pred in (('dot', 'cosine', 'euclidean') if relu else ('dot',))]
    for loss, pred, nt, relu in runs:
        model = make_model(args, loss, pred, nt, relu)
        w = {'feature_biases_user': bu[:, None], 'feature_biases_item': bi[:, None]}
        for t in range(nt):
            w['linear_weights_user_%d' % t] = wu if t == 0 else bench.make_weights(uf.shape[1], args.d, seed=20 + t)
        if relu:
            w['relu_weights_item'] = (0.5 * rng.standard_normal((itf.shape[1], args.hidden))).astype(np.float32)
            w['relu_biases_item'] = np.zeros((1, args.hidden), np.float32)
            w['linear_weights_item'] = (0.5 * rng.standard_normal((args.hidden, args.d))).astype(np.float32)
        else:
            w['linear_weights_item'] = wi
        model.set_weights(w, n_user_features=uf.shape[1], n_item_features=itf.shape[1])
        stepper = train_kernels.WmrbStep(model, dev, seed=0, bf16=False)
        serial = loss != 'wmrb'
        step_args = (int_in, uf_in, if_in, None if serial else args.n_sampled, 0.01,
                     1e-5 if serial else int_in.n_positive * 1e-5)
        for _ in range(args.warmup):
            stepper.step(*step_args)
        torch.cuda.synchronize()
        stepper.marks = []
        for _ in range(args.steps):
            stepper.step(*step_args)
        torch.cuda.synchronize()
        phases, ms = phase_split(stepper.marks)
        stepper.marks = None
        r = {'path': 'kernel', 'loss': loss, 'prediction': pred, 'n_tastes': nt,
             'item_graph': 'relu(%d)' % args.hidden if relu else 'linear', 'ms_per_step': round(ms, 3),
             'phases_ms': phases,
             'workload': '%d users x %d items (%d item features), d=%d, %d interactions, f32' % (
                 args.users, args.items, itf.shape[1], args.d, inter.nnz)}
        print(json.dumps(r), flush=True)
        results.append(r)
        del model, stepper
        torch.cuda.empty_cache()
    return results


def layer_alone(args):
    """The layer's kernels at rows = n_items against torch fp32 (cuBLAS, TF32 off), CUDA events over args.steps calls."""
    import torch
    from tensorrec_b200 import _lib
    from tensorrec_b200.kernels import _p, _stream
    torch.backends.cuda.matmul.allow_tf32 = False
    lib = _lib.load()
    n, h, d = args.items, args.hidden, args.d
    dev = torch.device('cuda', 0)
    g = torch.Generator(device=dev).manual_seed(0)
    pre = torch.randn((n, h), device=dev, generator=g)
    b = torch.randn((h,), device=dev, generator=g) * 0.1
    w2 = torch.randn((h, d), device=dev, generator=g) * 0.05
    d_out = torch.randn((n, d), device=dev, generator=g)
    out = torch.empty((n, d), device=dev)
    ws_bytes = int(lib.trk_relu_layer_workspace_bytes(n, h, d))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    db, dw2 = torch.empty((h,), device=dev), torch.empty((h, d), device=dev)
    scratch = pre.clone()

    def fwd():
        _lib.check(lib.trk_relu_layer_forward_f32(_p(pre), _p(b), _p(w2), n, h, d, _p(out), _stream()), 'fwd')

    def bwd():
        scratch.copy_(pre)     # the backward overwrites P; the copy is timed apart and subtracted
        _lib.check(lib.trk_relu_layer_backward_f32(_p(scratch), _p(b), _p(w2), _p(d_out), n, h, d, _p(db), _p(dw2),
                                                   _p(ws), ws_bytes, _stream()), 'bwd')

    def copy():
        scratch.copy_(pre)

    def torch_fwd():
        return torch.relu(pre + b) @ w2

    def torch_bwd():
        z = pre + b
        dz = (d_out @ w2.t()) * (z > 0)
        return dz, dz.sum(0), torch.relu(z).t() @ d_out

    def timed(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    t = {name: timed(fn) for name, fn in (('forward', fwd), ('backward_with_copy', bwd), ('copy', copy),
                                          ('torch_forward', torch_fwd), ('torch_backward', torch_bwd))}
    t['backward'] = t['backward_with_copy'] - t['copy']
    ref_out = torch_fwd()
    err = float((out - ref_out).abs().max())
    flops = {'forward': 2.0 * n * h * d, 'backward': 4.0 * n * h * d}
    nbytes = {'forward': 4.0 * (n * h + n * d), 'backward': 4.0 * (2 * n * h + n * d)}
    r = {'measure': 'relu_layer_alone', 'rows': n, 'hidden': h, 'd': d, 'max_abs_diff_forward_vs_torch_fp32': err}
    for k in ('forward', 'backward'):
        r[k] = {'ms': round(t[k], 3), 'tflops': round(3 * flops[k] / t[k] / 1e9, 1),
                'tflops_useful': round(flops[k] / t[k] / 1e9, 1), 'gbytes_per_s': round(nbytes[k] / t[k] / 1e6, 1),
                'torch_fp32_ms': round(t['torch_' + k], 3)}
    print(json.dumps(r), flush=True)
    return [r]


def against_torch(args):
    import torch
    from tensorrec_b200 import session_management as sm, train_kernels
    sm.set_session(None)
    ns = argparse.Namespace(users=args.small_users, items=args.small_items, d=args.d, scores='iid')
    uf, itf, _, _, _, _ = bench.make_problem(ns)
    inter = forms_bench.interactions_for(args.small_users, args.small_items)
    results = []
    for loss, pred in (('wmrb', 'dot'), ('rmse', 'dot')):
        times = {}
        for path in ('kernel', 'torch'):
            train_kernels.TRAIN_PATH = 'torch' if path == 'torch' else 'auto'
            model = make_model(args, loss, pred, 1, True)
            kw = {} if loss == 'rmse' else {'n_sampled_items': args.n_sampled}
            model.fit_partial(inter, uf, itf, epochs=1, **kw)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model.fit_partial(inter, uf, itf, epochs=args.small_epochs, **kw)
            torch.cuda.synchronize()
            times[path] = (time.perf_counter() - t0) * 1e3 / args.small_epochs
            assert (getattr(model, '_wmrb_step', None) is not None) == (path == 'kernel'), (loss, path)
        train_kernels.TRAIN_PATH = 'auto'
        r = {'path': 'kernel_vs_torch', 'loss': loss, 'prediction': pred, 'item_graph': 'relu(%d)' % args.hidden,
             'kernel_ms_per_step': round(times['kernel'], 2), 'torch_ms_per_step': round(times['torch'], 2),
             'speedup': round(times['torch'] / times['kernel'], 1),
             'workload': '%d users x %d items, d=%d, f32' % (args.small_users, args.small_items, args.d)}
        print(json.dumps(r), flush=True)
        results.append(r)
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--users', type=int, default=1000000)
    ap.add_argument('--items', type=int, default=1000000)
    ap.add_argument('--d', type=int, default=128)
    ap.add_argument('--hidden', type=int, default=512)
    ap.add_argument('--n-sampled', type=int, default=64)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--small-users', type=int, default=4096)
    ap.add_argument('--small-items', type=int, default=8192)
    ap.add_argument('--small-epochs', type=int, default=3)
    ap.add_argument('--no-steps', action='store_true', help='skip the 1M x 1M step table')
    ap.add_argument('--no-torch', action='store_true', help='skip the kernel path against torch path table')
    ap.add_argument('--out', default=None, help='also write every result line to this JSON file')
    args = ap.parse_args()
    import torch
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    torch.cuda.set_device(0)
    info = {'card': forms_bench.card()}
    print(json.dumps(info), flush=True)
    results = [info]
    if not args.no_steps:
        results += kernel_path(args)
    results += layer_alone(args)
    if not args.no_torch:
        results += against_torch(args)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(results, f, indent=1)


if __name__ == '__main__':
    main()
