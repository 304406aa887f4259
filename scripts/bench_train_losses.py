"""Times the serial-loss training step (RMSELossGraph, SeparationLossGraph on trk_serial_loss_step; DESIGN §3.11) on
bench_train_forms.py's workload (LinearRepr features, 1M users x 1M items, d = 128, 4 positives per user and one
negative in four users, so Separation has both groups), for the dot form and a mixture of three tastes, with
WmrbStep's phase split, the split of the serial step into its forward / statistics / backward launches (torch.profiler,
in a pass of its own), and the ratio to the WMRB dot step of the same run; then, at a size the torch path finishes, the
kernel path against the torch-autograd path (fit_partial, one epoch).

    python scripts/bench_train_losses.py [--users N] [--items N] [--steps K] [--warmup W] [--small-users N]

Prints one JSON line per measurement and records the card name and power limit read in the same run."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bench  # noqa: E402
import bench_train_forms as forms_bench  # noqa: E402

SERIAL_PHASES = ['representations', 'serial_loss_step', 'weight_gradients', 'adam']
LOSSES = ['rmse', 'separation']


def forms():
    from tensorrec_b200.representation_graphs import LinearRepresentationGraph
    return [('dot', {}), ('3_tastes', {'n_tastes': 3}),
            ('3_tastes_attention', {'n_tastes': 3, 'attention_graph': LinearRepresentationGraph()})]


def loss_graph(loss):
    from tensorrec_b200 import loss_graphs
    return {'wmrb': loss_graphs.WMRBLossGraph, 'rmse': loss_graphs.RMSELossGraph,
            'separation': loss_graphs.SeparationLossGraph}[loss]()


def launch_split(stepper, args_step, n_steps):
    """ms per step of the serial step's three launches, from the CUDA kernel records of torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n_steps):
            stepper.step(*args_step)
        torch.cuda.synchronize()
    split = {'forward': 0.0, 'statistics': 0.0, 'backward': 0.0}
    for ev in prof.key_averages():
        name = ev.key
        us = getattr(ev, 'device_time_total', None)
        us = ev.cuda_time_total if us is None else us
        if 'serial_stats_kernel' in name or 'serial_finish_kernel' in name:
            split['statistics'] += us
        elif 'wmrb_step_kernel' in name and name.replace(' ', '').endswith(',1>(trk::WmrbParams)'):
            split['forward'] += us
        elif 'wmrb_step_kernel' in name and name.replace(' ', '').endswith(',2>(trk::WmrbParams)'):
            split['backward'] += us
    return {k: round(v / 1e3 / n_steps, 3) for k, v in split.items()}


def kernel_path(args, dtype):
    import torch
    import tensorrec_b200
    from tensorrec_b200 import train_kernels
    from tensorrec_b200.input_utils import SparseInput
    ns = argparse.Namespace(users=args.users, items=args.items, d=args.d, scores='iid')
    uf, itf, wu, wi, bu, bi = bench.make_problem(ns)
    inter = forms_bench.interactions_for(args.users, args.items)
    int_in, uf_in, if_in = SparseInput(inter), SparseInput(uf), SparseInput(itf)
    dev = torch.device('cuda', 0)
    results, wmrb_ms = [], None
    runs = [('wmrb', 'dot', {})] + [(loss, name, kw) for loss in LOSSES for name, kw in forms()]
    for loss, name, kw in runs:
        model = tensorrec_b200.TensorRec(n_components=args.d, loss_graph=loss_graph(loss), **kw)
        model.set_weights(forms_bench.weights_for(kw, uf, itf, args.d, wu, wi, bu, bi))
        stepper = train_kernels.WmrbStep(model, dev, seed=0, bf16=dtype == 'bf16')
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
        phases = SERIAL_PHASES if serial else forms_bench.PHASES
        marks, per = stepper.marks, len(phases) + 1
        phase = {p: sum(marks[s * per + j][1].elapsed_time(marks[s * per + j + 1][1]) for s in range(args.steps))
                 / args.steps for j, p in enumerate(phases)}
        ms = sum(marks[s * per][1].elapsed_time(marks[s * per + per - 1][1]) for s in range(args.steps)) / args.steps
        stepper.marks = None
        wmrb_ms = ms if loss == 'wmrb' else wmrb_ms
        r = {'path': 'kernel', 'loss': loss, 'form': name, 'dtype': dtype, 'ms_per_step': round(ms, 3),
             'ratio_to_wmrb_dot': round(ms / wmrb_ms, 3), 'phases_ms': {k: round(v, 3) for k, v in phase.items()},
             'loss_value': float(stepper.last['loss'].sum()) if serial else None,
             'workload': '%d users x %d items, d=%d, %d interactions' % (args.users, args.items, args.d, inter.nnz)}
        if serial:
            r['serial_launches_ms'] = launch_split(stepper, step_args, args.steps)
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
    inter = forms_bench.interactions_for(args.small_users, args.small_items)
    results = []
    for loss in LOSSES:
        for name, kw in forms():
            times, losses = {}, {}
            for path in ('kernel', 'torch'):
                train_kernels.TRAIN_PATH = 'torch' if path == 'torch' else 'auto'
                model = tensorrec_b200.TensorRec(n_components=args.d, loss_graph=loss_graph(loss), **kw)
                model.set_weights(forms_bench.weights_for(kw, uf, itf, args.d, wu, wi, bu, bi))
                model.fit_partial(inter, uf, itf, epochs=1)       # warm-up
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                model.fit_partial(inter, uf, itf, epochs=args.small_epochs)
                torch.cuda.synchronize()
                times[path] = (time.perf_counter() - t0) * 1e3 / args.small_epochs
                assert (getattr(model, '_wmrb_step', None) is not None) == (path == 'kernel'), (loss, name, path)
            train_kernels.TRAIN_PATH = 'auto'
            r = {'path': 'kernel_vs_torch', 'loss': loss, 'form': name,
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
    ap.add_argument('--n-sampled', type=int, default=64, help='n_sampled_items of the WMRB dot step compared with')
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
    info = {'card': forms_bench.card()}
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
