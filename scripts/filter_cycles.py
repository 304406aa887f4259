"""Cycle accounting of the narrow filter kernel (GPU): where the consumer warps' clocks go.

    python scripts/filter_cycles.py [--tree DIR | --lib PATH] [--k K] [--launches N] [shape ...]

Builds the library with -DTRK_FILTER_CYCLES into a temporary directory (from this checkout, or from the checkout at
--tree; --lib takes such a library ready-made), runs score_filter on the seeded inputs of bench.py and prints, per
shape (default 1000000x1000000 and 1000000x125000, users x items, d128), each category's share of the consumer warps'
clocks and the producer warp's share of clocks spent waiting for a free item-tile slot.  Lane 0 of every warp reads
clock64(); the timers cost a few instructions per event, so the total runs slightly slower than the shipped kernel.
TRK_FILTER_MAX_STAGES and the other probe knobs of the launcher apply as usual."""
import argparse
import ctypes
import importlib.util
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from tensorrec_b200 import _lib, kernels  # noqa: E402

# FilterCycle in score_filter_tc.cu, in order
NAMES = ['b_full', 'mma', 'row_halves', 'slow', 'compact_mid', 'compact_tile_end', 'compact_final', 'output',
         'release', 'unit_start', 'warm', 'consumer', 'consumer_warps', 'producer_empty', 'producer', 'producer_warps']

ROWS = [   # (label, value from the sums)
    ('wait on b_full', lambda c: c['b_full']),
    ('filter_mma_rows (fence .. wait)', lambda c: c['mma']),
    ('register fast path', lambda c: c['row_halves'] - c['slow']),
    ('staged slow path (filter_32, exclusion)', lambda c: c['slow'] - c['compact_mid']),
    ('compaction, mid-tile', lambda c: c['compact_mid']),
    ('compaction, tile end', lambda c: c['compact_tile_end']),
    ('compaction, final', lambda c: c['compact_final']),
    ('output of the lists', lambda c: c['output']),
    ('slot release', lambda c: c['release']),
    ('user-block load', lambda c: c['unit_start']),
    ('warm start (its MMAs included)', lambda c: c['warm']),
]


def load_build(tree):
    spec = importlib.util.spec_from_file_location('trk_build', os.path.join(tree, 'tensorrec_b200', 'csrc', 'build.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def bind(path):
    lib = ctypes.CDLL(path)
    for name, (restype, argtypes) in _lib.SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    lib.trk_debug_filter_cycles.restype = ctypes.c_int
    lib.trk_debug_filter_cycles.argtypes = [ctypes.c_void_p, ctypes.c_int]
    return lib


def read_cycles(lib):
    buf = (ctypes.c_ulonglong * 64)()
    n = lib.trk_debug_filter_cycles(buf, 64)
    if n != len(NAMES):
        raise RuntimeError('trk_debug_filter_cycles returned %d (expected %d categories)' % (n, len(NAMES)))
    return {name: int(buf[i]) for i, name in enumerate(NAMES)}


def measure(lib, users, items, k, launches):
    class A:
        pass
    A.users, A.items, A.k, A.d = users, items, k, 128
    uf, itf, wu, wi, bu, bi = bench.make_problem(A)
    dev = torch.device('cuda', 0)
    d_pad = kernels.d_pad_for(A.d)
    ucsr, icsr = kernels.DeviceCSR.from_scipy(uf, device=dev), kernels.DeviceCSR.from_scipy(itf, device=dev)
    stats = torch.empty(3, device=dev)
    _, us, usc, unorm = kernels.gather_reduce(ucsr, torch.from_numpy(wu).to(dev), want_f32=False, split_d_pad=d_pad,
                                              want_norm=True)
    _, its, isc = kernels.gather_reduce(icsr, torch.from_numpy(wi).to(dev), want_f32=False, split_d_pad=d_pad,
                                        stats=stats)
    ub = kernels.project_biases(ucsr, torch.from_numpy(bu).to(dev))
    ib = kernels.project_biases(icsr, torch.from_numpy(bi).to(dev))
    f = kernels.FilterItems(kernels.SideOperands(None, its, isc, ib, items, A.d, d_pad, stats=stats))

    def run():
        return kernels.score_filter(us, usc, ub, unorm, f.hi, f.stats, f.bias_pad, f.block_max, f.perm, users, items,
                                    d_pad, k, block_bias_min=f.block_min)
    run()
    torch.cuda.synchronize()
    read_cycles(lib)   # drop the warm-up launch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        run()
    b.record()
    torch.cuda.synchronize()
    return read_cycles(lib), a.elapsed_time(b) / launches


def report(c, ms, users, items, launches):
    cons = max(c['consumer'], 1)
    n_warps = max(c['consumer_warps'] // launches, 1)
    print('\n%d users x %d items, k-sweep of %d launches: %.2f ms per launch (instrumented), %d consumer warps, '
          '%.0f clocks per consumer warp per launch' % (users, items, launches, ms, n_warps,
                                                        c['consumer'] / launches / n_warps))
    print('%-42s %8s' % ('consumer category', 'share'))
    acc = 0
    for label, fn in ROWS:
        v = fn(c)
        acc += v
        print('%-42s %7.2f%%' % (label, 100.0 * v / cons))
    print('%-42s %7.2f%%' % ('rest of the loop', 100.0 * (c['consumer'] - acc) / cons))
    print('%-42s %7.2f%%' % ('producer: wait on b_empty (of its clocks)',
                             100.0 * c['producer_empty'] / max(c['producer'], 1)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('shapes', nargs='*', default=['1000000x1000000', '1000000x125000'])
    ap.add_argument('--tree', default=ROOT, help='checkout whose sources are built (default: this one)')
    ap.add_argument('--lib', default=None, help='a library built with -DTRK_FILTER_CYCLES (skips the build)')
    ap.add_argument('--k', type=int, default=10)
    ap.add_argument('--launches', type=int, default=2)
    cli = ap.parse_args()
    assert torch.cuda.is_available(), 'filter_cycles.py measures on a CUDA device'
    with tempfile.TemporaryDirectory() as tmp:
        path = cli.lib or load_build(os.path.abspath(cli.tree)).build(force=True, defines=['TRK_FILTER_CYCLES'],
                                                                        out_dir=tmp)
        lib = bind(os.path.abspath(path))
        _lib._lib = lib
        print('library:', path, ' device:', torch.cuda.get_device_name(0))
        for shape in cli.shapes:
            users, items = (int(x) for x in shape.split('x'))
            c, ms = measure(lib, users, items, cli.k, cli.launches)
            report(c, ms, users, items, cli.launches)


if __name__ == '__main__':
    main()
