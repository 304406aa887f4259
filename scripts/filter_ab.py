"""A/B (GPU) of two builds of the library on the SAME box and the same device operands: the filter sweep timed back to
back (sustained, as inside bench.py) and as single launches after idle, alternating between the builds.
usage: python scripts/filter_ab.py <users> <items> [--k K] <other .so> [<other .so> ...]
k <= 12 (default 10) times score_filter; a larger k times the wide form, score_wide, with wide_splits item splits."""
import argparse
import ctypes
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from tensorrec_b200 import _lib, kernels  # noqa: E402


ap = argparse.ArgumentParser()
ap.add_argument('users', type=int)
ap.add_argument('items', type=int)
ap.add_argument('libs', nargs='*')
ap.add_argument('--k', type=int, default=10)
cli = ap.parse_intermixed_args()


class A:
    users, items, k = cli.users, cli.items, cli.k
    d = 128


def bind(path):
    lib = ctypes.CDLL(path)
    for name, (restype, argtypes) in _lib.SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    return lib


LIBS = {'head': _lib.load()}
for path in cli.libs:
    LIBS[os.path.basename(path).replace('lib_', '').replace('.so', '')] = bind(os.path.abspath(path))
ROUNDS = int(os.environ.get('AB_ROUNDS', '2'))
uf, itf, wu, wi, bu, bi = bench.make_problem(A)
dev = torch.device('cuda', 0)
d_pad = kernels.d_pad_for(A.d)
ucsr, icsr = kernels.DeviceCSR.from_scipy(uf, device=dev), kernels.DeviceCSR.from_scipy(itf, device=dev)
stats = torch.empty(3, device=dev)
_, us, usc, unorm = kernels.gather_reduce(ucsr, torch.from_numpy(wu).to(dev), want_f32=False, split_d_pad=d_pad,
                                          want_norm=True)
_, its, isc = kernels.gather_reduce(icsr, torch.from_numpy(wi).to(dev), want_f32=False, split_d_pad=d_pad, stats=stats)
ub = kernels.project_biases(ucsr, torch.from_numpy(bu).to(dev))
ib = kernels.project_biases(icsr, torch.from_numpy(bi).to(dev))
items = kernels.SideOperands(None, its, isc, ib, A.items, A.d, d_pad, stats=stats)
f = kernels.FilterItems(items)
WIDE = A.k > kernels.filter_max_k()
users = kernels.SideOperands(None, us, usc, ub, A.users, A.d, d_pad)
wide_splits = kernels.wide_splits(A.users, A.items, A.k) if WIDE else None


def run_filter():
    if WIDE:
        return kernels.score_wide(users, unorm, f, A.items, A.k, wide_splits)
    return kernels.score_filter(us, usc, ub, unorm, f.hi, f.stats, f.bias_pad, f.block_max, f.perm, A.users, A.items,
                                d_pad, A.k, block_bias_min=f.block_min)


def identical(a, b):
    """Narrow form: every output.  Wide form (list_item, count, theta): counts, thetas and the first `count` entries
    of each list; the entries past the count are scratch."""
    if not WIDE:
        return all(torch.equal(x, y) for x, y in zip(a, b))
    (la, ca, ta), (lb, cb, tb) = a, b
    if not (torch.equal(ca, cb) and torch.equal(ta, tb)):
        return False
    held = torch.arange(la.shape[-1], device=la.device) < ca.unsqueeze(-1)
    return torch.equal(torch.where(held, la, 0), torch.where(held, lb, 0))


def sustained(n):
    run_filter()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        run_filter()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def cool(n, pause=0.4):
    ts = []
    for _ in range(n):
        time.sleep(pause)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run_filter()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


n = 6 if A.items >= 500000 else 20
print('%s k=%d, shape %d users x %d items; sustained = %d launches back to back, cool = median of 5 single launches '
      'after idle' % ('score_wide' if WIDE else 'score_filter', A.k, A.users, A.items, n))
ref = {}
for rnd in range(ROUNDS):
    for name in LIBS:
        _lib._lib = LIBS[name]
        out = run_filter()
        torch.cuda.synchronize()
        if rnd == 0:
            ref[name] = [t.clone() for t in out]
        print('round %d %-12s sustained %.2f ms   cool %.2f ms' % (rnd, name, sustained(n), cool(5)), flush=True)
for name in LIBS:
    print('candidate lists of %s identical to head: %s' % (name, identical(ref['head'], ref[name])))
for trig in (() if WIDE else ('32',)):
    os.environ['TRK_FILTER_TILE_END_TRIGGER'] = trig
    _lib._lib = LIBS['head']
    print('head, tile-end trigger %s: sustained %.2f ms   cool %.2f ms' % (trig, sustained(n), cool(5)))
os.environ.pop('TRK_FILTER_TILE_END_TRIGGER', None)
