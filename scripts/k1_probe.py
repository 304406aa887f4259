"""K1 (csr_gather_reduce) timing at the bench shape (L2 flushed between launches): output variants, and with the
re-referenced tag rows of the indicator regime pinned in L2 (trk_l2_persist_window).
usage: python scripts/k1_probe.py [rows]"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from tensorrec_b200 import kernels  # noqa: E402


class A:
    users = int(sys.argv[1]) if len(sys.argv) > 1 else 1000000
    items, d, k = 1024, 128, 10


uf, itf, wu, wi, bu, bi = bench.make_problem(A)
dev = torch.device('cuda', 0)
ucsr = kernels.DeviceCSR.from_scipy(uf, device=dev)
w = torch.from_numpy(wu).to(dev)
bu_d = torch.from_numpy(bu).to(dev)
d_pad = kernels.d_pad_for(A.d)
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def timeit(fn, n=7):
    fn()
    ts = []
    for _ in range(n):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


nnz = uf.nnz
distinct = int(np.unique(uf.indices).shape[0])
survey = nnz * 8 + (A.users + 1) * 4 + distinct * A.d * 4 + A.users * A.d * 4
print('indicator regime: %d rows, nnz %d, distinct columns %d, SURVEY 8(d) bytes %.3f GB' % (A.users, nnz, distinct, survey / 1e9))


def report(name, ms):
    print('%-58s %.3f ms  %.0f GB/s on the 8(d) bytes = %.3f of the H100 SXM data sheet\'s 3350' % (
        name, ms, survey / ms / 1e6, survey / ms / 1e6 / 3350.0))


variants = [('split only', dict(want_f32=False, split_d_pad=d_pad)),
            ('split + norm (the filter path)', dict(want_f32=False, split_d_pad=d_pad, want_norm=True)),
            ('fp32 only', dict(want_f32=True)),
            ('fp32 + split', dict(want_f32=True, split_d_pad=d_pad))]
for name, kw in variants:
    report('K1 ' + name, timeit(lambda: kernels.gather_reduce(ucsr, w, **kw)))
report('project_biases', timeit(lambda: kernels.project_biases(ucsr, bu_d)))
# tag regime (tensorrec/util.py:61-85: 200 features, ~20 nnz per row): the 100 KB table lives in L2, the kernel is bound by
# the index stream and the output write -- SURVEY 8(d): 20*8 + 4 + 512 = 676 B per row
from tests import helpers as H  # noqa: E402
tf = H.tag_features(A.users, 200, 20, seed=0)
tcsr = kernels.DeviceCSR.from_scipy(tf, device=dev)
tw = torch.from_numpy(H.linear_weights(200, A.d, seed=2)).to(dev)
survey = tf.nnz * 8 + (A.users + 1) * 4 + 200 * A.d * 4 + A.users * A.d * 4
print('tag regime: %d rows, nnz %d, SURVEY 8(d) bytes %.3f GB' % (A.users, tf.nnz, survey / 1e9))
for name, kw in variants[:3]:
    report('K1 tag regime, ' + name, timeit(lambda: kernels.gather_reduce(tcsr, tw, **kw)))
