"""bench.py helpers that run without a GPU: the secondary workloads take the run's --steps / --warmup, and
--dump-outputs writes the top-k in the documented files, dtypes and size budget, identically from run to run."""
import argparse
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import bench  # noqa: E402


def test_extras_use_the_runs_steps_and_warmup(monkeypatch):
    seen = {}

    def fake(name):
        def run(a, emit=True):
            seen[name] = (a.steps, a.warmup)
            return {'steps': a.steps, 'warmup': a.warmup}
        return run

    for name in ('run_dense', 'run_full_ranks', 'run_train'):
        monkeypatch.setattr(bench, name, fake(name))
    args = argparse.Namespace(steps=1, warmup=0, users=10, items=10, d=8)
    extra = bench.run_extras(args)
    assert seen == {'run_dense': (1, 0), 'run_full_ranks': (1, 0), 'run_train': (1, 0)}
    assert all(extra[k]['steps'] == 1 for k in ('dense', 'ranks', 'train'))
    assert (args.users, args.items, args.d) == (10, 10, 8)     # the per-workload sizes do not leak back


def _fake_top(n, k, seed=0):
    rng = np.random.default_rng(seed)
    items = torch.from_numpy(rng.integers(0, 2 ** 31 - 1, size=(n, k), dtype=np.int64).astype(np.int32))
    scores = torch.from_numpy(rng.standard_normal((n, k)).astype(np.float32))
    return SimpleNamespace(items=items, scores=scores)


def test_dump_outputs_writes_every_row_when_they_fit(tmp_path):
    top = _fake_top(50, 10)
    bench.dump_outputs(str(tmp_path), top, user_lo=7)
    items = np.load(str(tmp_path / 'top_items.npy'))
    scores = np.load(str(tmp_path / 'top_scores.npy'))
    rows = np.load(str(tmp_path / 'user_rows.npy'))
    assert items.dtype == np.float64 and scores.dtype == np.float32 and rows.dtype == np.float64
    assert np.array_equal(items, top.items.numpy().astype(np.float64))      # int32 ids are exact in float64
    assert np.array_equal(scores, top.scores.numpy())
    assert np.array_equal(rows, np.arange(7, 57, dtype=np.float64))


def test_dump_outputs_samples_within_the_budget_and_repeats_exactly(tmp_path):
    top = _fake_top(5000, 10)
    budget = 64 * 1024
    for out in ('a', 'b'):
        bench.dump_outputs(str(tmp_path / out), top, user_lo=0, suffix='_rank1', max_bytes=budget)
    total = sum(os.path.getsize(str(tmp_path / 'a' / f)) for f in os.listdir(str(tmp_path / 'a')))
    assert total <= budget + 3 * 128                                       # + the three .npy headers
    rows = np.load(str(tmp_path / 'a' / 'user_rows_rank1.npy')).astype(np.int64)
    assert len(rows) == budget // (10 * 12 + 8) and np.all(np.diff(rows) > 0)
    assert np.array_equal(np.load(str(tmp_path / 'a' / 'top_items_rank1.npy')), top.items.numpy()[rows])
    for name in ('top_items_rank1.npy', 'top_scores_rank1.npy', 'user_rows_rank1.npy'):
        assert np.array_equal(np.load(str(tmp_path / 'a' / name)), np.load(str(tmp_path / 'b' / name)))


def test_dump_outputs_is_refused_outside_the_flagship_arm(tmp_path):
    out = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--impl', 'reference', '--dump-outputs',
                          str(tmp_path / 'd')], capture_output=True, text=True, timeout=120, cwd=ROOT)
    assert out.returncode != 0 and '--dump-outputs' in out.stderr
    assert not os.path.exists(str(tmp_path / 'd'))
