"""Host-side helpers of the predict / predict_rank(k) / training paths that need no device: sizing of the fallback buffer,
user blocking of predict, what the kernel training step covers, per-item positive sums, bench workload description."""
import argparse

import numpy as np
import scipy.sparse as sp

import bench
from tensorrec_b200 import TensorRec, kernels, train_kernels
from tensorrec_b200.input_utils import SparseInput
from tensorrec_b200.loss_graphs import BalancedWMRBLossGraph, RMSELossGraph, WMRBLossGraph
from tensorrec_b200.prediction_graphs import CosineSimilarityPredictionGraph
from tensorrec_b200.representation_graphs import NormalizedLinearRepresentationGraph


def test_fallback_capacity_is_an_eighth_in_whole_user_blocks():
    for n in (1, 5, 127, 128, 1000, 1024, 8191, 8192, 100000, 1000000, 10000001):
        cap = kernels.fallback_capacity(n)
        assert cap % 128 == 0 and cap >= min(n, 1024)
        assert cap <= max(((n + 127) // 128) * 128, 1024 + 127)            # never more than the batch (rounded up)
        if n >= 8 * 1024:
            assert abs(cap - n // 8) < 128
    assert kernels.fallback_capacity(1000000) == 125056
    assert kernels.fallback_capacity(2048) >= kernels.FALLBACK_SMALL_ROWS     # the small tier fits as soon as the batch does


def test_user_blocks_cover_every_row_once_in_order():
    model = TensorRec(n_components=8)
    feats = sp.random(1000, 30, density=0.1, format='coo', random_state=0, dtype=np.float32)
    whole = model._user_blocks(SparseInput(feats), n_items=50, user_batch_size=None)
    assert [(a, b) for a, b, _ in whole] == [(0, 1000)] and whole[0][2].matrix is feats
    blocks = model._user_blocks(SparseInput(feats), n_items=50, user_batch_size=300)
    assert [(a, b) for a, b, _ in blocks] == [(0, 300), (300, 600), (600, 900), (900, 1000)]
    stacked = sp.vstack([blk.matrix for _, _, blk in blocks]).toarray()
    assert np.array_equal(stacked, feats.toarray())
    # default block size: a multiple of 128 rows whose fp32 scores fit PREDICT_BLOCK_BYTES
    n_items = 100000
    rows = model._user_blocks(SparseInput(sp.random(10 ** 6, 4, density=0.25, format='csr', random_state=1,
                                                    dtype=np.float32)), n_items, None)[0][1]
    assert rows % 128 == 0 and rows * n_items * 4 <= model.PREDICT_BLOCK_BYTES < (rows + 128) * n_items * 4


def test_step_plan_gives_each_model_its_form(monkeypatch):
    monkeypatch.setattr(train_kernels, 'TRAIN_PATH', 'kernel')
    plan = train_kernels.step_plan
    dot = train_kernels.StepForm(pair='dot', n_tastes=1, attention=False, normalize_user=0, normalize_attn=0,
                                 normalize_item=0, d_pad=8, loss='wmrb')          # Linear x dot x WMRB, one taste
    assert plan(TensorRec(n_components=8, loss_graph=WMRBLossGraph())) == dot
    assert plan(TensorRec(n_components=128, loss_graph=BalancedWMRBLossGraph())) == dot._replace(d_pad=128)
    assert plan(TensorRec(n_components=8, loss_graph=RMSELossGraph())) == dot._replace(loss='rmse')
    assert plan(TensorRec(n_components=10, loss_graph=WMRBLossGraph())) == dot._replace(d_pad=12)    # zero-padded
    assert plan(TensorRec(n_components=8, n_tastes=2, loss_graph=WMRBLossGraph())) == dot._replace(n_tastes=2)
    assert plan(TensorRec(n_components=8, loss_graph=WMRBLossGraph(),
                          prediction_graph=CosineSimilarityPredictionGraph())) == dot._replace(normalize_user=1,
                                                                                                normalize_item=1)
    assert plan(TensorRec(n_components=8, loss_graph=WMRBLossGraph(),
                          item_repr_graph=NormalizedLinearRepresentationGraph())) == dot._replace(normalize_item=1)
    monkeypatch.setattr(train_kernels, 'TRAIN_PATH', 'torch')
    assert plan(TensorRec(n_components=8, loss_graph=WMRBLossGraph())) is None


def test_positive_item_sums_and_positive_count():
    m = sp.coo_matrix((np.array([1.0, -1.0, 2.0, 0.5, 0.0, 3.0], dtype=np.float32),
                       (np.array([0, 0, 1, 2, 2, 2]), np.array([1, 2, 1, 0, 3, 1]))), shape=(3, 5))
    sums = train_kernels.positive_item_sums(m, 5)
    assert sums.dtype == np.float32 and np.array_equal(sums, np.array([0.5, 6.0, 0.0, 0.0, 0.0], dtype=np.float32))
    assert SparseInput(m).n_positive == 4
    dup = sp.coo_matrix((np.array([1.0, 1.0], dtype=np.float32), (np.array([0, 0]), np.array([2, 2]))), shape=(1, 3))
    assert np.array_equal(train_kernels.positive_item_sums(dup, 3), np.array([0.0, 0.0, 2.0], dtype=np.float32))


def test_bench_config_is_a_function_of_the_workload_only():
    ns = argparse.Namespace(users=1000000, items=1000000, d=128, k=10, scores='iid')
    a, b = bench.workload_config(ns), bench.workload_config(argparse.Namespace(**vars(ns)))
    assert a == b and set(a) == {'workload', 'l2'}
    assert '1000000 users x 1000000 items' in a['workload'] and 'exceed L2' in a['l2']
    small = bench.workload_config(argparse.Namespace(users=2000, items=3000, d=64, k=10, scores='iid'))
    assert 'FIT in L2' in small['l2'] and small['workload'] != a['workload']
