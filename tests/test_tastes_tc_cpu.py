"""CPU tests of the mixture-of-tastes routes: topk_route with attention, TensorRec._tastes_tensor_ok by model kind, the
block plan of the taste-collapsing kernel, and the predicates that stay as they were."""
import pytest

import tensorrec_b200 as T
from tensorrec_b200 import kernels, tensorrec

R, P = T.representation_graphs, T.prediction_graphs


def route(k, n_items, sharded=False, attention=True, model_ok=True):
    return tensorrec.topk_route(k, n_items, model_ok, False, 16, 32, sharded=sharded, attention=attention)


def model(n_tastes=3, attention=True, prediction=P.DotProductPredictionGraph, d=64):
    return T.TensorRec(n_components=d, n_tastes=n_tastes, prediction_graph=prediction(),
                       attention_graph=R.LinearRepresentationGraph() if attention else None)


def test_attention_route_k_limits_and_catalogue_floor():
    floor = tensorrec.ATTENTION_MIN_ITEMS
    for k in (1, 10, 32):
        assert route(k, floor) == 'exact3'
        assert route(k, floor - 1) == 'dense+rank'
    assert route(33, 10 ** 6) == 'dense+rank'
    assert route(100, 10 ** 6) == 'dense+rank'
    assert route(10, 0) == 'dense+rank'
    assert route(10, 10 ** 6, model_ok=False) == 'dense+rank'


def test_attention_route_in_sharded_calls():
    assert route(10, 1, sharded=True) == 'exact3'      # every rank takes exact3, whatever its shard size
    assert route(33, 10 ** 6, sharded=True) == 'dense+rank'


@pytest.mark.parametrize('topk_path', ['auto', 'exact'])
def test_attention_route_ignores_topk_path(monkeypatch, topk_path):
    monkeypatch.setattr(tensorrec, 'TOPK_PATH', topk_path)
    assert route(10, 10 ** 6) == 'exact3'
    assert route(10, 10) == 'dense+rank'


def test_routes_without_the_keyword_are_unchanged():
    assert tensorrec.topk_route(10, 10 ** 6, True, False, 16, 32) == 'filter'
    assert tensorrec.topk_route(20, 10 ** 6, True, False, 16, 32) == 'exact3'
    assert tensorrec.topk_route(100, 10 ** 6, True, False, 16, 32) == 'dense+rank'
    assert tensorrec.topk_route(100, 10 ** 6, True, True, 16, 32) == 'wide'


def test_tastes_tensor_ok_by_model_kind(monkeypatch):
    assert not model(n_tastes=1, attention=False)._tastes_tensor_ok()
    assert model(n_tastes=3, attention=False)._tastes_tensor_ok()
    assert model(n_tastes=3, attention=True)._tastes_tensor_ok()
    assert model(prediction=P.CosineSimilarityPredictionGraph)._tastes_tensor_ok()
    assert not model(prediction=P.EuclideanSimilarityPredictionGraph)._tastes_tensor_ok()
    assert not model(d=200)._tastes_tensor_ok()
    assert model(d=128)._tastes_tensor_ok()
    assert model(n_tastes=64, attention=False)._tastes_tensor_ok()
    assert not model(n_tastes=65, attention=False)._tastes_tensor_ok()
    assert model(n_tastes=32, attention=True)._tastes_tensor_ok()
    assert not model(n_tastes=33, attention=True)._tastes_tensor_ok()
    monkeypatch.setattr(tensorrec, 'SCORE_PATH', 'exact')
    assert not model()._tastes_tensor_ok()
    monkeypatch.setattr(tensorrec, 'SCORE_PATH', 'tensor')
    assert model()._tastes_tensor_ok()


@pytest.mark.parametrize('n_tastes,attention,per_wg,rows', [
    (2, False, 32, 64), (3, False, 21, 63), (5, False, 12, 60), (64, False, 1, 64),
    (1, True, 32, 64), (3, True, 10, 60), (5, True, 6, 60), (32, True, 1, 64)])
def test_block_plan(n_tastes, attention, per_wg, rows):
    assert kernels.tastes_plan(n_tastes, attention) == (per_wg, 2 * per_wg, rows)


def test_block_plan_limits():
    assert kernels.tastes_plan(1, False) is None        # one operand row: the plain kernel
    assert kernels.tastes_plan(65, False) is None
    assert kernels.tastes_plan(33, True) is None


def test_unchanged_predicates(monkeypatch):
    m = model(n_tastes=3, attention=True)
    assert not m._tensor_path_ok(allow_tastes=True)     # attention stays off the plain tensor path
    assert not m._euclidean_tensor_ok()
    plain = model(n_tastes=3, attention=False)
    assert not plain._tensor_path_ok()
    assert plain._tensor_path_ok(allow_tastes=True)
    assert model(n_tastes=2, attention=False, prediction=P.EuclideanSimilarityPredictionGraph)._euclidean_tensor_ok()
