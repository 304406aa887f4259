"""CPU tests of the Euclidean user x item tensor-core route: topk_route with euclidean=True and the model predicate
_euclidean_tensor_ok, next to _tensor_path_ok (which keeps covering dot and cosine only)."""
import pytest


@pytest.fixture
def TR():
    from tensorrec_b200 import tensorrec
    return tensorrec


def route(TR, k, n_items=10 ** 6, single_taste=True, sharded=False):
    return TR.topk_route(k, n_items, True, single_taste, 12, 32, sharded=sharded, euclidean=True)


def test_route_k_limits_and_catalogue_floor(TR, monkeypatch):
    monkeypatch.setattr(TR, 'EUCLIDEAN_MIN_ITEMS', 5000)
    # no filter or wide form: every k <= 32 is exact3, larger k dense+rank
    assert {route(TR, k) for k in (1, 10, 12, 13, 32)} == {'exact3'}
    assert {route(TR, k) for k in (33, 100, 1024, 2000)} == {'dense+rank'}
    assert route(TR, 10, n_items=4999) == 'dense+rank' and route(TR, 10, n_items=5000) == 'exact3'
    assert route(TR, 10, n_items=0) == 'dense+rank'
    # tastes: one exact sweep per taste, then the de-duplicating merge
    assert route(TR, 10, single_taste=False) == 'exact3' and route(TR, 100, single_taste=False) == 'dense+rank'
    # not a tensor-core model: dense+rank whatever k
    assert TR.topk_route(10, 10 ** 6, False, True, 12, 32, euclidean=True) == 'dense+rank'


def test_sharded_route_does_not_depend_on_the_shard_size(TR, monkeypatch):
    monkeypatch.setattr(TR, 'EUCLIDEAN_MIN_ITEMS', 5000)
    assert {route(TR, 10, n_items=n, sharded=True) for n in (1, 4999, 5000, 10 ** 6)} == {'exact3'}
    assert {route(TR, 100, n_items=n, sharded=True) for n in (1, 10 ** 6)} == {'dense+rank'}


@pytest.mark.parametrize('topk_path', ['auto', 'exact'])
def test_topk_path_does_not_change_the_euclidean_route(TR, monkeypatch, topk_path):
    monkeypatch.setattr(TR, 'EUCLIDEAN_MIN_ITEMS', 5000)
    monkeypatch.setattr(TR, 'TOPK_PATH', topk_path)
    assert route(TR, 5) == 'exact3' and route(TR, 32) == 'exact3' and route(TR, 33) == 'dense+rank'


def test_default_route_is_unchanged_without_the_keyword(TR, monkeypatch):
    monkeypatch.setattr(TR, 'WIDE_MIN_ITEMS', 5000)
    args = (12, 32)
    assert TR.topk_route(10, 10 ** 6, True, True, *args) == 'filter'
    assert TR.topk_route(20, 10 ** 6, True, True, *args) == 'exact3'
    assert TR.topk_route(100, 10 ** 6, True, True, *args) == 'wide'


def test_euclidean_min_items_keeps_small_catalogues_on_dense_rank(TR):
    assert TR.EUCLIDEAN_MIN_ITEMS >= 1024        # the 700-item catalogue of the exclusion tests stays on dense+rank


def models():
    import tensorrec_b200 as T
    P = T.prediction_graphs
    attention = T.representation_graphs.LinearRepresentationGraph()
    return {
        'dot': (T.TensorRec(n_components=64), False, True),
        'cosine': (T.TensorRec(n_components=64, prediction_graph=P.CosineSimilarityPredictionGraph()), False, True),
        'euclidean': (T.TensorRec(n_components=64, prediction_graph=P.EuclideanSimilarityPredictionGraph()), True,
                      False),
        'euclidean_d128': (T.TensorRec(n_components=128, prediction_graph=P.EuclideanSimilarityPredictionGraph()), True,
                           False),
        'euclidean_tastes': (T.TensorRec(n_components=64, n_tastes=3,
                                         prediction_graph=P.EuclideanSimilarityPredictionGraph()), True, False),
        'euclidean_attention': (T.TensorRec(n_components=64, n_tastes=2, attention_graph=attention,
                                            prediction_graph=P.EuclideanSimilarityPredictionGraph()), False, False),
        'euclidean_d200': (T.TensorRec(n_components=200, prediction_graph=P.EuclideanSimilarityPredictionGraph()),
                           False, False),
        'dot_d200': (T.TensorRec(n_components=200), False, False),
        'dot_attention': (T.TensorRec(n_components=64, n_tastes=2, attention_graph=attention), False, False),
    }


@pytest.mark.parametrize('kind', sorted(models()))
def test_predicates_by_model_kind(TR, kind):
    model, euclidean_ok, tensor_ok = models()[kind]
    assert model._euclidean_tensor_ok() == euclidean_ok
    assert model._tensor_path_ok(allow_tastes=True) == tensor_ok     # _tensor_path_ok is unchanged: dot / cosine only


def test_score_path_exact_and_tensor(TR, monkeypatch):
    ms = models()
    monkeypatch.setattr(TR, 'SCORE_PATH', 'exact')
    assert not any(m._euclidean_tensor_ok() for m, _, _ in ms.values())
    assert not any(m._tensor_path_ok(True) for m, _, _ in ms.values())
    monkeypatch.setattr(TR, 'SCORE_PATH', 'tensor')
    # the Euclidean predicate never raises; _tensor_path_ok still raises for every model it does not cover
    assert ms['euclidean'][0]._euclidean_tensor_ok() and not ms['euclidean_d200'][0]._euclidean_tensor_ok()
    with pytest.raises(RuntimeError):
        ms['euclidean'][0]._tensor_path_ok(True)
    assert ms['dot'][0]._tensor_path_ok(True)
