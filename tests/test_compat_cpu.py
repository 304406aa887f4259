"""CPU tests of compat/: code written against jfkirk/tensorrec -- `import tensorrec`, `import tensorflow as tf` inside
plugin graphs, `nose_parameterized` -- runs on this package unchanged.  The custom graphs follow the reference README's
"custom representation / loss graph" examples."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'compat'))

import tensorrec                                # noqa: E402  (the alias package under compat/)
import tensorflow as tf                         # noqa: E402  (the stand-in under compat/)
import tensorrec_b200                           # noqa: E402
from nose_parameterized import parameterized    # noqa: E402


@pytest.fixture(autouse=True)
def cpu_session():
    from tensorrec_b200 import session_management as sm
    sm.set_session(sm.Session('cpu'))
    yield
    sm.set_session(None)


def test_tensorrec_alias_resolves_to_this_package():
    from tensorrec import TensorRec
    from tensorrec.loss_graphs import WMRBLossGraph
    assert TensorRec is tensorrec_b200.TensorRec and WMRBLossGraph is tensorrec_b200.loss_graphs.WMRBLossGraph
    for name in ('eval', 'util', 'input_utils', 'representation_graphs', 'prediction_graphs', 'errors'):
        assert getattr(tensorrec, name) is sys.modules['tensorrec_b200.' + name]


class TanhRepresentationGraph(tensorrec.representation_graphs.AbstractRepresentationGraph):
    def connect_representation_graph(self, tf_features, n_components, n_features, node_name_ending):
        tf_tanh_weights = tf.Variable(tf.random_normal([n_features, n_components], stddev=.5),
                                      name='tanh_weights_%s' % node_name_ending)
        tf_repr = tf.nn.tanh(tf.sparse_tensor_dense_matmul(tf_features, tf_tanh_weights))
        return tf_repr, [tf_tanh_weights]


class SimpleLossGraph(tensorrec.loss_graphs.AbstractLossGraph):
    def connect_loss_graph(self, tf_prediction_serial, tf_interactions_serial, **kwargs):
        return tf.reduce_mean(tf.abs(tf_prediction_serial - tf_interactions_serial))


def test_readme_custom_graphs_train_through_the_tf_stand_in():
    interactions, user_features, item_features = tensorrec.util.generate_dummy_data(
        num_users=30, num_items=40, interaction_density=.2, seed=3)
    model = tensorrec.TensorRec(n_components=5, user_repr_graph=TanhRepresentationGraph(),
                                item_repr_graph=TanhRepresentationGraph(), loss_graph=SimpleLossGraph())
    model.fit(interactions, user_features, item_features, epochs=1)
    assert 'tanh_weights_user_0' in model._variables and 'tanh_weights_item' in model._variables
    before = {k: v.detach().clone().numpy() for k, v in model._variables.items()}
    model.fit_partial(interactions, user_features, item_features, epochs=5)
    moved = [k for k in before if not np.array_equal(before[k], model._variables[k].detach().numpy())]
    assert 'tanh_weights_user_0' in moved and 'tanh_weights_item' in moved
    assert all(np.all(np.isfinite(v.detach().numpy())) for v in model._variables.values())


def test_tf_stand_in_ops_follow_tensorflow_semantics():
    x = np.array([[3.0, 4.0], [0.0, 0.0]], dtype=np.float32)
    assert np.allclose(tf.nn.l2_normalize(x, axis=1).numpy(), [[0.6, 0.8], [0.0, 0.0]])
    sp = tf.SparseTensor(indices=[[0, 1], [1, 0], [1, 0]], values=[2.0, 1.0, 3.0], dense_shape=[2, 2])
    w = np.array([[1.0, 10.0], [100.0, 1000.0]], dtype=np.float32)
    assert np.array_equal(tf.sparse_tensor_dense_matmul(sp, w).numpy(), [[200.0, 2000.0], [4.0, 40.0]])   # dups sum
    assert np.array_equal(tf.matmul(x, w, transpose_b=True).numpy(), x @ w.T)
    assert float(tf.reduce_mean(tf.abs(np.array([-1.0, 3.0], dtype=np.float32)))) == 2.0


def test_parameterized_expand_generates_one_named_method_per_case():
    import unittest

    class Case(unittest.TestCase):
        @parameterized.expand([('linear', 1), ('tanh graph', 2)])
        def test_it(self, name, n):
            self.assertGreater(n, 0)

    assert Case.test_it is None                  # the template itself is not a test
    assert hasattr(Case, 'test_it_0_linear') and hasattr(Case, 'test_it_1_tanh_graph')
    result = unittest.TestResult()
    unittest.defaultTestLoader.loadTestsFromTestCase(Case).run(result)
    assert result.testsRun == 2 and result.wasSuccessful()
