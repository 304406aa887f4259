"""tensorrec_b200 -- the predict / predict_rank hot path of jfkirk/tensorrec, H100-native (sm_90a), behind the
reference's own TensorRec class and RepresentationGraph / PredictionGraph / LossGraph plugin surface.

Export list mirrors tensorrec/__init__.py:1-14."""
from .tensorrec import TensorRec, TopK
from . import eval
from . import input_utils
from . import loss_graphs
from . import representation_graphs
from . import prediction_graphs
from . import recommendation_graphs
from . import session_management
from . import util
from . import errors

__version__ = '0.1.0'   # follows the API of tensorrec 0.26.2

__all__ = [
    'TensorRec', 'TopK', 'eval', 'util', 'loss_graphs', 'representation_graphs', 'prediction_graphs',
    'recommendation_graphs', 'session_management', 'input_utils', 'errors',
]
