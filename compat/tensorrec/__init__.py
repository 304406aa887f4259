"""`import tensorrec` for code written against jfkirk/tensorrec: every name resolves to tensorrec_b200.

Put this directory on PYTHONPATH (next to the repository root) and the reference's own modules -- tensorrec.eval,
tensorrec.util, tensorrec.loss_graphs, ... -- are the H100 implementations; `from tensorrec import TensorRec` works
unchanged."""
import importlib
import os
import sys

import tensorrec_b200 as _impl

# the reference's modules all import tensorflow; code written against them relies on what that import provides
# (tensor.eval(session=...), the numpy-1 aliases): load the stand-in that sits next to this package
if 'tensorflow' not in sys.modules:
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    try:
        importlib.import_module('tensorflow')
    finally:
        sys.path.pop(0)

_SUBMODULES = ('tensorrec', 'eval', 'input_utils', 'loss_graphs', 'representation_graphs', 'prediction_graphs',
               'recommendation_graphs', 'session_management', 'util', 'errors')
for _name in _SUBMODULES:
    _module = importlib.import_module('tensorrec_b200.' + _name)
    sys.modules[__name__ + '.' + _name] = _module
    globals()[_name] = _module

TensorRec = _impl.TensorRec
TopK = _impl.TopK
__version__ = _impl.__version__
__all__ = ['TensorRec', 'TopK'] + [n for n in _SUBMODULES if n != 'tensorrec']
