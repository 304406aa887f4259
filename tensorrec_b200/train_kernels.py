"""The sampled-rank training step on hand-written kernels (SURVEY 8 row f1; BASELINE config #4).

For the model family the reference's WMRB examples use -- LinearRepresentationGraph on both sides, DotProductPredictionGraph,
WMRBLossGraph or BalancedWMRBLossGraph, one taste, no attention -- one Adam step is, through the C ABI:

    K1  trk_csr_gather_reduce_f32      user / item representations             (tensorrec/representation_graphs.py:40)
        trk_csr_project_biases_f32     projected biases                        (tensorrec/recommendation_graphs.py:4-19)
        trk_f32_to_bf16                [bf16 form] representations rounded once, halving the gather traffic of the step
        trk_sample_items               n_sampled_items item ids per user       (tensorrec/util.py:12-21)
        trk_wmrb_step_tastes           serial predictions of the interactions and of the samples, WMRB loss, and the
                                       gradient with respect to representations and projected biases, fused
    K1^T trk_csr_gather_reduce_f32     on the transposed CSR: weight gradients (the gradient of sparse_tensor_dense_matmul)
        trk_csr_project_biases_f32     on the transposed CSR: feature-bias gradients
        trk_adam_step_f32              L2 term + Adam moments + parameter step (tensorrec/tensorrec.py:487-489)

The same step trains every other form step_plan() accepts (DESIGN §3.10): cosine and Euclidean prediction,
NormalizedLinearRepresentationGraph users / items / attention, mixtures of tastes with max or attention collapse, and
any n_components (zero-padded to a multiple of 4 inside the step).  There the user operand is NT taste planes (and NT
attention planes) stacked for trk_wmrb_step_tastes, normalised rows come from trk_l2_normalize_rows_step_f32 forward
and backward, and every weight gets its own K1^T and Adam pass.

RMSELossGraph and SeparationLossGraph models of those forms (step_plan's loss 'rmse' / 'separation'; DESIGN §3.11)
train on the same representations, K1^T and Adam, with trk_serial_loss_step in place of the sampler and
trk_wmrb_step_tastes: a forward launch writes the serial predictions, a statistics launch reduces them to the scalar
loss and a loss state on the device, and a backward launch turns each prediction into its gradient from that state.

ReLURepresentationGraph user, item or attention sides (relu_step_plan; DESIGN §3.14) add a hidden-layer stage: K1 of
X . W1 into the pre-activations P, trk_relu_layer_forward_f32 (relu(P + b) . W2) into the operand plane, and after the
loss kernel trk_relu_layer_backward_f32 (dP over P, d relu_biases, d linear_weights) before K1^T of dP and Adam.

Every other model family trains through the torch-autograd mirror of the reference's graph functions
(TensorRec._training_losses); TENSORREC_B200_TRAIN_PATH=torch forces that path."""
import collections
import ctypes
import os

import numpy as np
import scipy.sparse as sp
import torch

from . import _lib, kernels
from .kernels import _p, _stream

TRAIN_PATH = os.environ.get('TENSORREC_B200_TRAIN_PATH', 'auto')       # 'auto' | 'torch'
TRAIN_DTYPE = os.environ.get('TENSORREC_B200_TRAIN_DTYPE', 'f32')      # 'f32' | 'bf16' (representations only)

ADAM_BETA1, ADAM_BETA2, ADAM_EPSILON = 0.9, 0.999, 1e-8                # tf.train.AdamOptimizer defaults


def sample_items_device(n_items, n_users, n_sampled_items, replace, seed, step, device):
    """int32 [n_users, n_sampled_items] on the device (trk_sample_items)."""
    lib = kernels.require_cuda()
    if (not replace) and n_sampled_items > n_items:
        raise ValueError("Cannot take a larger sample than population when 'replace=False'")
    out = torch.empty((int(n_users), int(n_sampled_items)), dtype=torch.int32, device=device)
    rc = lib.trk_sample_items(int(n_users), int(n_items), int(n_sampled_items), 1 if replace else 0,
                              ctypes.c_uint64(int(seed) & (2 ** 64 - 1)), ctypes.c_uint32(int(step) & 0xffffffff),
                              _p(out), _stream())
    _lib.check(rc, 'trk_sample_items')
    return out


def sample_items_host(n_items, n_users, n_sampled_items, replace, seed, step):
    """The same sample computed on the host from the same Philox stream (trk_sample_stream_u64): the statement of what
    the device kernel must produce, used by the tests.  Pure Python: small sizes only."""
    lib = _lib.load()
    out = np.empty((n_users, n_sampled_items), dtype=np.int32)
    for u in range(n_users):
        chosen = []
        for j in range(n_sampled_items):
            r = int(lib.trk_sample_stream_u64(ctypes.c_uint64(seed), ctypes.c_uint32(step), ctypes.c_uint32(u),
                                              ctypes.c_uint32(j)))
            if replace:
                chosen.append((r * n_items) >> 64)
            else:
                top = n_items - n_sampled_items + j            # Floyd: t uniform in [0, top]
                t = (r * (top + 1)) >> 64
                chosen.append(top if t in chosen else t)
        out[u] = chosen
    return out


MAX_SAMPLED = 2048                 # n_sampled_items the fused step covers
MAX_D_ONE_TASTE = 512              # n_components with one taste
MAX_D_TASTES = 128                 # n_components with several tastes
MAX_TASTES = 8                     # n_tastes without attention
MAX_TASTES_ATTENTION = 4           # n_tastes with attention

MAX_HIDDEN = 2048                  # relu_size of a ReLURepresentationGraph (trk_relu_layer_*_f32)

# The form of the fused step that trains a model: pair 'dot' (dot and cosine) or 'euclidean'; how many times the user,
# attention and item rows are L2-normalised (NormalizedLinearRepresentationGraph once, cosine once more); d_pad the
# operand width (n_components rounded up to a multiple of 4).
# loss: 'wmrb' (WMRB / BalancedWMRB on trk_wmrb_step_tastes), or 'rmse' / 'separation' (trk_serial_loss_step).
# hidden: the hidden layer width of the user, attention and item graphs when they are ReLURepresentationGraph (relu_size
# rounded up to a multiple of 8), 0 for a Linear / NormalizedLinear graph (relu_step_plan; DESIGN §3.14).
StepForm = collections.namedtuple('StepForm', ['pair', 'n_tastes', 'attention', 'normalize_user', 'normalize_attn',
                                               'normalize_item', 'd_pad', 'loss', 'hidden'], defaults=((0, 0, 0),))
SERIAL_LOSS_KIND = {'rmse': 0, 'separation': 1}          # trk_serial_loss_step's loss_kind


def step_plan(model, n_sampled_items=None):
    """The StepForm of the fused training step for this model, or None when it trains on the torch path: loss 'wmrb'
    for a WMRB / BalancedWMRB loss with n_sampled_items <= 2048, 'rmse' / 'separation' for an RMSELossGraph /
    SeparationLossGraph (nothing sampled: no n_sampled_items limit); dot, cosine or Euclidean prediction; Linear or
    NormalizedLinear user, item and attention graphs (or no attention); n_components <= 512 for one taste, <= 128 with
    n_tastes <= 8 (<= 4 with attention)."""
    return _plan(model, n_sampled_items, relu=False)


def relu_step_plan(model, n_sampled_items=None):
    """The StepForm of the fused training step for a model with at least one ReLURepresentationGraph whose other
    graphs are Linear or NormalizedLinear, or None: step_plan's losses, predictions and limits, and relu_size <= 2048.
    A ReLU side adds its hidden layer (trk_relu_layer_forward_f32 / _backward_f32) between K1 and the loss kernels;
    cosine prediction normalises its output once.  step_plan answers None for every model this planner covers."""
    return _plan(model, n_sampled_items, relu=True)


def _relu_hidden(model, graph):
    """relu_size of a ReLURepresentationGraph (default 4 n_components), 0 for any other graph."""
    from .representation_graphs import ReLURepresentationGraph
    if type(graph) is not ReLURepresentationGraph:
        return 0
    return 4 * int(model.n_components) if graph.relu_size is None else int(graph.relu_size)


def _plan(model, n_sampled_items, relu):
    from .loss_graphs import BalancedWMRBLossGraph, RMSELossGraph, SeparationLossGraph, WMRBLossGraph
    from .prediction_graphs import (CosineSimilarityPredictionGraph, DotProductPredictionGraph,
                                    EuclideanSimilarityPredictionGraph)
    from .representation_graphs import (LinearRepresentationGraph, NormalizedLinearRepresentationGraph,
                                        ReLURepresentationGraph)
    loss = {WMRBLossGraph: 'wmrb', BalancedWMRBLossGraph: 'wmrb', RMSELossGraph: 'rmse',
            SeparationLossGraph: 'separation'}.get(type(model.loss_graph_factory))
    if TRAIN_PATH == 'torch' or loss is None:
        return None
    if loss == 'wmrb' and n_sampled_items is not None and n_sampled_items > MAX_SAMPLED:
        return None
    pred = type(model.prediction_graph_factory)
    if pred not in (DotProductPredictionGraph, CosineSimilarityPredictionGraph, EuclideanSimilarityPredictionGraph):
        return None
    attention = model.attention_graph_factory is not None
    graphs = [model.user_repr_graph_factory, model.item_repr_graph_factory]
    if attention:
        graphs.append(model.attention_graph_factory)
    kinds = (LinearRepresentationGraph, NormalizedLinearRepresentationGraph) + ((ReLURepresentationGraph,) if relu else ())
    if any(type(graph) not in kinds for graph in graphs):
        return None
    if relu and not any(type(graph) is ReLURepresentationGraph for graph in graphs):
        return None
    d, nt = int(model.n_components), int(model.n_tastes)
    if nt == 1:
        if attention or not 1 <= d <= MAX_D_ONE_TASTE:
            return None
    elif d > MAX_D_TASTES or nt > (MAX_TASTES_ATTENTION if attention else MAX_TASTES):
        return None
    hidden = [_relu_hidden(model, graph) for graph in graphs]
    if any(type(graph) is ReLURepresentationGraph and not 1 <= h <= MAX_HIDDEN for graph, h in zip(graphs, hidden)):
        return None
    cos = 1 if pred is CosineSimilarityPredictionGraph else 0

    def n_norm(graph):
        return (1 if type(graph) is NormalizedLinearRepresentationGraph else 0) + cos

    form = StepForm(pair='euclidean' if pred is EuclideanSimilarityPredictionGraph else 'dot', n_tastes=nt,
                    attention=attention, normalize_user=n_norm(model.user_repr_graph_factory),
                    normalize_attn=n_norm(model.attention_graph_factory) if attention else 0,
                    normalize_item=n_norm(model.item_repr_graph_factory), d_pad=(d + 3) // 4 * 4, loss=loss)
    if relu:
        pad8 = [(h + 7) // 8 * 8 for h in hidden]
        form = form._replace(hidden=(pad8[0], pad8[2] if attention else 0, pad8[1]))
    return form


def check_step_inputs(interactions_shape, n_users, n_items, n_sampled_items, samples=None):
    """Raises ValueError unless the interactions are (n_users, n_items) and the caller's samples, if any, are int32
    [n_users, n_sampled_items] item ids in [0, n_items): the step's kernels index item rows with both, unchecked."""
    if tuple(int(x) for x in interactions_shape) != (int(n_users), int(n_items)):
        raise ValueError('interactions have shape {} but the feature matrices give {} users x {} items'.format(
            tuple(interactions_shape), n_users, n_items))
    if samples is None:
        return
    if samples.dtype not in (torch.int32, np.int32):
        raise ValueError('samples must be int32, got {}'.format(samples.dtype))
    if tuple(samples.shape) != (int(n_users), int(n_sampled_items)):
        raise ValueError('samples have shape {} but the step needs ({}, {})'.format(tuple(samples.shape), n_users,
                                                                                 n_sampled_items))
    if samples.numel() if isinstance(samples, torch.Tensor) else samples.size:
        lo, hi = int(samples.min()), int(samples.max())
        if lo < 0 or hi >= n_items:
            raise ValueError('samples hold item ids in [{}, {}] outside [0, {})'.format(lo, hi, n_items))


class WmrbStep(object):
    """State of the kernel training path of one model: Adam moments per weight, the step counter of the sampler's
    stream and of Adam's bias correction."""

    def __init__(self, model, device, seed=None, bf16=None):
        self.model, self.device = model, device
        self.seed = int(np.random.SeedSequence().generate_state(2, dtype=np.uint32).view(np.uint64)[0]) \
            if seed is None else int(seed)
        self.bf16 = (TRAIN_DTYPE == 'bf16') if bf16 is None else bool(bf16)
        self.t = 0
        self.beta_powers = (np.float32(1.0), np.float32(1.0))    # beta1^t, beta2^t as float32 variables (TensorFlow)
        self.moments = {}            # weight name -> (m, v)
        self.last = {}
        self.marks = None            # bench.py: list that receives (phase name, CUDA event) pairs of a step

    def _mark(self, name):
        if self.marks is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self.marks.append((name, e))

    # -- weights ------------------------------------------------------------------------------------------
    def _weight(self, name, shape, init):
        store = self.model._variables
        if name not in store:
            store[name] = init().to(self.device).requires_grad_(True)
        w = store[name]
        if w.device != self.device:
            w = w.detach().to(self.device).requires_grad_(True)
            store[name] = w
        if tuple(w.shape) != tuple(shape):
            raise ValueError('weight {!r} has shape {} but the inputs need {}'.format(name, tuple(w.shape), shape))
        return w

    def _weights(self, n_user_features, n_item_features, form):
        """The weights in the creation order of the reference's graph: item, then user_<t> (and attn_<t>) per taste,
        then the feature biases.  A Linear / NormalizedLinear side has linear_weights_<end> [n_features, d]; a ReLU side
        has relu_weights_<end> [n_features, H], relu_biases_<end> [1, H] and linear_weights_<end> [H, d]
        (representation_graphs.py: ReLURepresentationGraph), H = relu_size."""
        d = self.model.n_components

        def normal_rows(n):       # representation_graphs.py:35-36: random_normal rows, L2-normalised
            def init():
                w = torch.randn(n, d, dtype=torch.float32)
                return w * torch.rsqrt(torch.clamp((w * w).sum(dim=1, keepdim=True), min=1e-12))
            return init

        def normal(shape):        # ReLURepresentationGraph: random_normal, stddev .5
            return lambda: torch.randn(*shape, dtype=torch.float32) * .5

        names, ws = [], {}

        def side(end, graph, n_features):
            h = _relu_hidden(self.model, graph)
            if h:
                specs = [('relu_weights_' + end, (n_features, h), normal((n_features, h))),
                         ('relu_biases_' + end, (1, h), lambda: torch.zeros(1, h, dtype=torch.float32)),
                         ('linear_weights_' + end, (h, d), normal((h, d)))]
            else:
                specs = [('linear_weights_' + end, (n_features, d), normal_rows(n_features))]
            for name, shape, init in specs:
                ws[name] = self._weight(name, shape, init)
                names.append(name)

        side('item', self.model.item_repr_graph_factory, n_item_features)
        for t in range(self.model.n_tastes):
            side('user_{}'.format(t), self.model.user_repr_graph_factory, n_user_features)
            if self.model.attention_graph_factory is not None:
                side('attn_{}'.format(t), self.model.attention_graph_factory, n_user_features)
        if self.model.biased:         # recommendation_graphs.py:11: zeros
            for name, n in (('feature_biases_user', n_user_features), ('feature_biases_item', n_item_features)):
                ws[name] = self._weight(name, (n, 1), lambda n=n: torch.zeros(n, 1, dtype=torch.float32))
                names.append(name)
        return names, ws

    # -- one step -----------------------------------------------------------------------------------------
    def step(self, interactions_in, user_in, item_in, n_sampled_items, learning_rate, l2, samples=None):
        """One Adam step on sum(WMRB loss) + l2 * sum_w 0.5 |w|^2.  `l2` is the coefficient of the L2 term in the
        SUMMED loss (the reference adds alpha * reg to every element of its loss vector, tensorrec.py:488, so it is
        n_positive_interactions * batched_alpha).  Returns the device tensors of the step (loss, pred_serial).

        For an RMSE / Separation model (step_plan's loss 'rmse' / 'separation') the loss is a scalar: `l2` is
        batched_alpha itself, the returned loss is a 1-element tensor, and n_sampled_items and samples are not used."""
        lib = kernels.require_cuda()
        form = step_plan(self.model) or relu_step_plan(self.model)
        if form is None:
            raise ValueError('the fused training step does not cover this model (train_kernels.step_plan, '
                             'relu_step_plan)')
        wmrb = form.loss == 'wmrb'
        if not wmrb:
            samples = None
        dev, d, dp = self.device, self.model.n_components, form.d_pad
        n_users, n_items = user_in.shape[0], item_in.shape[0]
        check_step_inputs(interactions_in.shape, n_users, n_items, n_sampled_items, samples)
        ucsr, icsr = user_in.device_csr(dev), item_in.device_csr(dev)
        ucsr_t, icsr_t = user_in.device_csr_t(dev), item_in.device_csr_t(dev)
        inter = interactions_in.device_csr(dev)
        if not wmrb and inter.nnz >= 2 ** 31:
            raise ValueError('{} interactions exceed the step\'s int32 indexing'.format(inter.nnz))
        names, ws = self._weights(user_in.shape[1], item_in.shape[1], form)
        # the user operand: taste planes, then attention planes, [n_rows, n_users, d_pad]; (end, normalisations, H)
        user_ops = [('user_{}'.format(t), form.normalize_user, form.hidden[0]) for t in range(form.n_tastes)]
        if form.attention:
            user_ops += [('attn_{}'.format(t), form.normalize_attn, form.hidden[1]) for t in range(form.n_tastes)]
        relu_sides = {}              # end -> (pre-activations P [rows, H_pad], b, W2 padded) of a ReLU side

        def operand(csr, end, n_norm, hp, out):
            """K1 of one side into `out`, or for a ReLU side into its pre-activations P (the layer runs after every
            K1).  Returns K1's raw rows when they are normalised (kept for the backward pass)."""
            if hp:
                h = ws['relu_weights_' + end].shape[1]
                w1 = ws['relu_weights_' + end].detach()
                b = ws['relu_biases_' + end].detach().reshape(-1)
                w2 = ws['linear_weights_' + end].detach()
                if hp != h or dp != d:     # zero units and columns change no prediction, norm or gradient
                    w1 = torch.nn.functional.pad(w1, (0, hp - h))
                    b = torch.nn.functional.pad(b, (0, hp - h))
                    w2 = torch.nn.functional.pad(w2, (0, dp - d, 0, hp - h))
                relu_sides[end] = (kernels.gather_reduce(csr, w1, want_f32=True)[0], b, w2)
                return None
            w = ws['linear_weights_' + end].detach()
            if dp != d:                # zero columns change no prediction, norm or gradient
                w = torch.nn.functional.pad(w, (0, dp - d))
            if n_norm == 0:
                kernels.gather_reduce(csr, w, want_f32=True, out_f32=out)
                return None
            raw, _, _ = kernels.gather_reduce(csr, w, want_f32=True)
            _lib.check(lib.trk_l2_normalize_rows_step_f32(_p(raw), raw.shape[0], dp, n_norm, _p(out), None, _stream()),
                       'trk_l2_normalize_rows_step_f32')
            return raw

        def layer(end, n_norm, out):
            """The hidden layer of a ReLU side into `out` (normalised for cosine: its raw rows are returned)."""
            pre, b, w2 = relu_sides[end]
            raw = out if n_norm == 0 else torch.empty(out.shape, dtype=torch.float32, device=dev)
            _lib.check(lib.trk_relu_layer_forward_f32(_p(pre), _p(b), _p(w2), pre.shape[0], pre.shape[1], dp, _p(raw),
                                                      _stream()), 'trk_relu_layer_forward_f32')
            if n_norm == 0:
                return None
            _lib.check(lib.trk_l2_normalize_rows_step_f32(_p(raw), raw.shape[0], dp, n_norm, _p(out), None, _stream()),
                       'trk_l2_normalize_rows_step_f32')
            return raw

        self._mark('start')
        # forward: representations and projected biases (K1)
        user_repr = torch.empty((len(user_ops), n_users, dp), dtype=torch.float32, device=dev)
        item_repr = torch.empty((n_items, dp), dtype=torch.float32, device=dev)
        item_raw = operand(icsr, 'item', form.normalize_item, form.hidden[2], item_repr)
        user_raw = [operand(ucsr, end, n_norm, hp, user_repr[r]) for r, (end, n_norm, hp) in enumerate(user_ops)]
        ub = ib = None
        if self.model.biased:
            ub = kernels.project_biases(ucsr, ws['feature_biases_user'].detach().reshape(-1))
            ib = kernels.project_biases(icsr, ws['feature_biases_item'].detach().reshape(-1))
        if relu_sides:
            self._mark('representations')
            # the hidden layers of the ReLU sides (trk_relu_layer_forward_f32), then their normalisation
            if form.hidden[2]:
                item_raw = layer('item', form.normalize_item, item_repr)
            for r, (end, n_norm, hp) in enumerate(user_ops):
                if hp:
                    user_raw[r] = layer(end, n_norm, user_repr[r])
        repr_u, repr_i = user_repr, item_repr
        if self.bf16:
            repr_u = torch.empty(user_repr.shape, dtype=torch.bfloat16, device=dev)
            repr_i = torch.empty(item_repr.shape, dtype=torch.bfloat16, device=dev)
            _lib.check(lib.trk_f32_to_bf16(_p(user_repr), user_repr.numel(), _p(repr_u), _stream()), 'trk_f32_to_bf16')
            _lib.check(lib.trk_f32_to_bf16(_p(item_repr), item_repr.numel(), _p(repr_i), _stream()), 'trk_f32_to_bf16')

        self._mark('layer_forward' if relu_sides else 'representations')
        # the loss and the gradient with respect to the operands
        if wmrb:
            samples, loss, pred, (d_user_repr, d_item_repr, d_ub, d_ib) = self._wmrb_loss(
                lib, form, interactions_in, inter, repr_u, repr_i, ub, ib, n_sampled_items, samples)
        else:
            loss, pred, (d_user_repr, d_item_repr, d_ub, d_ib) = self._serial_loss(lib, form, inter, repr_u, repr_i,
                                                                                   ub, ib)

        # backward through the normalisations and the ReLU layers, then through the sparse x dense products: K1 on
        # the transposed CSR
        grads = {}

        def layer_grad(end, raw, n_norm, d_rows):
            """d_rows -> the gradient K1^T takes: through the normalisations, and for a ReLU side through its layer
            (trk_relu_layer_backward_f32 replaces P by dP and gives the gradients of relu_biases and linear_weights)."""
            if raw is not None:
                _lib.check(lib.trk_l2_normalize_rows_step_f32(_p(raw), raw.shape[0], dp, n_norm, None, _p(d_rows),
                                                              _stream()), 'trk_l2_normalize_rows_step_f32')
            if end not in relu_sides:
                return d_rows
            pre, b, w2 = relu_sides[end]
            rows, hp = pre.shape
            h = ws['relu_biases_' + end].shape[1]
            ws_bytes = int(lib.trk_relu_layer_workspace_bytes(rows, hp, dp))
            workspace = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
            d_b = torch.empty((hp,), dtype=torch.float32, device=dev)
            d_w2 = torch.empty((hp, dp), dtype=torch.float32, device=dev)
            _lib.check(lib.trk_relu_layer_backward_f32(_p(pre), _p(b), _p(w2), _p(d_rows), rows, hp, dp, _p(d_b),
                                                       _p(d_w2), _p(workspace), ws_bytes, _stream()),
                       'trk_relu_layer_backward_f32')
            grads['relu_biases_' + end] = d_b[:h].reshape(1, h).contiguous()
            grads['linear_weights_' + end] = d_w2 if (hp, dp) == (h, d) else d_w2[:h, :d].contiguous()
            return pre

        def weight_grad(csr_t, end, d_rows):
            name = ('relu_weights_' if end in relu_sides else 'linear_weights_') + end
            g = kernels.gather_reduce(csr_t, d_rows, want_f32=True)[0]
            width = ws[name].shape[1]
            grads[name] = g if g.shape[1] == width else g[:, :width].contiguous()

        sides = [(icsr_t, 'item', layer_grad('item', item_raw, form.normalize_item, d_item_repr))]
        for r, (end, n_norm, _) in enumerate(user_ops):
            sides.append((ucsr_t, end, layer_grad(end, user_raw[r], n_norm, d_user_repr[r])))
        if relu_sides:
            self._mark('layer_backward')
        for csr_t, end, d_rows in sides:
            weight_grad(csr_t, end, d_rows)
        if self.model.biased:
            grads['feature_biases_user'] = kernels.project_biases(ucsr_t, d_ub)
            grads['feature_biases_item'] = kernels.project_biases(icsr_t, d_ib)
        self.last = {'loss': loss, 'pred_serial': pred, 'grads': grads, 'samples': samples, 'inter_val': inter.val}

        self._mark('weight_gradients')
        # Adam
        self.t += 1
        f32 = np.float32
        self.beta_powers = (f32(self.beta_powers[0] * f32(ADAM_BETA1)), f32(self.beta_powers[1] * f32(ADAM_BETA2)))
        lr_t = float(f32(learning_rate) * np.sqrt(f32(1.0) - self.beta_powers[1]) / (f32(1.0) - self.beta_powers[0]))
        for name in names:
            w = ws[name]
            if name not in self.moments:
                self.moments[name] = (torch.zeros_like(w, requires_grad=False), torch.zeros_like(w, requires_grad=False))
            m, v = self.moments[name]
            rc = lib.trk_adam_step_f32(_p(w), _p(grads[name]), _p(m), _p(v), w.numel(), ctypes.c_float(lr_t),
                                       ctypes.c_float(ADAM_BETA1), ctypes.c_float(ADAM_BETA2),
                                       ctypes.c_float(ADAM_EPSILON), ctypes.c_float(l2), _stream())
            _lib.check(rc, 'trk_adam_step_f32')
        self._mark('adam')
        return loss, pred

    def _operand_grads(self, repr_u, repr_i):
        """(d user rows, d item rows, d user biases, d item biases) for the loss kernels: the user side is written,
        the item side added to (zeroed here)."""
        dev, biased, n_users, n_items = self.device, self.model.biased, repr_u.shape[1], repr_i.shape[0]
        return (torch.empty(repr_u.shape, dtype=torch.float32, device=dev),
                torch.zeros(repr_i.shape, dtype=torch.float32, device=dev),
                torch.empty((n_users,), dtype=torch.float32, device=dev) if biased else None,
                torch.zeros((n_items,), dtype=torch.float32, device=dev) if biased else None)

    def _wmrb_loss(self, lib, form, interactions_in, inter, repr_u, repr_i, ub, ib, n_sampled_items, samples):
        """trk_sample_items (unless the caller gives the samples) and trk_wmrb_step_tastes: the samples, the loss
        [nnz] (0 for the non-positive interactions), pred_serial and the operand gradients of a WMRB / BalancedWMRB
        step."""
        from .loss_graphs import BalancedWMRBLossGraph
        dev, n_users, n_items, nnz = self.device, repr_u.shape[1], repr_i.shape[0], inter.nnz
        if samples is None:
            samples = sample_items_device(n_items, n_users, n_sampled_items,
                                          self.model.loss_graph_factory.is_sampled_with_replacement, self.seed, self.t,
                                          dev)
        weight_sum = None
        if type(self.model.loss_graph_factory) is BalancedWMRBLossGraph:
            weight_sum = interactions_in.positive_item_sums(dev)

        self._mark('sampler')
        loss = torch.empty((nnz,), dtype=torch.float32, device=dev)
        pred = torch.empty((nnz,), dtype=torch.float32, device=dev)
        coef = torch.empty((nnz,), dtype=torch.float32, device=dev)
        grads = d_user_repr, d_item_repr, d_ub, d_ib = self._operand_grads(repr_u, repr_i)
        rc = lib.trk_wmrb_step_tastes(_p(repr_u), _p(repr_i), 1 if self.bf16 else 0, form.n_tastes,
                                      1 if form.attention else 0, 1 if form.pair == 'euclidean' else 0, _p(ub), _p(ib),
                                      _p(inter.indptr), _p(inter.col), _p(inter.val), _p(weight_sum), _p(samples),
                                      n_users, n_items, form.d_pad, int(samples.shape[1]), _p(loss), _p(pred), _p(coef),
                                      _p(d_user_repr), _p(d_ub), _p(d_item_repr), _p(d_ib), _stream())
        _lib.check(rc, 'trk_wmrb_step_tastes')
        self._mark('wmrb_step')
        return samples, loss, pred, grads

    def _serial_loss(self, lib, form, inter, repr_u, repr_i, ub, ib):
        """trk_serial_loss_step: the scalar loss [1], pred_serial and the operand gradients of an RMSE / Separation
        step.  An interaction-free batch launches no kernel (loss NaN, zero gradients), as the mean of nothing gives."""
        dev, n_users, n_items, nnz = self.device, repr_u.shape[1], repr_i.shape[0], inter.nnz
        loss = torch.empty((1,), dtype=torch.float32, device=dev)
        pred = torch.empty((nnz,), dtype=torch.float32, device=dev)
        grads = d_user_repr, d_item_repr, d_ub, d_ib = self._operand_grads(repr_u, repr_i)
        ws_bytes = int(lib.trk_serial_loss_workspace_bytes(nnz))
        workspace = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        rc = lib.trk_serial_loss_step(SERIAL_LOSS_KIND[form.loss], _p(repr_u), _p(repr_i), 1 if self.bf16 else 0,
                                      form.n_tastes, 1 if form.attention else 0, 1 if form.pair == 'euclidean' else 0,
                                      _p(ub), _p(ib), _p(inter.indptr), _p(inter.col), _p(inter.val), n_users, n_items,
                                      form.d_pad, nnz, _p(loss), _p(pred), _p(d_user_repr), _p(d_ub), _p(d_item_repr),
                                      _p(d_ib), _p(workspace), ws_bytes, _stream())
        _lib.check(rc, 'trk_serial_loss_step')
        self._mark('serial_loss_step')
        return loss, pred, grads


def positive_item_sums(matrix, n_items):
    """BalancedWMRBLossGraph's listening_sum_per_item (tensorrec/loss_graphs.py:201): sum of the positive interaction
    values per item, float32 (host side, once per interaction matrix)."""
    coo = matrix if isinstance(matrix, sp.coo_matrix) else sp.coo_matrix(matrix)
    data = coo.data.astype(np.float32)
    mask = data > 0.0
    out = np.zeros(n_items, dtype=np.float32)
    np.add.at(out, coo.col[mask], data[mask])
    return out
