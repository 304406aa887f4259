"""The TensorRec model class: same constructor, fit / fit_partial / predict / predict_rank / predict_* / save / load
signatures and error behaviour as tensorrec/tensorrec.py, with the predict / predict_rank hot path evaluated by
hand-written sm_90a kernels through the C ABI (include/tensorrec_b200.h):

    sparse features --K1 trk_csr_gather_reduce_f32--> representations (fp32 and/or split-fp16 operand)
                    --trk_csr_project_biases_f32--> user / item biases
    predict():       K2 trk_score_dense_(euclid_)f16x3 (wgmma) or trk_score_f32 (exact fp32, any shape) -> [U, I] f32
    predict_rank():  ... + K3 trk_rank_full                                                      -> [U, I] int32
    predict_rank(k): K2+K3 fused trk_score_topk_f16x3 + trk_topk_merge (+ one NCCL all-gather when the item axis is
                     sharded over GPUs)                                                           -> top-k ids, scores

Training (fit) is outside that path: it is a torch-autograd step over the plugin graphs' differentiable forms
(SURVEY.md 8f rank 1)."""
import collections
import logging
import os
import pickle
from itertools import cycle

import numpy as np
import scipy.sparse as sp
import torch

from . import kernels
from .errors import (
    ModelNotBiasedException, ModelNotFitException, ModelWithoutAttentionException, BatchNonSparseInputException
)
from .input_utils import SparseInput, TensorRecDataset
from .loss_graphs import AbstractLossGraph, RMSELossGraph
from .prediction_graphs import (
    AbstractPredictionGraph, DotProductPredictionGraph, CosineSimilarityPredictionGraph,
    EuclideanSimilarityPredictionGraph
)
from .recommendation_graphs import (
    split_sparse_tensor_indices, bias_prediction_dense, bias_prediction_serial, densify_sampled_item_predictions,
    collapse_mixture_of_tastes
)
from .representation_graphs import (
    AbstractRepresentationGraph, LinearRepresentationGraph, NormalizedLinearRepresentationGraph
)
from .session_management import get_session, variable_scope, get_variable, name_scope
from .util import sample_items, calculate_batched_alpha

TopK = collections.namedtuple('TopK', ['items', 'scores'])
TopK.__doc__ = """predict_rank(k=...) result: items int32 [n_users, k] = the item ids holding reference ranks 1..k (in
rank order), scores float32 [n_users, k].  Slots beyond n_items hold id 2**31-1 / score -inf."""

_BUILTIN_REPR = (LinearRepresentationGraph, NormalizedLinearRepresentationGraph)
_BUILTIN_PRED = (DotProductPredictionGraph, CosineSimilarityPredictionGraph, EuclideanSimilarityPredictionGraph)

# 'auto': tensor cores whenever the shape allows; 'exact': always the fp32 CUDA-core kernel; 'tensor': insist.
SCORE_PATH = os.environ.get('TENSORREC_B200_SCORE_PATH', 'auto')
# predict_rank(k) on the tensor path: 'auto' = 1-pass filter + exact fp32 re-scoring when k allows, 'exact' = always the
# 3-pass split-product kernel
TOPK_PATH = os.environ.get('TENSORREC_B200_TOPK_PATH', 'auto')

# The wide form of the filter serves 32 < k <= WIDE_MAX_K on catalogues of at least WIDE_MIN_ITEMS items; below that,
# scoring the catalogue densely and ranking it costs less than a sweep (see README, "Large k").
WIDE_MAX_K = 1024
WIDE_MIN_ITEMS = 4096
# Euclidean user x item models take the exact 3-pass kernel for k <= 32 on catalogues of at least EUCLIDEAN_MIN_ITEMS
# items.  The fused route was faster at every measured catalogue size, from 1024 items up (see README, "Euclidean
# models"); smaller catalogues stay on dense scoring and ranking.
EUCLIDEAN_MIN_ITEMS = 1024
# Mixture-of-tastes models with an attention graph take the taste-collapsing exact kernel for k <= 32 on catalogues of
# at least ATTENTION_MIN_ITEMS items (see README, "Mixtures of tastes and attention").
ATTENTION_MIN_ITEMS = 1024
# Euclidean and attention models take the exact kernel's wide mode for 32 < k <= WIDE_MAX_K on catalogues of at least
# EXACT_WIDE_MIN_ITEMS items; below that, dense scoring and ranking (see README, "Large k for Euclidean and attention
# models").
EXACT_WIDE_MIN_ITEMS = 4096
# predict_rank_at counts on the exact kernel's counting mode (route 'exact3_count') on catalogues of at least
# RANK_AT_MIN_ITEMS items; below that, dense scoring and ranking of the user blocks (see README, "Ranks of listed
# pairs").
RANK_AT_MIN_ITEMS = 2048
# Euclidean mixtures of tastes with attention count from RANK_AT_EUCLID_ATTENTION_MIN_ITEMS items: the capture and the
# counting sweep each pay 2T roots and the softmax per pair, which costs more than one dense sweep and the sort on smaller
# catalogues (see README, "Euclidean mixtures of tastes").
RANK_AT_EUCLID_ATTENTION_MIN_ITEMS = 16384
# predict_at scores on the exact kernel's pairs mode (route 'exact3_pairs') on catalogues of at least
# PREDICT_AT_MIN_ITEMS items; below that, dense scoring of the user blocks gathered at the pairs is faster, as the pairs
# mode pays its host planner per pair (see README, "Scores of listed pairs").
PREDICT_AT_MIN_ITEMS = 1 << 20


def rank_at_route(n_items, tensor_scored, euclid_attention=False):
    """The route of a predict_rank_at call: 'exact3_count' when predict() scores the model on the exact tensor-core
    kernel (tensor_scored: TensorRec._tensor_score_form() is not None) and the catalogue has at least RANK_AT_MIN_ITEMS
    items (RANK_AT_EUCLID_ATTENTION_MIN_ITEMS for a Euclidean mixture of tastes with attention), 'dense+rank'
    otherwise."""
    floor = RANK_AT_EUCLID_ATTENTION_MIN_ITEMS if euclid_attention else RANK_AT_MIN_ITEMS
    return 'exact3_count' if tensor_scored and n_items >= floor else 'dense+rank'


def predict_at_route(n_items, tensor_scored):
    """The route of a predict_at call: 'exact3_pairs', the exact kernel's pairs mode, when predict() scores the model
    on the exact tensor-core kernel (tensor_scored: TensorRec._tensor_score_form() is not None) and the catalogue has at
    least PREDICT_AT_MIN_ITEMS items, 'dense+gather' (dense scores of the user blocks, gathered at the pairs)
    otherwise."""
    return 'exact3_pairs' if tensor_scored and n_items >= PREDICT_AT_MIN_ITEMS else 'dense+gather'


def rank_at_blocks(indptr, unit, max_rows, max_pairs):
    """User blocks [(u0, u1)] of a predict_rank_at call over the rows of the pair CSR indptr: every block starts at a
    multiple of `unit` (the kernel's user block, so every user keeps its accumulator row), has at most max_rows rows (a
    positive multiple of unit) and at most max_pairs pairs unless one unit alone holds more."""
    n = len(indptr) - 1
    indptr = np.asarray(indptr, dtype=np.int64)
    blocks, u0 = [], 0
    while u0 < n:
        u1 = min(n, u0 + max_rows)
        fit = int(np.searchsorted(indptr, indptr[u0] + max_pairs, side='right')) - 1   # last row end within max_pairs
        if fit < u1:
            u1 = min(n, max(u0 + unit, fit // unit * unit))
        blocks.append((u0, u1))
        u0 = u1
    return blocks


def topk_route(k, n_items, model_ok, single_taste, filter_max_k, exact_max_k, sharded=False, euclidean=False,
               attention=False, merge_max_k=32, exact_wide_max_k=0):
    """The route of a top-k call -- 'filter', 'exact3', 'wide', 'exact3_wide' or 'dense+rank' -- from k, the catalogue
    size and the
    model alone.  model_ok: the tensor-core kernels evaluate the model (built-in dot / cosine prediction, or any
    built-in similar-items graph, no attention, d_pad <= 128); single_taste: one taste; filter_max_k / exact_max_k:
    the k limits of the filter and of the exact 3-pass kernel; merge_max_k: the largest k whose per-taste lists the
    caller can merge with de-duplication (32: trk_topk_merge alone; WIDE_MAX_K: with trk_topk_merge_dedup_pair on the
    wide route), so a mixture of tastes takes the wide route under the one-taste conditions when k <= merge_max_k.
    sharded: an item-sharded call, where every rank must take the same route (the exchange is collective), so a
    rank's shard size does not decide the wide route.  TOPK_PATH='exact' means "no filter": k > exact_max_k then
    goes to dense+rank.  euclidean: a Euclidean user x item model (model_ok from _euclidean_tensor_ok), which has no
    filter or wide form: 'exact3' for k <= exact_max_k on catalogues of at least EUCLIDEAN_MIN_ITEMS items (any shard
    size in a sharded call), 'dense+rank' otherwise.  attention: a mixture of tastes with an attention graph (model_ok
    from _tastes_tensor_ok, or _euclid_tastes_tensor_ok for Euclidean prediction), whose softmax has no filter or wide form either: the same rule with ATTENTION_MIN_ITEMS.
    merge_max_k does not apply to either.  exact_wide_max_k: the largest k of the exact kernel's wide mode (0: none,
    WIDE_MAX_K: trk_score_topk_wide_*); Euclidean and attention models with exact_max_k < k <= exact_wide_max_k take
    'exact3_wide' on catalogues of at least EXACT_WIDE_MIN_ITEMS items (any shard size in a sharded call), with one
    taste or several."""
    if not model_ok:
        return 'dense+rank'
    if euclidean or attention:
        if n_items == 0 or k > max(exact_max_k, exact_wide_max_k):
            return 'dense+rank'
        if k > exact_max_k:
            return 'exact3_wide' if sharded or n_items >= EXACT_WIDE_MIN_ITEMS else 'dense+rank'
        min_items = ATTENTION_MIN_ITEMS if attention else EUCLIDEAN_MIN_ITEMS
        return 'exact3' if sharded or n_items >= min_items else 'dense+rank'
    if k <= exact_max_k:
        if n_items == 0:
            return 'dense+rank'
        return 'filter' if TOPK_PATH != 'exact' and k <= filter_max_k else 'exact3'
    if TOPK_PATH == 'exact' or k > WIDE_MAX_K or (not single_taste and k > merge_max_k):
        return 'dense+rank'
    return 'wide' if sharded or n_items >= WIDE_MIN_ITEMS else 'dense+rank'


def _names_argument(method, name):
    """Does `method` declare `name` as an explicit parameter (not just **kwargs)?"""
    import inspect
    try:
        return name in inspect.signature(method).parameters
    except (TypeError, ValueError):
        return True


class _Hook(object):
    """Placeholder stored in the tf_* attributes once the model is built (the reference stores TF nodes there and
    tests `self.tf_prediction is None` to detect an unfitted model, tensorrec.py:654)."""

    def __init__(self, name):
        self.name = name

    def __repr__(self):
        return '<graph hook {}>'.format(self.name)


def _checked_exclude(exclude, n_users, n_items, k, item_id_offset, sharded):
    """Validates predict_top_k's `exclude` (no device work) and returns it as a CSR matrix."""
    if k is None:
        raise ValueError('exclude needs k: exclusion applies to the top-k only, not to full ranks')
    if not sp.issparse(exclude):
        raise ValueError('exclude must be a scipy sparse matrix with one row per user')
    if exclude.shape[0] != n_users:
        raise ValueError('exclude has %d rows but there are %d users' % (exclude.shape[0], n_users))
    if sharded:
        if exclude.shape[1] < int(item_id_offset) + n_items:
            raise ValueError('exclude has %d columns; this shard needs >= item_id_offset + n_items = %d'
                             % (exclude.shape[1], int(item_id_offset) + n_items))
    elif exclude.shape[1] != n_items:
        raise ValueError('exclude has %d columns but there are %d items' % (exclude.shape[1], n_items))
    return exclude if isinstance(exclude, sp.csr_matrix) else sp.csr_matrix(exclude)


def _similar_exclusion_mask(exclude, exclude_self, ids, n_queries, n_items):
    """The excluded (query, item) pairs of predict_similar_items_top_k as a CSR matrix of ones (None = nothing excluded
    at all): the non-zero pairs of `exclude` (duplicates summed first) united with every query's own id when
    exclude_self.  A union of masks, not a sum of values: a -1 entry on the query's own id stays excluded."""
    mask = None
    if exclude is not None:
        mask = exclude.copy()
        mask.sum_duplicates()
        mask.eliminate_zeros()
        mask = sp.csr_matrix((np.ones(mask.nnz, np.float32), mask.indices, mask.indptr), shape=mask.shape)
    if exclude_self:
        own = np.arange(n_queries, dtype=np.int64) if ids is None else ids
        self_mask = sp.csr_matrix((np.ones(n_queries, np.float32), own, np.arange(n_queries + 1)),
                                  shape=(n_queries, n_items))
        mask = self_mask if mask is None else mask.maximum(self_mask)
    return mask


class TensorRec(object):

    def __init__(self,
                 n_components=100,
                 n_tastes=1,
                 user_repr_graph=LinearRepresentationGraph(),
                 item_repr_graph=LinearRepresentationGraph(),
                 attention_graph=None,
                 prediction_graph=DotProductPredictionGraph(),
                 loss_graph=RMSELossGraph(),
                 biased=True,):
        """A TensorRec recommendation model (arguments as tensorrec/tensorrec.py:28-61)."""
        # Arg Check (tensorrec.py:69-88)
        if (n_components is None) or (n_tastes is None) or (user_repr_graph is None) or (item_repr_graph is None) \
                or (prediction_graph is None) or (loss_graph is None):
            raise ValueError("All arguments to TensorRec() must be non-None")
        if n_components < 1:
            raise ValueError("n_components must be >= 1")
        if n_tastes < 1:
            raise ValueError("n_tastes must be >= 1")
        if not isinstance(user_repr_graph, AbstractRepresentationGraph):
            raise ValueError("user_repr_graph must inherit AbstractRepresentationGraph")
        if not isinstance(item_repr_graph, AbstractRepresentationGraph):
            raise ValueError("item_repr_graph must inherit AbstractRepresentationGraph")
        if not isinstance(prediction_graph, AbstractPredictionGraph):
            raise ValueError("prediction_graph must inherit AbstractPredictionGraph")
        if not isinstance(loss_graph, AbstractLossGraph):
            raise ValueError("loss_graph must inherit AbstractLossGraph")
        if attention_graph is not None:
            if not isinstance(attention_graph, AbstractRepresentationGraph):
                raise ValueError("attention_graph must be None or inherit AbstractRepresentationGraph")
            if n_tastes == 1:
                raise ValueError("attention_graph must be None if n_tastes == 1")

        self.n_components = n_components
        self.n_tastes = n_tastes
        self.user_repr_graph_factory = user_repr_graph
        self.item_repr_graph_factory = item_repr_graph
        self.attention_graph_factory = attention_graph
        self.prediction_graph_factory = prediction_graph
        self.loss_graph_factory = loss_graph
        self.biased = biased

        # graph hook attribute names, as the reference declares them (tensorrec.py:100-124)
        self.graph_tensor_hook_attr_names = [
            'tf_user_representation', 'tf_item_representation', 'tf_prediction_serial', 'tf_prediction', 'tf_rankings',
            'tf_predict_similar_items', 'tf_rank_similar_items',
            'tf_basic_loss', 'tf_weight_reg_loss', 'tf_loss',
            'tf_learning_rate', 'tf_alpha', 'tf_sample_indices', 'tf_n_sampled_items', 'tf_similar_items_ids',
        ]
        if self.biased:
            self.graph_tensor_hook_attr_names += ['tf_projected_user_biases', 'tf_projected_item_biases']
        if self.attention_graph_factory is not None:
            self.graph_tensor_hook_attr_names += ['tf_user_attention_representation']
        self.graph_operation_hook_attr_names = ['tf_optimizer']
        self.graph_iterator_hook_attr_names = ['tf_user_feature_iterator', 'tf_item_feature_iterator',
                                               'tf_interaction_iterator']
        self._break_graph_hooks()

        self.n_user_features = None
        self.n_item_features = None
        self._variables = collections.OrderedDict()   # name -> trainable tensor (the model's weights)
        self._optimizer = None
        self._optimizer_params = None
        self._stepped = False          # has any training step completed?

    # ------------------------------------------------------------------------------------------------
    # graph hooks (tensorrec.py:136-183).  Only their None-ness carries meaning here.
    # ------------------------------------------------------------------------------------------------
    def _all_hook_names(self):
        return (self.graph_tensor_hook_attr_names + self.graph_operation_hook_attr_names +
                self.graph_iterator_hook_attr_names)

    def _break_graph_hooks(self):
        for name in self._all_hook_names():
            self.__setattr__(name, None)

    def _attach_graph_hooks(self):
        for name in self._all_hook_names():
            self.__setattr__(name, _Hook(name))

    # ------------------------------------------------------------------------------------------------
    # input handling (tensorrec.py:185-263, util.py:34-58)
    # ------------------------------------------------------------------------------------------------
    @staticmethod
    def _inputs_from_raw(raw_input):
        """scipy sparse matrix / TensorRecDataset / list of those -> list of SparseInput."""
        def ok(v):
            return sp.issparse(v) or isinstance(v, (TensorRecDataset, SparseInput))

        def wrap(v):
            return v if isinstance(v, SparseInput) else SparseInput(v)

        if ok(raw_input):
            return [wrap(raw_input)]
        if isinstance(raw_input, list) and len(raw_input) > 0 and all(ok(v) for v in raw_input):
            return [wrap(v) for v in raw_input]
        if isinstance(raw_input, str) or (isinstance(raw_input, list) and raw_input and
                                          all(isinstance(v, str) for v in raw_input)):
            # TFRecord path(s) (tensorrec.py:203-215): every record of every file is one batch
            from .input_utils import create_tensorrec_dataset_from_tfrecord
            paths = [raw_input] if isinstance(raw_input, str) else raw_input
            return [wrap(ds) for path in paths for ds in create_tensorrec_dataset_from_tfrecord(path)]
        raise ValueError('Input must be a scipy sparse matrix, an iterable of scipy sprase matrices, or a TensorFlow '
                         'Dataset')

    @classmethod
    def _single_input(cls, raw_input, what):
        inputs = cls._inputs_from_raw(raw_input)
        if len(inputs) != 1:
            raise ValueError('{} must be one matrix at predict time (got a list of {})'.format(what, len(inputs)))
        return inputs[0]

    def _create_batched_inputs(self, interactions, user_features, item_features, user_batch_size=None):
        if user_batch_size is not None:
            if (not sp.issparse(interactions)) or (not sp.issparse(user_features)):
                raise BatchNonSparseInputException()
            if not isinstance(interactions, sp.csr_matrix):
                interactions = sp.csr_matrix(interactions)
            if not isinstance(user_features, sp.csr_matrix):
                user_features = sp.csr_matrix(user_features)
            n_users = user_features.shape[0]
            interactions_batched, user_features_batched = [], []
            start_batch = 0
            while start_batch < n_users:
                end_batch = min(start_batch + user_batch_size, n_users)
                interactions_batched.append(interactions[start_batch:end_batch])
                user_features_batched.append(user_features[start_batch:end_batch])
                start_batch = end_batch
            interactions, user_features = interactions_batched, user_features_batched

        int_in = self._inputs_from_raw(interactions)
        uf_in = self._inputs_from_raw(user_features)
        if_in = self._inputs_from_raw(item_features)
        if len(int_in) != len(uf_in):
            raise ValueError('Number of batches in user_features and interactions must be equal.')
        if (len(if_in) > 1) and (len(if_in) != len(uf_in)):
            raise ValueError('Number of batches in item_features must be 1 or equal to the number of batches in '
                             'user_features.')
        return [batch for batch in zip(int_in, uf_in, cycle(if_in))]

    # ------------------------------------------------------------------------------------------------
    # training step (define-by-run form of _build_tf_graph, tensorrec.py:270-492)
    # ------------------------------------------------------------------------------------------------
    def _training_losses(self, interactions, user_features, item_features, n_sampled_items, device):
        from .session_management import training_step
        with training_step():
            return self._training_losses_impl(interactions, user_features, item_features, n_sampled_items, device)

    def _training_losses_impl(self, interactions, user_features, item_features, n_sampled_items, device):
        tf_user_features = user_features.torch_sparse(device)
        tf_item_features = item_features.torch_sparse(device)
        tf_interactions = interactions.torch_sparse(device)
        n_users, n_items = user_features.shape[0], item_features.shape[0]
        loss_graph = self.loss_graph_factory
        tf_weights = []

        with name_scope('item'):
            item_repr, item_weights = self.item_repr_graph_factory.connect_representation_graph(
                tf_features=tf_item_features, n_components=self.n_components, n_features=self.n_item_features,
                node_name_ending='item')
        tf_weights.extend(item_weights)

        tf_x_user, tf_x_item = split_sparse_tensor_indices(tf_sparse_tensor=tf_interactions, n_dimensions=2)
        if loss_graph.is_sample_based:
            sample_indices = torch.from_numpy(sample_items(n_items, n_users, n_sampled_items,
                                                           replace=loss_graph.is_sampled_with_replacement)).to(device)
            tf_x_user_sample, tf_x_item_sample = sample_indices[:, 0], sample_indices[:, 1]

        pred_graph = self.prediction_graph_factory
        tastes_predictions, tastes_prediction_serials, tastes_sample_prediction_serials = [], [], []
        with_attention = self.attention_graph_factory is not None
        tastes_attentions = [] if with_attention else None
        tastes_attention_serials = [] if with_attention else None
        tastes_sample_attention_serials = [] if with_attention else None

        for taste in range(self.n_tastes):
            with name_scope('user_{}'.format(taste)):
                user_repr, user_weights = self.user_repr_graph_factory.connect_representation_graph(
                    tf_features=tf_user_features, n_components=self.n_components, n_features=self.n_user_features,
                    node_name_ending='user_{}'.format(taste))
            tf_weights.extend(user_weights)

            if with_attention:
                with name_scope('attn_{}'.format(taste)):
                    attention_repr, attention_weights = self.attention_graph_factory.connect_representation_graph(
                        tf_features=tf_user_features, n_components=self.n_components,
                        n_features=self.n_user_features, node_name_ending='attn_{}'.format(taste))
                tf_weights.extend(attention_weights)
                if loss_graph.is_dense:
                    tastes_attentions.append(pred_graph.connect_dense_prediction_graph(
                        tf_user_representation=attention_repr, tf_item_representation=item_repr))
                tastes_attention_serials.append(pred_graph.connect_serial_prediction_graph(
                    tf_user_representation=attention_repr, tf_item_representation=item_repr,
                    tf_x_user=tf_x_user, tf_x_item=tf_x_item))
                if loss_graph.is_sample_based:
                    # the reference feeds the USER representation here, not the attention one (tensorrec.py:367-372)
                    tastes_sample_attention_serials.append(pred_graph.connect_serial_prediction_graph(
                        tf_user_representation=user_repr, tf_item_representation=item_repr,
                        tf_x_user=tf_x_user_sample, tf_x_item=tf_x_item_sample))

            if loss_graph.is_dense:
                tastes_predictions.append(pred_graph.connect_dense_prediction_graph(
                    tf_user_representation=user_repr, tf_item_representation=item_repr))
            tastes_prediction_serials.append(pred_graph.connect_serial_prediction_graph(
                tf_user_representation=user_repr, tf_item_representation=item_repr,
                tf_x_user=tf_x_user, tf_x_item=tf_x_item))
            if loss_graph.is_sample_based:
                tastes_sample_prediction_serials.append(pred_graph.connect_serial_prediction_graph(
                    tf_user_representation=user_repr, tf_item_representation=item_repr,
                    tf_x_user=tf_x_user_sample, tf_x_item=tf_x_item_sample))

        tf_prediction = None
        if loss_graph.is_dense:
            tf_prediction = collapse_mixture_of_tastes(tastes_predictions, tastes_attentions if with_attention else None)
        tf_prediction_serial = collapse_mixture_of_tastes(tastes_prediction_serials, tastes_attention_serials)
        tf_sample_predictions_serial = None
        if loss_graph.is_sample_based:
            tf_sample_predictions_serial = collapse_mixture_of_tastes(tastes_sample_prediction_serials,
                                                                      tastes_sample_attention_serials)

        if self.biased:
            user_feature_biases = get_variable('feature_biases_user',
                                               lambda: torch.zeros([self.n_user_features, 1], device=device))
            item_feature_biases = get_variable('feature_biases_item',
                                               lambda: torch.zeros([self.n_item_features, 1], device=device))
            projected_user_biases = torch.sum(torch.sparse.mm(tf_user_features, user_feature_biases), dim=1)
            projected_item_biases = torch.sum(torch.sparse.mm(tf_item_features, item_feature_biases), dim=1)
            tf_weights.append(user_feature_biases)
            tf_weights.append(item_feature_biases)
            if tf_prediction is not None:
                tf_prediction = bias_prediction_dense(tf_prediction, projected_user_biases, projected_item_biases)
            tf_prediction_serial = bias_prediction_serial(tf_prediction_serial, projected_user_biases,
                                                          projected_item_biases, tf_x_user, tf_x_item)
            if tf_sample_predictions_serial is not None:
                tf_sample_predictions_serial = bias_prediction_serial(
                    tf_sample_predictions_serial, projected_user_biases, projected_item_biases,
                    tf_x_user_sample, tf_x_item_sample)

        # loss-graph kwargs with the reference's visibility rules (tensorrec.py:463-482)
        loss_graph_kwargs = {
            'tf_prediction_serial': tf_prediction_serial,
            'tf_interactions_serial': tf_interactions._values(),
            'tf_interactions': tf_interactions,
            'tf_n_users': n_users,
            'tf_n_items': n_items,
        }
        if loss_graph.is_dense:
            # In the reference tf_rankings is a graph node that costs nothing unless the loss graph consumes it; here it
            # is a full K3 sort of [n_users, n_items] per step, so it is evaluated only for a loss graph that names it
            tf_rankings = None
            if tf_prediction.is_cuda and _names_argument(loss_graph.connect_loss_graph, 'tf_rankings'):
                # ranks come from the K3 kernel; they carry no gradient (as tf.nn.top_k)
                tf_rankings = kernels.rank_full(tf_prediction.detach().contiguous())
            loss_graph_kwargs.update({'tf_prediction': tf_prediction, 'tf_rankings': tf_rankings})
        if loss_graph.is_sample_based:
            loss_graph_kwargs.update({
                'tf_sample_predictions': densify_sampled_item_predictions(
                    tf_sample_predictions_serial=tf_sample_predictions_serial,
                    tf_n_sampled_items=n_sampled_items, tf_n_users=n_users),
                'tf_n_sampled_items': n_sampled_items})

        with name_scope('loss'):
            basic_loss = loss_graph.connect_loss_graph(**loss_graph_kwargs)
        weight_reg_loss = sum(0.5 * torch.sum(w * w) for w in tf_weights)      # sum of tf.nn.l2_loss
        return basic_loss, weight_reg_loss, tf_prediction_serial, tf_weights

    def fit(self, interactions, user_features, item_features, epochs=100, learning_rate=0.1, alpha=0.00001,
            verbose=False, user_batch_size=None, n_sampled_items=None):
        """Constructs the model on first use and fits it (arguments as tensorrec/tensorrec.py:494-526)."""
        self.fit_partial(interactions=interactions, user_features=user_features, item_features=item_features,
                         epochs=epochs, learning_rate=learning_rate, alpha=alpha, verbose=verbose,
                         user_batch_size=user_batch_size, n_sampled_items=n_sampled_items)

    def fit_partial(self, interactions, user_features, item_features, epochs=1, learning_rate=0.1,
                    alpha=0.00001, verbose=False, user_batch_size=None, n_sampled_items=None):
        """One or more epochs of Adam on the loss graph (tensorrec/tensorrec.py:539-634)."""
        device = get_session().device

        if self.loss_graph_factory.is_sample_based:
            if (n_sampled_items is None) or (n_sampled_items <= 0):
                raise ValueError("n_sampled_items must be an integer >0")
        if (n_sampled_items is not None) and (not self.loss_graph_factory.is_sample_based):
            logging.warning('n_sampled_items was specified, but the loss graph is not sample-based')

        if verbose:
            logging.info('Processing interaction and feature data')
        batches = self._create_batched_inputs(interactions=interactions, user_features=user_features,
                                              item_features=item_features, user_batch_size=user_batch_size)

        first_build = self.tf_prediction is None
        if first_build:
            # feature counts are learned from the first batch and cannot change afterwards (tensorrec.py:598-605)
            self.n_user_features = batches[0][1].shape[1]
            self.n_item_features = batches[0][2].shape[1]
            self._attach_graph_hooks()

        batched_alpha = calculate_batched_alpha(num_batches=len(batches), alpha=alpha)
        if verbose:
            logging.info('Beginning fitting')
        try:
            self._fit_epochs(batches, epochs, learning_rate, alpha, batched_alpha, verbose, n_sampled_items, device)
            first_build = False
        finally:
            if first_build and not getattr(self, '_stepped', False):
                # the very first step failed (e.g. n_sampled_items > n_items): the model is still unbuilt -- predict()
                # must keep raising ModelNotFitException and a later fit may use other feature counts
                self._break_graph_hooks()
                self.n_user_features = self.n_item_features = None
                self._variables.clear()
                self._optimizer = None

    def _fit_epochs(self, batches, epochs, learning_rate, alpha, batched_alpha, verbose, n_sampled_items, device):
        from . import train_kernels
        # the training step on hand-written kernels (train_kernels.step_plan, relu_step_plan; DESIGN §3.10, §3.11,
        # §3.14), or the torch path
        plan = None
        if device.type == 'cuda':
            plan = train_kernels.step_plan(self, n_sampled_items) or train_kernels.relu_step_plan(self, n_sampled_items)
        serial = plan is not None and plan.loss != 'wmrb'         # RMSE / Separation: a scalar loss
        for epoch in range(epochs):
            for batch, (int_in, uf_in, if_in) in enumerate(batches):
                if uf_in.shape[1] != self.n_user_features or if_in.shape[1] != self.n_item_features:
                    raise ValueError('feature matrices have {} / {} columns but the model was built for {} / {}'.format(
                        uf_in.shape[1], if_in.shape[1], self.n_user_features, self.n_item_features))
                if plan is not None:
                    # the training step on hand-written kernels (train_kernels.py; SURVEY 8 f1)
                    if getattr(self, '_wmrb_step', None) is None or self._wmrb_step.device != device:
                        self._wmrb_step = train_kernels.WmrbStep(self, device)
                    n_pos = int_in.n_positive
                    # WMRB adds alpha * reg to each positive interaction's loss; a scalar loss adds it once
                    l2 = batched_alpha if serial else n_pos * batched_alpha
                    loss_vec, serial_predictions = self._wmrb_step.step(
                        int_in, uf_in, if_in, n_sampled_items, learning_rate, l2=l2)
                    self._stepped = True
                    if verbose:
                        mean_loss = float(loss_vec[0]) if serial else float(loss_vec.sum()) / max(n_pos, 1)
                        mean_pred = float(torch.mean(serial_predictions))
                        wr = sum(0.5 * float(torch.sum(w.detach() * w.detach())) for w in self._variables.values())
                        logging.info('EPOCH {} BATCH {} loss = {}, weight_reg_l2_loss = {}, mean_pred = {}'.format(
                            epoch, batch, mean_loss, alpha * wr, mean_pred))
                    continue
                with variable_scope(self._variables):
                    basic_loss, wr_loss, serial_predictions, tf_weights = self._training_losses(
                        int_in, uf_in, if_in, n_sampled_items, device)
                loss = basic_loss + batched_alpha * wr_loss
                params = [w for w in tf_weights if w.requires_grad and w.is_leaf]
                self._ensure_optimizer(params, learning_rate)
                self._optimizer.zero_grad(set_to_none=True)
                loss.sum().backward()       # tf.gradients of a vector loss (WMRB) is the gradient of its sum
                self._optimizer.step()
                self._stepped = True
                if verbose:
                    mean_loss = float(torch.mean(basic_loss.detach()))
                    mean_pred = float(torch.mean(serial_predictions.detach()))
                    weight_reg_l2_loss = alpha * float(wr_loss.detach())
                    logging.info('EPOCH {} BATCH {} loss = {}, weight_reg_l2_loss = {}, mean_pred = {}'.format(
                        epoch, batch, mean_loss, weight_reg_l2_loss, mean_pred))

    def _ensure_optimizer(self, params, learning_rate):
        ids = tuple(id(p) for p in params)
        if self._optimizer is None or self._optimizer_params != ids:
            self._optimizer = torch.optim.Adam(params, lr=learning_rate)     # tf.train.AdamOptimizer defaults
            self._optimizer_params = ids
        for group in self._optimizer.param_groups:
            group['lr'] = learning_rate

    # ------------------------------------------------------------------------------------------------
    # weights
    # ------------------------------------------------------------------------------------------------
    def get_weights(self):
        """name -> numpy array of every model weight (linear_weights_item, linear_weights_user_<t>,
        linear_weights_attn_<t>, feature_biases_user, feature_biases_item, ...)."""
        return collections.OrderedDict((k, v.detach().cpu().numpy().copy()) for k, v in self._variables.items())

    def set_weights(self, weights, n_user_features=None, n_item_features=None):
        """Injects weights (dict name -> array).  Marks the model as built, so predict* work without fit -- the
        parity-test hook: the reference never seeds its initialiser (representation_graphs.py:35), so values after
        fit() are unpinned."""
        device = get_session().device
        for name, value in weights.items():
            t = torch.as_tensor(np.asarray(value, dtype=np.float32)).to(device).clone()
            self._variables[name] = t.requires_grad_(True)
        self._optimizer = None
        self._wmrb_step = None          # Adam moments of the kernel training path belong to the replaced weights
        if n_user_features is None and 'linear_weights_user_0' in self._variables:
            n_user_features = self._variables['linear_weights_user_0'].shape[0]
        if n_item_features is None and 'linear_weights_item' in self._variables:
            n_item_features = self._variables['linear_weights_item'].shape[0]
        self.n_user_features = n_user_features if n_user_features is not None else self.n_user_features
        self.n_item_features = n_item_features if n_item_features is not None else self.n_item_features
        self._attach_graph_hooks()

    def _var(self, name, device):
        if name not in self._variables:
            raise RuntimeError('weight {!r} does not exist; fit the model or inject it with set_weights()'.format(name))
        v = self._variables[name]
        if v.device != device:     # fitted on another device: move once and keep
            v = v.detach().to(device).requires_grad_(True)
            self._variables[name] = v
            self._optimizer = None
        return v.detach()

    # ------------------------------------------------------------------------------------------------
    # the predict / predict_rank hot path
    # ------------------------------------------------------------------------------------------------
    @staticmethod
    def _cuda_device():
        kernels.require_cuda()
        return torch.device('cuda', torch.cuda.current_device())

    def _check_features(self, sparse_input, n_features, side):
        if n_features is not None and sparse_input.shape[1] != n_features:
            raise ValueError('{} feature matrix has {} columns but the model was built for {}'.format(
                side, sparse_input.shape[1], n_features))

    def _represent(self, graph, sparse_input, n_features, node_name_ending, device, extra_normalize=0,
                   want_f32=True, split_d_pad=None, want_norm=False, stats=None, split_out=None):
        """One representation on the device: (repr_f32 | None, split | None, scale | None[, norm]).  split_out:
        (split, scale) tensors the split operand is written to."""
        if type(graph) in _BUILTIN_REPR:
            weights = self._var(LinearRepresentationGraph.weight_name(node_name_ending), device)
            n_norm = (1 if graph.b200_kind == 'normalized_linear' else 0) + extra_normalize
            return kernels.gather_reduce(sparse_input.device_csr(device), weights, n_normalize=n_norm,
                                         want_f32=want_f32, split_d_pad=split_d_pad, want_norm=want_norm, stats=stats,
                                         split_out=split_out)
        # user-defined / non-linear plugin: run its own forward on the device, then hand the dense rows to the kernels
        with torch.no_grad(), variable_scope(self._variables), name_scope(node_name_ending):
            for k in list(self._variables):
                self._var(k, device)
            dense, _ = graph.connect_representation_graph(
                tf_features=sparse_input.torch_sparse(device), n_components=self.n_components, n_features=n_features,
                node_name_ending=node_name_ending)
        dense = dense.detach().to(torch.float32).contiguous().clone()
        for _ in range(extra_normalize):
            kernels.l2_normalize_rows_(dense)
        split = scale = None
        if split_d_pad is not None:
            split, scale = kernels.split_f32(dense, n_normalize=0, d_pad=split_d_pad, out=split_out)
        if stats is not None:
            stats.zero_()
        if want_norm or stats is not None:
            norm = kernels.operand_stats(split, scale, split_d_pad, want_norm=want_norm, stats=stats)
            if want_norm:
                return (dense if want_f32 else None), split, scale, norm
        return (dense if want_f32 else None), split, scale

    def _projected_biases(self, sparse_input, name, device):
        return kernels.project_biases(sparse_input.device_csr(device), self._var(name, device).reshape(-1))

    def _tensor_path_ok(self, allow_tastes=False):
        """Can the tensor-core kernels evaluate this model?  allow_tastes: the fused top-k also covers n_tastes > 1 without
        attention (one sweep per taste, then a de-duplicating merge: the prediction is the maximum over the tastes) --
        for k <= 32 one merge of all the per-taste lists, on the wide route a pairwise fold of each taste's list into
        the running result (DESIGN §3.6)."""
        if SCORE_PATH == 'exact':
            return False
        ok = (type(self.prediction_graph_factory) in (DotProductPredictionGraph, CosineSimilarityPredictionGraph)
              and (self.n_tastes == 1 or allow_tastes) and self.attention_graph_factory is None
              and kernels.d_pad_for(self.n_components) <= 128)
        if SCORE_PATH == 'tensor' and not ok:
            raise RuntimeError('TENSORREC_B200_SCORE_PATH=tensor but this model cannot use the tensor-core kernel')
        return ok

    def _euclidean_tensor_ok(self):
        """Can the tensor-core kernels evaluate this Euclidean user x item model?  The built-in Euclidean graph, no
        attention, d_pad <= 128; any number of tastes (the fused top-k merges one sweep per taste; dense scoring takes
        one taste only -- _score_plan checks that)."""
        return (SCORE_PATH != 'exact' and type(self.prediction_graph_factory) is EuclideanSimilarityPredictionGraph
                and self.attention_graph_factory is None and kernels.d_pad_for(self.n_components) <= 128)

    def _tastes_tensor_ok(self):
        """Can the taste-collapsing tensor-core kernels evaluate this mixture of tastes?  Built-in dot or cosine
        prediction, n_tastes >= 2 within the kernel's operand rows (T <= 64, T <= 32 with attention), any attention
        graph or none, d_pad <= 128."""
        return (SCORE_PATH != 'exact'
                and type(self.prediction_graph_factory) in (DotProductPredictionGraph, CosineSimilarityPredictionGraph)
                and self.n_tastes >= 2
                and kernels.tastes_plan(self.n_tastes, self.attention_graph_factory is not None) is not None
                and kernels.d_pad_for(self.n_components) <= 128)

    def _euclid_tastes_tensor_ok(self):
        """Can the taste-collapsing tensor-core kernels evaluate this Euclidean mixture of tastes (DESIGN §3.12)?  The
        built-in Euclidean graph, n_tastes >= 2 within the kernel's operand rows (T <= 64, T <= 32 with attention), any
        attention graph or none, d_pad <= 128."""
        return (SCORE_PATH != 'exact' and type(self.prediction_graph_factory) is EuclideanSimilarityPredictionGraph
                and self.n_tastes >= 2
                and kernels.tastes_plan(self.n_tastes, self.attention_graph_factory is not None) is not None
                and kernels.d_pad_for(self.n_components) <= 128)

    def _taste_operands(self, block_in, device):
        """The users of a mixture of tastes as kernels.SideOperands whose split is the stacked operand [n_ops, U,
        2 d_pad] (u_0 .. u_{T-1}, then a_0 .. a_{T-1} with attention) and scale [n_ops, U]; K1 writes every operand
        straight into its slice, normalised as the CUDA-core path normalises it.  With Euclidean prediction, hsq holds
        the half squared norms of every slice [n_ops, U] (one operand_half_sqnorm launch over the stacked rows)."""
        extra = 1 if type(self.prediction_graph_factory) is CosineSimilarityPredictionGraph else 0
        d_pad = kernels.d_pad_for(self.n_components)
        rows = block_in.shape[0]
        ops = [(self.user_repr_graph_factory, 'user_{}'.format(t)) for t in range(self.n_tastes)]
        if self.attention_graph_factory is not None:
            ops += [(self.attention_graph_factory, 'attn_{}'.format(t)) for t in range(self.n_tastes)]
        split = torch.empty((len(ops), rows, 2 * d_pad), dtype=torch.float16, device=device)
        scale = torch.empty((len(ops), rows), dtype=torch.float32, device=device)
        for j, (graph, name) in enumerate(ops):
            self._represent(graph, block_in, self.n_user_features, name, device, extra, want_f32=False,
                            split_d_pad=d_pad, split_out=(split[j], scale[j]))
        bias = self._projected_biases(block_in, 'feature_biases_user', device) if self.biased else None
        hsq = None
        if type(self.prediction_graph_factory) is EuclideanSimilarityPredictionGraph:
            hsq = kernels.operand_half_sqnorm(split.view(len(ops) * rows, 2 * d_pad), scale.view(-1), d_pad)
            hsq = hsq.view(len(ops), rows)
        return kernels.SideOperands(None, split, scale, bias, rows, self.n_components, d_pad, hsq=hsq)

    def _side_operands(self, side, sparse_in, device, for_filter=False, taste=0):
        """One side ('user' or 'item') as kernels.SideOperands: split-fp16 operand + scale, projected biases and -- for
        the filter form of the fused top-k -- the row norms (users) / the global statistics (items), all from K1."""
        extra = 1 if type(self.prediction_graph_factory) is CosineSimilarityPredictionGraph else 0
        d_pad = kernels.d_pad_for(self.n_components)
        is_user = side == 'user'
        graph = self.user_repr_graph_factory if is_user else self.item_repr_graph_factory
        n_features = self.n_user_features if is_user else self.n_item_features
        stats = norm = None
        if for_filter and not is_user:
            stats = torch.empty((3,), dtype=torch.float32, device=device)
        out = self._represent(graph, sparse_in, n_features, 'user_{}'.format(taste) if is_user else 'item', device, extra,
                              want_f32=False, split_d_pad=d_pad, want_norm=for_filter and is_user, stats=stats)
        split, scale = out[1], out[2]
        if for_filter and is_user:
            norm = out[3]
        bias = None
        if self.biased:
            bias = self._projected_biases(sparse_in, 'feature_biases_user' if is_user else 'feature_biases_item', device)
        return kernels.SideOperands(None, split, scale, bias, sparse_in.shape[0], self.n_components, d_pad, norm=norm,
                                    stats=stats)

    def _tensor_operands(self, user_in, item_in, device):
        return self._side_operands('user', user_in, device), self._side_operands('item', item_in, device)

    def _tensor_score_form(self):
        """How _score_plan scores this model on the exact tensor-core kernel: 'tastes' (the taste-collapsing form),
        'tastes_euclid' (its Euclidean form), 'euclidean' or 'dot' (dot / cosine); None when it scores it otherwise."""
        if self._tastes_tensor_ok():      # (checked first: SCORE_PATH='tensor' accepts these models)
            return 'tastes'
        if self._euclid_tastes_tensor_ok():
            return 'tastes_euclid'
        if self.n_tastes == 1 and self._euclidean_tensor_ok():
            return 'euclidean'
        return 'dot' if self._tensor_path_ok() else None

    def _score_plan(self, item_in, device):
        """Item-side work of the dense prediction, done once per call: returns score(user_block_in, out=None) ->
        float32 [rows, n_items] on the device.  Tensor cores (split-product kernel, dot / cosine / Euclidean) when the
        model allows, the exact CUDA-core kernel (tastes, attention, wide rows) or the plugin's own dense form
        otherwise."""
        n_items = item_in.shape[0]
        form = self._tensor_score_form()
        if form in ('tastes', 'tastes_euclid'):
            items = self._side_operands('item', item_in, device)
            meta = kernels.pack_item_meta(items.scale, items.bias, n_items)
            item_hsq = kernels.item_half_sqnorm(items) if form == 'tastes_euclid' else None
            attention = self.attention_graph_factory is not None

            def score(block_in, out=None):
                return kernels.score_dense_tastes(self._taste_operands(block_in, device), items.split, meta, n_items,
                                                  self.n_tastes, attention, out=out, item_hsq=item_hsq)
            return score
        euclidean = form == 'euclidean'
        if form is not None:
            items = self._side_operands('item', item_in, device)
            meta = kernels.pack_item_meta(items.scale, items.bias, n_items)
            item_hsq = kernels.item_half_sqnorm(items) if euclidean else None

            def score(block_in, out=None):
                users = self._side_operands('user', block_in, device)
                sqnorms = None
                if euclidean:
                    sqnorms = (kernels.operand_half_sqnorm(users.split, users.scale, users.d_pad), item_hsq)
                return kernels.score_dense_tc(users.split, users.scale, users.bias, items.split, meta,
                                              block_in.shape[0], n_items, users.d_pad, out=out, sqnorms=sqnorms)
            return score

        pred_graph = self.prediction_graph_factory
        builtin = type(pred_graph) in _BUILTIN_PRED
        extra = 1 if (builtin and pred_graph.b200_kind == 'cosine') else 0
        item_repr, _, _ = self._represent(self.item_repr_graph_factory, item_in, self.n_item_features, 'item', device,
                                          extra)
        item_bias = self._projected_biases(item_in, 'feature_biases_item', device) if self.biased else None

        def score(block_in, out=None):
            user_reprs = torch.stack([self._represent(self.user_repr_graph_factory, block_in, self.n_user_features,
                                                      'user_{}'.format(t), device, extra)[0]
                                      for t in range(self.n_tastes)])
            attention_reprs = None
            if self.attention_graph_factory is not None:
                attention_reprs = torch.stack([self._represent(self.attention_graph_factory, block_in,
                                                               self.n_user_features, 'attn_{}'.format(t), device,
                                                               extra)[0]
                                               for t in range(self.n_tastes)])
            user_bias = self._projected_biases(block_in, 'feature_biases_user', device) if self.biased else None
            if builtin and not (pred_graph.b200_kind == 'euclidean' and attention_reprs is not None):
                mode = 1 if pred_graph.b200_kind == 'euclidean' else 0
                return kernels.score_exact(user_reprs, item_repr, user_bias, item_bias, mode=mode,
                                           attention_repr=attention_reprs, out=out)
            # user-defined prediction graph: its own dense form per taste, then the reference's collapse + bias order
            with torch.no_grad():
                preds = [pred_graph.connect_dense_prediction_graph(tf_user_representation=user_reprs[t],
                                                                   tf_item_representation=item_repr)
                         for t in range(self.n_tastes)]
                atts = None
                if attention_reprs is not None:
                    atts = [pred_graph.connect_dense_prediction_graph(tf_user_representation=attention_reprs[t],
                                                                      tf_item_representation=item_repr)
                            for t in range(self.n_tastes)]
                pred = collapse_mixture_of_tastes(preds, atts)
                if self.biased:
                    pred = bias_prediction_dense(pred, user_bias, item_bias)
            pred = pred.to(torch.float32).contiguous()
            if out is not None:
                out.copy_(pred)
                return out
            return pred
        return score

    def _predict_device(self, user_in, item_in, device):
        """tf_prediction: dense float32 scores [n_users, n_items] on the device."""
        self._check_features(user_in, self.n_user_features, 'user')
        self._check_features(item_in, self.n_item_features, 'item')
        n_users, n_items = user_in.shape[0], item_in.shape[0]
        if n_users == 0 or n_items == 0:
            return torch.zeros((n_users, n_items), dtype=torch.float32, device=device)
        return self._score_plan(item_in, device)(user_in)

    # a dense [n_users, n_items] result beyond this many bytes is produced in user blocks (SURVEY 8d: BASELINE config #2,
    # 1M x 100K = 400 GB, exceeds the 80 GB of an H100): two device buffers + two page-locked host buffers of this size
    PREDICT_BLOCK_BYTES = 4 << 30

    def _user_blocks(self, user_in, n_items, user_batch_size):
        n_users = user_in.shape[0]
        if user_batch_size is None:
            user_batch_size = max(128, (self.PREDICT_BLOCK_BYTES // max(4 * n_items, 1)) // 128 * 128)
        step = max(1, int(user_batch_size))
        if step >= n_users:
            return [(0, n_users, user_in)]
        csr = user_in.matrix if isinstance(user_in.matrix, sp.csr_matrix) else sp.csr_matrix(user_in.matrix)
        return [(u0, min(n_users, u0 + step), SparseInput(csr[u0:min(n_users, u0 + step)]))
                for u0 in range(0, n_users, step)]

    def predict_batches(self, user_features, item_features, user_batch_size=None):
        """predict() as a stream of user blocks: yields (u0, u1, scores float32 ndarray [u1 - u0, n_items]).

        For results that fit neither HBM nor host memory at once (BASELINE config #2: 1M x 100K = 400 GB).  The item side
        is computed once; user blocks are scored into two alternating device buffers and copied into two alternating
        page-locked host buffers on a copy stream, so the device->host transfer of block b overlaps the kernels of block
        b + 1 (the path is bound by the host link, not by HBM).  The yielded array IS the page-locked buffer: it stays
        valid until the generator is advanced twice."""
        if self.tf_prediction is None:
            raise ModelNotFitException(method='predict')
        device = self._cuda_device()
        user_in = self._single_input(user_features, 'user_features')
        item_in = self._single_input(item_features, 'item_features')
        self._check_features(user_in, self.n_user_features, 'user')
        self._check_features(item_in, self.n_item_features, 'item')
        n_users, n_items = user_in.shape[0], item_in.shape[0]
        if n_users == 0 or n_items == 0:
            yield 0, n_users, np.zeros((n_users, n_items), dtype=np.float32)
            return
        blocks = self._user_blocks(user_in, n_items, user_batch_size)
        rows = max(u1 - u0 for u0, u1, _ in blocks)
        score = self._score_plan(item_in, device)
        n_buf = min(2, len(blocks))
        # the staging buffers (page-locking gigabytes takes seconds) are kept for the next call of the same shape
        key = (rows, n_items, n_buf, str(device))
        cached = getattr(self, '_stream_buffers', None)
        if cached is None or cached[0] != key:
            self._stream_buffers = None
            cached = (key,
                      [torch.empty((rows, n_items), dtype=torch.float32, device=device) for _ in range(n_buf)],
                      [torch.empty((rows, n_items), dtype=torch.float32, pin_memory=True) for _ in range(n_buf)])
            self._stream_buffers = cached
        dev_buf, host_buf = cached[1], cached[2]
        compute = torch.cuda.current_stream()
        copier = torch.cuda.Stream(device=device)
        copied = [None] * n_buf       # event: the copy out of dev_buf[j] / into host_buf[j] has finished
        pending = None
        for b, (u0, u1, block_in) in enumerate(blocks):
            j = b % n_buf
            if copied[j] is not None:
                compute.wait_event(copied[j])          # the kernels of this block overwrite dev_buf[j]
            score(block_in, out=dev_buf[j][:u1 - u0])
            done = torch.cuda.Event()
            done.record(compute)
            with torch.cuda.stream(copier):
                copier.wait_event(done)
                host_buf[j][:u1 - u0].copy_(dev_buf[j][:u1 - u0], non_blocking=True)
                copied[j] = torch.cuda.Event()
                copied[j].record(copier)
            if pending is not None:                    # hand out block b - 1 while block b is being computed / copied
                pj, p0, p1 = pending
                copied[pj].synchronize()
                yield p0, p1, host_buf[pj][:p1 - p0].numpy()
            pending = (j, u0, u1)
        pj, p0, p1 = pending
        copied[pj].synchronize()
        yield p0, p1, host_buf[pj][:p1 - p0].numpy()

    def predict(self, user_features, item_features, out=None, user_batch_size=None):
        """Scores for every user x item pair: float32 ndarray [n_users, n_items] (tensorrec/tensorrec.py:636-664).

        Results larger than PREDICT_BLOCK_BYTES (or any result when user_batch_size / out is given) are produced in user
        blocks (predict_batches) and assembled in `out` -- a caller-provided float32 array [n_users, n_items], e.g. a
        numpy.memmap when the matrix exceeds host memory -- or in a new array."""
        if self.tf_prediction is None:
            raise ModelNotFitException(method='predict')
        device = self._cuda_device()
        user_in = self._single_input(user_features, 'user_features')
        item_in = self._single_input(item_features, 'item_features')
        n_users, n_items = user_in.shape[0], item_in.shape[0]
        streamed = (out is not None or user_batch_size is not None or
                    4 * n_users * n_items > self.PREDICT_BLOCK_BYTES)
        if not streamed:
            return kernels.to_host(self._predict_device(user_in, item_in, device))
        if out is None:
            out = np.empty((n_users, n_items), dtype=np.float32)
        elif tuple(out.shape) != (n_users, n_items) or out.dtype != np.float32:
            raise ValueError('out must be a float32 array of shape ({}, {})'.format(n_users, n_items))
        for u0, u1, block in self.predict_batches(user_in, item_in, user_batch_size=user_batch_size):
            out[u0:u1] = block
        return out

    def predict_rank(self, user_features, item_features, k=None, exclude=None):
        """Ranks for every user x item pair: int32 ndarray [n_users, n_items], 1 = best, ties by lower item index
        (tensorrec/tensorrec.py:705-733).  With k (an addition for shapes whose rank matrix cannot be materialised)
        only the entries with rank <= k are produced, as a TopK(items, scores) -- see predict_top_k, also for
        `exclude` (top-k only: full ranks with exclusion raise ValueError)."""
        if self.tf_prediction is None:
            raise ModelNotFitException(method='predict_rank')
        if k is not None:
            if exclude is None:
                return self.predict_top_k(user_features, item_features, k)
            return self.predict_top_k(user_features, item_features, k, exclude=exclude)
        if exclude is not None:
            raise ValueError('exclude needs k: exclusion applies to the top-k only, not to full ranks')
        device = self._cuda_device()
        user_in = self._single_input(user_features, 'user_features')
        item_in = self._single_input(item_features, 'item_features')
        scores = self._predict_device(user_in, item_in, device)
        if scores.numel() == 0:
            return np.zeros(tuple(scores.shape), dtype=np.int32)
        return kernels.to_host(kernels.rank_full(scores))

    def predict_rank_at(self, user_features, item_features, pairs, exclude=None, user_batch_size=None):
        """The full rank of listed (user, item) pairs, without the [n_users, n_items] rank matrix: where each held-out
        item ranks for its user (recall / precision / ndcg at any k, hit rate, MRR, mean rank; tensorrec_b200.eval
        accepts the result).

        pairs: a scipy sparse matrix [n_users, n_items]; the pair (u, i) is listed when pairs[u, i] != 0 after
        duplicates are summed (explicit zeros list nothing).  Returns a scipy.sparse.csr_matrix of int32 [n_users,
        n_items] with sorted indices and one stored entry per listed pair: predict_rank(user_features,
        item_features)[u, i] = 1 + #{j: s_uj > s_ui} + #{j < i: s_uj == s_ui}, s the scores predict() returns, bit for
        bit (-0.0 and +0.0 compare equal).  exclude (validated as predict_top_k's single-GPU exclude): the rank among
        the items (u, j) not excluded plus the pair itself, 1 + #{j != i, (u, j) not excluded: s_uj > s_ui or (s_uj ==
        s_ui and j < i)} -- a listed pair that is itself excluded is ranked by its own score against the eligible
        items.  For a non-excluded pair of rank r <= k on an exact top-k route, predict_top_k(..., k,
        exclude=exclude).items[u, r - 1] == i.

        Users go in blocks that start at multiples of the kernel's user block (128 rows, or 2P for a mixture of tastes:
        DESIGN §3.5), so user_batch_size is rounded down to a positive multiple of it.  last_rank_info['path'] names
        the route (rank_at_route): 'exact3_count', the exact kernel's counting mode, or 'dense+rank', the scores of
        predict() ranked per block; last_rank_info['passes'] = the counting passes of the largest block (ceil of a
        row's most pairs / 32; 0 on dense+rank)."""
        if self.tf_prediction is None:
            raise ModelNotFitException(method='predict_rank_at')
        user_in = self._single_input(user_features, 'user_features')
        item_in = self._single_input(item_features, 'item_features')
        n_users, n_items = user_in.shape[0], item_in.shape[0]
        if not sp.issparse(pairs):
            raise ValueError('pairs must be a scipy sparse matrix with one row per user and one column per item')
        if tuple(pairs.shape) != (n_users, n_items):
            raise ValueError('pairs has shape %s but there are %d users and %d items'
                             % (tuple(pairs.shape), n_users, n_items))
        if exclude is not None:      # validated before any device work (the k argument does not apply here)
            exclude = _checked_exclude(exclude, n_users, n_items, 1, 0, False)
        self._check_features(user_in, self.n_user_features, 'user')
        self._check_features(item_in, self.n_item_features, 'item')
        indptr, ids = kernels.exclusion_host_csr(pairs, 0, n_items)   # the listing rule is the exclusion rule
        form = self._tensor_score_form()
        attention = self.attention_graph_factory is not None
        path = rank_at_route(n_items, form is not None, euclid_attention=form == 'tastes_euclid' and attention)
        self.last_rank_info = {'path': path, 'passes': 0}
        ranks = np.zeros(ids.shape[0], dtype=np.int32)
        result = lambda: sp.csr_matrix((ranks, ids, indptr), shape=(n_users, n_items))   # noqa: E731
        if ids.size == 0:
            return result()
        device = self._cuda_device()

        tastes_form = form in ('tastes', 'tastes_euclid')
        unit = kernels.tastes_plan(self.n_tastes, attention)[1] if tastes_form else kernels.TILE_USERS
        if path == 'exact3_count':
            n_ops = kernels.tastes_n_ops(self.n_tastes, attention) if tastes_form else 1
            # (tastes_euclid: 4 more bytes per operand row for its half squared norm)
            per_op = 4 * kernels.d_pad_for(self.n_components) + 8 + (4 if form == 'tastes_euclid' else 0)
            per_row = n_ops * per_op + 16
        else:
            per_row = kernels.DENSE_RANK_BYTES_PER_PAIR * n_items
        max_rows = self.PREDICT_BLOCK_BYTES // per_row if user_batch_size is None else int(user_batch_size)
        max_rows = max(unit, max_rows // unit * unit)
        blocks = rank_at_blocks(indptr, unit, max_rows, self.PREDICT_BLOCK_BYTES // kernels.RANK_AT_BYTES_PER_PAIR)
        csr = user_in.matrix if isinstance(user_in.matrix, sp.csr_matrix) else sp.csr_matrix(user_in.matrix)

        if path == 'exact3_count':
            items = self._side_operands('item', item_in, device)
            meta = kernels.pack_item_meta(items.scale, items.bias, n_items)
            item_hsq = kernels.item_half_sqnorm(items) if form in ('euclidean', 'tastes_euclid') else None
        else:
            score = self._score_plan(item_in, device)
        parts = []
        for u0, u1 in blocks:
            p0, p1 = int(indptr[u0]), int(indptr[u1])
            if p1 == p0:
                continue
            block_in = user_in if (u0, u1) == (0, n_users) else SparseInput(csr[u0:u1])
            b_indptr, b_ids = (indptr[u0:u1 + 1] - p0).astype(np.int32), ids[p0:p1]
            excl = None if exclude is None else kernels.DeviceExclusion.upload(
                *kernels.exclusion_host_csr(exclude, 0, n_items, u0, u1), device=device)
            if path == 'exact3_count':
                if tastes_form:
                    users, tastes = self._taste_operands(block_in, device), (self.n_tastes, attention)
                else:
                    users, tastes = self._side_operands('user', block_in, device), None
                counts, passes = kernels.count_listed_pairs(users, items, meta, b_indptr, b_ids, unit, excl=excl,
                                                            item_hsq=item_hsq, tastes=tastes)
                self.last_rank_info['passes'] = max(self.last_rank_info['passes'], passes)
                parts.append(counts + 1)
                del users
            else:
                rows = torch.from_numpy(np.repeat(np.arange(u1 - u0), np.diff(b_indptr))).to(device)
                cols = torch.from_numpy(b_ids.astype(np.int64)).to(device)
                parts.append(kernels.rank_listed_from_scores(score(block_in), rows, cols, excl=excl,
                                                             block_bytes=self.PREDICT_BLOCK_BYTES))
        ranks = (torch.cat(parts) if len(parts) > 1 else parts[0]).cpu().numpy()
        return result()

    def predict_at(self, user_features, item_features, pairs, user_batch_size=None):
        """The scores of listed (user, item) pairs, without the [n_users, n_items] score matrix: held-out ratings,
        the candidates of a re-ranking stage, the items a user was shown.

        pairs: a scipy sparse matrix [n_users, n_items]; the pair (u, i) is listed when pairs[u, i] != 0 after
        duplicates are summed (explicit zeros list nothing), as for predict_rank_at.  Returns a scipy.sparse.csr_matrix
        of float32 [n_users, n_items] with sorted indices and one stored entry per listed pair (a score of 0.0 is
        stored too): predict(user_features, item_features)[u, i], bit for bit.

        Users go in blocks that start at multiples of the kernel's user block (128 rows, or 2P for a mixture of
        tastes: DESIGN §3.5), so user_batch_size is rounded down to a positive multiple of it.
        last_predict_at_info['path'] names the route (predict_at_route): 'exact3_pairs', the exact kernel's pairs
        mode (catalogues of at least PREDICT_AT_MIN_ITEMS items), or 'dense+gather', predict()'s scores of each block
        gathered at the pairs; last_predict_at_info['tiles'] = the item tiles the pairs mode gathered (0 on
        dense+gather)."""
        if self.tf_prediction is None:
            raise ModelNotFitException(method='predict_at')
        user_in = self._single_input(user_features, 'user_features')
        item_in = self._single_input(item_features, 'item_features')
        n_users, n_items = user_in.shape[0], item_in.shape[0]
        if not sp.issparse(pairs):
            raise ValueError('pairs must be a scipy sparse matrix with one row per user and one column per item')
        if tuple(pairs.shape) != (n_users, n_items):
            raise ValueError('pairs has shape %s but there are %d users and %d items'
                             % (tuple(pairs.shape), n_users, n_items))
        self._check_features(user_in, self.n_user_features, 'user')
        self._check_features(item_in, self.n_item_features, 'item')
        indptr, ids = kernels.exclusion_host_csr(pairs, 0, n_items)   # the listing rule is the exclusion rule
        form = self._tensor_score_form()
        path = predict_at_route(n_items, form is not None)
        self.last_predict_at_info = {'path': path, 'tiles': 0}
        scores = np.zeros(ids.shape[0], dtype=np.float32)
        result = lambda: sp.csr_matrix((scores, ids, indptr), shape=(n_users, n_items))   # noqa: E731
        if ids.size == 0:
            return result()
        device = self._cuda_device()

        attention = self.attention_graph_factory is not None
        tastes_form = form in ('tastes', 'tastes_euclid')
        unit = kernels.tastes_plan(self.n_tastes, attention)[1] if tastes_form else kernels.TILE_USERS
        if path == 'exact3_pairs':
            n_ops = kernels.tastes_n_ops(self.n_tastes, attention) if tastes_form else 1
            # (tastes_euclid: 4 more bytes per operand row for its half squared norm)
            per_row = n_ops * (4 * kernels.d_pad_for(self.n_components) + 8 + (4 if form == 'tastes_euclid' else 0)) + 8
        else:
            per_row = 4 * n_items
        max_rows = self.PREDICT_BLOCK_BYTES // per_row if user_batch_size is None else int(user_batch_size)
        max_rows = max(unit, max_rows // unit * unit)
        blocks = rank_at_blocks(indptr, unit, max_rows, self.PREDICT_BLOCK_BYTES // kernels.PREDICT_AT_BYTES_PER_PAIR)
        csr = user_in.matrix if isinstance(user_in.matrix, sp.csr_matrix) else sp.csr_matrix(user_in.matrix)

        if path == 'exact3_pairs':
            items = self._side_operands('item', item_in, device)
            meta = kernels.pack_item_meta(items.scale, items.bias, n_items)
            item_hsq = kernels.item_half_sqnorm(items) if form in ('euclidean', 'tastes_euclid') else None
        else:
            score = self._score_plan(item_in, device)
        parts = []
        for u0, u1 in blocks:
            p0, p1 = int(indptr[u0]), int(indptr[u1])
            if p1 == p0:
                continue
            block_in = user_in if (u0, u1) == (0, n_users) else SparseInput(csr[u0:u1])
            b_indptr, b_ids = (indptr[u0:u1 + 1] - p0).astype(np.int32), ids[p0:p1]
            if path == 'exact3_pairs':
                if tastes_form:
                    users, tastes = self._taste_operands(block_in, device), (self.n_tastes, attention)
                else:
                    users, tastes = self._side_operands('user', block_in, device), None
                plan = kernels.pairs_plan(b_indptr, b_ids, u1 - u0, unit)
                self.last_predict_at_info['tiles'] += int(plan.tile_items.shape[0])
                parts.append(kernels.score_listed_pairs(users, items, meta, b_indptr, plan, item_hsq=item_hsq,
                                                        tastes=tastes))
                del users
            else:
                rows = torch.from_numpy(np.repeat(np.arange(u1 - u0), np.diff(b_indptr))).to(device)
                cols = torch.from_numpy(b_ids.astype(np.int64)).to(device)
                parts.append(score(block_in)[rows, cols])
        scores = (torch.cat(parts) if len(parts) > 1 else parts[0]).cpu().numpy()
        return result()

    def predict_top_k(self, user_features, item_features, k, item_id_offset=0, gather_group=None, to_host=True,
                      gather='all', user_batch_size=None, exclude=None):
        """The k best items per user in reference rank order, without materialising the score matrix.

        Single GPU: K2+K3 fused kernel (filter form: one tensor pass + re-scoring of the survivors; users the
        certificate rejects go through the exact kernel on the device) -> TopK(items, scores) for every user.
        Item axis sharded over ranks (`gather_group` = a torch.distributed process group whose ranks each pass THEIR
        rows of item_features and the global id of the first one as item_id_offset): one all-to-all of the per-shard
        top-k -- rank r receives the candidates of ITS slice of the users from every shard and merges them -- and,
        with gather='all', one all-gather of the merged slices so that every rank returns all users.  gather='slice'
        returns this rank's users only (rows `last_topk_info['user_rows']`).
        user_batch_size: users are processed in blocks of this many rows (bounds device memory at 10M+ users).
        32 < k <= WIDE_MAX_K on catalogues of at least WIDE_MIN_ITEMS items runs on the wide form of the filter (each
        user's candidates in a list in device memory, rows the certificate rejects scored dense and ranked); the default
        user blocks then keep those lists within PREDICT_BLOCK_BYTES.  A mixture of tastes without attention takes the
        same routes as one taste: one sweep per taste, and on the wide route each taste's top-k folded into the running
        result by a de-duplicating merge (last_topk_info['fallback_rows'] sums the tastes' fallback rows).  Euclidean
        models run k <= 32 on the exact kernel
        (catalogues of at least EUCLIDEAN_MIN_ITEMS items); so do mixtures of tastes with an attention graph
        (ATTENTION_MIN_ITEMS), on the taste-collapsing kernel, Euclidean prediction included.  Both run 32 < k <= WIDE_MAX_K on the exact kernel's wide
        mode on catalogues of at least EXACT_WIDE_MIN_ITEMS items (a Euclidean mixture of tastes: one sweep per taste,
        folded as on the wide route), and otherwise on dense+rank with tensor-core scoring.
        last_topk_info['path'] names the route (topk_route).

        exclude: None, or a scipy sparse matrix (any format) with n_users rows whose column index is the GLOBAL item id
        (the numbering of TopK.items).  The pair (u, i) is excluded when exclude[u, i] != 0 after duplicates are summed
        (explicit zeros exclude nothing, negative values do: "disliked" counts as seen).  Result: for every user the k
        best NON-excluded items in reference rank order (score descending, lower item id on ties) -- the result of a
        model whose excluded pairs score -inf, with excluded items never appearing; a user with fewer than k eligible
        items gets (id 2**31 - 1, score -inf) in the remaining slots.  With n_tastes > 1 an item is excluded for every
        taste.  exclude.shape[1] must equal n_items, or -- in sharded calls (item_id_offset != 0 or gather_group) -- be
        >= item_id_offset + n_items; entries outside this shard are ignored, so every rank can pass the same matrix.
        An exclude without non-zero entries gives results bit-identical to exclude=None."""
        if self.tf_prediction is None:
            raise ModelNotFitException(method='predict_rank')
        if exclude is not None:      # validated before any device work
            exclude = _checked_exclude(exclude, self._single_input(user_features, 'user_features').shape[0],
                                       self._single_input(item_features, 'item_features').shape[0], k,
                                       item_id_offset, item_id_offset != 0 or gather_group is not None)
        device = self._cuda_device()
        user_in = self._single_input(user_features, 'user_features')
        item_in = self._single_input(item_features, 'item_features')
        self._check_features(user_in, self.n_user_features, 'user')
        self._check_features(item_in, self.n_item_features, 'item')
        n_users, n_items = user_in.shape[0], item_in.shape[0]
        k = int(k)
        if k < 1:
            raise ValueError('k must be >= 1')
        if gather not in ('all', 'slice'):
            raise ValueError("gather must be 'all' or 'slice'")
        if n_users == 0:
            return TopK(np.zeros((0, k), np.int32), np.zeros((0, k), np.float32))
        from . import distributed

        attention = self.attention_graph_factory is not None
        euclidean = self._euclidean_tensor_ok()      # (checked first: SCORE_PATH='tensor' accepts these models)
        euclid_attention = attention and self._euclid_tastes_tensor_ok()
        if attention:
            model_ok = self._tastes_tensor_ok() or euclid_attention
        else:
            model_ok = euclidean or self._tensor_path_ok(allow_tastes=True)
        path = self._topk_path(k, n_items, model_ok, self.n_tastes == 1,
                               sharded=item_id_offset != 0 or gather_group is not None, euclidean=euclidean,
                               attention=attention)
        items = fitems = item_hsq = None
        if path != 'dense+rank' and n_items > 0:
            one_pass = path in ('filter', 'wide')
            items = self._side_operands('item', item_in, device, for_filter=one_pass)
            if one_pass:
                fitems = kernels.FilterItems(items)
            if euclidean or euclid_attention:
                item_hsq = kernels.item_half_sqnorm(items)

        if user_batch_size is None:
            # (an attention model collapses its tastes in one sweep: no per-taste fold to hold)
            user_batch_size = self._topk_block_rows(path, n_users, n_items, k, gather_group, device,
                                                    n_tastes=1 if attention else self.n_tastes)
        blocks = self._user_blocks(user_in, n_items, user_batch_size)

        def sweeps(block_in, u0, u1, route, excl):
            if attention:
                # the softmax mixes the tastes: one sweep of the taste-collapsing kernel, no device-side fallback
                users = self._taste_operands(block_in, device)
                topk = kernels.topk_tastes_wide if route == 'exact3_wide' else kernels.topk_tastes
                return topk(users, items, self.n_tastes, True, k, item_id_offset=item_id_offset, excl=excl,
                            item_hsq=item_hsq), [(None, 0)]
            # mixture of tastes (no attention): prediction = max over tastes (recommendation_graphs.py:107), so the top-k
            # lies in the union of the per-taste top-k lists: one fused sweep per taste, then a de-duplicating merge.
            # The wide routes (the wide filter, and the exact kernel's wide mode for Euclidean models) fold each taste's
            # list into the running result right after its sweep (DESIGN §3.6), so a block holds three lists of k
            # entries per row whatever the number of tastes.
            tops, counters, spare = [], [], None
            for t in range(self.n_tastes):
                users = self._side_operands('user', block_in, device, for_filter=route not in ('exact3', 'exact3_wide'),
                                            taste=t)
                taste_top, cnt, cap = kernels.topk_fused(route, users, items, k, fitems=fitems, excl=excl,
                                                         item_id_offset=item_id_offset, item_hsq=item_hsq,
                                                         block_bytes=self.PREDICT_BLOCK_BYTES)
                counters.append((cnt, cap))
                if route in ('wide', 'exact3_wide') and tops:
                    spare = kernels.topk_merge_dedup(tops[0], taste_top, out=spare)
                    tops[0], spare = spare, tops[0]
                else:
                    tops.append(taste_top)
                del users, taste_top
            top = tops[0]
            if len(tops) > 1:
                stacked = torch.stack([t.buf for t in tops]).contiguous()       # [T, U_block, 2k]
                top = kernels.topk_merge_received(stacked, block_in.shape[0], self.n_tastes, k, dedup=True)
            return top, counters

        def exchange(top, u0, u1):
            if gather_group is None:
                return top, np.arange(u0, u1)
            merged, (lo, hi) = distributed.exchange_and_merge(top, gather_group)
            if gather == 'all':
                return distributed.all_gather_rows(merged, u1 - u0, gather_group), np.arange(u0, u1)
            return merged, np.arange(u0 + lo, u0 + hi)

        results, rows = self._run_topk_blocks(path, k, blocks, n_items, item_id_offset, exclude, sweeps,
                                              lambda block_in, u0, u1: self._predict_device(block_in, item_in, device),
                                              exchange, gather_group)
        self.last_topk_info['user_rows'] = rows[0] if len(rows) == 1 else np.concatenate(rows)
        return self._topk_result(results, to_host)

    def _run_topk_blocks(self, path, k, blocks, n_items, item_id_offset, exclude, fused, dense_scores, exchange,
                         gather_group=None):
        """The block loop of a top-k call on `path`, for every (r0, r1, block_in) of `blocks`.  exclude: None, or a CSR
        matrix of excluded (row, GLOBAL item id) pairs; a block's lists over the items [item_id_offset, item_id_offset +
        n_items) are uploaded once for all its sweeps.  The block's top-k: on dense+rank from dense_scores(block_in, r0,
        r1) -> its float32 [r1 - r0, n_items] scores on the device, on a fused route fused(block_in, r0, r1, route,
        excl) -> (PackedTopK, [(device counters | None, capacity)] of its sweeps) (kernels.topk_fused); then
        exchange(top, r0, r1) -> (top, result rows).  Then one synchronisation for the whole call: how many rows the
        certificate rejected per sweep (device counters, summed into last_topk_info['fallback_rows']); a block with more
        rejected rows than the device-side fallback holds is re-run through the exact kernel.  Returns (the PackedTopK
        of every block, its result rows)."""
        info = self.last_topk_info
        device = self._cuda_device()

        def run_block(block_in, r0, r1, force_exact=False):
            excl = None if exclude is None else kernels.DeviceExclusion.upload(
                *kernels.exclusion_host_csr(exclude, item_id_offset, n_items, r0, r1), device=device)
            if path == 'dense+rank':
                return self._topk_from_dense(r1 - r0, n_items, k, item_id_offset, device,
                                             lambda: dense_scores(block_in, r0, r1), excl), [(None, 0)]
            if path == 'wide' and n_items == 0:     # an empty item shard: no candidates, the calls of the other ranks
                return kernels.empty_topk(r1 - r0, k, device), [(torch.zeros((4,), dtype=torch.int32, device=device), 0)]
            return fused(block_in, r0, r1, 'exact3' if force_exact and path == 'filter' else path, excl)

        results, counters, rows = [], [], []
        for (r0, r1, block_in) in blocks:
            top, sweeps = run_block(block_in, r0, r1)
            top, block_rows = exchange(top, r0, r1)
            results.append(top)
            counters.append(sweeps)
            rows.append(block_rows)

        live = [c for sweeps in counters for c, _ in sweeps if c is not None]
        if live:
            counts = iter(torch.stack([c[0] for c in live]).cpu().numpy().tolist())
            overflow = []
            for b, sweeps in enumerate(counters):
                for c, cap in sweeps:
                    if c is None:
                        continue
                    n_bad = next(counts)
                    info['fallback_rows'] += min(n_bad, cap)
                    if n_bad > cap and b not in overflow:
                        overflow.append(b)
            if gather_group is not None:     # every rank must take the same decision: the exchange is collective
                from . import distributed
                overflow = distributed.union_of_indices(overflow, len(blocks), gather_group, device)
            for b in overflow:
                r0, r1, block_in = blocks[b]
                top, _ = run_block(block_in, r0, r1, force_exact=True)
                results[b], rows[b] = exchange(top, r0, r1)
            info['overflow_blocks'] = len(overflow)
        return results, rows

    @staticmethod
    def _topk_result(results, to_host):
        """The PackedTopK of consecutive row blocks -> one TopK (device tensors, or numpy arrays with to_host)."""
        top_s = results[0].scores if len(results) == 1 else torch.cat([r.scores for r in results])
        top_i = results[0].items if len(results) == 1 else torch.cat([r.items for r in results])
        if not to_host:
            return TopK(top_i, top_s)
        return TopK(*kernels.to_host(top_i, top_s))

    def _topk_block_rows(self, path, n_rows, n_items, k, gather_group=None, device=None, n_tastes=1):
        """Default rows per block of a top-k call: every row at once on the k <= 32 fused routes; on dense+rank as many
        as keep the dense scores, ranks and selection masks within PREDICT_BLOCK_BYTES; on the wide routes ('wide',
        'exact3_wide') as many as keep the lists within PREDICT_BLOCK_BYTES at one item split per row, and with
        n_tastes > 1 (a user x item
        call of a mixture of tastes) the running, per-taste and merged PackedTopK of the pairwise fold (3 x 8k bytes per
        row) as well.  (A block splits the items only when it has fewer user blocks than the device has SMs; its rows x
        splits then stay below ~3 x 128 x the SM count, about 1.2 GB of lists at k = 1024 on an H100.)  In a sharded call
        (gather_group) every rank takes the smallest of the ranks' choices: each block ends in the collective exchange,
        so all ranks must cut the same blocks."""
        if path in ('wide', 'exact3_wide'):
            if path == 'wide':
                per_row = 8 * kernels.wide_list_capacity(k)
            else:      # two lists per row (the column halves) and their counts
                per_row = 2 * (8 * kernels.exact_wide_list_capacity(k) + 4)
            if n_tastes > 1:
                per_row += 3 * 8 * k
            rows = max(2 * kernels.TILE_USERS, self.PREDICT_BLOCK_BYTES // per_row // 256 * 256)
        elif path == 'dense+rank':
            rows = kernels.dense_rank_rows(n_items, self.PREDICT_BLOCK_BYTES)
        else:
            rows = n_rows
        if gather_group is not None:
            from . import distributed
            rows = distributed.common_block_rows(rows, gather_group, device)
        return rows

    def _topk_path(self, k, n_items, model_ok, single_taste, **route):
        """The route of a top-k call: topk_route(...) with the k limits of this model's kernels (the per-taste lists of
        the wide routes merge pairwise, up to WIDE_MAX_K, the k limit of the exact kernel's wide mode too).  Starts
        last_topk_info."""
        d_pad = kernels.d_pad_for(self.n_components)
        limits = (kernels.filter_max_k(), kernels.topk_max_k(d_pad)) if model_ok else (0, 0)
        path = topk_route(k, n_items, model_ok, single_taste, *limits, merge_max_k=WIDE_MAX_K,
                          exact_wide_max_k=WIDE_MAX_K if model_ok else 0, **route)
        self.last_topk_info = {'path': path, 'fallback_rows': 0}
        return path

    def _topk_from_dense(self, n_users, n_items, k, item_id_offset, device, score, excl=None):
        """Any model the fused kernel does not cover: dense scores -> exact full ranks -> the rank <= k entries.
        score() -> the float32 [n_users, n_items] scores of the rows on the device.  excl: the rows' DeviceExclusion
        -- those scores become -inf before the ranking and those entries are never emitted (their slots keep the
        sentinel)."""
        if n_items == 0:
            return kernels.empty_topk(n_users, k, device)
        ex = (None, None) if excl is None else kernels.exclusion_pairs(excl, torch.arange(n_users, device=device))
        return kernels.topk_from_scores(score(), k, item_id_offset, *ex)

    def predict_similar_items(self, item_features, item_ids, n_similar):
        """tensorrec/tensorrec.py:666-703: for each id, the n_similar (item_id, score) pairs of highest prediction
        between that item's representation and every item's.
        For whole catalogues (no [len(item_ids), n_items] matrix), use predict_similar_items_top_k."""
        if self.tf_prediction is None:
            raise ModelNotFitException(method='predict_similar_items')
        device = self._cuda_device()
        item_in = self._single_input(item_features, 'item_features')
        pred_graph = self.prediction_graph_factory
        builtin = type(pred_graph) in _BUILTIN_PRED
        extra = 1 if (builtin and pred_graph.b200_kind == 'cosine') else 0
        item_repr, _, _ = self._represent(self.item_repr_graph_factory, item_in, self.n_item_features, 'item', device,
                                          extra)
        ids = torch.as_tensor(np.asarray(item_ids), dtype=torch.long, device=device)
        gathered = item_repr[ids].contiguous()
        if builtin:
            sims = kernels.score_exact(gathered, item_repr, mode=1 if pred_graph.b200_kind == 'euclidean' else 0)
        else:
            with torch.no_grad():
                sims = pred_graph.connect_dense_prediction_graph(tf_user_representation=gathered,
                                                                 tf_item_representation=item_repr)
        sims = sims.cpu().numpy()
        results = []
        for i in range(len(item_ids)):
            item_sims = sims[i]
            best = np.argpartition(item_sims, -n_similar)[-n_similar:]
            results.append(sorted(zip(best, item_sims[best]), key=lambda x: -x[1]))
        return results

    def predict_similar_items_top_k(self, item_features, n_similar, item_ids=None, exclude=None, exclude_self=False,
                                    to_host=True, item_batch_size=None):
        """The n_similar most similar items of every query item, without materialising the [n_queries, n_items]
        similarity matrix: TopK(items int32 [n_queries, n_similar], scores float32 [n_queries, n_similar]).

        Similarity is predict_similar_items' score: the prediction graph (dot, cosine or Euclidean for the built-in
        graphs) between the query's item representation and every item's, without biases (biased, n_tastes and the
        attention graph do not enter it).  Row q holds the n_similar best items of query q in reference rank order
        (score descending, lower item id first on ties); slots that cannot be filled hold (id 2**31 - 1, score -inf).

        item_ids: 1-D integer array-like of query item ids in [0, n_items) (duplicates allowed); None = every item, in
        order (the whole "related items" table).  exclude: None or a scipy sparse matrix [n_queries, n_items] with the
        rules of predict_top_k's `exclude` (duplicates summed; a pair is excluded when its sum is non-zero).
        exclude_self: also exclude every query's own id (the reference returns the item itself, hence the default False).
        item_batch_size: queries are processed in blocks of this many rows (bit-identical results).

        Built-in prediction and representation graphs with n_components <= 128 and n_similar <= 32 run on the fused
        tensor-core top-k kernels (filter + re-scoring for n_similar <= 12, else the exact 3-pass kernel), and with
        32 < n_similar <= WIDE_MAX_K on catalogues of at least WIDE_MIN_ITEMS items on the wide filter; Euclidean
        similarity ranks -1/2 d^2 = q.i - 1/2 |q|^2 - 1/2 |i|^2 there and is mapped to -sqrt(d^2) at the end.  Everything
        else scores dense query blocks and ranks them.  last_topk_info['path'] names the route.  Single GPU: queries
        and items live on one device (there is no item-sharded form)."""
        if self.tf_prediction is None:
            raise ModelNotFitException(method='predict_similar_items_top_k')
        item_in = self._single_input(item_features, 'item_features')
        self._check_features(item_in, self.n_item_features, 'item')
        n_items = item_in.shape[0]
        n = int(n_similar)
        if n < 1:
            raise ValueError('n_similar must be >= 1')
        ids = None
        if item_ids is not None:
            ids = np.asarray(item_ids)
            if ids.ndim != 1:
                raise ValueError('item_ids must be a 1-D array of item ids')
            if ids.size == 0:
                ids = ids.astype(np.int64)
            if not np.issubdtype(ids.dtype, np.integer):
                raise ValueError('item_ids must hold integers')
            if ids.size and (ids.min() < 0 or ids.max() >= n_items):
                raise ValueError('item_ids must lie in [0, %d)' % n_items)
            ids = ids.astype(np.int64)
        n_queries = n_items if ids is None else ids.shape[0]
        if exclude is not None:
            exclude = _checked_exclude(exclude, n_queries, n_items, n, 0, False)
        mask = _similar_exclusion_mask(exclude, exclude_self, ids, n_queries, n_items)

        pred_graph = self.prediction_graph_factory
        kind = pred_graph.b200_kind if type(pred_graph) in _BUILTIN_PRED else None
        euclidean = kind == 'euclidean'
        device = self._cuda_device()
        d_pad = kernels.d_pad_for(self.n_components)
        model_ok = (SCORE_PATH != 'exact' and kind is not None and type(self.item_repr_graph_factory) in _BUILTIN_REPR
                    and d_pad <= 128)
        if SCORE_PATH == 'tensor' and not model_ok:
            raise RuntimeError('TENSORREC_B200_SCORE_PATH=tensor but this model cannot use the tensor-core kernel')
        path = self._topk_path(n, n_items, model_ok, True)
        fused = path != 'dense+rank'
        if n_queries == 0:
            return TopK(np.zeros((0, n), np.int32), np.zeros((0, n), np.float32))
        ids_dev = None if ids is None else torch.from_numpy(ids).to(device)

        def take(t, q0, q1):
            """Rows of the queries [q0, q1) of a per-item tensor (a view when the queries are all items in order)."""
            if t is None:
                return None
            return t[q0:q1] if ids_dev is None else t.index_select(0, ids_dev[q0:q1])

        extra = 1 if kind == 'cosine' else 0
        sweep = dense_scores = None
        if fused:
            # the item operand once: split fp16 + scale (+ row norms and statistics for the filter), no projected biases;
            # Euclidean: bias -1/2 |i|^2.  The queries are rows of this same operand.
            one_pass = path in ('filter', 'wide')
            stats = torch.empty((3,), dtype=torch.float32, device=device) if one_pass else None
            out = self._represent(self.item_repr_graph_factory, item_in, self.n_item_features, 'item', device, extra,
                                  want_f32=False, split_d_pad=d_pad, want_norm=one_pass, stats=stats)
            split, scale, norm = out[1], out[2], (out[3] if one_pass else None)
            bias = kernels.operand_half_sqnorm(split, scale, d_pad) if euclidean else None
            items = kernels.SideOperands(None, split, scale, bias, n_items, self.n_components, d_pad, stats=stats)
            fitems = kernels.FilterItems(items) if one_pass else None

            def sweep(_, q0, q1, route, excl):
                queries = kernels.SideOperands(None, take(split, q0, q1), take(scale, q0, q1), take(bias, q0, q1),
                                               q1 - q0, self.n_components, d_pad, norm=take(norm, q0, q1))
                top, cnt, cap = kernels.topk_fused(route, queries, items, n, fitems=fitems, excl=excl,
                                                   euclidean=euclidean, block_bytes=self.PREDICT_BLOCK_BYTES)
                return top, [(cnt, cap)]
        else:
            item_repr = self._represent(self.item_repr_graph_factory, item_in, self.n_item_features, 'item', device,
                                        extra)[0]

            def dense_scores(_, q0, q1):
                gathered = take(item_repr, q0, q1).contiguous()
                if kind is not None:
                    return kernels.score_exact(gathered, item_repr, mode=1 if euclidean else 0)
                with torch.no_grad():
                    sims = pred_graph.connect_dense_prediction_graph(tf_user_representation=gathered,
                                                                     tf_item_representation=item_repr)
                return sims.to(torch.float32).contiguous()

        if item_batch_size is not None:
            step = max(1, int(item_batch_size))
        else:
            step = self._topk_block_rows(path, n_queries, n_items, n)
        blocks = [(q0, min(n_queries, q0 + step), None) for q0 in range(0, n_queries, step)]
        results, _ = self._run_topk_blocks(path, n, blocks, n_items, 0, mask, sweep, dense_scores,
                                           lambda top, q0, q1: (top, None))
        if fused and euclidean and path != 'wide':     # (the wide route maps its survivors in the selection kernel)
            for top in results:
                kernels.topk_euclidean_finish(top)
        return self._topk_result(results, to_host)

    def predict_user_representation(self, user_features):
        """[n_users, n_components] (or [n_tastes, n_users, n_components] when n_tastes > 1) (tensorrec.py:735-762)."""
        if self.tf_prediction is None:
            raise ModelNotFitException(method='predict_user_representation')
        device = self._cuda_device()
        user_in = self._single_input(user_features, 'user_features')
        self._check_features(user_in, self.n_user_features, 'user')
        user_repr = torch.stack([self._represent(self.user_repr_graph_factory, user_in, self.n_user_features,
                                                 'user_{}'.format(t), device)[0]
                                 for t in range(self.n_tastes)]).cpu().numpy()
        if self.n_tastes == 1:
            user_repr = np.sum(user_repr, axis=0)
        return user_repr

    def predict_user_attention_representation(self, user_features):
        """tensorrec.py:764-793."""
        if self.tf_prediction is None:
            raise ModelNotFitException(method='predict_user_attention_representation')
        if self.attention_graph_factory is None:
            raise ModelWithoutAttentionException()
        device = self._cuda_device()
        user_in = self._single_input(user_features, 'user_features')
        attn = torch.stack([self._represent(self.attention_graph_factory, user_in, self.n_user_features,
                                            'attn_{}'.format(t), device)[0]
                            for t in range(self.n_tastes)]).cpu().numpy()
        if self.n_tastes == 1:
            attn = np.sum(attn, axis=0)
        return attn

    def predict_item_representation(self, item_features):
        """[n_items, n_components] (tensorrec.py:795-816)."""
        if self.tf_prediction is None:
            raise ModelNotFitException(method='predict_item_representation')
        device = self._cuda_device()
        item_in = self._single_input(item_features, 'item_features')
        self._check_features(item_in, self.n_item_features, 'item')
        return self._represent(self.item_repr_graph_factory, item_in, self.n_item_features, 'item',
                               device)[0].cpu().numpy()

    def predict_user_bias(self, user_features):
        """[n_users] (tensorrec.py:818-842)."""
        if self.tf_prediction is None:
            raise ModelNotFitException(method='predict_user_bias')
        if not self.biased:
            raise ModelNotBiasedException(actor='user')
        device = self._cuda_device()
        user_in = self._single_input(user_features, 'user_features')
        return self._projected_biases(user_in, 'feature_biases_user', device).cpu().numpy()

    def predict_item_bias(self, item_features):
        """[n_items] (tensorrec.py:844-868)."""
        if self.tf_prediction is None:
            raise ModelNotFitException(method='predict_item_bias')
        if not self.biased:
            raise ModelNotBiasedException(actor='item')
        device = self._cuda_device()
        item_in = self._single_input(item_features, 'item_features')
        return self._projected_biases(item_in, 'feature_biases_item', device).cpu().numpy()

    # ------------------------------------------------------------------------------------------------
    # persistence (tensorrec.py:870-917): weights as .npz beside the pickled Python object
    # ------------------------------------------------------------------------------------------------
    def __getstate__(self):
        state = dict(self.__dict__)
        state['_variables'] = collections.OrderedDict()
        state['_optimizer'] = None
        state['_optimizer_params'] = None
        state['_was_fit'] = self.tf_prediction is not None
        state.pop('_stream_buffers', None)
        state['_wmrb_step'] = None
        for name in self._all_hook_names():
            state[name] = None
        return state

    def save_model(self, directory_path):
        if self.tf_prediction is None:
            raise ModelNotFitException(method='save_model')
        if not os.path.exists(directory_path):
            os.makedirs(directory_path)
        np.savez(os.path.join(directory_path, 'tensorrec_session.npz'), **self.get_weights())
        with open(os.path.join(directory_path, 'tensorrec.pkl'), 'wb') as file:
            pickle.dump(file=file, obj=self)

    @classmethod
    def load_model(cls, directory_path):
        with open(os.path.join(directory_path, 'tensorrec.pkl'), 'rb') as file:
            model = pickle.load(file=file)
        with np.load(os.path.join(directory_path, 'tensorrec_session.npz')) as data:
            weights = collections.OrderedDict((k, data[k]) for k in data.files)
        model.set_weights(weights, n_user_features=model.n_user_features, n_item_features=model.n_item_features)
        return model
