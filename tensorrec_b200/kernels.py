"""Host-side launch layer: torch supplies device memory and streams, every computation is a call through the C ABI
(libtensorrec_b200.so).  No function here has a CPU path; all of them raise without a CUDA device."""
import collections
import ctypes

import numpy as np
import scipy.sparse as sp
import torch

from . import _lib

import os as _os
BIAS_ORDER = _os.environ.get('TENSORREC_B200_BIAS_ORDER', 'kernel')   # 'kernel' (trk_rank_full + trk_order_from_ranks) | 'torch'

TILE_ITEMS = 256     # item tile of the tensor-core kernel (item_meta is padded to a multiple of this)
TILE_USERS = 128


def require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError('tensorrec_b200 runs its predict / predict_rank path on a CUDA device (H100, sm_90a) only; '
                           'no CUDA device is visible and there is no CPU fallback')
    return _lib.load()


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _f32(t, device):
    if isinstance(t, np.ndarray):
        t = torch.from_numpy(np.ascontiguousarray(t, dtype=np.float32))
    return t.to(device=device, dtype=torch.float32).contiguous()


def d_pad_for(n_components):
    """Width of the split-fp16 operand: n_components rounded up to the 64-element swizzle row."""
    return ((int(n_components) + 63) // 64) * 64


class DeviceCSR(object):
    """Sparse features resident in HBM as CSR: int32 indptr[rows+1], int32 col[nnz], float32 val[nnz].

    Replaces the 5-tuple (row i64, col i64, val f32, d0, d1) of tensorrec/input_utils.py:15-40 and the
    tf.SparseTensor built from it (tensorrec/tensorrec.py:285-293).  Entry order inside a row is the order the
    reference's COO conversion yields (stable row sort), duplicates are kept, values are cast to float32."""

    def __init__(self, indptr, col, val, shape):
        self.indptr, self.col, self.val = indptr, col, val
        self.shape = (int(shape[0]), int(shape[1]))

    @property
    def nnz(self):
        return int(self.col.numel())

    @staticmethod
    def host_arrays(matrix):
        """scipy sparse matrix -> (indptr i32, col i32, val f32) numpy arrays, reference entry order."""
        if not sp.issparse(matrix):
            raise ValueError('Input must be a scipy sparse matrix')
        if matrix.shape[0] >= 2 ** 31 - 1 or matrix.shape[1] >= 2 ** 31 - 1 or matrix.nnz >= 2 ** 31 - 1:
            raise ValueError('feature matrix exceeds int32 indexing')
        if isinstance(matrix, sp.csr_matrix):
            # sp.coo_matrix(csr) walks the rows in storage order: the CSR arrays already are that order
            return (np.ascontiguousarray(matrix.indptr, dtype=np.int32),
                    np.ascontiguousarray(matrix.indices, dtype=np.int32),
                    np.ascontiguousarray(matrix.data, dtype=np.float32))
        coo = matrix if isinstance(matrix, sp.coo_matrix) else sp.coo_matrix(matrix)     # input_utils.py:29-30
        order = np.argsort(coo.row, kind='stable')
        counts = np.bincount(coo.row, minlength=coo.shape[0])
        indptr = np.zeros(coo.shape[0] + 1, dtype=np.int64)
        np.cumsum(counts, out=indptr[1:])
        return (indptr.astype(np.int32), np.ascontiguousarray(coo.col[order], dtype=np.int32),
                np.ascontiguousarray(coo.data[order], dtype=np.float32))

    @staticmethod
    def host_arrays_transposed(matrix):
        """CSR arrays of the TRANSPOSE (one row per feature column), entries of a column in ascending row order and,
        within a row, in reference entry order; duplicates are kept.  K1 on these arrays is the backward of K1:
        dW = A^T . dRepr (tf.sparse_tensor_dense_matmul's gradient w.r.t. the dense operand)."""
        indptr, col, val = DeviceCSR.host_arrays(matrix)
        n_rows, n_cols = matrix.shape
        rows = np.repeat(np.arange(n_rows, dtype=np.int32), np.diff(indptr))
        order = np.argsort(col, kind='stable')
        counts = np.bincount(col, minlength=n_cols)
        indptr_t = np.zeros(n_cols + 1, dtype=np.int64)
        np.cumsum(counts, out=indptr_t[1:])
        return indptr_t.astype(np.int32), np.ascontiguousarray(rows[order]), np.ascontiguousarray(val[order])

    @classmethod
    def from_scipy_transposed(cls, matrix, device='cuda'):
        require_cuda()
        indptr, col, val = cls.host_arrays_transposed(matrix)
        up = lambda a: torch.from_numpy(a).to(device, non_blocking=True)   # noqa: E731
        return cls(up(indptr), up(col), up(val), (matrix.shape[1], matrix.shape[0]))

    @classmethod
    def from_scipy(cls, matrix, device='cuda', pin=False):
        require_cuda()
        indptr, col, val = cls.host_arrays(matrix)

        def up(a):
            t = torch.from_numpy(a)
            if pin:
                t = t.pin_memory()
            return t.to(device, non_blocking=True)

        return cls(up(indptr), up(col), up(val), matrix.shape)

    def h2d_bytes(self):
        return 4 * (self.indptr.numel() + self.col.numel() + self.val.numel())


K1_MAX_WIDTH = 512      # widest row one K1 launch covers (256 when the width is not a multiple of 4)


def gather_reduce(csr, weights, n_normalize=0, want_f32=True, split_d_pad=None, want_norm=False, stats=None,
                  split_out=None, out_f32=None):
    """K1.  Returns (repr_f32 or None, split or None, scale or None[, norm]).

    want_norm: also return the row norms (upper bounds) formed in K1's epilogue; stats: float32[3] that receives the
    max norm / max row scale (zeroed by the call).  Both feed the filter form of the fused top-k.
    split_out: (split [rows, 2 split_d_pad] fp16, scale [rows] f32) contiguous tensors -- e.g. one operand's slice of a
    stacked mixture-of-tastes operand -- that K1 writes instead of new ones.  out_f32: a contiguous float32 [rows, d]
    tensor K1 writes the representation to instead of a new one (e.g. one plane of the training step's operand)."""
    lib = require_cuda()
    rows, n_features = csr.shape
    d = int(weights.shape[1])
    if int(weights.shape[0]) != n_features:
        raise ValueError('feature matrix has %d columns but the weights have %d rows' % (n_features, weights.shape[0]))
    dev = weights.device
    if split_d_pad is None and not want_norm and stats is None and (d > K1_MAX_WIDTH or (d % 4 != 0 and d > 256)):
        return _gather_reduce_wide(csr, weights, n_normalize), None, None
    out = None
    if want_f32:
        out = torch.empty((rows, d), dtype=torch.float32, device=dev) if out_f32 is None else out_f32
    split = scale = norm = None
    d_pad = 0
    if split_d_pad is not None:
        d_pad = int(split_d_pad)
        if split_out is not None:
            split, scale = split_out
        else:
            split = torch.empty((rows, 2 * d_pad), dtype=torch.float16, device=dev)
            scale = torch.empty((rows,), dtype=torch.float32, device=dev)
    if want_norm:
        norm = torch.empty((rows,), dtype=torch.float32, device=dev)
    rc = lib.trk_csr_gather_reduce_f32(_p(csr.indptr), _p(csr.col), _p(csr.val), _p(weights), rows, n_features, d,
                                       int(n_normalize), _p(out), _p(split), d_pad, _p(scale), _p(norm), _p(stats),
                                       _stream())
    _lib.check(rc, 'trk_csr_gather_reduce_f32')
    if want_norm:
        return out, split, scale, norm
    return out, split, scale


def _gather_reduce_wide(csr, weights, n_normalize):
    """Rows wider than one K1 launch covers (n_components > 512, e.g. the 4 x n_components hidden layer of a
    ReLURepresentationGraph): the component axis is cut into column blocks of at most 512, one K1 launch each (every
    output element is still the same fp32 FMA chain in CSR order), normalisation afterwards over the whole row."""
    rows = csr.shape[0]
    d = int(weights.shape[1])
    out = torch.empty((rows, d), dtype=torch.float32, device=weights.device)
    step = K1_MAX_WIDTH
    for c0 in range(0, d, step):
        c1 = min(d, c0 + step)
        block, _, _ = gather_reduce(csr, weights[:, c0:c1].contiguous(), want_f32=True)
        out[:, c0:c1] = block
    for _ in range(int(n_normalize)):
        _l2_normalize_rows_any_width_(out)
    return out


def _l2_normalize_rows_any_width_(x):
    if x.shape[1] <= 1024:
        return l2_normalize_rows_(x)
    # tf.nn.l2_normalize: x * rsqrt(max(sum x^2, 1e-12)); rows this wide are outside every kernel's row shape
    x.mul_(torch.rsqrt(torch.clamp((x * x).sum(dim=1, keepdim=True), min=1e-12)))
    return x


def split_f32(repr_f32, n_normalize=0, d_pad=None, out=None):
    """out: (split, scale) tensors to write, as gather_reduce's split_out."""
    lib = require_cuda()
    rows, d = repr_f32.shape
    d_pad = d_pad_for(d) if d_pad is None else int(d_pad)
    if out is not None:
        split, scale = out
    else:
        split = torch.empty((rows, 2 * d_pad), dtype=torch.float16, device=repr_f32.device)
        scale = torch.empty((rows,), dtype=torch.float32, device=repr_f32.device)
    rc = lib.trk_split_f32_to_f16x2(_p(repr_f32), rows, d, int(n_normalize), _p(split), d_pad, _p(scale), _stream())
    _lib.check(rc, 'trk_split_f32_to_f16x2')
    return split, scale


def l2_normalize_rows_(x):
    lib = require_cuda()
    rc = lib.trk_l2_normalize_rows_f32(_p(x), x.shape[0], x.shape[1], _stream())
    _lib.check(rc, 'trk_l2_normalize_rows_f32')
    return x


def project_biases(csr, feature_biases):
    lib = require_cuda()
    if int(feature_biases.numel()) != csr.shape[1]:
        raise ValueError('feature matrix has %d columns but there are %d feature biases'
                         % (csr.shape[1], feature_biases.numel()))
    out = torch.empty((csr.shape[0],), dtype=torch.float32, device=feature_biases.device)
    rc = lib.trk_csr_project_biases_f32(_p(csr.indptr), _p(csr.col), _p(csr.val), _p(feature_biases), csr.shape[0],
                                        _p(out), _stream())
    _lib.check(rc, 'trk_csr_project_biases_f32')
    return out


def score_exact(user_repr, item_repr, user_bias=None, item_bias=None, mode=0, attention_repr=None, out=None):
    """K2 on CUDA cores (exact fp32).  user_repr [T, U, d] or [U, d]; returns [U, I] float32."""
    lib = require_cuda()
    if user_repr.dim() == 2:
        user_repr = user_repr.unsqueeze(0)
    user_repr = user_repr.contiguous()
    n_tastes, n_users, d = user_repr.shape
    n_items = item_repr.shape[0]
    if item_repr.shape[1] != d:
        raise ValueError('user and item representations differ in n_components (%d vs %d)' % (d, item_repr.shape[1]))
    if out is None:
        out = torch.empty((n_users, n_items), dtype=torch.float32, device=user_repr.device)
    # grid.y carries 64-row user tiles (<= 65535 per launch): block the user axis for very tall inputs
    max_rows = 65535 * 64
    for u0 in range(0, max(n_users, 1), max_rows):
        u1 = min(n_users, u0 + max_rows)
        ur = user_repr[:, u0:u1].contiguous() if (u0 > 0 or u1 < n_users) else user_repr
        ub = None if user_bias is None else user_bias[u0:u1]
        if attention_repr is not None:
            ar = attention_repr[:, u0:u1].contiguous()
            rc = lib.trk_score_attention_f32(_p(ur), _p(ar), _p(item_repr), _p(ub), _p(item_bias), _p(out[u0:u1]),
                                             u1 - u0, n_items, d, n_tastes, _stream())
            _lib.check(rc, 'trk_score_attention_f32')
        else:
            rc = lib.trk_score_f32(_p(ur), _p(item_repr), _p(ub), _p(item_bias), _p(out[u0:u1]), u1 - u0, n_items, d,
                                   n_tastes, int(mode), _stream())
            _lib.check(rc, 'trk_score_f32')
    return out


def rank_full(scores):
    """K3 (full): the reference's rank_predictions on a dense [U, I] float32 matrix -> int32 ranks."""
    lib = require_cuda()
    scores = scores.contiguous()
    n_users, n_items = scores.shape
    ranks = torch.empty((n_users, n_items), dtype=torch.int32, device=scores.device)
    need = int(lib.trk_rank_full_workspace_bytes(n_users, n_items))
    ws = torch.empty((max(need, 8) // 8,), dtype=torch.int64, device=scores.device) if need else None
    rc = lib.trk_rank_full(_p(scores), _p(ranks), n_users, n_items, _p(ws), need, _stream())
    _lib.check(rc, 'trk_rank_full')
    return ranks


def padded_items(n_items):
    return ((int(n_items) + TILE_ITEMS - 1) // TILE_ITEMS) * TILE_ITEMS


def pack_item_meta(item_scale, item_bias, n_items):
    lib = require_cuda()
    n_pad = padded_items(n_items)
    meta = torch.empty((n_pad, 2), dtype=torch.float32, device=item_scale.device)
    rc = lib.trk_pack_item_meta(_p(item_scale), _p(item_bias), n_items, _p(meta), n_pad, _stream())
    _lib.check(rc, 'trk_pack_item_meta')
    return meta


def topk_max_k(d_pad):
    return int(require_cuda().trk_score_topk_max_k(int(d_pad)))


def default_splits(n_users, n_items):
    """Item-range splits so that (user blocks x splits) covers every SM about twice when there are few users."""
    n_sm = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    n_ub = (n_users + TILE_USERS - 1) // TILE_USERS
    n_tiles = (n_items + TILE_ITEMS - 1) // TILE_ITEMS
    if n_ub >= n_sm:
        return 1
    return int(max(1, min(n_tiles, 256, (2 * n_sm + n_ub - 1) // n_ub)))


def score_topk(user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad, k, n_splits=None,
               item_id_offset=0, n_users_live=None, excl=None, excl_row_map=None, sqnorms=None):
    """K2+K3 fused.  Returns (cand_score [U, n_splits, k] f32, cand_item [U, n_splits, k] i32).
    n_users_live: device int32 tensor; only its first element's worth of user rows is processed.
    excl: DeviceExclusion -- its items are left out of every row's top-k (user row u reads list row excl_row_map[u]).
    sqnorms: (user -1/2 |u|^2, item -1/2 |i|^2 padded by item_half_sqnorm) -> Euclidean similarity scores."""
    lib = require_cuda()
    if n_splits is None:
        n_splits = default_splits(n_users, n_items)
    dev = user_split.device
    cand_score = torch.empty((n_users, n_splits, k), dtype=torch.float32, device=dev)
    cand_item = torch.empty((n_users, n_splits, k), dtype=torch.int32, device=dev)
    if sqnorms is not None:
        name = 'trk_score_topk_euclid_f16x3'
        extra = (None, None, None) if excl is None else (_p(excl.indptr), _p(excl.ids), _p(excl_row_map))
        extra += (_p(sqnorms[0]), _p(sqnorms[1]))
    elif excl is None:
        name, extra = 'trk_score_topk_f16x3', ()
    else:
        name, extra = 'trk_score_topk_f16x3_excl', (_p(excl.indptr), _p(excl.ids), _p(excl_row_map))
    rc = getattr(lib, name)(_p(user_split), _p(user_scale), _p(user_bias), _p(item_split), _p(item_meta), n_users,
                            n_items, int(d_pad), int(k), int(n_splits), int(item_id_offset), _p(cand_score),
                            _p(cand_item), _p(n_users_live), *extra, _stream())
    _lib.check(rc, name)
    return cand_score, cand_item


def score_dense_tc(user_split, user_scale, user_bias, item_split, item_meta, n_users, n_items, d_pad, out=None,
                   sqnorms=None):
    """sqnorms: as for score_topk (Euclidean similarity)."""
    lib = require_cuda()
    if out is None:
        out = torch.empty((n_users, n_items), dtype=torch.float32, device=user_split.device)
    args = (_p(user_split), _p(user_scale), _p(user_bias), _p(item_split), _p(item_meta), n_users, n_items, int(d_pad),
            _p(out), out.stride(0))
    if sqnorms is None:
        name, extra = 'trk_score_dense_f16x3', ()
    else:
        name, extra = 'trk_score_dense_euclid_f16x3', (_p(sqnorms[0]), _p(sqnorms[1]))
    rc = getattr(lib, name)(*args, *extra, _stream())
    _lib.check(rc, name)
    return out


# ---------------------------------------------------------------------------------------------------------------
# mixtures of tastes on the tensor-core kernels: every user's n_ops operand rows (u_0 .. u_{T-1}, then a_0 .. a_{T-1}
# with attention) stacked as [n_ops, U, 2 d_pad]; the kernel collapses the tastes per (user, item)
# ---------------------------------------------------------------------------------------------------------------
TASTES_MAX_OPS = 64      # operand rows per user the kernel holds: one consumer warpgroup's accumulator rows


def tastes_n_ops(n_tastes, attention):
    return int(n_tastes) * (2 if attention else 1)


def tastes_plan(n_tastes, attention):
    """Block layout of the taste-collapsing kernel: (users per warpgroup P, users per 128-row block 2P, accumulator
    rows used per warpgroup n_ops * P, out of 64).  None when n_ops is outside [2, TASTES_MAX_OPS]."""
    n_ops = tastes_n_ops(n_tastes, attention)
    if n_ops < 2 or n_ops > TASTES_MAX_OPS:
        return None
    per_wg = TASTES_MAX_OPS // n_ops
    return per_wg, 2 * per_wg, n_ops * per_wg


def _tastes_entry(name, users, item_hsq):
    """The entry point of a mixture of tastes (name: trk_score_<mode>_tastes) and its trailing norm arguments: the
    Euclidean form (..._tastes_euclid_f16x3, users.hsq and item_hsq) when item_hsq is given."""
    if item_hsq is None:
        return name + '_f16x3', ()
    if users.hsq is None:
        raise ValueError('a Euclidean mixture of tastes needs the operand norms (SideOperands.hsq)')
    return name + '_euclid_f16x3', (_p(users.hsq), _p(item_hsq))


def score_topk_tastes(users, items, meta, n_tastes, attention, k, n_splits=None, item_id_offset=0, excl=None,
                      excl_row_map=None, item_hsq=None):
    """The fused top-k of a mixture of tastes (users: stacked SideOperands).  item_hsq (item_half_sqnorm(items)):
    Euclidean prediction, with the operand norms users.hsq.  Returns (cand_score, cand_item) [U, n_splits, k]."""
    lib = require_cuda()
    n_users = users.n_rows
    if n_splits is None:
        n_splits = default_splits(n_users, items.n_rows)
    dev = users.split.device
    cand_score = torch.empty((n_users, n_splits, k), dtype=torch.float32, device=dev)
    cand_item = torch.empty((n_users, n_splits, k), dtype=torch.int32, device=dev)
    ex = (None, None, None) if excl is None else (_p(excl.indptr), _p(excl.ids), _p(excl_row_map))
    name, norms = _tastes_entry('trk_score_topk_tastes', users, item_hsq)
    rc = getattr(lib, name)(_p(users.split), _p(users.scale), _p(users.bias), int(n_tastes), 1 if attention else 0,
                            _p(items.split), _p(meta), n_users, items.n_rows, int(users.d_pad), int(k), int(n_splits),
                            int(item_id_offset), _p(cand_score), _p(cand_item), *ex, *norms, _stream())
    _lib.check(rc, name)
    return cand_score, cand_item


def topk_tastes(users, items, n_tastes, attention, k, n_splits=None, item_id_offset=0, excl=None, out=None,
                item_hsq=None):
    """Fused top-k of a mixture of tastes + merge -> PackedTopK [U, k].  item_hsq: as for score_topk_tastes."""
    meta = pack_item_meta(items.scale, items.bias, items.n_rows)
    cs, ci = score_topk_tastes(users, items, meta, n_tastes, attention, k, n_splits=n_splits,
                               item_id_offset=item_id_offset, excl=excl, item_hsq=item_hsq)
    return topk_merge(cs, ci, k, out=out)


def score_dense_tastes(users, item_split, item_meta, n_items, n_tastes, attention, out=None, item_hsq=None):
    """Dense scores [U, n_items] of a mixture of tastes (users: stacked SideOperands).  item_hsq: as for
    score_topk_tastes."""
    lib = require_cuda()
    if out is None:
        out = torch.empty((users.n_rows, n_items), dtype=torch.float32, device=users.split.device)
    name, norms = _tastes_entry('trk_score_dense_tastes', users, item_hsq)
    rc = getattr(lib, name)(_p(users.split), _p(users.scale), _p(users.bias), int(n_tastes), 1 if attention else 0,
                            _p(item_split), _p(item_meta), users.n_rows, n_items, int(users.d_pad), _p(out),
                            out.stride(0), *norms, _stream())
    _lib.check(rc, name)
    return out


class PackedTopK(object):
    """Top-k result of a batch of users in the layout the multi-GPU exchange sends: int32 [n_users, 2k], row u =
    k scores (float32 bits) then k item ids.  `scores` / `items` are views."""

    def __init__(self, n_users, k, device, buf=None):
        self.k = int(k)
        self.buf = torch.empty((int(n_users), 2 * self.k), dtype=torch.int32, device=device) if buf is None else buf

    @property
    def n_users(self):
        return int(self.buf.shape[0])

    @property
    def scores(self):
        return self.buf[:, :self.k].view(torch.float32)

    @property
    def items(self):
        return self.buf[:, self.k:]

    def score_ptr(self):
        return ctypes.c_void_p(self.buf.data_ptr())

    def item_ptr(self):
        return ctypes.c_void_p(self.buf.data_ptr() + 4 * self.k)


def empty_topk(n_rows, k, device):
    """PackedTopK [n_rows, k] of sentinels only (id 2**31 - 1, score -inf): the result over an empty catalogue."""
    top = PackedTopK(n_rows, k, device)
    top.scores.fill_(float('-inf'))
    top.items.fill_(2 ** 31 - 1)
    return top


def topk_merge(cand_score, cand_item, k_out, out=None, n_users_live=None):
    """[U, L, k_in] candidate lists -> PackedTopK [U, k_out] (top scores, top item ids)."""
    lib = require_cuda()
    n_users, n_lists, k_in = cand_score.shape
    cand_score, cand_item = cand_score.contiguous(), cand_item.contiguous()
    if out is None:
        out = PackedTopK(n_users, k_out, cand_score.device)
    rc = lib.trk_topk_merge(_p(cand_score), _p(cand_item), n_users, n_lists, k_in, int(k_out), n_lists * k_in, k_in,
                            out.score_ptr(), out.item_ptr(), 2 * out.k, _p(n_users_live), 0, _stream())
    _lib.check(rc, 'trk_topk_merge')
    return out


def topk_merge_received(recv, n_users, n_lists, k, dedup=False):
    """Merge of int32 [n_lists, n_users, 2k] -> PackedTopK [n_users, k]: the exchange receive buffer (list l = the
    candidates rank l found for THIS rank's user slice), or -- with dedup -- the per-taste results of a
    mixture-of-tastes model (list t = the top-k of taste t; an item named by several tastes keeps its best score)."""
    lib = require_cuda()
    out = PackedTopK(n_users, k, recv.device)
    if n_users == 0:
        return out
    base = recv.data_ptr()
    rc = lib.trk_topk_merge(ctypes.c_void_p(base), ctypes.c_void_p(base + 4 * k), n_users, int(n_lists), int(k), int(k),
                            2 * k, n_users * 2 * k, out.score_ptr(), out.item_ptr(), 2 * k, None, 1 if dedup else 0,
                            _stream())
    _lib.check(rc, 'trk_topk_merge')
    return out


def topk_merge_dedup(a, b, out=None):
    """Two PackedTopK [U, k] of the same users -> PackedTopK [U, k]: the top-k of their union with every item once, at
    its higher score (trk_topk_merge_dedup_pair, any k <= wide_max_k()).  The fold of the per-taste lists of a mixture
    of tastes on the wide route; `out` must be a third buffer."""
    lib = require_cuda()
    if a.k != b.k or a.n_users != b.n_users:
        raise ValueError('topk_merge_dedup: lists of [%d, %d] and [%d, %d]' % (a.n_users, a.k, b.n_users, b.k))
    if out is None:
        out = PackedTopK(a.n_users, a.k, a.buf.device)
    if a.n_users == 0:
        return out
    rc = lib.trk_topk_merge_dedup_pair(a.score_ptr(), a.item_ptr(), 2 * a.k, b.score_ptr(), b.item_ptr(), 2 * b.k,
                                       a.n_users, a.k, out.score_ptr(), out.item_ptr(), 2 * out.k, _stream())
    _lib.check(rc, 'trk_topk_merge_dedup_pair')
    return out


# ---------------------------------------------------------------------------------------------------------------
# filter form of the fused top-k: 1 tensor pass + exact fp32 re-scoring of the survivors
# ---------------------------------------------------------------------------------------------------------------
def filter_max_k():
    return int(require_cuda().trk_score_filter_max_k())


def filter_list_width():
    return int(require_cuda().trk_score_filter_list_width())


def operand_stats(split, scale, d_pad, want_norm=True, stats=None):
    """Row norms (upper bounds) of a split operand and, if `stats` (zeroed float32[3]) is given, the global max norm /
    max row scale by device-side atomic max."""
    lib = require_cuda()
    rows = split.shape[0]
    norm = torch.empty((rows,), dtype=torch.float32, device=split.device) if want_norm else None
    rc = lib.trk_operand_stats(_p(split), _p(scale), rows, int(d_pad), _p(norm), _p(stats), _stream())
    _lib.check(rc, 'trk_operand_stats')
    return norm


def operand_half_sqnorm(split, scale, d_pad, out=None):
    """-1/2 |row|^2 of every row of a split operand (fp32 [rows], or the first rows entries of `out`): the biases that
    turn the fused top-k kernels' score q.i + ub + ib into -1/2 d^2(q, i) for Euclidean similar items, and the norms of
    the Euclidean user x item kernels."""
    lib = require_cuda()
    if out is None:
        out = torch.empty((split.shape[0],), dtype=torch.float32, device=split.device)
    rc = lib.trk_operand_half_sqnorm(_p(split), _p(scale), split.shape[0], int(d_pad), _p(out), _stream())
    _lib.check(rc, 'trk_operand_half_sqnorm')
    return out


def item_half_sqnorm(items):
    """-1/2 |i|^2 of an item SideOperands, zero-padded to padded_items(n) entries (the Euclidean kernels read whole
    item tiles)."""
    out = torch.zeros((padded_items(items.n_rows),), dtype=torch.float32, device=items.split.device)
    return operand_half_sqnorm(items.split, items.scale, items.d_pad, out=out)


def topk_euclidean_finish(top):
    """In place on a PackedTopK whose scores are -1/2 d^2: scores become -sqrt(max(d^2, 1e-16)) (the reference's
    Euclidean similarity) and every row is re-sorted by (score desc, id asc)."""
    lib = require_cuda()
    rc = lib.trk_topk_euclidean_finish(top.score_ptr(), top.item_ptr(), 2 * top.k, top.n_users, top.k, _stream())
    _lib.check(rc, 'trk_topk_euclidean_finish')
    return top


def rescale_hi_global(split, scale, stats, d_pad, perm=None):
    lib = require_cuda()
    rows = split.shape[0]
    out = torch.empty((rows, int(d_pad)), dtype=torch.float16, device=split.device)
    rc = lib.trk_rescale_hi_global(_p(split), _p(scale), _p(stats), _p(perm), rows, int(d_pad), _p(out), _stream())
    _lib.check(rc, 'trk_rescale_hi_global')
    return out


def pack_item_bias(item_bias, n_items, stats, device, perm=None, want_min=False):
    """Returns (bias in processing order padded with -inf, max bias per block of 128 positions[, min bias per block])."""
    lib = require_cuda()
    n_pad = padded_items(n_items)
    out = torch.empty((n_pad,), dtype=torch.float32, device=device)
    block_max = torch.empty((n_pad // 128,), dtype=torch.float32, device=device)
    block_min = torch.empty((n_pad // 128,), dtype=torch.float32, device=device) if want_min else None
    rc = lib.trk_pack_item_bias(_p(item_bias), _p(perm), n_items, _p(out), n_pad, _p(stats), _p(block_max),
                                _p(block_min), _stream())
    _lib.check(rc, 'trk_pack_item_bias')
    if want_min:
        return out, block_max, block_min
    return out, block_max


def bias_processing_order(item_bias):
    """Items by DESCENDING bias (stable, so the order is deterministic): int32 perm[position] = item index.
    Highest biases first: the running k-th best rises early, and every later block starts below it by its bias gap."""
    if item_bias is None:
        return None
    if BIAS_ORDER == 'torch':
        return torch.sort(item_bias, descending=True, stable=True).indices.to(torch.int32)
    # own kernels: the reference ranks of the 1 x I bias row (K3: value descending, lower index first on ties), inverted
    lib = require_cuda()
    n = int(item_bias.numel())
    ranks = rank_full(item_bias.contiguous().view(1, n))
    order = torch.empty((n,), dtype=torch.int32, device=item_bias.device)
    rc = lib.trk_order_from_ranks(_p(ranks), n, _p(order), _stream())
    _lib.check(rc, 'trk_order_from_ranks')
    return order


def score_filter(user_split, user_scale, user_bias, user_norm, item_hi, item_stats, item_bias_pad, block_bias_max,
                 item_perm, n_users, n_items, d_pad, k, n_splits=None, item_id_offset=0, block_bias_min=None,
                 excl=None):
    """Filter pass.  Returns (cand_score, cand_item [U, n_splits, 16], theta [U, n_splits]).
    excl: DeviceExclusion with its processing positions formed (exclusion_positions)."""
    lib = require_cuda()
    if n_splits is None:
        n_splits = default_splits(n_users, n_items)
    dev = user_split.device
    width = filter_list_width()      # one list of `width` candidates per (user, split)
    cand_s = torch.empty((n_users, n_splits, width), dtype=torch.float32, device=dev)
    cand_i = torch.empty((n_users, n_splits, width), dtype=torch.int32, device=dev)
    theta = torch.empty((n_users, n_splits), dtype=torch.float32, device=dev)
    if excl is None:
        name, extra = 'trk_score_filter_f16', ()
    else:
        name, extra = 'trk_score_filter_f16_excl', (_p(excl.indptr), _p(excl.pos))
    rc = getattr(lib, name)(_p(user_split), _p(user_scale), _p(user_bias), _p(user_norm), _p(item_hi), _p(item_stats),
                            _p(item_bias_pad), _p(block_bias_max), _p(block_bias_min), _p(item_perm), n_users, n_items,
                            int(d_pad), int(k), int(n_splits), int(item_id_offset), _p(cand_s), _p(cand_i), _p(theta),
                            *extra, _stream())
    _lib.check(rc, name)
    return cand_s, cand_i, theta


def rescore_topk(users, items, cand_item, theta, user_norm, item_stats, k, item_id_offset=0, out=None):
    """Survivors of the filter -> (PackedTopK [U, k], flags int32 [U]); flags mark users the certificate rejects."""
    lib = require_cuda()
    n_users = users.n_rows
    n_lists = theta.numel() // max(n_users, 1)
    width = cand_item.shape[-1]
    dev = users.split.device
    if out is None:
        out = PackedTopK(n_users, k, dev)
    out_f = torch.empty((n_users,), dtype=torch.int32, device=dev)
    rc = lib.trk_rescore_topk_split(_p(users.split), _p(users.scale), _p(items.split), _p(items.scale), _p(users.bias),
                                    _p(items.bias), _p(cand_item), _p(theta), _p(user_norm), _p(item_stats), n_users,
                                    items.n_rows, int(users.d_pad), n_lists, width, int(k), int(item_id_offset),
                                    out.score_ptr(), out.item_ptr(), 2 * out.k, _p(out_f), _stream())
    _lib.check(rc, 'trk_rescore_topk_split')
    return out, out_f


class _HostResults(object):
    """Device -> host copies of results land in page-locked buffers (a pageable destination costs a staging copy and
    page faults: ~3x the time of the PCIe transfer for the 80 MB top-k of 1M users).  The returned numpy arrays ARE the
    pinned buffers; a buffer is recycled only after the array handed out for it (and every view of it) has been
    garbage collected, so results never alias."""

    max_pinned_bytes = 1 << 30   # larger results (a dense [U, I] matrix) use an ordinary pageable copy

    def __init__(self, max_idle_bytes=2 << 30):
        self._idle = []          # [(pinned tensor, weakref to the ndarray handed out)]
        self._max_idle_bytes = max_idle_bytes

    def _take(self, shape, dtype):
        keep, found = [], None
        for buf, ref in self._idle:
            if ref() is not None:
                keep.append((buf, ref))
            elif found is None and buf.dtype == dtype and tuple(buf.shape) == tuple(shape):
                found = buf
            else:
                keep.append((buf, ref))
        self._idle = keep
        if found is None:
            found = torch.empty(tuple(shape), dtype=dtype, pin_memory=True)
        return found

    def fetch(self, *tensors):
        """numpy copies of CUDA tensors, transferred together (one synchronisation)."""
        import weakref
        bufs = []
        for t in tensors:
            t = t.detach().contiguous()
            nbytes = t.numel() * t.element_size()
            if nbytes == 0 or nbytes > self.max_pinned_bytes:
                bufs.append(t.cpu().numpy())      # empty, or too large to page-lock: ordinary pageable copy
                continue
            buf = self._take(t.shape, t.dtype)
            buf.copy_(t, non_blocking=True)
            bufs.append(buf)
        torch.cuda.current_stream().synchronize()
        out = []
        for buf in bufs:
            if isinstance(buf, np.ndarray):
                out.append(buf)
                continue
            arr = buf.numpy()
            self._idle.append((buf, weakref.ref(arr)))
            out.append(arr)
        # bound what sits in the pool once its arrays are gone
        idle_bytes, keep = 0, []
        for buf, ref in reversed(self._idle):
            nbytes = buf.numel() * buf.element_size()
            if ref() is None and idle_bytes + nbytes > self._max_idle_bytes:
                continue
            if ref() is None:
                idle_bytes += nbytes
            keep.append((buf, ref))
        self._idle = list(reversed(keep))
        return out


_host_results = _HostResults()


def to_host(*tensors):
    """CUDA tensors -> numpy arrays through page-locked buffers (see _HostResults)."""
    require_cuda()
    out = _host_results.fetch(*tensors)
    return out[0] if len(out) == 1 else tuple(out)


class SideOperands(object):
    """Everything the score kernels need from one side (users or items), all resident on the device.
    norm: row norms (users, filter path); stats: float32[3] max norm / max scale / max |bias| (items, filter path);
    hsq: -1/2 |x|^2 of every operand row of a stacked operand, [n_ops, U] (a Euclidean mixture of tastes)."""

    def __init__(self, repr_f32, split, scale, bias, n_rows, d, d_pad, norm=None, stats=None, hsq=None):
        self.repr_f32, self.split, self.scale, self.bias = repr_f32, split, scale, bias
        self.n_rows, self.d, self.d_pad = n_rows, d, d_pad
        self.norm, self.stats, self.hsq = norm, stats, hsq

    def rows(self, r0, r1):
        """The operands of rows [r0, r1) (views)."""
        cut = lambda t: None if t is None else t[r0:r1]   # noqa: E731
        return SideOperands(cut(self.repr_f32), cut(self.split), cut(self.scale), cut(self.bias), r1 - r0, self.d,
                            self.d_pad, norm=cut(self.norm), stats=self.stats)


def topk_exact(users, items, k, n_splits=None, item_id_offset=0, out=None, n_users_live=None, excl=None,
               excl_row_map=None, item_hsq=None):
    """Exact 3-pass fused kernel + merge -> PackedTopK [U, k].  item_hsq (item_half_sqnorm(items)): Euclidean
    similarity, with the user norms taken from users.split here."""
    meta = pack_item_meta(items.scale, items.bias, items.n_rows)
    sqnorms = None
    if item_hsq is not None:
        sqnorms = (operand_half_sqnorm(users.split, users.scale, users.d_pad), item_hsq)
    cs, ci = score_topk(users.split, users.scale, users.bias, items.split, meta, users.n_rows, items.n_rows,
                        users.d_pad, k, n_splits=n_splits, item_id_offset=item_id_offset, n_users_live=n_users_live,
                        excl=excl, excl_row_map=excl_row_map, sqnorms=sqnorms)
    return topk_merge(cs, ci, k, out=out, n_users_live=n_users_live)


class FilterItems(object):
    """Item-side inputs of the filter kernel, derived once per call from the K1 outputs (items.stats: max norm / max
    scale already formed in K1's epilogue; operands from a user-defined graph get them from trk_operand_stats)."""

    def __init__(self, items):
        dev = items.split.device
        if items.stats is not None:
            self.stats = items.stats
        else:
            self.stats = torch.zeros((3,), dtype=torch.float32, device=dev)
            operand_stats(items.split, items.scale, items.d_pad, want_norm=False, stats=self.stats)
        self.perm = bias_processing_order(items.bias)
        self.hi = rescale_hi_global(items.split, items.scale, self.stats, items.d_pad, perm=self.perm)
        self.bias_pad, self.block_max, self.block_min = pack_item_bias(items.bias, items.n_rows, self.stats, dev,
                                                                       perm=self.perm, want_min=True)


def _filter_inputs(users, items, fitems, excl):
    """What both filter forms read besides the operands: (user row norms, FilterItems), each formed here when the
    caller has none, and -- with exclusion lists -- their positions in fitems' processing order."""
    user_norm = users.norm if users.norm is not None else operand_stats(users.split, users.scale, users.d_pad)
    if fitems is None:
        fitems = FilterItems(items)
    if excl is not None and excl.pos is None:
        exclusion_positions(excl, fitems.perm, items.n_rows)
    return user_norm, fitems


def fallback_capacity(n_users):
    """Rows the device-side fallback can hold (the exact kernel is launched over this many rows and skips the unused
    ones): 1/8 of the batch, at least 1024, whole 128-row user blocks.  More flagged rows than this = a tie-heavy
    batch; the host layer then re-runs the whole batch through the exact kernel."""
    cap = min(int(n_users), max(1024, int(n_users) // 8))
    return ((cap + 127) // 128) * 128


FALLBACK_SMALL_ROWS = 1024     # the small re-scoring tier: at most this many flagged rows, many item splits


def _ptr_at(t, index):
    return ctypes.c_void_p(t.data_ptr() + index * t.element_size())


def _gather_flagged_rows(users, bad, counters, capacity, small=None):
    """Compacts the indices of the rows of `users` with bad != 0 into idx on the device (at most `capacity`;
    counters[0] = how many were flagged) and gathers those rows' operands.  Returns (idx, SideOperands of `capacity`
    rows whose first min(flagged, capacity) are filled; `small`: the bound of trk_gather_operand_rows' small tier).
    small=None: the count is read back first (one synchronisation) and exactly the flagged rows are gathered -- None
    when there are none."""
    lib = require_cuda()
    dev = users.split.device
    idx = torch.empty((capacity,), dtype=torch.int32, device=dev)
    rc = lib.trk_select_flagged_rows(_p(bad), users.n_rows, _p(idx), capacity, _p(counters), _stream())
    _lib.check(rc, 'trk_select_flagged_rows')
    rows = capacity
    if small is None:
        rows = small = int(counters[0].item())
        if rows == 0:
            return idx, None
    split = torch.empty((rows, 2 * users.d_pad), dtype=torch.float16, device=dev)
    scale = torch.empty((rows,), dtype=torch.float32, device=dev)
    bias = None if users.bias is None else torch.empty((rows,), dtype=torch.float32, device=dev)
    rc = lib.trk_gather_operand_rows(_p(idx), _p(counters), rows, small, _p(users.split), _p(users.scale),
                                     _p(users.bias), int(users.d_pad), _p(split), _p(scale), _p(bias), _stream())
    _lib.check(rc, 'trk_gather_operand_rows')
    return idx, SideOperands(None, split, scale, bias, rows, users.d, users.d_pad)


def rerun_uncertified(users, items, bad, top, k, item_id_offset=0, excl=None):
    """Users flagged by the certificate go through the exact kernel WITHOUT a host round trip: the flagged rows are
    compacted on the device, their operands gathered into a fixed-capacity buffer, the exact kernel runs over that buffer
    with the device-side count and the rows are scattered back into `top`.  Two tiers are launched, exactly one does
    work (decided on the device): up to FALLBACK_SMALL_ROWS rows (the normal case: ~0.01 % of the users) with as many
    item splits as it takes to fill the machine from one or two user blocks, or up to `capacity` rows with few splits.
    Returns (counters, capacity); counters[0] = flagged rows, > capacity means overflow (the caller checks it at its
    next synchronisation).  excl: the exclusion lists of the users; the gathered rows read them through idx."""
    lib = require_cuda()
    cap = fallback_capacity(users.n_rows)
    small = min(cap, FALLBACK_SMALL_ROWS)
    counters = torch.empty((4,), dtype=torch.int32, device=users.split.device)
    idx, sub = _gather_flagged_rows(users, bad, counters, cap, small=small)
    tiers = [(sub.rows(0, small), small, 2, default_splits(2 * TILE_USERS, items.n_rows))]
    if cap > small:
        tiers.append((sub, cap, 3, None))
    for tier_rows, n_rows, slot, n_splits in tiers:
        live = counters[slot:slot + 1]
        exact = topk_exact(tier_rows, items, k, n_splits=n_splits, item_id_offset=item_id_offset, n_users_live=live,
                           excl=excl, excl_row_map=None if excl is None else idx)
        rc = lib.trk_scatter_topk_rows(_p(idx), _ptr_at(counters, slot), n_rows, exact.score_ptr(), exact.item_ptr(),
                                       2 * exact.k, int(k), top.score_ptr(), top.item_ptr(), 2 * top.k, _stream())
        _lib.check(rc, 'trk_scatter_topk_rows')
    return counters, cap


def topk_filter(users, items, k, n_splits=None, item_id_offset=0, fitems=None, excl=None):
    """Filter form: one tensor pass + re-scoring from the split operands; users whose error bound cannot be certified
    (buffer overflow under massive ties, bound violated) are re-run through the exact kernel on the device.
    excl: DeviceExclusion of the users (its positions are formed here for fitems' processing order if missing).
    Returns (PackedTopK, counters device int32[2], capacity)."""
    user_norm, fitems = _filter_inputs(users, items, fitems, excl)
    _, ci, theta = score_filter(users.split, users.scale, users.bias, user_norm, fitems.hi, fitems.stats,
                                fitems.bias_pad, fitems.block_max, fitems.perm, users.n_rows, items.n_rows,
                                users.d_pad, k, n_splits=n_splits, item_id_offset=item_id_offset,
                                block_bias_min=fitems.block_min, excl=excl)
    top, bad = rescore_topk(users, items, ci, theta, user_norm, fitems.stats, k, item_id_offset=item_id_offset)
    counters, cap = rerun_uncertified(users, items, bad, top, k, item_id_offset=item_id_offset, excl=excl)
    return top, counters, cap


# ---------------------------------------------------------------------------------------------------------------
# wide form of the filter (32 < k <= 1024): candidate lists in global memory, re-scoring + selection + certificate in
# one CTA per row, rows the certificate rejects scored dense and ranked
# ---------------------------------------------------------------------------------------------------------------
WIDE_MAX_SLOTS = 16384      # candidates of one row trk_select_wide_topk sorts at once (n_splits x list capacity)
DENSE_RANK_BYTES_PER_PAIR = 35   # device bytes per (row, item) pair that dense scores + rank_full + selection hold


def wide_max_k():
    return int(require_cuda().trk_score_wide_max_k())


def wide_list_capacity(k):
    """Entries of one wide candidate list (per user and item split) for this k."""
    return int(require_cuda().trk_score_wide_list_capacity(int(k)))


def wide_splits(n_users, n_items, k):
    """default_splits, bounded so that a row's lists fit one selection (n_splits x capacity <= WIDE_MAX_SLOTS)."""
    return int(max(1, min(default_splits(n_users, n_items), WIDE_MAX_SLOTS // wide_list_capacity(k))))


def score_wide(users, user_norm, fitems, n_items, k, n_splits, item_id_offset=0, excl=None):
    """Wide filter pass.  Returns (list_item [U, n_splits, capacity], list_count [U, n_splits], theta [U, n_splits])."""
    lib = require_cuda()
    dev = users.split.device
    cap = wide_list_capacity(k)
    list_s = torch.empty((users.n_rows, n_splits, cap), dtype=torch.float32, device=dev)
    list_i = torch.empty((users.n_rows, n_splits, cap), dtype=torch.int32, device=dev)
    count = torch.empty((users.n_rows, n_splits), dtype=torch.int32, device=dev)
    theta = torch.empty((users.n_rows, n_splits), dtype=torch.float32, device=dev)
    if excl is None:
        name, extra = 'trk_score_wide_f16', ()
    else:
        name, extra = 'trk_score_wide_f16_excl', (_p(excl.indptr), _p(excl.pos))
    rc = getattr(lib, name)(_p(users.split), _p(users.scale), _p(users.bias), _p(user_norm), _p(fitems.hi),
                            _p(fitems.stats), _p(fitems.bias_pad), _p(fitems.block_max), _p(fitems.perm), users.n_rows,
                            n_items, int(users.d_pad), int(k), int(n_splits), int(item_id_offset), _p(list_s),
                            _p(list_i), _p(count), _p(theta), *extra, _stream())
    _lib.check(rc, name)
    return list_i, count, theta


def select_wide(users, items, cand_item, n_lists, width, k, count=None, theta=None, user_norm=None, item_stats=None,
                item_id_offset=0, euclidean=False, out=None):
    """Candidate ids per row (cand_item[row, l * width + e], e < count[row, l]) -> PackedTopK [U, k] re-scored from the
    split operands in (score desc, id asc) order, and -- when theta is given -- flags int32 [U] of the rows the
    certificate rejects (else None).  euclidean: scores -1/2 d^2 become -sqrt(max(d^2, 1e-16))."""
    lib = require_cuda()
    dev = users.split.device
    if out is None:
        out = PackedTopK(users.n_rows, k, dev)
    flags = None if theta is None else torch.empty((users.n_rows,), dtype=torch.int32, device=dev)
    rc = lib.trk_select_wide_topk(_p(users.split), _p(users.scale), _p(items.split), _p(items.scale), _p(users.bias),
                                  _p(items.bias), _p(cand_item), cand_item.stride(0), int(n_lists), int(width),
                                  _p(count), _p(theta), _p(user_norm), _p(item_stats), users.n_rows, items.n_rows,
                                  int(users.d_pad), int(k), int(item_id_offset), 1 if euclidean else 0,
                                  out.score_ptr(), out.item_ptr(), 2 * out.k, _p(flags), _stream())
    _lib.check(rc, 'trk_select_wide_topk')
    return out, flags


def exclusion_pairs(excl, rows):
    """(row position, local item id) long tensors of the excluded pairs of the list rows `rows` (long [n])."""
    dev = excl.indptr.device
    starts = excl.indptr[rows].long()
    lens = excl.indptr[rows + 1].long() - starts
    pair_row = torch.repeat_interleave(torch.arange(rows.numel(), device=dev), lens)
    first = torch.repeat_interleave(torch.cumsum(lens, 0) - lens, lens)
    offs = torch.arange(pair_row.numel(), device=dev) - first
    return pair_row, excl.ids[starts[pair_row] + offs].long()


def topk_from_scores(scores, k, item_id_offset=0, ex_rows=None, ex_cols=None):
    """Dense scores [n, n_items] (modified in place) -> PackedTopK [n, k] of the entries of rank <= k (exact full ranks,
    trk_rank_full).  ex_rows / ex_cols: excluded pairs -- they score -inf before the ranking and are never emitted
    (their slots keep the sentinel (-inf, 2**31 - 1))."""
    n_rows, n_items = scores.shape
    top = empty_topk(n_rows, k, scores.device)
    excluded = None
    if ex_rows is not None:
        scores[ex_rows, ex_cols] = float('-inf')
        excluded = torch.zeros((n_rows, n_items), dtype=torch.bool, device=scores.device)
        excluded[ex_rows, ex_cols] = True
    ranks = rank_full(scores).long()
    sel = ranks <= k
    if excluded is not None:
        sel &= ~excluded
    rows, cols = sel.nonzero(as_tuple=True)
    pos = ranks[rows, cols] - 1
    top.scores[rows, pos] = scores[rows, cols]
    top.items[rows, pos] = (cols + item_id_offset).to(torch.int32)
    return top


def dense_rank_rows(n_items, block_bytes):
    """Rows of one dense-score + full-rank block that stay within block_bytes (DENSE_RANK_BYTES_PER_PAIR per pair)."""
    return int(max(1, block_bytes // max(DENSE_RANK_BYTES_PER_PAIR * int(n_items), 1)))


def rerun_flagged_dense(users, items, bad, top, k, item_id_offset=0, excl=None, euclidean=False,
                        block_bytes=4 << 30):
    """Rows of `top` whose certificate failed (bad != 0): compacted on the device, their operands gathered, scored dense
    by the exact 3-pass kernel in blocks of at most block_bytes, ranked (trk_rank_full, exclusion as a mask), and their
    rank <= k items re-scored and ordered by trk_select_wide_topk (the arithmetic of every other row) before they are
    scattered back into `top`.  One host synchronisation per call, i.e. per user block: the count, which sizes the dense
    work.  (The default wide blocks are large: one block at k = 100 for up to 1.68M users, six at k = 1000 for 1M.)
    Returns the device counters (counters[0] = rows)."""
    lib = require_cuda()
    dev = users.split.device
    counters = torch.zeros((4,), dtype=torch.int32, device=dev)
    if users.n_rows == 0:
        return counters
    idx, sub = _gather_flagged_rows(users, bad, counters, users.n_rows)
    if sub is None:
        return counters
    n_bad = sub.n_rows
    meta = pack_item_meta(items.scale, items.bias, items.n_rows)
    cand = torch.empty((n_bad, k), dtype=torch.int32, device=dev)
    step = dense_rank_rows(items.n_rows, block_bytes)
    rows = idx[:n_bad].long()
    for r0 in range(0, n_bad, step):
        r1 = min(n_bad, r0 + step)
        part = sub.rows(r0, r1)
        scores = score_dense_tc(part.split, part.scale, part.bias, items.split, meta, r1 - r0, items.n_rows,
                                users.d_pad)
        ex = (None, None) if excl is None else exclusion_pairs(excl, rows[r0:r1])
        cand[r0:r1] = topk_from_scores(scores, k, item_id_offset, *ex).items
        del scores
    fixed, _ = select_wide(sub, items, cand, 1, k, k, item_id_offset=item_id_offset, euclidean=euclidean)
    rc = lib.trk_scatter_topk_rows(_p(idx), _p(counters), n_bad, fixed.score_ptr(), fixed.item_ptr(), 2 * fixed.k,
                                   int(k), top.score_ptr(), top.item_ptr(), 2 * top.k, _stream())
    _lib.check(rc, 'trk_scatter_topk_rows')
    return counters


def topk_wide(users, items, k, n_splits=None, item_id_offset=0, fitems=None, excl=None, euclidean=False,
              block_bytes=4 << 30):
    """Wide filter form for 32 < k <= wide_max_k(): one tensor pass that keeps every row's candidates in global memory,
    re-scoring + selection + certificate (trk_select_wide_topk), and the rows the certificate rejects scored dense and
    ranked (rerun_flagged_dense).  Returns (PackedTopK, counters device int32[4], capacity); counters[0] = rows that
    took the dense fallback (every flagged row fits: capacity = the number of rows)."""
    user_norm, fitems = _filter_inputs(users, items, fitems, excl)
    if n_splits is None:
        n_splits = wide_splits(users.n_rows, items.n_rows, k)
    cand, count, theta = score_wide(users, user_norm, fitems, items.n_rows, k, n_splits,
                                    item_id_offset=item_id_offset, excl=excl)
    cap = cand.shape[2]
    top, bad = select_wide(users, items, cand.view(users.n_rows, n_splits * cap), n_splits, cap, k, count=count,
                           theta=theta, user_norm=user_norm, item_stats=fitems.stats, item_id_offset=item_id_offset,
                           euclidean=euclidean)
    del cand, count, theta
    counters = rerun_flagged_dense(users, items, bad, top, k, item_id_offset=item_id_offset, excl=excl,
                                   euclidean=euclidean, block_bytes=block_bytes)
    return top, counters, users.n_rows


# ---------------------------------------------------------------------------------------------------------------
# wide mode of the exact kernel (k <= 1024, Euclidean and attention forms): every (user, item split, column half)
# keeps its exact top k in a list in global memory, then one selection per row -- no certificate, no fallback
# ---------------------------------------------------------------------------------------------------------------
def exact_wide_list_capacity(k):
    """Entries of one list of the exact kernel's wide mode (per user, item split and column half) for this k; 0 when k
    is outside [1, 1024]."""
    return int(require_cuda().trk_score_topk_wide_list_capacity(int(k)))


def exact_wide_splits(n_users, n_items, k):
    """default_splits, bounded so that a row's 2 n_splits lists fit one selection (2 n_splits keep <= WIDE_MAX_SLOTS,
    keep = half the capacity)."""
    return int(max(1, min(default_splits(n_users, n_items), WIDE_MAX_SLOTS // exact_wide_list_capacity(k))))


def _exact_wide_lists(n_users, n_splits, k, device):
    cap = exact_wide_list_capacity(k)
    return (torch.empty((n_users, n_splits, 2, cap), dtype=torch.float32, device=device),
            torch.empty((n_users, n_splits, 2, cap), dtype=torch.int32, device=device),
            torch.empty((n_users, n_splits, 2), dtype=torch.int32, device=device))


def select_topk_lists(list_s, list_i, count, k, out=None):
    """Lists [U, n_splits, 2, capacity] with counts [U, n_splits, 2] (the wide mode's output) -> PackedTopK [U, k] in
    (score desc, id asc) order, sentinels where a row has fewer than k entries (trk_select_topk_lists)."""
    lib = require_cuda()
    n_users, n_splits, _, cap = list_s.shape
    if out is None:
        out = PackedTopK(n_users, k, list_s.device)
    rc = lib.trk_select_topk_lists(_p(list_s), _p(list_i), _p(count), n_users, 2 * n_splits, cap, int(k),
                                   out.score_ptr(), out.item_ptr(), 2 * out.k, _stream())
    _lib.check(rc, 'trk_select_topk_lists')
    return out


def topk_exact_wide(users, items, k, n_splits=None, item_id_offset=0, out=None, excl=None, excl_row_map=None,
                    item_hsq=None):
    """Top-k of a Euclidean model for any 1 <= k <= 1024 on the exact kernel's wide mode + trk_select_topk_lists ->
    PackedTopK [U, k].  item_hsq: item_half_sqnorm(items), formed here when not given; the user norms come from
    users.split, as in topk_exact."""
    lib = require_cuda()
    if n_splits is None:
        n_splits = exact_wide_splits(users.n_rows, items.n_rows, k)
    if item_hsq is None:
        item_hsq = item_half_sqnorm(items)
    meta = pack_item_meta(items.scale, items.bias, items.n_rows)
    user_hsq = operand_half_sqnorm(users.split, users.scale, users.d_pad)
    list_s, list_i, count = _exact_wide_lists(users.n_rows, n_splits, k, users.split.device)
    ex = (None, None, None) if excl is None else (_p(excl.indptr), _p(excl.ids), _p(excl_row_map))
    rc = lib.trk_score_topk_wide_euclid_f16x3(_p(users.split), _p(users.scale), _p(users.bias), _p(items.split),
                                              _p(meta), users.n_rows, items.n_rows, int(users.d_pad), int(k),
                                              int(n_splits), int(item_id_offset), _p(list_s), _p(list_i), _p(count),
                                              None, *ex, _p(user_hsq), _p(item_hsq), _stream())
    _lib.check(rc, 'trk_score_topk_wide_euclid_f16x3')
    return select_topk_lists(list_s, list_i, count, k, out=out)


def topk_tastes_wide(users, items, n_tastes, attention, k, n_splits=None, item_id_offset=0, excl=None, out=None,
                     item_hsq=None):
    """topk_tastes for any 1 <= k <= 1024 on the exact kernel's wide mode (attention only: a mixture of tastes without
    attention takes the wide filter, or one Euclidean sweep per taste) -> PackedTopK [U, k].  item_hsq: as for
    score_topk_tastes."""
    lib = require_cuda()
    n_users = users.n_rows
    if n_splits is None:
        n_splits = exact_wide_splits(n_users, items.n_rows, k)
    meta = pack_item_meta(items.scale, items.bias, items.n_rows)
    list_s, list_i, count = _exact_wide_lists(n_users, n_splits, k, users.split.device)
    ex = (None, None, None) if excl is None else (_p(excl.indptr), _p(excl.ids), None)
    name, norms = _tastes_entry('trk_score_topk_wide_tastes', users, item_hsq)
    rc = getattr(lib, name)(_p(users.split), _p(users.scale), _p(users.bias), int(n_tastes), 1 if attention else 0,
                            _p(items.split), _p(meta), n_users, items.n_rows, int(users.d_pad), int(k), int(n_splits),
                            int(item_id_offset), _p(list_s), _p(list_i), _p(count), *ex, *norms, _stream())
    _lib.check(rc, name)
    return select_topk_lists(list_s, list_i, count, k, out=out)


def topk_fused(path, users, items, k, fitems=None, excl=None, item_id_offset=0, item_hsq=None, euclidean=False,
               block_bytes=4 << 30):
    """The fused top-k of one route of topk_route: 'filter' (topk_filter), 'exact3' (topk_exact, with item_hsq),
    'exact3_wide' (topk_exact_wide, Euclidean, with item_hsq) or 'wide' (topk_wide, with euclidean and block_bytes).
    Returns (PackedTopK [U, k], device counters of the rows the certificate rejected | None, capacity of the
    device-side fallback)."""
    if path == 'filter':
        return topk_filter(users, items, k, item_id_offset=item_id_offset, fitems=fitems, excl=excl)
    if path == 'wide':
        return topk_wide(users, items, k, item_id_offset=item_id_offset, fitems=fitems, excl=excl, euclidean=euclidean,
                         block_bytes=block_bytes)
    if path == 'exact3':
        return topk_exact(users, items, k, item_id_offset=item_id_offset, excl=excl, item_hsq=item_hsq), None, 0
    if path == 'exact3_wide':
        return topk_exact_wide(users, items, k, item_id_offset=item_id_offset, excl=excl, item_hsq=item_hsq), None, 0
    raise ValueError('%r is not a fused top-k route' % (path,))


# ---------------------------------------------------------------------------------------------------------------
# exclusion lists: the top-k among the items a user has not interacted with
# ---------------------------------------------------------------------------------------------------------------
def exclusion_host_csr(exclude, item_id_offset, n_items, u0=0, u1=None):
    """Host preparation of an exclusion matrix (pure numpy / scipy, no device).

    exclude: scipy sparse [n_users, >= item_id_offset + n_items], column = GLOBAL item id.  Returns the lists of user
    rows [u0, u1) over the items [item_id_offset, item_id_offset + n_items) as (indptr int32 [rows + 1], ids int32):
    duplicates summed, entries that are zero afterwards dropped (explicit zeros exclude nothing; negative values do
    exclude), ids LOCAL (global - item_id_offset) and ascending within each row."""
    csr = sp.csr_matrix(exclude)
    u1 = csr.shape[0] if u1 is None else int(u1)
    block = csr[int(u0):u1]
    csr = block.copy() if np.shares_memory(block.data, csr.data) else block   # the caller's matrix is never modified
    csr.sum_duplicates()             # sums duplicates and sorts the indices of every row
    csr.eliminate_zeros()
    keep = (csr.indices >= item_id_offset) & (csr.indices < item_id_offset + n_items)
    rows = np.repeat(np.arange(csr.shape[0]), np.diff(csr.indptr))[keep]
    ids = (csr.indices[keep].astype(np.int64) - item_id_offset).astype(np.int32)
    indptr = np.zeros(csr.shape[0] + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows, minlength=csr.shape[0]), out=indptr[1:])
    if indptr[-1] >= 2 ** 31 - 1:
        raise ValueError('exclude holds more entries than int32 indexing covers')
    return indptr.astype(np.int32), np.ascontiguousarray(ids)


class DeviceExclusion(object):
    """Exclusion lists of a block of user rows on the device: int32 indptr [rows + 1], int32 ids (local item ids,
    ascending per row) for the exact kernel and -- once exclusion_positions ran -- int32 pos (processing positions,
    ascending per row) for the filter kernel."""

    def __init__(self, indptr, ids):
        self.indptr, self.ids, self.pos = indptr, ids, None

    @property
    def n_rows(self):
        return int(self.indptr.numel()) - 1

    @classmethod
    def upload(cls, indptr, ids, device):
        require_cuda()
        up = lambda a: torch.from_numpy(a).to(device, non_blocking=True)   # noqa: E731
        # (an empty id array still gets a valid device pointer)
        return cls(up(indptr), up(ids) if ids.size else torch.zeros((1,), dtype=torch.int32, device=device))


def exclusion_positions(excl, perm, n_items):
    """excl.pos = every row's excluded items as filter processing positions (perm: position -> local id, None =
    identity), ascending: one kernel writes (row << 32 | position) keys, one sort of the keys orders every row (the
    rows are contiguous, so indptr is unchanged)."""
    if perm is None:
        excl.pos = excl.ids         # identity order: the ascending ids are the positions
        return excl
    lib = require_cuda()
    dev = excl.indptr.device
    keys = torch.empty((int(excl.ids.numel()),), dtype=torch.int64, device=dev)   # (an empty list: one unused key)
    inv = torch.empty((max(int(n_items), 1),), dtype=torch.int32, device=dev)
    rc = lib.trk_exclusion_positions(_p(perm), int(n_items), _p(inv), _p(excl.indptr), _p(excl.ids), excl.n_rows,
                                     _p(keys), _stream())
    _lib.check(rc, 'trk_exclusion_positions')
    excl.pos = (torch.sort(keys).values & 0xffffffff).to(torch.int32)
    return excl


# ---------------------------------------------------------------------------------------------------------------
# counting mode of the exact kernel: the full ranks of listed (user, item) pairs without the score matrix
# (DESIGN §3.9): one capture sweep for the pairs' scores, a sort of every row's pairs, then counting passes of up to
# COUNT_TARGETS pairs per row
# ---------------------------------------------------------------------------------------------------------------
COUNT_TARGETS = 32          # pairs of a row per counting pass
RANK_AT_BYTES_PER_PAIR = 48  # device bytes per listed pair: ids, scores and counts twice over, sort keys, permutation
RANK_AT_TEMP_BYTES_PER_ELEMENT = 8   # dense+rank with exclusion: bytes per (pair, item) of a chunk's temporaries


def pair_block_max(indptr, n_users, block_rows):
    """The most pairs of a row in each kernel user block of block_rows rows (host, int32 [ceil(n_users / block_rows)])."""
    per_row = np.zeros(-(-int(n_users) // block_rows) * block_rows, dtype=np.int64)
    per_row[:n_users] = np.diff(np.asarray(indptr, dtype=np.int64))
    return per_row.reshape(-1, block_rows).max(axis=1).astype(np.int32)


def count_passes(max_row_pairs):
    """Counting passes of a row with this many pairs."""
    return -(-int(max_row_pairs) // COUNT_TARGETS)


def rank_sort_order(score, pair_row):
    """The permutation that orders the pairs of every row by (score desc, position asc); positions ascend with the item
    id inside a row, so ties go to the lower id as in rank_full.  One stable sort of int64 keys (row << 32 | a key that
    descends with the score); the scores get + 0.0 first so that -0.0 sorts with +0.0."""
    bits = (score + 0.0).view(torch.int32).long()
    ascending = torch.where(bits < 0, 0x7fffffff - (bits & 0x7fffffff), bits + 0x80000000)
    return torch.sort((pair_row.long() << 32) | (0xffffffff - ascending), stable=True).indices


def count_listed_pairs(users, items, meta, indptr, ids, block_rows, excl=None, item_hsq=None, tastes=None,
                       n_splits=None):
    """Counting mode of the exact kernel over the users of `users` (SideOperands; a mixture of tastes: the stacked
    operand and tastes = (n_tastes, attention)).  indptr / ids: host int32 CSR of the listed pairs, ids LOCAL and
    ascending per row; block_rows: the kernel's user block (128, or 2P for a mixture of tastes); excl: DeviceExclusion
    of the same rows or None; item_hsq: item_half_sqnorm(items) for a Euclidean model (a Euclidean mixture of tastes:
    with the operand norms users.hsq).  Returns (int32 counts [nnz] on
    the device in the order of ids -- rank = 1 + count --, passes)."""
    lib = require_cuda()
    dev = users.split.device
    n_users, n_items = users.n_rows, items.n_rows
    nnz = int(indptr[-1])
    block_max = pair_block_max(indptr, n_users, block_rows)
    passes = count_passes(block_max.max()) if block_max.size else 0
    if nnz == 0:
        return torch.zeros((0,), dtype=torch.int32, device=dev), 0
    if n_splits is None:
        n_splits = default_splits(n_users, n_items)
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev, non_blocking=True)   # noqa: E731
    d_indptr, d_ids, d_block_max = up(indptr), up(ids), up(block_max)
    ex = (None, None, None) if excl is None else (_p(excl.indptr), _p(excl.ids), None)
    user_hsq = None
    if item_hsq is not None and tastes is None:
        user_hsq = operand_half_sqnorm(users.split, users.scale, users.d_pad)

    def launch(pair_ids, pair_score, pair_count, pass_):
        head = (_p(users.split), _p(users.scale), _p(users.bias))
        lists = (_p(d_indptr), _p(pair_ids), _p(pair_score), _p(pair_count), _p(d_block_max), int(pass_)) + ex
        shape = (n_users, n_items, int(users.d_pad), int(n_splits), 0)
        if tastes is not None:
            name, norms = _tastes_entry('trk_score_count_tastes', users, item_hsq)
            args = head + (int(tastes[0]), 1 if tastes[1] else 0, _p(items.split), _p(meta)) + shape + lists + norms
        elif item_hsq is not None:
            name = 'trk_score_count_euclid_f16x3'
            args = head + (_p(items.split), _p(meta)) + shape + lists + (_p(user_hsq), _p(item_hsq))
        else:
            name = 'trk_score_count_f16x3'
            args = head + (_p(items.split), _p(meta)) + shape + lists
        _lib.check(getattr(lib, name)(*args, _stream()), name)

    score = torch.empty((nnz,), dtype=torch.float32, device=dev)
    launch(d_ids, score, None, -1)
    pair_row = torch.repeat_interleave(torch.arange(n_users, device=dev), d_indptr[1:].long() - d_indptr[:-1].long())
    order = rank_sort_order(score, pair_row)
    sorted_ids, sorted_score = d_ids[order].contiguous(), score[order].contiguous()
    del score, pair_row
    counts = torch.zeros((nnz,), dtype=torch.int32, device=dev)
    for p in range(passes):
        launch(sorted_ids, sorted_score, counts, p)
    out = torch.empty_like(counts)
    out[order] = counts
    return out, passes


def rank_listed_from_scores(scores, pair_row, pair_col, excl=None, block_bytes=4 << 30):
    """Ranks of listed pairs (long device tensors pair_row / pair_col) from a block's dense scores [rows, n_items]
    (modified in place with excl).  Without excl: trk_rank_full, gathered.  With excl (DeviceExclusion of the rows):
    1 + #{j != i, (row, j) not excluded: s_j > s_i or (s_j == s_i and j < i)}, the pair's own score counted against
    the masked row, in chunks of pairs whose temporaries fit the part of block_bytes the scores leave free (at least
    one pair per chunk).  Returns int32 ranks on the device."""
    if excl is None:
        return rank_full(scores)[pair_row, pair_col]
    n_rows, n_items = scores.shape
    target = scores[pair_row, pair_col]
    ex_rows, ex_cols = exclusion_pairs(excl, torch.arange(n_rows, device=scores.device))
    scores[ex_rows, ex_cols] = float('-inf')
    cols = torch.arange(n_items, device=scores.device)
    out = torch.empty((pair_row.numel(),), dtype=torch.int32, device=scores.device)
    # per gathered element: its float32 score and at most three live bool masks (RANK_AT_TEMP_BYTES_PER_ELEMENT)
    free = max(0, int(block_bytes) - 4 * scores.numel())
    step = max(1, free // (RANK_AT_TEMP_BYTES_PER_ELEMENT * max(n_items, 1)))
    for p0 in range(0, pair_row.numel(), step):
        p1 = min(pair_row.numel(), p0 + step)
        row = scores[pair_row[p0:p1]]
        t = target[p0:p1, None]
        ahead = (row > t).sum(dim=1) + ((row == t) & (cols[None, :] < pair_col[p0:p1, None])).sum(dim=1)
        out[p0:p1] = (1 + ahead).to(torch.int32)
    return out


# ---------------------------------------------------------------------------------------------------------------
# pairs mode of the exact kernel: the scores of listed (user, item) pairs, bit for bit predict()'s, from item tiles
# gathered out of each user block's own listed items (DESIGN §3.13)
# ---------------------------------------------------------------------------------------------------------------
PAIR_TILE = 128             # columns of a gathered tile: item i sits at column i % PAIR_TILE, its dense-sweep column
PAIRS_TILES_PER_WORK = 16   # gathered tiles per work item: a block with many tiles is spread over several CTAs
# device bytes per listed pair at most: its virtual column, score and permutation, and -- when every tile holds a single
# listed item -- a whole tile of slots (item id, {scale, bias}, half squared norm)
PREDICT_AT_BYTES_PER_PAIR = 24 + PAIR_TILE * 16

PairsPlan = collections.namedtuple('PairsPlan', 'tile_items block_tiles work cols order')


def pairs_plan(indptr, ids, n_rows, block_rows, max_tiles=PAIRS_TILES_PER_WORK):
    """Host plan of a pairs-mode launch over n_rows user rows whose listed pairs are the CSR (indptr, ids: LOCAL item
    ids, ascending per row); block_rows = the kernel's user block (128, or 2P for a mixture of tastes).

    Every user block takes its distinct listed items (an item listed by several of its rows takes one slot), groups
    them by residue c = i % 128 and puts the j-th item (ascending) of residue c at column c of the block's tile j, so a
    block gets as many tiles as its largest residue class.  Returns a PairsPlan of numpy arrays:
      tile_items  int32 [T, 128], -1 = an empty slot;
      block_tiles int64 [n_blocks + 1]: block b owns tiles [block_tiles[b], block_tiles[b + 1]);
      work        int32 [W, 3]: (block, first tile, end tile), at most max_tiles tiles each, every tile in one item;
      cols        int32 [nnz]: the pairs' virtual columns tile * 128 + i % 128, ascending within each row;
      order       int64 [nnz]: pair k of the kernel's order (cols) is pair order[k] of the listing (ids)."""
    indptr = np.asarray(indptr, dtype=np.int64)
    ids = np.asarray(ids, dtype=np.int64)
    n_blocks = -(-int(n_rows) // int(block_rows))
    row = np.repeat(np.arange(n_rows, dtype=np.int64), np.diff(indptr))
    res, quo = ids % PAIR_TILE, ids // PAIR_TILE
    span = int(quo.max()) + 1 if ids.size else 1
    # one int64 key per pair whose order is (block, residue, item); its distinct values are the block's slots
    slots, inv = np.unique(((row // block_rows) * PAIR_TILE + res) * span + quo, return_inverse=True)
    group = slots // span                              # block * 128 + residue
    n = slots.size
    first = np.flatnonzero(np.r_[True, group[1:] != group[:-1]]) if n else np.zeros(0, np.int64)
    rank = np.arange(n) - np.repeat(first, np.diff(np.r_[first, n]))   # j: rank of the item in its residue class
    blk = group // PAIR_TILE
    block_tiles = np.zeros(n_blocks + 1, dtype=np.int64)
    if n:
        b_first = np.flatnonzero(np.r_[True, blk[1:] != blk[:-1]])
        block_tiles[blk[b_first] + 1] = np.maximum.reduceat(rank + 1, b_first)
    np.cumsum(block_tiles, out=block_tiles)
    n_tiles = int(block_tiles[-1])
    if n_tiles > 1 << 24:
        raise ValueError('%d gathered tiles exceed the int32 virtual columns of one launch' % n_tiles)
    tile = block_tiles[blk] + rank
    tile_items = np.full((n_tiles, PAIR_TILE), -1, dtype=np.int32)
    tile_items[tile, group % PAIR_TILE] = (slots % span) * PAIR_TILE + group % PAIR_TILE
    col = (tile * PAIR_TILE + group % PAIR_TILE)[inv.reshape(-1)]
    order = np.argsort(row * (n_tiles * PAIR_TILE) + col, kind='stable')
    per_block = np.diff(block_tiles)
    chunks = -(-per_block // max_tiles)
    w_blk = np.repeat(np.arange(n_blocks, dtype=np.int64), chunks)
    w_k = np.arange(w_blk.size) - np.repeat(np.cumsum(chunks) - chunks, chunks)
    t0 = block_tiles[w_blk] + w_k * max_tiles
    work = np.stack([w_blk, t0, np.minimum(t0 + max_tiles, block_tiles[w_blk + 1])], axis=1).astype(np.int32)
    return PairsPlan(tile_items, block_tiles, work, col[order].astype(np.int32), order)


def score_listed_pairs(users, items, meta, indptr, plan, item_hsq=None, tastes=None):
    """Pairs mode of the exact kernel over the users of `users` (SideOperands; a mixture of tastes: the stacked operand
    and tastes = (n_tastes, attention)); meta = pack_item_meta(items ...), item_hsq = item_half_sqnorm(items) for a
    Euclidean model; indptr / plan: the host pair CSR and its pairs_plan.  Returns float32 scores on the device in the
    order of the listing."""
    lib = require_cuda()
    dev = users.split.device
    nnz = int(indptr[-1])
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev, non_blocking=True)   # noqa: E731
    d_indptr, d_cols, d_tiles, d_work = up(indptr), up(plan.cols), up(plan.tile_items), up(plan.work)
    slot = d_tiles.view(-1).long()
    empty = slot < 0
    slot = slot.clamp(min=0)
    slot_meta = meta[slot]
    slot_meta[empty] = torch.tensor([0.0, float('-inf')], device=dev)   # an empty slot scores as a padding column
    slot_hsq = None
    if item_hsq is not None:
        slot_hsq = item_hsq[slot]
        slot_hsq[empty] = 0.0
    score = torch.empty((nnz,), dtype=torch.float32, device=dev)
    n_tiles, n_work = int(plan.tile_items.shape[0]), int(plan.work.shape[0])
    head = (_p(users.split), _p(users.scale), _p(users.bias))
    shape = (users.n_rows, items.n_rows, int(users.d_pad))
    lists = (_p(d_indptr), _p(d_cols), _p(score), _p(d_tiles), n_tiles, _p(d_work), n_work)
    if tastes is not None:
        name, norms = _tastes_entry('trk_score_pairs_tastes', users, slot_hsq)
        args = head + (int(tastes[0]), 1 if tastes[1] else 0, _p(items.split), _p(slot_meta)) + shape + lists + norms
    elif item_hsq is not None:
        name = 'trk_score_pairs_euclid_f16x3'
        user_hsq = operand_half_sqnorm(users.split, users.scale, users.d_pad)
        args = head + (_p(items.split), _p(slot_meta)) + shape + lists + (_p(user_hsq), _p(slot_hsq))
    else:
        name = 'trk_score_pairs_f16x3'
        args = head + (_p(items.split), _p(slot_meta)) + shape + lists
    _lib.check(getattr(lib, name)(*args, _stream()), name)
    out = torch.empty_like(score)
    out[up(plan.order)] = score
    return out
