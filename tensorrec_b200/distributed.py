"""Item-axis sharding of predict_rank(k) over the GPUs of one box (SURVEY.md 8e).

One process per GPU (torchrun); every rank holds the full user side and a contiguous range of item rows.  The path has
exactly one exchange step.  Each rank finds the top-k of ALL users over ITS items (kernels.PackedTopK: int32 [U, 2k],
row u = k scores then k global item ids), then

    all-to-all   rank r receives, from every rank, the rows of user slice r  ->  int32 [world, U_r, 2k]
                 (U * k * 8 * (world - 1) / world bytes leave each rank: 1/world of what an all-gather moves in)
    merge        trk_topk_merge over the `world` lists of each of ITS U_r users, ordered by (score desc, global id asc)
                 so cross-shard ties resolve to the lower id like tf.nn.top_k

so every user's global top-k is formed exactly once, on the rank that owns the user slice.  Callers that want all
users on every rank add one all-gather of the merged slices (all_gather_rows).  torch.distributed is the plumbing:
NCCL over NVLink on GPUs, gloo on CPU for the host-logic tests."""
import numpy as np
import torch
import torch.distributed as dist


def shard_bounds(n, world_size, rank):
    """Contiguous, balanced range [lo, hi) of `rank` out of n rows; the first n % world_size ranks get one extra."""
    base, extra = divmod(int(n), int(world_size))
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def exchange_rows(packed, group=None):
    """The all-to-all of the exchange on a [U, w] tensor: returns (recv [world, U_r, w], (lo, hi)) where [lo, hi) is
    this rank's user slice and recv[l] = rows [lo, hi) of rank l's tensor."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    n_users, width = packed.shape
    bounds = [shard_bounds(n_users, world, r) for r in range(world)]
    lo, hi = bounds[rank]
    recv = torch.empty((world * (hi - lo), width), dtype=packed.dtype, device=packed.device)
    dist.all_to_all_single(recv, packed.contiguous(), output_split_sizes=[hi - lo] * world,
                           input_split_sizes=[b - a for a, b in bounds], group=group)
    return recv.view(world, hi - lo, width), (lo, hi)


def exchange_and_merge(top, group=None):
    """kernels.PackedTopK of all users over this rank's items -> (PackedTopK of this rank's user slice over ALL items,
    (lo, hi) = the slice)."""
    from . import kernels
    recv, (lo, hi) = exchange_rows(top.buf, group)
    return kernels.topk_merge_received(recv, hi - lo, recv.shape[0], top.k), (lo, hi)


def all_gather_rows(merged, n_users, group=None):
    """Merged slices -> kernels.PackedTopK of all n_users users on every rank (one all-gather; slices may differ by
    one row, so the buffers are padded to the largest)."""
    from . import kernels
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    width = merged.buf.shape[1]
    largest = shard_bounds(n_users, world, 0)[1]
    send = merged.buf
    if send.shape[0] < largest:
        send = torch.cat([send, send.new_zeros((largest - send.shape[0], width))])
    out = torch.empty((world * largest, width), dtype=send.dtype, device=send.device)
    dist.all_gather_into_tensor(out, send.contiguous(), group=group)
    if n_users % world != 0:
        out = torch.cat([out[r * largest: r * largest + (b - a)]
                         for r, (a, b) in enumerate(shard_bounds(n_users, world, r) for r in range(world))])
    return kernels.PackedTopK(n_users, merged.k, out.device, buf=out)


def union_of_indices(indices, n, group, device):
    """The union over ranks of a small set of indices in [0, n) (all-reduce of a mask): every rank takes the same
    decision about which user blocks to re-run."""
    mask = torch.zeros((max(n, 1),), dtype=torch.int32, device=device)
    if indices:
        mask[torch.as_tensor(list(indices), device=device)] = 1
    dist.all_reduce(mask, op=dist.ReduceOp.MAX, group=group)
    return [int(i) for i in np.nonzero(mask.cpu().numpy())[0]]


def predict_top_k_sharded(model, user_features, item_features, k, group=None, to_host=True, gather='all',
                          user_batch_size=None, exclude=None):
    """Item-sharded predict_rank(k).  `item_features` is the FULL item matrix (scipy sparse); each rank slices its
    contiguous shard, runs the fused kernel on it and takes part in the exchange.  `exclude` (global item ids, see
    TensorRec.predict_top_k) is the same matrix on every rank; each rank uses the columns of its shard."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    lo, hi = shard_bounds(item_features.shape[0], world, rank)
    local_items = item_features.tocsr()[lo:hi] if hasattr(item_features, 'tocsr') else item_features[lo:hi]
    return model.predict_top_k(user_features, local_items, k, item_id_offset=lo,
                               gather_group=group if group is not None else dist.group.WORLD, to_host=to_host,
                               gather=gather, user_batch_size=user_batch_size, **({} if exclude is None else
                                                                               {'exclude': exclude}))


def common_block_rows(rows, group, device):
    """The smallest of the block sizes (user rows per block) the ranks chose.  Each rank sizes its blocks from its own
    item shard, and shards differ in size; but every block ends in the collective exchange, so every rank must cut the
    users into the same blocks."""
    t = torch.tensor([int(rows)], dtype=torch.int64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
    return int(t.item())
