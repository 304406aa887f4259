"""GPU tests of the exact kernel's wide mode ('exact3_wide', DESIGN §3.8): Euclidean models with one taste or three and
attention models, 32 < k <= 1024.  The wide mode and dense+rank score through the same epilogue, so every case is
bit for bit: against dense+rank forced on the same model, against the oracle on integer fixtures, and -- at the kernel
level -- against a numpy top-k of the dense tensor-core scores.  dense+rank scores Euclidean mixtures of tastes on the
fp32 CUDA-core kernel, so their float fixtures are held bit for bit to the numpy top-k of the maximum over the tastes of
the per-taste tensor-core dense scores instead, and agree with dense+rank to a few ulps."""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from tests.masked_topk import SENTINEL_ID, masked_top_k
from tests.test_euclidean_tc_gpu import exclusion
from tests.test_euclidean_tc_gpu import make_model as euclid_model
from tests.test_tastes_tc_gpu import crafted, float_model, identity_model, oracle_scores

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def T():
    import torch
    import tensorrec_b200
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    torch.cuda.set_device(0)
    return tensorrec_b200


def assert_same(a, b):
    assert np.array_equal(np.asarray(a.items), np.asarray(b.items))
    assert np.array_equal(np.asarray(a.scores), np.asarray(b.scores))


def both_routes(T, monkeypatch, model, uf, itf, k, **kw):
    """predict_top_k on 'exact3_wide' and on 'dense+rank', both forced."""
    monkeypatch.setattr(T.tensorrec, 'EXACT_WIDE_MIN_ITEMS', 0)
    wide = model.predict_top_k(uf, itf, k, **kw)
    assert model.last_topk_info['path'] == 'exact3_wide' and model.last_topk_info['fallback_rows'] == 0
    monkeypatch.setattr(T.tensorrec, 'EXACT_WIDE_MIN_ITEMS', 10 ** 9)
    dense = model.predict_top_k(uf, itf, k, **kw)
    assert model.last_topk_info['path'] == 'dense+rank'
    return wide, dense


U, I = 150, 1200 + 37           # neither a multiple of a block or a tile


def model_of(T, kind, d, integer, seed):
    """-> (model, uf, itf, oracle scores or None)."""
    if kind == 'attention':
        if integer:
            u, a, item, ub, ib = crafted(U, I, d, 3, True, seed=seed)
            model, uf, itf = identity_model(T, u, a, item, ub, ib)
            return model, uf, itf, oracle_scores(u, a, item, ub, ib)
        model, uf, itf, _ = float_model(T, U, I, d, 3, True, seed=seed)
        return model, uf, itf, None
    n_tastes = 3 if kind == 'euclid3' else 1
    model, uf, itf, scores, _, _ = euclid_model(T, U, I, d, integer, n_tastes=n_tastes, seed=seed)
    return model, uf, itf, scores if integer else None


def tastes_reference(T, model, uf, itf, k):
    """numpy top-k by (score desc, id asc) of max_t of the per-taste tensor-core Euclidean dense scores of a model.  The
    biases are added inside each taste's score; rounding is monotone, so the max commutes with them."""
    from tensorrec_b200 import kernels
    device = model._cuda_device()
    user_in, item_in = model._single_input(uf, 'user_features'), model._single_input(itf, 'item_features')
    items = model._side_operands('item', item_in, device)
    meta = kernels.pack_item_meta(items.scale, items.bias, items.n_rows)
    best = None
    for t in range(model.n_tastes):
        users = model._side_operands('user', user_in, device, taste=t)
        sq = (kernels.operand_half_sqnorm(users.split, users.scale, users.d_pad), kernels.item_half_sqnorm(items))
        s = kernels.score_dense_tc(users.split, users.scale, users.bias, items.split, meta, users.n_rows, items.n_rows,
                                   users.d_pad, sqnorms=sq).cpu().numpy()
        best = s if best is None else np.maximum(best, s)
    return oracle.top_k_from_scores(best, k)


@pytest.mark.parametrize('kind', ['euclid', 'euclid3', 'attention'])
@pytest.mark.parametrize('d', [40, 128])
@pytest.mark.parametrize('integer', [True, False])
def test_wide_equals_dense_rank(T, monkeypatch, kind, d, integer):
    model, uf, itf, scores = model_of(T, kind, d, integer, seed=d + len(kind))
    for k in (33, 100, 1000):
        wide, dense = both_routes(T, monkeypatch, model, uf, itf, k)
        if kind == 'euclid3' and not integer:
            # dense+rank scores a Euclidean mixture of tastes on the fp32 CUDA-core kernel, not on the tensor-core
            # epilogue: bit for bit against the top-k of the max of the per-taste tensor-core scores instead
            exp_i, exp_s = tastes_reference(T, model, uf, itf, k)
            assert np.array_equal(wide.items, exp_i) and np.array_equal(wide.scores, exp_s)
            assert np.allclose(wide.scores, dense.scores, rtol=2e-6, atol=2e-6)
        else:
            assert_same(wide, dense)
        if scores is not None:
            exp_i, exp_s = oracle.top_k_from_scores(scores, k)
            assert np.array_equal(wide.items, exp_i) and np.array_equal(wide.scores, exp_s)


@pytest.mark.parametrize('kind', ['euclid', 'euclid3', 'attention'])
def test_exclusion_and_user_blocks(T, monkeypatch, kind):
    model, uf, itf, scores = model_of(T, kind, 40, True, seed=7)
    k = 100
    ref = scores if scores is not None else model.predict(uf, itf)
    exclude = exclusion(ref, k, seed=8)
    wide, dense = both_routes(T, monkeypatch, model, uf, itf, k, exclude=exclude, user_batch_size=64)
    assert_same(wide, dense)
    assert (wide.items[4::6] == SENTINEL_ID).any() and (wide.items[3::6] == SENTINEL_ID).all()
    if scores is not None:
        exp_i, exp_s = masked_top_k(scores, exclude, k)
        assert np.array_equal(wide.items, exp_i) and np.array_equal(wide.scores, exp_s)
    monkeypatch.setattr(T.tensorrec, 'EXACT_WIDE_MIN_ITEMS', 0)
    empty = model.predict_top_k(uf, itf, k, exclude=sp.csr_matrix(ref.shape))
    assert_same(empty, model.predict_top_k(uf, itf, k))


# ---- the kernels --------------------------------------------------------------------------------------------------
def operands(T, n_users, n_items, d, seed, values=None, item_bias=None):
    import torch
    from tensorrec_b200 import kernels
    rng = np.random.default_rng(seed)
    d_pad = kernels.d_pad_for(d)
    if values is None:
        u = rng.integers(-3, 4, (n_users, d)).astype(np.float32)
        i = rng.integers(-3, 4, (n_items, d)).astype(np.float32)
    else:
        u, i = values
    ub = rng.integers(-4, 5, n_users).astype(np.float32)
    ib = rng.integers(-4, 5, n_items).astype(np.float32) if item_bias is None else item_bias

    def side(x, b):
        split, scale = kernels.split_f32(torch.from_numpy(x).cuda(), d_pad=d_pad)
        return kernels.SideOperands(None, split, scale, torch.from_numpy(b).cuda(), x.shape[0], d, d_pad)

    return side(u, ub), side(i, ib)


def dense_top(T, users, items, k, item_id_offset=0, excl_rows=None):
    """numpy top-k by (score desc, id asc) of the dense tensor-core Euclidean scores (the same epilogue)."""
    from tensorrec_b200 import kernels
    meta = kernels.pack_item_meta(items.scale, items.bias, items.n_rows)
    sq = (kernels.operand_half_sqnorm(users.split, users.scale, users.d_pad), kernels.item_half_sqnorm(items))
    scores = kernels.score_dense_tc(users.split, users.scale, users.bias, items.split, meta, users.n_rows,
                                    items.n_rows, users.d_pad, sqnorms=sq).cpu().numpy()
    if excl_rows is not None:
        for r, cols in excl_rows.items():
            scores[r, cols] = -np.inf
    ids = np.arange(items.n_rows) + item_id_offset
    out_i = np.full((users.n_rows, k), SENTINEL_ID, np.int32)
    out_s = np.full((users.n_rows, k), -np.inf, np.float32)
    for r in range(users.n_rows):
        ok = scores[r] > -np.inf
        order = np.lexsort((ids[ok], -scores[r][ok].astype(np.float64)))[:k]
        out_i[r, :len(order)] = ids[ok][order]
        out_s[r, :len(order)] = scores[r][ok][order]
    return out_i, out_s


def check_top(top, exp):
    assert np.array_equal(top.items.cpu().numpy(), exp[0])
    assert np.array_equal(top.scores.cpu().numpy(), exp[1])


@pytest.mark.parametrize('k', [1, 10, 32])
def test_small_k_equals_topk_exact(T, k):
    from tensorrec_b200 import kernels
    users, items = operands(T, 300, 2000 + 5, 64, seed=k)
    hsq = kernels.item_half_sqnorm(items)
    wide = kernels.topk_exact_wide(users, items, k, item_hsq=hsq)
    exact = kernels.topk_exact(users, items, k, item_hsq=hsq)
    assert np.array_equal(wide.buf.cpu().numpy(), exact.buf.cpu().numpy())


@pytest.mark.parametrize('n_splits', [1, 3, 8])
@pytest.mark.parametrize('k', [33, 257, 1024])
def test_splits_and_ragged_catalogues(T, n_splits, k):
    from tensorrec_b200 import kernels
    users, items = operands(T, 260, 3000 + 77, 128, seed=n_splits + k)
    top = kernels.topk_exact_wide(users, items, k, n_splits=n_splits)
    check_top(top, dense_top(T, users, items, k))


def test_tie_heavy_and_rising_scores(T):
    from tensorrec_b200 import kernels
    n_users, n_items, d = 140, 2500 + 3, 64
    zeros_u, zeros_i = np.zeros((n_users, d), np.float32), np.zeros((n_items, d), np.float32)
    # every score equal: the lowest ids win
    users, items = operands(T, n_users, n_items, d, 1, values=(zeros_u, zeros_i), item_bias=np.zeros(n_items, np.float32))
    for k in (33, 500):
        check_top(kernels.topk_exact_wide(users, items, k), dense_top(T, users, items, k))
    # scores rising with the item id: every item is admitted, lists compact as often as they can
    rising = np.arange(n_items, dtype=np.float32)
    users, items = operands(T, n_users, n_items, d, 2, values=(zeros_u, zeros_i), item_bias=rising)
    for k in (33, 1000):
        top = kernels.topk_exact_wide(users, items, k)
        check_top(top, dense_top(T, users, items, k))
        assert np.all(top.items.cpu().numpy() == np.arange(n_items - 1, n_items - 1 - k, -1))
    # few distinct integer scores
    users, items = operands(T, n_users, n_items, d, 3, values=(np.ones((n_users, d), np.float32),
                                                               np.random.default_rng(4).integers(0, 2, (n_items, d))
                                                               .astype(np.float32)))
    check_top(kernels.topk_exact_wide(users, items, 300), dense_top(T, users, items, 300))


def test_exclusion_lists_at_the_kernel(T):
    from tensorrec_b200 import kernels
    n_users, n_items, k = 130, 1500 + 11, 200
    users, items = operands(T, n_users, n_items, 40, seed=9)
    rng = np.random.default_rng(10)
    rows = {r: np.sort(rng.choice(n_items, [0, 50, n_items - k // 2, n_items][r % 4], replace=False))
            for r in range(n_users)}
    indptr = np.concatenate([[0], np.cumsum([len(rows[r]) for r in range(n_users)])]).astype(np.int32)
    ids = np.concatenate([rows[r] for r in range(n_users)]).astype(np.int32)
    excl = kernels.DeviceExclusion.upload(indptr, ids, 'cuda')
    top = kernels.topk_exact_wide(users, items, k, n_splits=2, excl=excl)
    check_top(top, dense_top(T, users, items, k, excl_rows=rows))
    got = top.items.cpu().numpy()
    assert (got[2::4] == SENTINEL_ID).any() and (got[3::4] == SENTINEL_ID).all()


def test_item_shards_merge_to_the_whole(T):
    import torch
    from tensorrec_b200 import kernels
    n_users, n_items, k, world = 150, 3000 + 41, 150, 3
    users, items = operands(T, n_users, n_items, 64, seed=11)
    whole = dense_top(T, users, items, k)
    cuts = np.linspace(0, n_items, world + 1).astype(int)
    per_shard = []
    for r in range(world):
        part = items.rows(int(cuts[r]), int(cuts[r + 1]))
        top = kernels.topk_exact_wide(users, part, k, item_id_offset=int(cuts[r]))
        per_shard.append(top.buf)
    merged = kernels.topk_merge_received(torch.stack(per_shard).contiguous(), n_users, world, k)
    assert np.array_equal(merged.items.cpu().numpy(), whole[0])
    assert np.array_equal(merged.scores.cpu().numpy(), whole[1])


def test_attention_kernel_matches_its_dense_scores(T):
    import torch
    from tensorrec_b200 import kernels
    from tests.test_tastes_tc_gpu import stacked_operand
    n_users, n_items, d, k = 77, 2000 + 9, 40, 400
    u, a, item, ub, ib = crafted(n_users, n_items, d, 3, True, seed=12)
    d_pad = kernels.d_pad_for(d)
    split, scale = stacked_operand(u, a, d_pad)
    its, isc = kernels.split_f32(torch.from_numpy(item).cuda(), d_pad=d_pad)
    users = kernels.SideOperands(None, split, scale, torch.from_numpy(ub).cuda(), n_users, d, d_pad)
    items = kernels.SideOperands(None, its, isc, torch.from_numpy(ib).cuda(), n_items, d, d_pad)
    exp = oracle.top_k_from_scores(oracle_scores(u, a, item, ub, ib), k)
    for n_splits in (1, 4):
        top = kernels.topk_tastes_wide(users, items, 3, True, k, n_splits=n_splits)
        check_top(top, exp)
    with pytest.raises(kernels._lib.TrkUnsupportedError):
        kernels.topk_tastes_wide(users, items, 3, False, k)


def test_attention_blocks_reserve_no_taste_fold(T, monkeypatch):
    """An attention model collapses its tastes in one sweep, so its blocks size for the lists alone."""
    model, uf, itf, _ = model_of(T, 'attention', 40, True, seed=13)
    seen = []
    real = type(model)._topk_block_rows
    monkeypatch.setattr(type(model), '_topk_block_rows',
                        lambda self, *a, **kw: seen.append(kw.get('n_tastes')) or real(self, *a, **kw))
    monkeypatch.setattr(T.tensorrec, 'EXACT_WIDE_MIN_ITEMS', 0)
    model.predict_top_k(uf, itf, 100)
    assert model.last_topk_info['path'] == 'exact3_wide' and seen == [1]
