"""GPU parity tests of every C-ABI kernel against the oracle (needs an H100: pytest -m gpu).

Bars (BASELINE.json north_star): integer / index results bit-exact; fp32 scores within 1e-5 relative to |u|.|i|."""
import json
import os

import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from tests import helpers as H

pytestmark = pytest.mark.gpu

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), 'golden', 'reference_known_answers.json')))
F32 = np.float32


@pytest.fixture(scope='module')
def K():
    import torch
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    torch.cuda.set_device(0)
    return kernels


def dev(a, dtype=None):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    return t.cuda()


def split_to_f32(split, scale, d):
    s = split.float().cpu().numpy().astype(np.float64)
    d_pad = s.shape[1] // 2
    return ((s[:, :d] + s[:, d_pad:d_pad + d]) * scale.cpu().numpy().astype(np.float64)[:, None])


# ------------------------------------------------------------------------------------------------- K1
@pytest.mark.parametrize('rows,n_features,d,kind', [
    (100, 200, 100, 'tag'), (150, 200, 128, 'tag'), (1000, 200, 64, 'tag'), (257, 200, 10, 'tag'),
    (64, 200, 1, 'tag'), (3000, None, 128, 'indicator'), (513, None, 32, 'indicator'), (300, 50, 256, 'tag'),
    (37, 23, 12, 'messy'), (90, 40, 7, 'messy'), (70, 31, 128, 'messy'),
])
@pytest.mark.parametrize('n_norm', [0, 1])
def test_gather_reduce_matches_oracle(K, rows, n_features, d, kind, n_norm):
    if kind == 'tag':
        m = H.tag_features(rows, n_features, min(20, n_features // 2), seed=rows)
    elif kind == 'indicator':
        m = H.indicator_features(rows, seed=rows)
        n_features = m.shape[1]
    else:
        m = H.messy_coo(rows, n_features, 6 * rows, seed=rows)
    w = H.linear_weights(n_features, d, seed=d)
    coo = oracle.coo_from_sparse(m)
    expect = oracle.sparse_dense_matmul(coo, w)
    for _ in range(n_norm):
        expect = oracle.l2_normalize(expect)
    csr = K.DeviceCSR.from_scipy(m)
    d_pad = K.d_pad_for(d)
    out, split, scale = K.gather_reduce(csr, dev(w), n_normalize=n_norm, want_f32=True, split_d_pad=d_pad)
    got = out.cpu().numpy()
    # fp32 accumulation in the same order; FMA contraction and the reduction tree of the norm differ by ulps
    scale_ref = np.maximum(np.abs(expect).max(axis=1, keepdims=True), 1e-30)
    assert np.all(np.abs(got - expect) <= 4e-6 * scale_ref + 1e-30)
    # split operand reproduces the fp32 row to ~2^-21 of the row maximum; the scale is an exact power of two
    rec = split_to_f32(split, scale, d)
    assert np.all(np.abs(rec - got) <= 2.0 ** -20 * np.abs(got).max(axis=1, keepdims=True) + 1e-37)
    sc = scale.cpu().numpy()
    assert np.all(np.log2(sc) == np.round(np.log2(sc)))
    pad = split.float().cpu().numpy()
    assert np.all(pad[:, d:d_pad] == 0) and np.all(pad[:, d_pad + d:] == 0)


def test_gather_reduce_integer_exact_and_deterministic(K):
    m = H.tag_features(500, 200, 20, seed=1, integer=True)
    w = H.linear_weights(200, 64, seed=2, integer=True)
    expect = oracle.sparse_dense_matmul(oracle.coo_from_sparse(m), w)
    csr = K.DeviceCSR.from_scipy(m)
    a, sa, sca = K.gather_reduce(csr, dev(w), split_d_pad=64)
    b, sb, scb = K.gather_reduce(csr, dev(w), split_d_pad=64)
    assert np.array_equal(a.cpu().numpy(), expect)
    assert np.array_equal(a.cpu().numpy(), b.cpu().numpy())                     # test/test_tensorrec.py:418-458
    assert np.array_equal(sa.cpu().numpy().view(np.uint16), sb.cpu().numpy().view(np.uint16))
    assert np.array_equal(split_to_f32(sa, sca, 64), expect.astype(np.float64))  # integers survive the split exactly


def test_gather_reduce_input_formats_keep_reference_order(K):
    # csc / lil / coo inputs must accumulate in the order sp.coo_matrix(...) gives the reference
    m = H.messy_coo(50, 30, 400, seed=3)
    w = H.linear_weights(30, 16, seed=4)
    for conv in (lambda x: x, sp.csc_matrix, sp.csr_matrix, sp.lil_matrix):
        mm = conv(m)
        expect = oracle.sparse_dense_matmul(oracle.coo_from_sparse(mm), w)
        out, _, _ = K.gather_reduce(K.DeviceCSR.from_scipy(mm), dev(w))
        assert np.all(np.abs(out.cpu().numpy() - expect) <= 4e-6 * np.abs(expect).max() + 1e-30)


def test_project_biases_golden_and_random(K):
    g = GOLDEN['project_biases']
    feats = sp.coo_matrix(np.array(g['features'], dtype=F32))
    out = K.project_biases(K.DeviceCSR.from_scipy(feats), dev(np.array(g['feature_biases'], dtype=F32)))
    assert np.array_equal(out.cpu().numpy(), np.array(g['expected'], dtype=F32))      # exact, as the reference test
    m = H.tag_features(1234, 200, 20, seed=9)
    b = H.feature_biases(200, seed=1)
    expect = oracle.project_biases(oracle.coo_from_sparse(m), b)
    got = K.project_biases(K.DeviceCSR.from_scipy(m), dev(b)).cpu().numpy()
    assert np.all(np.abs(got - expect) <= 1e-6)


def test_empty_rows_and_empty_matrix(K):
    m = sp.csr_matrix((5, 8), dtype=F32)
    w = H.linear_weights(8, 4)
    out, split, scale = K.gather_reduce(K.DeviceCSR.from_scipy(m), dev(w), n_normalize=1, split_d_pad=64)
    assert np.all(out.cpu().numpy() == 0) and np.all(split.float().cpu().numpy() == 0)
    assert np.all(scale.cpu().numpy() == 1.0)
    assert np.all(K.project_biases(K.DeviceCSR.from_scipy(m), dev(H.feature_biases(8))).cpu().numpy() == 0)


# ------------------------------------------------------------------------------------------------- K2 exact
def test_score_exact_golden(K):
    g = GOLDEN['dot_product_dense']
    got = K.score_exact(dev(np.array(g['user_repr'], dtype=F32)), dev(np.array(g['item_repr'], dtype=F32)))
    assert np.allclose(got.cpu().numpy(), np.array(g['expected']))
    g = GOLDEN['cosine_dense']
    u = K.l2_normalize_rows_(dev(np.array(g['user_repr'], dtype=F32)))
    i = K.l2_normalize_rows_(dev(np.array(g['item_repr'], dtype=F32)))
    assert np.allclose(K.score_exact(u, i).cpu().numpy(), np.array(g['expected']), atol=1e-6)
    g = GOLDEN['euclidean_dense']
    got = K.score_exact(dev(np.array(g['user_repr'], dtype=F32)), dev(np.array(g['item_repr'], dtype=F32)), mode=1)
    assert np.allclose(got.cpu().numpy(), -np.sqrt(np.array(g['expected_neg_sqrt_of'])), atol=1e-6)
    g = GOLDEN['bias_prediction_dense']
    # bias epilogue alone: a 1-component identity "matmul" reproduces the prediction matrix
    pred = np.array(g['predictions'], dtype=F32)
    u = np.eye(3, dtype=F32)
    got = K.score_exact(dev(u), dev(np.ascontiguousarray(pred.T)), dev(np.array(g['user_biases'], dtype=F32)),
                        dev(np.array(g['item_biases'], dtype=F32)))
    assert np.array_equal(got.cpu().numpy(), np.array(g['expected'], dtype=F32))


@pytest.mark.parametrize('U,I,d,T', [(100, 150, 100, 1), (65, 130, 17, 3), (300, 257, 128, 2), (1, 1, 1, 1)])
def test_score_exact_random(K, U, I, d, T):
    rng = np.random.default_rng(U + I)
    u = rng.standard_normal((T, U, d)).astype(F32)
    i = rng.standard_normal((I, d)).astype(F32)
    ub = rng.standard_normal(U).astype(F32)
    ib = rng.standard_normal(I).astype(F32)
    expect = oracle.bias_prediction_dense(
        oracle.collapse_mixture_of_tastes([oracle.dot_product_dense(u[t], i) for t in range(T)]), ub, ib)
    got = K.score_exact(dev(u), dev(i), dev(ub), dev(ib)).cpu().numpy()
    tol = H.norm_tolerance(u, i).max(axis=0) + 1e-6 * (np.abs(ub)[:, None] + np.abs(ib)[None, :])
    assert np.all(np.abs(got - expect) <= tol)
    eu = oracle.collapse_mixture_of_tastes([oracle.euclidean_dense(u[t], i) for t in range(T)])
    got = K.score_exact(dev(u), dev(i), mode=1).cpu().numpy()
    assert np.allclose(got, eu, rtol=1e-4, atol=1e-4)


def test_score_attention_golden_and_random(K):
    g = GOLDEN['collapse_mixture_of_tastes_with_attention']
    # 1 user, 4 items, d = 3 one-hot "tastes": pred[t, 0, i] = predictions[t][i] via identity representations
    preds = np.array(g['predictions'], dtype=F32)
    atts = np.array(g['attentions'], dtype=F32)
    T, I = preds.shape
    # item repr = columns; user repr for taste t picks row t of preds: use d = T*? -> build d = I with item one-hots
    item = np.eye(I, dtype=F32)
    u = preds[:, None, :]          # [T, 1, I]: dot with one-hot item i gives preds[t][i]
    a = atts[:, None, :]
    got = K.score_exact(dev(u), dev(item), attention_repr=dev(a)).cpu().numpy()[0]
    expect = np.array(g['expected'], dtype=F32)
    assert np.all(np.abs(got - expect) <= 4 * np.spacing(expect))
    rng = np.random.default_rng(0)
    u = rng.standard_normal((3, 40, 16)).astype(F32)
    a = rng.standard_normal((3, 40, 16)).astype(F32)
    it = rng.standard_normal((70, 16)).astype(F32)
    expect = oracle.collapse_mixture_of_tastes([oracle.dot_product_dense(u[t], it) for t in range(3)],
                                               [oracle.dot_product_dense(a[t], it) for t in range(3)])
    got = K.score_exact(dev(u), dev(it), attention_repr=dev(a)).cpu().numpy()
    assert np.allclose(got, expect, rtol=2e-5, atol=2e-5)


def test_taste_max_golden(K):
    g = GOLDEN['collapse_mixture_of_tastes']
    preds = np.array(g['predictions'], dtype=F32)
    got = K.score_exact(dev(preds[:, None, :]), dev(np.eye(4, dtype=F32))).cpu().numpy()[0]
    assert np.array_equal(got, np.array(g['expected'], dtype=F32))


# ------------------------------------------------------------------------------------------------- K3 full
def test_rank_full_golden(K):
    g = GOLDEN['rank_predictions']
    got = K.rank_full(dev(np.array(g['predictions'], dtype=F32))).cpu().numpy()
    assert got.dtype == np.int32 and np.array_equal(got, np.array(g['expected']))


@pytest.mark.parametrize('U,I', [(3, 1), (7, 2), (100, 150), (40, 256), (40, 257), (33, 1000), (17, 2048), (5, 4096), (9, 4097),
                                 (6, 9000), (4, 12293), (3, 20000), (2, 70001)])
def test_rank_full_matches_double_sort_with_ties(K, U, I):
    rng = np.random.default_rng(I)
    s = rng.integers(-4, 5, size=(U, I)).astype(F32)           # heavy ties
    s[0, ::3] = -0.0                                            # -0.0 ties with +0.0
    assert np.array_equal(K.rank_full(dev(s)).cpu().numpy(), oracle.rank_predictions(s))
    f = rng.standard_normal((U, I)).astype(F32)
    f[:, : I // 2] = f[:, I - I // 2:][:, : I // 2]             # exact float duplicates
    r = K.rank_full(dev(f)).cpu().numpy()
    assert np.array_equal(r, oracle.rank_predictions(f))
    assert r.min() == 1 and r.max() == I                        # test/test_tensorrec.py:204-212: ranks > 0


# ------------------------------------------------------------------------------------------------- K2+K3 fused
def make_case(U, I, d, integer, seed, biased=True, regime='tag'):
    if regime == 'tag':
        uf = H.tag_features(U, 200, 20, seed=seed, integer=integer)
        itf = H.tag_features(I, 200, 20, seed=seed + 1, integer=integer)
    else:
        uf = H.indicator_features(U, seed=seed)
        itf = H.indicator_features(I, seed=seed + 1)
    wu = H.linear_weights(uf.shape[1], d, seed=seed + 2, integer=integer)
    wi = H.linear_weights(itf.shape[1], d, seed=seed + 3, integer=integer)
    bu = H.feature_biases(uf.shape[1], seed=seed + 4, integer=integer) if biased else None
    bi = H.feature_biases(itf.shape[1], seed=seed + 5, integer=integer) if biased else None
    return uf, itf, wu, wi, bu, bi


def run_fused(K, uf, itf, wu, wi, bu, bi, k, n_splits=None, n_norm=0, offset=0):
    d = wu.shape[1]
    d_pad = K.d_pad_for(d)
    ucsr, icsr = K.DeviceCSR.from_scipy(uf), K.DeviceCSR.from_scipy(itf)
    _, us, usc = K.gather_reduce(ucsr, dev(wu), n_normalize=n_norm, want_f32=False, split_d_pad=d_pad)
    _, its, isc = K.gather_reduce(icsr, dev(wi), n_normalize=n_norm, want_f32=False, split_d_pad=d_pad)
    ub = K.project_biases(ucsr, dev(bu)) if bu is not None else None
    ib = K.project_biases(icsr, dev(bi)) if bi is not None else None
    meta = K.pack_item_meta(isc, ib, itf.shape[0])
    cs, ci = K.score_topk(us, usc, ub, its, meta, uf.shape[0], itf.shape[0], d_pad, k, n_splits=n_splits,
                          item_id_offset=offset)
    top = K.topk_merge(cs, ci, k)
    return top.scores.cpu().numpy(), top.items.cpu().numpy(), (us, usc, ub, its, meta, d_pad)


def oracle_scores(uf, itf, wu, wi, bu, bi, prediction='dot'):
    model = oracle.OracleModel([wu], wi, bu, bi, prediction=prediction)
    return model.predict(uf, itf)


@pytest.mark.parametrize('U,I,d,k,splits', [
    (100, 150, 100, 10, None), (256, 4096, 64, 10, 1), (256, 4096, 64, 10, 5), (130, 1000, 128, 32, 3),
    (1, 300, 64, 1, 2), (300, 257, 128, 7, None), (129, 513, 10, 10, 4),
])
def test_fused_topk_integer_fixture_exact(K, U, I, d, k, splits):
    """Integer-valued features/weights: every product and partial sum is exact in fp32 and in the split-fp16 MMA,
    so ids AND scores must equal the reference order bit for bit, with many ties (lower id first)."""
    uf, itf, wu, wi, bu, bi = make_case(U, I, d, True, seed=U + I)
    scores = oracle_scores(uf, itf, wu, wi, bu, bi)
    exp_i, exp_s = oracle.top_k_from_scores(scores, k)
    got_s, got_i, _ = run_fused(K, uf, itf, wu, wi, bu, bi, k, n_splits=splits)
    assert np.array_equal(got_i, exp_i)
    assert np.array_equal(got_s, exp_s)


@pytest.mark.parametrize('U,I,d,k,regime,cosine', [
    (100, 150, 100, 10, 'tag', False), (500, 3000, 128, 10, 'indicator', False), (200, 2000, 64, 20, 'tag', True),
])
def test_fused_topk_float_within_tolerance(K, U, I, d, k, regime, cosine):
    uf, itf, wu, wi, bu, bi = make_case(U, I, d, False, seed=U, regime=regime)
    model = oracle.OracleModel([wu], wi, bu, bi, prediction='cosine' if cosine else 'dot')
    scores = model.predict(uf, itf)
    ur, ir = model.user_representation(uf)[0], model.item_representation(itf)
    if cosine:
        ur, ir = oracle.l2_normalize(ur), oracle.l2_normalize(ir)
    tol = H.norm_tolerance(ur, ir, rel=1e-5) + 1e-6
    got_s, got_i, _ = run_fused(K, uf, itf, wu, wi, bu, bi, k, n_norm=1 if cosine else 0)
    rows = np.arange(U)[:, None]
    # 1) scores of the returned items agree with the oracle within 1e-5 * |u||i|
    assert np.all(np.abs(got_s - scores[rows, got_i]) <= tol[rows, got_i])
    # 2) the returned set is a valid top-k: nothing outside it beats the k-th returned score by more than tol
    kth = got_s[:, -1:]
    mask = np.ones_like(scores, dtype=bool)
    mask[rows, got_i] = False
    assert np.all((scores - tol)[mask.reshape(scores.shape)].reshape(U, -1) <= kth + 1e-6)
    # 3) ordered by score descending
    assert np.all(np.diff(got_s, axis=1) <= 0)


def test_fused_topk_offset_and_sharded_merge(K):
    """Item-axis shards (the multi-GPU layout) run one after the other on one GPU: merged result == unsharded."""
    import torch
    U, I, d, k = 200, 3000, 64, 10
    uf, itf, wu, wi, bu, bi = make_case(U, I, d, True, seed=7)
    exp_i, exp_s = oracle.top_k_from_scores(oracle_scores(uf, itf, wu, wi, bu, bi), k)
    shards = [(0, 1100), (1100, 1900), (1900, 3000)]
    cs, ci = [], []
    for lo, hi in shards:
        s, i, _ = run_fused(K, uf, itf[lo:hi], wu, wi, bu, bi, k, offset=lo)
        cs.append(torch.from_numpy(s).cuda())
        ci.append(torch.from_numpy(i).cuda())
    top = K.topk_merge(torch.stack(cs, 1), torch.stack(ci, 1), k)
    assert np.array_equal(top.items.cpu().numpy(), exp_i) and np.array_equal(top.scores.cpu().numpy(), exp_s)


def test_fused_topk_k_larger_than_items_pads_with_sentinels(K):
    uf, itf, wu, wi, bu, bi = make_case(40, 6, 64, True, seed=11)
    got_s, got_i, _ = run_fused(K, uf, itf, wu, wi, bu, bi, k=10)
    exp_i, exp_s = oracle.top_k_from_scores(oracle_scores(uf, itf, wu, wi, bu, bi), 6)
    assert np.array_equal(got_i[:, :6], exp_i) and np.array_equal(got_s[:, :6], exp_s)
    assert np.all(got_i[:, 6:] == 2 ** 31 - 1) and np.all(np.isneginf(got_s[:, 6:]))


def test_dense_tc_matches_exact(K):
    for (U, I, d, integer) in [(100, 150, 100, True), (300, 1000, 64, False), (129, 257, 128, False)]:
        uf, itf, wu, wi, bu, bi = make_case(U, I, d, integer, seed=U)
        scores = oracle_scores(uf, itf, wu, wi, bu, bi)
        _, _, (us, usc, ub, its, meta, d_pad) = run_fused(K, uf, itf, wu, wi, bu, bi, k=1)
        got = K.score_dense_tc(us, usc, ub, its, meta, U, I, d_pad).cpu().numpy()
        if integer:
            assert np.array_equal(got, scores)
        else:
            model = oracle.OracleModel([wu], wi, bu, bi)
            tol = H.norm_tolerance(model.user_representation(uf)[0], model.item_representation(itf)) + 1e-6
            assert np.all(np.abs(got - scores) <= tol)


def test_topk_merge_orders_ties_by_lower_id(K):
    import torch
    s = torch.tensor([[[5., 3., 1.], [5., 4., 1.], [9., 1., -float('inf')]]], device='cuda')
    i = torch.tensor([[[7, 1, 30], [2, 9, 11], [40, 10, 2 ** 31 - 1]]], dtype=torch.int32, device='cuda')
    top = K.topk_merge(s, i, 6)
    assert top.items.cpu().tolist() == [[40, 2, 7, 9, 1, 10]]
    assert top.scores.cpu().tolist() == [[9., 5., 5., 4., 3., 1.]]


def test_topk_merge_of_the_exchange_receive_layout(K):
    """[n_lists, U_slice, 2k] (what the all-to-all delivers) merges to the same result as the [U, L, k] layout."""
    import torch
    rng = np.random.default_rng(5)
    U, L, k = 77, 5, 10
    scores = np.sort(rng.integers(-4, 5, size=(U, L, k)).astype(F32), axis=2)[:, :, ::-1].copy()
    ids = np.stack([np.stack([np.sort(rng.choice(1000, k, replace=False)) + 1000 * l for l in range(L)])
                    for _ in range(U)]).astype(np.int32)
    # equal scores inside a list must be ordered by id: sort ids within runs of equal score
    for u in range(U):
        for l in range(L):
            order = np.lexsort((ids[u, l], -scores[u, l]))
            scores[u, l], ids[u, l] = scores[u, l][order], ids[u, l][order]
    ref = K.topk_merge(dev(scores), dev(ids), k)
    recv = np.empty((L, U, 2 * k), dtype=np.int32)
    recv[:, :, :k] = scores.view(np.int32).transpose(1, 0, 2)
    recv[:, :, k:] = ids.transpose(1, 0, 2)
    got = K.topk_merge_received(dev(recv), U, L, k)
    assert torch.equal(got.buf, ref.buf)


def test_unsupported_shapes_raise(K):
    from tensorrec_b200._lib import TrkUnsupportedError
    uf, itf, wu, wi, bu, bi = make_case(10, 20, 64, True, seed=1)
    with pytest.raises(TrkUnsupportedError):
        run_fused(K, uf, itf, wu, wi, bu, bi, k=K.topk_max_k(64) + 1)


# ------------------------------------------------------------------------------------------------- filter + rescore
def side_operands(K, feats, w, b, d, n_norm=0):
    """Operands as the host layer builds them for the filter path: norms and statistics come out of K1."""
    import torch
    csr = K.DeviceCSR.from_scipy(feats)
    d_pad = K.d_pad_for(d)
    stats = torch.empty(3, device='cuda')
    f32, split, scale, norm = K.gather_reduce(csr, dev(w), n_normalize=n_norm, want_f32=True, split_d_pad=d_pad,
                                              want_norm=True, stats=stats)
    bias = K.project_biases(csr, dev(b)) if b is not None else None
    return K.SideOperands(f32, split, scale, bias, feats.shape[0], d, d_pad, norm=norm, stats=stats)


def run_filter(K, uf, itf, wu, wi, bu, bi, k, n_splits=None, n_norm=0, offset=0):
    users = side_operands(K, uf, wu, bu, wu.shape[1], n_norm)
    items = side_operands(K, itf, wi, bi, wi.shape[1], n_norm)
    top, counters, cap = K.topk_filter(users, items, k, n_splits=n_splits, item_id_offset=offset)
    n_bad = int(counters[0])
    assert n_bad <= cap, 'device-side fallback overflowed in a test-sized batch'
    return top.scores.cpu().numpy(), top.items.cpu().numpy(), {'fallback_rows': n_bad}


def test_operand_stats_and_global_rescale(K):
    import torch
    uf, itf, wu, wi, bu, bi = make_case(300, 1000, 100, False, seed=3)
    items = side_operands(K, itf, wi, bi, 100)
    stats = torch.zeros(3, device='cuda')
    norm = K.operand_stats(items.split, items.scale, items.d_pad, stats=stats).cpu().numpy()
    true = np.linalg.norm(items.repr_f32.cpu().numpy().astype(np.float64), axis=1)
    assert np.all(norm >= true) and np.all(norm <= true * 1.01 + 1e-30)           # upper bounds, tight
    st = stats.cpu().numpy()
    assert st[0] == norm.max() and st[1] == items.scale.cpu().numpy().max()
    # the same quantities straight out of K1's epilogue (what the host layer uses): upper bounds, equally tight
    k1_norm, k1_st = items.norm.cpu().numpy(), items.stats.cpu().numpy()
    assert np.all(k1_norm >= true) and np.all(k1_norm <= true * 1.01 + 1e-30)
    assert k1_st[0] == k1_norm.max() and k1_st[1] == st[1]
    hi = K.rescale_hi_global(items.split, items.scale, stats, items.d_pad).float().cpu().numpy()
    x = items.repr_f32.cpu().numpy()
    rec = hi[:, :100] * st[1]
    assert np.all(np.abs(rec - x) <= 2.0 ** -11 * np.abs(x) + 2.0 ** -24 * np.abs(x).max())
    padded, bmax = K.pack_item_bias(items.bias, 1000, stats, 'cuda')
    padded, bmax = padded.cpu().numpy(), bmax.cpu().numpy()
    bias = items.bias.cpu().numpy()
    assert padded.shape == (1024,) and np.all(np.isneginf(padded[1000:]))
    assert np.array_equal(padded[:1000], bias)
    assert np.array_equal(bmax, padded.reshape(-1, 128).max(axis=1))
    assert stats.cpu().numpy()[2] == np.abs(bias).max()
    # processing order: items sorted by bias (stable), operands and biases permuted alike
    perm = K.bias_processing_order(items.bias)
    pn = perm.cpu().numpy()
    assert np.array_equal(pn, np.argsort(-bias, kind='stable'))
    hi_p = K.rescale_hi_global(items.split, items.scale, stats, items.d_pad, perm=perm).float().cpu().numpy()
    assert np.array_equal(hi_p, hi[pn])
    padded_p, bmax_p = K.pack_item_bias(items.bias, 1000, stats, 'cuda', perm=perm)
    assert np.array_equal(padded_p.cpu().numpy()[:1000], bias[pn])
    assert np.array_equal(bmax_p.cpu().numpy(), padded_p.cpu().numpy().reshape(-1, 128).max(axis=1))


@pytest.mark.parametrize('n', [1, 7, 4096, 5000, 300001])
def test_bias_processing_order_from_own_kernels(K, monkeypatch, n):
    """trk_rank_full on the 1 x n bias row + trk_order_from_ranks == the stable descending argsort (ties by lower item
    index, -0.0 == +0.0), and == the library-sort form."""
    rng = np.random.default_rng(n)
    bias = (rng.integers(-3, 4, size=n).astype(F32) * 0.25)          # many exact ties
    if n > 10:
        bias[3], bias[9] = -0.0, 0.0
    assert K.BIAS_ORDER == 'kernel'
    perm = K.bias_processing_order(dev(bias))
    assert perm.dtype.is_floating_point is False and perm.shape == (n,)
    assert np.array_equal(perm.cpu().numpy(), np.argsort(-bias, kind='stable'))
    monkeypatch.setattr(K, 'BIAS_ORDER', 'torch')
    assert np.array_equal(K.bias_processing_order(dev(bias)).cpu().numpy(), perm.cpu().numpy())


@pytest.mark.parametrize('U,I,d,k,regime,cosine,splits', [
    (100, 150, 100, 10, 'tag', False, None), (500, 3000, 128, 10, 'indicator', False, None),
    (200, 2000, 64, 12, 'tag', True, 3), (1000, 20000, 128, 10, 'indicator', False, 1),
    (130, 5000, 10, 5, 'tag', False, 7), (1, 700, 64, 1, 'tag', False, None),
])
def test_filter_topk_float_matches_oracle(K, U, I, d, k, regime, cosine, splits):
    uf, itf, wu, wi, bu, bi = make_case(U, I, d, False, seed=U + 1, regime=regime)
    model = oracle.OracleModel([wu], wi, bu, bi, prediction='cosine' if cosine else 'dot')
    scores = model.predict(uf, itf)
    ur, ir = model.user_representation(uf)[0], model.item_representation(itf)
    if cosine:
        ur, ir = oracle.l2_normalize(ur), oracle.l2_normalize(ir)
    tol = H.norm_tolerance(ur, ir, rel=1e-5) + 2e-6
    got_s, got_i, info = run_filter(K, uf, itf, wu, wi, bu, bi, k, n_splits=splits, n_norm=1 if cosine else 0)
    rows = np.arange(U)[:, None]
    assert got_i.min() >= 0 and got_i.max() < I
    assert np.all(np.abs(got_s - scores[rows, got_i]) <= tol[rows, got_i])      # exact fp32 re-scoring: 1e-5
    mask = np.ones_like(scores, dtype=bool)
    mask[rows, got_i] = False
    assert np.all((scores - tol)[mask].reshape(U, -1) <= got_s[:, -1:] + 1e-6)  # nothing better was left out
    assert np.all(np.diff(got_s, axis=1) <= 0)
    exp_i, _ = oracle.top_k_from_scores(scores, k)
    assert (got_i != exp_i).mean() < 0.01                                        # only sub-tolerance near-ties may swap
    assert info['fallback_rows'] <= U // 20                                      # continuous scores: the bound certifies


@pytest.mark.parametrize('U,I,d,k,splits', [(100, 150, 100, 10, None), (256, 4096, 64, 10, 2), (129, 513, 10, 3, 4)])
def test_filter_topk_integer_fixture_exact_through_fallback(K, U, I, d, k, splits):
    """Massive ties: the filter cannot separate equal scores within its bound, overflows and hands those rows to the
    exact kernel -- the combined result must still be the reference order bit for bit."""
    uf, itf, wu, wi, bu, bi = make_case(U, I, d, True, seed=U + I)
    scores = oracle_scores(uf, itf, wu, wi, bu, bi)
    exp_i, exp_s = oracle.top_k_from_scores(scores, k)
    got_s, got_i, info = run_filter(K, uf, itf, wu, wi, bu, bi, k, n_splits=splits)
    assert np.array_equal(got_i, exp_i) and np.array_equal(got_s, exp_s)


@pytest.mark.parametrize('sort_by_bias', [True, False])
def test_filter_candidates_respect_the_error_bound(K, sort_by_bias):
    """The approximate scores of the survivors are within m = 1.5*2^-10 |u| max|i| of the exact ones, and every true
    top-k item is among the survivors."""
    import torch
    U, I, d, k = 300, 6000, 128, 10
    uf, itf, wu, wi, bu, bi = make_case(U, I, d, False, seed=9, regime='indicator')
    users, items = side_operands(K, uf, wu, bu, d), side_operands(K, itf, wi, bi, d)
    stats = torch.zeros(3, device='cuda')
    unorm = K.operand_stats(users.split, users.scale, users.d_pad)
    K.operand_stats(items.split, items.scale, items.d_pad, want_norm=False, stats=stats)
    perm = K.bias_processing_order(items.bias) if sort_by_bias else None
    hi = K.rescale_hi_global(items.split, items.scale, stats, items.d_pad, perm=perm)
    bias_pad, bmax, bmin = K.pack_item_bias(items.bias, I, stats, 'cuda', perm=perm, want_min=True)
    assert np.array_equal(bmin.cpu().numpy(), bias_pad.cpu().numpy().reshape(-1, 128).min(axis=1))
    cs, ci, theta = K.score_filter(users.split, users.scale, users.bias, unorm, hi, stats, bias_pad, bmax, perm,
                                   U, I, users.d_pad, k, n_splits=2, block_bias_min=bmin)
    scores = oracle_scores(uf, itf, wu, wi, bu, bi)
    cs, ci = cs.cpu().numpy().reshape(U, -1), ci.cpu().numpy().reshape(U, -1)
    m = 1.5 * 2.0 ** -10 * unorm.cpu().numpy() * stats.cpu().numpy()[0] + 1e-5
    exp_i, _ = oracle.top_k_from_scores(scores, k)
    for u in range(U):
        real = ci[u] != 2 ** 31 - 1
        assert np.all(np.abs(cs[u][real] - scores[u, ci[u][real]]) <= m[u])
        assert set(exp_i[u]) <= set(ci[u][real])
        assert real.sum() <= 32


@pytest.mark.parametrize('U,I,d,k,integer', [(700, 9000, 128, 10, False), (300, 1500, 64, 5, True), (257, 513, 100, 12, False),
                                             (513, 40000, 64, 10, False), (1100, 3000, 128, 10, False)])
@pytest.mark.parametrize('cluster', ['1', '2'])
def test_filter_user_block_and_kblock_shapes(K, monkeypatch, cluster, U, I, d, k, integer):
    """Ragged user blocks (U not a multiple of 256: rows past the end arrive as zero rows), one and two
    k-blocks (d_pad 64 / 128), several work units per CTA; both launch forms: independent CTAs and clusters of two
    CTAs sharing the item tiles by TMA multicast (an odd number of 256-user groups leaves one CTA of the last cluster
    without users)."""
    monkeypatch.setenv('TRK_FILTER_CLUSTER', cluster)
    uf, itf, wu, wi, bu, bi = make_case(U, I, d, integer, seed=U + I, regime='tag' if integer else 'indicator')
    scores = oracle_scores(uf, itf, wu, wi, bu, bi)
    exp_i, exp_s = oracle.top_k_from_scores(scores, k)
    got_s, got_i, info = run_filter(K, uf, itf, wu, wi, bu, bi, k)
    if integer:
        assert np.array_equal(got_i, exp_i) and np.array_equal(got_s, exp_s)
    else:
        rows = np.arange(U)[:, None]
        model = oracle.OracleModel([wu], wi, bu, bi)
        tol = H.norm_tolerance(model.user_representation(uf)[0], model.item_representation(itf)) + 2e-6
        assert np.all(np.abs(got_s - scores[rows, got_i]) <= tol[rows, got_i])
        assert (got_i != exp_i).mean() < 0.01
        assert info['fallback_rows'] <= U // 20


# ------------------------------------------------------------------------------------------------- adversarial filter cases
def check_float_topk(scores, tol, got_s, got_i, k):
    U = scores.shape[0]
    rows = np.arange(U)[:, None]
    assert np.all(np.abs(got_s - scores[rows, got_i]) <= tol[rows, got_i])
    mask = np.ones_like(scores, dtype=bool)
    mask[rows, got_i] = False
    assert np.all((scores - tol)[mask].reshape(U, -1) <= got_s[:, -1:] + 1e-6)
    assert np.all(np.diff(got_s, axis=1) <= 0)


def test_filter_item_bias_dominates_the_dot_products(K):
    """|item bias| ~ 1e3 x the dot products: the admission bound, the 4-ulp bias term of m and the re-scoring all work
    on numbers whose fp32 spacing is of the order of the dot products themselves."""
    U, I, d, k = 300, 20000, 128, 10
    uf, itf, wu, wi, bu, bi = make_case(U, I, d, False, seed=21, regime='indicator')
    bi = (bi * 1e4).astype(F32)
    model = oracle.OracleModel([wu], wi, bu, bi)
    scores = model.predict(uf, itf)
    tol = H.norm_tolerance(model.user_representation(uf)[0], model.item_representation(itf)) + \
        8 * np.spacing(np.abs(scores).astype(F32))
    got_s, got_i, info = run_filter(K, uf, itf, wu, wi, bu, bi, k)
    check_float_topk(scores, tol, got_s, got_i, k)


def test_filter_norms_spanning_forty_binades(K):
    """Row norms from 2^-20 to 2^20 on both sides: the per-row power-of-two scales differ by 2^40, the global item
    rescale pushes small items into fp16 subnormals (flush is inside the bound), every user has its own margin."""
    U, I, d, k = 256, 6000, 64, 10
    uf, itf, wu, wi, bu, bi = make_case(U, I, d, False, seed=22, regime='indicator')
    rng = np.random.default_rng(0)
    wu = (wu * np.exp2(rng.integers(-20, 21, size=(wu.shape[0], 1)))).astype(F32)
    wi = (wi * np.exp2(rng.integers(-20, 21, size=(wi.shape[0], 1)))).astype(F32)
    model = oracle.OracleModel([wu], wi, None, None)
    scores = model.predict(uf, itf)
    ur, ir = model.user_representation(uf)[0], model.item_representation(itf)
    # the contract is relative to |u| max_j |i_j| (the filter's error unit), rows with tiny items carry that slack
    tol = (1e-5 * np.linalg.norm(ur, axis=1)[:, None] * np.linalg.norm(ir, axis=1).max()).astype(np.float64) + 1e-30
    tol = np.broadcast_to(tol, scores.shape)
    got_s, got_i, info = run_filter(K, uf, itf, wu, wi, None, None, k)
    check_float_topk(scores.astype(np.float64), tol, got_s.astype(np.float64), got_i, k)


@pytest.mark.parametrize('cluster', ['1', '2'])
def test_filter_all_scores_equal_at_200k_items(K, monkeypatch, cluster):
    """Every score identical (zero weights, constant bias): the top-k is items 0..k-1 for every user, the filter can
    certify nothing and every row goes through the device-side fallback."""
    monkeypatch.setenv('TRK_FILTER_CLUSTER', cluster)
    U, I, d, k = 64, 200000, 64, 12
    uf = H.indicator_features(U, seed=1)
    itf = H.indicator_features(I, seed=2, tags_per_row=0)      # one entry per item: every projected bias is 0.5
    wu = np.zeros((uf.shape[1], d), F32)
    wi = np.zeros((itf.shape[1], d), F32)
    bu = np.zeros(uf.shape[1], F32)
    bi = np.full(itf.shape[1], 0.5, F32)
    got_s, got_i, info = run_filter(K, uf, itf, wu, wi, bu, bi, k)
    scores = oracle_scores(uf, itf, wu, wi, bu, bi)
    exp_i, exp_s = oracle.top_k_from_scores(scores, k)
    assert np.array_equal(got_i, exp_i) and np.array_equal(got_s, exp_s)
    assert info['fallback_rows'] == U


def test_filter_cluster_pairs_with_splits_and_a_ragged_last_tile(K, monkeypatch):
    """2-CTA clusters x several item splits x an item count that leaves a 1-item last tile, U an odd number of
    256-user groups."""
    monkeypatch.setenv('TRK_FILTER_CLUSTER', '2')
    for (U, I, splits, integer) in [(769, 128 * 37 + 1, 3, False), (300, 128 * 9 + 1, 4, True)]:
        uf, itf, wu, wi, bu, bi = make_case(U, I, 128, integer, seed=U, regime='tag' if integer else 'indicator')
        scores = oracle_scores(uf, itf, wu, wi, bu, bi)
        exp_i, exp_s = oracle.top_k_from_scores(scores, 10)
        got_s, got_i, info = run_filter(K, uf, itf, wu, wi, bu, bi, 10, n_splits=splits)
        if integer:
            assert np.array_equal(got_i, exp_i) and np.array_equal(got_s, exp_s)
        else:
            model = oracle.OracleModel([wu], wi, bu, bi)
            tol = H.norm_tolerance(model.user_representation(uf)[0], model.item_representation(itf)) + 2e-6
            check_float_topk(scores, tol, got_s, got_i, 10)
            assert (got_i != exp_i).mean() < 0.01


@pytest.mark.parametrize('cluster', ['1', '2'])
def test_filter_variants_with_and_without_the_tile_end_pass_agree(K, monkeypatch, cluster):
    """Tile-end compaction at the default trigger, at another trigger, and turned off by the probe knob: same certified
    result, bit for bit, and equal to the oracle's."""
    monkeypatch.setenv('TRK_FILTER_CLUSTER', cluster)
    for (U, I, d, k, splits) in [(700, 40000, 128, 10, 1), (300, 9000, 64, 12, 2)]:
        uf, itf, wu, wi, bu, bi = make_case(U, I, d, False, seed=I, regime='indicator')
        got = {}
        for name, trigger in (('default', None), ('tile_end', '20'), ('plain', '32')):
            if trigger is None:
                monkeypatch.delenv('TRK_FILTER_TILE_END_TRIGGER', raising=False)
            else:
                monkeypatch.setenv('TRK_FILTER_TILE_END_TRIGGER', trigger)
            got[name] = run_filter(K, uf, itf, wu, wi, bu, bi, k, n_splits=splits)
        for name in ('tile_end', 'plain'):
            assert np.array_equal(got[name][1], got['default'][1]) and np.array_equal(got[name][0], got['default'][0])
        scores = oracle_scores(uf, itf, wu, wi, bu, bi)
        model = oracle.OracleModel([wu], wi, bu, bi)
        tol = H.norm_tolerance(model.user_representation(uf)[0], model.item_representation(itf)) + 2e-6
        check_float_topk(scores, tol, got['plain'][0], got['plain'][1], k)


def test_filter_infinite_item_biases_stay_nan_free(K):
    """-inf biases (items that must never be recommended) and a few +inf ones: no NaN reaches the result, the +inf
    items lead every list in id order, no -inf item is returned while finite ones remain."""
    U, I, d, k = 130, 3000, 64, 10
    uf, itf, wu, wi, bu, bi = make_case(U, I, d, False, seed=23, regime='indicator')
    itf = sp.csr_matrix(itf)
    # the identity column of an item carries its own bias entry: set those directly
    bi = bi.copy()
    bi[:I] = 0.0
    bi[5:I:7] = -np.inf
    bi[[11, 400]] = np.inf
    # tag columns keep finite biases; an item's projected bias = its identity entry + its tags
    got_s, got_i, info = run_filter(K, uf, itf, wu, wi, bu, bi, k)
    with np.errstate(invalid='ignore'):
        scores = oracle_scores(uf, itf, wu, wi, bu, bi)
    assert not np.isnan(got_s).any()
    exp_i, exp_s = oracle.top_k_from_scores(scores, k)
    assert np.array_equal(got_i[:, :2], exp_i[:, :2]) and np.all(np.isposinf(got_s[:, :2]))
    assert not np.isneginf(got_s).any()
    model = oracle.OracleModel([wu], wi, bu, bi)
    tol = H.norm_tolerance(model.user_representation(uf)[0], model.item_representation(itf)) + 2e-6
    rows = np.arange(U)[:, None]
    assert np.all(np.abs(got_s[:, 2:] - scores[rows, got_i[:, 2:]]) <= tol[rows, got_i[:, 2:]])


def test_certified_and_fallback_rows_are_bit_identical_on_an_integer_fixture(K):
    """A row's result must not depend on the route it took: re-scoring from the split operands (certified rows) and
    the exact tensor-core kernel (rows routed through the device-side fallback) give the same bits when the arithmetic
    is exact.  Continuous biases make the certificate pass for most rows of this integer-weight fixture; then every
    row is forced through the fallback and the two results are compared."""
    import torch
    U, I, d, k = 300, 5000, 64, 10
    uf, itf, wu, wi, bu, bi = make_case(U, I, d, True, seed=31)
    bi = (np.arange(bi.shape[0]) % 97 * 0.125).astype(F32)         # exact in fp32, spreads the scores: few ties
    users, items = side_operands(K, uf, wu, bu, d), side_operands(K, itf, wi, bi, d)
    top, counters, cap = K.topk_filter(users, items, k)
    certified = U - int(counters[0])
    assert certified > U // 2, 'fixture should certify most rows (got %d of %d)' % (certified, U)
    forced = K.PackedTopK(U, k, 'cuda')
    forced.buf.zero_()
    c2, _ = K.rerun_uncertified(users, items, torch.ones(U, dtype=torch.int32, device='cuda'), forced, k)
    assert int(c2[0]) == U
    assert torch.equal(top.buf, forced.buf)
    exp_i, exp_s = oracle.top_k_from_scores(oracle_scores(uf, itf, wu, wi, bu, bi), k)
    assert np.array_equal(top.items.cpu().numpy(), exp_i) and np.array_equal(top.scores.cpu().numpy(), exp_s)


def test_device_side_fallback_overflow_is_reported(K):
    """More flagged rows than the fallback buffer holds: counters[0] > capacity tells the host layer to re-run the batch
    through the exact kernel; the device-side tiers then do no work and nothing is written out of bounds."""
    import torch
    U = 5000
    uf, itf, wu, wi, bu, bi = make_case(U, 300, 64, True, seed=33)
    users, items = side_operands(K, uf, wu, bu, 64), side_operands(K, itf, wi, bi, 64)
    top = K.PackedTopK(U, 5, 'cuda')
    top.buf.fill_(-7)
    counters, cap = K.rerun_uncertified(users, items, torch.ones(U, dtype=torch.int32, device='cuda'), top, 5)
    assert cap == 1024 and int(counters[0]) == U
    assert bool((top.buf == -7).all())


def test_device_side_fallback_large_tier(K, monkeypatch):
    """More flagged rows than the small tier holds but fewer than the capacity: the large tier re-scores them."""
    import torch
    monkeypatch.setattr(K, 'FALLBACK_SMALL_ROWS', 128)
    U, I, k = 1500, 700, 5
    uf, itf, wu, wi, bu, bi = make_case(U, I, 64, True, seed=34)
    users, items = side_operands(K, uf, wu, bu, 64), side_operands(K, itf, wi, bi, 64)
    exp_i, exp_s = oracle.top_k_from_scores(oracle_scores(uf, itf, wu, wi, bu, bi), k)
    flags = torch.zeros(U, dtype=torch.int32, device='cuda')
    chosen = np.arange(0, U, 3)                                  # 500 rows: > 128, < capacity (1024)
    flags[torch.from_numpy(chosen).cuda()] = 1
    top = K.PackedTopK(U, k, 'cuda')
    top.buf.fill_(-7)
    counters, cap = K.rerun_uncertified(users, items, flags, top, k)
    c = counters.cpu().numpy()
    assert c[0] == len(chosen) and c[2] == 0 and c[3] == len(chosen)
    got_i, got_s = top.items.cpu().numpy(), top.scores.cpu().numpy()
    assert np.array_equal(got_i[chosen], exp_i[chosen]) and np.array_equal(got_s[chosen], exp_s[chosen])
    rest = np.setdiff1d(np.arange(U), chosen)
    assert np.all(top.buf.cpu().numpy()[rest] == -7)
