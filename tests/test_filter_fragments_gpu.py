"""The filter kernel's per-row ownership of the wgmma fragments, position by position (needs an H100: pytest -m gpu).

A consumer warp owns the 32 user rows whose accumulator fragments it holds, finds each row's maximum of a 32-column
chunk by shuffles and stages a chunk only when some row passes.  Here every one of 256 user rows (both user blocks of
a work unit, so every warp, lane and register class) has one dominant item in a chunk of its own, whose processing
column is the row's index mod 32: over the rows the winners run through all 32 columns of a chunk and all four chunks
of a tile.  Items have distinct biases, so their processing order is their index.  One split makes the sweep one work
unit: after the first tile the threshold sits far above every item but the winners, so a winner is found only if the
register maximum of its row reaches the row's owner.  A wrong owner, shuffle source or staging address reports a wrong
item rather than a slightly different score; the scores are exact, so the result must equal the oracle's top-k
exactly, with every row certified by the filter (none left to the exact fallback kernel)."""
import numpy as np
import pytest
import scipy.sparse as sp

import oracle
from tests.masked_topk import masked_top_k

pytestmark = pytest.mark.gpu

U, D, K = 256, 128, 10
FIRST = 256                       # winners start past the first two tiles (the first one sets the threshold)
N_ITEMS = FIRST + 32 * U + 37     # one 32-column chunk per user row, and a ragged last tile


def winner(r):
    return FIRST + 32 * r + r % 32


def second_winner(r):
    return FIRST + 32 * r + (7 * r + 5) % 32      # != r % 32 for every r


@pytest.fixture(scope='module')
def Kn():
    import torch
    from tensorrec_b200 import kernels
    kernels.require_cuda()
    torch.cuda.set_device(0)
    return kernels


def make_case(second):
    """Identity features: the representations are the weight rows.  User r is 16 s e_j (j = r % 128, s = -1 for the
    second user block); its winners have the same vector, so they score 256 for r, -256 for r +- 128 and 0 for every
    other user.  Every other item is the zero vector.  Biases descend with the item index: 1/4 apart on the first tile
    (the k-th best of every row sits there), 1/256 apart after it, 32 or more below the first tile."""
    wu = np.zeros((U, D), np.float32)
    wi = np.zeros((N_ITEMS, D), np.float32)
    for r in range(U):
        v = np.zeros(D, np.float32)
        v[r % D] = 16.0 if r < D else -16.0
        wu[r] = v
        wi[winner(r)] = v
        if second and r % 3 == 0:
            wi[second_winner(r)] = v
    pos = np.arange(N_ITEMS, dtype=np.float64)
    bi = np.where(pos < 128, -0.25 * pos, -32.0 - pos / 256.0).astype(np.float32)
    bu = np.zeros(U, np.float32)
    uf = sp.identity(U, dtype=np.float32, format='csr')
    itf = sp.identity(N_ITEMS, dtype=np.float32, format='csr')
    return uf, itf, wu, wi, bu, bi


def side_operands(Kn, feats, w, b):
    import torch
    csr = Kn.DeviceCSR.from_scipy(feats)
    d_pad = Kn.d_pad_for(D)
    stats = torch.empty(3, device='cuda')
    f32, split, scale, norm = Kn.gather_reduce(csr, torch.from_numpy(w).cuda(), want_f32=True, split_d_pad=d_pad,
                                               want_norm=True, stats=stats)
    bias = Kn.project_biases(csr, torch.from_numpy(b).cuda())
    return Kn.SideOperands(f32, split, scale, bias, feats.shape[0], D, d_pad, norm=norm, stats=stats)


@pytest.mark.parametrize('cluster', ['1', '2'])
@pytest.mark.parametrize('second', [False, True])
@pytest.mark.parametrize('mask_winner', [False, True])
def test_every_fragment_position_reaches_its_owner(Kn, monkeypatch, cluster, second, mask_winner):
    monkeypatch.setenv('TRK_FILTER_CLUSTER', cluster)
    uf, itf, wu, wi, bu, bi = make_case(second)
    scores = oracle.OracleModel([wu], wi, bu, bi).predict(uf, itf)
    rows = np.arange(U)
    excl = None
    if mask_winner:
        exclude = sp.csr_matrix((np.ones(U), (rows, [winner(r) for r in rows])), shape=(U, N_ITEMS))
        exp_i, exp_s = masked_top_k(scores, exclude, K)
        indptr, ids = Kn.exclusion_host_csr(exclude, 0, N_ITEMS)
        excl = Kn.DeviceExclusion.upload(indptr, ids, 'cuda')
    else:
        exp_i, exp_s = oracle.top_k_from_scores(scores, K)
    # the fixture does what it says: each row's dominant items lead its top-k
    lead = exp_i[:, 0]
    if not mask_winner:
        assert np.all((lead == [winner(r) for r in rows]) | (lead == [second_winner(r) for r in rows]))
    elif second:
        assert np.array_equal(lead[::3], [second_winner(r) for r in rows[::3]])
    users, items = side_operands(Kn, uf, wu, bu), side_operands(Kn, itf, wi, bi)
    top, counters, cap = Kn.topk_filter(users, items, K, n_splits=1, excl=excl)
    assert int(counters[0]) == 0, 'the certificate, not the exact kernel, must decide every row'
    assert np.array_equal(top.items.cpu().numpy(), exp_i)
    assert np.array_equal(top.scores.cpu().numpy(), exp_s)
