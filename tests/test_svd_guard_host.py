"""Host side of the reference's SVD degeneracy guard (rigid_docking_model.py:570-586): the fp64 restatement of
tests/heads_ref.py against the numpy oracle with the same draws, its autograd gradient through a perturbed covariance
against central finite differences, and its replay of the engine's CPU-generator draws (IEGMNEngine._resolve_status,
run here on host covariances with the guard test of kabsch_apply_kernel done on the host).  Needs no GPU."""
import types

import numpy as np
import pytest
import torch

import heads_ref as hr
import iegmn_oracle as orc
from equidock_public_b200 import _native as nat
from equidock_public_b200.engine import IEGMNEngine, draw_dropout

CPU = torch.device('cpu')
F64 = torch.float64


def _sd(K):
    return {k: v.detach().double() for k, v in hr.build_model('dips', CPU, K, seed=K).state_dict().items()}


def _protein(rng, n, collapsed=False):
    h = rng.normal(0, 0.7, (n, 64))
    x = rng.normal(0, 8.0, (n, 3))
    return h, np.tile(x[:1], (n, 1)) if collapsed else x


def _noise(seed, n=12):
    rng = np.random.default_rng(seed)
    return [rng.uniform(0, 1, 3) for _ in range(n)]


def _counting(draws):
    it, used = iter(draws), [0]

    def nxt():
        used[0] += 1
        return next(it)
    return nxt, used


def _tail(sd, K, hl, xl, hr_, xr, rand_diag, x_lig=None, trace=None):
    h = torch.from_numpy(np.concatenate([hl, hr_]))
    x = torch.from_numpy(np.concatenate([xl, xr]))
    seg = [0, len(hl), len(hl) + len(hr_)]
    return hr.keypoint_tail(sd, h, x, x[:len(hl)] if x_lig is None else x_lig, seg, 1, K, 0.01, rand_diag=rand_diag,
                            trace=trace)


CASES = [(1, 'natural'), (2, 'natural'), (3, 'natural'), (4, 'natural'), (4, 'collapsed'), (50, 'natural'),
         (50, 'collapsed')]


@pytest.mark.parametrize('K,kind', CASES)
def test_tail_equals_the_numpy_oracle_with_the_same_draws(K, kind):
    """K <= 3 keypoints span at most a plane after centring, so the guard fires on every pair; at K = 4 and 50 it fires
    only when all receptor nodes coincide (A = 0)."""
    sd = _sd(K)
    rng = np.random.default_rng([K, len(kind)])
    hl, xl = _protein(rng, 37)
    hr_, xr = _protein(rng, 52, kind == 'collapsed')
    noise = _noise(K)
    cfg = orc.OracleConfig(8, 0.5, 0.0, 0.01, K)
    nxt_o, used_o = _counting(noise)
    T, b, y_l, y_r, info = orc.keypoints_and_kabsch({k: v.numpy() for k, v in sd.items()}, cfg, hl, xl, hr_, xr,
                                                    np.float64, rand_diag=_Iter(nxt_o))
    nxt, used = _counting(noise)
    trace = {}
    co, Y, R, t, draws = _tail(sd, K, hl, xl, hr_, xr, nxt, trace=trace)
    fires = K <= 3 or kind == 'collapsed'
    assert info['flagged'] == fires and (draws[0] > 0) == fires
    assert draws[0] == used[0] == used_o[0], (draws, used, used_o)
    if fires:
        assert orc.svd_guard_flags(np.linalg.svd(info['A'] - sum(np.diag(n) for n in noise[:draws[0]]),
                                                 compute_uv=False).astype(np.float32))
    assert not orc.svd_guard_flags(torch.linalg.svdvals(trace['A'][0]).float().numpy())
    s2 = np.linalg.svd(trace['A'][0].numpy(), compute_uv=False) ** 2
    print(f'\nK={K} {kind}: draws {draws[0]}, smallest squared-singular-value gap {np.abs(np.diff(s2)).min():.3e}')
    assert np.abs(trace['A'][0].numpy() - info['A']).max() <= 1e-12 * np.abs(info['A']).max()
    assert np.abs(Y[0].numpy() - y_l).max() <= 1e-12 * np.abs(y_l).max()
    assert np.abs(Y[1].numpy() - y_r).max() <= 1e-12 * np.abs(y_r).max()
    assert np.abs(R[0].numpy() - T).max() <= 1e-10
    assert abs(np.linalg.det(R[0].numpy()) - 1.0) <= 1e-12
    assert np.abs(t.numpy() - b).max() <= 1e-10 * max(1.0, np.abs(b).max())
    assert np.abs(co.numpy() - (xl @ T.T + b)).max() <= 1e-10 * max(1.0, np.abs(co.numpy()).max())


class _Iter:
    """An iterator over a callable's results (the oracle takes an iterator, the restatement a callable)."""

    def __init__(self, fn):
        self.fn = fn

    def __iter__(self):
        return self

    def __next__(self):
        return self.fn()


def test_tail_without_a_noise_source_refuses_to_compare_against_unperturbed_kabsch():
    sd = _sd(2)
    rng = np.random.default_rng(0)
    with pytest.raises(RuntimeError, match='no noise source'):
        _tail(sd, 2, *_protein(rng, 20), *_protein(rng, 30), None)


@pytest.mark.parametrize('K', [2, 50])
def test_autograd_through_the_perturbed_covariance_matches_central_differences(K):
    """d/dh, d/dx and d/d(key weights) of a fixed linear functional of the pose and the keypoints, through a covariance
    the guard perturbed (K = 2: every pair; K = 50: a receptor collapsed to one point), against central differences at
    the same draws."""
    sd = _sd(K)
    rng = np.random.default_rng(7 + K)
    hl, xl = _protein(rng, 23)
    hr_, xr = _protein(rng, 31, collapsed=K == 50)
    noise = _noise(100 + K)
    wc = torch.from_numpy(rng.normal(0, 1, (23, 3)))
    wy = torch.from_numpy(rng.normal(0, 1, (2, K, 3)))
    h0 = torch.from_numpy(np.concatenate([hl, hr_]))
    x0 = torch.from_numpy(np.concatenate([xl, xr]))
    seg = [0, 23, 54]

    def f(h, x, wk):
        s = dict(sd, **{'iegmn_original.att_mlp_key_ROT.0.weight': wk})
        nxt, _ = _counting(noise)
        co, Y, _, _, draws = hr.keypoint_tail(s, h, x, x[:23], seg, 1, K, 0.01, rand_diag=nxt)
        assert draws[0] > 0
        return (co * wc).sum() + (Y * wy).sum(), draws

    leaves = [h0.clone().requires_grad_(True), x0.clone().requires_grad_(True),
              sd['iegmn_original.att_mlp_key_ROT.0.weight'].clone().requires_grad_(True)]
    val, draws = f(*leaves)
    val.backward()
    eps = 1e-6
    for i, leaf in enumerate(leaves):
        flat = leaf.detach().reshape(-1)
        for j in np.random.default_rng(i).choice(flat.numel(), 6, replace=False):
            args = [v.detach().clone() for v in leaves]
            args[i].view(-1)[j] += eps
            fp, dp = f(*args)
            args[i].view(-1)[j] -= 2 * eps
            fm, dm_ = f(*args)
            assert dp == dm_ == draws
            fd = float(fp - fm) / (2 * eps)
            ad = float(leaf.grad.reshape(-1)[j])
            assert abs(fd - ad) <= 1e-5 * max(1.0, abs(ad)), (i, j, fd, ad)


# ---- the engine's host loop, with the device's guard test done on the host -------------------------------------------

def _host_engine():
    eng = object.__new__(IEGMNEngine)
    eng.device = CPU
    return eng


def _flag(cov):
    return nat.STATUS_SVD_DEGENERATE if orc.svd_guard_flags(torch.linalg.svdvals(cov.view(3, 3)).float().numpy()) else 0


def _engine_resolve(covs, log=None):
    """IEGMNEngine._resolve_status over host covariances (B,9): kabsch_apply's status from the fp32-rounded singular
    values, as the kernel sets it.  Returns the engine's output dict."""
    B = covs.shape[0]
    status = torch.tensor([_flag(c) for c in covs], dtype=torch.int32)
    out = {'status_event': types.SimpleNamespace(synchronize=lambda: None), 'cov': covs.clone(), 'status': status,
           'status_host': torch.cat([status, torch.zeros(2, dtype=torch.int32)])}

    def kab(mask):
        for b in torch.nonzero(mask).reshape(-1).tolist():
            out['status'][b] = _flag(out['cov'][b])
    _host_engine()._resolve_status(types.SimpleNamespace(n_pairs=B), out, kab, log)
    return out


def _covs(rng):
    """Pairs: A = 0, well conditioned, rank 1, well conditioned, two equal singular values."""
    Q = lambda: np.linalg.qr(rng.normal(size=(3, 3)))[0]
    good = lambda: Q() @ np.diag([9.0, 4.0, 1.5]) @ Q().T
    v = rng.normal(size=3)
    return torch.from_numpy(np.stack([np.zeros((3, 3)), good(), np.outer(v, v), good(),
                                      Q() @ np.diag([2.0, 2.0, 0.5]) @ Q().T]).reshape(5, 9))


@pytest.mark.parametrize('p', [0.0, 0.25])
def test_replay_reproduces_the_engine_draw_order(p):
    """A training forward draws its dropout seed (p > 0) and then the guard's noise, flagged pairs in order: replay_draws
    + guarded_kabsch pair by pair take the same draws (same counts, bitwise the same perturbed covariances, the same
    generator state after)."""
    covs = _covs(np.random.default_rng(5))
    torch.manual_seed(77)
    dropout = draw_dropout(p)
    out = _engine_resolve(covs)
    state = torch.get_rng_state()
    assert out['guard_draws'][1] == out['guard_draws'][3] == 0
    assert all(out['guard_draws'][b] > 0 for b in (0, 2, 4))
    d2, rand_diag = hr.replay_draws(77, p)
    assert (d2 is None) == (p == 0) and (d2 is None or d2 == dropout)
    for b in range(covs.shape[0]):
        _, n, A = hr.guarded_kabsch(covs[b].view(3, 3).clone(), rand_diag)
        assert n == out['guard_draws'][b], b
        assert torch.equal(A.reshape(9), out['cov'][b]), b
    assert torch.equal(torch.get_rng_state(), state)
    # the dropout draw shifts the noise: the replay without it would read other values
    if p > 0:
        _, rd0 = hr.replay_draws(77, 0.0)
        _, n, A = hr.guarded_kabsch(covs[0].view(3, 3).clone(), rd0)
        assert not torch.equal(A.reshape(9), out['cov'][0])


def test_guard_exits_after_eleven_draws_like_the_reference():
    """Two singular values of 1e12: their fp32 squares coincide whatever noise of size 1 is added, so the guard never
    passes.  The engine, the restatement and the numpy oracle all exit after the 11th draw with the reference's message."""
    c = torch.diag(torch.tensor([1e12, 1e12, 3.0], dtype=F64)).reshape(1, 9)
    covs = torch.cat([_covs(np.random.default_rng(1))[1:2], c])
    logged = []
    torch.manual_seed(3)
    with pytest.raises(SystemExit):
        _engine_resolve(covs, logged.append)
    state = torch.get_rng_state()
    assert logged == [hr.GUARD_EXIT]
    torch.manual_seed(3)
    for _ in range(11):
        torch.rand(3, 3)
    assert torch.equal(torch.get_rng_state(), state)
    _, rand_diag = hr.replay_draws(3)
    with pytest.raises(SystemExit, match=hr.GUARD_EXIT.strip()):
        hr.guarded_kabsch(c.view(3, 3).clone(), rand_diag)
    assert torch.equal(torch.get_rng_state(), state)


def test_kink_branch_keeps_values_and_sets_the_derivative_near_the_kink():
    orig = torch.nn.functional.leaky_relu
    z = torch.tensor([[1e-9, -1e-9, 2.0, -3.0], [0.0, 4e-6, -1.0, 0.5]], dtype=F64, requires_grad=True)
    ref = torch.nn.functional.leaky_relu(z.detach(), 0.01)
    for positive, d in ((True, 1.0), (False, 0.01)):
        with hr.kink_branch(1e-5, positive):
            y = torch.nn.functional.leaky_relu(z, 0.01)
        assert torch.equal(y.detach(), ref)
        z.grad = None
        y.sum().backward()
        # within 1e-5 of the row's max |z|: the chosen side; farther, and exactly 0: leaky_relu's own derivative
        assert z.grad.tolist() == [[d, d, 1.0, 0.01], [0.01, d, 0.01, 1.0]]
    assert torch.nn.functional.leaky_relu is orig
