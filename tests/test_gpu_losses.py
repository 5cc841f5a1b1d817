"""GPU (H100): the training losses of csrc/losses.cu against fp64 references, where the solver and the reductions go wrong:
every storage layout of the exact-EMD solver, tied and degenerate costs, large coordinates, oversize and empty pockets,
the batch shape of a training step, and MSE / body-intersection reductions whose threads loop several times.

Every transport plan the device returns is certified optimal by oracle/loss_oracle.ot_certify (exact integer marginals,
no negative residual cycle), so a non-unique optimum is never a reason to skip a check: the OT value and BOTH keypoint
gradients are compared with fp64 sums over the kernel's own plan.  Loss weights are not the reference's defaults (a
missing weight would hide behind 1.0), except in one run of the training shape."""
import numpy as np
import pytest
import torch

import bench_train
import loss_oracle as lo
from equidock_public_b200 import _native as nat
from equidock_public_b200 import synthetic
from equidock_public_b200.engine import GraphPlan
from equidock_public_b200.losses import PocketBatch, check_loss_status, device_losses

pytestmark = pytest.mark.gpu
M = nat.HEADS
_f32 = lambda v: float(np.float32(v))   # the C ABI takes the weights as float
WEIGHTS = dict(w_ot=_f32(0.37), w_int=_f32(3.1), sigma=_f32(17.0), ct=_f32(6.5))
DEFAULTS = dict(w_ot=1.0, w_int=10.0, sigma=25.0, ct=10.0)
KINK_REL = 1e-9       # |ct - G| below this x (|ct| + sigma |log S|): the kernel (fp64, same fp32 inputs) may take either side
KINK_MAX_FRACTION = 0.01


def _plan(sizes, dev):
    """GraphPlan of a batch with the given (N_lig, N_rec) per pair and no edges: the losses read only the node ranges."""
    z = torch.zeros(0, dtype=torch.int32)
    he = torch.zeros(0, nat.EDGE_FEATS)
    return GraphPlan([a for a, _ in sizes], [b for _, b in sizes], z, z, z, z, he, he, dev)


def _pockets(rng, kind, n):
    """(pocket_lig, pocket_rec) fp32 (n, 3) and (keypts_lig, keypts_rec) fp64 (50, 3) of one pair."""
    if kind == 'random':
        pl, pr = rng.normal(0, 12, (n, 3)), rng.normal(0, 12, (n, 3))
        kl, kr = rng.normal(0, 15, (M, 3)), rng.normal(0, 15, (M, 3))
    elif kind == 'one_keypoint':            # all 50 keypoints identical: every column of C is the same
        pl, pr = rng.normal(0, 12, (n, 3)), rng.normal(0, 12, (n, 3))
        kl, kr = np.repeat(rng.normal(0, 15, (1, 3)), M, 0), np.repeat(rng.normal(0, 15, (1, 3)), M, 0)
    elif kind == 'with_replacement':        # bench_train.make_targets: midpoints of residue pairs drawn with replacement
        a, b = rng.normal(0, 8, (24, 3)), rng.normal(0, 8, (24, 3)) + 8.0
        pl = 0.5 * (a[rng.integers(0, 24, n)] + b[rng.integers(0, 24, n)])
        pr = pl
        kl, kr = rng.normal(0, 10, (M, 3)), rng.normal(0, 10, (M, 3))
    elif kind == 'grid':                    # integer coordinates: many exactly equal costs
        pl, pr = rng.integers(-3, 4, (n, 3)), rng.integers(-3, 4, (n, 3))
        kl, kr = rng.integers(-3, 4, (M, 3)), rng.integers(-3, 4, (M, 3))
    elif kind == 'far':                     # ~1e3 A: |C| ~ 1e6, the lazy potential offsets grow large
        c = np.array([1e3, -1e3, 1e3])
        pl, pr = c + rng.normal(0, 300, (n, 3)), -c + rng.normal(0, 300, (n, 3))
        kl, kr = c + rng.normal(0, 300, (M, 3)), -c + rng.normal(0, 300, (M, 3))
    elif kind == 'same_pockets':            # pocket_lig == pocket_rec
        pl = rng.normal(0, 12, (n, 3))
        pr = pl
        kl, kr = rng.normal(0, 15, (M, 3)), rng.normal(0, 15, (M, 3))
    else:
        raise ValueError(kind)
    f32 = lambda a: np.asarray(a, np.float32)
    f64 = lambda a: np.asarray(a, np.float64)
    return f32(pl), f32(pr), f64(kl), f64(kr)


def _case(rng, n_pockets, kind='random', prot_sizes=None, geometry='overlap'):
    """One batch: per-pair fp32 predicted / bound ligand, bound receptor, pockets, and fp64 keypoints."""
    B = len(n_pockets)
    sizes = prot_sizes or [(20 + 3 * b, 25 + 2 * b) for b in range(B)]
    c = dict(sizes=sizes, pred=[], bl=[], br=[], pl=[], pr=[], kl=[], kr=[])
    for (nl, nr), n in zip(sizes, n_pockets):
        if geometry == 'overlap':           # overlapping bodies
            pred, rec = rng.normal(0, 6, (nl, 3)), rng.normal(2, 6, (nr, 3))
        elif geometry == 'all_active':      # tight clusters on top of each other: every term of both sums is active
            pred, rec = rng.normal(0, 0.3, (nl, 3)), rng.normal(0, 0.3, (nr, 3))
        elif geometry == 'none_active':     # 500 A apart: ct - G = ct + sigma log(1e-3) < 0 everywhere
            pred, rec = rng.normal(0, 6, (nl, 3)), rng.normal(0, 6, (nr, 3)) + 500.0
        elif geometry == 'straddle':        # half-overlapping: the ct - G = 0 kink runs through both bodies
            pred, rec = rng.normal(0, 4, (nl, 3)), rng.normal(0, 4, (nr, 3)) + np.array([8.0, 0, 0])
        else:
            raise ValueError(geometry)
        c['pred'].append(pred.astype(np.float32))
        c['bl'].append((pred + rng.normal(0, 1.5, pred.shape)).astype(np.float32))
        c['br'].append(rec.astype(np.float32))
        for key, v in zip(('pl', 'pr', 'kl', 'kr'), _pockets(rng, kind, n)):
            c[key].append(v)
    return c


def _run(c, W, dev):
    plan = _plan(c['sizes'], dev)
    t = lambda L: [torch.from_numpy(a) for a in L]
    tgt = PocketBatch(t(c['bl']), t(c['br']), t(c['pl']), t(c['pr']), dev)
    res = device_losses(plan, torch.from_numpy(np.concatenate(c['pred'])).to(dev),
                        torch.from_numpy(np.stack(c['kl'] + c['kr'])).to(dev), tgt, W['w_ot'], W['w_int'], W['sigma'], W['ct'])
    torch.cuda.synchronize()
    return plan, res


def _cost(c, b):
    return lo.sq_dist_mat(c['pl'][b], c['kl'][b]) + lo.sq_dist_mat(c['pr'][b], c['kr'][b])


def _check_ot_pair(c, res, W, b, p0, highs, worst):
    """Certified plan, value from the plan (1e-12), HiGHS optimum (1e-9, if `highs`), both keypoint gradients from the
    plan (1e-12 of the sum of magnitudes: the signed sum can cancel).  Returns the solver statistics parts[b, 3]."""
    B, n = len(c['pl']), c['pl'][b].shape[0]
    cost = _cost(c, b)
    x = res['plan'][p0:p0 + n].cpu().numpy()
    lo.ot_certify(cost, x)
    parts = res['parts'].cpu().numpy()
    val = float((x * cost).sum()) / (M * n)
    e = abs(parts[b, 1] - val)
    assert e <= 1e-12 * abs(val), (b, n, parts[b, 1], val)
    worst['ot_vs_plan'] = max(worst.get('ot_vs_plan', 0.0), e / max(abs(val), 1e-300))
    if highs:
        opt = lo.ot_emd(cost)[0]
        e = abs(parts[b, 1] - opt)
        assert e <= 1e-9 * max(abs(opt), 1.0), (b, n, parts[b, 1], opt)
        worst['ot_vs_highs'] = max(worst.get('ot_vs_highs', 0.0), e / max(abs(opt), 1.0))
    T = x.astype(np.float64) / (M * n)
    gsc = 2.0 * W['w_ot'] / B
    dk = res['dkeypts'].cpu().numpy()
    for row, P, Y in ((b, c['pl'][b], c['kl'][b]), (B + b, c['pr'][b], c['kr'][b])):
        diff = Y[None, :, :] - P.astype(np.float64)[:, None, :]                 # (n, 50, 3)
        ref = gsc * (T[:, :, None] * diff).sum(0)
        bound = 1e-12 * gsc * (T[:, :, None] * np.abs(diff)).sum(0)
        err = np.abs(dk[row] - ref)
        assert (err <= bound).all(), (b, row, n, float((err - bound).max()))
        worst['dkeypts'] = max(worst.get('dkeypts', 0.0), float((err / np.maximum(bound / 1e-12, 1e-300)).max()))
    return float(parts[b, 3])


def _check_coors(c, res, W, plan, worst, exclude_kink=True):
    """Per pair: MSE and intersection parts (1e-12 / 1e-10) and dcoors (1e-5 of the pair's max) against torch fp64
    autograd.  Ligand points whose fp64 margin to the ct - G = 0 kink is within KINK_REL, or that weigh on a receptor
    point within it, are left out of the dcoors comparison (at most KINK_MAX_FRACTION of the pair, at least 2 allowed).
    Returns (n active, n inactive) terms over the batch."""
    B = len(c['pred'])
    s, ct, w_int = W['sigma'], W['ct'], W['w_int']
    parts = res['parts'].cpu().numpy()
    dco = res['dcoors'].cpu().numpy().astype(np.float64)
    act = [0, 0]
    for b in range(B):
        p = torch.tensor(c['pred'][b].astype(np.float64), requires_grad=True)
        rec = torch.tensor(c['br'][b].astype(np.float64))
        E = torch.exp(-((p[:, None] - rec[None]) ** 2).sum(2) / s)                # (n_l, n_r)
        Sl, Sr = 1e-3 + E.sum(1), 1e-3 + E.sum(0)
        vl, vr = ct + s * torch.log(Sl), ct + s * torch.log(Sr)                    # ct - G_rec(l_j), ct - G_lig(r_i)
        mse = ((p - torch.tensor(c['bl'][b].astype(np.float64))) ** 2).mean()
        inter = torch.clamp(vl, min=0).mean() + torch.clamp(vr, min=0).mean()
        ((mse + w_int * inter) / B).backward()
        assert abs(parts[b, 0] - mse.item()) <= 1e-12 * max(mse.item(), 1e-300), (b, parts[b, 0], mse.item())
        assert abs(parts[b, 2] - inter.item()) <= 1e-10 * max(inter.item(), 1.0), (b, parts[b, 2], inter.item())
        worst['inter'] = max(worst.get('inter', 0.0), abs(parts[b, 2] - inter.item()) / max(inter.item(), 1.0))
        vl_, vr_, E_ = vl.detach().numpy(), vr.detach().numpy(), E.detach().numpy()
        act[0] += int((vl_ > 0).sum() + (vr_ > 0).sum())
        act[1] += int((vl_ <= 0).sum() + (vr_ <= 0).sum())
        keep = np.ones(len(vl_), bool)
        if exclude_kink:
            near_l = np.abs(vl_) <= KINK_REL * (abs(ct) + s * np.abs(np.log(Sl.detach().numpy())))
            near_r = np.abs(vr_) <= KINK_REL * (abs(ct) + s * np.abs(np.log(Sr.detach().numpy())))
            keep &= ~near_l
            if near_r.any():
                keep &= ~(E_[:, near_r] > 1e-9 * Sr.detach().numpy()[near_r]).any(1)
            assert (~keep).sum() <= max(2, KINK_MAX_FRACTION * len(keep)), (b, int((~keep).sum()))
        lo_, hi_ = plan.seg_ptr_host[b], plan.seg_ptr_host[b + 1]
        g, ref = dco[lo_:hi_][keep], p.grad.numpy()[keep]
        e = float(np.abs(g - ref).max() / max(np.abs(p.grad.numpy()).max(), 1e-300)) if keep.any() else 0.0
        assert e < 1e-5, (b, c['sizes'][b], e)
        worst['dcoors'] = max(worst.get('dcoors', 0.0), e)
    return act


def _check_totals(c, res, W, worst):
    ref, parts = lo.batch_loss(c['pred'], c['bl'], c['br'], c['kl'], c['kr'], c['pl'], c['pr'],
                               W['w_ot'], W['w_int'], W['sigma'], W['ct'])
    tot = res['total'].cpu().numpy()
    for got, want in ((tot[0], ref), (tot[1], parts['mse']), (tot[2], parts['ot']), (tot[3], parts['intersection'])):
        assert abs(got - want) <= 1e-9 * max(1.0, abs(want)), (tot, ref, parts)
        worst['totals'] = max(worst.get('totals', 0.0), abs(got - want) / max(1.0, abs(want)))


def _check_all(c, res, W, plan, highs_pairs, tag):
    """err == 0 and every check of every pair; prints the largest observed error of each check."""
    assert int(res['err'].item()) == 0, int(res['err'].item())
    worst, stats, p0 = {}, [], 0
    for b, P in enumerate(c['pl']):
        stats.append(_check_ot_pair(c, res, W, b, p0, b in highs_pairs, worst))
        p0 += P.shape[0]
    _check_coors(c, res, W, plan, worst)
    _check_totals(c, res, W, worst)
    big = [(P.shape[0], st, 64 * (P.shape[0] + M) + 1024) for P, st in zip(c['pl'], stats) if P.shape[0] >= 398]
    print(f'\n[{tag}] worst={worst} (n, augmentations + 1e-9 search rounds, max_aug) for n >= 398: {big}')


# cap = the batch's largest pocket picks the layout (cost matrix C / per-sink source lists in shared or global memory):
# <= 310 both shared, 311..370 C shared, 371..870 lists shared, 871..1024 both global.  Most pairs have n < cap.
LAYOUT_BATCHES = [[1, 49, 310, 50, 51], [51, 311, 1, 310], [50, 370, 49, 311], [1, 371, 49, 370],
                  [51, 870, 371, 1], [871, 50, 870], [49, 1024, 871, 1]]


@pytest.mark.parametrize('sizes', LAYOUT_BATCHES, ids=lambda s: f'cap{max(s)}')
def test_ot_solver_layouts_vs_fp64(sizes, cuda_device):
    c = _case(np.random.default_rng(max(sizes)), sizes)
    plan, res = _run(c, WEIGHTS, cuda_device)
    _check_all(c, res, WEIGHTS, plan, highs_pairs={0, 1}, tag=f'layout cap={max(sizes)}')


TIE_KINDS = ['one_keypoint', 'with_replacement', 'grid', 'far', 'same_pockets']


@pytest.mark.parametrize('kind', TIE_KINDS)
def test_ot_ties_and_degenerate_costs_vs_fp64(kind, cuda_device):
    """Tied costs (identical keypoints, repeated pocket points, integer grids, pocket_lig == pocket_rec) and |C| ~ 1e6
    at n = 48, 398, 1024: the plan is certified optimal and the device result is bitwise reproducible."""
    c = _case(np.random.default_rng(TIE_KINDS.index(kind) + 100), [48, 398, 1024], kind=kind)
    plan, res = _run(c, WEIGHTS, cuda_device)
    _check_all(c, res, WEIGHTS, plan, highs_pairs={0, 1}, tag=f'ties {kind}')
    _assert_bitwise_equal(res, _run(c, WEIGHTS, cuda_device)[1])


def _assert_bitwise_equal(r1, r2):
    for k in ('plan', 'parts', 'total', 'dcoors', 'dkeypts'):
        assert torch.equal(r1[k], r2[k]), k


@pytest.mark.parametrize('weights', [WEIGHTS, DEFAULTS], ids=['weights', 'defaults'])
def test_training_batch_shape_vs_fp64(weights, cuda_device):
    """64 pairs with the targets of bench_train.make_targets (pocket = midpoints of residue pairs drawn with replacement,
    the same array for both sides) and keypoints bunched together as at initialisation, in one call."""
    rng = np.random.default_rng(64)
    c = dict(sizes=[], pred=[], bl=[], br=[], pl=[], pr=[], kl=[], kr=[])
    for b in range(64):
        nl, nr = int(rng.integers(40, 300)), int(rng.integers(40, 300))
        pair = synthetic.synthetic_pair(rng, nl, nr, 1)
        t = bench_train.make_targets(pair, rng)
        c['sizes'].append((nl, nr))
        c['bl'].append(t['bound_lig'])
        c['br'].append(t['bound_rec'])
        c['pred'].append((t['bound_lig'] + rng.normal(0, 2, t['bound_lig'].shape)).astype(np.float32))
        c['pl'].append(t['pocket_lig'])
        c['pr'].append(t['pocket_rec'])
        c['kl'].append(t['bound_lig'].mean(0) + rng.normal(0, 0.5, (M, 3)))
        c['kr'].append(t['bound_rec'].mean(0) + rng.normal(0, 0.5, (M, 3)))
    plan, res = _run(c, weights, cuda_device)
    _check_all(c, res, weights, plan, highs_pairs={0, 1, 2}, tag=f'training shape w_ot={weights["w_ot"]}')
    _assert_bitwise_equal(res, _run(c, weights, cuda_device)[1])


def test_oversize_and_empty_pockets(cuda_device):
    """Pocket sizes [1025, 40, 0]: err bit 1 is set and check_loss_status raises; the 40-point pair is still exact; the
    oversize and the empty pair contribute ot = 0 and zero keypoint gradients; the totals are the means over all three
    pairs (built here: the LP oracle has no empty pocket)."""
    W = WEIGHTS
    c = _case(np.random.default_rng(1025), [1025, 40, 0])
    plan, res = _run(c, W, cuda_device)
    assert int(res['err'].item()) & 1
    with pytest.raises(nat.NativeLibraryError):
        check_loss_status(res)
    worst = {}
    _check_ot_pair(c, res, W, 1, 1025, True, worst)
    parts, dk = res['parts'].cpu().numpy(), res['dkeypts'].cpu().numpy()
    for b in (0, 2):
        assert parts[b, 1] == 0.0
        assert not dk[b].any() and not dk[3 + b].any()
    _check_coors(c, res, W, plan, worst)
    ot = [0.0, float((res['plan'][1025:1065].cpu().numpy() * _cost(c, 1)).sum()) / (M * 40), 0.0]
    mse = [float(((c['pred'][b].astype(np.float64) - c['bl'][b]) ** 2).mean()) for b in range(3)]
    inter = [lo.body_intersection_loss(c['pred'][b].astype(np.float64), c['br'][b].astype(np.float64), W['sigma'], W['ct'])
             for b in range(3)]
    want = [np.mean(mse) + W['w_ot'] * np.mean(ot) + W['w_int'] * np.mean(inter), np.mean(mse), np.mean(ot), np.mean(inter)]
    tot = res['total'].cpu().numpy()
    assert np.all(np.abs(tot - want) <= 1e-9 * np.maximum(1.0, np.abs(want))), (tot, want)


MSE_SIZES = [(1, 2000), (2000, 1), (129, 257), (700, 700)]


@pytest.mark.parametrize('geometry', ['all_active', 'none_active', 'straddle'])
def test_mse_intersection_ragged_sizes_vs_fp64(geometry, cuda_device):
    """N_lig / N_rec up to 2000 (the 128-thread loops run up to 16 times, with ragged tails) for overlapping bodies (every
    term active), bodies 500 A apart (none) and bodies straddling the ct - G = 0 kink."""
    W = WEIGHTS
    c = _case(np.random.default_rng(7), [7, 7, 7, 7], prot_sizes=MSE_SIZES, geometry=geometry)
    plan, res = _run(c, W, cuda_device)
    assert int(res['err'].item()) == 0
    worst = {}
    act, inact = _check_coors(c, res, W, plan, worst)
    if geometry == 'all_active':
        assert inact == 0
    elif geometry == 'none_active':
        assert act == 0
    else:
        assert min(act, inact) > 0.1 * (act + inact), (act, inact)
    _check_totals(c, res, W, worst)
    print(f'\n[mse {geometry}] worst={worst} active={act} inactive={inact}')
