"""GPU (H100): the reference's SVD degeneracy guard (rigid_docking_model.py:570-586) in the forward and the CUDA backward.
When the keypoint covariance A has a singular value below 1e-3 or two squared singular values closer than 1e-2, the
reference adds diag(torch.rand(3, 3)) from the CPU generator until the test passes: the engine flags the pair on the
device (kabsch_apply_kernel), IEGMNEngine.resolve_status adds the noise to the forward's ``cov`` and re-solves, and
eqd_bwd_head differentiates through that perturbed ``cov``.  The guard fires on every pair of a model at random
initialisation (its keypoints sit near their centroid) and of every model with K <= 3 keypoints (the centred keypoints
have rank <= K - 1).

Everything is compared with torch.autograd on the fp64 restatement of tests/heads_ref.py, whose guard loop replays the
engine's CPU-generator draws (heads_ref.replay_draws).  Every case asserts the same draws per pair on both sides and the
same CPU-generator state after them, and prints the draws, the smallest squared-singular-value gap of the perturbed
covariances and the worst relative error per tensor group."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

import dropout_masks as dm
import golden_io as gio
import heads_ref as hr
from equidock_public_b200 import _native as nat
from equidock_public_b200 import hetero_graph as hg
from equidock_public_b200 import synthetic
from equidock_public_b200.engine import GraphPlan
from equidock_public_b200.losses import PocketBatch, device_losses
from equidock_public_b200.rigid_docking_model import Rigid_Body_Docking_Net, graph_inputs
from test_gpu_dropout import _loss, _oracle_inputs
from test_gpu_dropout import _pairs as _model_pairs
from test_gpu_heads import _coord_bound, _guard_loop, _pairs, _rel, _targets, _twice
from test_gpu_layer_norm_options import _fp64_state, _grad_mismatches

pytestmark = pytest.mark.gpu
F64 = torch.float64
DEG = nat.STATUS_SVD_DEGENERATE


def _min_gap(covs):
    """Smallest |s_i^2 - s_j^2| over the pairs' 3x3 covariances (fp64)."""
    s2 = torch.linalg.svdvals(torch.as_tensor(covs).detach().cpu().double().reshape(-1, 3, 3)) ** 2
    return float(torch.stack([(s2[:, 0] - s2[:, 1]).abs(), (s2[:, 1] - s2[:, 2]).abs()]).min())


# ---- head kernels -----------------------------------------------------------------------------------------------------

HEAD_CASES = ([(K, kind, 0.0, False) for K in (1, 2, 3, 4, 50) for kind in ('single', 'ragged3', 'sizes')]
              + [(K, 'ragged3', 0.25, False) for K in (1, 2, 3, 4, 50)]
              + [(K, 'ragged3', 0.0, True) for K in (4, 50)]
              + [(K, 'bulk', 0.25, False) for K in (25, 50, 64)])


def _head_batch(kind, dev):
    """(graph, plan) of a head case: test_gpu_heads' pairs, or test_gpu_backward_kernels' bulk batch (109 pairs,
    41 510 nodes, 422 node tiles)."""
    if kind == 'bulk':
        from test_gpu_backward_kernels import _batch
        return _batch('bulk', dev)
    g = gio.make_batch(_pairs(kind), dev)
    return g, GraphPlan.from_graph(g, dev, 10)


@pytest.mark.parametrize('K,kind,p,small', HEAD_CASES)
def test_head_kernels_through_the_perturbed_covariance_vs_fp64(K, kind, p, small, cuda_device):
    """eqd_keypoints, eqd_kabsch_apply + the engine's host loop, then eqd_bwd_head (eqd_bwd_head_dropout for p > 0) on the
    perturbed ``cov``, each run twice (bitwise equal), against torch.autograd of the fp64 tail (heads_ref.keypoint_tail)
    evaluated from the kernels' own h / x and at the kernels' own fp32 segment means of the head's activations, at the
    1e-5 of tests/test_gpu_backward_kernels.py.  Because the tail takes those means' values from the kernel, an error in
    them would not show here: the means themselves are checked against fp64 by test_gpu_heads.py's forward-kernel test
    (qbar), and their gradient path (dpre) here.  Trained weights (the shipped checkpoint with seeded K-head key / query
    projections), and ``small``: key / query weights scaled by 1e-3, so that the keypoints collapse onto their centroid as
    at initialisation and the guard fires on every pair.  `bulk` (p = 0.25, K = 25, 50, 64): the dropout backward over
    109 pairs, its site-3 mask replayed on 41 510 nodes, after a re-run of the forward's mean kernel (422 node tiles on
    264 CTAs: 158 of them walk a second tile).

    K = 2 and 3 with trained weights are tested here, at the head level, only: after the noise the perturbed A has one
    large singular value next to two of size ~1 (e.g. S = (7.1e3, 0.68, 0.57)), so the rotation about the two small axes
    is set by the noise and moves by about S_max * delta / S_min under a change delta of the keypoints.  Evaluated from the
    kernels' own h / x / means the fp64 tail sees delta at fp64 level; a whole-model comparison would see the fp32-level
    delta of the layers, amplified by ~1e4."""
    dev, lib = cuda_device, nat.load()
    g, plan = _head_batch(kind, dev)
    if kind == 'bulk':      # the mean kernel that eqd_bwd_head_dropout re-runs (grid 264) walks a second tile
        assert plan.n_node_tiles > 264 and plan.n_pairs > 100
    model = hr.build_model('dips', dev, K, seed=K)
    net = model.iegmn_original
    if small:
        with torch.no_grad():
            net.att_mlp_key_ROT[0].weight.mul_(1e-3)
            net.att_mlp_query_ROT[0].weight.mul_(1e-3)
    head = net.packed_head(dev)
    B, N, NL = plan.n_pairs, plan.N, plan.N_l
    gen = torch.Generator(device=dev).manual_seed(300 + K)
    h = torch.randn(N, 64, generator=gen, device=dev) * 0.7
    x = (torch.randn(N, 3, generator=gen, device=dev, dtype=F64) * 8.0).contiguous()
    xl = x[:NL].float().contiguous()
    dcoors = (torch.randn(NL, 3, generator=gen, device=dev) * 0.05).contiguous()
    dkp = (torch.randn(2 * B, K, 3, generator=gen, device=dev) * 0.05).double().contiguous()
    ws_bytes = int(lib.eqd_workspace_bytes_k(N, plan.n_node_tiles, B, K))
    bws_bytes = int(lib.eqd_bwd_head_workspace_bytes_k(N, plan.n_node_tiles, B, K))
    a256 = lambda v: (v + 255) // 256 * 256
    q_off = a256(max(plan.n_node_tiles, 1) * 256) + a256((2 * B + 1) * 4)
    layer, dseed = 5, 0x1234_5678_9ABC_DEF0 + K
    dr = nat.dropout_descriptor(p, dseed, layer) if p > 0 else None
    seed = 4000 + K
    gs = C.byref(plan.struct)

    def run():
        ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device=dev)
        kp = torch.full((2 * B, K, 3), float('nan'), dtype=F64, device=dev)
        ym = torch.full((2 * B, 3), float('nan'), dtype=F64, device=dev)
        cov = torch.full((B, 9), float('nan'), dtype=F64, device=dev)
        nat.check(lib.eqd_keypoints_dropout(gs, C.byref(head.struct), C.byref(dr) if dr is not None else None,
                                            nat.ptr(h), nat.ptr(x), nat.ptr(ws), ws_bytes, nat.ptr(kp), nat.ptr(ym),
                                            nat.ptr(cov), None), 'eqd_keypoints_dropout')
        qbar = ws[q_off:q_off + 2 * B * 512].view(F64).view(2 * B, 64).clone()
        rot, trans = torch.full((B, 9), float('nan'), device=dev), torch.full((B, 3), float('nan'), device=dev)
        lig = torch.full((NL, 3), float('nan'), device=dev)
        sing = torch.full((B, 3), float('nan'), dtype=F64, device=dev)
        status = torch.zeros(B, dtype=torch.int32, device=dev)
        kab = lambda mask: nat.check(lib.eqd_kabsch_apply(gs, nat.ptr(cov), nat.ptr(ym), nat.ptr(xl), nat.ptr(mask),
                                                          nat.ptr(rot), nat.ptr(trans), nat.ptr(lig), nat.ptr(sing),
                                                          nat.ptr(status), None), 'eqd_kabsch_apply')
        kab(None)
        flagged = status.clone()
        draws = torch.tensor(_guard_loop(dev, plan, cov, status, kab, seed))
        state = torch.get_rng_state()
        bws = torch.full((bws_bytes,), 0xFF, dtype=torch.uint8, device=dev)
        dh = torch.full((N, 64), float('nan'), device=dev)
        dx = torch.full((N, 3), float('nan'), dtype=F64, device=dev)
        dpre = torch.full((N, 64), float('nan'), device=dev)
        gk, gq = torch.zeros(K * 64, 64, device=dev), torch.zeros(K * 64, 64, device=dev)
        nat.check(lib.eqd_bwd_head_dropout(gs, C.byref(head.struct), C.byref(dr) if dr is not None else None,
                                           nat.ptr(h), nat.ptr(x), nat.ptr(cov), nat.ptr(xl), nat.ptr(dcoors),
                                           nat.ptr(dkp), None, None, nat.ptr(bws), bws_bytes, nat.ptr(dh), nat.ptr(dx),
                                           nat.ptr(dpre), nat.ptr(gk), nat.ptr(gq), None), 'eqd_bwd_head_dropout')
        return rot, trans, lig, kp, cov, qbar, flagged, status, draws, state, dh, dx, dpre, gk, gq

    rot, trans, lig, kp, cov, qbar, flagged, status, draws, state, dh, dx, dpre, gk, gq = _twice(run)
    assert not bool((status & DEG).any())
    # the fp64 tail from the kernels' own h / x / means, its guard replaying the same draws
    sd = _fp64_state(model, requires_grad=True)
    h64 = h.double().cpu().requires_grad_(True)
    x64 = x.cpu().requires_grad_(True)
    seg = [int(v) for v in plan.seg_ptr_host]
    mask3 = dm.mask(dseed, 0, layer, 3, N, 64, p) if p > 0 else None
    _, rand_diag = hr.replay_draws(seed)
    trace = {}
    co, Y, R, t, draws_ref = hr.keypoint_tail(sd, h64, x64, xl.double().cpu(), seg, B, K, float(net.leakyrelu_neg_slope),
                                               mask3, rand_diag, qbar_value=qbar.cpu(), trace=trace)
    assert torch.equal(torch.get_rng_state(), state)
    assert draws.tolist() == draws_ref, (draws.tolist(), draws_ref)
    assert [bool(v) for v in (flagged & DEG).tolist()] == [n > 0 for n in draws_ref]
    if K <= 3 or small:
        assert all(n > 0 for n in draws_ref), draws_ref
    ((co * dcoors.double().cpu()).sum() + (Y * dkp.cpu()).sum()).backward()
    wk, wq = sd['iegmn_original.att_mlp_key_ROT.0.weight'], sd['iegmn_original.att_mlp_query_ROT.0.weight']
    errs = {'cov': _rel(cov, trace['A'].reshape(B, 9)), 'keypts': _rel(kp, Y.detach()),
            'pose': max(_rel(rot, R.detach().reshape(B, 9)), _rel(trans, t.detach()), _rel(lig, co.detach())),
            'dh': _rel(dh, h64.grad), 'dx': _rel(dx, x64.grad), 'dpre': _rel(dpre, trace['pre'].grad),
            'dW_key/query': max(_rel(gk, wk.grad), _rel(gq, wq.grad))}
    print(f'\nguard head K={K} {kind} p={p}{" small" if small else ""}: draws {draws.tolist()} (fp64 {draws_ref}), '
          f'min gap {_min_gap(cov):.3e}, ' + ', '.join(f'{k} {e:.1e}' for k, e in errs.items()))
    assert all(e <= 1e-5 for e in errs.values()), errs


# ---- whole models at random initialisation ----------------------------------------------------------------------------

def _random_model(ds, K, dev, p=0.0, init_seed=0):
    """Rigid_Body_Docking_Net(args) with torch's default initialisation from torch.manual_seed(init_seed)."""
    args = hr.args_with(ds, K, dropout=p)
    torch.manual_seed(init_seed)
    return Rigid_Body_Docking_Net(dict(args, device=dev)).to(dev).train(), args


def _module_step(model, pairs, tg, dev, seed):
    """loss.backward() through the module from torch.manual_seed(seed), the graph's input tensors requiring grad."""
    torch.manual_seed(seed)
    g = gio.make_batch(pairs, dev)
    ins = graph_inputs(g)
    for t in ins:
        t.requires_grad_(True)
    coors, kp_l, kp_r, _, _ = model(g, epoch=0)
    state = torch.get_rng_state()
    model.zero_grad(set_to_none=True)
    loss = _loss(coors, (kp_l, kp_r), tg, [len(l['res_feat']) for l, _ in pairs])
    loss.backward()
    fwd = model.iegmn_original.last_outputs
    return {'g': g, 'fwd': fwd, 'loss': loss.detach(), 'coors': torch.cat([c.detach() for c in coors]), 'state': state,
            'grads': {n: q.grad.detach().clone() for n, q in model.named_parameters()},
            'ins': {'x': torch.cat([ins[0].grad, ins[1].grad]), 'mu_r_norm': torch.cat([ins[2].grad, ins[3].grad]),
                    'he': torch.cat([ins[4].grad, ins[5].grad])}}


KINK_BAND = 1e-5


def _ref_step(model, args, r, tg, seed, p, kink=None):
    """The same step on the fp64 restatement, its dropout seed and guard noise replayed from torch.manual_seed(seed).
    ``kink`` = True / False: LeakyReLU inputs within KINK_BAND of the kink take the derivative of the positive / negative
    side (heads_ref.kink_branch)."""
    fwd, plan = r['fwd'], r['fwd']['plan']
    assert plan.edge_perm is None
    inp = _oracle_inputs(r['g'], plan)
    for k in ('x', 'mu_r_norm', 'he'):
        inp[k] = inp[k].detach().requires_grad_(True)
    sd = _fp64_state(model, requires_grad=True)
    dropout, rand_diag = hr.replay_draws(seed, p)
    masks = None
    if dropout is not None:
        assert dropout[1] == fwd['dropout_layers'][0].dropout.seed
        masks = dm.BatchMasks(p, dropout[1], 0, plan.N, plan.E, int(args['iegmn_n_lays']))
    with hr.kink_branch(KINK_BAND, kink) if kink is not None else contextlib.nullcontext():
        co, Y, _, _, draws = hr.model_forward(sd, args, inp, masks, rand_diag)
        state = torch.get_rng_state()
        B = plan.n_pairs
        loss = _loss(co, (Y[:B], Y[B:]), tg, plan.n_lig_list)
        loss.backward()
    return {'coors': co.detach().numpy(), 'loss': loss.item(), 'draws': draws, 'state': state,
            'grads': {k: v.grad.numpy() for k, v in sd.items()},
            'ins': {k: inp[k].grad.numpy() for k in ('x', 'mu_r_norm', 'he')}}


def _check_step(tag, r, ref, sides=None):
    """The module step r against the fp64 step ref at the bounds of tests/test_gpu_dropout.py /
    tests/test_gpu_input_grads.py: 2e-3 max(1, |x|/100) on coordinates, 3e-3 max|ref| + 2e-6 max|all gradients| on
    parameter gradients, 3e-3 max|ref| on input gradients.  ``sides`` = the fp64 steps with the LeakyReLU inputs near
    the kink on the positive / the negative side (_ref_step(kink=...)): each gradient bound grows by what that choice
    alone changes, max|g_positive - g_negative|.  The printout gives the draws, the smallest gap, every group's error as a
    fraction of its bound and the gradients whose bound the kink term dominates, with its size."""
    draws = r['fwd']['guard_draws']
    assert draws == ref['draws'], (draws, ref['draws'])
    assert torch.equal(r['state'], ref['state'])
    cr = ref['coors']
    err = {'coors': float(np.abs(r['coors'].cpu().double().numpy() - cr).max()) / _coord_bound(cr),
           'loss': abs(r['loss'].item() - ref['loss']) / (1e-3 * abs(ref['loss']))}
    got = {**{n: q.cpu().double().numpy() for n, q in r['grads'].items()},
           **{'d' + k: v.detach().cpu().double().numpy() for k, v in r['ins'].items()}}
    rf = {**ref['grads'], **{'d' + k: v for k, v in ref['ins'].items()}}
    gmax = max(np.abs(v).max() for v in ref['grads'].values())
    base = {n: 3e-3 * np.abs(rf[n]).max() + (2e-6 * gmax if n in ref['grads'] else 0.0) for n in got}
    kink = {n: 0.0 for n in got}
    if sides is not None:
        hi, lo = ({**s['grads'], **{'d' + k: v for k, v in s['ins'].items()}} for s in sides)
        kink = {n: float(np.abs(hi[n] - lo[n]).max()) for n in got}
    frac = {n: float(np.abs(got[n] - rf[n]).max()) / (base[n] + kink[n]) for n in got}
    err['params'] = max(f for n, f in frac.items() if n in ref['grads'])
    err.update({n: f for n, f in frac.items() if n not in ref['grads']})
    widened = sorted((kink[n] / base[n], n.replace('iegmn_original.', '')) for n in got if kink[n] > base[n])
    print(f'\n{tag}: draws {draws} (fp64 {ref["draws"]}), min gap {_min_gap(r["fwd"]["cov"]):.3e}, '
          + ', '.join(f'{k} {e:.1e}' for k, e in err.items()) + ' (fractions of the bounds)'
          + (f'; the kink term exceeds the base bound for {len(widened)} of {len(got)} gradients, by up to '
             f'{widened[-1][0]:.1f}x ({widened[-1][1]})' if widened else ''))
    bad = {k: e for k, e in err.items() if not e <= 1}
    bad.update({n: f for n, f in frac.items() if not f <= 1})
    assert not bad, bad


def _head_gradients(model, args, r, tg, seed, p):
    """Localises a gradient error: the engine's gradient w.r.t. the last layer's h / x (eqd_bwd_head, captured by
    TrainEngine.backward for the step's own loss) against fp64 autograd of the keypoint head and guarded Kabsch
    (heads_ref.keypoint_tail) evaluated from the engine's own last-layer h / x.  Returns the relative errors."""
    from equidock_public_b200.training import TrainEngine
    eng = TrainEngine(model)
    torch.manual_seed(seed)
    fwd = eng.forward(r['g'])
    plan, B, L = fwd['plan'], fwd['plan'].n_pairs, int(args['iegmn_n_lays'])
    c = torch.from_numpy(np.concatenate([t['c'] for t in tg])).to(fwd['keypts'].device)
    y = torch.from_numpy(np.stack([t['yl'] for t in tg] + [t['yr'] for t in tg])).to(fwd['keypts'].device)
    cap = []
    eng.backward(fwd, 2 * (fwd['ligand_coors'].double() - c), 2 * (fwd['keypts'] - y), capture=cap)
    head = cap[0]
    sd = _fp64_state(model)
    h = fwd['h'].double().cpu().requires_grad_(True)
    x = fwd['x64'].cpu().requires_grad_(True)
    dropout, rand_diag = hr.replay_draws(seed, p)
    mask3 = dm.mask(dropout[1], 0, L, 3, plan.N, 64, p) if dropout is not None else None
    seg = [int(v) for v in plan.seg_ptr_host]
    co, Y, _, _, draws = hr.keypoint_tail(sd, h, x, fwd['x_lig_in'].detach().double().cpu(), seg, B, model.iegmn_original.num_att_heads,
                                          float(args['leakyrelu_neg_slope']), mask3, rand_diag)
    assert draws == fwd['guard_draws'], (draws, fwd['guard_draws'])
    _loss(co, (Y[:B], Y[B:]), tg, plan.n_lig_list).backward()
    return {'head dh': _rel(head['dh'], h.grad), 'head dx': _rel(head['dx'], x.grad)}


TRAIN_CASES = [(ds, K, p) for ds in ('db5', 'dips') for K in (1, 2, 3, 50) for p in (0.0, 0.25)]


@pytest.mark.parametrize('ds,K,p', TRAIN_CASES)
def test_training_from_random_initialisation_vs_fp64(ds, K, p, cuda_device):
    """The first training step of a run from scratch: torch.manual_seed, Rigid_Body_Docking_Net(args), a ragged batch of
    3 (40+131, 129+20, 64+64), DB5 (5 shared layers) and DIPS (8 layers), K = 1, 2, 3 and 50, dropout 0 and 0.25.  The
    guard fires on every pair (the keypoint attention is nearly uniform, A's singular values are 1e-2 .. 1e-5 before the
    noise).  The same seed is bitwise reproducible.  Two comparisons with fp64 autograd under the same draws (and masks):

      - the head alone: the engine's gradient w.r.t. the last layer's h / x against the fp64 head and guarded Kabsch from
        the engine's own h / x, at 1e-5 (_head_gradients).  This is what the guard's branch changes.
      - the whole step: loss, coordinates, every parameter gradient and the gradients of new_x / x, mu_r_norm and he.  At
        default initialisation many LeakyReLU inputs of the layers lie closer to the kink than the fp32 forward resolves
        (4e-9 .. 4e-7 of their row's max |input| in the fp64 restatement, in every one of these configurations); the
        engine may take the other side there, and the derivative differs by 0.99 x the upstream gradient.  So each
        gradient bound of tests/test_gpu_dropout.py is extended by max|g_positive - g_negative| of two fp64 evaluations
        that put every input within KINK_BAND = 1e-5 of its row's scale on one side or the other (_check_step)."""
    dev = cuda_device
    model, args = _random_model(ds, K, dev, p, init_seed=K)
    pairs = _model_pairs(ds, 'ragged3')
    tg = _targets(pairs, K)
    r = _module_step(model, pairs, tg, dev, 21)
    r2 = _module_step(model, pairs, tg, dev, 21)
    assert torch.equal(r['loss'], r2['loss']) and torch.equal(r['coors'], r2['coors'])
    assert all(torch.equal(r['grads'][n], r2['grads'][n]) for n in r['grads'])
    assert all(torch.equal(r['ins'][k], r2['ins'][k]) for k in r['ins'])
    assert r['fwd']['guard_draws'] == r2['fwd']['guard_draws'] and all(n > 0 for n in r['fwd']['guard_draws'])
    hd = _head_gradients(model, args, r, tg, 21, p)
    print(f'\ntrain {ds} K={K} p={p}: ' + ', '.join(f'{k} {e:.1e}' for k, e in hd.items()))
    assert all(e <= 1e-5 for e in hd.values()), hd
    _check_step(f'train {ds} K={K} p={p}', r, _ref_step(model, args, r, tg, 21, p),
                [_ref_step(model, args, r, tg, 21, p, kink) for kink in (True, False)])


@pytest.mark.parametrize('K', [1, 2, 3])
def test_trainer_step_at_few_keypoints_matches_the_module_path(K, cuda_device):
    """DataParallelTrainer.step (device exact-EMD / MSE / intersection losses and their backward with K keypoints) against
    the module path -> device_losses -> loss.backward(), from the same random initialisation and the same torch seed, so
    the same guard draws."""
    from equidock_public_b200.training import DataParallelTrainer
    dev = cuda_device
    rng = np.random.default_rng(12)
    pairs = [synthetic.synthetic_pair(rng, a, b, 10) for a, b in [(60, 75), (90, 50)]]
    g = gio.make_batch(pairs, dev)
    bl = [torch.from_numpy(q[0]['x']) for q in pairs]
    br = [torch.from_numpy(q[1]['x'] + 8.0) for q in pairs]
    pk = [torch.from_numpy((0.5 * (q[0]['x'][:9] + q[1]['x'][:9] + 8.0)).astype(np.float32)) for q in pairs]
    tgt = PocketBatch(bl, br, pk, pk, dev)
    m1, _ = _random_model('dips', K, dev, init_seed=40 + K)
    m2, _ = _random_model('dips', K, dev, init_seed=40 + K)
    tr = DataParallelTrainer(m1, lr=1e-3, weight_decay=1e-4, clip=1e30)
    torch.manual_seed(7)
    r1 = tr.step(g, tgt)
    s1 = torch.get_rng_state()
    torch.manual_seed(7)
    coors, kl, kr, _, _ = m2(g, epoch=0)
    assert torch.equal(torch.get_rng_state(), s1)
    d1, d2 = r1['fwd']['guard_draws'], m2.iegmn_original.last_outputs['guard_draws']
    assert d1 == d2 and all(n > 0 for n in d1), (d1, d2)
    plan = m2.iegmn_original.last_outputs['plan']
    kp = torch.cat([torch.stack(kl), torch.stack(kr)]).double()
    res = device_losses(plan, torch.cat(coors), kp, tgt, 1.0, 10.0, 25.0, 10.0)
    assert res['dkeypts'].shape == (4, K, 3) and res['plan'].shape == (18, K)
    ((torch.cat(coors) * res['dcoors']).sum() + (kp * res['dkeypts']).sum()).backward()
    assert abs(float(r1['loss'][0]) - float(res['total'][0])) < 1e-6 * max(1.0, abs(float(res['total'][0])))
    by_param = {id(q): v for q, v in zip(tr.layout.params, tr.layout.views(tr.flat_g))}
    flat = {n: by_param[id(q)].double().cpu().numpy() for n, q in m1.named_parameters()}
    ref = {n: q.grad.detach().double().cpu().numpy() for n, q in m2.named_parameters()}
    print(f'\ntrainer K={K}: draws {d1}, min gap {_min_gap(r1["fwd"]["cov"]):.3e}')
    bad = _grad_mismatches(flat, ref)
    assert not bad, bad


def _collapsed_mixed_pairs():
    """The first shipped DIPS test pair with all receptor residues at one point (A = 0: the guard fires) between two
    other shipped pairs."""
    names, pairs, _, _ = gio.load_pairs('dips')
    lig, rec = [dict(d) for d in pairs[names[0]]]
    rec['x'] = np.tile(rec['x'][:1], (rec['x'].shape[0], 1))
    return [pairs[names[1]], (lig, rec), pairs[names[2]]]


def test_mixed_batch_gradient_is_the_sum_of_the_per_pair_gradients(cuda_device):
    """Trained weights: the guard fires on the collapsed pair alone.  The batch step against fp64 under the same draws,
    and the batch's parameter gradient against the sum of the three one-pair steps, each from the same torch seed, so
    each with its own draws (only the collapsed pair draws)."""
    dev = cuda_device
    model = gio.build_model('dips', dev).train()
    args = gio.load_args('dips')
    pairs = _collapsed_mixed_pairs()
    tg = _targets(pairs, 50)
    r = _module_step(model, pairs, tg, dev, 31)
    draws = r['fwd']['guard_draws']
    assert draws[1] > 0 and draws[0] == draws[2] == 0, draws
    _check_step('mixed batch', r, _ref_step(model, args, r, tg, 31, 0.0))
    total, per_pair = None, []
    for b in range(3):
        rb = _module_step(model, [pairs[b]], [tg[b]], dev, 31)
        per_pair.append(rb['fwd']['guard_draws'][0])
        total = rb['grads'] if total is None else {n: total[n] + v for n, v in rb['grads'].items()}
    assert per_pair == draws
    bad = _grad_mismatches({n: v.cpu().double().numpy() for n, v in r['grads'].items()},
                           {n: v.cpu().double().numpy() for n, v in total.items()})
    assert not bad, bad


# ---- serving paths ----------------------------------------------------------------------------------------------------

def test_graph_replay_and_pipelined_serving_replay_the_eager_draws(cuda_device):
    """Eval mode at random initialisation (the guard fires on every pair): model.graphed(g).launch().result() and
    PipelinedInference (with and without CUDA graphs) return what the eager forward returns from the same generator state,
    and leave the generator where it leaves it.  Seeded after capture: a capture runs two eager forwards, which draw."""
    from equidock_public_b200.serving import PipelinedInference
    dev = cuda_device
    model, _ = _random_model('dips', 50, dev, init_seed=3)
    model.eval()
    pairs = _model_pairs('dips', 'ragged3')
    g = gio.make_batch(pairs, dev)

    def eager(batch, seed):
        torch.manual_seed(seed)
        with torch.no_grad():
            out = model(batch, epoch=0)
        assert all(n > 0 for n in model.iegmn_original.last_outputs['guard_draws'])
        return out, torch.get_rng_state()

    gf = model.graphed(g)
    ref, state = eager(g, 5)
    torch.manual_seed(5)
    res = gf.launch().result()
    assert torch.equal(torch.get_rng_state(), state)
    for a, b in zip(res, ref):
        assert all(torch.equal(x, y) for x, y in zip(a, b))
    hb = hg.batch_pairs(synthetic.to_torch_pairs(pairs)).pin_memory()
    for use_graph in (True, False):
        pipe = PipelinedInference(model, dev, use_cuda_graph=use_graph)
        if use_graph:
            for o in pipe.run(iter([hb])):      # the capture
                o['_event'].synchronize()
        torch.manual_seed(6)
        got = []
        for o in pipe.run(iter([hb])):
            o['_event'].synchronize()
            got.append((o['ligand_coors'].clone(), o['rotation'].clone()))
        st = torch.get_rng_state()
        ref, state = eager(hb.to(dev), 6)
        assert torch.equal(st, state)
        assert torch.equal(got[0][0], torch.cat(ref[0]).cpu()) and torch.equal(got[0][1], torch.stack(ref[3]).cpu())


# ---- the exit ---------------------------------------------------------------------------------------------------------

def test_guard_exits_after_the_reference_number_of_draws(cuda_device):
    """A covariance the guard can never pass (two singular values of 1e12: their fp32 squares coincide whatever the noise)
    in pair 1 of a batch: IEGMNEngine.resolve_status re-solves on the device after every draw and exits after the 11th,
    as the reference does, with the reference's message; the fp64 restatement exits after the same draws."""
    dev = cuda_device
    model = gio.build_model('dips', dev)
    g = gio.make_batch(_model_pairs('dips', 'ragged3'), dev)
    raw = model.iegmn_original.run_engine(g, check_status=False)
    raw['status_event'].synchronize()
    assert not bool(raw['status_host'][:3].any())
    crafted = torch.diag(torch.tensor([1e12, 1e12, 3.0], dtype=F64))
    raw['cov'][1] = crafted.reshape(9).to(dev)
    mask = torch.tensor([0, 1, 0], dtype=torch.int32, device=dev)
    raw['kabsch'](mask)                         # kabsch_apply flags the crafted pair on the device
    raw['status_host'][:3] = raw['status'][:3].cpu()
    assert raw['status_host'][:3].tolist() == [0, DEG, 0], (raw['status_host'].tolist(), raw['sing'][1].tolist())
    logged = []
    torch.manual_seed(8)
    with pytest.raises(SystemExit):
        raw['engine'].resolve_status(raw['plan'], raw, raw['kabsch'], logged.append)
    state = torch.get_rng_state()
    assert logged == [hr.GUARD_EXIT]
    assert raw['guard_draws'] == [0, 11, 0]
    torch.manual_seed(8)
    A = crafted.clone()
    for _ in range(11):
        A = A + torch.diag(torch.rand(3, 3).diagonal().double())
    assert torch.equal(torch.get_rng_state(), state)
    assert torch.equal(raw['cov'][1].cpu(), A.reshape(9))
    assert bool(raw['status'][1].item() & DEG)
    _, rand_diag = hr.replay_draws(8)
    with pytest.raises(SystemExit, match=hr.GUARD_EXIT.strip()):
        hr.guarded_kabsch(crafted.clone(), rand_diag)
    assert torch.equal(torch.get_rng_state(), state)
