"""GPU (H100): training with dropout > 0.  The CUDA forward and backward under the engine's masks against torch.autograd on
the fp64 batch restatement (tests/dropout_masks.py) under the same masks, recomputed on the host from the forward's seed.
A single mask bit that differs between the device and the host gives an O(1) error in the outputs or the gradients, so
these comparisons also pin the device masks to the numpy Philox.  Bounds are those of test_gpu_backward.py."""
import numpy as np
import pytest
import torch

import dropout_masks as dm
import golden_io as gio
from equidock_public_b200 import synthetic
from equidock_public_b200.engine import draw_dropout
from equidock_public_b200.hetero_graph import LIGAND, LL, RECEPTOR, RR

pytestmark = pytest.mark.gpu
P = 0.25
PAIR = {'db5': '1QA9', 'dips': 'kq_1kq1.pdb1_2.dill'}


def _args(ds, p=P):
    a = gio.load_args(ds)
    a['dropout'] = p
    return a


def _pairs(ds, kind):
    if kind == 'single':
        _, pairs, _, _ = gio.load_pairs(ds)
        return [pairs[PAIR[ds]]]
    rng = np.random.default_rng(9)
    return [synthetic.synthetic_pair(rng, a, b, 10) for a, b in [(40, 131), (129, 20), (64, 64)]]


def _oracle_inputs(graph, plan):
    nl, nr = graph.nodes[LIGAND].data, graph.nodes[RECEPTOR].data
    c = lambda a, b: torch.cat([a.detach().cpu(), b.detach().cpu()]).double()
    seg = np.concatenate([[0], np.cumsum(list(plan.n_lig_list) + list(plan.n_rec_list))]).tolist()
    return {'B': plan.n_pairs, 'seg': seg, 'src': plan.col_src.long().cpu(), 'dst': plan.edge_dst.long().cpu(),
            'res': c(nl['res_feat'], nr['res_feat']).reshape(-1).long(), 'mu_r_norm': c(nl['mu_r_norm'], nr['mu_r_norm']),
            'x': c(nl['new_x'], nr['x']),
            'he': torch.cat([plan.he_l[:plan.E_l].cpu(), plan.he_r[:plan.E_r].cpu()]).double()}


def _targets(pairs, seed=3):
    rng = np.random.default_rng(seed)
    return [{'c': rng.normal(0, 5, (len(l['res_feat']), 3)), 'yl': rng.normal(0, 10, (50, 3)),
             'yr': rng.normal(0, 10, (50, 3))} for l, r in pairs]


def _loss(coors, Y, tg, n_lig):
    """sum over pairs of |coors - c|^2 + |Y_l - yl|^2 + |Y_r - yr|^2 (coors concatenated, Y [2B][50][3] or lists)."""
    B, off, tot = len(tg), 0, 0.
    for b, t in enumerate(tg):
        dev = coors[b].device if isinstance(coors, list) else coors.device
        T = lambda a: torch.from_numpy(a).to(dev)
        cb = coors[b] if isinstance(coors, list) else coors[off:off + n_lig[b]]
        off += n_lig[b]
        tot = tot + ((cb.double() - T(t['c'])) ** 2).sum() + ((Y[0][b].double() - T(t['yl'])) ** 2).sum() \
            + ((Y[1][b].double() - T(t['yr'])) ** 2).sum()
    return tot


def _run_module(model, pairs, tg, dev, torch_seed):
    torch.manual_seed(torch_seed)
    g = gio.make_batch(pairs, dev)
    coors, kp_l, kp_r, rot, trans = model(g, epoch=0)
    model.zero_grad(set_to_none=True)
    loss = _loss(coors, (kp_l, kp_r), tg, [len(l['res_feat']) for l, _ in pairs])
    loss.backward()
    fwd = model.iegmn_original.last_outputs
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters()}
    return g, fwd, loss.detach(), torch.cat([c.detach() for c in coors]), grads


@pytest.mark.parametrize('ds', ['db5', 'dips'])
@pytest.mark.parametrize('kind', ['single', 'ragged3'])
def test_module_training_with_dropout_matches_fp64_autograd_under_the_same_masks(ds, kind, cuda_device):
    args = _args(ds)
    pairs, model = _pairs(ds, kind), gio.build_model(ds, cuda_device, args=args).train()
    tg = _targets(pairs)
    g, fwd, loss, coors, grads = _run_module(model, pairs, tg, cuda_device, 11)
    d0 = fwd['dropout_layers'][0].dropout
    assert d0.p == np.float32(P) and fwd['dropout_head'].layer == int(args['iegmn_n_lays'])
    plan = fwd['plan']
    inp = _oracle_inputs(g, plan)
    masks = dm.BatchMasks(P, d0.seed, 0, plan.N, plan.E, int(args['iegmn_n_lays']))
    leaves, sd = {}, {}     # one fp64 leaf per parameter tensor: the weight-shared DB5 layers 1..4 sum their gradients
    for k, v in model.state_dict(keep_vars=True).items():
        if v.data_ptr() not in leaves:
            leaves[v.data_ptr()] = torch.from_numpy(v.detach().cpu().double().numpy()).requires_grad_(True)
        sd[k] = leaves[v.data_ptr()]
    co_ref, Y, _, _ = dm.model_forward(sd, args, inp, masks)
    B = plan.n_pairs
    loss_ref = _loss(co_ref, (Y[:B], Y[B:]), tg, plan.n_lig_list)
    loss_ref.backward()
    cr = co_ref.detach().numpy()
    assert np.abs(coors.cpu().numpy() - cr).max() < 2e-3 * max(1.0, np.abs(cr).max() / 100)
    assert abs(loss.item() - loss_ref.item()) < 1e-3 * abs(loss_ref.item())
    # the masks matter: without them the fp64 restatement lands elsewhere
    co_nomask = dm.model_forward({k: v.detach() for k, v in sd.items()}, args, inp)[0].numpy()
    assert np.abs(co_nomask - cr).max() > 100 * 2e-3 * max(1.0, np.abs(cr).max() / 100)
    ref = {k: v.grad.numpy() for k, v in sd.items()}
    gmax = max(np.abs(v).max() for v in ref.values())
    bad = [(n, float(np.abs(grads[n].cpu().double().numpy() - ref[n]).max() / np.abs(ref[n]).max()))
           for n in grads if np.abs(grads[n].cpu().double().numpy() - ref[n]).max() > 3e-3 * np.abs(ref[n]).max() + 2e-6 * gmax]
    assert not bad, bad


def test_same_torch_seed_is_bitwise_reproducible_and_another_seed_is_not(cuda_device):
    args = _args('dips')
    pairs = _pairs('dips', 'ragged3')
    tg = _targets(pairs)
    model = gio.build_model('dips', cuda_device, args=args).train()
    _, f1, l1, c1, g1 = _run_module(model, pairs, tg, cuda_device, 5)
    _, f2, l2, c2, g2 = _run_module(model, pairs, tg, cuda_device, 5)
    _, f3, l3, c3, g3 = _run_module(model, pairs, tg, cuda_device, 6)
    seed = lambda f: f['dropout_layers'][0].dropout.seed
    assert seed(f1) == seed(f2) != seed(f3)
    assert torch.equal(l1, l2) and torch.equal(c1, c2)
    assert all(torch.equal(g1[n], g2[n]) for n in g1)
    assert not torch.equal(c1, c3) and not torch.equal(l1, l3)


def test_eval_mode_ignores_dropout(cuda_device):
    pairs = _pairs('db5', 'ragged3')
    outs = []
    for p in (P, 0.0):
        model = gio.build_model('db5', cuda_device, args=_args('db5', p)).eval()
        with torch.no_grad():
            coors, kp_l, _, rot, _ = model(gio.make_batch(pairs, cuda_device), epoch=0)
        outs.append(torch.cat(coors))
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize('ds', ['db5', 'dips'])
@pytest.mark.parametrize('li', [0, 1])
def test_layer_autograd_with_dropout_matches_fp64_autograd(ds, li, cuda_device):
    """One IEGMN_Layer call in training mode (its own seed, layer position 0) on a ragged batch: outputs and every
    parameter gradient against torch.autograd on the fp64 layer restatement under the same masks."""
    args = _args(ds)
    model = gio.build_model(ds, cuda_device, args=args).train()
    lay = model.iegmn_original.iegmn_layers[li]
    pairs = _pairs(ds, 'ragged3')
    g = gio.make_batch(pairs, cuda_device)
    nl, nr = g.nodes[LIGAND].data, g.nodes[RECEPTOR].data
    emb = model.iegmn_original.residue_emb_layer.weight.detach()
    h0 = [torch.cat([emb[d['res_feat'].reshape(-1).long()], torch.log(d['mu_r_norm'])], 1) for d in (nl, nr)]
    rng = np.random.default_rng(li)
    dh = 69 if li == 0 else 64
    h = h0 if li == 0 else [torch.from_numpy(rng.normal(0, 1, (t.shape[0], 64)).astype(np.float32)).to(cuda_device)
                            for t in h0]
    x = [nl['new_x'], nr['x']]
    he = [g.edges[LL].data['he'], g.edges[RR].data['he']]
    torch.manual_seed(21)
    seed = draw_dropout(P)[1]
    torch.manual_seed(21)
    xl, hl, xr, hr = lay(g, x[0], h[0], h0[0], he[0], x[0], x[1], h[1], h0[1], he[1], x[1])
    wx = torch.from_numpy(rng.normal(0, 1, (xl.shape[0] + xr.shape[0], 3))).to(cuda_device)
    wh = torch.from_numpy(rng.normal(0, 1, (hl.shape[0] + hr.shape[0], 64))).to(cuda_device)
    lay.zero_grad(set_to_none=True)
    ((torch.cat([xl, xr]).double() * wx).sum() + (torch.cat([hl, hr]).double() * wh).sum()).backward()
    plan = g._eqd_plan
    inp = _oracle_inputs(g, plan)
    masks = dm.BatchMasks(P, seed, 0, plan.N, plan.E, 1)
    p = {k: torch.from_numpy(v.detach().cpu().double().numpy()).requires_grad_(True) for k, v in lay.state_dict().items()}
    cpu = lambda a, b: torch.cat([a.detach().cpu(), b.detach().cpu()]).double()
    x_ref, h_ref = dm.layer_forward(p, inp['x'], cpu(h[0], h[1]), inp['x'], cpu(h0[0], h0[1]), inp['src'], inp['dst'],
                                    inp['he'], inp['seg'], plan.n_pairs, float(args['leakyrelu_neg_slope']),
                                    float(args['skip_weight_h']), float(args['x_connection_init']), masks, 0)
    ((x_ref * wx.cpu()).sum() + (h_ref * wh.cpu()).sum()).backward()
    xg, hg = torch.cat([xl, xr]).detach().cpu().double(), torch.cat([hl, hr]).detach().cpu().double()
    assert (xg - x_ref.detach()).abs().max() < 2e-3 * max(1.0, x_ref.abs().max().item() / 100)
    assert (hg - h_ref.detach()).abs().max() < 2e-3 * h_ref.abs().max().item()
    ref = {k: v.grad.numpy() for k, v in p.items()}
    gmax = max(np.abs(v).max() for v in ref.values())
    got = {n: q.grad.detach().cpu().double().numpy() for n, q in lay.named_parameters()}
    bad = [(n, float(np.abs(got[n] - ref[n]).max() / np.abs(ref[n]).max())) for n in got
           if np.abs(got[n] - ref[n]).max() > 3e-3 * np.abs(ref[n]).max() + 2e-6 * gmax]
    assert not bad, bad
    assert dh == p['att_mlp_Q.0.weight'].shape[0]


@pytest.mark.parametrize('ds', ['db5', 'dips'])
def test_input_tensor_gradients_with_dropout_match_fp64_autograd(ds, cuda_device):
    """.grad of the graph's new_x / x, mu_r_norm and he after loss.backward() under dropout (ragged batch of 3)."""
    from equidock_public_b200.rigid_docking_model import graph_inputs
    args = _args(ds)
    pairs, model = _pairs(ds, 'ragged3'), gio.build_model(ds, cuda_device, args=args).train()
    tg = _targets(pairs, 4)
    torch.manual_seed(13)
    g = gio.make_batch(pairs, cuda_device)
    ins = graph_inputs(g)
    for t in ins:
        t.requires_grad_(True)
    coors, kp_l, kp_r, _, _ = model(g, epoch=0)
    _loss(coors, (kp_l, kp_r), tg, [len(l['res_feat']) for l, _ in pairs]).backward()
    fwd = model.iegmn_original.last_outputs
    plan = fwd['plan']
    assert plan.edge_perm is None
    inp = _oracle_inputs(g, plan)
    for k in ('x', 'mu_r_norm', 'he'):
        inp[k] = inp[k].detach().requires_grad_(True)
    sd = {k: torch.from_numpy(v.detach().cpu().double().numpy()) for k, v in model.state_dict().items()}
    masks = dm.BatchMasks(P, fwd['dropout_layers'][0].dropout.seed, 0, plan.N, plan.E, int(args['iegmn_n_lays']))
    co_ref, Y, _, _ = dm.model_forward(sd, args, inp, masks)
    B = plan.n_pairs
    _loss(co_ref, (Y[:B], Y[B:]), tg, plan.n_lig_list).backward()
    got = {'x': torch.cat([ins[0].grad, ins[1].grad]), 'mu_r_norm': torch.cat([ins[2].grad, ins[3].grad]),
           'he': torch.cat([ins[4].grad, ins[5].grad])}
    for k, v in got.items():
        ref = inp[k].grad.numpy()
        err = np.abs(v.detach().cpu().double().numpy() - ref).max()
        assert err <= 3e-3 * np.abs(ref).max(), (k, err / np.abs(ref).max())


def test_fused_trainer_step_with_dropout_matches_the_module_path(cuda_device):
    """DataParallelTrainer.step under dropout against model.train(); outputs -> the same device losses through autograd
    -> loss.backward(), from the same parameters and with the same torch seed (so the same masks: the trainer's rank is
    0), for two seeds: the same loss, and the trainer's flat gradient (clip norm out of reach, so unscaled) equal to every
    param.grad within the bounds of test_gpu_backward.py."""
    from equidock_public_b200.losses import PocketBatch, device_losses
    from equidock_public_b200.training import DataParallelTrainer
    rng = np.random.default_rng(12)
    pairs = [synthetic.synthetic_pair(rng, a, b, 10) for a, b in [(60, 75), (90, 50)]]
    g = gio.make_batch(pairs, cuda_device)
    bl = [torch.from_numpy(p[0]['x']) for p in pairs]
    br = [torch.from_numpy(p[1]['x'] + 8.0) for p in pairs]
    pk = [torch.from_numpy((0.5 * (p[0]['x'][:9] + p[1]['x'][:9] + 8.0)).astype(np.float32)) for p in pairs]
    tgt = PocketBatch(bl, br, pk, pk, cuda_device)
    seeds = []
    for step in range(2):
        m1 = gio.build_model('db5', cuda_device, args=_args('db5')).train()
        m2 = gio.build_model('db5', cuda_device, args=_args('db5')).train()
        tr = DataParallelTrainer(m1, lr=1e-3, weight_decay=1e-4, clip=1e30)   # no clipping: flat_g stays unscaled
        assert tr.engine.rank == 0
        torch.manual_seed(100 + step)
        r1 = tr.step(g, tgt)
        seeds.append(r1['fwd']['dropout_layers'][0].dropout.seed)
        assert float(r1['grad_norm'][0]) < 1e30
        torch.manual_seed(100 + step)
        coors, kl, kr, _, _ = m2(g, epoch=0)
        assert m2.iegmn_original.last_outputs['dropout_layers'][0].dropout.seed == seeds[-1]
        plan = m2.iegmn_original.last_outputs['plan']
        kp = torch.cat([torch.stack(kl), torch.stack(kr)]).double()
        res = device_losses(plan, torch.cat(coors), kp, tgt, 1.0, 10.0, 25.0, 10.0)
        ((torch.cat(coors) * res['dcoors']).sum() + (kp * res['dkeypts']).sum()).backward()
        assert abs(float(r1['loss'][0]) - float(res['total'][0])) < 1e-6 * max(1.0, abs(float(res['total'][0])))
        by_param = {id(p): v for p, v in zip(tr.layout.params, tr.layout.views(tr.flat_g))}
        flat = {n: by_param[id(p)] for n, p in m1.named_parameters()}
        ref = {n: p.grad.detach().double().cpu().numpy() for n, p in m2.named_parameters()}
        gmax = max(np.abs(v).max() for v in ref.values())
        bad = [n for n in ref if np.abs(flat[n].double().cpu().numpy() - ref[n]).max() > 3e-3 * np.abs(ref[n]).max() + 2e-6 * gmax]
        assert not bad, bad
    assert seeds[0] != seeds[1]


def test_graph_capture_refuses_training_mode_dropout(cuda_device):
    """A captured graph would replay one seed's masks: capture refuses a training-mode model with dropout > 0, capture
    in eval() works, and switching the model to train() makes launch() re-capture and so refuse."""
    pairs = _pairs('db5', 'ragged3')
    model = gio.build_model('db5', cuda_device, args=_args('db5')).train()
    g = gio.make_batch(pairs, cuda_device)
    with pytest.raises(NotImplementedError, match='dropout'):
        model.graphed(g)
    model.eval()
    gf = model.graphed(g)
    with torch.no_grad():
        ref = torch.cat(model(g, epoch=0)[0])
    assert torch.equal(torch.cat(gf.launch().result()[0]), ref)
    model.train()
    with pytest.raises(NotImplementedError, match='dropout'):
        gf.launch()
