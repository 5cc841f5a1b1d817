"""GPU (H100): autograd through the exported IEGMN_Layer and IEGMN modules, against torch.autograd on the fp64 TorchOracle.

IEGMN_Layer: one layer (the 69-wide layer 0 and a 64-wide layer of both checkpoints) on a single golden pair, a ragged
batch of 3 with the 128 + 1 / 128 + 3 node-tile boundaries, and that batch with its edges in random order; the shared DB5
layer called twice in a row; every layer of a checkpoint chained by hand.  The loss is a seeded random linear form of the
layer outputs (x_final, node_upd) of both proteins, and for the whole stack the quadratic side-output loss of
test_gpu_input_grads.py.  A tensor passes if max|got - ref| <= tol max|ref| + 2e-6 G, G the
largest reference magnitude of its group (coordinates, features, edge features, parameters): tol 2e-3 for the input
gradients and 3e-3 for the parameter gradients of one layer, 3e-3 for everything through a whole stack (the bounds of
test_gpu_backward.py).  x_connection_init is 0.3 so that the original coordinates get a gradient.

IEGMN: IEGMN.forward under train() is the same autograd node as Rigid_Body_Docking_Net.forward: bitwise equal gradients."""
import numpy as np
import pytest
import torch

import golden_io as gio
import iegmn_oracle_torch as ot
from equidock_public_b200 import _native as nat
from equidock_public_b200 import synthetic
from equidock_public_b200.hetero_graph import LL, RR
from equidock_public_b200.rigid_docking_model import graph_inputs

pytestmark = pytest.mark.gpu
PAIR = {'db5': '1QA9', 'dips': 'kq_1kq1.pdb1_2.dill'}
ETA = 0.3
WIDE = {'db5': 1, 'dips': 4}                  # the 64-wide layer tested per checkpoint
SIDE_KEYS = ('x', 'h', 'h0', 'he', 'x0')      # per-protein tensor order of IEGMN_Layer.forward
GROUP = {'x': 'x', 'x0': 'x', 'h': 'h', 'h0': 'h', 'he': 'he'}


def _np(t):
    return t.detach().double().cpu().numpy()


def _model(ds, dev):
    args = dict(gio.load_args(ds), x_connection_init=ETA)
    return gio.build_model(ds, dev, args=args), args


def _oracle(model, args):
    sd = {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}
    m = ot.TorchOracle(sd, args['iegmn_n_lays'], args['skip_weight_h'], args['x_connection_init'],
                       args['leakyrelu_neg_slope'], args['num_att_heads'], dtype=torch.float64)
    return m, m.parameters_for_grad()


def _pairs(ds, batch):
    if batch == 'single':
        _, pairs, _, _ = gio.load_pairs(ds)
        return [pairs[PAIR[ds]]]
    rng = np.random.default_rng(9)
    pairs = [synthetic.synthetic_pair(rng, a, b, 10) for a, b in [(40, 131), (129, 20), (64, 64)]]
    if batch == 'unsorted':          # every edge list in random order (not grouped by destination)
        shuffled = []
        for lig, rec in pairs:
            sides = []
            for d in (lig, rec):
                q = rng.permutation(d['dst'].shape[0])
                sides.append(dict(d, src=d['src'][q], dst=d['dst'][q], he=d['he'][q]))
            shuffled.append(tuple(sides))
        pairs = shuffled
    return pairs


def _layer_inputs(m, pairs, li):
    """Per pair, both proteins' fp64 tensors entering layer li of the oracle stack (x, h, h0, he, x0, src, dst)."""
    emb = m.sd['iegmn_original.residue_emb_layer.weight'].detach()
    out = []
    with torch.no_grad():
        for lig, rec in pairs:
            sides = []
            for s, ck in ((lig, 'new_x'), (rec, 'x')):
                idx = torch.as_tensor(s['res_feat']).reshape(-1).long()
                h0 = torch.cat([emb[idx], torch.log(torch.as_tensor(s['mu_r_norm']).double())], dim=1)
                x0 = torch.as_tensor(s[ck]).double()
                sides.append({'x': x0, 'x0': x0, 'h': h0, 'h0': h0, 'he': torch.as_tensor(s['he']).double(),
                              'src': torch.as_tensor(s['src']).long(), 'dst': torch.as_tensor(s['dst']).long()})
            for j in range(li):
                m._layer(j, sides)
            out.append(sides)
    return out


def _upstream(per_pair, seed, quad=False):
    """Seeded loss weights (a_x (n,3), a_h (n,64), t_x (n,3) or None) of both proteins of every pair (see _term)."""
    rng = np.random.default_rng(seed)
    out = []
    for sides in per_pair:
        ups = []
        for s in sides:
            n = s['x'].shape[0]
            if quad:
                ups.append((torch.from_numpy(rng.uniform(0, 1, (n, 3)) / n), torch.from_numpy(rng.uniform(0, 1, (n, 64)) / n),
                            s['x'] + torch.from_numpy(rng.normal(0, 1, (n, 3)))))
            else:
                ups.append((torch.from_numpy(rng.normal(0, 1, (n, 3))), torch.from_numpy(rng.normal(0, 1, (n, 64))), None))
        out.append(ups)
    return out


def _term(x, h, ax, ah, tx):
    """fp64 loss of one protein's layer outputs: sum a_x x + sum a_h h (random upstream gradients a_x, a_h), or with
    targets t_x the quadratic sum a_x (x - t_x)^2 + sum a_h h^2 (test_gpu_input_grads.py's side-output loss)."""
    x, h = x.double(), h.double()
    if tx is None:
        return (ax * x).sum() + (ah * h).sum()
    return (ax * (x - tx) ** 2).sum() + (ah * h ** 2).sum()


def _oracle_grads(m, psd, per_pair, layers, ups):
    """fp64 autograd of the _term losses of the outputs of the oracle layers `layers` (indices, in call order):
    (gradients of the ten inputs in engine order, {layer index: {param name: grad}})."""
    leaves, loss = [], 0.0
    for sides, up in zip(per_pair, ups):
        lv = [{k: s[k].detach().clone().requires_grad_(True) for k in SIDE_KEYS} for s in sides]
        run = [dict(v, src=s['src'], dst=s['dst']) for v, s in zip(lv, sides)]
        for li in layers:
            m._layer(li, run)
        for r, u in zip(run, up):
            loss = loss + _term(r['x'], r['h'], *u)
        leaves.append(lv)
    loss.backward()
    g = lambda v: v.grad.numpy() if v.grad is not None else np.zeros(tuple(v.shape))
    ref_in = [np.concatenate([g(lv[side][k]) for lv in leaves]) for side in (0, 1) for k in SIDE_KEYS]
    ref_p = {}
    for key, v in psd.items():
        if '.iegmn_layers.' in key and v.requires_grad:
            li, name = key.split('.iegmn_layers.')[1].split('.', 1)
            ref_p.setdefault(int(li), {})[name] = g(v)
    return ref_in, ref_p


def _engine_inputs(per_pair, g, dev):
    """The ten IEGMN_Layer.forward tensors in engine order (ligands of all pairs, then receptors), fp32 leaves; the edge
    features are the graph's own tensors."""
    ins = []
    for side, et in ((0, LL), (1, RR)):
        for k in SIDE_KEYS:
            if k == 'he':
                t = g.edges[et].data['he']
            else:
                t = torch.cat([pp[side][k] for pp in per_pair]).to(dev, torch.float32)
            ins.append(t.requires_grad_(True))
    return ins


def _engine_loss(outs, ups, dev):
    cat = lambda side, j: None if ups[0][side][j] is None else torch.cat([u[side][j] for u in ups]).to(dev)
    x_l, h_l, x_r, h_r = outs
    return _term(x_l, h_l, cat(0, 0), cat(0, 1), cat(0, 2)) + _term(x_r, h_r, cat(1, 0), cat(1, 1), cat(1, 2))


def _report(rows):
    """rows: (group, tag, got, ref, tol).  Prints every tensor's error; returns the lines out of bound."""
    G = {}
    for grp, _, _, ref, _ in rows:
        G[grp] = max(G.get(grp, 0.0), float(np.abs(ref).max()))
    bad = []
    for grp, tag, got, ref, tol in rows:
        err, rmax = float(np.abs(got - ref).max()), float(np.abs(ref).max())
        ok = err <= tol * rmax + 2e-6 * G[grp]
        line = f'{"ok  " if ok else "BAD "}{tag:44s} abs {err:.2e}  rel {err / max(rmax, 1e-30):.2e}  max|ref| {rmax:.3e}'
        print(line)
        if not ok:
            bad.append(line)
    return bad


def _input_rows(ins, ref_in, tol):
    tags = [f'd {k}_{"lig" if i < 5 else "rec"}' for i, k in enumerate(SIDE_KEYS * 2)]
    return [(GROUP[SIDE_KEYS[i % 5]], tags[i], _np(t.grad) if t.grad is not None else np.zeros(r.shape), r, tol)
            for i, (t, r) in enumerate(zip(ins, ref_in))]


def _param_rows(module, ref, tol, tag):
    return [('param', f'{tag}.{n}', _np(p.grad).reshape(ref[n].shape) if p.grad is not None else np.zeros(ref[n].shape),
             ref[n], tol) for n, p in module.named_parameters()]


@pytest.mark.parametrize('batch', ['single', 'ragged', 'unsorted'])
@pytest.mark.parametrize('which', ['layer0', 'wide'])
@pytest.mark.parametrize('ds', ['db5', 'dips'])
def test_one_layer_grads_vs_fp64_oracle(ds, which, batch, cuda_device):
    model, args = _model(ds, cuda_device)
    model.train()
    li = 0 if which == 'layer0' else WIDE[ds]
    lay = model.iegmn_original.iegmn_layers[li]
    pairs = _pairs(ds, batch)
    m, psd = _oracle(model, args)
    per_pair = _layer_inputs(m, pairs, li)
    ups = _upstream(per_pair, 31 + li)
    g = gio.make_batch(pairs, cuda_device)
    ins = _engine_inputs(per_pair, g, cuda_device)
    outs = lay(g, *ins)
    assert all(o.grad_fn is not None for o in outs)
    _engine_loss(outs, ups, cuda_device).backward()
    ref_in, ref_p = _oracle_grads(m, psd, per_pair, [li], ups)
    bad = _report(_input_rows(ins, ref_in, 2e-3) + _param_rows(lay, ref_p[li], 3e-3, f'layer{li}'))
    assert not bad, '\n'.join(bad)


def test_shared_layer_called_twice_accumulates(cuda_device):
    """The DB5 shared layer applied twice in a row: .grad holds the sum of both calls' parameter gradients."""
    model, args = _model('db5', cuda_device)
    model.train()
    lay = model.iegmn_original.iegmn_layers[1]
    pairs = _pairs('db5', 'ragged')
    m, psd = _oracle(model, args)
    per_pair = _layer_inputs(m, pairs, 1)
    ups = _upstream(per_pair, 41)
    g = gio.make_batch(pairs, cuda_device)
    ins = _engine_inputs(per_pair, g, cuda_device)
    x_l, h_l, x_r, h_r = lay(g, *ins)
    outs = lay(g, x_l, h_l, ins[2], ins[3], ins[4], x_r, h_r, ins[7], ins[8], ins[9])
    _engine_loss(outs, ups, cuda_device).backward()
    ref_in, ref_p = _oracle_grads(m, psd, per_pair, [1, 1], ups)
    bad = _report(_input_rows(ins, ref_in, 3e-3) + _param_rows(lay, ref_p[1], 3e-3, 'layer1 x2'))
    assert not bad, '\n'.join(bad)


@pytest.mark.parametrize('ds', ['db5', 'dips'])
def test_layer_stack_by_hand_vs_fp64_oracle(ds, cuda_device):
    """Every IEGMN_Layer of a checkpoint chained by hand from (x0, h0), the quadratic loss of _term on the last layer's
    outputs.  The edge features enter as a product with 1 (not the graph's tensors: each call builds its own plan)."""
    model, args = _model(ds, cuda_device)
    model.train()
    layers = model.iegmn_original.iegmn_layers
    L = len(layers)
    pairs = _pairs(ds, 'ragged')
    m, psd = _oracle(model, args)
    per_pair = _layer_inputs(m, pairs, 0)
    ups = _upstream(per_pair, 51, quad=True)
    g = gio.make_batch(pairs, cuda_device)
    ins = _engine_inputs(per_pair, g, cuda_device)
    xo_l, h0_l, he_l, xo_r, h0_r, he_r = ins[4], ins[2], ins[3] * 1.0, ins[9], ins[7], ins[8] * 1.0
    x_l, h_l, x_r, h_r = ins[0], ins[1], ins[5], ins[6]
    for lay in layers:
        x_l, h_l, x_r, h_r = lay(g, x_l, h_l, h0_l, he_l, xo_l, x_r, h_r, h0_r, he_r, xo_r)
    _engine_loss((x_l, h_l, x_r, h_r), ups, cuda_device).backward()
    ref_in, ref_p = _oracle_grads(m, psd, per_pair, list(range(L)), ups)
    rows = _input_rows(ins, ref_in, 3e-3)
    seen = set()
    for li, lay in enumerate(layers):
        if id(lay) in seen:
            continue
        seen.add(id(lay))
        uses = [j for j in range(L) if layers[j] is lay]        # a shared module's gradient sums over its uses
        ref = {n: sum(ref_p[j][n] for j in uses) for n in ref_p[li]}
        rows += _param_rows(lay, ref, 3e-3, f'layer{li}')
    bad = _report(rows)
    assert not bad, '\n'.join(bad)


def test_layer_autograd_outputs_bitwise_and_idle_input_kernels(cuda_device, monkeypatch):
    """eval() with one input requiring grad takes the autograd node: its outputs are bitwise those of the torch.no_grad()
    inference path.  With neither the edge features nor the original coordinates requiring grad, eqd_bwd_layer_inputs is
    not launched."""
    lib = nat.load()
    calls = {'n': 0}
    fn = lib.eqd_bwd_layer_inputs

    def counted(*a):
        calls['n'] += 1
        return fn(*a)
    monkeypatch.setattr(lib, 'eqd_bwd_layer_inputs', counted)
    model, args = _model('dips', cuda_device)
    model.eval()
    pairs = _pairs('dips', 'ragged')
    m, _ = _oracle(model, args)
    for li in (0, 1):
        lay = model.iegmn_original.iegmn_layers[li]
        per_pair = _layer_inputs(m, pairs, li)
        g = gio.make_batch(pairs, cuda_device)
        ins = [t.detach() for t in _engine_inputs(per_pair, g, cuda_device)]
        with torch.no_grad():
            ref = lay(g, *ins)
        ins[1].requires_grad_(True)
        outs = lay(g, *ins)
        assert outs[1].grad_fn is not None
        for a, b in zip(outs, ref):
            assert a.dtype == b.dtype and torch.equal(a.detach(), b)
        outs[1].sum().backward()
        assert ins[1].grad is not None and bool(ins[1].grad.abs().sum() > 0)
        assert all(p.grad is not None for p in lay.parameters())
    assert calls['n'] == 0


def _kabsch_loss(rot, trans, kp_l, kp_r, seed):
    rng = np.random.default_rng(seed)
    loss = 0.0
    for r, t, yl, yr in zip(rot, trans, kp_l, kp_r):
        w = lambda a: torch.from_numpy(rng.normal(0, 1, tuple(a.shape))).to(a.device)
        loss = loss + (r.double() * w(r)).sum() + (t.double() * w(t)).sum() + (yl.double() * w(yl)).sum() \
            + (yr.double() * w(yr)).sum()
    return loss


@pytest.mark.parametrize('ds', ['db5', 'dips'])
def test_iegmn_forward_grads_bitwise_equal_to_docking_net(ds, cuda_device):
    """The same loss on T, b and both keypoint sets through IEGMN.forward and through Rigid_Body_Docking_Net.forward
    (train mode, same inputs): bitwise equal parameter and graph-input gradients; x_iegmn_out / hv_iegmn_out in the graph
    are autograd-connected.  Under torch.no_grad() IEGMN.forward keeps the inference path."""
    model, _ = _model(ds, cuda_device)
    model.train()
    pairs = _pairs(ds, 'ragged')

    def run(call):
        model.zero_grad(set_to_none=True)
        g = gio.make_batch(pairs, cuda_device)
        ins = graph_inputs(g)
        for t in ins:
            t.requires_grad_(True)
        rot, trans, kp_l, kp_r = call(g)
        _kabsch_loss(rot, trans, kp_l, kp_r, 61).backward()
        return [p.grad.clone() for p in model.parameters()], [t.grad.clone() for t in ins], g

    def net(g):
        _, kp_l, kp_r, rot, trans = model(g, 0)
        return rot, trans, kp_l, kp_r

    gp_net, gi_net, _ = run(net)
    gp_ieg, gi_ieg, g = run(lambda g: model.iegmn_original(g, 0))
    for (n, _), a, b in zip(model.named_parameters(), gp_net, gp_ieg):
        assert torch.equal(a, b), n
    for a, b in zip(gi_net, gi_ieg):
        assert torch.equal(a, b)
    from equidock_public_b200.hetero_graph import LIGAND, RECEPTOR
    for nt in (LIGAND, RECEPTOR):
        assert g.nodes[nt].data['x_iegmn_out'].grad_fn is not None
        assert g.nodes[nt].data['hv_iegmn_out'].grad_fn is not None
    with torch.no_grad():
        out = model.iegmn_original(gio.make_batch(pairs, cuda_device), 0)
    assert all(t.grad_fn is None for lst in out for t in lst)
