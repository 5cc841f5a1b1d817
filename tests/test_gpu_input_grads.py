"""GPU (H100): gradients with respect to the graph's input tensors (ligand new_x, receptor x, both mu_r_norm, both edge
types' he) and through the x_iegmn_out / hv_iegmn_out side outputs, through ``loss.backward()`` on the drop-in module,
against torch.autograd on the fp64 TorchOracle.

The loss is probe_loss (ligand coordinates and both keypoint sets) plus a seeded quadratic term on the last layer's
coordinates and features of both proteins.  Every tensor passes if max|got - ref| <= 3e-3 max|ref| + 2e-6 G, G = the
largest reference magnitude of its group: the bound of the backward's own tests (test_gpu_backward.py), with the groups
coordinate gradients (new_x, x), mu_r_norm gradients, he gradients and parameter gradients.  Printed per tensor: the
absolute error and the error relative to max|ref|."""
import numpy as np
import pytest
import torch

import golden_io as gio
import iegmn_oracle_torch as ot
from equidock_public_b200 import _native as nat
from equidock_public_b200 import synthetic
from equidock_public_b200.hetero_graph import LIGAND, LL, RECEPTOR, RR
from equidock_public_b200.rigid_docking_model import graph_inputs

pytestmark = pytest.mark.gpu
PAIR = {'db5': '1QA9', 'dips': 'kq_1kq1.pdb1_2.dill'}
INPUTS = ('new_x', 'x', 'mu_lig', 'mu_rec', 'he_ll', 'he_rr')    # graph_inputs order


class _Oracle(ot.TorchOracle):
    """TorchOracle that keeps the last layer's coordinates and features of both proteins."""

    def _layer(self, li, sides):
        super()._layer(li, sides)
        if li == self.L - 1:
            self.last = [(s['x'], s['h']) for s in sides]


def _np(t):
    return t.detach().double().cpu().numpy()


def _pairs(ds, batch):
    if batch == 'golden':
        _, pairs, _, _ = gio.load_pairs(ds)
        return [pairs[PAIR[ds]]]
    rng = np.random.default_rng(9)
    return [synthetic.synthetic_pair(rng, a, b, 10) for a, b in [(40, 131), (129, 20), (64, 64)]]


def _targets(pairs, seed, probe=True, side=True):
    rng = np.random.default_rng(seed)
    tg = []
    for lig, rec in pairs:
        nl, nr = lig['new_x'].shape[0], rec['x'].shape[0]
        tg.append({'probe': probe, 'side': side, 'coors': rng.normal(0, 5, (nl, 3)) + lig['x'].mean(0),
                   'w_l': rng.uniform(0, 1, 50), 'p_l': rng.normal(0, 10, (50, 3)),
                   'w_r': rng.uniform(0, 1, 50), 'p_r': rng.normal(0, 10, (50, 3)),
                   'ax_l': rng.uniform(0, 1, (nl, 3)) / nl, 'tx_l': rng.normal(0, 5, (nl, 3)),
                   'ax_r': rng.uniform(0, 1, (nr, 3)) / nr, 'tx_r': rng.normal(0, 5, (nr, 3)),
                   'ah_l': rng.uniform(0, 1, (nl, 64)) / nl, 'ah_r': rng.uniform(0, 1, (nr, 64)) / nr})
    return tg


def _loss(coors, y_l, y_r, x_l, h_l, x_r, h_r, t):
    """fp64 scalar: probe_loss + sum a_x (x - t_x)^2 + sum a_h h^2 over both proteins' last-layer outputs."""
    T = lambda k: torch.as_tensor(t[k]).to(device=coors.device, dtype=torch.float64)
    d = lambda v: v.to(torch.float64)
    loss = torch.zeros((), dtype=torch.float64, device=coors.device)
    if t['probe']:
        loss = loss + ot.probe_loss(d(coors), d(y_l), d(y_r), {k: T(k) for k in ('coors', 'w_l', 'p_l', 'w_r', 'p_r')})
    if t['side']:
        loss = loss + (T('ax_l') * (d(x_l) - T('tx_l')) ** 2).sum() + (T('ax_r') * (d(x_r) - T('tx_r')) ** 2).sum() \
            + (T('ah_l') * d(h_l) ** 2).sum() + (T('ah_r') * d(h_r) ** 2).sum()
    return loss


def _oracle(model, args, pairs, tgts):
    """fp64 torch.autograd through the TorchOracle, pair by pair: (input gradients in engine order, parameter gradients
    keyed like model.named_parameters())."""
    sd = {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}
    m = _Oracle(sd, args['iegmn_n_lays'], args['skip_weight_h'], args['x_connection_init'], args['leakyrelu_neg_slope'],
                args['num_att_heads'], dtype=torch.float64)
    psd = m.parameters_for_grad()
    leaves = []
    loss = 0.0
    for (lig, rec), t in zip(pairs, tgts):
        lf = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)
        l2, r2 = dict(lig), dict(rec)
        for d, ck in ((l2, 'new_x'), (r2, 'x')):
            for k in (ck, 'mu_r_norm', 'he'):
                d[k] = lf(d[k])
        out = m.forward_pair_grad(l2, r2)
        (xl, hl), (xr, hr) = m.last
        loss = loss + _loss(out['ligand_coors'], out['keypts_ligand'], out['keypts_receptor'], xl, hl, xr, hr, t)
        leaves.append((l2, r2))
    loss.backward()
    g = lambda v: v.grad.numpy() if v.grad is not None else np.zeros(tuple(v.shape))
    cat = lambda side, k: np.concatenate([g(lv[side][k]) for lv in leaves])
    ref_in = [cat(0, 'new_x'), cat(1, 'x'), cat(0, 'mu_r_norm'), cat(1, 'mu_r_norm'), cat(0, 'he'), cat(1, 'he')]
    shared = bool(args['shared_layers'])
    ref_p = {}
    for name, _ in model.named_parameters():
        ref_p[name] = g(psd[name])
        if shared and '.iegmn_layers.' in name and int(name.split('.iegmn_layers.')[1].split('.')[0]) >= 1:
            # one leaf per layer index in the restatement; the shared module's gradient is their sum
            suffix = name.split('.iegmn_layers.')[1].split('.', 1)[1]
            ref_p[name] = sum(g(psd[f'iegmn_original.iegmn_layers.{j}.{suffix}']) for j in range(1, args['iegmn_n_lays']))
    return ref_in, ref_p


def _graph(pairs, dev, dtype=torch.float32):
    g = gio.make_batch(pairs, dev)
    nl, nr = g.nodes[LIGAND].data, g.nodes[RECEPTOR].data
    nl['new_x'], nr['x'] = nl['new_x'].to(dtype), nr['x'].to(dtype)
    nl['mu_r_norm'], nr['mu_r_norm'] = nl['mu_r_norm'].to(dtype), nr['mu_r_norm'].to(dtype)
    g.edges[LL].data['he'], g.edges[RR].data['he'] = g.edges[LL].data['he'].to(dtype), g.edges[RR].data['he'].to(dtype)
    return g


def _engine_loss(model, g, tgts):
    coors, kp_l, kp_r, rot, trans = model(g, epoch=0)
    raw = model.iegmn_original.last_outputs
    B = len(tgts)
    assert not bool(raw['status_host'][:B].any()), raw['status_host'][:B].tolist()   # the oracle has no guard branch
    plan = raw['plan']
    nl, nr = g.nodes[LIGAND].data, g.nodes[RECEPTOR].data
    split = lambda t, n: torch.split(t, n, dim=0)
    xl, hl = split(nl['x_iegmn_out'], plan.n_lig_list), split(nl['hv_iegmn_out'], plan.n_lig_list)
    xr, hr = split(nr['x_iegmn_out'], plan.n_rec_list), split(nr['hv_iegmn_out'], plan.n_rec_list)
    loss = sum(_loss(coors[i], kp_l[i], kp_r[i], xl[i], hl[i], xr[i], hr[i], tgts[i]) for i in range(B))
    return loss, (coors, kp_l, kp_r, rot, trans, nl['x_iegmn_out'], nl['hv_iegmn_out'], nr['x_iegmn_out'],
                  nr['hv_iegmn_out'])


def _report(got_in, ref_in, model, ref_p, amp=1.0):
    """Prints every tensor's error; returns the ones out of bound (``amp`` times the bound)."""
    rows = [(grp, f'd {n}', _np(a).reshape(r.shape), r)
            for n, grp, a, r in zip(INPUTS, ('x', 'x', 'mu', 'mu', 'he', 'he'), got_in, ref_in) if a is not None]
    rows += [('param', n.replace('iegmn_original.', ''), _np(p.grad).reshape(ref_p[n].shape) if p.grad is not None
              else np.zeros(ref_p[n].shape), ref_p[n]) for n, p in model.named_parameters()]
    G = {grp: max(float(np.abs(r).max()) for g_, _, _, r in rows if g_ == grp) for grp in {row[0] for row in rows}}
    bad = []
    for grp, tag, got, ref in rows:
        err, rmax = float(np.abs(got - ref).max()), float(np.abs(ref).max())
        ok = err <= amp * (3e-3 * rmax + 2e-6 * G[grp])
        line = f'{"ok  " if ok else "BAD "}{tag:52s} abs {err:.2e}  rel {err / max(rmax, 1e-30):.2e}  max|ref| {rmax:.3e}'
        print(line)
        if not ok:
            bad.append(line)
    return bad


def _model(ds, dev, eta):
    args = dict(gio.load_args(ds), x_connection_init=eta)
    return gio.build_model(ds, dev, args=args), args


def _check(ds, batch, eta, cuda_device, mode='train', probe=True, side=True):
    model, args = _model(ds, cuda_device, eta)
    model.train() if mode == 'train' else model.eval()
    pairs = _pairs(ds, batch)
    tgts = _targets(pairs, 21, probe, side)
    g = _graph(pairs, cuda_device)
    ins = graph_inputs(g)
    for t in ins:
        t.requires_grad_(True)
    loss, _ = _engine_loss(model, g, tgts)
    loss.backward()
    ref_in, ref_p = _oracle(model, args, pairs, tgts)
    bad = _report([t.grad for t in ins], ref_in, model, ref_p)
    assert not bad, '\n'.join(bad)


@pytest.mark.parametrize('eta', [0.0, 0.3])
@pytest.mark.parametrize('batch', ['golden', 'ragged'])
@pytest.mark.parametrize('ds', ['db5', 'dips'])
def test_input_and_parameter_grads_vs_fp64_oracle(ds, batch, eta, cuda_device):
    """Both checkpoints (5 shared layers / 8 layers), one golden pair and a ragged batch of 3 with the 128 + 1 / 128 + 3
    tile-boundary sizes, x_connection_init 0 (the shipped value) and 0.3 (the eta share of every layer's coordinate
    gradient reaches the input coordinates)."""
    _check(ds, batch, eta, cuda_device)


def test_eval_mode_input_grads_and_bitwise_outputs(cuda_device):
    """model.eval() with an input requiring grad takes the autograd path: its outputs are bitwise those of the
    torch.no_grad() inference path, and its gradients pass the same bounds."""
    model, args = _model('dips', cuda_device, 0.3)
    model.eval()
    pairs = _pairs('dips', 'ragged')
    tgts = _targets(pairs, 22)
    with torch.no_grad():
        _, ref_out = _engine_loss(model, _graph(pairs, cuda_device), tgts)
    g = _graph(pairs, cuda_device)
    ins = graph_inputs(g)
    ins[0].requires_grad_(True)
    ins[5].requires_grad_(True)
    loss, out = _engine_loss(model, g, tgts)
    assert out[0][0].requires_grad
    flat = lambda o: [t for v in o for t in (v if isinstance(v, (list, tuple)) else [v])]
    for a, b in zip(flat(out), flat(ref_out)):
        assert a.dtype == b.dtype and torch.equal(a.detach(), b)
    loss.backward()
    ref_in, ref_p = _oracle(model, args, pairs, tgts)
    bad = _report([ins[0].grad, None, None, None, None, ins[5].grad], ref_in, model, ref_p)
    assert not bad, '\n'.join(bad)


def test_side_output_loss_only(cuda_device):
    """A loss on hv_iegmn_out / x_iegmn_out alone: parameter (and input) gradients within the bound."""
    _check('db5', 'ragged', 0.3, cuda_device, probe=False)


def test_parameter_grads_unchanged_and_new_kernels_idle_without_input_grads(cuda_device, monkeypatch):
    """No input requiring grad: the input-gradient entry points are never called, and every parameter gradient is bitwise
    the one of a run that also produced input gradients."""
    lib = nat.load()
    calls = {'eqd_bwd_layer_inputs': 0, 'eqd_bwd_inputs': 0}
    for name in calls:
        fn = getattr(lib, name)

        def counted(*a, _fn=fn, _name=name):
            calls[_name] += 1
            return _fn(*a)
        monkeypatch.setattr(lib, name, counted)
    model, args = _model('dips', cuda_device, 0.3)
    model.train()
    pairs = _pairs('dips', 'ragged')
    tgts = _targets(pairs, 23)

    def grads(with_inputs):
        model.zero_grad(set_to_none=True)
        g = _graph(pairs, cuda_device)
        if with_inputs:
            for t in graph_inputs(g):
                t.requires_grad_(True)
        _engine_loss(model, g, tgts)[0].backward()
        return [p.grad.clone() for p in model.parameters()]

    plain = grads(False)
    assert calls == {'eqd_bwd_layer_inputs': 0, 'eqd_bwd_inputs': 0}
    with_in = grads(True)
    assert calls == {'eqd_bwd_layer_inputs': args['iegmn_n_lays'], 'eqd_bwd_inputs': 1}
    for a, b in zip(plain, with_in):
        assert torch.equal(a, b)


def test_shuffled_edges_grad_in_caller_order(cuda_device):
    """Edge lists out of destination order (each destination's in-edges keep their relative order, so the sorted copy is
    the original batch): he.grad arrives in the caller's order and equals the sorted case's gradient permuted."""
    model, _ = _model('db5', cuda_device, 0.3)
    model.train()
    pairs = _pairs('db5', 'ragged')
    tgts = _targets(pairs, 24)
    shuffled, perms = [], []
    for lig, rec in pairs:
        sides, ps = [], []
        for d in (lig, rec):
            q = np.argsort(-d['dst'].astype(np.int64), kind='stable')      # destinations descending
            d2 = dict(d)
            d2['src'], d2['dst'], d2['he'] = d['src'][q], d['dst'][q], d['he'][q]
            sides.append(d2)
            ps.append(q)
        shuffled.append(tuple(sides))
        perms.append(ps)

    def run(prs):
        model.zero_grad(set_to_none=True)
        g = _graph(prs, cuda_device)
        ins = graph_inputs(g)
        for t in ins:
            t.requires_grad_(True)
        _engine_loss(model, g, tgts)[0].backward()
        return [t.grad for t in ins], [p.grad.clone() for p in model.parameters()]

    (gi_s, gp_s), (gi_u, gp_u) = run(pairs), run(shuffled)
    for side, k in ((0, 4), (1, 5)):
        off, idx = 0, []
        for ps, pr in zip(perms, pairs):
            idx.append(torch.from_numpy(ps[side]) + off)
            off += pr[side]['he'].shape[0]
        idx = torch.cat(idx).to(cuda_device)
        assert torch.equal(gi_u[k], gi_s[k][idx])
    for a, b in zip(gi_s[:4], gi_u[:4]):
        assert torch.equal(a, b)
    for a, b in zip(gp_s, gp_u):
        assert torch.equal(a, b)


def test_misaligned_he_slice_and_fp64_inputs(cuda_device):
    """he given as a row slice the engine must copy (not 16-byte aligned): the gradient lands in the caller's tensor.
    fp64 input tensors get fp64 gradients (the engine computes in the same precision, so they round to the fp32 case's).
    torch.autograd.grad(loss, [new_x, he]) works."""
    model, _ = _model('db5', cuda_device, 0.3)
    model.train()
    pairs = _pairs('db5', 'ragged')
    tgts = _targets(pairs, 25)
    g = _graph(pairs, cuda_device)
    ins = graph_inputs(g)
    for t in ins:
        t.requires_grad_(True)
    _engine_loss(model, g, tgts)[0].backward()
    ref = [t.grad for t in ins]

    g = _graph(pairs, cuda_device)
    he = g.edges[LL].data['he']
    big = torch.zeros(he.shape[0] + 1, he.shape[1], device=cuda_device)
    big[1:] = he
    big.requires_grad_(True)
    g.edges[LL].data['he'] = big[1:]
    assert big[1:].data_ptr() % 16 != 0
    _engine_loss(model, g, tgts)[0].backward()
    assert torch.equal(big.grad[1:], ref[4]) and not bool(big.grad[0].any())

    g = _graph(pairs, cuda_device, torch.float64)
    ins = graph_inputs(g)
    for t in ins:
        t.requires_grad_(True)
    _engine_loss(model, g, tgts)[0].backward()
    for t, r in zip(ins, ref):
        # the outputs the loss reads are fp64 here (keypoints, x_iegmn_out), so the upstream gradients differ in the
        # last fp32 bits from the fp32 case's
        assert t.grad.dtype == torch.float64 and t.grad.shape == r.shape
        assert float((t.grad - r.double()).abs().max()) <= 1e-5 * float(r.abs().max())

    g = _graph(pairs, cuda_device)
    nx, he_l = graph_inputs(g)[0], graph_inputs(g)[4]
    nx.requires_grad_(True)
    he_l.requires_grad_(True)
    d_nx, d_he = torch.autograd.grad(_engine_loss(model, g, tgts)[0], [nx, he_l])
    assert torch.equal(d_nx, ref[0]) and torch.equal(d_he, ref[4])
