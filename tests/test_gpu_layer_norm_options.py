"""GPU (H100): models with the reference's coordinate LayerNorm (layer_norm_coors='LN', coors_mlp.3) and final feature
LayerNorm (final_h_layer_norm='LN', final_h_layernorm_layer), alone and together, on the tensor-core and fp32 edge and node
stages and in the CUDA backward, against the fp64 restatement of tests/layer_norm_ref.py.

Bounds.  Those of the shipped configuration: tests/test_gpu_edge_stage.py's 1e-5 relative for the edge-stage kernels and
tests/test_gpu_dropout.py's 2e-3 on coordinates scaled by max(1, |x|/100) and 3e-3 relative per parameter gradient for
whole models.  The coordinate LayerNorm needs no extra allowance: it normalises a row of the same kind as edge_mlp.3 and
its measured errors stay within those bounds.  The final LayerNorm normalises every layer's node output, so an fp32 error e
of the row y reaches h' as about |gamma_f| e / sigma_y, once per layer; on the 8-layer DIPS model with |gamma_f| <= 1.5
this was measured on an H100 at 2.8x the coordinate bound and 1.8x the gradient bound.  Models with the final LayerNorm
are therefore held to FINAL_LN_AMP = 4 times the bounds (SIGMA_AMP = 1 otherwise)."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dropout_masks as dm
import fp64_stages as fs
import golden_io as gio
import layer_norm_ref as nr
from equidock_public_b200 import _native as nat
from equidock_public_b200 import synthetic
from equidock_public_b200.engine import GraphPlan
from equidock_public_b200.hetero_graph import LIGAND, LL, RECEPTOR, RR
from test_gpu_dropout import _loss, _oracle_inputs, _pairs, _run_module, _targets

pytestmark = pytest.mark.gpu
SIGMA_AMP = 1.0
FINAL_LN_AMP = 4.0
N_LAYS = {'db5': 5, 'dips': 8}


def _amp(args=None):
    return FINAL_LN_AMP if args is not None and args['final_h_layer_norm'] == 'LN' else SIGMA_AMP


def _coord_bound(ref, args=None):
    return _amp(args) * 2e-3 * max(1.0, float(np.abs(ref).max()) / 100)


def _grad_mismatches(got, ref, args=None):
    gmax = max(np.abs(v).max() for v in ref.values())
    return [(n, float(np.abs(got[n] - ref[n]).max() / max(np.abs(ref[n]).max(), 1e-30))) for n in got
            if np.abs(got[n] - ref[n]).max() > _amp(args) * 3e-3 * np.abs(ref[n]).max() + 2e-6 * gmax]


def _fp64_state(model, requires_grad=False):
    leaves, sd = {}, {}     # one fp64 leaf per parameter tensor: weight-shared layers sum their gradients
    for k, v in model.state_dict(keep_vars=True).items():
        if v.data_ptr() not in leaves:
            leaves[v.data_ptr()] = torch.from_numpy(v.detach().cpu().double().numpy()).requires_grad_(requires_grad)
        sd[k] = leaves[v.data_ptr()]
    return sd


# ---- forward ------------------------------------------------------------------------------------------------------------

COMBOS = [('LN', '0'), ('0', 'LN'), ('LN', 'LN')]     # (layer_norm_coors, final_h_layer_norm)


@pytest.mark.parametrize('ds', ['db5', 'dips'])
@pytest.mark.parametrize('kind', ['single', 'ragged3', 'gamma0'])
@pytest.mark.parametrize('combo', COMBOS)
def test_forward_matches_fp64(ds, kind, combo, cuda_device):
    """Eval-mode forward of the 5-layer (shared) / 8-layer model on the tensor cores against the fp64 restatement; the
    CUDA-graph replay and the bf16x3 mode of the same batch.  gamma0: the coordinate LayerNorm's gamma = 0."""
    args = nr.args_with(ds, combo[0], final_h_layer_norm=combo[1])
    model = nr.build_model(ds, cuda_device, args, seed=1, gamma_zero=kind == 'gamma0')
    pairs = _pairs(ds, 'single' if kind == 'single' else 'ragged3')
    g = gio.make_batch(pairs, cuda_device)
    with torch.no_grad():
        coors, kp_l, kp_r, rot, trans = model(g, epoch=0)
        again = model(g, epoch=0)
    got = torch.cat(coors)
    assert torch.equal(got, torch.cat(again[0]))
    plan = model.iegmn_original.last_outputs['plan']
    co_ref, Y, R, _ = nr.model_forward(_fp64_state(model), args, _oracle_inputs(g, plan))
    cr = co_ref.numpy()
    err = float(np.abs(got.cpu().double().numpy() - cr).max())
    print(f'forward {ds} {kind} {combo}: max |coors - fp64| = {err:.3e} (bound {_coord_bound(cr, args):.3e})')
    assert err <= _coord_bound(cr, args)
    assert float(np.abs(torch.stack(rot).cpu().double().numpy() - R.numpy()).max()) <= _amp(args) * 2e-4
    gf = model.graphed(g)
    assert torch.equal(torch.cat(gf.launch().result()[0]), got)
    model.precision = 'bf16x3'
    with torch.no_grad():
        c3 = torch.cat(model(g, epoch=0)[0])
    assert torch.equal(torch.cat(model.graphed(g).launch().result()[0]), c3)
    e3 = float(np.abs(c3.cpu().double().numpy() - cr).max())
    print(f'forward bf16x3 {ds} {kind} {combo}: max |coors - fp64| = {e3:.3e}')
    # bf16x3 carries ~2^-16 relative error per product instead of ~2^-24: 2^8 x the fp32-level error, capped by the
    # coordinate bound of the shipped RMSD gate (1e-1 A at these sizes)
    assert e3 <= max(_coord_bound(cr, args), 0.1)


def test_options_off_runs_the_parent_path(cuda_device):
    """layer_norm_coors='0' in the args is the shipped configuration: the model equals gio.build_model bit for bit."""
    pairs = _pairs('dips', 'ragged3')
    g = gio.make_batch(pairs, cuda_device)
    a = nr.build_model('dips', cuda_device, nr.args_with('dips', '0'))
    b = gio.build_model('dips', cuda_device)
    with torch.no_grad():
        assert torch.equal(torch.cat(a(g, 0)[0]), torch.cat(b(g, 0)[0]))


# ---- the edge-stage kernels ---------------------------------------------------------------------------------------------

def _edge_ref(mod, plan, proj, x_in):
    """fp64 edge stage (fp64_stages.edge_stage) with the coordinate LayerNorm: aggr [n][64], x update [n][3]."""
    slope, dh = float(mod.leakyrelu_neg_slope), int(mod.att_mlp_Q[0].weight.shape[0])
    w, b = fs._w, fs._b
    lin1, ln, lin2, lin3, lnc, lin4 = (mod.edge_mlp[0], mod.edge_mlp[3], mod.edge_mlp[4], mod.coors_mlp[0],
                                       mod.coors_mlp[3], mod.coors_mlp[4])
    N, dev = plan.N, x_in.device
    src, dst = plan.col_src.long(), plan.edge_dst.long()
    he = torch.cat([plan.he_l[:plan.E_l], plan.he_r[:plan.E_r]]).to(fs.F64)
    xrel = x_in[src] - x_in[dst]
    d2 = (xrel ** 2).sum(1, keepdim=True)
    ein = torch.cat([he] + [torch.exp(-d2 / sg) for sg in fs.SIGMAS], 1)
    z1 = proj[src, 0:64] + proj[dst, 64:128] + ein @ w(lin1)[:, 2 * dh:].t()
    msg = F.layer_norm(F.leaky_relu(z1, slope), (64,), w(ln), b(ln), ln.eps) @ w(lin2).t() + b(lin2)
    c3 = F.layer_norm(F.leaky_relu(msg @ w(lin3).t() + b(lin3), slope), (64,), w(lnc), b(lnc), lnc.eps)
    phi = c3 @ w(lin4).t() + b(lin4)
    deg = (plan.row_ptr[1:] - plan.row_ptr[:-1]).to(dev, fs.F64).clamp(min=1)[:, None]
    aggr = torch.zeros(N, 64, dtype=fs.F64, device=dev).index_add_(0, dst, msg) / deg
    xupd = torch.zeros(N, 3, dtype=fs.F64, device=dev).index_add_(0, dst, xrel * phi) / deg
    return aggr, xupd


@pytest.mark.parametrize('k,sizes,shift', [(10, ((23, 31), (38, 17), (1, 1)), 0.0), (1, ((40, 37),), 0.0),
                                           (9, ((129, 131),), 1e3), (64, ((70, 80), (66, 90)), 0.0),
                                           (70, ((75, 110),), 0.0)])
def test_edge_stage_kernels_vs_fp64(k, sizes, shift, cuda_device):
    """eqd_edge_stage (tensor cores, P = 6 and P = 3; the fp32 kernel above in-degree 64) and eqd_edge_stage_ffma with the
    coordinate LayerNorm, each launched twice (bitwise equal), against the fp64 edge stage.  In-degrees 0 (ligand nodes
    without in-edges, a 1-node protein), 1, 9, 10, 64 and 70; proteins of 129 and 131 nodes; coordinates near 1e3 A."""
    dev = cuda_device
    rng = np.random.default_rng(k)
    pairs = [synthetic.synthetic_pair(rng, a, b, min(k, a - 1, b - 1) if min(a, b) > 1 else 0) for a, b in sizes]
    if k == 10:                                       # ligand nodes 4..8 of pair 0 lose their in-edges
        lig = pairs[0][0]
        keep = (lig['dst'] < 4) | (lig['dst'] >= 9)
        for key in ('src', 'dst', 'he'):
            lig[key] = lig[key][keep]
    g = gio.make_batch(pairs, dev)
    plan = GraphPlan.from_graph(g, dev, k)
    N = plan.N
    model = nr.build_model('dips', dev, nr.args_with('dips'), seed=k)
    mod = model.iegmn_original.iegmn_layers[1]
    lay = mod.packed(dev)
    torch.manual_seed(k)
    proj = torch.randn(N, 320, device=dev)
    x = torch.randn(N, 3, device=dev, dtype=torch.float64) * 5 + shift
    x0 = torch.randn(N, 3, device=dev, dtype=torch.float64) * 5 + shift
    lib = nat.load()
    aggr_ref, xupd_ref = _edge_ref(mod, plan, proj.double(), x)
    eta = float(mod.x_connection_init)
    x_ref = eta * x0 + (1 - eta) * x + xupd_ref
    for fn, desc in ((lib.eqd_edge_stage, lay.descriptor(0)), (lib.eqd_edge_stage, lay.descriptor(3)),
                     (lib.eqd_edge_stage_ffma, lay.descriptor(0))):
        outs = []
        for _ in range(2):
            aggr = torch.full((N, 64), float('nan'), device=dev)
            xo = torch.full((N, 3), float('nan'), device=dev, dtype=torch.float64)
            st = torch.zeros(plan.n_pairs + 1, dtype=torch.int32, device=dev)
            rc = fn(C.byref(plan.struct), C.byref(desc), nat.ptr(proj), nat.ptr(x), nat.ptr(x0), nat.ptr(aggr),
                    nat.ptr(xo), nat.ptr(st), None)
            torch.cuda.synchronize()
            assert rc == 0 and int(st.abs().sum()) == 0
            outs.append((aggr, xo))
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
        aggr, xo = outs[0]
        # P = 3 keeps its own bound: 2^-16 relative error per product (eqd_layer_params.mma_products)
        tol = 1e-5 if desc.dev.mma_products != 3 or k > 64 else 3e-4
        ea = float((aggr.double() - aggr_ref).abs().max()) / max(1.0, float(aggr_ref.abs().max()))
        ex = float((xo - x_ref).abs().max()) / max(1.0, float(xupd_ref.abs().max()))
        print(f'edge stage k={k} {fn.__name__} P={desc.dev.mma_products}: aggr {ea:.2e}, x {ex:.2e}')
        assert ea <= SIGMA_AMP * tol and ex <= SIGMA_AMP * tol, (ea, ex)
    half = lay.descriptor(0).__class__.from_buffer_copy(lay.descriptor(0))
    half.norms.coors_ln_b = None
    assert lib.eqd_edge_stage(C.byref(plan.struct), C.byref(half), nat.ptr(proj), nat.ptr(x), nat.ptr(x0),
                              nat.ptr(aggr), nat.ptr(xo), nat.ptr(st), None) == -1     # EQD_ERR_BAD_ARG


# ---- training -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('ds', ['db5', 'dips'])
@pytest.mark.parametrize('p', [0.0, 0.25])
@pytest.mark.parametrize('combo', COMBOS)
def test_training_matches_fp64_autograd(ds, p, combo, cuda_device):
    """loss.backward() through the module (CUDA backward with the coordinate LayerNorm; p > 0: the fp32 forward kernels
    with their dropout masks) on a ragged batch of 3: coordinates, loss and every parameter gradient, the coordinate
    LayerNorm's gamma / beta included, against torch.autograd on the fp64 restatement under the same masks.  The same
    torch seed reproduces the run bit for bit."""
    args = nr.args_with(ds, combo[0], dropout=p, final_h_layer_norm=combo[1])
    model = nr.build_model(ds, cuda_device, args, seed=2).train()
    pairs = _pairs(ds, 'ragged3')
    tg = _targets(pairs)
    g, fwd, loss, coors, grads = _run_module(model, pairs, tg, cuda_device, 11)
    _, _, loss2, coors2, grads2 = _run_module(model, pairs, tg, cuda_device, 11)
    assert torch.equal(loss, loss2) and torch.equal(coors, coors2) and all(torch.equal(grads[n], grads2[n]) for n in grads)
    plan = fwd['plan']
    masks = None
    if p > 0:
        masks = dm.BatchMasks(p, fwd['dropout_layers'][0].dropout.seed, 0, plan.N, plan.E, N_LAYS[ds])
    sd = _fp64_state(model, requires_grad=True)
    co_ref, Y, _, _ = nr.model_forward(sd, args, _oracle_inputs(g, plan), masks)
    B = plan.n_pairs
    loss_ref = _loss(co_ref, (Y[:B], Y[B:]), tg, plan.n_lig_list)
    loss_ref.backward()
    cr = co_ref.detach().numpy()
    err = float(np.abs(coors.cpu().numpy() - cr).max())
    assert err < _coord_bound(cr, args)
    assert abs(loss.item() - loss_ref.item()) < _amp(args) * 1e-3 * abs(loss_ref.item())
    ref = {k: v.grad.numpy() for k, v in sd.items()}
    got = {n: q.cpu().double().numpy() for n, q in grads.items()}
    assert any('coors_mlp.3' in n for n in got) == (combo[0] == 'LN')
    assert any('final_h_layernorm_layer' in n for n in got) == (combo[1] == 'LN')
    bad = _grad_mismatches(got, ref, args)
    worst = max(float(np.abs(got[n] - ref[n]).max() / max(np.abs(ref[n]).max(), 1e-30)) for n in got)
    print(f'training {ds} p={p} {combo}: coors {err:.2e}, worst relative gradient error {worst:.2e}')
    assert not bad, bad


@pytest.mark.parametrize('ds', ['db5', 'dips'])
@pytest.mark.parametrize('li', [0, 1])
@pytest.mark.parametrize('combo', COMBOS)
def test_layer_autograd_matches_fp64_autograd(ds, li, combo, cuda_device):
    """One IEGMN_Layer call with the coordinate LayerNorm under autograd: outputs and every parameter gradient against
    torch.autograd on the fp64 layer restatement."""
    args = nr.args_with(ds, combo[0], final_h_layer_norm=combo[1])
    model = nr.build_model(ds, cuda_device, args, seed=3)
    lay = model.iegmn_original.iegmn_layers[li]
    lay.force_autograd = True
    g = gio.make_batch(_pairs(ds, 'ragged3'), cuda_device)
    nl, nr_ = g.nodes[LIGAND].data, g.nodes[RECEPTOR].data
    emb = model.iegmn_original.residue_emb_layer.weight.detach()
    h0 = [torch.cat([emb[d['res_feat'].reshape(-1).long()], torch.log(d['mu_r_norm'])], 1) for d in (nl, nr_)]
    rng = np.random.default_rng(li)
    h = h0 if li == 0 else [torch.from_numpy(rng.normal(0, 1, (t.shape[0], 64)).astype(np.float32)).to(cuda_device)
                            for t in h0]
    x = [nl['new_x'], nr_['x']]
    he = [g.edges[LL].data['he'], g.edges[RR].data['he']]
    xl, hl, xr, hr = lay(g, x[0], h[0], h0[0], he[0], x[0], x[1], h[1], h0[1], he[1], x[1])
    wx = torch.from_numpy(rng.normal(0, 1, (xl.shape[0] + xr.shape[0], 3))).to(cuda_device)
    wh = torch.from_numpy(rng.normal(0, 1, (hl.shape[0] + hr.shape[0], 64))).to(cuda_device)
    lay.zero_grad(set_to_none=True)
    ((torch.cat([xl, xr]).double() * wx).sum() + (torch.cat([hl, hr]).double() * wh).sum()).backward()
    plan = g._eqd_plan
    inp = _oracle_inputs(g, plan)
    p = {k: torch.from_numpy(v.detach().cpu().double().numpy()).requires_grad_(True) for k, v in lay.state_dict().items()}
    cpu = lambda a, b: torch.cat([a.detach().cpu(), b.detach().cpu()]).double()
    x_ref, h_ref = nr.layer_forward(p, inp['x'], cpu(h[0], h[1]), inp['x'], cpu(h0[0], h0[1]), inp['src'], inp['dst'],
                                    inp['he'], inp['seg'], plan.n_pairs, float(args['leakyrelu_neg_slope']),
                                    float(args['skip_weight_h']), float(args['x_connection_init']))
    ((x_ref * wx.cpu()).sum() + (h_ref * wh.cpu()).sum()).backward()
    xg, hg = torch.cat([xl, xr]).detach().cpu().double(), torch.cat([hl, hr]).detach().cpu().double()
    assert (xg - x_ref.detach()).abs().max() < _coord_bound(x_ref.detach().numpy(), args)
    assert (hg - h_ref.detach()).abs().max() < _amp(args) * 2e-3 * h_ref.abs().max().item()
    ref = {k: v.grad.numpy() for k, v in p.items()}
    got = {n: q.grad.detach().cpu().double().numpy() for n, q in lay.named_parameters()}
    assert ('coors_mlp.3.weight' in got) == (combo[0] == 'LN')
    assert ('final_h_layernorm_layer.weight' in got) == (combo[1] == 'LN')
    bad = _grad_mismatches(got, ref, args)
    assert not bad, bad


@pytest.mark.parametrize('combo', COMBOS)
def test_fused_trainer_step_matches_the_module_path(combo, cuda_device):
    """DataParallelTrainer.step of a DB5-shaped (weight-shared) model with the coordinate LayerNorm against model.train();
    outputs -> the same device losses through autograd -> loss.backward(): the same loss, and the trainer's flat gradient
    (clip out of reach) equal to every param.grad within the bounds above."""
    from equidock_public_b200.losses import PocketBatch, device_losses
    from equidock_public_b200.training import DataParallelTrainer
    rng = np.random.default_rng(12)
    pairs = [synthetic.synthetic_pair(rng, a, b, 10) for a, b in [(60, 75), (90, 50)]]
    g = gio.make_batch(pairs, cuda_device)
    bl = [torch.from_numpy(p[0]['x']) for p in pairs]
    br = [torch.from_numpy(p[1]['x'] + 8.0) for p in pairs]
    pk = [torch.from_numpy((0.5 * (p[0]['x'][:9] + p[1]['x'][:9] + 8.0)).astype(np.float32)) for p in pairs]
    tgt = PocketBatch(bl, br, pk, pk, cuda_device)
    args = nr.args_with('db5', combo[0], final_h_layer_norm=combo[1])
    m1 = nr.build_model('db5', cuda_device, args, seed=4).train()
    m2 = nr.build_model('db5', cuda_device, args, seed=4).train()
    tr = DataParallelTrainer(m1, lr=1e-3, weight_decay=1e-4, clip=1e30)
    r1 = tr.step(g, tgt)
    coors, kl, kr, _, _ = m2(g, epoch=0)
    plan = m2.iegmn_original.last_outputs['plan']
    kp = torch.cat([torch.stack(kl), torch.stack(kr)]).double()
    res = device_losses(plan, torch.cat(coors), kp, tgt, 1.0, 10.0, 25.0, 10.0)
    ((torch.cat(coors) * res['dcoors']).sum() + (kp * res['dkeypts']).sum()).backward()
    assert abs(float(r1['loss'][0]) - float(res['total'][0])) < 1e-6 * max(1.0, abs(float(res['total'][0])))
    by_param = {id(q): v for q, v in zip(tr.layout.params, tr.layout.views(tr.flat_g))}
    flat = {n: by_param[id(q)].double().cpu().numpy() for n, q in m1.named_parameters()}
    ref = {n: q.grad.detach().double().cpu().numpy() for n, q in m2.named_parameters()}
    assert any('coors_mlp.3' in n for n in ref) == (combo[0] == 'LN')
    bad = _grad_mismatches(flat, ref, args)
    assert not bad, bad
