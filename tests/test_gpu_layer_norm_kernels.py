"""GPU (H100): every entry point with a layer-norm option compiled in (layer_norm_coors='LN': the coordinate
LayerNorm coors_mlp.3, CLN; final_h_layer_norm='LN': the final feature LayerNorm final_h_layernorm_layer, HLN) called
directly on seeded inputs and compared with torch fp64 (autograd) of its stage formula with the LayerNorm(s) added, and
the graph-input gradients of models with these options or with K != 50 keypoints.  The layer-norm counterpart of
test_gpu_forward_kernels.py and test_gpu_backward_kernels.py, whose batches, Report, _twice and _kink_rows it reuses.

The layers come from a layer_norm_ref.build_model DIPS model whose LayerNorm gamma / beta are then overwritten with
distinct per-channel values of both signs (|gamma| in [0.4, 1.6]), so that a swapped or permuted gamma / beta is an O(1)
error; `gamma_c = 0` is the coordinate LayerNorm as reset_parameters leaves it.

The backward kernels are persistent (grid = min(tiles, 132)): on `bulk` every CTA walks at least two edge tiles and two
node tiles, so the per-CTA partial sums of d gamma / d beta (384 floats per CTA for the edge kernel with CLN, 272 for
the node kernel with HLN) accumulate over several tiles, and with HLN the in-place rewrite of dh_out (the gradient
w.r.t. the pre-norm row y) runs in every tile a CTA takes.  The per-CTA partials also go through the layer's own
reduction table (LayerTrainPack maps, eqd_grad_reduce) into a flat gradient, whose ParamLayout views are compared at
the same bound.

Every output is allocated with GUARD rows past its end, pre-filled with the finite SENT; after the launch those rows
must be untouched (the N / E-row outputs, x_out, proj_next, the rewritten dh_out, and the per-CTA partial rows >=
n_partials).  Every kernel runs twice on the same inputs: the outputs must be bitwise equal.

Tolerance: max |kernel - reference| over the compared rows / max |reference|, 1e-5, or 3e-4 for the P = 3 (bf16x3)
products, as test_gpu_layer_norm_options.py's edge test uses.  LeakyReLU kinks are handled as in
test_gpu_backward_kernels.py: rows with a pre-activation within the fp32 error band of 0 are left out of the per-row
comparisons that depend on the branch, at most 0.5 % of the rows.  Measured on an H100 80GB HBM3 (700 W power limit),
largest value over the cases of each test (`pytest -s` prints every value):
  edge stage CLN     tc P=6 aggr 4.5e-7, update 3.8e-7;  tc P=3 aggr 7.8e-7, update 1.2e-8;
                     fp32 aggr 5.1e-7, update 7.4e-7;  fp32 with dropout aggr 6.4e-7, update 3.7e-7
  node MLP HLN       tc P=6 h_out 1.9e-7, P=3 1.5e-5;  layer 0 (tc0) h_out 3.3e-7
  node stage HLN     tc: mu 5.5e-7, h_out 4.1e-7, next-layer Psrc / Pdst / Q / K / V 4.0e-7 .. 5.9e-7;
                     tc0: mu 1.7e-6, h_out 3.9e-6, next-layer projections 1.7e-6 .. 3.4e-6;
                     fp32: mu 2.1e-7, h_out 5.2e-7, proj_next 4.5e-7 .. 5.9e-7
  bwd edge CLN       ein 5.9e-9, n1 5.5e-7, msg 1.1e-6, dz3 5.7e-6, dmsg 7.0e-6, dz1 6.9e-6, dxrel 7.1e-6,
                     dgamma 2.3e-7, dbeta 4.5e-7, dw4 1.0e-6, db4 1.6e-6, dgamma_c 6.8e-7, dbeta_c 2.0e-6
                     (dz3 .. dxrel: the bulk layer-0 case with dropout; every other case stays under 6e-7)
  bwd node HLN       dh_in 1.4e-6, daggr 1.1e-6, dmu 1.2e-6, dh0_acc 1.4e-6, n5 1.5e-6, du 1.3e-6, dh_out rewritten
                     4.0e-7, dgamma 7.6e-7, dbeta 4.0e-7, dgamma_f 3.1e-7, dbeta_f 1.7e-7
  reduction table    the same errors as the per-CTA partial sums it reduces
  input gradients    largest error / max|ref| 4.1e-4 (d x, DIPS with both options and K = 25); parameter gradients
                     1.8e-3 (att_mlp_Q of layer 0, K = 25), within 3e-3 max|ref| + 2e-6 G
The file runs in about 40 s on that GPU.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dropout_masks as dm
import fp64_stages as fs
import layer_norm_ref as nr
import test_gpu_input_grads as ig
from equidock_public_b200 import _native as nat
from equidock_public_b200.hetero_graph import LL, RR
from equidock_public_b200.rigid_docking_model import graph_inputs
from equidock_public_b200.training import TrainEngine
from test_gpu_backward_kernels import KINK_BAND, SMS, Report, _batch, _d, _gen, _kink_rows, _leaf, _reduce, _twice
from test_gpu_dropout import _oracle_inputs
from test_gpu_dropout import _pairs as _dpairs
from test_gpu_forward_kernels import ETA, SENT, _coords, _decode_kv, _fbatch, _np_gen
from test_gpu_layer_norm_options import FINAL_LN_AMP, _fp64_state

pytestmark = pytest.mark.gpu

F64 = torch.float64
GUARD = 3                                    # rows past the end of every output, pre-filled with SENT
P_DROP, SEED = 0.25, 0x5EED_0123_4567_89AB   # the dropout of the kernel cases (rank 3, as test_gpu_dropout_kernels)
SHIFT = (1.0e3, -0.7e3, 0.4e3)               # coordinates around 1e3 A (the range layer-evolved coordinates reach)

_MODELS = {}


# ---- models, descriptors, guarded outputs ---------------------------------------------------------------------

def _distinct(rng):
    """64 distinct per-channel values of both signs for gamma (|gamma| in [0.4, 1.6]) and beta (in [-0.5, 0.5])."""
    g = rng.permutation(np.linspace(0.4, 1.6, 64)) * rng.choice([-1.0, 1.0], 64)
    b = rng.permutation(np.linspace(-0.5, 0.5, 64))
    return torch.from_numpy(g.astype(np.float32)), torch.from_numpy(b.astype(np.float32))


def _ln_model(dev, cln='LN', hln='0', gamma_c0=False):
    """(model, TrainEngine) of the DIPS checkpoint with the given options, gamma / beta of every LayerNorm option
    overwritten with _distinct values (gamma_c0: the coordinate LayerNorm's gamma = 0)."""
    key = (cln, hln, gamma_c0)
    if key not in _MODELS:
        model = nr.build_model('dips', dev, nr.args_with('dips', cln, final_h_layer_norm=hln), seed=5)
        rng = np.random.default_rng(50)
        with torch.no_grad():
            for lay in model.iegmn_original.iegmn_layers:
                lns = [lay.coors_mlp[3]] if cln == 'LN' else []
                lns += [lay.final_h_layernorm_layer] if hln == 'LN' else []
                for ln in lns:
                    g, b = _distinct(rng)
                    ln.weight.copy_(g)
                    ln.bias.copy_(b)
                if gamma_c0:
                    lay.coors_mlp[3].weight.zero_()
        _MODELS[key] = (model, TrainEngine(model))
    return _MODELS[key]


def _layer(li, dev, cln='LN', hln='0', gamma_c0=False):
    model, eng = _ln_model(dev, cln, hln, gamma_c0)
    mod = model.iegmn_original.iegmn_layers[li]
    return mod, mod.packed(dev), eng.layer_pack(mod), eng


def _desc(lay, products=0, drop_layer=None, eta=None):
    """A copy of the layer's eqd_layer with mma_products, dropout (P_DROP at layer position drop_layer) and
    x_connection_init set as given."""
    s = nat.EqdLayer.from_buffer_copy(lay.descriptor(products))
    if drop_layer is not None:
        s.dropout = nat.dropout_descriptor(P_DROP, SEED, drop_layer, 3)
    if eta is not None:
        s.dev.x_connection_init = eta
    return s


def _mask(layer, site, rows, cols, dev):
    return dm.mask(SEED, 3, layer, site, rows, cols, P_DROP).to(dev)


def _out(rows, cols, dev, dtype=torch.float32):
    return torch.full((rows + GUARD, cols), SENT, dtype=dtype, device=dev)


def _guarded(name, t, rows):
    assert bool((t[rows:] == SENT).all()), f'{name}: rows past {rows} were written'


def _kink_kept(pre, terms, what, keep=None):
    """_kink_rows over the elements a dropout mask keeps (dropped ones enter the LeakyReLU as an exact 0)."""
    return _kink_rows(pre if keep is None else torch.where(keep, pre, torch.inf), terms, what)


def _table(lib, tp, eng, name, vec, nparts, ncols, dev):
    """The per-CTA partials through the layer's reduction `name` (LayerTrainPack maps) into a zeroed flat gradient."""
    src, dst = tp.maps[name][1]
    flat = torch.zeros(eng.layout.total, device=dev)
    nat.check(lib.eqd_grad_reduce(nat.ptr(vec), nparts, ncols, nat.ptr(src), nat.ptr(dst), int(src.numel()),
                                  nat.ptr(flat), None), 'eqd_grad_reduce')
    return flat


def _view(eng, flat, li, pname, numel):
    off = eng.layout.name_offset[f'iegmn_original.iegmn_layers.{li}.{pname}']
    return flat[off:off + numel]


# ---- fp64 stage formulas with the LayerNorms ------------------------------------------------------------------------

def _edge_fwd_ref(mod, plan, proj, x_in, m0=1.0, m1=1.0):
    """fp64 edge stage with the coordinate LayerNorm and the dropout factors m0 (z1) / m1 (z3): aggr [n][64],
    xupd [n][3]."""
    slope, dh = float(mod.leakyrelu_neg_slope), int(mod.att_mlp_Q[0].weight.shape[0])
    w, b = fs._w, fs._b
    lin1, ln, lin2, lin3, lnc, lin4 = (mod.edge_mlp[0], mod.edge_mlp[3], mod.edge_mlp[4], mod.coors_mlp[0],
                                       mod.coors_mlp[3], mod.coors_mlp[4])
    N, dev = plan.N, x_in.device
    src, dst = plan.col_src.long(), plan.edge_dst.long()
    he = torch.cat([plan.he_l[:plan.E_l], plan.he_r[:plan.E_r]]).to(F64)
    xrel = x_in[src] - x_in[dst]
    d2 = (xrel ** 2).sum(1, keepdim=True)
    ein = torch.cat([he] + [torch.exp(-d2 / sg) for sg in fs.SIGMAS], 1)
    z1 = (proj[src, 0:64] + proj[dst, 64:128] + ein @ w(lin1)[:, 2 * dh:].t()) * m0
    msg = F.layer_norm(F.leaky_relu(z1, slope), (64,), w(ln), b(ln), ln.eps) @ w(lin2).t() + b(lin2)
    z3 = (msg @ w(lin3).t() + b(lin3)) * m1
    phi = F.layer_norm(F.leaky_relu(z3, slope), (64,), w(lnc), b(lnc), lnc.eps) @ w(lin4).t() + b(lin4)
    deg = (plan.row_ptr[1:] - plan.row_ptr[:-1]).to(dev, F64).clamp(min=1)[:, None]
    aggr = torch.zeros(N, 64, dtype=F64, device=dev).index_add_(0, dst, msg) / deg
    xupd = torch.zeros(N, 3, dtype=F64, device=dev).index_add_(0, dst, xrel * phi) / deg
    return aggr, xupd


def _node_fwd_ref(mod, h, aggr, mu, h0, m2=1.0):
    """LN_f(skip(node_mlp([h | aggr | mu | h0]))) in fp64, with the dropout factor m2 on u5."""
    w, b = fs._w, fs._b
    slope, sk = float(mod.leakyrelu_neg_slope), float(mod.skip_weight_h)
    lin0, ln, lin4, lnf = mod.node_mlp[0], mod.node_mlp[3], mod.node_mlp[4], mod.final_h_layernorm_layer
    u5 = (torch.cat([h, aggr, mu, h0], 1) @ w(lin0).t() + b(lin0)) * m2
    o = F.layer_norm(F.leaky_relu(u5, slope), (u5.shape[1],), w(ln), b(ln), ln.eps) @ w(lin4).t() + b(lin4)
    y = sk * o + (1.0 - sk) * h if h.shape[1] == o.shape[1] else o
    return F.layer_norm(y, (64,), w(lnf), b(lnf), lnf.eps)


# ---- forward: edge stage with the coordinate LayerNorm --------------------------------------------------------------

def _edge_run(fn, plan, desc, proj, x_in, x_orig, dev):
    N, B = plan.N, plan.n_pairs

    def run():
        aggr, xo = _out(N, 64, dev), _out(N, 3, dev, F64)
        st = torch.zeros(B + 1, dtype=torch.int32, device=dev)
        nat.check(fn(C.byref(plan.struct), C.byref(desc), nat.ptr(proj), nat.ptr(x_in), nat.ptr(x_orig), nat.ptr(aggr),
                     nat.ptr(xo), nat.ptr(st), None), 'edge stage')
        return aggr, xo, st

    aggr, xo, st = _twice(run)
    assert int(st.abs().sum()) == 0, 'status words must stay 0'
    _guarded('aggr', aggr, N)
    _guarded('x_out', xo, N)
    return aggr[:N], xo[:N]


def _edge_inputs(kind, li, seed, dev):
    g, plan = _fbatch(kind, dev)
    mod, lay, tp, _ = _layer(li, dev)
    r = _np_gen(seed, dev)
    proj = r(plan.N, tp.pw, s=0.5).contiguous()
    x_in = (_coords(g, dev) + torch.tensor(SHIFT, dtype=F64, device=dev)).contiguous()
    x_orig = (x_in + r(plan.N, 3, s=3.0).double()).contiguous()
    return plan, mod, lay, proj, x_in, x_orig


@pytest.mark.parametrize('kind,li', [('bench', 1), ('bench', 0), ('bulk', 1), ('bulk', 0), ('mixed', 1), ('mixed', 0),
                                     ('k64', 1), ('k70', 1), ('k70', 0)])
def test_edge_stage_cln_vs_fp64(kind, li, cuda_device):
    """eqd_edge_stage (tensor cores; P = 6, and P = 3 for the 64-wide layer) and eqd_edge_stage_ffma with CLN.  `bench`
    (330 pairs) and `bulk` give every warpgroup chain many tiles; `mixed` has in-degrees 0 / 1 / 9 / 10 and proteins of
    1 and 2 nodes; k64 the largest tensor-core in-degree, k70 the fp32 route."""
    dev, lib = cuda_device, nat.load()
    plan, mod, lay, proj, x_in, x_orig = _edge_inputs(kind, li, 1400 + li, dev)
    if kind in ('bench', 'bulk'):
        assert (plan.N + 5) // 6 >= 3 * 132 * 4
    if kind == 'mixed':
        deg = (plan.row_ptr[1:] - plan.row_ptr[:-1]).cpu()
        assert all(int((deg == d).sum()) > 0 for d in (0, 1, 9, 10))
    aggr, xupd = _edge_fwd_ref(mod, plan, _d(proj), x_in)
    base = ETA * x_orig + (1.0 - ETA) * x_in
    runs = [('tc P=6', lib.eqd_edge_stage, 0, 1e-5), ('ffma', lib.eqd_edge_stage_ffma, 0, 1e-5)]
    if li == 1 and kind != 'k70':
        runs.append(('tc P=3', lib.eqd_edge_stage, 3, 3e-4))
    for tag, fn, products, tol in runs:
        a, xo = _edge_run(fn, plan, _desc(lay, products, eta=ETA), proj, x_in, x_orig, dev)
        rep = Report(f'edge CLN[{kind}, L{li}] {tag}', tol)
        rep.rel('aggr', a, aggr)
        rep.rel('update', xo - base, xupd)
        rep.check()


@pytest.mark.parametrize('kind,li', [('ragged', 0), ('ragged', 1), ('mixed', 0), ('mixed', 1)])
def test_edge_stage_cln_with_dropout_vs_fp64(kind, li, cuda_device):
    """The fp32 edge stage with CLN and dropout sites 0 / 1 (p = 0.25) against the fp64 stage under the same masks;
    eqd_edge_stage routes the same launch to it."""
    dev, lib = cuda_device, nat.load()
    plan, mod, lay, proj, x_in, x_orig = _edge_inputs(kind, li, 1410 + li, dev)
    layer = 2 + li
    desc = _desc(lay, drop_layer=layer, eta=ETA)
    ff = _edge_run(lib.eqd_edge_stage_ffma, plan, desc, proj, x_in, x_orig, dev)
    routed = _edge_run(lib.eqd_edge_stage, plan, desc, proj, x_in, x_orig, dev)
    assert torch.equal(routed[0], ff[0]) and torch.equal(routed[1], ff[1])
    E = plan.E
    aggr, xupd = _edge_fwd_ref(mod, plan, _d(proj), x_in, _mask(layer, 0, E, 64, dev), _mask(layer, 1, E, 64, dev))
    rep = Report(f'edge CLN dropout[{kind}, L{li}]')
    rep.rel('aggr', ff[0], aggr)
    rep.rel('update', ff[1] - (ETA * x_orig + (1.0 - ETA) * x_in), xupd)
    rep.check()


# ---- forward: node kernels with the final LayerNorm -----------------------------------------------------------------

def _node_inputs(n, seed, dev):
    r = _np_gen(seed, dev)
    h, aggr, mu = r(n, 64, s=0.7), r(n, 64, s=0.3), r(n, 64, s=0.5)
    h0 = torch.zeros(n, 72, device=dev)
    h0[:, :69] = r(n, 69)
    return h, aggr, mu, h0


@pytest.mark.parametrize('n', [1, 63, 64, 65, 264 * 64 + 4, 'bench'])
@pytest.mark.parametrize('products', [6, 3])
def test_node_mlp_tc_hln_vs_fp64(n, products, cuda_device):
    """eqd_node_mlp_tc with HLN: tile edges of the 64-row warpgroup chains, one chain running a second tile
    (264 * 64 + 4 nodes), and the bench batch's 132 000 nodes (several tiles per chain)."""
    dev, lib = cuda_device, nat.load()
    if n == 'bench':
        n = _fbatch('bench', dev)[1].N
    mod, lay, _, _ = _layer(1, dev, '0', 'LN')
    h, aggr, mu, h0 = _node_inputs(n, 1500 + n % 1000, dev)
    g = nat.EqdGraph()
    g.n_nodes = n
    desc = _desc(lay, products)

    def run():
        out = _out(n, 64, dev)
        nat.check(lib.eqd_node_mlp_tc(C.byref(g), C.byref(desc), nat.ptr(h), nat.ptr(aggr), nat.ptr(mu), nat.ptr(h0),
                                      nat.ptr(out), None), 'eqd_node_mlp_tc')
        return (out,)

    out, = _twice(run)
    _guarded('h_out', out, n)
    rep = Report(f'node_mlp_tc HLN[n={n}, P={products}]', 1e-5 if products == 6 else 3e-4)
    rep.rel('h_out', out[:n], _node_fwd_ref(mod, _d(h), _d(aggr), _d(mu), _d(h0[:, :69])))
    rep.check()


@pytest.mark.parametrize('kind', ['sizes', 'bench'])
def test_node_mlp_tc0_hln_vs_fp64(kind, cuda_device):
    """eqd_node_mlp_tc0 (layer 0, 69 wide, no skip) with HLN over the first n nodes of the batch; rows >= n stay
    untouched."""
    dev, lib = cuda_device, nat.load()
    _, plan = _fbatch(kind, dev)
    mod, lay, _, _ = _layer(0, dev, '0', 'LN')
    N = plan.N
    r = _np_gen(1510, dev)
    h0 = torch.zeros(N, 72, device=dev)
    h0[:, :69] = r(N, 69)
    aggr = r(N, 64, s=0.3)
    mu = torch.zeros(N, 72, device=dev)
    mu[:, :69] = r(N, 69, s=0.5)
    h69 = _d(h0[:, :69])
    ref = _node_fwd_ref(mod, h69, _d(aggr), _d(mu[:, :69]), h69)
    rep = Report(f'node_mlp_tc0 HLN[{kind}]')
    for n in ([1, 63, 64, 65, N] if kind == 'bench' else [N]):
        gn = nat.EqdGraph.from_buffer_copy(plan.struct)
        gn.n_nodes = n

        def run():
            out = _out(N, 64, dev)
            nat.check(lib.eqd_node_mlp_tc0(C.byref(gn), C.byref(lay.struct), nat.ptr(h0), nat.ptr(aggr), nat.ptr(mu),
                                           nat.ptr(out), None), 'eqd_node_mlp_tc0')
            return (out,)

        out, = _twice(run)
        _guarded(f'h_out n={n}', out, n)
        rep.rel(f'h_out n={n}', out[:n], ref[:n])
    rep.check()


def _next_report(rep, mod_next, h_ref, pn, kv, N):
    """proj_next (Psrc | Pdst | Q) and the next layer's K / V blocks against the projections of the fp64 h' (the
    normalised row: the pre-norm row is an O(1) error here)."""
    ref = fs.projections(mod_next, h_ref)
    rep.rel('proj_next Psrc', pn[:N, 0:64], ref['Psrc'])
    rep.rel('proj_next Pdst', pn[:N, 64:128], ref['Pdst'])
    rep.rel('proj_next Q', pn[:N, 128:192], ref['Q'])
    K, V = _decode_kv(kv, N)
    rep.rel('next K blocks', K, ref['K'])
    rep.rel('next V blocks', V, ref['V'])


@pytest.mark.parametrize('kind', ['sizes', 'bench'])
def test_node_stage_tc_hln_vs_fp64(kind, cuda_device):
    """eqd_node_stage_tc of layer 1 with p_next = layer 2, both with HLN: mu, h_out = LN_f(skip(.)) and the fused
    next-layer projections of h_out."""
    dev, lib = cuda_device, nat.load()
    _, plan = _fbatch(kind, dev)
    mod, lay, _, _ = _layer(1, dev, '0', 'LN')
    mod2, lay2, _, _ = _layer(2, dev, '0', 'LN')
    N, seg = plan.N, plan.seg_ptr_host
    G, L, Ln = C.byref(plan.struct), C.byref(lay.struct), C.byref(lay2.struct)
    r = _np_gen(1520, dev)
    h, aggr = r(N, 64, s=0.7), r(N, 64, s=0.3)
    h0 = torch.zeros(N, 72, device=dev)
    h0[:, :69] = r(N, 69)
    proj = torch.zeros(N, 320, device=dev)
    kv = torch.zeros(lib.eqd_kv_blocks_bytes(N), dtype=torch.uint8, device=dev)
    nat.check(lib.eqd_project_tc(G, L, nat.ptr(h), nat.ptr(proj), None, None), 'eqd_project_tc')    # proj K / V too
    nat.check(lib.eqd_project_tc(G, L, nat.ptr(h), nat.ptr(proj), nat.ptr(kv), None), 'eqd_project_tc')

    def run():
        kv2 = kv.clone()
        mu, h_out, pn = _out(N, 64, dev), _out(N, 64, dev), _out(N, 320, dev)
        nat.check(lib.eqd_node_stage_tc(G, L, Ln, nat.ptr(h), nat.ptr(h0), nat.ptr(proj), nat.ptr(aggr), nat.ptr(kv2),
                                        nat.ptr(mu), nat.ptr(h_out), nat.ptr(pn), None), 'eqd_node_stage_tc')
        return mu, h_out, pn, kv2

    mu, h_out, pn, kv2 = _twice(run)
    for name, t in (('mu', mu), ('h_out', h_out), ('proj_next', pn)):
        _guarded(name, t, N)
    P = _d(proj)
    mu_ref = fs.attention(seg, P[:, 128:192], P[:, 192:256], P[:, 256:320])
    h_ref = _node_fwd_ref(mod, _d(h), _d(aggr), mu_ref, _d(h0[:, :69]))
    rep = Report(f'node stage tc HLN[{kind}]')
    rep.rel('mu', mu[:N], mu_ref)
    rep.rel('h_out', h_out[:N], h_ref)
    _next_report(rep, mod2, h_ref, pn, kv2, N)
    rep.check()


@pytest.mark.parametrize('kind', ['sizes', 'bench'])
def test_node_stage_tc0_hln_vs_fp64(kind, cuda_device):
    """eqd_node_stage_tc0 of layer 0 with p_next = layer 1, both with HLN."""
    from test_gpu_forward_kernels import _l0_inputs, _project_tc0, _qkv69
    dev, lib = cuda_device, nat.load()
    _, plan = _fbatch(kind, dev)
    mod, lay, _, _ = _layer(0, dev, '0', 'LN')
    mod1, lay1, _, _ = _layer(1, dev, '0', 'LN')
    N, seg = plan.N, plan.seg_ptr_host
    h0, aggr = _l0_inputs(plan, dev, 1530)
    proj, kv, x5 = _project_tc0(plan, lay, h0, dev)
    mu_ref = fs.attention(seg, *_qkv69(proj, kv, x5, N))

    def run():
        kv2 = kv.clone()
        mu, h_out, pn = _out(N, 72, dev), _out(N, 64, dev), _out(N, 320, dev)
        nat.check(lib.eqd_node_stage_tc0(C.byref(plan.struct), C.byref(lay.struct), C.byref(lay1.struct), nat.ptr(h0),
                                         nat.ptr(proj), nat.ptr(aggr), nat.ptr(kv2), nat.ptr(x5), nat.ptr(mu),
                                         nat.ptr(h_out), nat.ptr(pn), None), 'eqd_node_stage_tc0')
        return mu, h_out, pn, kv2

    mu, h_out, pn, kv2 = _twice(run)
    for name, t in (('mu', mu), ('h_out', h_out), ('proj_next', pn)):
        _guarded(name, t, N)
    h69 = _d(h0[:, :69])
    h_ref = _node_fwd_ref(mod, h69, _d(aggr), mu_ref, h69)
    rep = Report(f'node stage tc0 HLN[{kind}]')
    rep.rel('mu', mu[:N, :69], mu_ref)
    rep.rel('h_out', h_out[:N], h_ref)
    _next_report(rep, mod1, h_ref, pn, kv2, N)
    rep.check()


@pytest.mark.parametrize('kind,li,drop', [('sizes', 0, False), ('sizes', 0, True), ('sizes', 1, False),
                                          ('sizes', 1, True), ('ragged', 0, True), ('ragged', 1, False),
                                          ('mixed', 0, False), ('mixed', 1, True)])
def test_node_stage_fp32_hln_vs_fp64(kind, li, drop, cuda_device):
    """eqd_node_stage (the fp32 node stage: training with dropout, layers without tensor-core panels) with HLN and
    p_next = the next layer: mu, h_out and all 320 columns of proj_next (Psrc | Pdst | Q | K | V of h_out)."""
    dev, lib = cuda_device, nat.load()
    _, plan = _fbatch(kind, dev)
    mod, lay, tp, _ = _layer(li, dev, '0', 'LN')
    mod_n, lay_n, _, _ = _layer(li + 1, dev, '0', 'LN')
    N, dh, dhp, seg = plan.N, tp.dh, tp.dhp, plan.seg_ptr_host
    r = _np_gen(1540 + li, dev)
    h0 = torch.zeros(N, 72, device=dev)
    h0[:, :69] = r(N, 69)
    h = h0 if li == 0 else r(N, 64)
    ldh = 72 if li == 0 else 64
    proj = r(N, tp.pw, s=0.3)
    for c0 in (128, 128 + dhp, 128 + 2 * dhp):
        proj[:, c0 + dh:c0 + dhp] = 0.0
    aggr = r(N, 64)
    layer = 1 + li
    desc = _desc(lay, drop_layer=layer if drop else None)

    def run():
        mu, h_out, pn = _out(N, dhp, dev), _out(N, 64, dev), _out(N, 320, dev)
        nat.check(lib.eqd_node_stage(C.byref(plan.struct), C.byref(desc), C.byref(lay_n.struct), nat.ptr(h), ldh,
                                     nat.ptr(h0), nat.ptr(proj), nat.ptr(aggr), nat.ptr(mu), nat.ptr(h_out),
                                     nat.ptr(pn), None), 'eqd_node_stage')
        return mu, h_out, pn

    mu, h_out, pn = _twice(run)
    for name, t in (('mu', mu), ('h_out', h_out), ('proj_next', pn)):
        _guarded(name, t, N)
    P = _d(proj)
    mu_ref = fs.attention(seg, *(P[:, c0:c0 + dh] for c0 in (128, 128 + dhp, 128 + 2 * dhp)))
    m2 = _mask(layer, 2, N, dh, dev) if drop else 1.0
    h_ref = _node_fwd_ref(mod, _d(h)[:, :dh], _d(aggr), mu_ref, _d(h0[:, :69]), m2)
    ref = fs.projections(mod_n, h_ref)
    rep = Report(f'node stage fp32 HLN[{kind}, L{li}, {"dropout" if drop else "no dropout"}]')
    rep.rel('mu', mu[:N, :dh], mu_ref)
    rep.rel('h_out', h_out[:N], h_ref)
    for name, c0 in (('Psrc', 0), ('Pdst', 64), ('Q', 128), ('K', 192), ('V', 256)):
        rep.rel(f'proj_next {name}', pn[:N, c0:c0 + 64], ref[name])
    rep.check()


# ---- backward: edge kernel with the coordinate LayerNorm ------------------------------------------------------------

@pytest.mark.parametrize('kind,li,drop,gamma_c', [('bulk', 1, False, 'seeded'), ('bulk', 0, True, 'seeded'),
                                                ('bulk', 1, True, 'zero'), ('k70', 1, False, 'seeded'),
                                                ('k70', 0, True, 'zero'), ('ragged', 0, False, 'zero'),
                                                ('ragged', 1, True, 'seeded')])
def test_bwd_edge_cln_vs_fp64_autograd(kind, li, drop, gamma_c, cuda_device):
    """eqd_bwd_edge with CLN (and dropout sites 0 / 1) against torch fp64 autograd of the edge stage.  gamma 'zero':
    gamma_c = 0, what reset_parameters leaves; then dz3 is exactly 0 and d gamma_c is the only signal moving gamma_c."""
    zero = gamma_c == 'zero'
    dev, lib = cuda_device, nat.load()
    g, plan = _batch(kind, dev)
    mod, lay, tp, eng = _layer(li, dev, 'LN', '0', zero)
    N, E, pw = plan.N, plan.E, tp.pw
    ntiles = (E + 127) // 128
    if kind == 'bulk':
        assert ntiles >= 2 * SMS
    nparts = min(ntiles, SMS)
    layer = 2 + li
    desc = _desc(lay, drop_layer=layer if drop else None)
    r = _gen(1600 + li, dev)
    proj = r(N, pw, s=0.5).contiguous()
    x_in = (_coords(g, dev) + torch.tensor(SHIFT, dtype=F64, device=dev)).contiguous()
    daggr = r(N, 64, s=0.1)
    dx_out = r(N, 3).double().contiguous()

    def run():
        outs = [_out(E, w, dev) for w in (44, 64, 64, 64, 64, 64)]
        dxrel = _out(E, 3, dev, F64)
        vec = torch.full(((SMS + GUARD) * 384,), SENT, device=dev)
        n = C.c_int32(0)
        nat.check(lib.eqd_bwd_edge(C.byref(plan.struct), C.byref(desc), nat.ptr(tp.t['w2lin']), nat.ptr(tp.t['w3lin']),
                                   nat.ptr(proj), nat.ptr(x_in), nat.ptr(daggr), nat.ptr(dx_out),
                                   *[nat.ptr(t) for t in outs], nat.ptr(dxrel), nat.ptr(vec), C.byref(n), None),
                  'eqd_bwd_edge')
        assert n.value == nparts
        return (*outs, dxrel, vec)

    res = _twice(run)
    for name, t in zip(('ein', 'n1', 'msg', 'dz3', 'dmsg', 'dz1', 'dxrel'), res[:7]):
        _guarded(name, t, E)
    ein, n1, msg, dz3, dmsg, dz1, dxrel = (t[:E] for t in res[:7])
    vec = res[7]
    assert bool((vec[nparts * 384:] == SENT).all()), 'per-CTA partial rows >= n_partials were written'
    sums = _reduce(lib, vec, nparts, 384, list(range(193)) + list(range(256, 384)), dev)
    flat = _table(lib, tp, eng, 'edgevec', vec, nparts, 384, dev)

    # fp64 autograd of the edge stage with coors_mlp.3 between LeakyReLU(z3) and coors_mlp.4
    lin1, ln, lin2 = mod.edge_mlp[0], mod.edge_mlp[3], mod.edge_mlp[4]
    lin3, lnc, lin4 = mod.coors_mlp[0], mod.coors_mlp[3], mod.coors_mlp[4]
    slope, dh = float(mod.leakyrelu_neg_slope), tp.dh
    ones = torch.ones(E, 64, dtype=F64, device=dev)
    m0, m1 = (_mask(layer, 0, E, 64, dev), _mask(layer, 1, E, 64, dev)) if drop else (ones, ones)
    src, dst = plan.col_src.long(), plan.edge_dst.long()
    deg = (plan.row_ptr[1:] - plan.row_ptr[:-1]).long()
    he = torch.cat([plan.he_l, plan.he_r]).to(F64)
    xrel = (x_in[src] - x_in[dst]).requires_grad_(True)
    d2 = (xrel ** 2).sum(1, keepdim=True)
    ein_ref = torch.cat([he, torch.cat([torch.exp(-d2 / sg) for sg in fs.SIGMAS], 1)], 1)
    w1e = _d(lin1.weight)[:, 2 * dh:]
    P = _d(proj)
    z1 = P[src, 0:64] + P[dst, 64:128] + ein_ref @ w1e.t()
    z1.retain_grad()
    gamma, beta, w4, b4 = _leaf(ln.weight), _leaf(ln.bias), _leaf(lin4.weight), _leaf(lin4.bias)
    gc, bc = _leaf(lnc.weight), _leaf(lnc.bias)
    a1 = F.leaky_relu(z1 * m0, slope)
    n1_ref = F.layer_norm(a1, (64,), gamma, beta, ln.eps)
    nhat = F.layer_norm(a1, (64,)).detach()
    msg_ref = n1_ref @ _d(lin2.weight).t() + _d(lin2.bias)
    msg_ref.retain_grad()
    z3 = msg_ref @ _d(lin3.weight).t() + _d(lin3.bias)
    z3.retain_grad()
    c3 = F.leaky_relu(z3 * m1, slope)
    c3.retain_grad()
    phi = F.layer_norm(c3, (64,), gc, bc, lnc.eps) @ w4.t() + b4
    inv = 1.0 / deg.clamp(min=1).to(F64)[:, None]
    aggr = torch.zeros(N, 64, dtype=F64, device=dev).index_add_(0, dst, msg_ref) * inv
    xupd = torch.zeros(N, 3, dtype=F64, device=dev).index_add_(0, dst, xrel * phi) * inv
    ((aggr * _d(daggr)).sum() + (xupd * dx_out).sum()).backward()

    t1 = (P[src, 0:64].abs() + P[dst, 64:128].abs() + ein_ref.detach().abs() @ w1e.abs().t()) * m0
    t3 = (msg_ref.detach().abs() @ _d(lin3.weight).abs().t() + _d(lin3.bias).abs()) * m1
    pre1, pre3 = z1.detach() * m0, z3.detach() * m1
    near3 = (pre3.abs() < KINK_BAND * t3) & (m1 != 0)
    ok = ~(_kink_kept(pre1, t1, 'z1', m0 != 0) | _kink_kept(pre3, t3, 'z3', m1 != 0))
    # A z3 element j inside the band may take the other LeakyReLU branch in the kernel.  Its value lrelu(z3) is
    # continuous there, so n-hat_c, n3 and phi move by fp32 rounding only; only the derivative changes, and dz3_j moves
    # by (1 - slope) |dc3_j m1_j| (dc3 = the coordinate LayerNorm's input gradient).  d gamma_c = sum dn3 n-hat_c and
    # d beta_c = sum dn3 take dn3 = dphi w4, which is upstream of that derivative, so they (and dw4, db4) need no
    # slack.  edge_mlp.3's d gamma / d beta take dn = dmsg . W2 with dmsg += dz3 . W3: the moved dz3_j reaches channel c
    # of dn with weight |W3 W2|[j][c] (times |n-hat_c| for d gamma), as in test_gpu_backward_kernels.py.
    rows, cols = near3.nonzero(as_tuple=True)
    mag = (1.0 - slope) * (c3.grad[rows, cols] * m1[rows, cols]).abs()
    w32 = (_d(lin3.weight) @ _d(lin2.weight)).abs()
    slack_b = (mag[:, None] * w32[cols]).sum(0)
    slack_g = (mag[:, None] * w32[cols] * nhat[rows].abs()).sum(0)

    name = f'edge CLN[{kind}, L{li}, {"dropout" if drop else "no dropout"}, gamma_c {gamma_c}]'
    rep = Report(name)
    rep.rel('ein', ein[:, :42], ein_ref.detach())
    assert float(ein[:, 42:].abs().max()) == 0.0
    rep.rel('n1', n1, n1_ref.detach())
    rep.rel('msg', msg, msg_ref.detach())
    if zero:
        assert float(dz3.abs().max()) == 0.0, 'gamma_c = 0: dz3 must be exactly 0'
    else:
        rep.rel('dz3', dz3, z3.grad, ok)
    rep.rel('dmsg', dmsg, msg_ref.grad, ok)
    rep.rel('dz1', dz1, z1.grad, ok)
    rep.rel('dxrel', dxrel, xrel.grad, ok)
    rep.rel(f'dgamma ({rows.numel()} z3 in band)', sums[0:64], gamma.grad, slack=slack_g)
    rep.rel('dbeta', sums[64:128], beta.grad, slack=slack_b)
    rep.rel('dw4', sums[128:192], w4.grad[0])
    rep.rel('db4', sums[192:193], b4.grad)
    rep.rel('dgamma_c', sums[193:257], gc.grad)
    rep.rel('dbeta_c', sums[257:321], bc.grad)
    rep.rel('table coors_mlp.3.weight', _view(eng, flat, li, 'coors_mlp.3.weight', 64), gc.grad)
    rep.rel('table coors_mlp.3.bias', _view(eng, flat, li, 'coors_mlp.3.bias', 64), bc.grad)
    rep.rel('table coors_mlp.4.weight', _view(eng, flat, li, 'coors_mlp.4.weight', 64), w4.grad[0])
    rep.rel('table coors_mlp.4.bias', _view(eng, flat, li, 'coors_mlp.4.bias', 1), b4.grad)
    rep.check()


# ---- backward: node MLP kernel with the final LayerNorm -------------------------------------------------------------

@pytest.mark.parametrize('kind,li,drop', [(k, li, d) for k in ('bulk', 'ragged') for li in (1, 0)
                                          for d in (False, True)])
def test_bwd_node_mlp_hln_vs_fp64_autograd(kind, li, drop, cuda_device):
    """eqd_bwd_node_mlp with HLN (and dropout site 2) against torch fp64 autograd of h' = LN_f(skip(node_mlp(.))): the
    input gradients, dh0 accumulated into a non-zero buffer, n5, du, the rewritten dh_out (= d/dy of the pre-norm row y)
    and the four LayerNorm affine gradients of the 272-float per-CTA partials."""
    dev, lib = cuda_device, nat.load()
    _, plan = _batch(kind, dev)
    mod, lay, tp, eng = _layer(li, dev, '0', 'LN')
    N, dh, dhp = plan.N, tp.dh, tp.dhp
    ntiles = (N + 127) // 128
    if kind == 'bulk':
        assert ntiles >= 2 * SMS
    nparts = min(ntiles, SMS)
    layer = 1 + li
    desc = _desc(lay, drop_layer=layer if drop else None)
    r = _gen(1700 + li, dev)
    pad = lambda t: torch.cat([t, torch.zeros(N, dhp - dh, device=dev)], 1).contiguous()
    h, aggr, mu = pad(r(N, dh, s=0.7)), r(N, 64, s=0.3), pad(r(N, dh, s=0.5))
    h0 = torch.cat([r(N, nat.H0), torch.zeros(N, nat.H0_PAD - nat.H0, device=dev)], 1).contiguous()
    dh_out0 = _out(N, 64, dev)
    dh_out0[:N] = r(N, 64, s=0.1)
    dh0_init = _out(N, nat.H0_PAD, dev)
    dh0_init[:N] = torch.cat([r(N, nat.H0, s=0.2), torch.zeros(N, nat.H0_PAD - nat.H0, device=dev)], 1)

    def run():
        dh_in, daggr, dmu, n5, du = (_out(N, w, dev) for w in (dhp, 64, dhp, dhp, dhp))
        dy, dh0 = dh_out0.clone(), dh0_init.clone()
        vec = torch.full(((SMS + GUARD) * 272,), SENT, device=dev)
        n = C.c_int32(0)
        nat.check(lib.eqd_bwd_node_mlp(C.byref(plan.struct), C.byref(desc), nat.ptr(tp.t['w_node1_lin']),
                                       nat.ptr(tp.t['w_node2_lin']), nat.ptr(h), dhp, nat.ptr(aggr), nat.ptr(mu), dhp,
                                       nat.ptr(h0), nat.ptr(dy), nat.ptr(dh_in), nat.ptr(daggr), nat.ptr(dmu),
                                       nat.ptr(dh0), nat.ptr(n5), nat.ptr(du), nat.ptr(vec), C.byref(n), None),
                  'eqd_bwd_node_mlp')
        assert n.value == nparts
        return dh_in, daggr, dmu, dh0, n5, du, dy, vec

    res = _twice(run)
    for name, t in zip(('dh_in', 'daggr', 'dmu', 'dh0_acc', 'n5', 'du', 'dh_out (rewritten)'), res[:7]):
        _guarded(name, t, N)
    dh_in, daggr, dmu, dh0, n5, du, dy = (t[:N] for t in res[:7])
    vec = res[7]
    assert bool((vec[nparts * 272:] == SENT).all()), 'per-CTA partial rows >= n_partials were written'
    sums = _reduce(lib, vec, nparts, 272, list(range(dh)) + [72 + c for c in range(dh)] + list(range(144, 272)), dev)
    flat = _table(lib, tp, eng, 'nodevec', vec, nparts, 272, dev)

    lin0, ln, lin4, lnf = mod.node_mlp[0], mod.node_mlp[3], mod.node_mlp[4], mod.final_h_layernorm_layer
    slope, sk = float(mod.leakyrelu_neg_slope), float(mod.skip_weight_h)
    m2 = _mask(layer, 2, N, dh, dev) if drop else torch.ones(N, dh, dtype=F64, device=dev)
    xh, xa, xm, x0 = _leaf(h[:, :dh]), _leaf(aggr), _leaf(mu[:, :dh]), _leaf(h0[:, :nat.H0])
    gamma, beta, gamma_f, beta_f = _leaf(ln.weight), _leaf(ln.bias), _leaf(lnf.weight), _leaf(lnf.bias)
    x = torch.cat([xh, xa, xm, x0], 1)
    u5 = x @ _d(lin0.weight).t() + _d(lin0.bias)
    u5.retain_grad()
    n5_ref = F.layer_norm(F.leaky_relu(u5 * m2, slope), (dh,), gamma, beta, ln.eps)
    o = n5_ref @ _d(lin4.weight).t() + _d(lin4.bias)
    y = sk * o + (1.0 - sk) * xh if dh == nat.HID else o
    y.retain_grad()
    (F.layer_norm(y, (64,), gamma_f, beta_f, lnf.eps) * _d(dh_out0[:N])).sum().backward()
    terms = (x.detach().abs() @ _d(lin0.weight).abs().t() + _d(lin0.bias).abs()) * m2
    ok = ~_kink_kept(u5.detach() * m2, terms, 'u5', m2 != 0)

    # dy, n5 and the four affine gradients are upstream of the LeakyReLU derivative: compared over every row
    rep = Report(f'node_mlp HLN[{kind}, L{li}, {"dropout" if drop else "no dropout"}]')
    rep.rel('dh_in', dh_in[:, :dh], xh.grad, ok)
    rep.rel('daggr', daggr, xa.grad, ok)
    rep.rel('dmu', dmu[:, :dh], xm.grad, ok)
    rep.rel('dh0_acc (accumulated)', dh0[:, :nat.H0], _d(dh0_init[:N, :nat.H0]) + x0.grad, ok)
    rep.rel('n5', n5[:, :dh], n5_ref.detach())
    rep.rel('du', du[:, :dh], u5.grad, ok)
    rep.rel('dh_out rewritten (dy)', dy, y.grad)
    rep.rel('dgamma', sums[:dh], gamma.grad)
    rep.rel('dbeta', sums[dh:2 * dh], beta.grad)
    rep.rel('dgamma_f', sums[2 * dh:2 * dh + 64], gamma_f.grad)
    rep.rel('dbeta_f', sums[2 * dh + 64:], beta_f.grad)
    rep.rel('table node_mlp.3.weight', _view(eng, flat, li, 'node_mlp.3.weight', dh), gamma.grad)
    rep.rel('table node_mlp.3.bias', _view(eng, flat, li, 'node_mlp.3.bias', dh), beta.grad)
    rep.rel('table final_h_layernorm_layer.weight', _view(eng, flat, li, 'final_h_layernorm_layer.weight', 64),
            gamma_f.grad)
    rep.rel('table final_h_layernorm_layer.bias', _view(eng, flat, li, 'final_h_layernorm_layer.bias', 64), beta_f.grad)
    rep.check()
    if dhp > dh:      # layer 0: channels 69..71 are padding and must come out exactly 0
        for name, t in (('dh_in', dh_in), ('dmu', dmu), ('n5', n5), ('du', du), ('dh0_acc', dh0)):
            assert float(t[:, dh:].abs().max()) == 0.0, name


# ---- graph-input gradients of models with the layer-norm options or K keypoints -------------------------------------

def _ref_forward(sd, args, inp):
    """fp64 forward of layer_norm_ref's layers under heads_ref's K-head read-out: (ligand coordinates, keypoints
    (2B,K,3), the last layer's (x, h))."""
    import heads_ref as hr
    last = []

    def layer(*a, **k):
        out = nr.layer_forward(*a, **k)
        last[:] = [out]
        return out

    saved = dm.layer_forward
    dm.layer_forward = layer
    try:
        coors, Y, _, _, _ = hr.model_forward(sd, args, inp)
    finally:
        dm.layer_forward = saved
    return coors, Y, last[0]


def _k_targets(pairs, seed, K):
    """test_gpu_input_grads._targets with K transport weights and points per protein."""
    rng = np.random.default_rng(seed + 1000)
    tg = ig._targets(pairs, seed)
    for t in tg:
        t.update({'w_l': rng.uniform(0, 1, K), 'p_l': rng.normal(0, 10, (K, 3)),
                  'w_r': rng.uniform(0, 1, K), 'p_r': rng.normal(0, 10, (K, 3))})
    return tg


@pytest.mark.parametrize('ds,cln,hln,K', [('db5', 'LN', '0', 50), ('db5', '0', 'LN', 50), ('db5', 'LN', 'LN', 50),
                                          ('dips', 'LN', '0', 50), ('dips', '0', 'LN', 50), ('dips', 'LN', 'LN', 50),
                                          ('dips', '0', '0', 25), ('dips', '0', '0', 64), ('dips', 'LN', 'LN', 25)])
def test_input_grads_with_norm_options_and_k_heads_vs_fp64(ds, cln, hln, K, cuda_device):
    """loss.backward() through the module with every graph input requiring grad (test_gpu_input_grads' probe loss plus
    its side-output term on x_iegmn_out / hv_iegmn_out) on the ragged batch of 3, x_connection_init 0.3, against fp64
    autograd of layer_norm_ref's layers and heads_ref's K-head read-out with x, mu_r_norm and he as leaves.  With the
    final LayerNorm on, the hv_iegmn_out gradient enters the last layer through eqd_bwd_node_mlp's in-place dh_out
    rewrite.  Bound: test_gpu_input_grads', times FINAL_LN_AMP with the final LayerNorm on."""
    dev = cuda_device
    args = dict(nr.args_with(ds, cln, final_h_layer_norm=hln), x_connection_init=0.3, num_att_heads=K)
    model = nr.build_model(ds, dev, args, seed=6, heads=K).train()
    pairs = _dpairs(ds, 'ragged3')
    tgts = _k_targets(pairs, 26, K)
    g = ig._graph(pairs, dev)
    ins = graph_inputs(g)
    for t in ins:
        t.requires_grad_(True)
    loss, _ = ig._engine_loss(model, g, tgts)
    loss.backward()

    plan = model.iegmn_original.last_outputs['plan']
    assert torch.equal(plan.he_l[:plan.E_l].cpu(), g.edges[LL].data['he'].detach().cpu())
    assert torch.equal(plan.he_r[:plan.E_r].cpu(), g.edges[RR].data['he'].detach().cpu())
    inp = _oracle_inputs(g, plan)
    for k in ('x', 'mu_r_norm', 'he'):
        inp[k].requires_grad_(True)
    sd = _fp64_state(model, requires_grad=True)
    coors, Y, (x_last, h_last) = _ref_forward(sd, args, inp)
    B, seg, NL = plan.n_pairs, inp['seg'], plan.N_l
    ref_loss = sum(ig._loss(coors[seg[b]:seg[b + 1]], Y[b], Y[B + b], x_last[seg[b]:seg[b + 1]],
                            h_last[seg[b]:seg[b + 1]], x_last[seg[B + b]:seg[B + b + 1]],
                            h_last[seg[B + b]:seg[B + b + 1]], tgts[b]) for b in range(B))
    ref_loss.backward()
    print(f'\ninput grads {ds} coors LN {cln} final LN {hln} K {K}: loss {loss.item():.6e} fp64 {ref_loss.item():.6e}')
    amp = FINAL_LN_AMP if hln == 'LN' else 1.0
    assert abs(loss.item() - ref_loss.item()) <= amp * 1e-3 * abs(ref_loss.item())
    xg, mg, hg = (inp[k].grad.numpy() for k in ('x', 'mu_r_norm', 'he'))
    ref_in = [xg[:NL], xg[NL:], mg[:NL], mg[NL:], hg[:plan.E_l], hg[plan.E_l:]]
    ref_p = {n: sd[n].grad.numpy() if sd[n].grad is not None else np.zeros(tuple(sd[n].shape))
             for n, _ in model.named_parameters()}
    bad = ig._report([t.grad for t in ins], ref_in, model, ref_p, amp)
    assert not bad, '\n'.join(bad)
