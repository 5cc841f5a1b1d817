"""GPU (H100): every backward entry point (csrc/bwd_*.cu and the backward half of head.cu) called directly on seeded
inputs and compared with a torch fp64 autograd of the forward formula of its stage -- independent of
oracle/backward_manual.py, except for the head, whose reference is that file's kabsch_bwd / keypoints_bwd.  The
graph-input gradient kernels (eqd_bwd_layer_inputs, eqd_bwd_inputs) are compared with their fp64 formulas; the dropout
variants of the edge and node kernels are in test_gpu_dropout_backward_kernels.py.

The tile kernels are persistent (grid = min(tiles, 132), a CTA walks tile, tile + 132, ...).  The `bulk` batch (the
ragged pairs of test_gpu_node_stage.py plus 100 pairs of 200 + 200 nodes, 41 510 nodes, 415 k edges) gives every CTA
several node, attention and edge tiles, so the second trips through the tile loops, the per-CTA partial sums that span
several tiles and long key / query chunk walks all run.  `long` is one 2000 + 150 pair: 32 key chunks on one side, 3 on
the other.  `k70` is built with 70 in-edges per node.

Tolerance: max |kernel - reference| over the compared rows, relative to the largest reference magnitude of the tensor.
One kernel on exact fp32 inputs shows only fp32 rounding, and the bound is 1e-5 for every tensor except the attention
gradients with sharpened logits (4e-5, justified in that test).  Measured on an H100 80GB HBM3 (largest value over the
cases of each test):
  node MLP   dh_in 4.8e-7, daggr 4.3e-7, dmu 5.9e-7, dh0_acc 3.4e-7, n5 1.2e-6, du 5.1e-7, dgamma 4.2e-7, dbeta 3.5e-7
  attention  dQpre 1.3e-6, dKpre 1.6e-6, dV 1.5e-6; sharpened logits: dQpre 1.6e-5, dKpre 5.1e-6, dV 1.5e-6
  edge       ein 5.9e-9, n1 4.3e-7, msg 1.0e-6, dz3 8.0e-8, dmsg 5.3e-7, dz1 5.2e-7, dxrel 1.6e-7,
             dgamma 1.5e-7, dbeta 3.4e-7, dw4 5.3e-7, db4 4.6e-7
  gather     dPsrc 3.6e-7, dPdst 2.9e-7, dx 2.8e-9;  project dh 1.9e-7;  embed demb 5.2e-7;  head dh 3.0e-7, dx 2.5e-7
  inputs     layer inputs dhe 1.1e-7 (dx_orig exact);  d mu_r_norm within 1.47 fp32 ulp, dx 7.0e-17 (700 W power limit)
(the printed report of `pytest -s` lists every value).

The graph-input gradient kernels have their own bounds: eqd_bwd_layer_inputs' dhe 1e-5, its dx_orig += eta dx_out exact
(one fp64 rounding, or none through an FMA); eqd_bwd_inputs' d mu_r_norm within 2 fp32 ulp (a sum and a quotient in
fp32) and its dx within 1e-14 (products of fp32 values are exact in fp64, leaving three fp64 additions).

The LeakyReLU kink: the kernels recompute z1, z3 (edge) and u5 (node) in fp32.  Where an fp64 pre-activation lies
within the fp32 error of its dot product of 0, the kernel may take the other branch and its derivative differs by
(1 - slope) x the upstream gradient.  Rows with a pre-activation |z| < 32 * 2^-24 * (sum of |terms| of z) are left out
of the per-row comparisons that depend on that branch; at most 0.5 % of the rows may be left out (measured: u5 up to
2.6e-3, 4 of 1510 rows of layer 0; z1 and z3 up to 3.3e-4).  The per-CTA LayerNorm sums of the edge kernel include
those rows, so their bound adds the most the flagged z3 elements can change them by.

Every kernel is also run twice on the same inputs: the outputs must be bitwise equal (no float atomics, fixed
reduction order, DESIGN.md section 4.2).
"""
import ctypes as C
import hashlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import backward_manual as bm
import fp64_stages as fs
import golden_io as gio
import iegmn_oracle as orc
from equidock_public_b200 import _native as nat
from equidock_public_b200 import synthetic
from equidock_public_b200.engine import GraphPlan
from equidock_public_b200.training import BackwardWorkspace, TrainEngine, tn_gemm_shapes
from test_gpu_node_stage import RAGGED

pytestmark = pytest.mark.gpu

F64 = torch.float64
SMS = 132
TOL = 1e-5
KINK_BAND = 32 * 2.0 ** -24      # times the sum of |terms| of a pre-activation
KINK_MAX_FRACTION = 5e-3         # of the rows of a batch
SIGMAS = [1.5 ** s for s in range(nat.N_RBF)]

_CACHE = {}


def _pairs(kind):
    if kind == 'bulk':
        rng = np.random.default_rng(31)
        return [synthetic.synthetic_pair(rng, a, b, 10) for a, b in RAGGED] + synthetic.synthetic_batch(100, seed=32)
    if kind == 'ragged':
        rng = np.random.default_rng(33)
        return [synthetic.synthetic_pair(rng, a, b, 10) for a, b in RAGGED]
    if kind == 'long':
        return [synthetic.synthetic_pair(np.random.default_rng(34), 2000, 150, 10)]
    if kind == 'k70':
        rng = np.random.default_rng(35)
        return [synthetic.synthetic_pair(rng, 300, 250, 70), synthetic.synthetic_pair(rng, 75, 110, 70),
                synthetic.synthetic_pair(rng, 1, 90, 70)]
    if kind == 'train':           # exactly 100 pairs of 200 + 200 nodes, ten in-edges per node: N = 40 000, E = 400 000
        return synthetic.synthetic_batch(100, seed=36)
    raise ValueError(kind)


def _batch(kind, dev):
    """(graph, plan) of a named batch, built once per session."""
    if kind not in _CACHE:
        g = gio.make_batch(_pairs(kind), dev)
        _CACHE[kind] = (g, GraphPlan.from_graph(g, dev, 70 if kind == 'k70' else 10))
    return _CACHE[kind]


def _model(dev):
    if 'model' not in _CACHE:
        model = gio.build_model('dips', dev)
        _CACHE['model'] = (model, TrainEngine(model))
    return _CACHE['model']


def _layer(li, dev):
    model, eng = _model(dev)
    mod = model.iegmn_original.iegmn_layers[li]
    return mod, mod.packed(dev), eng.layer_pack(mod)


def _gen(seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    return lambda *shape, s=1.0: torch.randn(*shape, generator=g, device=dev) * s


def _d(t):
    return t.detach().to(F64)


def _leaf(t):
    return _d(t).clone().requires_grad_(True)


class Report:
    """Relative errors of one test, printed, and asserted together so that one run shows every tensor's error."""

    def __init__(self, name, tol=TOL):
        self.name, self.rows, self.tol = name, [], tol

    def rel(self, tag, got, ref, rows=None, slack=None):
        """max |got - ref| (over `rows`, less an elementwise `slack`) / max |ref|."""
        got, ref = _d(got), _d(ref)
        assert torch.isfinite(got).all(), f'{self.name} {tag}: non-finite values'
        diff = (got - ref).abs()
        if slack is not None:
            diff = (diff - slack).clamp(min=0.0)
        if rows is not None:
            diff = diff[rows]
        err = float(diff.max()) / max(float(ref.abs().max()), 1e-30) if diff.numel() else 0.0
        self.rows.append((tag, err))

    def check(self):
        lines = [f'{"ok " if e <= self.tol else "BAD"} {self.name} {tag:28s} {e:.2e}' for tag, e in self.rows]
        print('\n' + '\n'.join(lines))
        bad = [ln for ln in lines if ln.startswith('BAD')]
        assert not bad, '\n'.join(bad)


def _twice(run):
    """Runs a kernel launch twice on the same inputs; the outputs must be bitwise equal.  Returns the first outputs."""
    a = run()
    b = run()
    torch.cuda.synchronize()
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), f'output {i} differs between two runs on the same inputs'
    return a


def _kink_rows(pre, terms, what):
    """Rows with an fp64 pre-activation closer to 0 than the fp32 error bound of its dot product."""
    near = (pre.abs() < KINK_BAND * terms).any(1)
    frac = float(near.double().mean())
    print(f'\n{what}: {int(near.sum())} of {near.numel()} rows ({frac:.1e}) within the kink band')
    assert frac <= KINK_MAX_FRACTION, f'{what}: {frac:.2e} of the rows lie within the kink band'
    return near


def _reduce(lib, vec, nparts, stride, src, dev):
    src_t = torch.tensor(src, dtype=torch.int32, device=dev)
    dst_t = torch.arange(len(src), dtype=torch.int32, device=dev)
    out = torch.zeros(len(src), device=dev)
    nat.check(lib.eqd_grad_reduce(nat.ptr(vec), nparts, stride, nat.ptr(src_t), nat.ptr(dst_t), len(src), nat.ptr(out),
                                  None), 'eqd_grad_reduce')
    return out


# ---- node MLP -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('kind,li', [('bulk', 1), ('bulk', 0), ('ragged', 1), ('ragged', 0)])
def test_bwd_node_mlp_vs_fp64_autograd(kind, li, cuda_device):
    dev, lib = cuda_device, nat.load()
    _, plan = _batch(kind, dev)
    mod, lay, tp = _layer(li, dev)
    N, dh, dhp = plan.N, tp.dh, tp.dhp
    ntiles = (N + 127) // 128
    if kind == 'bulk':
        assert ntiles >= 2 * SMS
    r = _gen(100 + li, dev)
    pad = lambda t: torch.cat([t, torch.zeros(N, dhp - dh, device=dev)], 1).contiguous()
    h, aggr, mu = pad(r(N, dh, s=0.7)), r(N, 64, s=0.3), pad(r(N, dh, s=0.5))
    h0 = torch.cat([r(N, nat.H0), torch.zeros(N, nat.H0_PAD - nat.H0, device=dev)], 1).contiguous()
    dh_out = r(N, 64, s=0.1)
    dh0_init = torch.cat([r(N, nat.H0, s=0.2), torch.zeros(N, nat.H0_PAD - nat.H0, device=dev)], 1).contiguous()

    def run():
        outs = [torch.full((N, w), float('nan'), device=dev) for w in (dhp, 64, dhp, dhp, dhp)]
        dh_in, daggr, dmu, n5, du = outs
        dh0 = dh0_init.clone()
        vec = torch.full((SMS * 144,), float('nan'), device=dev)
        nparts = C.c_int32(0)
        nat.check(lib.eqd_bwd_node_mlp(C.byref(plan.struct), C.byref(lay.struct), nat.ptr(tp.t['w_node1_lin']),
                                       nat.ptr(tp.t['w_node2_lin']), nat.ptr(h), dhp, nat.ptr(aggr), nat.ptr(mu), dhp,
                                       nat.ptr(h0), nat.ptr(dh_out), nat.ptr(dh_in), nat.ptr(daggr), nat.ptr(dmu),
                                       nat.ptr(dh0), nat.ptr(n5), nat.ptr(du), nat.ptr(vec), C.byref(nparts), None),
                  'eqd_bwd_node_mlp')
        assert nparts.value == min(ntiles, SMS)
        gb = _reduce(lib, vec, nparts.value, 144, list(range(dh)) + [72 + c for c in range(dh)], dev)
        return dh_in, daggr, dmu, dh0, n5, du, gb

    dh_in, daggr, dmu, dh0, n5, du, gb = _twice(run)

    # fp64 autograd of node_mlp (:319-337)
    lin0, ln, lin4 = mod.node_mlp[0], mod.node_mlp[3], mod.node_mlp[4]
    slope, sk = float(mod.leakyrelu_neg_slope), float(mod.skip_weight_h)
    xh, xa, xm, x0 = _leaf(h[:, :dh]), _leaf(aggr), _leaf(mu[:, :dh]), _leaf(h0[:, :nat.H0])
    gamma, beta = _leaf(ln.weight), _leaf(ln.bias)
    x = torch.cat([xh, xa, xm, x0], 1)
    u5 = x @ _d(lin0.weight).t() + _d(lin0.bias)
    u5.retain_grad()
    n5_ref = F.layer_norm(F.leaky_relu(u5, slope), (dh,), gamma, beta, ln.eps)
    o = n5_ref @ _d(lin4.weight).t() + _d(lin4.bias)
    out = sk * o + (1.0 - sk) * xh if dh == nat.HID else o
    (out * _d(dh_out)).sum().backward()
    terms = x.detach().abs() @ _d(lin0.weight).abs().t() + _d(lin0.bias).abs()
    ok = ~_kink_rows(u5.detach(), terms, 'u5')

    rep = Report(f'node_mlp[{kind}, L{li}]')
    rep.rel('dh_in', dh_in[:, :dh], xh.grad, ok)
    rep.rel('daggr', daggr, xa.grad, ok)
    rep.rel('dmu', dmu[:, :dh], xm.grad, ok)
    rep.rel('dh0_acc (accumulated)', dh0[:, :nat.H0], _d(dh0_init[:, :nat.H0]) + x0.grad, ok)
    rep.rel('n5', n5[:, :dh], n5_ref.detach())
    rep.rel('du', du[:, :dh], u5.grad, ok)
    rep.rel('dgamma', gb[:dh], gamma.grad)
    rep.rel('dbeta', gb[dh:], beta.grad)
    rep.check()
    if dhp > dh:      # layer 0: channels 69..71 are padding and must come out exactly 0
        for name, t in (('dh_in', dh_in), ('dmu', dmu), ('n5', n5), ('du', du), ('dh0_acc', dh0)):
            assert float(t[:, dh:].abs().max()) == 0.0, name


# ---- cross attention ----------------------------------------------------------------------------------------------

def _attn_inputs(plan, dhp, dh, slope, qk_scale, seed, dev):
    """proj with post-activation Q, K (LeakyReLU of N(0, qk_scale^2) pre-activations), V, padding columns 0."""
    N, pw = plan.N, 128 + 3 * dhp
    r = _gen(seed, dev)
    proj = r(N, pw)
    for base, act in ((128, True), (128 + dhp, True), (128 + 2 * dhp, False)):
        blk = r(N, dh, s=qk_scale if act else 0.5)
        proj[:, base:base + dh] = F.leaky_relu(blk, slope) if act else blk
        proj[:, base + dh:base + dhp] = 0.0
    dmu = torch.zeros(N, dhp, device=dev)
    dmu[:, :dh] = r(N, dh, s=0.1)
    return proj.contiguous(), dmu


@pytest.mark.parametrize('kind,li,qk_scale', [('bulk', 1, 0.3), ('bulk', 0, 0.3), ('ragged', 1, 0.3), ('ragged', 0, 0.3),
                                              ('long', 1, 0.3), ('long', 0, 0.3), ('ragged', 1, 1.5), ('long', 0, 1.5)])
def test_bwd_attention_vs_fp64_autograd(kind, li, qk_scale, cuda_device):
    """qk_scale = 1.5: logits with a standard deviation of about 18, so most softmax rows saturate on one key.  Their
    bound is 4e-5: the kernels recompute logits of up to |s| ~ 70 in fp32, whose rounding (|s| 2^-24 ~ 4e-6) moves P by
    that much relative, and dS = P (dP - D) cancels in a saturated row, where D ~ dP of the dominant key."""
    dev, lib = cuda_device, nat.load()
    _, plan = _batch(kind, dev)
    mod, lay, tp = _layer(li, dev)
    N, dh, dhp = plan.N, tp.dh, tp.dhp
    pw = 128 + 3 * dhp
    if kind == 'bulk':
        assert plan.n_node_tiles >= 2 * SMS
    slope = float(mod.leakyrelu_neg_slope)
    proj, dmu = _attn_inputs(plan, dhp, dh, slope, qk_scale, 200 + li, dev)
    Q, K, V = (_d(proj[:, b:b + dh]) for b in (128, 128 + dhp, 128 + 2 * dhp))
    # pre-activations that LeakyReLU maps back onto the given Q, K: the kernels see the same branch as the reference
    qpre = torch.where(Q > 0, Q, Q / slope).requires_grad_(True)
    kpre = torch.where(K > 0, K, K / slope).requires_grad_(True)
    v = V.clone().requires_grad_(True)
    q, k = F.leaky_relu(qpre, slope), F.leaky_relu(kpre, slope)
    mu_ref = fs.attention(plan.seg_ptr_host, q, k, v)
    (mu_ref * _d(dmu[:, :dh])).sum().backward()
    mu = torch.zeros(N, dhp, device=dev)
    mu[:, :dh] = mu_ref.detach().float()           # the stashed forward output, rounded to fp32
    sentinel = 1234.5

    def run():
        dP = torch.full((N, pw), sentinel, device=dev)
        rowstat = torch.empty(N, 4, device=dev)
        nat.check(lib.eqd_bwd_attention(C.byref(plan.struct), C.byref(lay.struct), nat.ptr(proj), nat.ptr(mu), dhp,
                                        nat.ptr(dmu), nat.ptr(dP), nat.ptr(rowstat), None), 'eqd_bwd_attention')
        return (dP,)

    dP, = _twice(run)
    assert bool((dP[:, :128] == sentinel).all()), 'dP[:, 0:128] (dPsrc | dPdst) must be left untouched'
    rep = Report(f'attention[{kind}, L{li}, qk x{qk_scale}]', TOL if qk_scale < 1 else 4e-5)
    rep.rel('dQpre', dP[:, 128:128 + dh], qpre.grad)
    rep.rel('dKpre', dP[:, 128 + dhp:128 + dhp + dh], kpre.grad)
    rep.rel('dV', dP[:, 128 + 2 * dhp:128 + 2 * dhp + dh], v.grad)
    rep.check()
    if dhp > dh:      # layer 0: channels 69..71 of dQpre, dKpre and dV are padding
        for base in (128, 128 + dhp, 128 + 2 * dhp):
            assert float(dP[:, base + dh:base + dhp].abs().max()) == 0.0


# ---- edge stage ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('kind,li', [('bulk', 1), ('k70', 1), ('ragged', 0)])
def test_bwd_edge_vs_fp64_autograd(kind, li, cuda_device):
    """Coordinates around 1e3 A (the range layer-evolved coordinates reach).  The bulk and ragged batches have edge tiles
    that straddle n_lig_edges, a short last tile and nodes without in-edges (proteins of 1 node)."""
    dev, lib = cuda_device, nat.load()
    _, plan = _batch(kind, dev)
    mod, lay, tp = _layer(li, dev)
    N, E, dhp = plan.N, plan.E, tp.dhp
    pw = 128 + 3 * dhp
    ntiles = (E + 127) // 128
    assert E % 128 != 0 and plan.E_l % 128 != 0
    if kind == 'bulk':
        assert ntiles >= 2 * SMS
    deg = (plan.row_ptr[1:] - plan.row_ptr[:-1]).long()
    if kind != 'k70':
        assert int((deg == 0).sum()) > 0
    else:
        assert int(deg.max()) == 70
    r = _gen(300 + li, dev)
    proj = r(N, pw, s=0.5).contiguous()
    g, _ = _batch(kind, dev)
    from equidock_public_b200.hetero_graph import LIGAND, RECEPTOR
    x = torch.cat([g.nodes[LIGAND].data['new_x'], g.nodes[RECEPTOR].data['x']]).to(dev, F64)
    x_in = (x + torch.tensor([1.0e3, -0.7e3, 0.4e3], dtype=F64, device=dev)).contiguous()
    daggr = r(N, 64, s=0.1)
    dx_out = r(N, 3).double().contiguous()

    def run():
        outs = [torch.full((E, w), float('nan'), device=dev) for w in (44, 64, 64, 64, 64, 64)]
        dxrel = torch.full((E, 3), float('nan'), dtype=F64, device=dev)
        vec = torch.full((SMS * 256,), float('nan'), device=dev)
        nparts = C.c_int32(0)
        nat.check(lib.eqd_bwd_edge(C.byref(plan.struct), C.byref(lay.struct), nat.ptr(tp.t['w2lin']), nat.ptr(tp.t['w3lin']),
                                   nat.ptr(proj), nat.ptr(x_in), nat.ptr(daggr), nat.ptr(dx_out),
                                   *[nat.ptr(t) for t in outs], nat.ptr(dxrel), nat.ptr(vec), C.byref(nparts), None),
                  'eqd_bwd_edge')
        assert nparts.value == min(ntiles, SMS)
        sums = _reduce(lib, vec, nparts.value, 256, list(range(193)), dev)
        return (*outs, dxrel, sums)

    ein, n1, msg, dz3, dmsg, dz1, dxrel, sums = _twice(run)
    ref = _bwd_edge_ref(mod, plan, proj, x_in, daggr, dx_out)
    _bwd_edge_report(Report(f'edge[{kind}, L{li}]'), ref, ein, n1, msg, dz3, dmsg, dz1, dxrel, sums).check()


def _bwd_edge_ref(mod, plan, proj, x_in, daggr, dx_out, m0=None, m1=None):
    """fp64 autograd of the edge stage (:204-237, 263-292), with the dropout factors m0 / m1 [E][64] (site 0 on z1,
    site 1 on z3) when given.  Returns the reference tensors, the rows outside the LeakyReLU kink band (`ok`) and the
    slack of d gamma / d beta for the z3 elements inside it."""
    lin1, ln, lin2 = mod.edge_mlp[0], mod.edge_mlp[3], mod.edge_mlp[4]
    lin3, lin4 = mod.coors_mlp[0], mod.coors_mlp[4]
    slope, dh = float(mod.leakyrelu_neg_slope), int(mod.att_mlp_Q[0].weight.shape[0])
    N, E, dev = plan.N, plan.E, x_in.device
    ones = torch.ones(E, 64, dtype=F64, device=dev)
    m0 = ones if m0 is None else m0
    m1 = ones if m1 is None else m1
    src, dst = plan.col_src.long(), plan.edge_dst.long()
    deg = (plan.row_ptr[1:] - plan.row_ptr[:-1]).long()
    he = torch.cat([plan.he_l, plan.he_r]).to(F64)
    xrel = (x_in[src] - x_in[dst]).requires_grad_(True)
    d2 = (xrel ** 2).sum(1, keepdim=True)
    rbf = torch.cat([torch.exp(-d2 / sg) for sg in SIGMAS], 1)
    ein_ref = torch.cat([he, rbf], 1)
    w1e = _d(lin1.weight)[:, 2 * dh:]
    P = _d(proj)
    z1 = P[src, 0:64] + P[dst, 64:128] + ein_ref @ w1e.t()
    gamma, beta, w4, b4 = _leaf(ln.weight), _leaf(ln.bias), _leaf(lin4.weight), _leaf(lin4.bias)
    z1.retain_grad()
    a1 = F.leaky_relu(z1 * m0, slope)
    n1_ref = F.layer_norm(a1, (64,), gamma, beta, ln.eps)
    nhat = F.layer_norm(a1, (64,)).detach()
    msg_ref = n1_ref @ _d(lin2.weight).t() + _d(lin2.bias)
    msg_ref.retain_grad()
    z3 = msg_ref @ _d(lin3.weight).t() + _d(lin3.bias)
    z3.retain_grad()
    c3 = F.leaky_relu(z3 * m1, slope)
    c3.retain_grad()
    phi = c3 @ w4.t() + b4
    inv = 1.0 / deg.clamp(min=1).to(F64)[:, None]
    aggr = torch.zeros(N, 64, dtype=F64, device=dev).index_add_(0, dst, msg_ref) * inv
    xupd = torch.zeros(N, 3, dtype=F64, device=dev).index_add_(0, dst, xrel * phi) * inv
    ((aggr * _d(daggr)).sum() + (xupd * dx_out).sum()).backward()

    # the kink test over the elements the masks keep (a dropped element enters the LeakyReLU as an exact 0)
    t1 = (P[src, 0:64].abs() + P[dst, 64:128].abs() + ein_ref.detach().abs() @ w1e.abs().t()) * m0
    t3 = (msg_ref.detach().abs() @ _d(lin3.weight).abs().t() + _d(lin3.bias).abs()) * m1
    pre1, pre3 = z1.detach() * m0, z3.detach() * m1
    near3 = (pre3.abs() < KINK_BAND * t3) & (m1 != 0)
    ok = ~(_kink_rows(torch.where(m0 != 0, pre1, torch.inf), t1, 'z1')
           | _kink_rows(torch.where(m1 != 0, pre3, torch.inf), t3, 'z3'))
    # dgamma / dbeta sum over every edge: a z3 element inside the band can move them by (1 - slope) |dc3_j m1_j| (dc3 =
    # the gradient w.r.t. LeakyReLU(z3 m1) = dphi w4_j) times row j of |W3 W2| (times |n-hat| for dgamma)
    rows, cols = near3.nonzero(as_tuple=True)
    mag = (1.0 - slope) * (c3.grad[rows, cols] * m1[rows, cols]).abs()
    w32 = (_d(lin3.weight) @ _d(lin2.weight)).abs()               # [j][c]: dn_c per unit dz3_j
    return {'ein': ein_ref.detach(), 'n1': n1_ref.detach(), 'msg': msg_ref.detach(), 'dz3': z3.grad,
            'dmsg': msg_ref.grad, 'dz1': z1.grad, 'dxrel': xrel.grad, 'dgamma': gamma.grad, 'dbeta': beta.grad,
            'dw4': w4.grad[0], 'db4': b4.grad, 'ok': ok, 'n_band3': rows.numel(),
            'slack_b': (mag[:, None] * w32[cols]).sum(0), 'slack_g': (mag[:, None] * w32[cols] * nhat[rows].abs()).sum(0)}


def _bwd_edge_report(rep, ref, ein, n1, msg, dz3, dmsg, dz1, dxrel, sums):
    """eqd_bwd_edge's per-edge outputs and its reduced 193 per-CTA sums against _bwd_edge_ref."""
    ok = ref['ok']
    rep.rel('ein', ein[:, :42], ref['ein'])
    assert float(ein[:, 42:].abs().max()) == 0.0
    rep.rel('n1', n1, ref['n1'])
    rep.rel('msg', msg, ref['msg'])
    rep.rel('dz3', dz3, ref['dz3'], ok)
    rep.rel('dmsg', dmsg, ref['dmsg'], ok)
    rep.rel('dz1', dz1, ref['dz1'], ok)
    rep.rel('dxrel', dxrel, ref['dxrel'], ok)
    rep.rel(f'dgamma ({ref["n_band3"]} z3 in band)', sums[0:64], ref['dgamma'], slack=ref['slack_g'])
    rep.rel('dbeta', sums[64:128], ref['dbeta'], slack=ref['slack_b'])
    rep.rel('dw4', sums[128:192], ref['dw4'])
    rep.rel('db4', sums[192:193], ref['db4'])
    return rep

# ---- gather, projections, embedding -------------------------------------------------------------------------------

@pytest.mark.parametrize('kind', ['bulk', 'k70'])
def test_bwd_edge_gather_vs_fp64_autograd(kind, cuda_device):
    dev, lib = cuda_device, nat.load()
    _, plan = _batch(kind, dev)
    ws = BackwardWorkspace(plan, dev)            # the by-source edge order of the training backward
    N, E, pw = plan.N, plan.E, 344
    eta = 0.3
    r = _gen(400, dev)
    dz1, dxrel, dx_out = r(E, 64), r(E, 3).double(), r(N, 3).double()
    sentinel = -777.25

    def run():
        dP = torch.full((N, pw), sentinel, device=dev)
        dx = torch.full((N, 3), float('nan'), dtype=F64, device=dev)
        nat.check(lib.eqd_bwd_edge_gather(C.byref(plan.struct), nat.ptr(ws.out_ptr), nat.ptr(ws.out_edge), nat.ptr(dz1),
                                          nat.ptr(dxrel), nat.ptr(dx_out), eta, nat.ptr(dP), pw, nat.ptr(dx), None),
                  'eqd_bwd_edge_gather')
        return dP, dx

    dP, dx = _twice(run)
    src, dst = plan.col_src.long(), plan.edge_dst.long()
    psrc, pdst = torch.zeros(N, 64, dtype=F64, device=dev, requires_grad=True), torch.zeros(N, 64, dtype=F64, device=dev,
                                                                                            requires_grad=True)
    x = torch.zeros(N, 3, dtype=F64, device=dev, requires_grad=True)
    z1 = psrc[src] + pdst[dst]
    xrel = x[src] - x[dst]
    ((z1 * _d(dz1)).sum() + (xrel * dxrel).sum() + ((1.0 - eta) * x * dx_out).sum()).backward()
    assert bool((dP[:, 128:] == sentinel).all()), 'dP[:, 128:] must be left untouched'
    rep = Report(f'gather[{kind}]')
    rep.rel('dPsrc', dP[:, 0:64], psrc.grad)
    rep.rel('dPdst', dP[:, 64:128], pdst.grad)
    rep.rel('dx', dx, x.grad)
    rep.check()


@pytest.mark.parametrize('li', [1, 0])
def test_bwd_project_vs_fp64_autograd(li, cuda_device):
    """dh += dP . Wproj^T, accumulated into a non-zero dh; layer 0's padding columns 69..71 stay exactly 0 even when
    the padding columns of dP are not zero."""
    dev, lib = cuda_device, nat.load()
    _, plan = _batch('bulk', dev)
    mod, lay, tp = _layer(li, dev)
    N, dh, dhp = plan.N, tp.dh, tp.dhp
    pw = 128 + 3 * dhp
    r = _gen(500 + li, dev)
    dP = r(N, pw, s=0.1)
    dh_init = r(N, dhp)
    dh_init[:, dh:] = 0.0

    def run():
        out = dh_init.clone()
        nat.check(lib.eqd_bwd_project(C.byref(plan.struct), C.byref(lay.struct), nat.ptr(tp.t['w_projT']), nat.ptr(dP),
                                      nat.ptr(out), None), 'eqd_bwd_project')
        return (out,)

    out, = _twice(run)
    h = torch.zeros(N, dh, dtype=F64, device=dev, requires_grad=True)
    w1 = _d(mod.edge_mlp[0].weight)
    groups = [(0, h @ w1[:, :dh].t()), (64, h @ w1[:, dh:2 * dh].t()), (128, h @ _d(mod.att_mlp_Q[0].weight).t()),
              (128 + dhp, h @ _d(mod.att_mlp_K[0].weight).t()), (128 + 2 * dhp, h @ _d(mod.att_mlp_V[0].weight).t())]
    sum((y * _d(dP[:, b:b + y.shape[1]])).sum() for b, y in groups).backward()
    rep = Report(f'project[L{li}]')
    rep.rel('dh (accumulated)', out[:, :dh], _d(dh_init[:, :dh]) + h.grad)
    rep.check()
    if dhp > dh:
        assert float(out[:, dh:].abs().max()) == 0.0


def test_bwd_embed_vs_fp64(cuda_device):
    """All 21 residue types over the bulk batch, accumulated into a non-zero demb."""
    dev, lib = cuda_device, nat.load()
    _, plan = _batch('bulk', dev)
    N, NL = plan.N, plan.N_l
    g = torch.Generator(device=dev).manual_seed(600)
    res = torch.randint(0, nat.N_RES_TYPES, (N,), generator=g, device=dev)
    assert res.unique().numel() == nat.N_RES_TYPES
    res_f = res.float()
    res_l, res_r = res_f[:NL].contiguous(), res_f[NL:].contiguous()
    r = _gen(601, dev)
    dh0, dhl0, demb0 = r(N, nat.H0_PAD), r(N, nat.H0_PAD), r(nat.N_RES_TYPES, 64)

    def run():
        out = demb0.clone()
        nat.check(lib.eqd_bwd_embed(C.byref(plan.struct), nat.ptr(res_l), nat.ptr(res_r), nat.ptr(dh0), nat.ptr(dhl0),
                                    nat.ptr(out), None), 'eqd_bwd_embed')
        return (out,)

    out, = _twice(run)
    emb = torch.zeros(nat.N_RES_TYPES, 64, dtype=F64, device=dev, requires_grad=True)
    ((emb[res] * (_d(dh0) + _d(dhl0))[:, :64]).sum()).backward()
    rep = Report('embed[bulk]')
    rep.rel('demb (accumulated)', out, _d(demb0) + emb.grad)
    rep.check()


# ---- graph-input gradients ----------------------------------------------------------------------------------------

def _fma_or_two_roundings(got, a, b, c):
    """True where got == fl(a + fl(b c)) or == fma(b, c, a) (the compiler may contract the update), in fp64."""
    got, a, b, c = (t.cpu().numpy().ravel() for t in (got, a, b, c))
    ok = got == a + b * c
    from fractions import Fraction
    for i in np.flatnonzero(~ok):
        ok[i] = float(got[i]) == float(Fraction(float(a[i])) + Fraction(float(b[i])) * Fraction(float(c[i])))
    return bool(ok.all())


@pytest.mark.parametrize('li,eta', [(1, 0.0), (1, 0.3), (0, 0.0), (0, 0.3)])
def test_bwd_layer_inputs_vs_fp64(li, eta, cuda_device):
    """eqd_bwd_layer_inputs on the bulk batch: dhe += dz1 . W1[:, 2 dh : 2 dh + 27]^T (edge_mlp.0.weight's he block,
    69 + 69 columns in front of it in layer 0), accumulated into a non-zero dhe, and dx_orig += eta dx_out, exact (eta =
    0: bitwise unchanged).  The grid is min(max(edge tiles, 3N / 128), 4 x 132) = 528 CTAs: each walks about 6 edge
    tiles (the last one short) and takes two passes over the 3N coordinates."""
    dev, lib = cuda_device, nat.load()
    _, plan = _batch('bulk', dev)
    mod, lay, _ = _layer(li, dev)
    N, E, dh = plan.N, plan.E, int(mod.att_mlp_Q[0].weight.shape[0])
    grid = min(max((E + 127) // 128, (3 * N + 127) // 128), 4 * SMS)
    assert (E + 127) // 128 >= 2 * grid and 3 * N > grid * 128 and E % 128 != 0
    desc = nat.EqdLayer.from_buffer_copy(lay.struct)
    desc.dev.x_connection_init = eta
    eta32 = float(np.float32(eta))
    r = _gen(650 + li, dev)
    dz1 = r(E, 64, s=0.1)
    dx_out = r(N, 3).double()
    dhe0, dxo0 = r(E + 3, 27), r(N + 1, 3).double()
    sentinel = -777.25
    dhe0[E:], dxo0[N:] = sentinel, sentinel

    def run():
        dhe, dxo = dhe0.clone(), dxo0.clone()
        nat.check(lib.eqd_bwd_layer_inputs(C.byref(plan.struct), C.byref(desc), nat.ptr(dz1), nat.ptr(dx_out),
                                           nat.ptr(dhe), nat.ptr(dxo), None), 'eqd_bwd_layer_inputs')
        return dhe, dxo

    dhe, dxo = _twice(run)
    assert bool((dhe[E:] == sentinel).all()) and bool((dxo[N:] == sentinel).all()), 'rows past the end were written'
    w_he = _d(mod.edge_mlp[0].weight)[:, 2 * dh:2 * dh + 27]
    rep = Report(f'layer inputs[bulk, L{li}, eta {eta}]')
    rep.rel('dhe (accumulated)', dhe[:E], _d(dhe0[:E]) + _d(dz1) @ w_he)
    rep.check()
    if eta == 0.0:
        assert torch.equal(dxo, dxo0), 'eta = 0: dx_orig must be bitwise unchanged'
    else:
        assert _fma_or_two_roundings(dxo[:N], dxo0[:N], torch.full_like(dx_out, eta32), dx_out), \
            'dx_orig += eta dx_out is not exact'


def _pair_of_node(n_lig):
    """[N_l] pair index of every ligand node (ligands in pair order, n_lig[b] nodes each)."""
    return torch.repeat_interleave(torch.arange(len(n_lig)), torch.tensor(n_lig))


@pytest.mark.parametrize('kind,with_dcoors', [('bench', True), ('bench', False), ('ragged', True), ('ragged', False)])
def test_bwd_inputs_vs_fp64(kind, with_dcoors, cuda_device):
    """eqd_bwd_inputs (one thread per node, each ligand node finding its pair by a binary search over seg_ptr): on the
    bench batch's 330 ligands and the ragged batch's ligands of 1 .. 200 nodes, with a distinct rotation per pair.
    d mu_r_norm = (dh0_acc + dh_layer0)[64:69] / mu_r_norm within 2 fp32 ulp; dx = dx_layer0 + dx_orig (+ T_b^T dcoors
    on ligand rows) within 1e-14 (the fp32 products are exact in fp64); receptor rows, and every row without dcoors,
    bitwise equal to dx_layer0 + dx_orig; the first and the last node of every ligand checked on their own."""
    from test_gpu_forward_kernels import _fbatch
    dev, lib = cuda_device, nat.load()
    _, plan = _fbatch(kind, dev)
    N, NL, B = plan.N, plan.N_l, plan.n_pairs
    seg = [int(v) for v in plan.seg_ptr_host]
    n_lig = [seg[b + 1] - seg[b] for b in range(B)]
    if kind == 'bench':
        assert B == 330
    else:
        assert min(n_lig) == 1 and max(n_lig) >= 129
    r = _gen(660, dev)
    dh0, dhl0 = r(N, nat.H0_PAD), r(N, nat.H0_PAD)
    mu = torch.exp(r(N, 5, s=0.5))
    mu_l, mu_r = mu[:NL].contiguous(), mu[NL:].contiguous()
    dx_l0, dx_orig = r(N, 3).double(), r(N, 3).double()
    rot = torch.linalg.qr(r(B, 3, 3).double())[0].float().contiguous()    # a distinct rotation per pair
    dcoors = r(NL, 3, s=0.05) if with_dcoors else None

    def run():
        dmu = torch.full((N + 2, 5), -777.25, device=dev)
        dx = torch.full((N + 2, 3), -777.25, dtype=F64, device=dev)
        nat.check(lib.eqd_bwd_inputs(C.byref(plan.struct), nat.ptr(dh0), nat.ptr(dhl0), nat.ptr(mu_l), nat.ptr(mu_r),
                                     nat.ptr(dx_l0), nat.ptr(dx_orig), nat.ptr(rot),
                                     nat.ptr(dcoors) if dcoors is not None else None, nat.ptr(dmu), nat.ptr(dx), None),
                  'eqd_bwd_inputs')
        return dmu, dx

    dmu, dx = _twice(run)
    assert bool((dmu[N:] == -777.25).all()) and bool((dx[N:] == -777.25).all()), 'rows past the end were written'
    dmu, dx = dmu[:N], dx[:N]
    dmu_ref = (_d(dh0) + _d(dhl0))[:, 64:69] / _d(mu)
    ulp = torch.from_numpy(np.spacing(np.abs(dmu_ref.cpu().numpy()).astype(np.float32)).astype(np.float64)).to(dev)
    worst = float(((_d(dmu) - dmu_ref).abs() / ulp).max())
    print(f'\nbwd inputs[{kind}, dcoors {with_dcoors}]: dmu {worst:.2f} fp32 ulp')
    assert worst <= 2.0, f'dmu: {worst:.2f} ulp'
    base = dx_l0 + dx_orig
    assert torch.equal(dx[NL:], base[NL:]), 'receptor rows must be dx_layer0 + dx_orig, bitwise'
    if dcoors is None:
        assert torch.equal(dx[:NL], base[:NL]), 'without dcoors every row must be dx_layer0 + dx_orig, bitwise'
        return
    pair = _pair_of_node(n_lig).to(dev)
    ref = base[:NL] + torch.einsum('nrc,nr->nc', _d(rot).view(B, 3, 3)[pair], _d(dcoors))
    firsts = torch.tensor(seg[:B], device=dev)
    lasts = torch.tensor(seg[1:B + 1], device=dev) - 1
    rep = Report(f'bwd inputs[{kind}]', 1e-14)
    rep.rel('dx ligand rows', dx[:NL], ref)
    for tag, rows in (('first', firsts), ('last', lasts)):
        err = (dx[rows] - ref[rows]).abs().max(1).values / float(ref.abs().max())
        rep.rel(f'dx {tag} node of every ligand', dx[rows], ref[rows])
        assert bool((err <= 1e-14).all()), f'{tag} nodes of pairs {torch.nonzero(err > 1e-14).flatten().tolist()}'
    rep.check()


# ---- head ---------------------------------------------------------------------------------------------------------

def test_bwd_head_vs_manual_oracle(cuda_device):
    """eqd_bwd_head on the bulk batch (the forward's last-layer h, x and Kabsch covariances) against the fp64
    kabsch_bwd / keypoints_bwd of oracle/backward_manual.py on a sample of pairs, from the same h and x.  Every pair's
    dh and dx must be finite."""
    dev, lib = cuda_device, nat.load()
    g, plan = _batch('bulk', dev)
    model, eng = _model(dev)
    fwd = eng.forward(g)
    torch.cuda.synchronize()
    B, N, NL = plan.n_pairs, plan.N, plan.N_l
    r = _gen(700, dev)
    dcoors = r(NL, 3, s=0.05).contiguous()
    dkp = r(2 * B, nat.HEADS, 3, s=0.05).double().contiguous()
    ws_bytes = int(lib.eqd_bwd_head_workspace_bytes(N, plan.n_node_tiles, B))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)

    def run():
        dh = torch.full((N, 64), float('nan'), device=dev)
        dx = torch.full((N, 3), float('nan'), dtype=F64, device=dev)
        dpre = torch.full((N, 64), float('nan'), device=dev)
        gk, gq = torch.zeros(nat.HEADS * 64, 64, device=dev), torch.zeros(nat.HEADS * 64, 64, device=dev)
        nat.check(lib.eqd_bwd_head(C.byref(plan.struct), C.byref(fwd['head'].struct), nat.ptr(fwd['h']), nat.ptr(fwd['x64']),
                                   nat.ptr(fwd['cov']), nat.ptr(fwd['x_lig_in']), nat.ptr(dcoors), nat.ptr(dkp), None, None,
                                   nat.ptr(ws), ws_bytes, nat.ptr(dh), nat.ptr(dx), nat.ptr(dpre), nat.ptr(gk), nat.ptr(gq),
                                   None), 'eqd_bwd_head')
        return dh, dx, dpre, gk, gq

    dh, dx, *_ = _twice(run)
    assert torch.isfinite(dh).all() and torch.isfinite(dx).all()
    status = fwd['status_host'][:B].numpy()
    clean = [b for b in range(B) if status[b] == 0]
    assert len(clean) >= B - 5, status
    sample = [b for b in (0, 3, 4, 8) if b in clean] + [b for b in clean if b >= 9][::15]
    args = gio.load_args('dips')
    sd = gio.load_checkpoint('dips')
    cfg = orc.OracleConfig.from_args(args)
    seg = plan.seg_ptr_host
    h64, x64, xin = fwd['h'].double().cpu().numpy(), fwd['x64'].cpu().numpy(), fwd['x_lig_in'].double().cpu().numpy()
    dco, dk = dcoors.double().cpu().numpy(), dkp.cpu().numpy()
    dh_np, dx_np = dh.double().cpu().numpy(), dx.cpu().numpy()
    rep = Report('head[bulk]')
    for b in sample:
        (la, lb), (ra, rb) = (seg[b], seg[b + 1]), (seg[B + b], seg[B + b + 1])
        c = bm.head_forward(sd, cfg, h64[la:lb], x64[la:lb], h64[ra:rb], x64[ra:rb])
        G = {'wm': np.zeros((64, 64)), 'bm': np.zeros(64), 'wk': np.zeros_like(c['wk']), 'wq': np.zeros_like(c['wq'])}
        dY = bm.kabsch_bwd(c, xin[la:lb], dco[la:lb], (dk[b], dk[B + b]))
        dh_ref, dx_ref = bm.keypoints_bwd(cfg, c, dY, G)
        for side, (a, z) in enumerate(((la, lb), (ra, rb))):
            rep.rel(f'dh pair {b} side {side}', torch.from_numpy(dh_np[a:z]), torch.from_numpy(dh_ref[side]))
            rep.rel(f'dx pair {b} side {side}', torch.from_numpy(dx_np[a:z]), torch.from_numpy(dx_ref[side]))
    rep.check()


# ---- one whole training backward: bit pin and workspace bounds ------------------------------------------------------

class _RecordingLib:
    """Stands in for TrainEngine.lib and records every eqd_tn_gemm call."""

    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def eqd_tn_gemm(self, X, ldx, K, D, ldd, ncols, nrows, alpha, partial, colsum, nch, stream):
        self.calls.append((int(nrows), int(K), int(ncols), partial.value, None if colsum is None else colsum.value))
        return self._lib.eqd_tn_gemm(X, ldx, K, D, ldd, ncols, nrows, alpha, partial, colsum, nch, stream)


def _train_backward(dev):
    """TrainEngine.forward + backward of the 8-layer DIPS checkpoint on 100 pairs of 200 + 200 nodes (N = 40 000,
    E = 400 000: 313 node tiles, 400 attention tiles, 3 125 edge tiles on 132 CTAs), with seeded upstream gradients."""
    if 'train_bwd' not in _CACHE:
        g, plan = _batch('train', dev)
        model = gio.build_model('dips', dev).train()
        eng = TrainEngine(model)
        rec = _RecordingLib(eng.lib)
        eng.lib = rec
        fwd = eng.forward(g)
        r = _gen(800, dev)
        torch.manual_seed(0)          # the CPU generator of the SVD guard's perturbation (:578), should a pair need it
        flat = eng.backward(fwd, r(plan.N_l, 3, s=0.01), r(2 * plan.n_pairs, nat.HEADS, 3, s=0.01).double())
        torch.cuda.synchronize()
        _CACHE['train_bwd'] = (plan, eng._ws, rec.calls, flat.cpu().numpy())
    return _CACHE['train_bwd']


# sha256 of the flat gradient of _train_backward.  Every gradient keeps its summation order (fixed-order tile sums,
# row-chunk partials, fp64 second stage), so a change of that order shows here even inside the tolerances above.
TRAIN_GRAD_SHA256 = '1872fdcb0cbb43d6320d9184f087967cd5107508e7267868bfc7a48793cace97'


def test_train_backward_gradient_bits_pinned(cuda_device):
    plan, _, _, flat = _train_backward(cuda_device)
    assert (plan.N, plan.E) == (40000, 400000)
    assert np.isfinite(flat).all()
    digest = hashlib.sha256(flat.tobytes()).hexdigest()
    print(f'\ntrain backward flat gradient sha256 {digest}')
    assert digest == TRAIN_GRAD_SHA256


def test_train_backward_tn_gemm_calls_fit_the_workspace(cuda_device):
    lib = nat.load()
    plan, ws, calls, _ = _train_backward(cuda_device)
    assert len(calls) == 1 + 8 * 9
    listed = set(tn_gemm_shapes(plan.N, plan.E))
    for rows, K, nc, partial, colsum in calls:
        assert (rows, K, nc) in listed
        nch = C.c_int32(0)
        need = int(lib.eqd_tn_partial_floats(rows, K, nc, None, C.byref(nch)))
        assert partial == ws.partial.data_ptr() and need <= ws.partial.numel(), ((rows, K, nc), need, ws.partial.numel())
        if colsum is not None:
            assert colsum == ws.colsum.data_ptr() and nch.value * nc <= ws.colsum.numel()
    assert (plan.N, 64, 320) in {c[:3] for c in calls}
