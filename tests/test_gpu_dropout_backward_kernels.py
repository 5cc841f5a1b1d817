"""GPU (H100): the backward kernels of a dropout training step in the shipped configuration (layer_norm_coors = '0',
final_h_layer_norm = '0', the setting of both checkpoints) called directly on seeded inputs and compared with torch fp64
autograd of their stage under the numpy masks of tests/dropout_masks.py (p = 0.25, rank 3): eqd_bwd_edge (sites 0 / 1
on z1 / z3) and eqd_bwd_node_mlp (site 2 on u5).  The dropout counterpart of test_gpu_backward_kernels.py, whose
batches, Report, _twice, fp64 edge reference and kink rule it reuses, with the guarded outputs, descriptors and reduction
tables of test_gpu_layer_norm_kernels.py.  The keypoint head's dropout backward is tested in test_gpu_svd_guard.py.

Both kernels are persistent (grid = min(tiles, 132), a CTA walks tile, tile + 132, ...).  On `bulk` (41 510 nodes,
415 k edges: 325 node tiles and 3 243 edge tiles) every CTA walks at least two tiles, so a mask row taken from the CTA
instead of the tile, or a per-CTA partial sum reset between tiles, shows as an O(1) error of those rows.  `k70` has 70
in-edges per node, `ragged` edge tiles that straddle the ligand / receptor boundary and proteins of 1 node.

Every output has GUARD rows past its end, pre-filled with a finite sentinel, that must stay untouched, as must the
per-CTA partial rows >= n_partials.  Every kernel runs twice on the same inputs: the outputs must be bitwise equal.  The
per-CTA partials are reduced directly and through the layer's reduction table (LayerTrainPack maps) into the flat
gradient, whose ParamLayout views are compared at the same bound.

Tolerance: max |kernel - reference| / max |reference|, 1e-5.  Rows with a kept pre-activation inside the LeakyReLU kink
band are left out of the comparisons that depend on the branch (an element the mask drops enters the LeakyReLU as an
exact 0 and cannot take the other branch); d gamma / d beta of edge_mlp.3 get the slack of the z3 elements inside the
band, as in test_gpu_backward_kernels.py.  Measured on an H100 80GB HBM3 (700 W power limit), largest value over the
cases of each test (`pytest -s` prints every value):
  bwd edge   ein 5.9e-9, n1 5.1e-7, msg 1.1e-6, dz3 8.5e-8, dmsg 4.9e-7, dz1 4.6e-7, dxrel 3.1e-7, dw4 7.2e-7,
             db4 5.6e-7, dgamma 0 and dbeta 7.0e-11 after the slack (18 .. 71 z3 elements in the band on bulk); the
             reduction-table views the same
  bwd node   dh_in 4.3e-7, daggr 5.6e-7, dmu 1.1e-6, dh0_acc 3.4e-7, n5 1.2e-6, du 9.1e-7, dgamma 4.0e-7, dbeta 2.6e-7
             (table views the same)
The file runs in about 30 s on that GPU, most of it drawing the bulk batch's edge masks in numpy.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from equidock_public_b200 import _native as nat
from test_gpu_backward_kernels import (SMS, Report, _batch, _bwd_edge_ref, _bwd_edge_report, _d, _gen, _leaf, _reduce,
                                       _twice)
from test_gpu_forward_kernels import _coords
from test_gpu_layer_norm_kernels import (GUARD, SENT, SHIFT, _desc, _guarded, _kink_kept, _layer, _mask, _out,
                                         _table, _view)

pytestmark = pytest.mark.gpu

F64 = torch.float64


@pytest.mark.parametrize('kind,li', [('bulk', 1), ('bulk', 0), ('k70', 1), ('ragged', 0)])
def test_bwd_edge_with_dropout_vs_fp64_autograd(kind, li, cuda_device):
    """eqd_bwd_edge with dropout sites 0 / 1 and no coordinate LayerNorm (bwd_edge_kernel<DROP = true, CLN = false>):
    ein, n1, msg, dz3, dmsg, dz1, dxrel and the 256-float per-CTA partials (d edge_mlp.3 gamma / beta, d coors_mlp.4)."""
    dev, lib = cuda_device, nat.load()
    g, plan = _batch(kind, dev)
    mod, lay, tp, eng = _layer(li, dev, '0', '0')
    N, E, pw = plan.N, plan.E, tp.pw
    ntiles = (E + 127) // 128
    if kind == 'bulk':
        assert ntiles >= 2 * SMS
    nparts = min(ntiles, SMS)
    layer = 2 + li                   # the layer position of the forward dropout tests: the same masks
    desc = _desc(lay, drop_layer=layer)
    r = _gen(1800 + li, dev)
    proj = r(N, pw, s=0.5).contiguous()
    x_in = (_coords(g, dev) + torch.tensor(SHIFT, dtype=F64, device=dev)).contiguous()
    daggr = r(N, 64, s=0.1)
    dx_out = r(N, 3).double().contiguous()

    def run():
        outs = [_out(E, w, dev) for w in (44, 64, 64, 64, 64, 64)]
        dxrel = _out(E, 3, dev, F64)
        vec = torch.full(((SMS + GUARD) * 256,), SENT, device=dev)
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
    vec = res[7]
    assert bool((vec[nparts * 256:] == SENT).all()), 'per-CTA partial rows >= n_partials were written'
    sums = _reduce(lib, vec, nparts, 256, list(range(193)), dev)
    flat = _table(lib, tp, eng, 'edgevec', vec, nparts, 256, dev)

    ref = _bwd_edge_ref(mod, plan, proj, x_in, daggr, dx_out, _mask(layer, 0, E, 64, dev), _mask(layer, 1, E, 64, dev))
    rep = _bwd_edge_report(Report(f'edge dropout[{kind}, L{li}]'), ref, *(t[:E] for t in res[:7]), sums)
    # the reduction table sums the same partials: d gamma / d beta keep the slack of the z3 elements inside the band
    rep.rel('table edge_mlp.3.weight', _view(eng, flat, li, 'edge_mlp.3.weight', 64), ref['dgamma'],
            slack=ref['slack_g'])
    rep.rel('table edge_mlp.3.bias', _view(eng, flat, li, 'edge_mlp.3.bias', 64), ref['dbeta'], slack=ref['slack_b'])
    rep.rel('table coors_mlp.4.weight', _view(eng, flat, li, 'coors_mlp.4.weight', 64), ref['dw4'])
    rep.rel('table coors_mlp.4.bias', _view(eng, flat, li, 'coors_mlp.4.bias', 1), ref['db4'])
    rep.check()


@pytest.mark.parametrize('kind,li', [('bulk', 0), ('bulk', 1), ('ragged', 1)])
def test_bwd_node_mlp_with_dropout_vs_fp64_autograd(kind, li, cuda_device):
    """eqd_bwd_node_mlp with dropout site 2 and no final LayerNorm (bwd_node_mlp_kernel<EXTRA, DROP = true,
    HLN = false>): dh_in, daggr, dmu, dh0 accumulated into a non-zero buffer, n5, du and the 144-float per-CTA partials
    (d node_mlp.3 gamma / beta); dh_out is an input only and must stay unchanged."""
    dev, lib = cuda_device, nat.load()
    _, plan = _batch(kind, dev)
    mod, lay, tp, eng = _layer(li, dev, '0', '0')
    N, dh, dhp = plan.N, tp.dh, tp.dhp
    ntiles = (N + 127) // 128
    if kind == 'bulk':
        assert ntiles >= 2 * SMS
    nparts = min(ntiles, SMS)
    layer = 1 + li                   # the layer position of the forward node-stage dropout tests
    desc = _desc(lay, drop_layer=layer)
    r = _gen(1900 + li, dev)
    pad = lambda t: torch.cat([t, torch.zeros(N, dhp - dh, device=dev)], 1).contiguous()
    h, aggr, mu = pad(r(N, dh, s=0.7)), r(N, 64, s=0.3), pad(r(N, dh, s=0.5))
    h0 = torch.cat([r(N, nat.H0), torch.zeros(N, nat.H0_PAD - nat.H0, device=dev)], 1).contiguous()
    dh_out = r(N, 64, s=0.1)
    dh0_init = _out(N, nat.H0_PAD, dev)
    dh0_init[:N] = torch.cat([r(N, nat.H0, s=0.2), torch.zeros(N, nat.H0_PAD - nat.H0, device=dev)], 1)

    def run():
        dh_in, daggr, dmu, n5, du = (_out(N, w, dev) for w in (dhp, 64, dhp, dhp, dhp))
        dy, dh0 = dh_out.clone(), dh0_init.clone()
        vec = torch.full(((SMS + GUARD) * 144,), SENT, device=dev)
        n = C.c_int32(0)
        nat.check(lib.eqd_bwd_node_mlp(C.byref(plan.struct), C.byref(desc), nat.ptr(tp.t['w_node1_lin']),
                                       nat.ptr(tp.t['w_node2_lin']), nat.ptr(h), dhp, nat.ptr(aggr), nat.ptr(mu), dhp,
                                       nat.ptr(h0), nat.ptr(dy), nat.ptr(dh_in), nat.ptr(daggr), nat.ptr(dmu),
                                       nat.ptr(dh0), nat.ptr(n5), nat.ptr(du), nat.ptr(vec), C.byref(n), None),
                  'eqd_bwd_node_mlp')
        assert n.value == nparts
        return dh_in, daggr, dmu, dh0, n5, du, dy, vec

    res = _twice(run)
    for name, t in zip(('dh_in', 'daggr', 'dmu', 'dh0_acc', 'n5', 'du'), res[:6]):
        _guarded(name, t, N)
    dh_in, daggr, dmu, dh0, n5, du = (t[:N] for t in res[:6])
    assert torch.equal(res[6], dh_out), 'dh_out must stay unchanged without the final LayerNorm'
    vec = res[7]
    assert bool((vec[nparts * 144:] == SENT).all()), 'per-CTA partial rows >= n_partials were written'
    sums = _reduce(lib, vec, nparts, 144, list(range(dh)) + [72 + c for c in range(dh)], dev)
    flat = _table(lib, tp, eng, 'nodevec', vec, nparts, 144, dev)

    # fp64 autograd of node_mlp (:319-337) with the site-2 factor on u5
    lin0, ln, lin4 = mod.node_mlp[0], mod.node_mlp[3], mod.node_mlp[4]
    slope, sk = float(mod.leakyrelu_neg_slope), float(mod.skip_weight_h)
    m2 = _mask(layer, 2, N, dh, dev)
    xh, xa, xm, x0 = _leaf(h[:, :dh]), _leaf(aggr), _leaf(mu[:, :dh]), _leaf(h0[:, :nat.H0])
    gamma, beta = _leaf(ln.weight), _leaf(ln.bias)
    x = torch.cat([xh, xa, xm, x0], 1)
    u5 = x @ _d(lin0.weight).t() + _d(lin0.bias)
    u5.retain_grad()
    n5_ref = F.layer_norm(F.leaky_relu(u5 * m2, slope), (dh,), gamma, beta, ln.eps)
    o = n5_ref @ _d(lin4.weight).t() + _d(lin4.bias)
    out = sk * o + (1.0 - sk) * xh if dh == nat.HID else o
    (out * _d(dh_out)).sum().backward()
    terms = (x.detach().abs() @ _d(lin0.weight).abs().t() + _d(lin0.bias).abs()) * m2
    ok = ~_kink_kept(u5.detach() * m2, terms, 'u5', m2 != 0)

    # n5 and the affine gradients are upstream of the LeakyReLU derivative: compared over every row
    rep = Report(f'node_mlp dropout[{kind}, L{li}]')
    rep.rel('dh_in', dh_in[:, :dh], xh.grad, ok)
    rep.rel('daggr', daggr, xa.grad, ok)
    rep.rel('dmu', dmu[:, :dh], xm.grad, ok)
    rep.rel('dh0_acc (accumulated)', dh0[:, :nat.H0], _d(dh0_init[:N, :nat.H0]) + x0.grad, ok)
    rep.rel('n5', n5[:, :dh], n5_ref.detach())
    rep.rel('du', du[:, :dh], u5.grad, ok)
    rep.rel('dgamma', sums[:dh], gamma.grad)
    rep.rel('dbeta', sums[dh:], beta.grad)
    rep.rel('table node_mlp.3.weight', _view(eng, flat, li, 'node_mlp.3.weight', dh), gamma.grad)
    rep.rel('table node_mlp.3.bias', _view(eng, flat, li, 'node_mlp.3.bias', dh), beta.grad)
    rep.check()
    if dhp > dh:      # layer 0: channels 69..71 are padding and must come out exactly 0
        for name, t in (('dh_in', dh_in), ('dmu', dmu), ('n5', n5), ('du', du), ('dh0_acc', dh0)):
            assert float(t[:, dh:].abs().max()) == 0.0, name
