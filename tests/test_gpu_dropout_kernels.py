"""GPU (H100): each forward entry point with dropout on, called directly at p = 0.25 and compared with a torch fp64
evaluation of its formula under the numpy masks of tests/dropout_masks.py (one wrong mask bit is an O(1) error of its
row, far above the bound).  Batches, layers, tolerance and the run-twice-bitwise check are those of
test_gpu_forward_kernels.py: mixed in-degrees 0 / 1 / 9 / 10, in-degree 64 and 70 (> 64), the ragged batch with 128+1
and 128+3 edge tiles, proteins of every node-tile edge, layer 0 (69 wide) and a 64-wide layer.

The fp32 edge stage, the fp32 node stage and the head's mean kernel are persistent with a grid of at most 2 x 132 CTAs.
The `bulk` edge cases (3 460 tiles), the `bench` node-stage cases (1 032 node tiles) and the `bench` keypoint cases
(1 032 node tiles, K = 50 and 64) give every CTA several tiles, so a mask row taken from the CTA's first tile instead
of the current one is an O(1) error there; each case asserts its tile count.  Measured on an H100 80GB HBM3 (700 W
power limit), largest value over the cases of each test: edge aggr 6.4e-7, update 2.2e-7; node mu 1.1e-6, h_out
5.8e-7, proj_next 5.4e-7 .. 8.3e-7; keypoints 7.8e-8.  The file runs in about 30 s on that GPU."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dropout_masks as dm
import fp64_stages as fs
from equidock_public_b200 import _native as nat
from test_gpu_backward_kernels import Report, _d, _layer, _twice
from test_gpu_forward_kernels import ETA, _coords, _edge_run, _fbatch, _np_gen
from test_gpu_layer_norm_kernels import _guarded, _out

pytestmark = pytest.mark.gpu
F64 = torch.float64
P, SEED = 0.25, 0x5EED_0123_4567_89AB
GRID = 2 * 132          # the grid cap of the fp32 edge stage, the fp32 node stage and the head's mean kernel


def _desc(lay, layer, eta=None):
    s = nat.EqdLayer.from_buffer_copy(lay.struct)
    if eta is not None:
        s.dev.x_connection_init = eta
    s.dropout = nat.dropout_descriptor(P, SEED, layer, 3)
    return s


def _m(layer, site, rows, cols, dev):
    return dm.mask(SEED, 3, layer, site, rows, cols, P).to(dev)


def _edge_ref(mod, plan, proj, x_in, layer):
    """fs.edge_stage with the site-0 / site-1 masks on z1 / z3."""
    w, b = fs._w, fs._b
    slope, dh = float(mod.leakyrelu_neg_slope), int(mod.att_mlp_Q[0].weight.shape[0])
    N, E, dev = plan.N, plan.E, x_in.device
    src, dst = plan.col_src.long(), plan.edge_dst.long()
    he = torch.cat([plan.he_l[:plan.E_l], plan.he_r[:plan.E_r]]).to(F64)
    xrel = x_in[src] - x_in[dst]
    d2 = (xrel ** 2).sum(1, keepdim=True)
    ein = torch.cat([he] + [torch.exp(-d2 / sg) for sg in fs.SIGMAS], 1)
    z1 = (proj[src, 0:64] + proj[dst, 64:128] + ein @ w(mod.edge_mlp[0])[:, 2 * dh:].t()) * _m(layer, 0, E, 64, dev)
    n1 = F.layer_norm(F.leaky_relu(z1, slope), (64,), w(mod.edge_mlp[3]), b(mod.edge_mlp[3]), mod.edge_mlp[3].eps)
    msg = n1 @ w(mod.edge_mlp[4]).t() + b(mod.edge_mlp[4])
    z3 = (msg @ w(mod.coors_mlp[0]).t() + b(mod.coors_mlp[0])) * _m(layer, 1, E, 64, dev)
    phi = F.leaky_relu(z3, slope) @ w(mod.coors_mlp[4]).t() + b(mod.coors_mlp[4])
    deg = (plan.row_ptr[1:] - plan.row_ptr[:-1]).to(dev, F64).clamp(min=1)[:, None]
    aggr = torch.zeros(N, 64, dtype=F64, device=dev).index_add_(0, dst, msg) / deg
    xupd = torch.zeros(N, 3, dtype=F64, device=dev).index_add_(0, dst, xrel * phi) / deg
    return aggr, xupd


@pytest.mark.parametrize('kind,li', [('ragged', 0), ('ragged', 1), ('mixed', 0), ('mixed', 1), ('k64', 1), ('k70', 0),
                                     ('long', 1), ('bulk', 1), ('bulk', 0)])
def test_edge_stage_with_dropout_vs_fp64(kind, li, cuda_device):
    """`bulk` (415 k edges, 3 460 node tiles of 12 nodes on 264 CTAs): every CTA of the fp32 kernel walks several tiles,
    so the mask rows of its second and later tiles are checked."""
    dev = cuda_device
    g, plan = _fbatch(kind, dev)
    if kind == 'bulk':
        tn = 128 // int(plan.struct.max_in_degree)
        assert (plan.N + tn - 1) // tn >= 2 * GRID
    mod, lay, tp = _layer(li, dev)
    N, pw = plan.N, 128 + 3 * tp.dhp
    r = _np_gen(910 + li, dev)
    proj = r(N, pw, s=0.5).contiguous()
    x_in = (_coords(g, dev) + torch.tensor([1.0e3, -0.7e3, 0.4e3], dtype=F64, device=dev)).contiguous()
    x_orig = (x_in + r(N, 3, s=3.0).double()).contiguous()
    layer = 2 + li                     # any position: it only enters the counter
    st = _desc(lay, layer, ETA)
    routed = _edge_run(nat.load().eqd_edge_stage, plan, st, proj, x_in, x_orig, dev)
    ffma = _edge_run(nat.load().eqd_edge_stage_ffma, plan, st, proj, x_in, x_orig, dev)
    assert torch.equal(routed[0], ffma[0]) and torch.equal(routed[1], ffma[1])   # dropout routes to the fp32 kernel
    aggr, xupd = _edge_ref(mod, plan, _d(proj), x_in, layer)
    base = ETA * x_orig + (1.0 - ETA) * x_in
    rep = Report(f'dropout edge[{kind}, L{li}]')
    rep.rel('aggr', ffma[0], aggr)
    rep.rel('update', ffma[1] - base, xupd)
    rep.check()
    # the masks are on: the same launch without them lands elsewhere
    off = _edge_run(nat.load().eqd_edge_stage_ffma, plan, _off(lay, ETA), proj, x_in, x_orig, dev)
    assert float((off[0] - ffma[0]).abs().max()) > 1e-2 * float(aggr.abs().max())


def _off(lay, eta):
    s = nat.EqdLayer.from_buffer_copy(lay.struct)
    s.dev.x_connection_init = eta
    return s


def _node_ref(mod, seg, proj, h, h0, aggr, dh, dhp, layer, dev):
    q, k, v = proj[:, 128:128 + dh], proj[:, 128 + dhp:128 + dhp + dh], proj[:, 128 + 2 * dhp:128 + 2 * dhp + dh]
    mu = fs.attention(seg, q, k, v)
    w, b = fs._w, fs._b
    slope, sk = float(mod.leakyrelu_neg_slope), float(mod.skip_weight_h)
    u5 = torch.cat([h, aggr, mu, h0], 1) @ w(mod.node_mlp[0]).t() + b(mod.node_mlp[0])
    u5 = u5 * _m(layer, 2, u5.shape[0], dh, dev)
    o = F.layer_norm(F.leaky_relu(u5, slope), (dh,), w(mod.node_mlp[3]), b(mod.node_mlp[3]), mod.node_mlp[3].eps)
    o = o @ w(mod.node_mlp[4]).t() + b(mod.node_mlp[4])
    return mu, (sk * o + (1.0 - sk) * h if h.shape[1] == o.shape[1] else o)


@pytest.mark.parametrize('kind,li,nxt', [('sizes', 0, False), ('sizes', 1, False), ('ragged', 0, False),
                                         ('mixed', 1, False), ('bench', 0, False), ('bench', 1, False),
                                         ('bench', 1, True)])
def test_node_stage_with_dropout_vs_fp64(kind, li, nxt, cuda_device):
    """eqd_node_stage (fp32, the node stage of a forward with dropout on): site 2 on u5, 69 wide in layer 0 (the mask's
    columns 64..68 live in the kernel's extra column), 64 wide otherwise.  `bench` has 1 032 node tiles on 264 CTAs, so
    every CTA applies the mask to several tiles; `nxt`: p_next = layer 2, and proj_next (Psrc | Pdst | Q | K | V of the
    masked h_out) against the fp64 projections of the reference h_out.  Outputs carry guard rows that must stay
    untouched."""
    dev = cuda_device
    g, plan = _fbatch(kind, dev)
    mod, lay, tp = _layer(li, dev)
    N, dh, dhp = plan.N, tp.dh, tp.dhp
    if kind == 'bench':
        assert plan.n_node_tiles >= 2 * GRID
    r = _np_gen(920 + li, dev)
    h0 = torch.zeros(N, 72, device=dev)
    h0[:, :69] = r(N, 69)
    h = h0 if li == 0 else r(N, 64)
    ldh = 72 if li == 0 else 64
    proj = r(N, 128 + 3 * dhp, s=0.3)
    for c0 in (128, 128 + dhp, 128 + 2 * dhp):      # Q, K, V pad columns are 0, as the packed projections leave them
        proj[:, c0 + dh:c0 + dhp] = 0.0
    aggr = r(N, 64)
    layer = 1 + li
    st = _desc(lay, layer)
    mod_n, lay_n, _ = _layer(li + 1, dev) if nxt else (None, None, None)

    def run():
        mu, h_out, pn = _out(N, dhp, dev), _out(N, 64, dev), _out(N if nxt else 0, 320, dev)
        nat.check(nat.load().eqd_node_stage(C.byref(plan.struct), C.byref(st),
                                            C.byref(lay_n.struct) if nxt else None, nat.ptr(h), ldh, nat.ptr(h0),
                                            nat.ptr(proj), nat.ptr(aggr), nat.ptr(mu), nat.ptr(h_out),
                                            nat.ptr(pn) if nxt else None, None), 'eqd_node_stage')
        return mu, h_out, pn

    mu, h_out, pn = _twice(run)
    for name, t in (('mu', mu), ('h_out', h_out), ('proj_next', pn)):
        _guarded(name, t, N)
    seg = plan.seg_ptr.cpu().tolist()
    mu_ref, h_ref = _node_ref(mod, seg, _d(proj), _d(h)[:, :dh], _d(h0)[:, :69], _d(aggr), dh, dhp, layer, dev)
    rep = Report(f'dropout node[{kind}, L{li}{", p_next" if nxt else ""}]')
    rep.rel('mu', mu[:N, :dh], mu_ref)
    rep.rel('h_out', h_out[:N], h_ref)
    if nxt:
        ref = fs.projections(mod_n, h_ref)
        for name, c0 in (('Psrc', 0), ('Pdst', 64), ('Q', 128), ('K', 192), ('V', 256)):
            rep.rel(f'proj_next {name}', pn[:N, c0:c0 + 64], ref[name])
    rep.check()


@pytest.mark.parametrize('kind,K', [('head_sizes', 50), ('ragged', 50), ('bench', 50), ('bench', 64)])
def test_keypoints_with_dropout_vs_fp64(kind, K, cuda_device):
    """eqd_keypoints_dropout: site 3 on W_m h + b_m before the LeakyReLU and the per-protein mean (node tiles of every
    size up to 128 + 1 and a protein of 2000 nodes).  `bench`: 1 032 node tiles on the mean kernel's 264 CTAs, with the
    checkpoint's 50 heads and with 64 (heads_ref.build_model)."""
    from test_gpu_backward_kernels import _model
    import heads_ref as hr
    dev = cuda_device
    g, plan = _fbatch(kind, dev)
    if kind == 'bench':
        assert plan.n_node_tiles >= 2 * GRID
    model = _model(dev)[0] if K == 50 else hr.build_model('dips', dev, K, seed=K)
    ieg = model.iegmn_original
    head = ieg.packed_head(dev)
    N, B = plan.N, plan.n_pairs
    r = _np_gen(930, dev)
    h, x = r(N, 64), (_coords(g, dev) + r(N, 3, s=2.0).double()).contiguous()
    L = 8
    drop = nat.dropout_descriptor(P, SEED, L, 3)
    lib = nat.load()
    ws_bytes = int(lib.eqd_workspace_bytes_k(N, plan.n_node_tiles, B, K))

    def run():
        ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=dev)
        kp = _out(2 * B, K * 3, dev, F64)
        ym, cov = torch.empty(2 * B, 3, dtype=F64, device=dev), torch.empty(B, 9, dtype=F64, device=dev)
        nat.check(lib.eqd_keypoints_dropout(C.byref(plan.struct), C.byref(head.struct), C.byref(drop), nat.ptr(h),
                                            nat.ptr(x), nat.ptr(ws), ws_bytes, nat.ptr(kp), nat.ptr(ym), nat.ptr(cov),
                                            None), 'eqd_keypoints_dropout')
        return kp, ym, cov

    kp, _, _ = _twice(run)
    _guarded('keypts', kp, 2 * B)
    kp = kp[:2 * B].view(2 * B, K, 3)
    w = lambda m: m.weight.detach().to(F64)
    pre = (_d(h) @ w(ieg.mlp_h_mean_ROT[0]).t() + ieg.mlp_h_mean_ROT[0].bias.detach().to(F64)) * _m(L, 3, N, 64, dev)
    act = F.leaky_relu(pre, float(ieg.leakyrelu_neg_slope))
    seg = plan.seg_ptr.cpu().tolist()
    Y = []
    for s in range(2 * B):
        o = s + B if s < B else s - B
        qbar = act[seg[o]:seg[o + 1]].mean(0)
        keys = (_d(h)[seg[s]:seg[s + 1]] @ w(ieg.att_mlp_key_ROT[0]).t()).view(-1, K, 64)
        qry = (qbar @ w(ieg.att_mlp_query_ROT[0]).t()).view(K, 64)
        att = torch.softmax(torch.einsum('nkd,kd->kn', keys, qry) / 8.0, dim=1)
        Y.append(att @ x[seg[s]:seg[s + 1]])
    rep = Report(f'dropout keypoints[{kind}, K={K}]')
    rep.rel('keypts', kp, torch.stack(Y))
    rep.check()
