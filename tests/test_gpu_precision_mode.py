"""The opt-in bf16x3 inference mode (IEGMN.precision = 'bf16x3', eqd_layer_params.mma_products = 3) of the 64-wide
layers: each of its four tensor-core kernels against fp64, the default path untouched, all 125 shipped pairs end to end,
capture / determinism, and the refusals.

Error bound of a kernel (max |kernel - fp64| over a tensor, relative to the tensor's largest fp64 magnitude, as in
test_gpu_forward_kernels.py).  In bf16x3 each operand keeps two bf16 terms (|v - v0 - v1| <= 2^-18 |v|) and the product
a1 w1 is dropped, so every product a_k w_k carries a relative error below 3 * 2^-18 < 2^-16, and a GEMM output
sum_k a_k w_k is off by at most 2^-16 sum_k |a_k w_k| <= 2^-16 K max|a| max|w|.  Taking K (the GEMM's depth) as the
factor from that sum to the largest output, a kernel whose outputs pass through GEMMs of depths K1, K2, ... is bounded by
(K1 + K2 + ...) * 2^-16:
  projections           K = 64                       -> 64 * 2^-16  = 9.8e-4
  edge stage            GEMM1 K = 48, GEMM2/3 K = 64  -> 112 * 2^-16 = 1.7e-3 (aggr and the coordinate update)
  node MLP (h_out)      K = 272, then K = 64          -> 336 * 2^-16 = 5.1e-3
  attention (mu)        S = Q K^T (K = 64) enters exp(): an absolute logit error of 2^-16 max_ij sum_d |q_id k_jd| is a
                        relative error of the weights; then P V (K = 64):  2^-16 (2 max sum|q k| + 64)
The fp32 arithmetic of the epilogues adds about 1e-6 and is covered by these bounds.  Each launch runs twice and must be
bitwise equal.

End to end, an operand error 2^8 times that of bf16x6 (2^-16 against 2^-24) moves the output by at most about 2^8 times
as much: the per-pair bounds of test_gpu_acceptance.py (C-alpha coordinates max(1e-4, the pair's fp32-vs-fp64 yardstick),
rotation 3e-5) times 256.  The C-RMSD / I-RMSD table of BASELINE.md section 1 must come out as in the default mode: every
entry within one unit of its printed 0.01 A digit, the criterion of test_gpu_acceptance.py.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import fp64_stages as fs
import golden_io as gio
from equidock_public_b200 import _native as nat
from test_gpu_backward_kernels import Report, _d, _layer, _twice
from test_gpu_forward_kernels import ETA, SENT, _coords, _decode_kv, _edge_run, _fbatch, _np_gen

pytestmark = pytest.mark.gpu

U16 = 2.0 ** -16
TOL_PROJ, TOL_EDGE, TOL_NODE_MLP = 64 * U16, 112 * U16, 336 * U16


def _desc(lay, products, eta=None):
    """A copy of a packed layer's descriptor with mma_products (and x_connection_init) set."""
    s = nat.EqdLayer.from_buffer_copy(lay.struct)
    s.dev.mma_products = products
    if eta is not None:
        s.dev.x_connection_init = eta
    return s


# ---- edge stage -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('kind,eta', [('bench', ETA), ('bulk', 0.0), ('ragged', ETA), ('long', 0.0), ('mixed', ETA),
                                      ('mixed', 0.0), ('k1', ETA), ('k33', 0.0), ('k64', ETA)])
def test_edge_stage_bf16x3_vs_fp64(kind, eta, cuda_device):
    """eqd_edge_stage of layer 1 with mma_products = 3: coordinates around 1e3 A, x_connection_init 0 and 0.3 with
    x_orig != x_in; `mixed` puts nodes of in-degree 0, 1, 9 and 10 in one tile; k1 / k33 / k64: tiles of 32, 1 and 1
    nodes (max_in_degree 1, 33, 64)."""
    dev = cuda_device
    g, plan = _fbatch(kind, dev)
    mod, lay, _ = _layer(1, dev)
    N = plan.N
    r = _np_gen(1900, dev)
    proj = r(N, 320, s=0.5).contiguous()
    x_in = (_coords(g, dev) + torch.tensor([1.0e3, -0.7e3, 0.4e3], dtype=torch.float64, device=dev)).contiguous()
    x_orig = (x_in + r(N, 3, s=3.0).double()).contiguous()
    if kind == 'mixed':
        deg = (plan.row_ptr[1:] - plan.row_ptr[:-1]).cpu()
        assert all(int((deg == d).sum()) > 0 for d in (0, 1, 9, 10))
    aggr, xo = _edge_run(nat.load().eqd_edge_stage, plan, _desc(lay, 3, eta), proj, x_in, x_orig, dev)
    aggr6, xo6 = _edge_run(nat.load().eqd_edge_stage, plan, _desc(lay, 6, eta), proj, x_in, x_orig, dev)
    ref_a, ref_u = fs.edge_stage(mod, plan, _d(proj), x_in)
    base = ETA * x_orig + (1.0 - ETA) * x_in if eta else x_in
    isolated = (plan.row_ptr[1:] - plan.row_ptr[:-1]) == 0
    if bool(isolated.any()):
        assert float(aggr[isolated].abs().max()) == 0.0
    rep = Report(f'edge bf16x3[{kind}, eta {eta:.1f}]', tol=TOL_EDGE)
    rep.rel('aggr', aggr, ref_a)
    rep.rel('update', xo - base, ref_u)
    rep.check()
    assert not torch.equal(aggr, aggr6), 'mma_products = 3 must select the three-product kernel'


# ---- projections, attention, node MLP ---------------------------------------------------------------------------------

def _attention_bound(seg, q, k):
    """2^-16 (2 max_ij sum_d |q_id k_jd| + 64) over the partner blocks of the batch."""
    B, m = (len(seg) - 1) // 2, 0.0
    for s in range(2 * B):
        p = s + B if s < B else s - B
        a, b, c, d = int(seg[s]), int(seg[s + 1]), int(seg[p]), int(seg[p + 1])
        if b > a and d > c:
            m = max(m, float((q[a:b].abs() @ k[c:d].abs().t()).max()))
    return U16 * (2.0 * m + 64.0), m


@pytest.mark.parametrize('kind', ['bench', 'ragged', 'long', 'sizes'])
def test_node_stage_bf16x3_vs_fp64(kind, cuda_device):
    """eqd_project_tc of layer 1 (Psrc | Pdst | Q and the K / V blocks), then eqd_node_stage_tc of layer 1 with p_next =
    layer 2 (attention mu, node MLP h_out, layer 2's projections and K / V blocks), all with mma_products = 3, against
    fp64 on the kernels' own inputs.  `sizes` has proteins of 1 ... 2000 nodes (every query-tile and key-chunk edge),
    `bench` is bench.py's 330-pair batch."""
    dev, lib = cuda_device, nat.load()
    _, plan = _fbatch(kind, dev)
    mod, lay, _ = _layer(1, dev)
    mod2, lay2, _ = _layer(2, dev)
    N, seg = plan.N, plan.seg_ptr_host
    L, Ln = _desc(lay, 3), _desc(lay2, 3)
    G = C.byref(plan.struct)
    r = _np_gen(1910, dev)
    h, aggr = r(N, 64, s=0.7), r(N, 64, s=0.3)
    h0 = torch.zeros(N, 72, device=dev)
    h0[:, :69] = r(N, 69)

    def project():
        proj = torch.full((N, 320), SENT, device=dev)
        kv = torch.zeros(lib.eqd_kv_blocks_bytes(N), dtype=torch.uint8, device=dev)
        nat.check(lib.eqd_project_tc(G, C.byref(L), nat.ptr(h), nat.ptr(proj), nat.ptr(kv), None), 'eqd_project_tc')
        return proj, kv

    proj, kv = _twice(project)
    rep = Report(f'node stage bf16x3[{kind}]', tol=TOL_PROJ)
    ref = fs.projections(mod, _d(h))
    K, V = _decode_kv(kv, N)
    for name, got in (('Psrc', proj[:, 0:64]), ('Pdst', proj[:, 64:128]), ('Q', proj[:, 128:192]), ('K blocks', K),
                      ('V blocks', V)):
        rep.rel(f'proj {name}', got, ref[name.split()[0]])

    def stage():
        kv2 = kv.clone()
        mu = torch.full((N, 64), float('nan'), device=dev)
        h_out = torch.full((N, 64), float('nan'), device=dev)
        pn = torch.full((N, 320), SENT, device=dev)
        nat.check(lib.eqd_node_stage_tc(G, C.byref(L), C.byref(Ln), nat.ptr(h), nat.ptr(h0), nat.ptr(proj),
                                        nat.ptr(aggr), nat.ptr(kv2), nat.ptr(mu), nat.ptr(h_out), nat.ptr(pn), None),
                  'eqd_node_stage_tc')
        return mu, h_out, pn, kv2

    mu, h_out, pn, kv2 = _twice(stage)
    q = _d(proj[:, 128:192])
    mu_ref = fs.attention(seg, q, K, V)
    tol_mu, qk = _attention_bound(seg, q, K)
    print(f'\n{kind}: max_ij sum_d |q_id k_jd| = {qk:.1f}: attention bound {tol_mu:.2e}')
    att = Report(f'attention bf16x3[{kind}]', tol=tol_mu)
    att.rel('mu', mu, mu_ref)
    nm = Report(f'node MLP bf16x3[{kind}]', tol=TOL_NODE_MLP)
    nm.rel('h_out', h_out, fs.node_mlp(mod, _d(h), _d(aggr), _d(mu), _d(h0[:, :69])))
    ref2 = fs.projections(mod2, _d(h_out))
    K2, V2 = _decode_kv(kv2, N)
    for name, got in (('Psrc', pn[:, 0:64]), ('Pdst', pn[:, 64:128]), ('Q', pn[:, 128:192]), ('K blocks', K2),
                      ('V blocks', V2)):
        rep.rel(f'proj_next {name}', got, ref2[name.split()[0]])
    for rp in (rep, att, nm):
        rp.check()


# ---- the default path, capture, determinism --------------------------------------------------------------------------

_MODELS = {}


def _small_batch(dev):
    from equidock_public_b200 import synthetic
    rng = np.random.default_rng(77)
    return gio.make_batch([synthetic.synthetic_pair(rng, a, b, 10) for a, b in ((60, 75), (130, 41), (9, 200))], dev)


def _run(model, g):
    coors, kl, kr, rot, trans = model(g, epoch=0)
    return torch.cat([c.reshape(-1) for c in coors] + [k.reshape(-1) for k in kl + kr]
                     + [t.reshape(-1) for t in rot + trans])


def test_default_precision_is_unchanged(cuda_device):
    """precision='fp32' set explicitly gives the bits of a model that never touched the attribute; bf16x3 gives other
    bits; switching back restores the fp32 bits, also on a CUDA graph captured before the switches (it re-captures)."""
    dev = cuda_device
    g = _small_batch(dev)
    untouched = gio.build_model('dips', dev)
    ref = _run(untouched, g)
    m = gio.build_model('dips', dev)
    assert m.precision == 'fp32' and m.iegmn_original.precision == 'fp32'
    m.precision = 'fp32'
    assert torch.equal(_run(m, g), ref)
    gf = m.graphed(g)
    assert torch.equal(gf.launch().raw_result()['ligand_coors'], untouched.iegmn_original.last_outputs['ligand_coors'])
    m.precision = 'bf16x3'
    assert m.iegmn_original.precision == 'bf16x3'
    low = _run(m, g)
    assert not torch.equal(low, ref)
    low_graphed = gf.launch().raw_result()['ligand_coors'].clone()
    assert torch.equal(low_graphed, m.iegmn_original.last_outputs['ligand_coors'])
    m.precision = 'fp32'
    assert torch.equal(_run(m, g), ref)
    assert torch.equal(gf.launch().raw_result()['ligand_coors'], untouched.iegmn_original.last_outputs['ligand_coors'])


def test_mma_products_6_equals_0(cuda_device):
    """mma_products = 6 selects the same kernels as 0: the whole forward (eqd_iegmn_forward) and every tensor-core
    entry point give the same bits."""
    from equidock_public_b200.engine import IEGMNEngine
    dev = cuda_device
    g = _small_batch(dev)
    m = gio.build_model('dips', dev)
    ref = _run(m, g)
    orig = IEGMNEngine.forward
    IEGMNEngine.forward = lambda self, *a, **k: orig(self, *a, **{**k, 'mma_products': 6})
    try:
        six = _run(m, g)
    finally:
        IEGMNEngine.forward = orig
    assert torch.equal(six, ref)
    layers = m.iegmn_original.iegmn_layers
    assert layers[1].packed(dev).descriptor(6).dev.mma_products == 6
    assert layers[0].packed(dev).descriptor(3).dev.mma_products == 0       # layer 0 is never switched


def test_bf16x3_eager_graphed_pipelined_bitwise(cuda_device):
    """In bf16x3 mode the eager forward, GraphedForward and PipelinedInference return the same bits, twice."""
    from equidock_public_b200 import hetero_graph as hg
    from equidock_public_b200 import synthetic
    from equidock_public_b200.serving import PipelinedInference
    dev = cuda_device
    m = gio.build_model('dips', dev)
    m.precision = 'bf16x3'
    host = hg.batch_pairs(synthetic.to_torch_pairs(synthetic.synthetic_batch(12, 90, 70, seed=5))).pin_memory()
    g = host.to(dev)
    eager = [m(g, epoch=0) for _ in range(2)]
    ref = m.iegmn_original.last_outputs
    ref = {k: ref[k].clone() for k in ('ligand_coors', 'rotation', 'translation')}
    assert all(torch.equal(a, b) for a, b in zip(eager[0][0], eager[1][0]))
    gf = m.graphed(g)
    for _ in range(2):
        raw = gf.launch().raw_result()
        for k, v in ref.items():
            assert torch.equal(raw[k], v), k
    for use_graph in (True, False):
        outs = list(PipelinedInference(m, dev, use_cuda_graph=use_graph).run(host for _ in range(3)))
        for o in outs:
            o['_event'].synchronize()
            for k, v in ref.items():
                assert torch.equal(o[k].to(dev), v), (use_graph, k)


# ---- refusals -------------------------------------------------------------------------------------------------------

def test_bf16x3_refused_under_autograd_and_in_training(cuda_device):
    from equidock_public_b200.training import DataParallelTrainer
    dev = cuda_device
    g = _small_batch(dev)
    m = gio.build_model('dips', dev)
    m.precision = 'bf16x3'
    m.train()
    with pytest.raises(NotImplementedError, match='bf16x3'):
        m(g, epoch=0)
    with pytest.raises(NotImplementedError, match='bf16x3'):
        m.iegmn_original(g, 0)
    with pytest.raises(NotImplementedError, match='bf16x3'):
        DataParallelTrainer(m, lr=1e-4)
    with torch.no_grad():       # inference under no_grad is fine in training mode
        m(g, epoch=0)
    m.eval()
    m.precision = 'fp32'
    tr = DataParallelTrainer(m, lr=1e-4)
    m.precision = 'bf16x3'
    with pytest.raises(NotImplementedError, match='bf16x3'):
        tr.step(g, None)


def test_mma_products_refused_through_the_c_abi(cuda_device):
    """mma_products = 3 on the 69-wide layer 0, and any value other than 0 / 3 / 6, return EQD_ERR_UNSUPPORTED from the
    tensor-core entry points; so does the whole forward with such a layer 0."""
    from equidock_public_b200.engine import IEGMNEngine
    dev, lib = cuda_device, nat.load()
    g, plan = _fbatch('ragged', dev)
    N, G = plan.N, C.byref(plan.struct)
    _, lay0, _ = _layer(0, dev)
    _, lay1, _ = _layer(1, dev)
    proj = torch.zeros(N, 344, device=dev)
    x = _coords(g, dev).contiguous()
    aggr, xo = torch.zeros(N, 64, device=dev), torch.zeros(N, 3, dtype=torch.float64, device=dev)
    st = torch.zeros(plan.n_pairs + 1, dtype=torch.int32, device=dev)
    h0 = torch.zeros(N, 72, device=dev)
    kv = torch.zeros(lib.eqd_kv_blocks_bytes(N), dtype=torch.uint8, device=dev)
    x5 = torch.zeros(((N + 7) // 8 + 8) * 8, 16, device=dev)
    h = torch.zeros(N, 64, device=dev)
    P = nat.ptr
    for lay, bad in ((lay0, 3), (lay0, 5), (lay1, 5), (lay1, -1), (lay1, 12)):
        d = C.byref(_desc(lay, bad))
        assert lib.eqd_edge_stage(G, d, P(proj), P(x), P(x), P(aggr), P(xo), P(st), None) == -2, (lay.dh, bad)
        if lay.dh == 69:
            assert lib.eqd_project_tc0(G, d, P(h0), P(proj), P(kv), P(x5), None) == -2
            assert lib.eqd_node_mlp_tc0(G, d, P(h0), P(aggr), P(h0), P(h), None) == -2
            assert lib.eqd_node_stage_tc0(G, d, None, P(h0), P(proj), P(aggr), P(kv), P(x5), P(h0), P(h), None,
                                          None) == -2
        else:
            assert lib.eqd_project_tc(G, d, P(h), P(proj), P(kv), None) == -2
            assert lib.eqd_node_mlp_tc(G, d, P(h), P(aggr), P(h), P(h0), P(h), None) == -2
            assert lib.eqd_node_stage_tc(G, d, None, P(h), P(h0), P(proj), P(aggr), P(kv), P(h), P(h), None, None) == -2
    # the whole forward with a layer 0 that asks for three products
    m = gio.build_model('dips', dev)
    packed = [lay.packed(dev) for lay in m.iegmn_original.iegmn_layers]
    bad0 = _desc(packed[0], 3)
    orig = packed[0].descriptor
    packed[0].descriptor = lambda products=0: bad0
    try:
        with pytest.raises(nat.NativeLibraryError, match='EQD_ERR_UNSUPPORTED'):
            m(g, epoch=0)
    finally:
        packed[0].descriptor = orig
    torch.cuda.synchronize()


# ---- all 125 shipped pairs end to end ---------------------------------------------------------------------------------

BASELINE = {'db5': {'crmsd': (14.14, 14.73, 5.31), 'irmsd': (11.97, 13.23, 4.93)},
            'dips': {'crmsd': (13.30, 14.53, 7.14), 'irmsd': (10.19, 11.92, 7.01)}}


def _np(t):
    return t.detach().cpu().numpy()


@pytest.mark.parametrize('ds', ['db5', 'dips'])
def test_bf16x3_all_shipped_pairs_rmsd_table(ds, cuda_device):
    """Compact inputs -> GPU graph build -> engine in bf16x3 mode -> batched RMSD meter on every shipped pair of a set:
    per pair, C-alpha coordinates and rotation against the fp64 oracle on the same GPU-built inputs within 256 times the
    bf16x6 bounds of test_gpu_acceptance.py; the BASELINE.md section 1 table at its printed precision."""
    import iegmn_oracle as orc
    from equidock_public_b200 import hetero_graph as hg
    from equidock_public_b200.engine import GraphPlan
    from equidock_public_b200.eval import Meter_Unbound_Bound
    from equidock_public_b200.graph_build import ResidueBatch, build_graphs
    from test_gpu_acceptance import _interface
    names, allp = gio.load_all(ds)
    model = gio.build_model(ds, cuda_device)
    model.precision = 'bf16x3'
    sd, cfg = gio.load_checkpoint(ds), orc.OracleConfig.from_args(gio.load_args(ds))
    R, T, rows = {}, {}, []
    order = sorted(names, key=lambda n: allp[n]['lig']['nca_c'].shape[0] + allp[n]['rec']['nca_c'].shape[0])
    for c0 in range(0, len(order), 25):
        chunk = order[c0:c0 + 25]
        g = build_graphs(ResidueBatch([(allp[n]['lig'], allp[n]['rec']) for n in chunk]), cuda_device)
        coors, _, _, rot, trans = model(g, epoch=0)
        for n, r, t, co, part in zip(chunk, rot, trans, coors, hg.unbatch(g)):
            R[n], T[n] = _np(r).astype(np.float64), _np(t).astype(np.float64).reshape(3)
            f = lambda nt, et, new_x: {'src': _np(part.edges(etype=et)[0]), 'dst': _np(part.edges(etype=et)[1]),
                                       'he': _np(part.edges[et].data['he']), 'res_feat': _np(part.nodes[nt].data['res_feat']),
                                       'x': _np(part.nodes[nt].data['x']), 'mu_r_norm': _np(part.nodes[nt].data['mu_r_norm']),
                                       **({'new_x': _np(part.nodes[nt].data['new_x'])} if new_x else {})}
            ref = orc.forward_pair(sd, cfg, f('ligand', 'll', True), f('receptor', 'rr', False))
            err = float(np.abs(_np(co) - ref['ligand_coors']).max())
            rerr = float(np.abs(R[n] - ref['rotation']).max())
            terr = float(np.abs(T[n] - ref['translation'].reshape(3)).max())
            rows.append((n, err, 256 * max(1e-4, allp[n]['yard']), rerr, terr))
    rows.sort(key=lambda r: -r[1] / r[2])
    print(f'\n{ds} bf16x3: worst coords err / bound = {rows[0][1] / rows[0][2]:.3f}; max coords err {max(r[1] for r in rows):.2e} A, '
          f'max rotation err {max(r[3] for r in rows):.2e}, max translation err {max(r[4] for r in rows):.2e} A')
    for n, err, bound, rerr, terr in rows:
        print(f'  {n}: coords {err:.2e} (bound {bound:.2e}) rotation {rerr:.2e} translation {terr:.2e}')
    assert all(r[1] <= r[2] for r in rows), rows[:5]
    assert all(r[3] <= 256 * 3e-5 for r in rows), sorted(rows, key=lambda r: -r[3])[:5]

    def table(sel):
        lp, rp, lt, rt, nl, nr = [], [], [], [], [], []
        for n in names:
            e = allp[n]['ca']
            pred = ((R[n] @ e['ligand_in'].astype(np.float64).T).T + T[n]).astype(np.float32)
            li, ri = sel(e)
            lp.append(pred[li]); lt.append(e['ligand_gt'][li]); rp.append(e['receptor_gt'][ri]); rt.append(e['receptor_gt'][ri])
            nl.append(len(li)); nr.append(len(ri))
        z = torch.zeros(0, dtype=torch.int32, device=cuda_device)
        he = torch.zeros(0, 27, device=cuda_device)
        plan = GraphPlan(nl, nr, z, z, z, z, he, he, cuda_device)
        tt = lambda L: torch.from_numpy(np.concatenate(L)).to(cuda_device)
        out = Meter_Unbound_Bound().update_rmsd_batch(plan, tt(lp), tt(rp), tt(lt), tt(rt)).cpu().numpy()[:, 0]
        return float(np.median(out)), float(np.mean(out)), float(np.std(out))
    c = table(lambda e: (np.arange(e['ligand_gt'].shape[0]), np.arange(e['receptor_gt'].shape[0])))
    i = table(lambda e: _interface(e['ligand_gt'], e['receptor_gt']))
    print(f'{ds} bf16x3: C-RMSD median/mean/std = {c[0]:.2f}/{c[1]:.2f}/{c[2]:.2f}   I-RMSD = {i[0]:.2f}/{i[1]:.2f}/{i[2]:.2f}')
    # the criterion test_gpu_acceptance.py holds the default mode to
    for got, ref in zip(c, BASELINE[ds]['crmsd']):
        assert abs(got - ref) < 0.0151, (ds, 'crmsd', c)
    for got, ref in zip(i, BASELINE[ds]['irmsd']):
        assert abs(got - ref) < 0.0151, (ds, 'irmsd', i)
