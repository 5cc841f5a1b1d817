"""GPU (H100): every forward entry point (edge stage, layer-0 and 64-wide node stage, keypoint head, Kabsch, embedding)
called directly on seeded inputs and compared with a torch fp64 evaluation of the same formula (tests/fp64_stages.py and
the references below; rigid_docking_model.py line numbers).  The forward counterpart of test_gpu_backward_kernels.py,
whose batches (`bulk`, `ragged`, `long`), Report and _twice it reuses.

`bench` is the db5-shaped step batch of bench.py: 330 pairs of 200 + 200 nodes, k = 10 (132 000 nodes, 1.32 M edges,
11 000 edge tiles, 1032 node tiles, 660 proteins: the head's u kernel loops over two stripes of 512 proteins).

Tolerance: max |kernel - reference| over every row, relative to the largest reference magnitude of the tensor (no
LeakyReLU kink exclusion: forward outputs are continuous in the pre-activations).  Kernels with bf16x3 operands or fp32
arithmetic: 1e-5, except the layer-0 attention with sharpened logits (4e-5, justified in that test).  The fp64 stages
of the head: 1e-12 (m_qk, ymean, cov 1e-14; u 1e-13).  The coordinate update is compared as
x_out - (eta x_orig + (1 - eta) x_in), relative to the largest update.  Measured on an H100 80GB HBM3 (700 W power
limit), largest value over the cases of each test (`pytest -s` prints every value):
  edge stage       tensor cores: aggr 3.5e-7, update 2.5e-7;  fp32 kernel: aggr 6.7e-7, update 4.2e-7
  layer 0, TC      Psrc 2.0e-7, Pdst 1.8e-7, Q 1.9e-7, K / V blocks 1.7e-7, x5 1.7e-7, mu 2.1e-6 (sharpened 1.4e-5),
                   node MLP 3.8e-7;  node stage: mu 3.0e-6, h_out 1.5e-6, proj_next 2.0e-7, layer-1 K / V 1.9e-7
  layer 0, fp32    proj 4.1e-7, h_out 6.0e-6, proj_next 4.5e-7, K / V blocks 4.2e-7
  64-wide TC       bench batch: mu 4.3e-7, h_out 3.6e-7, proj_next 2.0e-7, next K / V blocks 2.0e-7
  head             m_qk 0, u 0, keypts 2.4e-15, ymean 3.8e-16, cov 6.6e-16 (each from the kernel's own inputs);
                   qbar 2.7e-7; keypoints end to end 7.9e-7 (vs backward_manual.head_forward 9.6e-7)
  Kabsch           rot, trans and ligand_out within 1 fp32 ulp, sing within 1e-12 relative
The file runs in about 20 s on that GPU.
"""
import ctypes as C
import hashlib

import numpy as np
import pytest
import torch

import backward_manual as bm
import fp64_stages as fs
import golden_io as gio
import iegmn_oracle as orc
from equidock_public_b200 import _native as nat
from equidock_public_b200 import synthetic
from equidock_public_b200.engine import GraphPlan
from test_gpu_backward_kernels import _CACHE, Report, _batch, _d, _layer, _model, _twice

pytestmark = pytest.mark.gpu

F64 = torch.float64
ETA = float(np.float32(0.3))     # x_connection_init as the kernels see it (fp32 in eqd_layer_params)
SIZES = [1, 8, 63, 64, 65, 127, 128, 129, 2000]
SENT = -777.25                   # pre-fill of outputs a kernel writes in part (finite: _twice compares bitwise)


def _fpairs(kind):
    if kind == 'bench':
        return synthetic.synthetic_batch(330, seed=37)
    if kind == 'sizes':           # proteins of every query-tile / key-chunk edge, one of 2000 nodes
        rng = np.random.default_rng(38)
        return [synthetic.synthetic_pair(rng, a, b, 10) for a, b in zip(SIZES, SIZES[::-1])]
    if kind == 'head_sizes':      # keypoint chunks: nc <= 32, 64-row chunks, 128-row head_mean tiles
        rng = np.random.default_rng(39)
        s = [1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 2000]
        return [synthetic.synthetic_pair(rng, a, b, 10) for a, b in zip(s, s[::-1])]
    if kind == 'p257':            # 514 proteins: a second u stripe holding 2
        rng = np.random.default_rng(40)
        return [synthetic.synthetic_pair(rng, 3 + i % 5, 2 + i % 7, 10) for i in range(257)]
    if kind == 'mixed':           # k = 10 tiles mixing nodes of in-degree 0, 1, 9 and 10; proteins of 1 and 2 nodes
        rng = np.random.default_rng(41)
        pairs = [synthetic.synthetic_pair(rng, a, b, 10) for a, b in ((40, 33), (1, 2), (2, 1), (61, 47))]
        for i, side in ((0, 0), (3, 1)):
            prot = dict(pairs[i][side])
            n = prot['x'].shape[0]
            want = np.full(n, 10)
            want[1::7], want[3::7], want[5::11] = 0, 1, 9
            first = np.searchsorted(prot['dst'], prot['dst'])
            keep = (np.arange(prot['dst'].shape[0]) - first) < want[prot['dst']]
            for key in ('src', 'dst', 'he'):
                prot[key] = prot[key][keep]
            pairs[i] = (prot, pairs[i][1]) if side == 0 else (pairs[i][0], prot)
        return pairs
    if kind.startswith('k'):      # k in-edges per node (proteins larger than k), plus proteins of 1 and 2 nodes
        k = int(kind[1:])
        rng = np.random.default_rng(42 + k)
        return [synthetic.synthetic_pair(rng, k + 37, k + 20, k), synthetic.synthetic_pair(rng, 2, 1, k),
                synthetic.synthetic_pair(rng, 2 * k + 9, 3, k)]
    raise ValueError(kind)


def _fbatch(kind, dev, bound=None):
    """(graph, plan) of a named batch, built once per session; `bound` plans the same graph with another
    max_in_degree."""
    if kind in ('bulk', 'ragged', 'long'):
        g, plan = _batch(kind, dev)
    else:
        if kind not in _CACHE:
            k = int(kind[1:]) if kind.startswith('k') else 10
            g = gio.make_batch(_fpairs(kind), dev)
            _CACHE[kind] = (g, GraphPlan.from_graph(g, dev, k))
        g, plan = _CACHE[kind]
    if bound is not None and bound != plan.struct.max_in_degree:
        key = (kind, bound)
        if key not in _CACHE:
            _CACHE[key] = (g, GraphPlan.from_graph(g, dev, bound))
        g, plan = _CACHE[key]
    return g, plan


def _coords(g, dev):
    from equidock_public_b200.hetero_graph import LIGAND, RECEPTOR
    return torch.cat([g.nodes[LIGAND].data['new_x'], g.nodes[RECEPTOR].data['x']]).to(dev, F64)


def _np_gen(seed, dev):
    rng = np.random.default_rng(seed)
    return lambda *shape, s=1.0: torch.from_numpy((rng.standard_normal(shape) * s).astype(np.float32)).to(dev)


def _decode_kv(kv, N):
    """K and V [N][64] of bf16x3 8-node blocks, as the sum of their three splits."""
    ng = (N + 7) // 8 + 8
    blocks = kv.view(torch.bfloat16).view(2, 3, ng, 8, 8, 8).double().sum(1)      # [which][n/8][d/8][n%8][d%8]
    dec = blocks.permute(0, 1, 3, 2, 4).reshape(2, ng * 8, 64)[:, :N]
    return dec[0], dec[1]


def _with_eta(lay, eta):
    """A copy of a packed layer's descriptor with another x_connection_init (the cached layer keeps its own)."""
    s = nat.EqdLayer.from_buffer_copy(lay.struct)
    s.dev.x_connection_init = eta
    return s


# ---- edge stage ---------------------------------------------------------------------------------------------------

def _edge_run(fn, plan, lay_struct, proj, x_in, x_orig, dev):
    N, B = plan.N, plan.n_pairs

    def run():
        aggr = torch.full((N, 64), float('nan'), device=dev)
        xo = torch.full((N, 3), float('nan'), dtype=F64, device=dev)
        st = torch.zeros(B + 1, dtype=torch.int32, device=dev)
        nat.check(fn(C.byref(plan.struct), C.byref(lay_struct), nat.ptr(proj), nat.ptr(x_in), nat.ptr(x_orig),
                     nat.ptr(aggr), nat.ptr(xo), nat.ptr(st), None), 'edge stage')
        return aggr, xo, st

    aggr, xo, st = _twice(run)
    assert int(st.abs().sum()) == 0, 'status words must stay 0'
    return aggr, xo


def _edge_case(kind, li, eta, dev, bound=None, coincide=False):
    """Runs eqd_edge_stage and eqd_edge_stage_ffma on one batch and layer; returns their outputs and the fp64 reference."""
    g, plan = _fbatch(kind, dev, bound)
    mod, lay, tp = _layer(li, dev)
    N, pw = plan.N, 128 + 3 * tp.dhp
    r = _np_gen(900 + li, dev)
    proj = r(N, pw, s=0.5).contiguous()
    x_in = _coords(g, dev) + torch.tensor([1.0e3, -0.7e3, 0.4e3], dtype=F64, device=dev)
    if coincide:      # one edge with identical endpoints: d = 0, every RBF = 1
        e = plan.E_l + 5
        x_in[plan.edge_dst[e].long()] = x_in[plan.col_src[e].long()]
    x_in = x_in.contiguous()
    x_orig = (x_in + r(N, 3, s=3.0).double()).contiguous()
    st = _with_eta(lay, eta)
    tc = _edge_run(nat.load().eqd_edge_stage, plan, st, proj, x_in, x_orig, dev)
    ff = _edge_run(nat.load().eqd_edge_stage_ffma, plan, st, proj, x_in, x_orig, dev)
    aggr, xupd = fs.edge_stage(mod, plan, _d(proj), x_in)
    base = ETA * x_orig + (1.0 - ETA) * x_in if eta else x_in
    return plan, tc, ff, aggr, xupd, base


def _edge_report(name, outs, aggr, xupd, base):
    rep = Report(name)
    for tag, (a, xo) in outs:
        rep.rel(f'{tag} aggr', a, aggr)
        rep.rel(f'{tag} update', xo - base, xupd)
    rep.check()


@pytest.mark.parametrize('kind,li,eta', [('bench', 1, 0.0), ('bench', 0, ETA), ('bulk', 0, 0.0), ('bulk', 1, ETA),
                                         ('ragged', 0, ETA), ('ragged', 1, 0.0), ('long', 1, ETA), ('long', 0, 0.0),
                                         ('mixed', 1, ETA), ('mixed', 0, 0.0)])
def test_edge_stage_vs_fp64(kind, li, eta, cuda_device):
    """Layer 0 (projection rows of 344 floats) and layer 1 (320), x_connection_init 0 and 0.3 with x_orig != x_in,
    coordinates around 1e3 A.  `bench` and `bulk` give every warpgroup chain many tiles; `mixed` has tiles of
    degree-10 nodes next to nodes of degree 0, 1 and 9 (the fixed-degree path off) and proteins of 1 and 2 nodes."""
    plan, tc, ff, aggr, xupd, base = _edge_case(kind, li, eta, cuda_device)
    if kind in ('bench', 'bulk'):
        assert (plan.N + 5) // 6 >= 3 * 132 * 4
    if kind == 'mixed':
        deg = (plan.row_ptr[1:] - plan.row_ptr[:-1]).cpu()
        assert all(int((deg == d).sum()) > 0 for d in (0, 1, 9, 10))
    isolated = (plan.row_ptr[1:] - plan.row_ptr[:-1]) == 0
    if bool(isolated.any()):
        for a, _ in (tc, ff):
            assert float(a[isolated].abs().max()) == 0.0
    _edge_report(f'edge[{kind}, L{li}, eta {eta:.1f}]', (('tc', tc), ('ffma', ff)), aggr, xupd, base)


@pytest.mark.parametrize('k', [1, 2, 10, 11, 21, 32, 33, 64, 65, 70, 128])
def test_edge_stage_tile_shapes_vs_fp64(k, cuda_device):
    """max_in_degree = k: tensor-core tiles of min(64 // k, 32) nodes up to 64 (one node per tile), the fp32 route
    above.  Layer 0, eta = 0.3, one edge of length 0."""
    plan, tc, ff, aggr, xupd, base = _edge_case(f'k{k}', 0, ETA, cuda_device, coincide=k > 2)
    assert int((plan.row_ptr[1:] - plan.row_ptr[:-1]).max()) == k
    if k > 64:
        assert torch.equal(tc[0], ff[0]) and torch.equal(tc[1], ff[1])
    _edge_report(f'edge[k{k}]', (('tc', tc), ('ffma', ff)), aggr, xupd, base)


def test_edge_stage_loose_bounds_bitwise(cuda_device):
    """The k = 10 `ragged` graph planned with max_in_degree 10, 12, 32 and 64: tiles of 6, 5, 2 and 1 nodes.  Every
    edge row is computed the same way whatever the tile, so the tensor-core outputs are bitwise equal; 65 takes the fp32
    route and is compared with fp64."""
    ref = None
    for bound in (10, 12, 32, 64, 65):
        plan, tc, ff, aggr, xupd, base = _edge_case('ragged', 1, ETA, cuda_device, bound=bound)
        assert plan.struct.max_in_degree == bound
        if bound <= 64:
            if ref is None:
                ref = tc
            assert torch.equal(tc[0], ref[0]) and torch.equal(tc[1], ref[1]), bound
        _edge_report(f'edge[ragged, bound {bound}]', (('tc', tc), ('ffma', ff)), aggr, xupd, base)


# ---- layer 0 on the tensor cores and on the fp32 CUDA cores ----------------------------------------------------------

def _l0_inputs(plan, dev, seed, scale=1.0):
    N = plan.N
    r = _np_gen(seed, dev)
    h0 = torch.zeros(N, 72, device=dev)
    h0[:, :69] = r(N, 69, s=scale)
    return h0, r(N, 64, s=0.3)


def _project_tc0(plan, lay, h0, dev):
    lib, N = nat.load(), plan.N
    rows = ((N + 7) // 8 + 8) * 8

    def run():
        proj = torch.full((N, 344), SENT, device=dev)
        kv = torch.zeros(lib.eqd_kv_blocks_bytes(N), dtype=torch.uint8, device=dev)
        x5 = torch.full((rows, 16), float('nan'), device=dev)
        x5[N:] = 0.0
        nat.check(lib.eqd_project_tc0(C.byref(plan.struct), C.byref(lay.struct), nat.ptr(h0), nat.ptr(proj), nat.ptr(kv),
                                      nat.ptr(x5), None), 'eqd_project_tc0')
        return proj, kv, x5

    return _twice(run)


def _qkv69(proj, kv, x5, N):
    """Q, K, V [N][69] as eqd_attention_tc0 reads them: channels 0..63 from proj / the K/V blocks, 64..68 from x5."""
    K, V = _decode_kv(kv, N)
    x = _d(x5[:N])
    return (torch.cat([_d(proj[:, 128:192]), x[:, 10:15]], 1), torch.cat([K, x[:, 0:4], x[:, 8:9]], 1),
            torch.cat([V, x[:, 4:8], x[:, 9:10]], 1))


@pytest.mark.parametrize('kind', ['bench', 'ragged', 'long', 'sizes'])
def test_layer0_tc_kernels_vs_fp64(kind, cuda_device):
    """eqd_project_tc0, eqd_attention_tc0 (also with logits sharpened by h0 x 3) and eqd_node_mlp_tc0, each on its own
    inputs."""
    dev, lib = cuda_device, nat.load()
    _, plan = _fbatch(kind, dev)
    mod, lay, _ = _layer(0, dev)
    N, seg = plan.N, plan.seg_ptr_host
    rep = Report(f'layer0 tc[{kind}]')
    # Sharpened logits reach |s| ~ 950; the kernel rounds them to fp32 (|s| 2^-24 ~ 6e-5), which moves the softmax
    # weights by that much relative: measured 1.4e-5 on the bench batch, bound 4e-5 as for the backward attention.
    sharp = Report(f'layer0 tc[{kind}] sharpened logits', 4e-5)
    for scale in (1.0, 3.0):
        h0, aggr = _l0_inputs(plan, dev, 1000, scale)
        proj, kv, x5 = _project_tc0(plan, lay, h0, dev)
        ref = fs.projections(mod, _d(h0[:, :69]))
        tag = '' if scale == 1.0 else ' (sharp)'
        if scale == 1.0:
            rep.rel('Psrc', proj[:, 0:64], ref['Psrc'])
            rep.rel('Pdst', proj[:, 64:128], ref['Pdst'])
            rep.rel('Q[0:64]', proj[:, 128:192], ref['Q'][:, :64])
            K, V = _decode_kv(kv, N)
            rep.rel('K[0:64] blocks', K, ref['K'][:, :64])
            rep.rel('V[0:64] blocks', V, ref['V'][:, :64])
            x5_ref = torch.cat([ref['K'][:, 64:68], ref['V'][:, 64:68], ref['K'][:, 68:69], ref['V'][:, 68:69],
                                ref['Q'][:, 64:69]], 1)
            rep.rel('x5[0:15]', x5[:N, :15], x5_ref)
            assert float(x5[:N, 15].abs().max()) == 0.0 and float(x5[N:].abs().max()) == 0.0
        q, k, v = _qkv69(proj, kv, x5, N)

        def attn():
            mu = torch.full((N, 72), float('nan'), device=dev)
            nat.check(lib.eqd_attention_tc0(C.byref(plan.struct), nat.ptr(proj), nat.ptr(kv), nat.ptr(x5), nat.ptr(mu),
                                            None), 'eqd_attention_tc0')
            return (mu,)

        mu, = _twice(attn)
        (rep if scale == 1.0 else sharp).rel('mu[:, :69]' + tag, mu[:, :69], fs.attention(seg, q, k, v))
        assert float(mu[:, 69:].abs().max()) == 0.0, 'mu columns 69..71 must be written as 0'
    # LeakyReLU is positively homogeneous: h0 x 3 scales every logit by exactly 9
    logits = max(float((q[int(seg[s]):int(seg[s + 1])] @ k[int(seg[p]):int(seg[p + 1])].t()).abs().max())
                 for s, p in ((0, plan.n_pairs), (plan.n_pairs, 0)))
    print(f'\nsharpened attention: max |logit| = {logits:.1f}')
    sharp.check()

    h0, aggr = _l0_inputs(plan, dev, 1001)
    mu = torch.zeros(N, 72, device=dev)
    mu[:, :69] = _np_gen(1002, dev)(N, 69, s=0.5)
    ref = fs.node_mlp(mod, _d(h0[:, :69]), _d(aggr), _d(mu[:, :69]), _d(h0[:, :69]))
    counts = [1, 63, 64, 65, N] if kind == 'bench' else [N]
    for n in counts:
        gn = nat.EqdGraph.from_buffer_copy(plan.struct)
        gn.n_nodes = n

        def mlp():
            out = torch.full((N, 64), SENT, device=dev)
            nat.check(lib.eqd_node_mlp_tc0(C.byref(gn), C.byref(lay.struct), nat.ptr(h0), nat.ptr(aggr), nat.ptr(mu),
                                           nat.ptr(out), None), 'eqd_node_mlp_tc0')
            return (out,)

        out, = _twice(mlp)
        rep.rel(f'node_mlp n={n}', out[:n], ref[:n])
        assert bool((out[n:] == SENT).all()), 'rows >= n must be left untouched'
    rep.check()


def _layer1_next(mod1, h_out, pn, kv, N, rep, tag):
    ref = fs.projections(mod1, _d(h_out))
    rep.rel(f'{tag} proj_next Psrc', pn[:, 0:64], ref['Psrc'])
    rep.rel(f'{tag} proj_next Pdst', pn[:, 64:128], ref['Pdst'])
    rep.rel(f'{tag} proj_next Q', pn[:, 128:192], ref['Q'])
    K, V = _decode_kv(kv, N)
    rep.rel(f'{tag} next K blocks', K, ref['K'])
    rep.rel(f'{tag} next V blocks', V, ref['V'])


@pytest.mark.parametrize('kind', ['bench', 'ragged', 'long', 'sizes'])
def test_layer0_node_stage_tc0_and_panelless_fp32_route_vs_fp64(kind, cuda_device):
    """eqd_node_stage_tc0 with p_next = layer 1 (h_out; Psrc | Pdst | Q of proj_next; layer 1's K/V blocks), and the
    fp32 CUDA-core route of a layer 0 without tensor-core panels: eqd_project (ldh 72), eqd_node_stage at dh 69 with its
    attention output mu [n][72] (what the training stash keeps for such a layer), eqd_kv_blocks."""
    dev, lib = cuda_device, nat.load()
    _, plan = _fbatch(kind, dev)
    mod, lay, _ = _layer(0, dev)
    mod1, lay1, _ = _layer(1, dev)
    N, seg = plan.N, plan.seg_ptr_host
    G, L, Ln = C.byref(plan.struct), C.byref(lay.struct), C.byref(lay1.struct)
    h0, aggr = _l0_inputs(plan, dev, 1003)
    h069 = _d(h0[:, :69])
    rep = Report(f'layer0 node stage[{kind}]')

    proj, kv, x5 = _project_tc0(plan, lay, h0, dev)
    mu_ref = fs.attention(seg, *_qkv69(proj, kv, x5, N))

    def tc0():
        kv2 = kv.clone()
        mu = torch.full((N, 72), float('nan'), device=dev)
        h_out = torch.full((N, 64), float('nan'), device=dev)
        pn = torch.full((N, 320), SENT, device=dev)
        nat.check(lib.eqd_node_stage_tc0(G, L, Ln, nat.ptr(h0), nat.ptr(proj), nat.ptr(aggr), nat.ptr(kv2), nat.ptr(x5),
                                         nat.ptr(mu), nat.ptr(h_out), nat.ptr(pn), None), 'eqd_node_stage_tc0')
        return mu, h_out, pn, kv2

    mu, h_out, pn, kv2 = _twice(tc0)
    rep.rel('tc0 mu', mu[:, :69], mu_ref)
    rep.rel('tc0 h_out', h_out, fs.node_mlp(mod, h069, _d(aggr), mu_ref, h069))
    _layer1_next(mod1, h_out, pn, kv2, N, rep, 'tc0')

    def fp32():
        p = torch.full((N, 344), SENT, device=dev)
        nat.check(lib.eqd_project(G, L, nat.ptr(h0), 72, nat.ptr(p), None), 'eqd_project')
        mu = torch.full((N, 72), SENT, device=dev)
        h_out = torch.full((N, 64), float('nan'), device=dev)
        pn = torch.full((N, 320), SENT, device=dev)
        nat.check(lib.eqd_node_stage(G, L, Ln, nat.ptr(h0), 72, nat.ptr(h0), nat.ptr(p), nat.ptr(aggr), nat.ptr(mu),
                                     nat.ptr(h_out), nat.ptr(pn), None), 'eqd_node_stage')
        kvf = torch.zeros(lib.eqd_kv_blocks_bytes(N), dtype=torch.uint8, device=dev)
        nat.check(lib.eqd_kv_blocks(G, nat.ptr(pn), 320, 192, 256, nat.ptr(kvf), None), 'eqd_kv_blocks')
        return p, mu, h_out, pn, kvf

    p, mu, h_out, pn, kvf = _twice(fp32)
    ref = fs.projections(mod, h069)
    for name, base in (('Psrc', 0), ('Pdst', 64), ('Q', 128), ('K', 200), ('V', 272)):
        w = 64 if name.startswith('P') else 69
        rep.rel(f'fp32 proj {name}', p[:, base:base + w], ref[name])
    mu_ref = fs.attention(seg, _d(p[:, 128:197]), _d(p[:, 200:269]), _d(p[:, 272:341]))
    rep.rel('fp32 mu', mu[:, :69], mu_ref)
    assert torch.equal(mu[:, 69:], torch.zeros(N, 3, device=dev))      # the padded V columns are 0
    rep.rel('fp32 h_out', h_out, fs.node_mlp(mod, h069, _d(aggr), mu_ref, h069))
    _layer1_next(mod1, h_out, pn, kvf, N, rep, 'fp32')
    rep.rel('fp32 proj_next K, V (fp32 columns)', pn[:, 192:320],
            torch.cat([fs.projections(mod1, _d(h_out))[c] for c in ('K', 'V')], 1))
    rep.check()


def test_node_stage_tc_bench_vs_fp64(cuda_device):
    """eqd_node_stage_tc of layer 1 (p_next = layer 2) on the bench batch: mu, h_out and proj_next against fp64."""
    dev, lib = cuda_device, nat.load()
    _, plan = _fbatch('bench', dev)
    mod, lay, _ = _layer(1, dev)
    mod2, lay2, _ = _layer(2, dev)
    N, seg = plan.N, plan.seg_ptr_host
    G, L, Ln = C.byref(plan.struct), C.byref(lay.struct), C.byref(lay2.struct)
    r = _np_gen(1100, dev)
    h, aggr = r(N, 64, s=0.7), r(N, 64, s=0.3)
    h0 = torch.zeros(N, 72, device=dev)
    h0[:, :69] = r(N, 69)
    proj = torch.zeros(N, 320, device=dev)
    kv = torch.zeros(lib.eqd_kv_blocks_bytes(N), dtype=torch.uint8, device=dev)
    nat.check(lib.eqd_project_tc(G, L, nat.ptr(h), nat.ptr(proj), None, None), 'eqd_project_tc')
    nat.check(lib.eqd_project_tc(G, L, nat.ptr(h), nat.ptr(proj), nat.ptr(kv), None), 'eqd_project_tc')

    def run():
        kv2 = kv.clone()
        mu = torch.full((N, 64), float('nan'), device=dev)
        h_out = torch.full((N, 64), float('nan'), device=dev)
        pn = torch.full((N, 320), SENT, device=dev)
        nat.check(lib.eqd_node_stage_tc(G, L, Ln, nat.ptr(h), nat.ptr(h0), nat.ptr(proj), nat.ptr(aggr), nat.ptr(kv2),
                                        nat.ptr(mu), nat.ptr(h_out), nat.ptr(pn), None), 'eqd_node_stage_tc')
        return mu, h_out, pn, kv2

    mu, h_out, pn, kv2 = _twice(run)
    rep = Report('node stage tc[bench]')
    P = _d(proj)
    mu_ref = fs.attention(seg, P[:, 128:192], P[:, 192:256], P[:, 256:320])
    rep.rel('mu', mu, mu_ref)
    rep.rel('h_out', h_out, fs.node_mlp(mod, _d(h), _d(aggr), mu_ref, _d(h0[:, :69])))
    _layer1_next(mod2, h_out, pn, kv2, N, rep, 'L2')
    rep.check()


# ---- keypoint head --------------------------------------------------------------------------------------------------

def _head_ws_views(ws, plan):
    """qbar [2B][64] and u [2B][50][64] inside the eqd_keypoints workspace (layout in include/eqd_iegmn.h)."""
    a256 = lambda v: (v + 255) // 256 * 256
    B = plan.n_pairs
    off = a256(max(plan.n_node_tiles, 1) * 64 * 4) + a256((2 * B + 1) * 4)
    qbar = ws[off:off + 2 * B * 64 * 8].view(F64).view(2 * B, 64)
    off += a256(2 * B * 64 * 8)
    u = ws[off:off + 2 * B * nat.HEADS * 64 * 8].view(F64).view(2 * B, nat.HEADS, 64)
    return qbar, u


def _seg_ids(plan, dev):
    seg = torch.from_numpy(plan.seg_ptr_host).to(dev)
    return torch.repeat_interleave(torch.arange(2 * plan.n_pairs, device=dev), seg[1:] - seg[:-1])


def _partner(B, dev):
    s = torch.arange(2 * B, device=dev)
    return torch.where(s < B, s + B, s - B)


def _keypts_ref(plan, h64, x, u):
    out = []
    for s in range(2 * plan.n_pairs):
        a, b = int(plan.seg_ptr_host[s]), int(plan.seg_ptr_host[s + 1])
        att = torch.softmax(h64[a:b] @ u[s].t(), 0)           # [n][50], softmax over the protein's nodes (:546)
        out.append(att.t() @ x[a:b])
    return torch.stack(out)


@pytest.mark.parametrize('kind,case', [('bench', 'plain'), ('p257', 'plain'), ('head_sizes', 'plain'),
                                       ('head_sizes', 'zero_h'), ('ragged', 'sharp'), ('bench', 'offset')])
def test_keypoint_head_vs_fp64(kind, case, cuda_device):
    """eqd_head_fold and eqd_keypoints, each fp64 stage from the kernel's own inputs: m_qk, qbar (the fp32 GEMM),
    u = m_qk[k]^T qbar[partner] (the stripe loop over > 512 proteins), keypoints, their means and covariances; then the
    keypoints end to end against backward_manual.head_forward on sampled pairs."""
    dev, lib = cuda_device, nat.load()
    g, plan = _fbatch(kind, dev)
    model, _ = _model(dev)
    net = model.iegmn_original
    head = net.packed_head(dev)
    B, N = plan.n_pairs, plan.N
    h = _np_gen(1200, dev)(N, 64, s=0.7)
    x = _coords(g, dev)
    if case == 'offset':
        x = x + torch.tensor([1.0e3, -0.7e3, 0.4e3], dtype=F64, device=dev)
    if case == 'zero_h':
        zs = B                                                # the receptor of 2000 nodes
        h[int(plan.seg_ptr_host[zs]):int(plan.seg_ptr_host[zs + 1])] = 0.0
    if case == 'sharp':
        h = h * 6.0
    x = x.contiguous()
    ws_bytes = int(lib.eqd_workspace_bytes(N, plan.n_node_tiles, B))

    def run():
        ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device=dev)
        m = torch.full((nat.HEADS, 64, 64), float('nan'), dtype=F64, device=dev)
        nat.check(lib.eqd_head_fold(C.byref(head.struct), nat.ptr(m), None), 'eqd_head_fold')
        kp = torch.full((2 * B, nat.HEADS, 3), float('nan'), dtype=F64, device=dev)
        ym = torch.full((2 * B, 3), float('nan'), dtype=F64, device=dev)
        cov = torch.full((B, 9), float('nan'), dtype=F64, device=dev)
        nat.check(lib.eqd_keypoints(C.byref(plan.struct), C.byref(head.struct), nat.ptr(h), nat.ptr(x), nat.ptr(ws),
                                    ws_bytes, nat.ptr(kp), nat.ptr(ym), nat.ptr(cov), None), 'eqd_keypoints')
        qbar, u = _head_ws_views(ws, plan)
        return m, qbar.clone(), u.clone(), kp, ym, cov

    m, qbar, u, kp, ym, cov = _twice(run)
    slope = float(net.leakyrelu_neg_slope)
    wq = _d(net.att_mlp_query_ROT[0].weight).view(nat.HEADS, 64, 64)      # [k][e][d']
    wk = _d(net.att_mlp_key_ROT[0].weight).view(nat.HEADS, 64, 64)        # [k][e][d]
    m_ref = torch.einsum('kec,ked->kcd', wq, wk) / 8.0
    lin = net.mlp_h_mean_ROT[0]
    h64 = _d(h)
    pre = torch.nn.functional.leaky_relu(h64 @ _d(lin.weight).t() + _d(lin.bias), slope)
    seg = torch.from_numpy(plan.seg_ptr_host).to(dev)
    n_seg = (seg[1:] - seg[:-1]).to(F64)[:, None]
    qbar_ref = torch.zeros(2 * B, 64, dtype=F64, device=dev).index_add_(0, _seg_ids(plan, dev), pre) / n_seg
    part = _partner(B, dev)
    u_ref = torch.einsum('kcd,sc->skd', _d(m), qbar[part])
    kp_ref = _keypts_ref(plan, h64, x, u)
    ym_ref = kp.mean(1)
    yc = kp - ym_ref[:, None]
    cov_ref = torch.einsum('bkr,bkc->brc', yc[B:], yc[:B]).reshape(B, 9)

    tight = Report(f'head[{kind}, {case}] fp64 stages', 1e-12)
    tight.rel('m_qk (1e-14)', m, m_ref)
    tight.rel('u (1e-13)', u, u_ref)
    tight.rel('keypts', kp, kp_ref)
    tight.rel('ymean (1e-14)', ym, ym_ref)
    tight.rel('cov (1e-14)', cov, cov_ref)
    tight.check()
    for tag, tol in (('m_qk', 1e-14), ('u', 1e-13), ('ymean', 1e-14), ('cov', 1e-14)):
        err = next(e for t, e in tight.rows if t.startswith(tag))
        assert err <= tol, (tag, err)
    rep = Report(f'head[{kind}, {case}]')
    rep.rel('qbar (fp32 GEMM)', qbar, qbar_ref)
    kp_e2e = _keypts_ref(plan, h64, x, torch.einsum('kcd,sc->skd', m_ref, qbar_ref[part]))
    rep.rel('keypts end to end', kp, kp_e2e)
    rep.check()
    if case == 'zero_h':
        a, b = int(plan.seg_ptr_host[zs]), int(plan.seg_ptr_host[zs + 1])
        centroid = x[a:b].mean(0)
        assert float((kp[zs] - centroid).abs().max()) <= 1e-12 * float(x[a:b].abs().max())
    if case == 'sharp':
        lg = max(float((h64[int(seg[s]):int(seg[s + 1])] @ u[s].t()).abs().max()) for s in range(2 * B))
        print(f'\nsharpened: max |logit| = {lg:.0f}')
    # end to end against the numpy fp64 head of oracle/backward_manual.py on sampled pairs (the last ones sit in the
    # second u stripe of the bench and p257 batches)
    sd, cfg = gio.load_checkpoint('dips'), orc.OracleConfig.from_args(gio.load_args('dips'))
    e2e = Report(f'head[{kind}, {case}] vs backward_manual.head_forward')
    hn, xn = h64.cpu().numpy(), x.cpu().numpy()
    for b in sorted({0, B // 2, B - 2, B - 1}):
        (la, lb), (ra, rb) = (int(seg[b]), int(seg[b + 1])), (int(seg[B + b]), int(seg[B + b + 1]))
        c = bm.head_forward(sd, cfg, hn[la:lb], xn[la:lb], hn[ra:rb], xn[ra:rb])
        e2e.rel(f'keypts pair {b} ligand', kp[b], torch.from_numpy(c['Y'][0]).to(dev))
        e2e.rel(f'keypts pair {b} receptor', kp[B + b], torch.from_numpy(c['Y'][1]).to(dev))
    e2e.check()


# ---- Kabsch + rigid transform -----------------------------------------------------------------------------------------

def _rand_rot(rng):
    q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
    return q * np.sign(np.linalg.det(q))


def _kabsch_cases(rng):
    """(name, A, compare rot) with A = U diag(S) V^T."""
    def mk(S, reflect=False, scale=1.0):
        U, V = _rand_rot(rng), _rand_rot(rng)
        A = U @ np.diag(S) @ V.T * scale
        return -A if reflect else A
    cases = [('random', mk([9.0, 4.0, 1.5]), True), ('reflection', mk([7.0, 3.0, 0.8], reflect=True), True),
             ('rank 2', mk([5.0, 2.0, 0.0]), False), ('zero', np.zeros((3, 3)), False),
             ('min S 0.9e-3', mk([3.0, 1.0, 0.9e-3]), False), ('min S 1.1e-3', mk([3.0, 1.0, 1.1e-3]), False),
             ('gap 0.9e-2', mk([3.0, np.sqrt(1.0 + 0.9e-2), 1.0]), False),
             ('gap 1.1e-2', mk([3.0, np.sqrt(1.0 + 1.1e-2), 1.0]), False),
             ('scale 1e-6', mk([9.0, 4.0, 1.5], scale=1e-6), True), ('scale 1e6', mk([9.0, 4.0, 1.5], scale=1e6), True),
             ('nan', mk([9.0, 4.0, 1.5]), False), ('random 2', mk([20.0, 6.0, 2.5], reflect=True), True)]
    cases[10][1][1, 2] = np.nan
    return cases


def _kabsch_batch(dev):
    if 'kabsch' not in _CACHE:
        rng = np.random.default_rng(43)
        lig = [1, 127, 128, 129, 300, 1, 127, 128, 129, 300, 2, 64]
        g = gio.make_batch([synthetic.synthetic_pair(rng, n, 3, 10) for n in lig], dev)
        _CACHE['kabsch'] = (g, GraphPlan.from_graph(g, dev, 10))
    return _CACHE['kabsch']


def _kabsch_run(plan, cov, ym, xl, mask, dev, fill=None):
    B = plan.n_pairs
    o = fill() if fill else (torch.full((B, 9), float('nan'), device=dev), torch.full((B, 3), float('nan'), device=dev),
                             torch.full((plan.N_l, 3), float('nan'), device=dev),
                             torch.full((B, 3), float('nan'), dtype=F64, device=dev),
                             torch.zeros(B, dtype=torch.int32, device=dev))
    nat.check(nat.load().eqd_kabsch_apply(C.byref(plan.struct), nat.ptr(cov), nat.ptr(ym), nat.ptr(xl), nat.ptr(mask),
                                          *[nat.ptr(t) for t in o], None), 'eqd_kabsch_apply')
    return o


def test_kabsch_apply_vs_numpy(cuda_device):
    """eqd_kabsch_apply on covariances built as U diag(S) V^T: proper and reflected, rank 2, zero, singular values on
    either side of the 1e-3 / 1e-2 guard thresholds, a NaN entry, scales 1e-6 and 1e6; ligands of 1 .. 300 nodes (the
    128-thread loop).  rot / trans within 1 fp32 ulp + 1e-12 of numpy's fp64 Kabsch where the rotation is well
    conditioned, sing within 1e-12 relative, ligand_out within 1 fp32 ulp, and the status bits."""
    dev = cuda_device
    g, plan = _kabsch_batch(dev)
    B = plan.n_pairs
    cases = _kabsch_cases(np.random.default_rng(44))
    assert len(cases) == B
    A = np.stack([c[1] for c in cases])
    rng = np.random.default_rng(45)
    ym_np = rng.uniform(-50, 50, size=(2 * B, 3))
    cov = torch.from_numpy(A.reshape(B, 9).copy()).to(dev)
    ym = torch.from_numpy(ym_np).to(dev)
    xl = (_coords(g, dev)[:plan.N_l].float() + 20.0).contiguous()
    # the NaN pair's outputs are NaN: compare the two runs with NaN mapped to a sentinel
    finite = lambda o: tuple(t.nan_to_num(SENT) if t.is_floating_point() else t for t in o)
    rot, trans, lo, sing, status = _twice(lambda: finite(_kabsch_run(plan, cov, ym, xl, None, dev)))
    rot, trans, lo, sing, status = (t.cpu().numpy() for t in (rot, trans, lo, sing, status))
    xl_np = xl.double().cpu().numpy()
    seg = plan.seg_ptr_host
    ulp = lambda v: float(np.spacing(np.float32(np.abs(v).max())))
    for b, (name, Ab, cmp_rot) in enumerate(cases):
        if name == 'nan':
            assert status[b] & nat.STATUS_NAN, name
            continue
        U, S, Vt = np.linalg.svd(Ab)
        flag = orc.svd_guard_flags(S.astype(np.float32))
        assert bool(status[b] & nat.STATUS_SVD_DEGENERATE) == flag, (name, S, status[b])
        assert not status[b] & nat.STATUS_NAN
        assert np.abs(sing[b] - S).max() <= 1e-12 * S[0], (name, sing[b], S)
        if name == 'rank 2':
            assert flag
        if not cmp_rot:
            continue
        T = U @ np.diag([1.0, 1.0, np.sign(np.linalg.det(Ab))]) @ Vt
        assert abs(np.linalg.det(T) - 1.0) < 1e-12
        t = ym_np[B + b] - T @ ym_np[b]
        assert np.abs(rot[b] - T.reshape(-1)).max() <= ulp(T) + 1e-12, name
        assert np.abs(trans[b] - t).max() <= ulp(t) + 1e-12 * np.abs(ym_np).max(), name
        pts = xl_np[seg[b]:seg[b + 1]]
        out = pts @ T.T + t
        assert np.abs(lo[seg[b]:seg[b + 1]] - out).max() <= ulp(out), name
    assert bool(status[2] & nat.STATUS_SVD_DEGENERATE) and bool(status[3] & nat.STATUS_SVD_DEGENERATE)


def test_kabsch_apply_pair_mask(cuda_device):
    """pair_mask: masked-out pairs keep every sentinel (rot, trans, sing, status, ligand rows) bitwise; masked-in
    pairs are bitwise those of an unmasked call."""
    dev = cuda_device
    g, plan = _kabsch_batch(dev)
    B = plan.n_pairs
    cases = _kabsch_cases(np.random.default_rng(46))
    cov = torch.from_numpy(np.stack([c[1] for c in cases]).reshape(B, 9).copy()).to(dev)
    ym = torch.from_numpy(np.random.default_rng(47).uniform(-50, 50, size=(2 * B, 3))).to(dev)
    xl = (_coords(g, dev)[:plan.N_l].float() - 5.0).contiguous()
    full = _kabsch_run(plan, cov, ym, xl, None, dev)
    mask = torch.tensor([b % 2 for b in range(B)], dtype=torch.int32, device=dev)
    sentinels = lambda: (torch.full((B, 9), -3.5, device=dev), torch.full((B, 3), 7.25, device=dev),
                         torch.full((plan.N_l, 3), -11.0, device=dev), torch.full((B, 3), 13.5, dtype=F64, device=dev),
                         torch.full((B,), 0x55, dtype=torch.int32, device=dev))
    masked = _kabsch_run(plan, cov, ym, xl, mask, dev, fill=sentinels)
    torch.cuda.synchronize()
    fresh = sentinels()
    seg = plan.seg_ptr_host
    for b in range(B):
        rows = slice(int(seg[b]), int(seg[b + 1]))
        src = full if b % 2 else fresh
        for i, (got, want) in enumerate(zip(masked, src)):
            part = (lambda t: t[rows]) if i == 2 else (lambda t: t[b])
            assert torch.equal(part(got), part(want)), (b, i)


# ---- embedding ------------------------------------------------------------------------------------------------------

RESIDUES = [(0.0, True), (20.0, True), (20.9, True), (-0.5, True), (-1.0, False), (21.0, False), (1e10, False),
            (float('inf'), False), (float('-inf'), False), (float('nan'), False)]


def test_embed_vs_fp64_and_residue_range(cuda_device):
    """eqd_embed_checked: h0[:, :64] is the embedding row of .long()(res) bitwise (20.9 -> 20, -0.5 -> 0), h0[:, 64:69]
    = log(mu) within 2 fp32 ulp, columns 69..71 exactly 0, x64 exact; EQD_STATUS_BAD_RESIDUE exactly for ids outside
    [0, 21) -- NaN included."""
    dev, lib = cuda_device, nat.load()
    g, plan = _fbatch('ragged', dev)
    N, NL, B = plan.N, plan.N_l, plan.n_pairs
    rng = np.random.default_rng(48)
    emb = torch.from_numpy(rng.standard_normal((nat.N_RES_TYPES, 64)).astype(np.float32)).to(dev)
    mu = torch.from_numpy(rng.uniform(1e-3, 2.0, size=(N, 5)).astype(np.float32)).to(dev)
    xs = torch.from_numpy((rng.standard_normal((N, 3)) * 300).astype(np.float32)).to(dev)

    def call(res):
        h0 = torch.full((N, 72), float('nan'), device=dev)
        x64 = torch.full((N, 3), float('nan'), dtype=F64, device=dev)
        st = torch.zeros(B + 1, dtype=torch.int32, device=dev)
        rl, rr = res[:NL].contiguous(), res[NL:].contiguous()
        nat.check(lib.eqd_embed_checked(C.byref(plan.struct), nat.ptr(emb), nat.ptr(rl), nat.ptr(rr), nat.ptr(mu[:NL]),
                                        nat.ptr(mu[NL:].contiguous()), nat.ptr(xs[:NL]), nat.ptr(xs[NL:].contiguous()),
                                        nat.ptr(h0), nat.ptr(x64), nat.ptr(st), None), 'eqd_embed_checked')
        return h0, x64, st

    res = torch.from_numpy(rng.integers(0, 21, size=N).astype(np.float32)).to(dev)
    good = [v for v, ok in RESIDUES if ok]
    res[:len(good)] = torch.tensor(good, device=dev)
    res[NL:NL + len(good)] = torch.tensor(good, device=dev)
    h0, x64, st = _twice(lambda: call(res))
    assert int(st.abs().sum()) == 0
    idx = torch.from_numpy(np.trunc(res.cpu().numpy()).astype(np.int64)).to(dev)
    assert torch.equal(h0[:, :64], emb[idx])
    logmu = torch.log(mu.double())
    ulp = torch.from_numpy(np.spacing(np.abs(logmu.float().cpu().numpy()))).to(dev).double()
    assert bool(((h0[:, 64:69].double() - logmu).abs() <= 2 * ulp).all())
    assert float(h0[:, 69:].abs().max()) == 0.0
    assert torch.equal(x64, xs.double())
    for v, ok in RESIDUES:
        for node in (3, NL + 5):                     # a ligand and a receptor node
            bad = res.clone()
            bad[node] = v
            _, _, st = call(bad)
            torch.cuda.synchronize()
            assert bool(int(st[B]) & nat.STATUS_BAD_RESIDUE) == (not ok), (v, node)
            assert int(st[:B].abs().sum()) == 0


# ---- bit pins -------------------------------------------------------------------------------------------------------

def _edge_bits(dev):
    """sha256 of aggr and x_out of eqd_edge_stage (layer 1) on the bulk batch, inputs from numpy's seeded generator."""
    g, plan = _batch('bulk', dev)
    _, lay, _ = _layer(1, dev)
    N = plan.N
    r = _np_gen(1300, dev)
    proj = r(N, 320, s=0.5).contiguous()
    x_in = (_coords(g, dev) + 1.0e3).contiguous()
    x_orig = (x_in + r(N, 3).double()).contiguous()
    aggr, xo = _edge_run(nat.load().eqd_edge_stage, plan, _with_eta(lay, ETA), proj, x_in, x_orig, dev)
    digest = hashlib.sha256()
    for t in (aggr, xo):
        digest.update(t.cpu().numpy().tobytes())
    return digest.hexdigest()


def _node_stage_tc0_bits(dev):
    """sha256 of everything eqd_node_stage_tc0 writes (mu, h_out, Psrc | Pdst | Q of proj_next, layer 1's K/V blocks)
    on the bulk batch, inputs from numpy's seeded generator."""
    lib = nat.load()
    _, plan = _batch('bulk', dev)
    _, lay, _ = _layer(0, dev)
    _, lay1, _ = _layer(1, dev)
    N = plan.N
    h0, aggr = _l0_inputs(plan, dev, 1301)
    proj, kv, x5 = _project_tc0(plan, lay, h0, dev)
    mu, h_out, pn = torch.zeros(N, 72, device=dev), torch.zeros(N, 64, device=dev), torch.zeros(N, 320, device=dev)
    nat.check(lib.eqd_node_stage_tc0(C.byref(plan.struct), C.byref(lay.struct), C.byref(lay1.struct), nat.ptr(h0),
                                     nat.ptr(proj), nat.ptr(aggr), nat.ptr(kv), nat.ptr(x5), nat.ptr(mu), nat.ptr(h_out),
                                     nat.ptr(pn), None), 'eqd_node_stage_tc0')
    torch.cuda.synchronize()
    digest = hashlib.sha256()
    for t in (mu, h_out, pn[:, :192].contiguous(), kv):
        digest.update(t.cpu().numpy().tobytes())
    return digest.hexdigest()


# Every per-element sum of these kernels keeps its order (split products, chunk sums, softmax row chains, the per-node
# aggregation), so a change of summation order shows here even inside the 1e-5 tolerance of the comparisons above.
EDGE_STAGE_SHA256 = 'fab087a8fa4dc9de8a98fa8adfd05e4a18bbb7a3053ea58261522244521bca03'
NODE_STAGE_TC0_SHA256 = 'b3c4f095a820d37e70a2ec9f58c3115817bb56aed320208857341c0976a4d4b5'


def test_edge_stage_bits_pinned(cuda_device):
    digest = _edge_bits(cuda_device)
    print(f'\nedge stage sha256 {digest}')
    assert digest == EDGE_STAGE_SHA256


def test_node_stage_tc0_bits_pinned(cuda_device):
    digest = _node_stage_tc0_bits(cuda_device)
    print(f'\nnode stage tc0 sha256 {digest}')
    assert digest == NODE_STAGE_TC0_SHA256
