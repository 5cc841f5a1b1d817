"""CPU: the C-ABI library loads and exports every symbol include/eqd_iegmn.h declares; host-side logic
(graph container, batch plan, weight repacking, launch accounting) -- no kernel is launched here."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import golden_io as gio
from equidock_public_b200 import _native as nat
from equidock_public_b200 import hetero_graph as hg
from equidock_public_b200 import synthetic
from equidock_public_b200.engine import GraphPlan, IEGMNEngine, PackedHead, PackedLayer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    with open(os.path.join(ROOT, 'include', 'eqd_iegmn.h')) as fh:
        return fh.read()


def test_library_exports_every_declared_symbol():
    declared = set(re.findall(r'^\s*(?:int|size_t|void\*?|float)\s+(eqd_\w+)\s*\(', _header(), flags=re.M))
    assert declared == set(nat.PROTOTYPES), (declared ^ set(nat.PROTOTYPES))
    lib = nat.load()
    for name in declared:
        assert getattr(lib, name) is not None
    assert lib.eqd_abi_version() == nat.ABI_VERSION


def test_header_constants_match_binding():
    h = _header()
    for name, val in (('EQD_EDGE_FEATS', nat.EDGE_FEATS), ('EQD_N_RBF', nat.N_RBF), ('EQD_HID', nat.HID),
                      ('EQD_H0', nat.H0), ('EQD_H0_PAD', nat.H0_PAD), ('EQD_HEADS', nat.HEADS),
                      ('EQD_TILE_ROWS', nat.TILE_ROWS), ('EQD_ABI_VERSION', nat.ABI_VERSION)):
        assert int(re.search(rf'#define {name} (\d+)', h).group(1)) == val


def test_abi_v11_struct_layouts_are_natural_c_layouts():
    assert ctypes.sizeof(nat.EqdGraph) == 24 + 6 * 8 + 8 + 8
    assert nat.EqdGraph.seg_ptr.offset == 24 and nat.EqdGraph.node_tiles.offset == 80
    assert nat.EqdLayerParams.w_proj.offset == 8 and nat.EqdLayerParams.b_coor2.offset == 8 + 10 * 8
    assert nat.EqdLayerParams.w_edge_tc.offset == 96 and nat.EqdLayerParams.w_node_tc.offset == 104
    assert nat.EqdLayerParams.w_proj_tc.offset == 112 and nat.EqdLayerParams.w_node1.offset == 120
    # eqd_layer = device part first (a binding may upload / keep it wholesale), host constants BY VALUE after it
    assert nat.EqdLayer.dev.offset == 0 and nat.EqdLayer.consts.offset == ctypes.sizeof(nat.EqdLayerParams)
    assert ctypes.sizeof(nat.EqdLayerConsts) == (5 * 64 + 304 + 320) * 4
    assert not any(n.endswith('_host') for n, _ in nat.EqdLayerParams._fields_)
    assert ctypes.sizeof(nat.EqdHeadParams) == 5 * 8 + 8
    assert nat.EqdHeadParams.m_qk.offset == 32 and nat.EqdHeadParams.leaky_slope.offset == 40
    assert ctypes.sizeof(nat.EqdForwardIO) == 18 * 8 + 16 and nat.EqdForwardIO.stage_events.offset == 17 * 8
    assert nat.EqdForwardIO.train_stash.offset == 18 * 8 and nat.EqdForwardIO.train_stash_bytes.offset == 19 * 8


def _header_struct_fields(name):
    """Field names of `typedef struct <name> { ... } <name>;` in declaration order (comments stripped)."""
    body = re.search(r'typedef struct %s \{(.*?)\} %s;' % (name, name), _header(), flags=re.S).group(1)
    body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
    fields = []
    for decl in body.split(';'):
        decl = decl.strip()
        if not decl:
            continue
        for part in decl.split(','):
            fields.append(re.findall(r'(\w+)\s*$', re.sub(r'(\[\d+\])+\s*$', '', part.strip()))[0])   # name, array extents dropped
    return fields


@pytest.mark.parametrize('cname,ctype', [('eqd_graph', nat.EqdGraph), ('eqd_layer_params', nat.EqdLayerParams),
                                         ('eqd_head_params', nat.EqdHeadParams), ('eqd_forward_io', nat.EqdForwardIO),
                                         ('eqd_layer_consts', nat.EqdLayerConsts), ('eqd_layer', nat.EqdLayer)])
def test_ctypes_structs_list_the_header_fields_in_order(cname, ctype):
    assert _header_struct_fields(cname) == [f[0] for f in ctype._fields_]


def test_forward_workspace_bytes_host_arithmetic():
    lib = nat.load()
    g = nat.EqdGraph()
    g.n_pairs, g.n_nodes, g.n_node_tiles = 256, 102400, 1024
    need = lib.eqd_forward_workspace_bytes(ctypes.byref(g))
    # two projection buffers (344 floats per node) dominate; everything is 256-byte aligned
    assert need > 2 * 102400 * 344 * 4 and need % 256 == 0
    assert need >= lib.eqd_kv_blocks_bytes(102400) + lib.eqd_workspace_bytes(102400, 1024, 256)
    assert lib.eqd_forward_workspace_bytes(None) == 0


def test_workspace_bytes_host_arithmetic():
    lib = nat.load()
    assert lib.eqd_workspace_bytes(1000, 10, 3) >= 10 * 64 * 4 + 7 * 4
    assert lib.eqd_workspace_bytes(0, 0, 0) > 0


def test_backward_workspace_covers_every_weight_gradient_reduction():
    """BackwardWorkspace's partial / colsum sizes cover eqd_tn_partial_floats (and nchunks * ncols) of every eqd_tn_gemm
    call TrainEngine.backward makes, listed here from the backward itself.  The row chunking depends on the number of
    64 x 64 output blocks, so the largest buffer is not the largest shape: at N = 40 000 the 64-wide layers' projection
    reduction (N, 64, 320) needs 16 384 floats more than the 69-wide layer's (N, 72, 344)."""
    from equidock_public_b200.training import tn_gemm_shapes, tn_workspace_floats
    lib = nat.load()

    def need(rows, K, nc):
        nch = ctypes.c_int32(0)
        return int(lib.eqd_tn_partial_floats(rows, K, nc, None, ctypes.byref(nch))), nch.value * nc

    Ns = list(range(1, 3000, 23)) + list(range(3000, 200001, 1009)) + [9600, 23700, 40000, 132000, 200000]
    for N in Ns:
        for E in (N // 2, N, 4 * N, 10 * N, 16 * N):
            partial, colsum = tn_workspace_floats(N, E)
            listed = set(tn_gemm_shapes(N, E))
            for dhp in (nat.H0_PAD, nat.HID):
                calls = [(N, 64, 64),                                                   # head: mlp_h_mean_ROT.0
                         (N, dhp, 64), (N, dhp, dhp), (N, 64, dhp), (N, nat.H0_PAD, dhp),   # node_mlp.4, node_mlp.0 blocks
                         (N, dhp, 128 + 3 * dhp),                                      # projections
                         (E, 44, 64), (E, 64, 64)]                                      # edge_mlp.0 / .4, coors_mlp.0
                for shape in calls:
                    assert shape in listed, (N, E, shape)
                    p, c = need(*shape)
                    assert p <= partial and c <= colsum, (N, E, shape, p, partial, c, colsum)
    # the batch where the parent's five-shape list fell short: 100 pairs of 200 + 200 nodes, ten edges per node
    assert need(40000, 64, 320)[0] == 2150400 <= tn_workspace_floats(40000, 400000)[0]


def test_engine_refuses_cpu_device():
    with pytest.raises(nat.NativeLibraryError):
        IEGMNEngine(torch.device('cpu'))


def test_missing_library_is_loud(monkeypatch):
    monkeypatch.setattr(nat, '_lib', None)
    monkeypatch.setattr(nat, 'LIB_PATH', '/nonexistent/libeqd_iegmn.so')
    with pytest.raises(nat.NativeLibraryError):
        nat.load()


def test_pair_graph_batch_roundtrip():
    pairs = synthetic.to_torch_pairs(synthetic.synthetic_batch(3, 17, 23, k=5, seed=1) +
                                     synthetic.synthetic_batch(1, 9, 4, k=3, seed=2))
    g = hg.batch_pairs(pairs)
    assert g.batch_num_nodes('ligand').tolist() == [17, 17, 17, 9]
    assert g.batch_num_nodes('receptor').tolist() == [23, 23, 23, 4]
    assert g.num_edges(hg.LL) == 3 * 17 * 5 + 9 * 3 and g.num_edges('rr') == 3 * 23 * 5 + 4 * 3
    s, d = g.edges(etype=('receptor', 'rr', 'receptor'))
    assert int(d.max()) == 23 * 3 + 4 - 1                       # ids are offset per type like dgl.batch
    assert g.edges['ll'].data['he'].shape == (g.num_edges(hg.LL), 27)
    assert g.num_edges(hg.CROSS_LR) == 0
    parts = hg.unbatch(g)
    assert len(parts) == 4
    for (lig, rec), one in zip(pairs, parts):
        assert torch.equal(one.nodes['ligand'].data['new_x'], lig['new_x'])
        assert torch.equal(one.edges['rr'].data['he'], rec['he'])
        assert torch.equal(one.edges(etype=hg.RR)[0], rec['src'])


def test_graph_plan_topology_on_cpu():
    pairs = synthetic.to_torch_pairs(synthetic.synthetic_batch(2, 130, 5, k=4, seed=3))
    g = hg.batch_pairs(pairs)
    plan = GraphPlan.from_graph(g, torch.device('cpu'), max_in_degree=4)
    assert plan.N == 270 and plan.N_l == 260 and plan.E == 2 * (130 * 4 + 5 * 4)
    assert plan.seg_ptr.tolist() == [0, 130, 260, 265, 270]
    rp = plan.row_ptr.numpy()
    assert rp[0] == 0 and rp[-1] == plan.E and (np.diff(rp) == 4).all()
    assert not bool(plan.unsorted)
    tiles = plan.node_tiles.view(-1, 2).tolist()                 # 130 nodes -> tiles of 128 + 2
    assert tiles == [[0, 0], [0, 128], [1, 130], [1, 258], [2, 260], [3, 265]]
    assert int(plan.col_src[plan.E_l:].min()) >= plan.N_l        # receptor ids are global
    # unsorted edges are detected (device-side flag, resolved by the slow path)
    bad = hg.batch_pairs(pairs)
    s, d = bad._edges[hg.LL]
    bad._edges[hg.LL] = (s.flip(0), d.flip(0))
    assert bool(GraphPlan.from_graph(bad, torch.device('cpu'), 4).unsorted)


@pytest.mark.parametrize('ds,li', [('dips', 0), ('dips', 3), ('db5', 1)])
def test_weight_repacking_reproduces_the_linear_layers(ds, li):
    """Packed k-major panels (with the edge-MLP split and zero padding) == the reference's nn.Linear algebra."""
    sd = {k: torch.from_numpy(v) for k, v in gio.load_checkpoint(ds).items()}
    pre = f'iegmn_original.iegmn_layers.{li}.'
    lsd = {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}
    P = PackedLayer(lsd, torch.device('cpu'), 0.75, 0.0, 0.01)
    dh, dhp = P.dh, P.dhp
    assert (dh, dhp) == ((69, 72) if li == 0 else (64, 64))
    g = torch.Generator().manual_seed(0)
    h_src, h_dst = torch.randn(5, dh, generator=g), torch.randn(5, dh, generator=g)
    ef = torch.randn(5, 42, generator=g)
    pad = lambda t, w: torch.cat([t, torch.zeros(t.shape[0], w - t.shape[1])], 1)
    proj_s = pad(h_src, dhp) @ P.t['w_proj'] + P.t['b_proj']
    proj_d = pad(h_dst, dhp) @ P.t['w_proj'] + P.t['b_proj']
    pre_act = proj_s[:, 0:64] + proj_d[:, 64:128] + pad(ef, 44) @ P.t['w_edge1']
    ref = torch.cat([h_src, h_dst, ef], 1) @ lsd['edge_mlp.0.weight'].t() + lsd['edge_mlp.0.bias']
    assert torch.allclose(pre_act, ref, atol=1e-4)
    assert torch.allclose(proj_s[:, 128:128 + dh], h_src @ lsd['att_mlp_Q.0.weight'].t(), atol=1e-4)
    assert torch.allclose(proj_s[:, 128 + 2 * dhp:128 + 2 * dhp + dh], h_src @ lsd['att_mlp_V.0.weight'].t(), atol=1e-4)
    if dhp > dh:
        assert float(proj_s[:, 128 + dh:128 + dhp].abs().max()) == 0.0          # padded columns stay zero
    aggr, mu, h0 = torch.randn(5, 64, generator=g), torch.randn(5, dh, generator=g), torch.randn(5, 69, generator=g)
    cat_p = torch.cat([pad(h_src, dhp), aggr, pad(mu, dhp), pad(h0, 72)], 1)
    hid = cat_p @ P.t['w_node1'] + P.t['b_node1']
    ref = torch.cat([h_src, aggr, mu, h0], 1) @ lsd['node_mlp.0.weight'].t() + lsd['node_mlp.0.bias']
    assert torch.allclose(hid[:, :dh], ref, atol=1e-4)
    out = pad(ref, dhp) @ P.t['w_node2'] + P.t['b_node2']
    assert torch.allclose(out, ref @ lsd['node_mlp.4.weight'].t() + lsd['node_mlp.4.bias'], atol=1e-4)


def test_module_surface_and_checkpoints_load_strict():
    import equidock_public_b200.rigid_docking_model as m
    for name in ('nn', 'math', 'torch', 'dgl', 'fn', 'sys', 'IEGMN_Layer', 'IEGMN', 'Rigid_Body_Docking_Net',
                 'compute_cross_attention', 'get_mask', 'get_non_lin', 'get_layer_norm', 'get_final_h_layer_norm',
                 'apply_final_h_layer_norm'):
        assert hasattr(m, name), name
    for ds, n_unique in (('db5', 525671), ('dips', 842477)):
        model = gio.build_model(ds, torch.device('cpu'))
        assert sum(p.numel() for p in model.parameters()) == n_unique      # SURVEY 5: unique parameter counts
    db5 = gio.build_model('db5', torch.device('cpu'))
    assert db5.iegmn_original.iegmn_layers[1] is db5.iegmn_original.iegmn_layers[4]   # shared_layers=True
    mask = m.get_mask([2, 1], [1, 3], torch.device('cpu'))
    assert mask.tolist() == [[1, 0, 0, 0], [1, 0, 0, 0], [0, 1, 1, 1]]


def test_unsupported_configurations_raise():
    import equidock_public_b200.rigid_docking_model as m
    args = gio.load_args('db5')
    args['device'] = 'cpu'
    for k, v in (('nonlin', 'swish'), ('layer_norm', 'BN'), ('fine_tune', True), ('cross_msgs', False)):
        bad = dict(args)
        bad[k] = v
        with pytest.raises(NotImplementedError):
            m.Rigid_Body_Docking_Net(bad)


def test_launch_accounting():
    assert IEGMNEngine.launches_per_forward(8) == 40 and IEGMNEngine.launches_per_forward(5) == 28


def _umma_decode(flat, n, k):
    """Inverse of engine.umma_bf16x3: 3 bf16 splits in the K-major no-swizzle core-matrix layout -> fp32 [n][k]
    (element (n,k) of a split at (k/8)*n*8 + (n/8)*64 + (n%8)*8 + (k%8) bf16 elements)."""
    parts = flat.view(3, k // 8, n // 8, 8, 8).float()          # [split][k/8][n/8][n%8][k%8]
    return parts.sum(0).permute(1, 2, 0, 3).reshape(n, k)


@pytest.mark.parametrize('ds,li', [('dips', 0), ('dips', 2), ('db5', 0), ('db5', 1)])
def test_tensor_core_panels_decode_to_the_reference_weights(ds, li):
    """The bf16x3 panels the tensor-core kernels read (edge stage, projections, node MLP; 64-wide layers and the
    69-wide layer 0 with its K = 80 padding, folded h/h0 blocks and the [K5|V5|Q5] group) reproduce the nn.Linear
    weights of the checkpoint to 3-term bf16 precision (2^-24 relative)."""
    sd = {k: torch.from_numpy(v) for k, v in gio.load_checkpoint(ds).items()}
    pre = f'iegmn_original.iegmn_layers.{li}.'
    w = {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}
    P = PackedLayer(w, torch.device('cpu'), 0.75, 0.0, 0.01)
    dh = P.dh
    close = lambda a, b: float((a - b).abs().max()) <= 2e-7 * max(1.0, float(b.abs().max()))
    # edge stage: [W1e (64 x 48) | stacked [W2 ; W3 W2] (128 x 64)]
    e = P.t['w_edge_tc'].view(torch.bfloat16) if P.t['w_edge_tc'].dtype != torch.bfloat16 else P.t['w_edge_tc']
    w1e = _umma_decode(e[:3 * 64 * 48], 64, 48)
    assert close(w1e[:, :42], w['edge_mlp.0.weight'][:, 2 * dh:]) and float(w1e[:, 42:].abs().max()) == 0.0
    w23 = _umma_decode(e[3 * 64 * 48:], 128, 64)
    assert close(w23[:64], w['edge_mlp.4.weight'])
    assert close(w23[64:], (w['coors_mlp.0.weight'].double() @ w['edge_mlp.4.weight'].double()).float())
    pj, nd = P.t['w_proj_tc'], P.t['w_node_tc']
    w1, w5, w6 = w['edge_mlp.0.weight'], w['node_mlp.0.weight'], w['node_mlp.4.weight']
    wq, wk, wv = w['att_mlp_Q.0.weight'], w['att_mlp_K.0.weight'], w['att_mlp_V.0.weight']
    if dh == 64:
        groups = [w1[:, :64], w1[:, 64:128], wq, wk, wv]
        for gi, ref in enumerate(groups):
            assert close(_umma_decode(pj[gi * 3 * 4096:(gi + 1) * 3 * 4096], 64, 64), ref)
        w5d = _umma_decode(nd[:3 * 64 * 272], 64, 272)
        assert close(w5d[:, :261], w5) and float(w5d[:, 261:].abs().max()) == 0.0
        assert close(_umma_decode(nd[3 * 64 * 272:], 64, 64), w6)
    else:   # layer 0: K = 80
        g64 = 3 * 64 * 80
        refs = [w1[:, :69], w1[:, 69:138], wq[:64], wk[:64], wv[:64]]
        for gi, ref in enumerate(refs):
            d = _umma_decode(pj[gi * g64:(gi + 1) * g64], 64, 80)
            assert close(d[:, :69], ref) and float(d[:, 69:].abs().max()) == 0.0
        x = _umma_decode(pj[5 * g64:], 16, 80)[:, :69]
        assert close(x[0:4], wk[64:68]) and close(x[4:8], wv[64:68]) and close(x[8], wk[68]) and close(x[9], wv[68])
        assert close(x[10:15], wq[64:69]) and float(x[15].abs().max()) == 0.0
        w5d = _umma_decode(nd[:3 * 80 * 224], 80, 224)
        assert close(w5d[:69, 0:69], (w5[:, 0:69].double() + w5[:, 202:271].double()).float())   # h and h0 blocks folded
        assert close(w5d[:69, 80:144], w5[:, 69:133]) and close(w5d[:69, 144:213], w5[:, 133:202])
        assert float(w5d[69:].abs().max()) == 0.0 and float(w5d[:, 69:80].abs().max()) == 0.0
        w6d = _umma_decode(nd[3 * 80 * 224:], 64, 80)
        assert close(w6d[:, :69], w6) and float(w6d[:, 69:].abs().max()) == 0.0


def test_default_bench_batch_fills_whole_rounds_of_tile_groups():
    """bench.py's headline batch (330 pairs of 200 + 200 residues per GPU) is sized to the machine: the tile kernels are persistent
    with one tile group on each of the 132 SMs of an H100, and 330 pairs give (nearly) whole rounds of attention / node / edge
    tiles where 370 pairs left the last attention round 7 % empty."""
    import math
    import bench
    B = bench.WORKLOADS['db5-shaped']['pairs_per_gpu']
    groups = 132
    def eff(b):
        tiles = {'attention': 2 * b * math.ceil(200 / nat.TILE_ROWS), 'node': math.ceil(400 * b / nat.TILE_ROWS),
                 'edge': math.ceil(400 * b / (nat.TILE_ROWS // 10))}
        return {k: (t / groups) / math.ceil(t / groups) for k, t in tiles.items()}
    e = eff(B)
    assert B == 330 and min(e.values()) > 0.97, e
    assert eff(370)['attention'] < 0.95
