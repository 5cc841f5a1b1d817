"""GPU: the tensor-core edge stage (64-row warpgroup tiles, in-degree <= 64) at its boundaries, and the fp32 route
that eqd_edge_stage takes for in-degrees in (64, 128]."""
import ctypes as C

import numpy as np
import pytest
import torch

import golden_io as gio
import iegmn_oracle as orc
from equidock_public_b200 import _native as nat
from equidock_public_b200 import synthetic
from equidock_public_b200.engine import GraphPlan

pytestmark = pytest.mark.gpu


def _np(t):
    return t.detach().cpu().numpy()


def test_in_degree_above_64_vs_oracle(cuda_device):
    """k = 70 in-edges per node, more than one 64-row tensor-core tile holds: eqd_edge_stage runs the fp32 kernel (its
    outputs are bitwise those of eqd_edge_stage_ffma), and the 8-layer DIPS model on ragged 100+90 / 75+110 pairs built
    with k = 70 matches the numpy fp64 oracle."""
    args = dict(gio.load_args('dips'), graph_max_neighbor=70)
    model = gio.build_model('dips', cuda_device, args=args)
    rng = np.random.default_rng(70)
    pairs = [synthetic.synthetic_pair(rng, 100, 90, 70), synthetic.synthetic_pair(rng, 75, 110, 70)]
    g = gio.make_batch(pairs, cuda_device)
    coors, kp_l, kp_r, rot, trans = model(g, epoch=0)
    cfg = orc.OracleConfig.from_args(args)
    checked = 0
    for i, (lig, rec) in enumerate(pairs):
        ref = orc.forward_pair(gio.load_checkpoint('dips'), cfg, lig, rec)
        if ref['kabsch']['flagged']:
            continue
        scale = max(1.0, float(np.abs(ref['ligand_coors']).max()) / 100.0)
        assert np.abs(_np(coors[i]) - ref['ligand_coors']).max() <= 2e-4 * scale, i
        assert np.abs(_np(rot[i]) - ref['rotation']).max() <= 5e-5, i
        checked += 1
    assert checked > 0
    (a_ref, x_ref), (a, x) = _edge_stage_both(g, 70, cuda_device)
    assert torch.equal(a, a_ref) and torch.equal(x, x_ref)


def _edge_stage_both(g, max_in_degree, dev):
    """One edge-stage launch of eqd_edge_stage_ffma and one of eqd_edge_stage on the same seeded inputs."""
    lib = nat.load()
    plan = GraphPlan.from_graph(g, dev, max_in_degree)
    N = plan.N
    lay = gio.build_model('dips', dev).iegmn_original.iegmn_layers[1].packed(dev)
    torch.manual_seed(0)
    proj = torch.randn(N, 128 + 3 * 64, device=dev)
    x = torch.randn(N, 3, device=dev, dtype=torch.float64) * 5
    x0 = torch.randn(N, 3, device=dev, dtype=torch.float64) * 5
    outs = []
    for fn in (lib.eqd_edge_stage_ffma, lib.eqd_edge_stage):
        aggr = torch.full((N, 64), float('nan'), device=dev)
        xo = torch.full((N, 3), float('nan'), device=dev, dtype=torch.float64)
        st = torch.zeros(plan.n_pairs + 1, dtype=torch.int32, device=dev)
        rc = fn(C.byref(plan.struct), C.byref(lay.struct), nat.ptr(proj), nat.ptr(x), nat.ptr(x0), nat.ptr(aggr),
                nat.ptr(xo), nat.ptr(st), None)
        torch.cuda.synchronize()
        assert rc == 0 and int(st.abs().sum()) == 0
        outs.append((aggr, xo))
    return outs


def test_tile_boundaries_tensor_core_vs_fp32_twin(cuda_device):
    """Nodes without in-edges, tiles straddling the ligand / receptor edge arrays (61 ligand nodes in all: not a multiple
    of the 6 nodes of a k = 10 tile) and a last tile with fewer nodes: eqd_edge_stage == eqd_edge_stage_ffma."""
    rng = np.random.default_rng(3)
    pairs = [synthetic.synthetic_pair(rng, a, b, 10) for a, b in ((23, 31), (38, 17))]
    lig, rec = pairs[0]
    keep = (lig['dst'] < 4) | (lig['dst'] >= 9)      # ligand nodes 4..8 of pair 0 lose their in-edges
    for key in ('src', 'dst', 'he'):
        lig[key] = lig[key][keep]
    rec = dict(rec)
    keep = rec['dst'] < 29                            # the last receptor nodes of pair 0 too
    for key in ('src', 'dst', 'he'):
        rec[key] = rec[key][keep]
    pairs[0] = (lig, rec)
    g = gio.make_batch(pairs, cuda_device)
    N = sum(a + b for a, b in ((23, 31), (38, 17)))
    assert N % 6 != 0 and (23 + 38) % 6 != 0
    (a_ref, x_ref), (a_tc, x_tc) = _edge_stage_both(g, 10, cuda_device)
    plan = GraphPlan.from_graph(g, cuda_device, 10)
    isolated = (plan.row_ptr[1:] - plan.row_ptr[:-1]) == 0
    assert int(isolated.sum()) >= 5
    assert float(a_tc[isolated].abs().max()) == 0.0
    _assert_twins_agree(a_ref, x_ref, a_tc, x_tc)


@pytest.mark.parametrize('k,sizes', [(64, ((70, 80), (66, 90))), (2, ((40, 37), (29, 51)))])
def test_tile_shapes_tensor_core_vs_fp32_twin(k, sizes, cuda_device):
    """max_in_degree = 64, the largest the tensor-core kernel takes (one node fills a 64-row tile), and 2 (32 nodes per
    tile, the cap: the coordinate update spans 96 threads): eqd_edge_stage == eqd_edge_stage_ffma."""
    rng = np.random.default_rng(k)
    g = gio.make_batch([synthetic.synthetic_pair(rng, a, b, k) for a, b in sizes], cuda_device)
    (a_ref, x_ref), (a_tc, x_tc) = _edge_stage_both(g, k, cuda_device)
    _assert_twins_agree(a_ref, x_ref, a_tc, x_tc)


def _assert_twins_agree(a_ref, x_ref, a_tc, x_tc):
    assert torch.isfinite(a_tc).all() and torch.isfinite(x_tc).all()
    assert float((a_tc - a_ref).abs().max()) <= 1e-5 * max(1.0, float(a_ref.abs().max()))
    assert float((x_tc - x_ref).abs().max()) <= 1e-5 * max(1.0, float(x_ref.abs().max()))

