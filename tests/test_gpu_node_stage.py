"""GPU: the tensor-core node stage of a 64-wide layer (cross attention on 64-row query tiles, node MLP, next layer's
projections and K/V blocks) against its fp32 CUDA-core twin eqd_node_stage, at the tile and chunk boundaries."""
import ctypes as C
import hashlib

import numpy as np
import pytest
import torch

import golden_io as gio
from equidock_public_b200 import _native as nat
from equidock_public_b200 import synthetic
from equidock_public_b200.engine import GraphPlan

pytestmark = pytest.mark.gpu

# (ligand, receptor) sizes.  Proteins of 1, 8, 63, 64, 65, 127, 128, 129 and 200 nodes: 64-row query tiles with one valid
# row, with none (a 128-row tile whose second half is empty) and full ones.  785 ligand nodes in all, so every receptor
# key range starts inside an 8-node block; receptors of 5 and 1 nodes are shorter than one block, those of 127 and more
# cross a 64-key chunk boundary.
RAGGED = [(1, 129), (8, 200), (63, 5), (64, 127), (65, 128), (127, 64), (128, 63), (129, 8), (200, 1)]


def _node_stage_bits(dev):
    """sha256 of everything eqd_node_stage_tc writes (mu, h_out, Psrc | Pdst | Q of proj_next, the next layer's K/V
    blocks) for the RAGGED pairs plus 4 pairs of 200 + 200 nodes, on inputs drawn from numpy's seeded generator."""
    lib = nat.load()
    rng = np.random.default_rng(11)
    pairs = [synthetic.synthetic_pair(rng, a, b, 10) for a, b in RAGGED] + synthetic.synthetic_batch(4, seed=2)
    plan = GraphPlan.from_graph(gio.make_batch(pairs, dev), dev, 10)
    N = plan.N
    net = gio.build_model('dips', dev).iegmn_original
    lay, lay_next = net.iegmn_layers[1].packed(dev), net.iegmn_layers[2].packed(dev)
    G, L, Ln = C.byref(plan.struct), C.byref(lay.struct), C.byref(lay_next.struct)
    f = lambda *shape: torch.from_numpy(rng.standard_normal(shape).astype(np.float32)).to(dev)
    h, aggr = f(N, 64) * 0.7, f(N, 64) * 0.3
    h0 = torch.zeros(N, 72, device=dev)
    h0[:, :69] = f(N, 69)
    proj = torch.zeros(N, 320, device=dev)
    kv = torch.zeros(lib.eqd_kv_blocks_bytes(N), dtype=torch.uint8, device=dev)
    assert lib.eqd_project_tc(G, L, nat.ptr(h), nat.ptr(proj), nat.ptr(kv), None) == 0
    mu, h_out, pn = torch.zeros(N, 64, device=dev), torch.zeros(N, 64, device=dev), torch.zeros(N, 320, device=dev)
    assert lib.eqd_node_stage_tc(G, L, Ln, nat.ptr(h), nat.ptr(h0), nat.ptr(proj), nat.ptr(aggr), nat.ptr(kv),
                                 nat.ptr(mu), nat.ptr(h_out), nat.ptr(pn), None) == 0
    torch.cuda.synchronize()
    digest = hashlib.sha256()
    for t in (mu, h_out, pn[:, :192].contiguous(), kv):
        digest.update(t.cpu().numpy().tobytes())
    return digest.hexdigest()


# The bits of the shared-memory 128-row attention and projection kernels, which the warpgroup-chain kernels reproduce
# (computed with both builds: equal).  Every per-element sum keeps
# its order (the split products, the chunk- and piece-wise round-to-nearest sums, the softmax row-sum chains), so a
# change of summation order shows here even where it stays inside the 1e-5 tolerance of the comparisons below.
NODE_STAGE_SHA256 = '2346c7c983fd362bad14a167edc313a334fb037fae4f2eb0846f9f6ecf0de546'


def test_node_stage_bits_pinned(cuda_device):
    assert _node_stage_bits(cuda_device) == NODE_STAGE_SHA256


def _rel_err(a, ref):
    return float((a.double() - ref.double()).abs().max()) / max(1.0, float(ref.double().abs().max()))


@pytest.mark.parametrize('n_bulk', [0, 80])
def test_node_stage_tensor_core_vs_fp32_twin_with_mu(n_bulk, cuda_device):
    """The tensor-core node stage against its fp32 CUDA-core twin, and the attention output mu of both (the fp32 twin
    writes it when given a buffer) against fp64.  n_bulk = 80 adds 80 pairs of 200 + 200 nodes: 640 query tiles of 64 rows, more than the resident tile chains hold,
    so every chain runs several tiles and prefetches across them.  n_nodes is not a multiple of 64 in either case."""
    dev = cuda_device
    lib = nat.load()
    rng = np.random.default_rng(64)
    pairs = [synthetic.synthetic_pair(rng, a, b, 10) for a, b in RAGGED] + synthetic.synthetic_batch(n_bulk, seed=1)
    plan = GraphPlan.from_graph(gio.make_batch(pairs, dev), dev, 10)
    N, B = plan.N, plan.n_pairs
    assert N % 64 != 0
    net = gio.build_model('dips', dev).iegmn_original
    lay, lay_next = net.iegmn_layers[1].packed(dev), net.iegmn_layers[2].packed(dev)
    G, L, Ln = C.byref(plan.struct), C.byref(lay.struct), C.byref(lay_next.struct)
    torch.manual_seed(5)
    h = torch.randn(N, 64, device=dev) * 0.7
    h0 = torch.zeros(N, 72, device=dev)
    h0[:, :69] = torch.randn(N, 69, device=dev)
    aggr = torch.randn(N, 64, device=dev) * 0.3
    proj = torch.zeros(N, 320, device=dev)
    kv = torch.zeros(lib.eqd_kv_blocks_bytes(N), dtype=torch.uint8, device=dev)
    assert lib.eqd_project_tc(G, L, nat.ptr(h), nat.ptr(proj), None, None) == 0          # all five groups as fp32
    assert lib.eqd_project_tc(G, L, nat.ptr(h), nat.ptr(proj), nat.ptr(kv), None) == 0   # + this layer's K/V blocks

    h_ref = torch.full((N, 64), float('nan'), device=dev)
    pn_ref = torch.full((N, 320), float('nan'), device=dev)
    mu_ff = torch.full((N, 64), float('nan'), device=dev)
    assert lib.eqd_node_stage(G, L, Ln, nat.ptr(h), 64, nat.ptr(h0), nat.ptr(proj), nat.ptr(aggr), nat.ptr(mu_ff),
                              nat.ptr(h_ref), nat.ptr(pn_ref), None) == 0
    mu = torch.full((N, 64), float('nan'), device=dev)
    h_tc = torch.full((N, 64), float('nan'), device=dev)
    pn_tc = torch.full((N, 320), float('nan'), device=dev)
    assert lib.eqd_node_stage_tc(G, L, Ln, nat.ptr(h), nat.ptr(h0), nat.ptr(proj), nat.ptr(aggr), nat.ptr(kv),
                                 nat.ptr(mu), nat.ptr(h_tc), nat.ptr(pn_tc), None) == 0
    torch.cuda.synchronize()

    # mu against a torch fp64 softmax(Q K^T) V of every pair, from the same projections
    seg = plan.seg_ptr_host
    P = proj.double()
    mu_ref = torch.zeros(N, 64, dtype=torch.float64, device=dev)
    for s in range(2 * B):
        p = s + B if s < B else s - B
        q, k, v = P[seg[s]:seg[s + 1], 128:192], P[seg[p]:seg[p + 1], 192:256], P[seg[p]:seg[p + 1], 256:320]
        mu_ref[seg[s]:seg[s + 1]] = torch.softmax(q @ k.t(), 1) @ v
    assert torch.isfinite(mu).all()
    assert _rel_err(mu, mu_ref) <= 1e-5
    assert torch.isfinite(mu_ff).all()
    assert _rel_err(mu_ff, mu_ref) <= 1e-5

    assert torch.isfinite(h_tc).all()
    assert _rel_err(h_tc, h_ref) <= 1e-5
    assert torch.isfinite(pn_tc[:, :192]).all()
    assert _rel_err(pn_tc[:, :192], pn_ref[:, :192]) <= 1e-5
    # the next layer's K and V blocks, decoded as the sum of their three bf16 splits
    ng = (N + 7) // 8 + 8
    blocks = kv.view(torch.bfloat16).view(2, 3, ng, 8, 8, 8).double().sum(1)      # [which][n/8][d/8][n%8][d%8]
    kv_dec = blocks.permute(0, 1, 3, 2, 4).reshape(2, ng * 8, 64)[:, :N]
    assert _rel_err(kv_dec[0], pn_ref[:, 192:256]) <= 1e-5
    assert _rel_err(kv_dec[1], pn_ref[:, 256:320]) <= 1e-5
