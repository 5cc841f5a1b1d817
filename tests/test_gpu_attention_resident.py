"""GPU: the 64-wide attention with each partner protein's K / V resident in shared memory (attention64_res_kernel) against
the streaming kernel it replaces for batches whose proteins all fit (attention64_tc_kernel): mu bitwise equal in both
product modes, at the bench shape, ragged and mid-block partner ranges, every partner size around a block or chunk edge
and at capacity, query proteins of 1 to 4 non-empty 64-row halves, fewer proteins than SMs and a protein count that is
not a multiple of the grid.  Also which kernel eqd_graph.max_segment_nodes selects, that every host path that builds an
eqd_graph sets it, and mu against fp64 for one case."""
import ctypes as C

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import golden_io as gio
from bench_train import make_targets
from equidock_public_b200 import _native as nat
from equidock_public_b200 import synthetic
from equidock_public_b200.datasets import DevicePairDataset
from equidock_public_b200.engine import GraphPlan
from equidock_public_b200.formats import PairArchive, save_pairs
from equidock_public_b200.graph_build import ResidueBatch, build_graphs

pytestmark = pytest.mark.gpu

# AT_RES_MAX_NODES in attn_tc.cu: 4 chunks of 8 blocks, less the block a partner starting mid-block adds
RES_MAX_NODES = 248
SMS = 132

# A 3-residue ligand first, so that partner key ranges start at every offset inside their 8-node blocks.  Partners of
# 1..248 nodes (block and chunk edges, capacity) against queries of 1..4 non-empty 64-row halves.
PARTNERS = [1, 7, 8, 9, 15, 16, 17, 63, 64, 65, 128, RES_MAX_NODES]
QUERIES = [1, 64, 65, 129, 193, RES_MAX_NODES]
CASES = {
    'bench': [(200, 200)] * 330,
    'ragged': [(3, 5)] + [(q, p) for p in PARTNERS for q in QUERIES[::2]] + [(p, q) for p in PARTNERS for q in QUERIES[1::2]],
    'few_proteins': [(3, 65), (129, RES_MAX_NODES), (RES_MAX_NODES, 1)],
    'grid_remainder': [(3, 9)] + [(193, 129)] * 69,   # 140 proteins on 132 CTAs
}


def _kernel_names(fn, attempts=3):
    """Names of the attention64 kernels fn launches, from the CUDA activity trace of torch.profiler.  fn always launches
    one attention kernel (eqd_node_stage_tc returned 0 and wrote mu), so a trace without any attention64 launch is a
    session in which the profiler recorded none of it, not an answer: it is taken again, up to `attempts` times.  A trace
    that names the wrong kernel, or more than one, is returned as it is."""
    for i in range(attempts):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if 'attention64' in e.name}
        if names:
            return names
        print(f'\nprofiler session {i + 1} recorded no attention64 launch; kernels seen: '
              f'{sorted({e.name for e in prof.events()})[:8]}')
    return names


class _Setup:
    def __init__(self, pairs, dev, seed=0):
        self.lib = lib = nat.load()
        self.plan = plan = GraphPlan.from_graph(gio.make_batch(pairs, dev), dev, 10)
        N = plan.N
        net = gio.build_model('dips', dev).iegmn_original
        self.lay = net.iegmn_layers[1].packed(dev)
        gen = torch.Generator(device=dev).manual_seed(seed)
        h = torch.randn(N, 64, device=dev, generator=gen) * 0.7
        self.h0 = torch.zeros(N, 72, device=dev)
        self.h0[:, :69] = torch.randn(N, 69, device=dev, generator=gen)
        self.h, self.aggr = h, torch.randn(N, 64, device=dev, generator=gen) * 0.3
        self.proj = torch.zeros(N, 320, device=dev)
        self.kv = torch.zeros(lib.eqd_kv_blocks_bytes(N), dtype=torch.uint8, device=dev)
        G, L = C.byref(plan.struct), C.byref(self.lay.struct)
        assert lib.eqd_project_tc(G, L, nat.ptr(h), nat.ptr(self.proj), None, None) == 0
        assert lib.eqd_project_tc(G, L, nat.ptr(h), nat.ptr(self.proj), nat.ptr(self.kv), None) == 0
        self.dev = dev

    def mu(self, products, max_segment_nodes):
        """mu of eqd_node_stage_tc (attention, then node MLP; no next layer) with the given bound in the descriptor."""
        g = nat.EqdGraph.from_buffer_copy(self.plan.struct)
        g.max_segment_nodes = max_segment_nodes
        N = self.plan.N
        mu = torch.full((N, 64), float('nan'), device=self.dev)
        h_out = torch.empty(N, 64, device=self.dev)
        L = self.lay.descriptor(products)
        rc = self.lib.eqd_node_stage_tc(C.byref(g), C.byref(L), None, nat.ptr(self.h), nat.ptr(self.h0), nat.ptr(self.proj),
                                        nat.ptr(self.aggr), nat.ptr(self.kv), nat.ptr(mu), nat.ptr(h_out), None, None)
        assert rc == 0
        torch.cuda.synchronize()
        return mu


def _bits(t):
    return t.view(torch.int32)


@pytest.mark.parametrize('case', list(CASES))
@pytest.mark.parametrize('products', [6, 3])
def test_resident_mu_bitwise_equals_streaming(case, products, cuda_device):
    pairs = CASES[case]
    rng = np.random.default_rng(7)
    st = _Setup([synthetic.synthetic_pair(rng, a, b, 10) for a, b in pairs], cuda_device, seed=len(pairs))
    bound = st.plan.struct.max_segment_nodes
    assert bound == max(max(p) for p in pairs) <= RES_MAX_NODES
    ref = st.mu(products, 0)
    assert torch.isfinite(ref).all()
    names = _kernel_names(lambda: st.mu(products, bound))
    assert len(names) == 1 and 'attention64_res_kernel' in names.pop()
    for _ in range(2):   # every launch gives the same bits
        assert torch.equal(_bits(st.mu(products, bound)), _bits(ref))


def test_bound_selects_kernel(cuda_device):
    rng = np.random.default_rng(3)
    st = _Setup([synthetic.synthetic_pair(rng, a, b, 10) for a, b in [(3, 65), (200, 129)]], cuda_device)
    for bound, kernel in ((0, 'attention64_tc_kernel'), (RES_MAX_NODES + 1, 'attention64_tc_kernel'),
                          (RES_MAX_NODES, 'attention64_res_kernel'), (200, 'attention64_res_kernel')):
        names = _kernel_names(lambda: st.mu(6, bound))
        assert len(names) == 1 and kernel in names.pop(), bound


def test_resident_mu_vs_fp64(cuda_device):
    """mu against a torch fp64 softmax(Q K^T) V of every protein, at the bound of the existing node-stage tests."""
    rng = np.random.default_rng(9)
    pairs = CASES['ragged']
    st = _Setup([synthetic.synthetic_pair(rng, a, b, 10) for a, b in pairs], cuda_device, seed=1)
    mu = st.mu(6, st.plan.struct.max_segment_nodes)
    B, seg, P = st.plan.n_pairs, st.plan.seg_ptr_host, st.proj.double()
    ref = torch.zeros_like(P[:, :64])
    for s in range(2 * B):
        p = s + B if s < B else s - B
        q, k, v = P[seg[s]:seg[s + 1], 128:192], P[seg[p]:seg[p + 1], 192:256], P[seg[p]:seg[p + 1], 256:320]
        ref[seg[s]:seg[s + 1]] = torch.softmax(q @ k.t(), 1) @ v
    assert torch.isfinite(mu).all()
    assert float((mu.double() - ref).abs().max()) / max(1.0, float(ref.abs().max())) <= 1e-5


def _residue_protein(rng, n):
    ca = np.cumsum(rng.normal(0, 2.2, (n, 3)), axis=0).astype(np.float32)
    nca_c = np.stack([ca + rng.normal(0, 1, (n, 3)), ca, ca + rng.normal(0, 1, (n, 3))], axis=1).astype(np.float32)
    return {'atoms': ca, 'atom_ptr': np.arange(n + 1, dtype=np.int32), 'nca_c': nca_c,
            'res_feat': rng.integers(0, 21, (n, 1)).astype(np.float32)}


def test_every_host_path_sets_max_segment_nodes(tmp_path, cuda_device):
    dev = cuda_device
    sizes = [(37, 120), (201, 15), (64, 64)]
    rng = np.random.default_rng(5)
    # GraphPlan from a batched graph
    plan = GraphPlan.from_graph(gio.make_batch([synthetic.synthetic_pair(rng, a, b, 10) for a, b in sizes], dev), dev, 10)
    assert plan.struct.max_segment_nodes == 201
    # the on-device residue graph build
    g = build_graphs(ResidueBatch([(_residue_protein(rng, a), _residue_protein(rng, b)) for a, b in sizes]), dev)
    assert g._eqd_plan.struct.max_segment_nodes == 201
    # the device-resident pair dataset, for a minibatch without the largest protein
    pairs, labels = [], []
    for a, b in sizes:
        lig, rec = synthetic.synthetic_protein(rng, a, 10), synthetic.synthetic_protein(rng, b, 10)
        lig['new_x'] = lig['x'].copy()
        tg = make_targets((lig, rec), rng)
        pairs.append((lig, rec))
        labels.append({'pocket_coors': tg['pocket_lig'], 'bound_lig': tg['bound_lig'], 'bound_rec': tg['bound_rec']})
    save_pairs(str(tmp_path / 'p.eqd'), pairs, labels)
    ds = DevicePairDataset(PairArchive(str(tmp_path / 'p.eqd')), dev)
    gd, _ = ds.batch([0, 2])
    assert gd._eqd_plan.struct.max_segment_nodes == 120
