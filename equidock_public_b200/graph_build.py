"""Residue k-NN graph construction on the GPU (csrc/graph_build.cu): the device-side replacement of the reference's
``protein_to_graph_unbound_bound`` (src/utils/protein_utils.py:212-397), producing the model's input contract -- CSR edges
grouped by destination, the 27 edge features, ``x``, ``mu_r_norm`` -- for a whole batch of pairs from compact all-atom
inputs.  The batch then needs ~50 KB per pair over PCIe instead of ~480 KB of edge features, and the 3.2 s/pair of Python
in front of the hot path disappears.

``ResidueBatch`` is the host-side container (pinned, ragged): proteins in engine order (ligand proteins of all pairs, then
receptor proteins).  ``build_graphs(residue_batch, device)`` returns a ``PairGraphBatch`` whose ``GraphPlan`` is already
attached, so ``model(graph, epoch)`` / ``model.graphed(graph)`` run on it directly.
"""
from __future__ import annotations

import ctypes as C
from types import SimpleNamespace
from typing import Dict, Sequence, Tuple

import numpy as np
import torch

from . import _native as nat
from .engine import GraphPlan, node_tiles_for
from .graphed import GraphedForward
from .hetero_graph import CROSS_LR, CROSS_RL, LIGAND, LL, RECEPTOR, RR, PairGraphBatch

MAXK = 16


class ResidueBatch:
    """Compact all-atom inputs of B protein pairs (the format of oracle/graph_oracle.py): per protein ``atoms`` (A,3) f32,
    ``atom_ptr`` (N+1,) i32, ``nca_c`` (N,3,3) f32, ``res_feat`` (N,1) f32 and optionally ``bound_ca`` (N,3) f32."""

    def __init__(self, pairs: Sequence[Tuple[Dict, Dict]], pin: bool = False):
        prots = [p[0] for p in pairs] + [p[1] for p in pairs]
        self.n_pairs = len(pairs)
        n = [int(np.asarray(p['nca_c']).shape[0]) for p in prots]
        self.n_lig, self.n_rec = n[:self.n_pairs], n[self.n_pairs:]
        self.max_protein_nodes = max(n)
        seg = np.zeros(len(prots) + 1, np.int32)
        seg[1:] = np.cumsum(n)
        a_ptr, a_off = [np.zeros(1, np.int32)], 0
        for p in prots:
            ap = np.asarray(p['atom_ptr'], np.int64)
            a_ptr.append((ap[1:] + a_off).astype(np.int32))
            a_off += int(ap[-1])
        f = lambda k, shape: torch.from_numpy(np.ascontiguousarray(np.concatenate([np.asarray(p[k], np.float32).reshape(shape) for p in prots])))
        self.t = {'seg_ptr': torch.from_numpy(seg), 'atom_ptr': torch.from_numpy(np.concatenate(a_ptr)),
                  'atoms': f('atoms', (-1, 3)), 'nca_c': f('nca_c', (-1, 9)), 'res_feat': f('res_feat', (-1, 1)),
                  'bound_ca': torch.from_numpy(np.ascontiguousarray(np.concatenate(
                      [np.asarray(p.get('bound_ca', np.asarray(p['nca_c'])[:, 1]), np.float32).reshape(-1, 3) for p in prots])))}
        if pin:
            self.t = {k: v.pin_memory() for k, v in self.t.items()}
        self.N = int(seg[-1])

    def nbytes(self) -> int:
        return int(sum(v.numel() * v.element_size() for v in self.t.values()))


def _edge_counts(ne_l, ne_r, B):
    z = torch.zeros(B, dtype=torch.int64)
    return {LL: torch.tensor(ne_l, dtype=torch.int64), RR: torch.tensor(ne_r, dtype=torch.int64), CROSS_RL: z, CROSS_LR: z.clone()}


class GraphBuffers:
    """Static device buffers of one graph build (inputs and outputs), so that a same-shaped batch can be rebuilt in place
    -- every pointer the forward's GraphPlan holds stays valid, which is what a CUDA-graph capture of
    [graph build + forward] needs (``ResidueGraphedForward``)."""

    def __init__(self, rb: ResidueBatch, device, max_neighbor: int = 10):
        dev = torch.device(device)
        N = rb.N
        i32, f32 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.float32, device=dev)
        self.inputs = {k: torch.empty_like(v, device=dev) for k, v in rb.t.items()}
        self.signature = tuple((k, tuple(v.shape)) for k, v in rb.t.items()) + (tuple(rb.n_lig), tuple(rb.n_rec))
        self.ws = torch.empty(int(nat.load().eqd_graph_build_workspace_bytes(N)), dtype=torch.uint8, device=dev)
        self.deg, self.x, self.mu = torch.empty(N, **i32), torch.empty(N, 3, **f32), torch.empty(N, 5, **f32)
        self.row_ptr = torch.zeros(N + 1, **i32)
        e_cap = N * int(max_neighbor)
        self.col_src, self.edge_dst = torch.zeros(e_cap, **i32), torch.zeros(e_cap, **i32)
        self.he = torch.zeros(e_cap + 1, 27, **f32)

    def matches(self, rb: ResidueBatch) -> bool:
        return self.signature == tuple((k, tuple(v.shape)) for k, v in rb.t.items()) + (tuple(rb.n_lig), tuple(rb.n_rec))

    def upload(self, rb: ResidueBatch, stream=None):
        with torch.cuda.stream(stream) if stream is not None else _null():
            for k, v in rb.t.items():
                self.inputs[k].copy_(v, non_blocking=True)


class _null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def build_graphs(rb: ResidueBatch, device, cutoff: float = 30.0, max_neighbor: int = 10, sync_sizes: bool = True,
                 dev_inputs: Dict[str, torch.Tensor] | None = None, buffers: 'GraphBuffers | None' = None) -> PairGraphBatch:
    """H2D of the compact inputs (unless ``dev_inputs`` already holds them) + the three graph kernels + one prefix sum.
    ``sync_sizes=True`` reads the edge counts back (one small D2H) so that the result is a fully formed PairGraphBatch;
    ``False`` keeps everything asynchronous: edge buffers stay sized for N x max_neighbor edges and the attached GraphPlan
    serves the forward pass (inference) without the host ever learning E."""
    dev = torch.device(device)
    N, B = rb.N, rb.n_pairs
    N_l = sum(rb.n_lig)
    e_cap = N * int(max_neighbor)
    if buffers is None:
        i32, f32 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.float32, device=dev)
        buffers = SimpleNamespace(
            inputs=dev_inputs or {k: v.to(dev, non_blocking=True) for k, v in rb.t.items()},
            ws=torch.empty(int(nat.load().eqd_graph_build_workspace_bytes(N)), dtype=torch.uint8, device=dev),
            deg=torch.empty(N, **i32), x=torch.empty(N, 3, **f32), mu=torch.empty(N, 5, **f32),
            row_ptr=torch.zeros(N + 1, **i32), col_src=torch.empty(e_cap, **i32), edge_dst=torch.empty(e_cap, **i32),
            he=torch.empty(e_cap + 1, 27, **f32))                  # +1 row: readable past the end for the TMA over-read
    rebuild_in_place(rb, buffers, cutoff, max_neighbor)     # (the inputs of a GraphBuffers were uploaded by the caller)
    d, x, mu = buffers.inputs, buffers.x, buffers.mu
    row_ptr, col_src, edge_dst, he = buffers.row_ptr, buffers.col_src, buffers.edge_dst, buffers.he
    with torch.cuda.device(dev):
        if sync_sizes:       # ONE small D2H: the edge offsets at the 2B + 1 protein boundaries
            bounds = row_ptr[d['seg_ptr'].long()].cpu().tolist()
            E_l, E = int(bounds[B]), int(bounds[2 * B])
            ne_l = [bounds[i + 1] - bounds[i] for i in range(B)]
            ne_r = [bounds[B + i + 1] - bounds[B + i] for i in range(B)]
        else:
            E_l = E = e_cap
            ne_l = ne_r = None
    g = PairGraphBatch({LIGAND: N_l, RECEPTOR: N - N_l},
                       {LL: (col_src[:E_l], edge_dst[:E_l]), RR: (col_src[E_l:E] - N_l, edge_dst[E_l:E] - N_l)} if sync_sizes else {},
                       {LIGAND: torch.tensor(rb.n_lig, dtype=torch.int64), RECEPTOR: torch.tensor(rb.n_rec, dtype=torch.int64)},
                       _edge_counts(ne_l, ne_r, B) if sync_sizes else None)
    g._ndata[LIGAND] = {'res_feat': d['res_feat'][:N_l], 'x': x[:N_l], 'new_x': x[:N_l], 'mu_r_norm': mu[:N_l]}
    g._ndata[RECEPTOR] = {'res_feat': d['res_feat'][N_l:], 'x': x[N_l:], 'mu_r_norm': mu[N_l:]}
    if sync_sizes:
        g._edata[LL]['he'], g._edata[RR]['he'] = he[:E_l], he[E_l:E]
    seg, seg_ptr, node_tiles = node_tiles_for(rb.n_lig, rb.n_rec, dev)
    g._eqd_plan = GraphPlan.from_device_arrays(rb.n_lig, rb.n_rec, E_l, E, col_src, edge_dst, row_ptr, he, he, seg_ptr,
                                               node_tiles, seg, dev, int(max_neighbor), keep=(buffers.ws, buffers.deg, d))
    return g


def rebuild_in_place(rb: ResidueBatch, buffers: GraphBuffers, cutoff: float = 30.0, max_neighbor: int = 10):
    """The three graph kernels + one prefix sum (an index op), from ``buffers.inputs`` into the output tensors of
    ``buffers`` (nothing allocated: capturable)."""
    lib = nat.load()
    d = buffers.inputs
    dev = buffers.x.device
    N, B = rb.N, rb.n_pairs
    with torch.cuda.device(dev):
        st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        nat.check(lib.eqd_graph_build_knn(2 * B, N, rb.max_protein_nodes, nat.ptr(d['seg_ptr']), nat.ptr(d['atom_ptr']),
                                          nat.ptr(d['atoms']), nat.ptr(d['nca_c']), nat.ptr(d['bound_ca']), float(cutoff),
                                          int(max_neighbor), nat.ptr(buffers.ws), int(buffers.ws.numel()), nat.ptr(buffers.deg),
                                          nat.ptr(buffers.x), nat.ptr(buffers.mu), st), 'eqd_graph_build_knn')
        torch.cumsum(buffers.deg, 0, dtype=torch.int32, out=buffers.row_ptr[1:])
        nat.check(lib.eqd_graph_build_edges(N, nat.ptr(buffers.row_ptr), nat.ptr(buffers.deg), nat.ptr(buffers.ws),
                                            nat.ptr(buffers.col_src), nat.ptr(buffers.edge_dst), nat.ptr(buffers.he), st),
                  'eqd_graph_build_edges')


class ResidueGraphedForward:
    """[graph construction + whole forward] of a fixed-shape residue batch as ONE CUDA graph: per batch the host uploads
    ~50 KB per pair of compact all-atom inputs into the static input buffers and launches one graph; the model's input
    graph (k-NN edges, 27 edge features, surface features) never exists on the host."""

    def __init__(self, model, rb: ResidueBatch, device, cutoff: float = 30.0, max_neighbor: int = 10):
        self.model, self.device = model, torch.device(device)
        self.cutoff, self.max_neighbor = cutoff, max_neighbor
        self.buffers = GraphBuffers(rb, device, max_neighbor)
        self.rb = rb
        self.buffers.upload(rb)
        self.graph = build_graphs(rb, device, cutoff, max_neighbor, sync_sizes=False, buffers=self.buffers)
        self.gf = GraphedForward(model, self.graph, before_forward=lambda: rebuild_in_place(
            self.rb, self.buffers, self.cutoff, self.max_neighbor))

    def upload(self, rb: ResidueBatch, stream=None):
        if not self.buffers.matches(rb):
            raise ValueError('ResidueGraphedForward: batch shape differs from the captured one')
        self.buffers.upload(rb, stream)

    def launch(self):
        return self.gf.launch()
