"""Pipelined host->device->host inference over the reference-facing module: the public "serve a stream of batches"
call.  While the engine works on batch k (compute stream), batch k+1 is copied from pinned host memory on a second
stream and batch k-1's status words / results are read back -- so end-to-end throughput is max(PCIe, compute)
instead of their sum.  Every batch still goes through ``Rigid_Body_Docking_Net.forward_async`` (same kernels, same
status handling as ``model(graph, epoch)``).

Device input buffers and pinned result buffers live in three reusable slots (keyed by the batch's tensor shapes), so a
steady stream of same-shaped batches performs no allocation at all; the copy stream waits for a slot's previous
consumer before overwriting it.  With ``use_cuda_graph=True`` (default) every slot also owns a captured CUDA graph of the
forward (``graphed.GraphedForward``): a same-shaped batch is served by refreshing the slot's plan in place and ONE graph
launch, so the host-side cost of a step is a dozen copies and a launch instead of ~60 calls."""
from __future__ import annotations

from typing import Dict, Iterable, Iterator, Optional, Tuple

import torch

from .hetero_graph import CANONICAL_ETYPES, PairGraphBatch


def _tensors(g: PairGraphBatch):
    for et in CANONICAL_ETYPES:
        s, d = g._edges[et]
        yield ('e', et, 0), s
        yield ('e', et, 1), d
    for nt in g.ntypes:
        for k, v in g._ndata[nt].items():
            yield ('n', nt, k), v
    for et in CANONICAL_ETYPES:
        for k, v in g._edata[et].items():
            yield ('d', et, k), v


class _Slot:
    """One device-resident copy of a host batch plus the events that guard its reuse."""

    def __init__(self):
        self.signature = None
        self.graph: Optional[PairGraphBatch] = None
        self.consumed = None      # recorded on the compute stream after the forward that read this slot
        self.results: Dict[str, torch.Tensor] = {}
        self.graphed = None       # GraphedForward over this slot's device tensors (same signature only)
        self.fresh = True         # the device tensors were (re)allocated by the last fill

    def fill(self, hb: PairGraphBatch, device, copy_stream) -> Tuple[PairGraphBatch, torch.cuda.Event]:
        sig = tuple((key, tuple(t.shape), t.dtype) for key, t in _tensors(hb)) + tuple(
            tuple(v.tolist()) for v in hb._batch_num_nodes.values())
        with torch.cuda.stream(copy_stream):
            if self.consumed is not None:
                copy_stream.wait_event(self.consumed)           # the previous batch in this slot has been read
            self.fresh = sig != self.signature
            if self.fresh:                                      # new shape: (re)allocate this slot's device tensors
                self.graph = hb.to(device, non_blocking=True)
                self.signature = sig                            # (the slot owns these tensors for good: no record_stream)
                self.graphed = None
            else:
                dst = dict(_tensors(self.graph))
                for key, t in _tensors(hb):
                    dst[key].copy_(t, non_blocking=True)
                self.graph._batch_num_nodes = hb._batch_num_nodes
                self.graph._batch_num_edges = hb._batch_num_edges
            if hasattr(self.graph, '_eqd_plan') and self.graphed is None:
                self.graph._eqd_plan = None                     # a new batch has a new topology: rebuild the plan
                                                                # (a graphed slot refreshes its plan in place instead)
            ev = torch.cuda.Event()
            ev.record(copy_stream)
        return self.graph, ev


class PipelinedInference:
    def __init__(self, model, device, use_cuda_graph: bool = True):
        self.model, self.device = model, torch.device(device)
        self.use_cuda_graph = use_cuda_graph
        self.copy_stream = torch.cuda.Stream(self.device)
        self.slots = [_Slot(), _Slot(), _Slot()]

    def run(self, host_batches: Iterable[PairGraphBatch]) -> Iterator[Dict[str, torch.Tensor]]:
        """``host_batches``: pinned ``PairGraphBatch`` objects.  Yields, in order, for every batch a dict of pinned
        host tensors ``ligand_coors`` (sum N_l, 3), ``rotation`` (B, 3, 3), ``translation`` (B, 1, 3) and the CUDA
        event ``_event`` that marks their arrival (the buffers are reused three batches later)."""
        compute = torch.cuda.current_stream(self.device)
        it = iter(host_batches)
        k = 0

        def stage(hb, idx):
            slot = self.slots[idx % len(self.slots)]
            g, ev = slot.fill(hb, self.device, self.copy_stream)
            return slot, g, ev

        nxt = next(it, None)
        staged = stage(nxt, k) if nxt is not None else None
        in_flight = None
        while staged is not None:
            slot, g, ev = staged
            compute.wait_event(ev)
            pending = self._launch(slot, g)
            slot.consumed = torch.cuda.Event()
            slot.consumed.record(compute)
            k += 1
            nxt = next(it, None)
            staged = stage(nxt, k) if nxt is not None else None   # H2D of the next batch overlaps this batch's kernels
            if in_flight is not None:
                yield self._finish(*in_flight)
            in_flight = (pending, slot)
        if in_flight is not None:
            yield self._finish(*in_flight)

    def _launch(self, slot: _Slot, g):
        if not self.use_cuda_graph:
            return self.model.forward_async(g, 0)
        from .graphed import GraphedForward
        if slot.graphed is None or not slot.graphed.refresh():
            slot.graphed = GraphedForward(self.model, g)     # first batch of this shape in this slot: capture
        return slot.graphed.launch()

    def _finish(self, pending, slot: _Slot):
        raw = pending.raw_result()     # batched device tensors, no per-pair split / re-concatenation
        res = {'ligand_coors': raw['ligand_coors'], 'rotation': raw['rotation'], 'translation': raw['translation']}
        out = {}
        for key, t in res.items():
            hbuf = slot.results.get(key)
            if hbuf is None or hbuf.shape != t.shape:
                hbuf = slot.results[key] = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
            hbuf.copy_(t, non_blocking=True)
            out[key] = hbuf
        done = torch.cuda.Event()
        done.record(torch.cuda.current_stream(self.device))    # the copies' stream, also when another device is current
        out['_event'] = done
        return out
