"""CUDA-graph replay of the whole forward for a fixed-shape batch.

One forward of the engine is ~43 kernel launches, 8 memsets and one small D2H copy issued by ``eqd_iegmn_forward``.
Captured once into a CUDA graph, a step costs the host ONE ``cudaGraphLaunch`` -- the GPU no longer waits for a Python
process that shares its cores with seven other ranks (round-1 SCALE run: 7 ms of GPU idle per 4 ms of kernels).

``GraphedForward(model, device_batch)`` owns the captured graph together with everything it points at: the batch's
device tensors, its ``GraphPlan`` (topology arrays), the workspace, the outputs and one pinned status buffer.  A new
batch of the SAME shape signature is served by overwriting the batch tensors in place and calling ``refresh()``
(``GraphPlan.refresh`` re-derives the CSR in place); ``launch()`` replays the graph and returns a handle whose
``result()`` waits for the replay, inspects the per-pair status words and -- only if the SVD guard, a NaN, an unsorted
edge list or a bad residue index was flagged -- falls back to the eager path, which replays the reference's host-side
control flow (rigid_docking_model.py:570-584).  The captured work is exactly the eager path's: same kernels, same
order, same buffers.

The graph is tied to the parameter version and the precision (``IEGMN.precision``) it was captured with (kernel
parameter banks hold small per-layer vectors and the product count selects the kernels): ``launch()`` re-captures when
either changed.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import _native as nat


def refuse_dropout_capture(iegmn):
    """A captured graph replays the kernel parameters of its capture, dropout seed included: every replay would apply the
    same masks.  Capture therefore refuses a model in training mode with dropout > 0 (launch() re-captures, and so
    refuses, when the model is switched to training mode after capture)."""
    if iegmn.training and iegmn.iegmn_layers[0].dropout_p > 0:
        raise NotImplementedError('CUDA-graph capture of a training-mode forward with dropout > 0 would replay one '
                                  'set of dropout masks: call model.eval(), or run the model eagerly')


class GraphedForward:
    def __init__(self, model, device_batch, before_forward=lambda: None):
        """``before_forward()`` is run (and recorded) in front of every forward of a capture: work on the capture stream
        that produces the batch's tensors in place (``graph_build.ResidueGraphedForward``: the graph build)."""
        self.model, self.batch, self.before_forward = model, device_batch, before_forward
        self.iegmn = model.iegmn_original
        self.device = self.iegmn.residue_emb_layer.weight.device
        if self.device.type != 'cuda':
            raise nat.NativeLibraryError('GraphedForward needs a CUDA device (no CPU fallback)')
        self.stream = torch.cuda.Stream(self.device)
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.raw: Optional[Dict] = None
        self.key = None
        self._capture()

    def _param_key(self):
        return tuple((p.data_ptr(), p._version) for p in self.model.parameters()) + (self.iegmn.precision,
                                                                                     self.iegmn.training)

    def _capture(self):
        refuse_dropout_capture(self.iegmn)
        with torch.cuda.device(self.device):
            cur = torch.cuda.current_stream(self.device)
            self.stream.wait_stream(cur)
            with torch.cuda.stream(self.stream):
                # eager warm-up on the capture stream: builds / caches the plan, the packed weights and every
                # one-time attribute, and proves the batch is servable before anything is recorded
                for _ in range(2):
                    self.before_forward()
                    self.iegmn.resolve(self.iegmn.run_engine(self.batch, check_status=False))
            self.stream.synchronize()
            self.plan = self.batch._eqd_plan
            self.key = self._param_key()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, stream=self.stream):
                self.before_forward()
                self.raw = self.iegmn.run_engine(self.batch, check_status=False, record_event=False)
            cur.wait_stream(self.stream)

    def refresh(self) -> bool:
        """Call after overwriting the batch's device tensors in place with a new same-shaped batch (on the current
        stream).  False = the shapes changed: build a new GraphedForward."""
        return self.plan.refresh(self.batch)

    def launch(self) -> 'GraphedPending':
        if self._param_key() != self.key:
            self._capture()
        with torch.cuda.device(self.device):
            self.graph.replay()
            ev = torch.cuda.Event()
            ev.record()
        return GraphedPending(self, ev)


class GraphedPending:
    def __init__(self, owner: GraphedForward, event):
        self.owner, self.event = owner, event

    def raw_result(self) -> Dict:
        """Waits for the replay and returns the engine's raw output dict (batched tensors: ``ligand_coors`` (sum N_l, 3),
        ``rotation`` (B, 3, 3), ``translation`` (B, 1, 3), ``keypts`` (2B, 50, 3) ...).  They are the graph's static
        buffers: valid until this GraphedForward is launched again."""
        o = self.owner
        self.event.synchronize()
        st = o.raw['status_host']
        if bool(st.any()):      # rare: some flag is set -> the eager path owns the reference's host-side control flow
            return o.iegmn.run_engine(o.batch, check_status=True)
        return o.raw

    def result(self):
        """The reference's 5-tuple (rigid_docking_model.py:690-692)."""
        raw = self.raw_result()
        iegmn = self.owner.iegmn
        return self.owner.model._assemble(iegmn.package(raw, self.owner.batch))
