"""Training side of the H100 engine: forward with a layer stash, the hand-written backward (csrc/bwd_*.cu, head.cu,
losses.cu) driven over the C ABI, a ``torch.autograd.Function`` so that the reference's own training loop
(``loss.backward()``, src/train.py:154) works on the drop-in module unchanged, and a fused data-parallel trainer
(device losses, flat-gradient NCCL all-reduce overlapped with the tail of backward, clip + Adam in one kernel;
src/train.py:98-165, 302).

PyTorch is plumbing here too: device memory, streams, ``torch.distributed``; a few index ops build the by-source edge
permutation once per batch topology.  No gradient arithmetic is done by torch beyond adding the upstream gradients of
the last layer's outputs (``x_iegmn_out`` / ``hv_iegmn_out``) to the head's.  There is no CPU fallback.

Gradient layout: ONE flat fp32 buffer holding every unique parameter in the order [head, layer L-1, ..., layer 0,
embedding] (the order the backward finishes them in, so that all-reduce buckets are contiguous and can start while
earlier layers are still being differentiated); ``param.grad`` tensors are views of it.
"""
from __future__ import annotations

import ctypes as C
import functools
from collections import namedtuple
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _native as nat
from .engine import (GraphPlan, IEGMNEngine, PackedLayer, _upload_blob, _host_f32, plan_for, retry_sorted, run_layer,
                     with_dropout)
from .hetero_graph import LIGAND, RECEPTOR

_f32 = torch.float32


def _padded(numel: int) -> int:
    """Floats one parameter takes in a flat buffer: every parameter starts on a 64-float (256-byte) boundary, because
    the kernels read weights 16 bytes at a time straight from the flat buffer (the index maps are built against it)."""
    return (numel + 63) & ~63


class ParamLayout:
    """Flat layout of a model's unique parameters in backward-completion order.  ``model`` is a Rigid_Body_Docking_Net or
    its IEGMN module (the same parameters; names keep the ``iegmn_original.`` prefix either way)."""

    def __init__(self, model):
        iegmn = getattr(model, 'iegmn_original', model)
        seen, self.entries = set(), []          # (qualified name, param)
        self.buckets: List[tuple] = []          # (label, lo, hi) contiguous slices, in completion order
        self.module_bucket: Dict[int, str] = {}  # id(layer module) -> its bucket label
        self.total = 0
        self._offs: List[int] = []

        def add(prefix, module, label):
            lo = self.total
            for n, p in module.named_parameters():
                if id(p) in seen:
                    continue
                seen.add(id(p))
                self.entries.append((f'{prefix}{n}', p))
                self._offs.append(self.total)
                self.total += _padded(p.numel())
            if self.total > lo:
                self.buckets.append((label, lo, self.total))
                self.module_bucket[id(module)] = label

        add('iegmn_original.att_mlp_key_ROT.', iegmn.att_mlp_key_ROT, 'head')
        add('iegmn_original.att_mlp_query_ROT.', iegmn.att_mlp_query_ROT, 'head')
        add('iegmn_original.mlp_h_mean_ROT.', iegmn.mlp_h_mean_ROT, 'head')
        # merge the three head modules into one bucket
        self.buckets = [('head', 0, self.total)]
        for li in reversed(range(len(iegmn.iegmn_layers))):
            add(f'iegmn_original.iegmn_layers.{li}.', iegmn.iegmn_layers[li], f'layer{li}')
        add('iegmn_original.residue_emb_layer.', iegmn.residue_emb_layer, 'emb')
        self.offset: Dict[int, int] = {}
        self.name_offset: Dict[str, int] = {}
        for (name, p), o in zip(self.entries, self._offs):
            self.offset[id(p)] = o
            self.name_offset[name] = o
        self.params = [p for _, p in self.entries]
        self.n_param_elements = sum(p.numel() for p in self.params)

    def views(self, flat: torch.Tensor) -> List[torch.Tensor]:
        return [flat[self.offset[id(p)]:self.offset[id(p)] + p.numel()].view(p.shape) for p in self.params]


def _i32(a, device):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(device)


# A weight block: partial [k][c0 + n] -> param [n][k0 + k] (an nn.Linear weight [out][width]), k < rows, n < cols.
Block = namedtuple('Block', 'param width k0 c0 rows cols')
# One weight-gradient reduction, launched right after the kernel of its ``stage`` ('node': eqd_bwd_node_mlp, 'edge':
# eqd_bwd_edge, 'proj': eqd_bwd_project, 'head': eqd_bwd_head_dropout): ws.partial / colsum / vec are reused between
# stages.  With X, eqd_tn_gemm computes alpha * X^T D over ``rows`` ('N' nodes or 'E' edges) into the row-chunk
# partials ws.partial [K][ncols] and, when there are ``sums``, the column sums of D into ws.colsum; alpha is the layer's
# skip_weight_h if ``skip``, else 1.  X and D name a stage operand or a BackwardWorkspace tensor.  Without X, the stage
# kernel left per-CTA sums in ws.vec, ``ncols`` floats per CTA.  eqd_grad_reduce adds the partials' ``blocks`` and the
# ``sums`` ((parameter, first column), each covering the whole parameter) into the flat gradient.
Reduction = namedtuple('Reduction', 'name stage X ldx K D ldd ncols rows blocks sums skip', defaults=((), (), False))


@functools.lru_cache(maxsize=None)
def layer_reductions(dh: int, dhp: int, coors_ln: bool = False, final_ln: bool = False) -> tuple:
    """The weight-gradient reductions of one IEGMN_Layer of width dh whose node rows are padded to dhp, in launch order
    (see Reduction); ``coors_ln`` / ``final_ln``: the layer has the coordinate LayerNorm coors_mlp.3
    (layer_norm_coors='LN') / the final feature LayerNorm final_h_layernorm_layer (final_h_layer_norm='LN').  h_in and
    mu have row stride dhp, h0 has H0_PAD."""
    pw = 128 + 3 * dhp                                # projection width: [Psrc | Pdst | Q | K | V]
    edgevec = (('edge_mlp.3.weight', 0), ('edge_mlp.3.bias', 64), ('coors_mlp.4.weight', 128), ('coors_mlp.4.bias', 192))
    if coors_ln:
        edgevec += (('coors_mlp.3.weight', 256), ('coors_mlp.3.bias', 320))
    nodevec = (('node_mlp.3.weight', 0), ('node_mlp.3.bias', 72))
    if final_ln:
        nodevec += (('final_h_layernorm_layer.weight', 144), ('final_h_layernorm_layer.bias', 208))
    ein, w1n = 2 * dh + 42, 2 * dh + 64 + nat.H0      # input widths of edge_mlp.0 and node_mlp.0
    R, B, w5 = Reduction, Block, 'node_mlp.0.weight'
    return (
        # R(name, stage, X, ldx, K, D, ldd, ncols, rows, blocks, sums): B(param, width, k0, c0, rows, cols), (param, c0)
        R('nodevec', 'node', None, 0, 0, None, 0, 272 if final_ln else 144, None, (), nodevec),
        R('node2', 'node', 'n5', dhp, dhp, 'dh_out', 64, 64, 'N', (B('node_mlp.4.weight', dh, 0, 0, dh, 64),),
          (('node_mlp.4.bias', 0),), skip=dh == nat.HID),
        R('node_h', 'node', 'h_in', dhp, dhp, 'du', dhp, dhp, 'N', (B(w5, w1n, 0, 0, dh, dh),),
          (('node_mlp.0.bias', 0),)),
        R('node_aggr', 'node', 'aggr', 64, 64, 'du', dhp, dhp, 'N', (B(w5, w1n, dh, 0, 64, dh),)),
        R('node_mu', 'node', 'mu', dhp, dhp, 'du', dhp, dhp, 'N', (B(w5, w1n, dh + 64, 0, dh, dh),)),
        R('node_h0', 'node', 'h0', nat.H0_PAD, nat.H0_PAD, 'du', dhp, dhp, 'N',
          (B(w5, w1n, 2 * dh + 64, 0, nat.H0, dh),)),
        R('edgevec', 'edge', None, 0, 0, None, 0, 384 if coors_ln else 256, None, (), edgevec),
        R('edge1', 'edge', 'ein', 44, 44, 'dz1', 64, 64, 'E', (B('edge_mlp.0.weight', ein, 2 * dh, 0, 42, 64),)),
        R('edge2', 'edge', 'n1', 64, 64, 'dmsg', 64, 64, 'E', (B('edge_mlp.4.weight', 64, 0, 0, 64, 64),),
          (('edge_mlp.4.bias', 0),)),
        R('edge3', 'edge', 'msg', 64, 64, 'dz3', 64, 64, 'E', (B('coors_mlp.0.weight', 64, 0, 0, 64, 64),),
          (('coors_mlp.0.bias', 0),)),
        R('proj', 'proj', 'h_in', dhp, dhp, 'dP', pw, pw, 'N',
          (B('edge_mlp.0.weight', ein, 0, 0, dh, 64), B('edge_mlp.0.weight', ein, dh, 64, dh, 64),
           B('att_mlp_Q.0.weight', dh, 0, 128, dh, dh), B('att_mlp_K.0.weight', dh, 0, 128 + dhp, dh, dh),
           B('att_mlp_V.0.weight', dh, 0, 128 + 2 * dhp, dh, dh)),
          (('edge_mlp.0.bias', 64),)),
    )


# Floats per CTA of the widest per-CTA partial sums a stage kernel leaves in BackwardWorkspace.vec
VEC_FLOATS = max(r.ncols for r in layer_reductions(nat.H0, nat.H0_PAD, True, True) if r.X is None)

HEAD_REDUCTION = Reduction('head', 'head', 'h', 64, 64, 'dpre', 64, 64, 'N',
                           (Block('iegmn_original.mlp_h_mean_ROT.0.weight', 64, 0, 0, 64, 64),),
                           (('iegmn_original.mlp_h_mean_ROT.0.bias', 0),))


def _block_map(off: int, b: Block, ncols: int):
    k, n = np.meshgrid(np.arange(b.rows), np.arange(b.cols), indexing='ij')     # k = input feature, n = output unit
    return (k * ncols + b.c0 + n).reshape(-1), (off + n * b.width + b.k0 + k).reshape(-1)


def reduction_maps(table, named_params, layout, device) -> Dict[str, tuple]:
    """{reduction name: (blocks map, sums map)} of the reductions in ``table``: each map is the (source index,
    destination index) int32 pair eqd_grad_reduce reads (partial, colsum or vec -> flat gradient at ``layout.offset``),
    or None.  ``named_params`` yields the (name, parameter) pairs the table's names refer to."""
    params = dict(named_params)
    off = lambda name: layout.offset[id(params[name])]
    span = lambda name: np.arange(params[name].numel())
    join = lambda pieces: tuple(_i32(np.concatenate(a), device) for a in zip(*pieces)) if pieces else None
    return {r.name: (join([_block_map(off(b.param), b, r.ncols) for b in r.blocks]),
                     join([(c0 + span(p), off(p) + span(p)) for p, c0 in r.sums])) for r in table}


class LayerTrainPack:
    """Backward-side tensors of one IEGMN_Layer module: the nn.Linear-layout weight panels the data-gradient GEMMs
    read, and the (source index, destination index) maps of every weight-gradient reduction (packed k-major partial ->
    flat state_dict-layout gradient).  The maps depend on the layout only: ``maps`` passes those of an earlier pack."""

    def __init__(self, layer_module, packed: PackedLayer, layout: ParamLayout, device, maps=None):
        dh, dhp = packed.dh, packed.dhp
        pw = 128 + 3 * dhp
        win = 2 * dhp + 64 + nat.H0_PAD
        sd = {k: _host_f32(v) for k, v in layer_module.state_dict(keep_vars=True).items()}
        w5, w6 = sd['node_mlp.0.weight'], sd['node_mlp.4.weight']
        w1lin = torch.zeros(dhp, win)
        w1lin[:dh, 0:dh] = w5[:, 0:dh]
        w1lin[:dh, dhp:dhp + 64] = w5[:, dh:dh + 64]
        w1lin[:dh, dhp + 64:dhp + 64 + dh] = w5[:, dh + 64:2 * dh + 64]
        w1lin[:dh, 2 * dhp + 64:2 * dhp + 64 + nat.H0] = w5[:, 2 * dh + 64:]
        w2lin = torch.zeros(64, dhp)
        w2lin[:, :dh] = w6
        self.t = _upload_blob({'w_node1_lin': w1lin, 'w_node2_lin': w2lin,
                               'w_projT': packed.t['w_proj'].detach().cpu().t().contiguous(),
                               'w2lin': sd['edge_mlp.4.weight'].contiguous(),
                               'w3lin': sd['coors_mlp.0.weight'].contiguous()}, device)
        self.dh, self.dhp, self.pw = dh, dhp, pw
        self.reductions = layer_reductions(dh, dhp, packed.layer_norm_coors == 'LN', packed.final_h_layer_norm == 'LN')
        self.maps = maps or reduction_maps(self.reductions, layer_module.named_parameters(), layout, device)


def tn_gemm_shapes(N: int, E: int, dhps: Sequence[int] = (nat.H0_PAD, nat.HID)) -> List[tuple]:
    """Every (rows, K, ncols) that TrainEngine.backward passes to eqd_tn_gemm, for a batch of N nodes and E edges whose
    layers have the padded widths ``dhps`` (72 for the 69-wide layer 0, 64 for the others)."""
    table = [HEAD_REDUCTION] + [r for dhp in dhps for r in layer_reductions(nat.HID if dhp == nat.HID else nat.H0, dhp)]
    return sorted({(N if r.rows == 'N' else E, r.K, r.ncols) for r in table if r.X is not None})


def tn_workspace_floats(N: int, E: int, dhps: Sequence[int] = (nat.H0_PAD, nat.HID)) -> tuple:
    """(partial, colsum) floats that cover every eqd_tn_gemm call of one backward (see tn_gemm_shapes)."""
    lib = nat.load()
    partial = colsum = 1
    for rows, K, nc in tn_gemm_shapes(N, E, dhps):
        nch = C.c_int32(0)
        partial = max(partial, int(lib.eqd_tn_partial_floats(rows, K, nc, None, C.byref(nch))))
        colsum = max(colsum, nch.value * nc)
    return partial, colsum


class BackwardWorkspace:
    """Device buffers of one backward, sized for a plan (reused across steps with the same sizes)."""

    def __init__(self, plan: GraphPlan, device, n_heads: int = nat.HEADS):
        N, E, B = plan.N, plan.E, plan.n_pairs
        f = lambda *s: torch.empty(*s, dtype=_f32, device=device)
        d = lambda *s: torch.empty(*s, dtype=torch.float64, device=device)
        self.key = (N, E, B)
        self.proj, self.dP = f(N, 344), f(N, 344)
        self.dh = [f(N, 72), f(N, 72)]
        self.dx = [d(N, 3), d(N, 3)]
        self.daggr, self.dmu, self.dh0 = f(N, 64), f(N, 72), f(N, 72)
        self.n5, self.du, self.rowstat, self.dpre = f(N, 72), f(N, 72), f(N, 4), f(N, 64)
        self.ein = f(max(E, 1), 44)
        self.n1, self.msg, self.dz3, self.dmsg, self.dz1 = (f(max(E, 1), 64) for _ in range(5))
        self.dxrel = d(max(E, 1), 3)
        lib = nat.load()
        n_partial, n_colsum = tn_workspace_floats(N, E)
        self.partial, self.colsum = f(n_partial), f(n_colsum)
        self.vec = f(132 * VEC_FLOATS)   # per-CTA partial sums of bwd_node / bwd_edge (grid <= EQD_SMS)
        self.head_ws_bytes = int(lib.eqd_bwd_head_workspace_bytes_k(N, plan.n_node_tiles, B, n_heads))
        self.head_ws = torch.empty(self.head_ws_bytes, dtype=torch.uint8, device=device)
        # edges grouped by SOURCE node (ascending edge id inside a group): the transpose index of the CSR-by-destination
        order = torch.sort(plan.col_src.long(), stable=True)
        self.out_edge = order.indices.to(torch.int32).contiguous()
        self.out_ptr = torch.searchsorted(order.values.to(torch.int32).contiguous(),
                                          torch.arange(N + 1, dtype=torch.int32, device=device), out_int32=True).contiguous()


def _vp(t):
    """A device pointer given as a tensor or already as c_void_p (a slice of the forward stash)."""
    return t if t is None or isinstance(t, C.c_void_p) else nat.ptr(t)


def _weight_grads(lib, ws, table, maps, stage, operands, N, E, flat, st, nparts=0, skip_weight_h=1.0):
    """Launches the reductions of ``table`` that follow ``stage``, in table order (see Reduction).  ``operands`` holds
    the stage's named operands that are not BackwardWorkspace tensors; ``nparts`` is the number of per-CTA sums in
    ws.vec."""
    opd = lambda name: _vp(operands[name] if name in operands else getattr(ws, name))
    partial, colsum, vec, grad = nat.ptr(ws.partial), nat.ptr(ws.colsum), nat.ptr(ws.vec), nat.ptr(flat)
    for r in table:
        if r.stage != stage:
            continue
        nch = C.c_int32(nparts)          # partial sums per element: eqd_tn_gemm sets its row-chunk count
        if r.X is not None:
            nat.check(lib.eqd_tn_gemm(opd(r.X), r.ldx, r.K, opd(r.D), r.ldd, r.ncols, N if r.rows == 'N' else E,
                                      skip_weight_h if r.skip else 1.0, partial, colsum if r.sums else None,
                                      C.byref(nch), st), 'eqd_tn_gemm')
        for src, stride, mp in zip((partial, colsum if r.X else vec), (r.K * r.ncols, r.ncols), maps[r.name]):
            if mp is not None:
                nat.check(lib.eqd_grad_reduce(src, nch.value, stride, nat.ptr(mp[0]), nat.ptr(mp[1]),
                                              int(mp[0].numel()), grad, st), 'eqd_grad_reduce')


def layer_backward(lib, plan: GraphPlan, lp_obj: PackedLayer, tp: LayerTrainPack, ws: BackwardWorkspace, h_in, x_in, aggr,
                   mu, h0, dh_out, dx_out, dh_in, dx_in, flat, st, dhe=None, dx_orig=None, capture=None, li=None, desc=None):
    """Backward of ONE IEGMN_Layer, the fixed kernel sequence eqd_project (recompute) -> eqd_bwd_node_mlp ->
    eqd_bwd_attention -> eqd_bwd_edge -> (eqd_bwd_layer_inputs) -> eqd_bwd_edge_gather -> eqd_bwd_project, with the weight
    gradients of each stage through eqd_tn_gemm + eqd_grad_reduce (``tp.reductions``, see layer_reductions).

    The layer's stashed inputs (tensors or device pointers): h_in [N][dhp] f32 (row stride 72 for the 69-wide layer 0,
    else 64), x_in [N][3] f64, aggr [N][64] f32, mu [N][dhp] f32, h0 [N][72] f32.  Upstream gradients: dh_out [N][64] f32
    and dx_out [N][3] f64 of the layer's output features and coordinates (with the final LayerNorm on, eqd_bwd_node_mlp
    overwrites dh_out with the gradient w.r.t. the pre-norm row, which the node_mlp.4 reductions read).  Writes dh_in [N][dhp] and dx_in [N][3] f64
    (overwritten), adds the gradient w.r.t. h0 into ws.dh0 and the parameter gradients into `flat` (through the index maps
    of `tp`).  With dhe [E][27] f32 / dx_orig [N][3] f64 given, it also adds the gradients w.r.t. the edge features and the
    original coordinates there (eqd_bwd_layer_inputs); without them that kernel is not launched.  ``desc`` is the eqd_layer
    the forward ran with when it differs from ``lp_obj.struct`` (training-mode dropout: the backward replays its masks).
    Returns (dh_in, dx_in, ws.dh0, dhe, dx_orig)."""
    g = C.byref(plan.struct)
    N, E = plan.N, plan.E
    lp = C.byref(desc if desc is not None else lp_obj.struct)
    dh, dhp, pw = tp.dh, tp.dhp, tp.pw
    ld = nat.H0_PAD if dh == nat.H0 else nat.HID     # row stride of h_in and of mu
    h_in, x_in, aggr, mu, h0 = _vp(h_in), _vp(x_in), _vp(aggr), _vp(mu), _vp(h0)
    ops = {'h_in': h_in, 'aggr': aggr, 'mu': mu, 'h0': h0, 'dh_out': dh_out}
    nat.check(lib.eqd_project(g, lp, h_in, ld, nat.ptr(ws.proj), st), 'eqd_project')
    nparts = C.c_int32(0)
    nat.check(lib.eqd_bwd_node_mlp(g, lp, nat.ptr(tp.t['w_node1_lin']), nat.ptr(tp.t['w_node2_lin']), h_in, ld,
                                   aggr, mu, ld, h0, nat.ptr(dh_out), nat.ptr(dh_in), nat.ptr(ws.daggr),
                                   nat.ptr(ws.dmu), nat.ptr(ws.dh0), nat.ptr(ws.n5), nat.ptr(ws.du),
                                   nat.ptr(ws.vec), C.byref(nparts), st), 'eqd_bwd_node_mlp')
    _weight_grads(lib, ws, tp.reductions, tp.maps, 'node', ops, N, E, flat, st, nparts.value,
                  float(lp_obj.struct.dev.skip_weight_h))
    nat.check(lib.eqd_bwd_attention(g, lp, nat.ptr(ws.proj), mu, ld, nat.ptr(ws.dmu), nat.ptr(ws.dP),
                                    nat.ptr(ws.rowstat), st), 'eqd_bwd_attention')
    nat.check(lib.eqd_bwd_edge(g, lp, nat.ptr(tp.t['w2lin']), nat.ptr(tp.t['w3lin']), nat.ptr(ws.proj), x_in,
                               nat.ptr(ws.daggr), nat.ptr(dx_out), nat.ptr(ws.ein), nat.ptr(ws.n1),
                               nat.ptr(ws.msg), nat.ptr(ws.dz3), nat.ptr(ws.dmsg), nat.ptr(ws.dz1),
                               nat.ptr(ws.dxrel), nat.ptr(ws.vec), C.byref(nparts), st), 'eqd_bwd_edge')
    if dhe is not None:
        nat.check(lib.eqd_bwd_layer_inputs(g, lp, nat.ptr(ws.dz1), nat.ptr(dx_out), nat.ptr(dhe),
                                           nat.ptr(dx_orig), st), 'eqd_bwd_layer_inputs')
    _weight_grads(lib, ws, tp.reductions, tp.maps, 'edge', ops, N, E, flat, st, nparts.value)
    nat.check(lib.eqd_bwd_edge_gather(g, nat.ptr(ws.out_ptr), nat.ptr(ws.out_edge), nat.ptr(ws.dz1),
                                      nat.ptr(ws.dxrel), nat.ptr(dx_out), float(lp_obj.struct.dev.x_connection_init),
                                      nat.ptr(ws.dP), pw, nat.ptr(dx_in), st), 'eqd_bwd_edge_gather')
    if capture is not None:
        rows = lambda t, w, n=N: t.reshape(-1)[:n * w].clone().view(n, w)
        capture.append({'layer': li, 'dh_part': rows(dh_in, dhp), 'daggr': ws.daggr.clone(), 'dmu': rows(ws.dmu, dhp),
                        'dz1': ws.dz1[:E].clone(), 'dxrel': ws.dxrel[:E].clone(), 'dP': rows(ws.dP, pw),
                        'dx': dx_in.clone(), 'dh0': ws.dh0.clone()})
    nat.check(lib.eqd_bwd_project(g, lp, nat.ptr(tp.t['w_projT']), nat.ptr(ws.dP), nat.ptr(dh_in), st),
              'eqd_bwd_project')
    if capture is not None:
        capture[-1]['dh'] = dh_in.reshape(-1)[:N * dhp].clone().view(N, dhp)
    _weight_grads(lib, ws, tp.reductions, tp.maps, 'proj', ops, N, E, flat, st)
    return dh_in, dx_in, ws.dh0, dhe, dx_orig


class TrainEngine:
    """Forward-with-stash and backward of one model on one device (a Rigid_Body_Docking_Net, or an IEGMN module)."""

    def __init__(self, model):
        self.model = model
        self.iegmn = getattr(model, 'iegmn_original', model)
        self.device = self.iegmn.residue_emb_layer.weight.device
        if self.device.type != 'cuda':
            raise nat.NativeLibraryError('training runs on a CUDA device only (no CPU fallback)')
        self.lib = nat.load()
        self.layout = ParamLayout(model)
        self._packs: Dict[int, tuple] = {}
        self._maps: Dict[int, dict] = {}
        self._ws: Optional[BackwardWorkspace] = None
        self._head_maps = reduction_maps((HEAD_REDUCTION,), self.layout.entries, self.layout, self.device)
        self.rank = 0        # data-parallel rank: an input of the dropout masks (DataParallelTrainer sets it)

    # ---- packs ----------------------------------------------------------------------------------------------------
    def layer_pack(self, lay_module) -> LayerTrainPack:
        packed = lay_module.packed(self.device)
        hit = self._packs.get(id(lay_module))
        if hit is None or hit[0] is not packed:
            maps = self._maps.get(id(lay_module))
            tp = LayerTrainPack(lay_module, packed, self.layout, self.device, maps)
            self._maps[id(lay_module)] = tp.maps
            hit = (packed, tp)
            self._packs[id(lay_module)] = hit
        return hit[1]

    # ---- forward with stash -----------------------------------------------------------------------------------------
    def forward(self, graph, log=None):
        iegmn = self.iegmn
        dropout = iegmn.iegmn_layers[0].dropout_now(self.rank) if iegmn.training else None
        return retry_sorted(graph, plan_for(graph, self.device, iegmn.graph_max_neighbor),
                            lambda plan: self._forward_plan(graph, plan, log, dropout))

    def _forward_plan(self, graph, plan, log, dropout=None):
        iegmn, dev, lib = self.iegmn, self.device, self.lib
        layers = [lay.packed(dev) for lay in iegmn.iegmn_layers]
        head = iegmn.packed_head(dev)
        nl, nr = graph.nodes[LIGAND].data, graph.nodes[RECEPTOR].data
        L = len(layers)
        with torch.cuda.device(dev):
            g = C.byref(plan.struct)
            stash_bytes = int(lib.eqd_forward_stash_bytes(g, L))
            offs = (C.c_size_t * 9)()
            nat.check(lib.eqd_forward_stash_offsets(g, L, offs), 'eqd_forward_stash_offsets')
            stash = torch.empty(stash_bytes, dtype=torch.uint8, device=dev)
            eng = IEGMNEngine(dev)
            emb32 = iegmn.residue_emb_layer.weight.detach().to(_f32).contiguous()
            out = eng.forward(plan, emb32, layers, head, nl['res_feat'], nr['res_feat'], nl['mu_r_norm'], nr['mu_r_norm'],
                              nl['new_x'], nr['x'], True, log, train_stash=stash, dropout=dropout)
        out.update(plan=plan, engine=eng, graph=graph, stash=stash, stash_offsets=list(offs), layers=layers, head=head,
                   res_l=nl['res_feat'].to(_f32).contiguous(), res_r=nr['res_feat'].to(_f32).contiguous(),
                   x_lig_in=nl['new_x'].to(_f32).contiguous())
        return out

    # ---- backward -------------------------------------------------------------------------------------------------
    def backward(self, fwd, d_coors, d_keypts, d_rot=None, d_trans=None, flat: Optional[torch.Tensor] = None,
                 on_bucket_done=None, capture: Optional[list] = None, d_x_out=None, d_h_out=None,
                 inputs_out: Optional[dict] = None) -> torch.Tensor:
        """Gradients of every parameter for upstream gradients w.r.t. the four raw outputs (ligand coordinates
        (N_l,3) f32, keypoints (2B,K,3) f64, rotations (B,3,3) f32, translations (B,1,3) f32; any may be None) and
        w.r.t. the last layer's coordinates and features (``d_x_out`` (N,3), ``d_h_out`` (N,64), global node order;
        None = no loss on them).
        Returns the flat gradient buffer (see ParamLayout).  ``on_bucket_done(label, lo, hi)`` is called on the host
        right after the kernels that complete a bucket have been queued (the data-parallel trainer launches that
        bucket's all-reduce there).  A dict ``inputs_out`` receives the gradients w.r.t. the graph's input tensors:
        'x_lig' (N_l,3) and 'x_rec' (N_r,3) f64, 'mu_lig' / 'mu_rec' (N,5) f32, 'he_lig' / 'he_rec' (E,27) f32 in the
        graph's own edge order.  Without it the input-gradient kernels are not launched; the parameter gradients are
        the same either way."""
        lib, dev, lay_out = self.lib, self.device, self.layout
        plan: GraphPlan = fwd['plan']
        iegmn = self.iegmn
        N, E, B = plan.N, plan.E, plan.n_pairs
        L = len(fwd['layers'])
        with torch.cuda.device(dev):
            st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            if self._ws is None or self._ws.key != (N, E, B) or self._ws_plan is not plan:
                self._ws = BackwardWorkspace(plan, dev, fwd['head'].n_heads)
                self._ws_plan = plan
            ws = self._ws
            if flat is None:
                flat = torch.zeros(lay_out.total, dtype=_f32, device=dev)
            g = C.byref(plan.struct)
            cf = lambda t, dt: None if t is None else t.detach().to(device=dev, dtype=dt).contiguous()
            d_coors, d_rot, d_trans = cf(d_coors, _f32), cf(d_rot, _f32), cf(d_trans, _f32)
            d_keypts = cf(d_keypts, torch.float64)
            off = lay_out.name_offset
            gk = flat[off['iegmn_original.att_mlp_key_ROT.0.weight']:]
            gq = flat[off['iegmn_original.att_mlp_query_ROT.0.weight']:]
            dh_cur, dh_nxt = ws.dh
            dx_cur, dx_nxt = ws.dx
            hd = fwd.get('dropout_head')
            nat.check(lib.eqd_bwd_head_dropout(g, C.byref(fwd['head'].struct), C.byref(hd) if hd is not None else None,
                                       nat.ptr(fwd['h']), nat.ptr(fwd['x64']),
                                       nat.ptr(fwd['cov']), nat.ptr(fwd['x_lig_in']), nat.ptr(d_coors), nat.ptr(d_keypts),
                                       nat.ptr(d_rot), nat.ptr(d_trans), nat.ptr(ws.head_ws), ws.head_ws_bytes,
                                       nat.ptr(dh_cur), nat.ptr(dx_cur), nat.ptr(ws.dpre), nat.ptr(gk), nat.ptr(gq), st),
                      'eqd_bwd_head_dropout')
            # eqd_bwd_head overwrote dh / dx: add the gradients that reach the last layer's outputs directly
            if d_x_out is not None:
                dx_cur.add_(d_x_out.detach().to(device=dev, dtype=torch.float64))
            if d_h_out is not None:
                dh_cur.reshape(-1)[:N * 64].view(N, 64).add_(d_h_out.detach().to(device=dev, dtype=_f32))
            dhe = dx_orig = None
            if inputs_out is not None:
                dhe = torch.zeros(max(E, 1), nat.EDGE_FEATS, dtype=_f32, device=dev)
                dx_orig = torch.zeros(N, 3, dtype=torch.float64, device=dev)
            if capture is not None:
                capture.append({'head': True, 'dh': dh_cur.reshape(-1)[:N * 64].clone().view(N, 64), 'dx': dx_cur.clone()})
            _weight_grads(lib, ws, (HEAD_REDUCTION,), self._head_maps, 'head', {'h': fwd['h']}, N, E, flat, st)
            buckets = {lab: (lo, hi) for lab, lo, hi in lay_out.buckets}
            if on_bucket_done:
                on_bucket_done('head', *buckets['head'])
            so = fwd['stash_offsets']
            sbase = fwd['stash'].data_ptr()
            sp = lambda o: C.c_void_p(sbase + o)
            h0_ptr = sp(so[0])
            ws.dh0.zero_()
            done_modules = set()
            first_use = {}
            for li, lm in enumerate(iegmn.iegmn_layers):
                first_use.setdefault(id(lm), li)
            for li in reversed(range(L)):
                lm = iegmn.iegmn_layers[li]
                h_in = h0_ptr if li == 0 else sp(so[3] + li * so[4])
                x_in = sp(so[1] + li * so[2])
                aggr, mu = sp(so[5] + li * so[6]), sp(so[7] + li * so[8])
                descs = fwd.get('dropout_layers')
                layer_backward(lib, plan, fwd['layers'][li], self.layer_pack(lm), ws, h_in, x_in, aggr, mu, h0_ptr,
                               dh_cur, dx_cur, dh_nxt, dx_nxt, flat, st, dhe, dx_orig, capture, li,
                               desc=descs[li] if descs is not None else None)
                dh_cur, dh_nxt = dh_nxt, dh_cur
                dx_cur, dx_nxt = dx_nxt, dx_cur
                if on_bucket_done and first_use[id(lm)] == li:   # a shared module completes at its FIRST use
                    lab = lay_out.module_bucket[id(lm)]
                    on_bucket_done(lab, *buckets[lab])
            demb = flat[off['iegmn_original.residue_emb_layer.weight']:]
            nat.check(lib.eqd_bwd_embed(g, nat.ptr(fwd['res_l']), nat.ptr(fwd['res_r']), nat.ptr(ws.dh0), nat.ptr(dh_cur),
                                        nat.ptr(demb), st), 'eqd_bwd_embed')
            if on_bucket_done:
                on_bucket_done('emb', *buckets['emb'])
            if inputs_out is not None:
                dmu = torch.empty(N, 5, dtype=_f32, device=dev)
                dx_in = torch.empty(N, 3, dtype=torch.float64, device=dev)
                mu = [fwd['graph'].nodes[nt].data['mu_r_norm'].detach().to(device=dev, dtype=_f32).contiguous()
                      for nt in (LIGAND, RECEPTOR)]
                nat.check(lib.eqd_bwd_inputs(g, nat.ptr(ws.dh0), nat.ptr(dh_cur), nat.ptr(mu[0]), nat.ptr(mu[1]),
                                             nat.ptr(dx_cur), nat.ptr(dx_orig), nat.ptr(fwd['rotation']), nat.ptr(d_coors),
                                             nat.ptr(dmu), nat.ptr(dx_in), st), 'eqd_bwd_inputs')
                N_l = plan.N_l
                dhe_l, dhe_r = plan.caller_edge_order(dhe)
                inputs_out.update(x_lig=dx_in[:N_l], x_rec=dx_in[N_l:], mu_lig=dmu[:N_l], mu_rec=dmu[N_l:],
                                  he_lig=dhe_l, he_rec=dhe_r)
        return flat


_INPUT_KEYS = ('x_lig', 'x_rec', 'mu_lig', 'mu_rec', 'he_lig', 'he_rec')   # TrainEngine.backward's inputs_out keys


class _HotPath(torch.autograd.Function):
    """autograd node of the whole hot path: forward = eqd_iegmn_forward with a stash, backward = the CUDA backward.
    Inputs: the graph's differentiable tensors (rigid_docking_model.graph_inputs; the forward reads them from the graph)
    and every parameter.  Outputs: the four raw outputs, then the last layer's coordinates (N,3) f64 and features
    (N,64) f32."""

    @staticmethod
    def forward(ctx, holder, x_lig, x_rec, mu_lig, mu_rec, he_lig, he_rec, *params):
        eng: TrainEngine = holder['engine']
        fwd = eng.forward(holder['graph'], holder.get('log'))
        holder['fwd'] = fwd
        ctx.holder = holder
        ctx.input_meta = [(t.dtype, t.device) for t in (x_lig, x_rec, mu_lig, mu_rec, he_lig, he_rec)]
        ctx.set_materialize_grads(False)    # an unused side output then costs nothing in the backward
        return fwd['ligand_coors'], fwd['keypts'], fwd['rotation'], fwd['translation'], fwd['x64'], fwd['h']

    @staticmethod
    def backward(ctx, d_coors, d_keypts, d_rot, d_trans, d_x, d_h):
        holder = ctx.holder
        eng: TrainEngine = holder['engine']
        fwd = holder['fwd']
        # zeros for the raw outputs without a gradient, as autograd would materialise them
        z = lambda d, key: torch.zeros_like(fwd[key]) if d is None else d
        d_coors, d_keypts = z(d_coors, 'ligand_coors'), z(d_keypts, 'keypts')
        d_rot, d_trans = z(d_rot, 'rotation'), z(d_trans, 'translation')
        need = ctx.needs_input_grad[1:1 + len(_INPUT_KEYS)]
        inputs = {} if any(need) else None
        flat = eng.backward(fwd, d_coors, d_keypts, d_rot, d_trans, d_x_out=d_x, d_h_out=d_h, inputs_out=inputs)
        in_grads = [inputs[k].to(device=dev, dtype=dt) if want else None
                    for k, want, (dt, dev) in zip(_INPUT_KEYS, need, ctx.input_meta)]
        return (None, *in_grads, *eng.layout.views(flat))


def check_fp32_precision(model):
    """The CUDA backward recomputes every layer from the stash in fp32 arithmetic: under ``precision='bf16x3'`` its
    gradients would not belong to the forward that ran, so training and autograd refuse that mode."""
    precision = getattr(model, 'iegmn_original', model).precision
    if precision != 'fp32':
        raise NotImplementedError(f"precision={precision!r} is an inference mode: autograd and training need "
                                  "precision='fp32' (the CUDA backward recomputes the forward in fp32)")


def autograd_forward(model, graph, log=None):
    """Runs the model's hot path as ONE autograd node and returns (raw outputs dict, the six differentiable outputs:
    ligand coordinates, keypoints, rotations, translations, last-layer coordinates (N,3) f64, last-layer features).
    ``model`` is a Rigid_Body_Docking_Net or an IEGMN module."""
    from .rigid_docking_model import graph_inputs
    check_fp32_precision(model)
    eng = getattr(model, '_eqd_train_engine', None)
    if eng is None or eng.device != getattr(model, 'iegmn_original', model).residue_emb_layer.weight.device:
        eng = TrainEngine(model)
        model._eqd_train_engine = eng
    holder = {'engine': eng, 'graph': graph, 'log': log}
    outs = _HotPath.apply(holder, *graph_inputs(graph), *eng.layout.params)
    return holder['fwd'], outs


# ---- one IEGMN_Layer as an autograd node ------------------------------------------------------------------------------

class LayerLayout:
    """Flat gradient layout of ONE IEGMN_Layer module: its parameters in ``module.parameters()`` order, each on a 256-byte
    boundary as in ParamLayout (LayerTrainPack's index maps read ``offset``)."""

    def __init__(self, layer_module):
        self.params, self.offset, self.total = [], {}, 0
        for p in layer_module.parameters():
            self.offset[id(p)] = self.total
            self.params.append(p)
            self.total += _padded(p.numel())

    views = ParamLayout.views


def layer_train_pack(layer_module, packed: PackedLayer, device):
    """(LayerLayout, LayerTrainPack) of a layer module for its current packed weights, cached on the module; the index
    maps are built once per module and device."""
    hit = getattr(layer_module, '_eqd_layer_train', None)
    if hit is not None and hit[0] is packed:
        return hit[1], hit[2]
    if hit is not None and hit[2].maps['proj'][0][0].device == torch.device(device):
        layout, maps = hit[1], hit[2].maps
    else:
        layout, maps = LayerLayout(layer_module), None
    tp = LayerTrainPack(layer_module, packed, layout, device, maps)
    layer_module._eqd_layer_train = (packed, layout, tp)
    return layout, tp


class _LayerFn(torch.autograd.Function):
    """autograd node of one IEGMN_Layer call: forward = eqd_project + eqd_iegmn_layer_forward (with mu), backward =
    layer_backward.  Inputs: the ten floating-point tensors of IEGMN_Layer.forward (ligand coordinates, features, original
    features, edge features, original coordinates, then the receptor's five) and the layer's parameters.  Outputs: the
    layer's coordinates (N,3) f64 and features (N,64) f32 of both proteins in global node order."""

    @staticmethod
    def forward(ctx, holder, x_l, h_l, h0_l, he_l, xo_l, x_r, h_r, h0_r, he_r, xo_r, *params):
        module, plan = holder['module'], holder['plan']
        inputs = (x_l, h_l, h0_l, he_l, xo_l, x_r, h_r, h0_r, he_r, xo_r)
        lay = module.packed(x_l.device)
        layout, tp = layer_train_pack(module, lay, x_l.device)
        desc = with_dropout([lay.struct], module.dropout_now())[0]   # each call is its own forward: own seed, layer 0
        h, h0, x_in, aggr, mu, h_out, x_out = run_layer(plan, lay, desc, inputs, keep_mu=True)
        ctx.saved = (plan, lay, layout, tp, h, h0, x_in, aggr, mu, desc)
        ctx.input_meta = [(t.dtype, t.device) for t in inputs]
        ctx.set_materialize_grads(False)    # a loss on only one of the two outputs launches nothing for the other
        return x_out, h_out

    @staticmethod
    def backward(ctx, d_x, d_h):
        plan, lay, layout, tp, h, h0, x_in, aggr, mu, desc = ctx.saved
        n_in = len(ctx.input_meta)
        if d_x is None and d_h is None:
            return (None,) * (1 + n_in + len(layout.params))
        dev, lib = h.device, nat.load()
        N, E, N_l = plan.N, plan.E, plan.N_l
        need = ctx.needs_input_grad[1:1 + n_in]
        with torch.cuda.device(dev):
            st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            ws = getattr(plan, '_eqd_layer_ws', None)
            if ws is None:
                ws = plan._eqd_layer_ws = BackwardWorkspace(plan, dev)
            # fresh, 16-byte aligned operands: every gradient handed to autograd is its own tensor, never the workspace
            dh_out = torch.zeros(N, nat.HID, dtype=_f32, device=dev)
            dx_out = torch.zeros(N, 3, dtype=torch.float64, device=dev)
            if d_h is not None:
                dh_out.copy_(d_h)
            if d_x is not None:
                dx_out.copy_(d_x)
            dh_in = torch.empty(N, lay.dhp, dtype=_f32, device=dev)
            dx_in = torch.empty(N, 3, dtype=torch.float64, device=dev)
            dhe = dx_orig = None
            if need[3] or need[4] or need[8] or need[9]:
                dhe = torch.zeros(max(E, 1), nat.EDGE_FEATS, dtype=_f32, device=dev)
                dx_orig = torch.zeros(N, 3, dtype=torch.float64, device=dev)
            flat = torch.zeros(layout.total, dtype=_f32, device=dev)
            ws.dh0.zero_()
            layer_backward(lib, plan, lay, tp, ws, h, x_in, aggr, mu, h0, dh_out, dx_out, dh_in, dx_in, flat, st, dhe,
                           dx_orig, desc=desc)
            dh0 = ws.dh0[:, :nat.H0].clone() if need[2] or need[7] else None
            if dhe is not None:
                dhe_l, dhe_r = plan.caller_edge_order(dhe)
        dh_in = dh_in[:, :lay.dh]
        per_side = {0: dx_in, 1: dh_in, 2: dh0, 4: dx_orig}
        grads = []
        for i, ((dt, d), want) in enumerate(zip(ctx.input_meta, need)):
            k, lig = i % 5, i < 5
            if not want:
                grads.append(None)
            elif k == 3:
                grads.append((dhe_l if lig else dhe_r).to(device=d, dtype=dt))
            else:
                t = per_side[k]
                grads.append((t[:N_l] if lig else t[N_l:]).to(device=d, dtype=dt))
        p_need = ctx.needs_input_grad[1 + n_in:]
        return (None, *grads, *[v if want else None for v, want in zip(layout.views(flat), p_need)])


def layer_autograd(module, plan: GraphPlan, inputs):
    """Runs one IEGMN_Layer call as an autograd node (see _LayerFn); ``inputs`` are the ten floating-point tensors of
    IEGMN_Layer.forward in its argument order.  Returns (coordinates (N,3) f64, features (N,64) f32), global node order."""
    return _LayerFn.apply({'module': module, 'plan': plan}, *inputs, *module.parameters())


# ---- fused data-parallel training step -------------------------------------------------------------------------------

def allreduce_buckets(flat: torch.Tensor, buckets, world: int, group=None):
    """Sum-all-reduce of a flat gradient buffer bucket by bucket (same result as one all-reduce of the whole buffer:
    buckets are disjoint slices).  Host-side helper shared by the trainer and the gloo test."""
    if world <= 1:
        return
    import torch.distributed as dist
    for _, lo, hi in buckets:
        dist.all_reduce(flat[lo:hi], op=dist.ReduceOp.SUM, group=group)


class DataParallelTrainer:
    """One training step of the reference (src/train.py:88-169) on the engine, data-parallel over pairs:

        forward (stash) -> device losses (MSE + exact-EMD OT + intersection, losses.cu) -> CUDA backward into ONE flat
        fp32 gradient -> per-bucket NCCL all-reduce on a side stream, launched as soon as a bucket's last kernel is
        queued (head first: 49 % of the parameters; then the layers last to first) so that it overlaps the rest of the
        backward -> global-norm partials -> fused clip_grad_norm_ + Adam on the flat parameter buffer.

    Each rank normalises its loss by its LOCAL pair count (train.py:143-146); gradients are averaged over ranks, which is
    the reference's global-batch mean when ranks hold equally many pairs.  The model's parameters are re-pointed at
    slices of one flat buffer (``param.data`` views), so the update is a single kernel and the all-reduce needs no
    packing."""

    def __init__(self, model, lr: float, weight_decay: float = 0.0, clip: float = 100.0, betas=(0.9, 0.999), eps: float = 1e-8,
                 pocket_ot_loss_weight: float = 1.0, intersection_loss_weight: float = 10.0, intersection_sigma: float = 25.0,
                 intersection_surface_ct: float = 10.0, world: int = 1, group=None):
        check_fp32_precision(model)
        self.model = model.train()
        self.engine = TrainEngine(model)
        self.layout = self.engine.layout
        dev = self.engine.device
        self.device, self.world, self.group = dev, int(world), group
        # zeroed: the alignment padding between parameters must stay 0, or Adam's weight decay would carry whatever it
        # held into m and v, and flat_w would differ between ranks there
        self.flat_w = torch.zeros(self.layout.total, dtype=_f32, device=dev)
        with torch.no_grad():
            for p, v in zip(self.layout.params, self.layout.views(self.flat_w)):
                v.copy_(p.detach().to(_f32))
                p.data = v                                       # parameters now live in the flat buffer
        self.m = torch.zeros_like(self.flat_w)
        self.v = torch.zeros_like(self.flat_w)
        self.flat_g = torch.zeros_like(self.flat_w)
        self.sq = torch.empty(256, dtype=torch.float64, device=dev)
        self.norm = torch.zeros(1, dtype=_f32, device=dev)
        self.hp = dict(lr=float(lr), wd=float(weight_decay), clip=float(clip), b1=float(betas[0]), b2=float(betas[1]), eps=float(eps))
        self.loss_args = (pocket_ot_loss_weight, intersection_loss_weight, intersection_sigma, intersection_surface_ct)
        self.steps = 0
        self.comm = torch.cuda.Stream(dev) if self.world > 1 else None
        if self.world > 1:
            import torch.distributed as dist
            self.engine.rank = dist.get_rank(group)
        self.lib = nat.load()

    def invalidate_packed(self):
        """Tells every cache of the weights that they changed.  eqd_clip_adam writes flat_w through a raw pointer, which
        moves neither a parameter's data_ptr nor its version counter; bumping the versions reaches every cache keyed on
        them: the packed layers and head (IEGMN_Layer.packed, IEGMN.packed_head), the training packs built on those
        (TrainEngine.layer_pack) and the CUDA graphs of the model's forward (graphed.GraphedForward), which re-capture
        at their next launch."""
        torch.autograd.graph.increment_version(self.layout.params)

    def step(self, graph, targets) -> Dict:
        from .losses import device_losses
        check_fp32_precision(self.model)
        dev, eng = self.device, self.engine
        with torch.cuda.device(dev):
            compute = torch.cuda.current_stream(dev)
            fwd = eng.forward(graph, self.model.log)
            res = device_losses(fwd['plan'], fwd['ligand_coors'], fwd['keypts'], targets, *self.loss_args)
            self.flat_g.zero_()                                  # optimizer.zero_grad() (train.py:88)

            def bucket_done(label, lo, hi):
                if self.world <= 1:
                    return
                import torch.distributed as dist
                ev = torch.cuda.Event()
                ev.record(compute)
                with torch.cuda.stream(self.comm):
                    self.comm.wait_event(ev)
                    dist.all_reduce(self.flat_g[lo:hi], op=dist.ReduceOp.SUM, group=self.group)

            eng.backward(fwd, res['dcoors'], res['dkeypts'], flat=self.flat_g, on_bucket_done=bucket_done)
            if self.world > 1:
                compute.wait_stream(self.comm)
            st = C.c_void_p(compute.cuda_stream)
            self.steps += 1
            nat.check(self.lib.eqd_sqnorm_partials(nat.ptr(self.flat_g), self.layout.total, nat.ptr(self.sq), 256, st), 'eqd_sqnorm_partials')
            h = self.hp
            nat.check(self.lib.eqd_clip_adam(nat.ptr(self.flat_w), nat.ptr(self.flat_g), nat.ptr(self.m), nat.ptr(self.v),
                                             self.layout.total, nat.ptr(self.sq), 256, h['clip'], h['lr'], h['b1'], h['b2'], h['eps'],
                                             h['wd'], self.steps, 1.0 / self.world, nat.ptr(self.norm), st), 'eqd_clip_adam')
            self.invalidate_packed()
        return {'loss': res['total'], 'grad_norm': self.norm, 'err': res['err'], 'fwd': fwd, 'parts': res['parts']}
