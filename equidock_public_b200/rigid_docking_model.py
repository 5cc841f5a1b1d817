"""Drop-in replacement for the reference's ``src/model/rigid_docking_model.py`` whose arithmetic
runs in hand-written sm_90a CUDA kernels (``csrc/``) behind the C ABI of ``include/eqd_iegmn.h``.

Same public surface as the reference module (it is star-imported by ``src/utils/train_utils.py:14``,
which ``train.py`` / ``inference_rigid.py`` star-import in turn, so the module-level names ``nn``,
``math``, ``torch``, ``dgl``, ``fn``, ``sys`` are part of the contract):

* ``IEGMN_Layer(orig_h_feats_dim, h_feats_dim, out_feats_dim, fine_tune, args, log=None)``  (:83-91)
* ``IEGMN(args, n_lays, fine_tune, log=None)``                                              (:362)
* ``Rigid_Body_Docking_Net(args, log=None)`` / ``model(batch_hetero_graph, epoch)``          (:613, :642)
* ``compute_cross_attention``, ``get_mask``, ``get_non_lin``, ``get_layer_norm``,
  ``get_final_h_layer_norm``, ``apply_final_h_layer_norm``                                  (:10-78)

Parameter names and shapes equal the reference's ``state_dict`` (SURVEY 8b), so both shipped
checkpoints load with ``strict=True``.  The graph argument may be a batched DGL heterograph
(``train_utils.py:61-100``) or this package's DGL-free ``PairGraphBatch``.

Scope of this engine: forward AND backward of the configuration the shipped checkpoints use
(``nonlin='lkyrelu'``, ``layer_norm='LN'``, ``layer_norm_coors='0'``, ``final_h_layer_norm='0'``,
``cross_msgs``, ``use_dist_in_layers``, ``rot_model='kb_att'``, ``fine_tune=False``), and ``layer_norm_coors='LN'`` (the
coordinate MLP's ``coors_mlp.3`` LayerNorm) and ``final_h_layer_norm='LN'`` (``final_h_layernorm_layer`` on each layer's
node output), both in the CUDA forward and backward.  ``dropout > 0`` is applied in
training mode, as ``nn.Dropout`` does, with masks from a counter-based generator seeded per forward from torch's default
CPU generator (``engine.draw_dropout``): same distribution as torch's, a different random stream.
Anything else raises ``NotImplementedError``; a missing CUDA library raises -- there is no CPU path.
In training mode (``model.train()`` with grad enabled), and in any mode when one of the graph's ``new_x`` / ``x`` /
``mu_r_norm`` / ``he`` requires grad, the outputs of ``Rigid_Body_Docking_Net.forward`` are autograd-connected: the whole
path is one autograd node backed by the CUDA backward kernels (``training.py``), differentiable with respect to every
parameter and to those graph tensors.  ``IEGMN.forward`` runs the same node under the same condition.  ``IEGMN_Layer.forward``
is differentiable on its own under that condition (its ten tensor arguments in place of the graph tensors): each call is
one autograd node whose backward is the CUDA per-layer backward (``training.layer_backward``), so models built from the
layers train like the reference's.
"""
import math  # noqa: F401  (re-exported, see module docstring)
import numbers
import sys  # noqa: F401

import torch
from torch import nn

try:  # the real DGL when the reference's environment provides it
    import dgl
    from dgl import function as fn
except ImportError:  # DGL-free deployments use the package's own container
    from . import hetero_graph as dgl
    fn = None

from . import _native as nat
from .engine import (PRECISIONS, GraphPlan, IEGMNEngine, PackedHead, PackedLayer, check_precision, draw_dropout, plan_for,
                     retry_sorted, run_layer, with_dropout)
from .hetero_graph import LIGAND, LL, RECEPTOR, RR


# ---- factory helpers (reference :10-42) --------------------------------------------------------

def get_non_lin(type, negative_slope):
    if type == 'swish':
        return nn.SiLU()
    assert type == 'lkyrelu'
    return nn.LeakyReLU(negative_slope=negative_slope)


def get_layer_norm(layer_norm_type, dim):
    if layer_norm_type == 'BN':
        return nn.BatchNorm1d(dim)
    if layer_norm_type == 'LN':
        return nn.LayerNorm(dim)
    return nn.Identity()


def get_final_h_layer_norm(layer_norm_type, dim):
    if layer_norm_type == 'BN':
        return nn.BatchNorm1d(dim)
    if layer_norm_type == 'LN':
        return nn.LayerNorm(dim)
    if layer_norm_type == 'GN':
        raise NotImplementedError("final_h_layer_norm='GN' is outside the CUDA engine's scope")
    assert layer_norm_type == '0'
    return nn.Identity()


def apply_final_h_layer_norm(g, h, node_type, norm_type, norm_layer):
    if norm_type == 'GN':
        return norm_layer(g, h, node_type)
    return norm_layer(h)


def get_mask(ligand_batch_num_nodes, receptor_batch_num_nodes, device):
    """Block-diagonal 0/1 mask of the reference's dense batched attention (:68-78).  Kept for API
    parity only: the engine's attention is segmented per pair and never materialises it."""
    rows, cols = int(sum(ligand_batch_num_nodes)), int(sum(receptor_batch_num_nodes))
    mask = torch.zeros(rows, cols, device=device)
    r = c = 0
    for l_n, r_n in zip(ligand_batch_num_nodes, receptor_batch_num_nodes):
        l_n, r_n = int(l_n), int(r_n)
        mask[r:r + l_n, c:c + r_n] = 1
        r, c = r + l_n, c + r_n
    return mask


def compute_cross_attention(queries, keys, values, mask, cross_msgs):
    """Dense masked attention with the reference's formula (:46-64), in plain torch ops.  API parity
    helper for callers outside the hot path; the engine itself uses the fused segmented kernel."""
    if not cross_msgs:
        return queries * 0.
    a = mask * torch.mm(queries, keys.t()) - 1000. * (1. - mask)
    return torch.mm(torch.softmax(a, dim=1), values)


# ---- shared host-side plumbing -------------------------------------------------------------------

# args values the CUDA engine implements (the first is the shipped checkpoints' configuration)
_SUPPORTED = {'nonlin': ('lkyrelu',), 'layer_norm': ('LN',), 'layer_norm_coors': ('0', 'LN'), 'final_h_layer_norm': ('0', 'LN'),
              'cross_msgs': (True,), 'use_dist_in_layers': (True,)}


def _check_layer_args(args):
    for k, vs in _SUPPORTED.items():
        if args[k] not in vs:
            raise NotImplementedError(f"args[{k!r}]={args[k]!r}: the CUDA engine implements {' / '.join(map(repr, vs))} only")


def _layer_plan(graph, device, max_in_degree, he_l, he_r):
    """GraphPlan of an IEGMN_Layer call under autograd: the graph's cached plan when ``he_l`` / ``he_r`` are the tensors it
    was built from, else one built with the caller's edge features.  Edges not grouped by destination get a
    destination-sorted copy whose ``edge_perm`` maps edge gradients back to the caller's order."""
    plan = plan_for(graph, device, max_in_degree)
    if plan.edge_perm is None and bool(plan.unsorted.item()):
        plan = plan_for(graph, device, max_in_degree, sort=True)
    if plan.edge_perm is None and he_l.data_ptr() == plan.he_l.data_ptr() and he_r.data_ptr() == plan.he_r.data_ptr():
        return plan
    return GraphPlan.from_graph(graph, device, max_in_degree, (he_l.detach(), he_r.detach()), sort=plan.edge_perm is not None)


def _wants_autograd(module, tensors):
    """The condition under which a module's forward runs as an autograd node: grad mode on, and training mode,
    ``force_autograd``, or an input tensor that requires grad."""
    return torch.is_grad_enabled() and (module.training or getattr(module, 'force_autograd', False)
                                        or any(t.requires_grad for t in tensors))


def graph_inputs(graph):
    """The graph's floating-point tensors the reference differentiates through: ligand ``new_x``, receptor ``x``,
    ligand / receptor ``mu_r_norm``, ``he`` of the ligand / receptor edges.  (``res_feat`` enters through ``.long()``.)"""
    nl, nr = graph.nodes[LIGAND].data, graph.nodes[RECEPTOR].data
    return nl['new_x'], nr['x'], nl['mu_r_norm'], nr['mu_r_norm'], graph.edges[LL].data['he'], graph.edges[RR].data['he']


def _module_state(module):
    return {k: v for k, v in module.state_dict(keep_vars=True).items()}


def _version_key(module):
    return tuple((p.data_ptr(), p._version) for p in module.parameters())


def _reset_parameters(module):
    for p in module.parameters():
        if p.dim() > 1:
            torch.nn.init.xavier_normal_(p, gain=1.)
        else:
            torch.nn.init.zeros_(p)


class IEGMN_Layer(nn.Module):
    """Parameters of one IEGMN layer (same names/shapes as the reference, :119-159) and its
    per-layer operator ``forward`` (:189-352) on the CUDA engine."""

    def __init__(self, orig_h_feats_dim, h_feats_dim, out_feats_dim, fine_tune, args, log=None):
        super().__init__()
        _check_layer_args(args)
        if fine_tune:
            raise NotImplementedError("fine_tune=True ('didn't work', args.py:110) is outside the engine's scope")
        edge_in = args['input_edge_feats_dim']
        drop, slope = args['dropout'], args['leakyrelu_neg_slope']
        act = lambda: get_non_lin(args['nonlin'], slope)
        self.cross_msgs = args['cross_msgs']
        self.final_h_layer_norm = args['final_h_layer_norm']
        self.layer_norm_coors = args['layer_norm_coors']
        self.use_dist_in_layers = args['use_dist_in_layers']
        self.skip_weight_h = args['skip_weight_h']
        self.x_connection_init = args['x_connection_init']
        self.leakyrelu_neg_slope = slope
        self.dropout_p = drop
        self.fine_tune = fine_tune
        self.debug, self.device, self.log = args['debug'], args['device'], log
        self.h_feats_dim, self.out_feats_dim = h_feats_dim, out_feats_dim
        self.graph_max_neighbor = int(args.get('graph_max_neighbor', 10) or 10)
        self.all_sigmas_dist = [1.5 ** x for x in range(15)]
        n_rbf = len(self.all_sigmas_dist)

        self.edge_mlp = nn.Sequential(nn.Linear(2 * h_feats_dim + edge_in + n_rbf, out_feats_dim), nn.Dropout(drop),
                                      act(), get_layer_norm(args['layer_norm'], out_feats_dim),
                                      nn.Linear(out_feats_dim, out_feats_dim))
        self.node_norm = nn.Identity()
        self.att_mlp_Q = nn.Sequential(nn.Linear(h_feats_dim, h_feats_dim, bias=False), act())
        self.att_mlp_K = nn.Sequential(nn.Linear(h_feats_dim, h_feats_dim, bias=False), act())
        self.att_mlp_V = nn.Sequential(nn.Linear(h_feats_dim, h_feats_dim, bias=False))
        self.node_mlp = nn.Sequential(nn.Linear(orig_h_feats_dim + 2 * h_feats_dim + out_feats_dim, h_feats_dim),
                                      nn.Dropout(drop), act(), get_layer_norm(args['layer_norm'], h_feats_dim),
                                      nn.Linear(h_feats_dim, out_feats_dim))
        self.final_h_layernorm_layer = get_final_h_layer_norm(self.final_h_layer_norm, out_feats_dim)
        self.coors_mlp = nn.Sequential(nn.Linear(out_feats_dim, out_feats_dim), nn.Dropout(drop), act(),
                                       get_layer_norm(args['layer_norm_coors'], out_feats_dim),
                                       nn.Linear(out_feats_dim, 1))
        if edge_in != nat.EDGE_FEATS or out_feats_dim != nat.HID or orig_h_feats_dim != nat.H0:
            raise NotImplementedError('CUDA engine widths: input_edge_feats_dim=27, hidden 64, node input 69')
        self._packed, self._packed_key = None, None

    reset_parameters = _reset_parameters

    def packed(self, device) -> PackedLayer:
        """Kernel-layout copy of the parameters, rebuilt only when a parameter changed."""
        key = (_version_key(self), str(device))
        if self._packed is None or self._packed_key != key:
            self._packed = PackedLayer(_module_state(self), device, float(self.skip_weight_h),
                                       float(self.x_connection_init), float(self.leakyrelu_neg_slope),
                                       layer_norm_coors=self.layer_norm_coors,
                                       final_h_layer_norm=self.final_h_layer_norm)
            self._packed_key = key
        return self._packed

    def dropout_now(self, rank: int = 0):
        """The dropout of one call of this layer (or of a stack it leads): engine.draw_dropout's (p, seed, rank) in
        training mode with dropout > 0, else None (no draw from the generator)."""
        return draw_dropout(self.dropout_p, rank) if self.training else None

    def forward(self, hetero_graph, coors_ligand, h_feats_ligand, original_ligand_node_features,
                original_edge_feats_ligand, orig_coors_ligand, coors_receptor, h_feats_receptor,
                original_receptor_node_features, original_edge_feats_receptor, orig_coors_receptor):
        """Per-layer operator with the reference's signature and return value
        ``(x_final_ligand, node_upd_ligand, x_final_receptor, node_upd_receptor)``.  In training mode (grad enabled), with
        ``force_autograd``, or when an input requires grad, the call is one autograd node whose backward is the CUDA
        per-layer backward (``training.layer_backward``): gradients reach the layer's parameters and all ten tensor
        inputs."""
        inputs = (coors_ligand, h_feats_ligand, original_ligand_node_features, original_edge_feats_ligand,
                  orig_coors_ligand, coors_receptor, h_feats_receptor, original_receptor_node_features,
                  original_edge_feats_receptor, orig_coors_receptor)
        dev = coors_ligand.device
        if _wants_autograd(self, inputs):
            from .training import layer_autograd
            plan = _layer_plan(hetero_graph, dev, self.graph_max_neighbor, inputs[3], inputs[8])
            x_out, h_out = layer_autograd(self, plan, inputs)
        else:
            plan = plan_for(hetero_graph, dev, self.graph_max_neighbor)
            if original_edge_feats_ligand.data_ptr() != plan.he_l.data_ptr():  # caller scaled / replaced he
                plan = GraphPlan.from_graph(hetero_graph, dev, self.graph_max_neighbor,
                                            (original_edge_feats_ligand, original_edge_feats_receptor))
            lay = self.packed(dev)
            desc = with_dropout([lay.struct], self.dropout_now())[0]   # each call is its own forward: own seed, layer 0
            h_out, x_out = run_layer(plan, lay, desc, inputs, keep_mu=False)[5:]
            if bool(plan.unsorted.item()):
                raise nat.NativeLibraryError('IEGMN_Layer.forward: edges must be grouped by destination')
        x_out = x_out.to(coors_ligand.dtype)
        return x_out[:plan.N_l], h_out[:plan.N_l], x_out[plan.N_l:], h_out[plan.N_l:]

    def __repr__(self):
        return 'IEGMN Layer (H100 engine) ' + str({k: v for k, v in self.__dict__.items() if not k.startswith('_')})


class IEGMN(nn.Module):
    """Embedding + IEGMN layer stack + keypoint attention + Kabsch (reference :360-606)."""

    def __init__(self, args, n_lays, fine_tune, log=None):
        super().__init__()
        self.debug, self.log = args['debug'], log
        self.device = args['device']
        self.graph_nodes = args['graph_nodes']
        self.rot_model = args['rot_model']
        self.noise_decay_rate, self.noise_initial = args['noise_decay_rate'], args['noise_initial']
        self.use_edge_features_in_gmn = args['use_edge_features_in_gmn']
        self.use_mean_node_features = args['use_mean_node_features']
        self.leakyrelu_neg_slope = args['leakyrelu_neg_slope']
        self.graph_max_neighbor = int(args.get('graph_max_neighbor', 10) or 10)
        assert self.graph_nodes == 'residues'
        assert args['rot_model'] == 'kb_att'
        if not (self.use_edge_features_in_gmn and self.use_mean_node_features):
            raise NotImplementedError('CUDA engine: use_edge_features_in_gmn and use_mean_node_features must be on')

        if int(args['residue_emb_dim']) != nat.HID:
            raise NotImplementedError(f'CUDA engine: residue_emb_dim must be {nat.HID}')
        self.residue_emb_layer = nn.Embedding(num_embeddings=21, embedding_dim=args['residue_emb_dim'])
        in_dim = args['residue_emb_dim'] + 5  # + mu_r_norm surface features (:387-388)
        hid = args['iegmn_lay_hid_dim']
        self.iegmn_layers = nn.ModuleList()
        self.iegmn_layers.append(IEGMN_Layer(in_dim, in_dim, hid, fine_tune, args, log))
        if args['shared_layers']:
            shared = IEGMN_Layer(in_dim, hid, hid, fine_tune, args, log)
            for _ in range(1, n_lays):
                self.iegmn_layers.append(shared)
        else:
            for _ in range(1, n_lays):
                self.iegmn_layers.append(IEGMN_Layer(in_dim, hid, hid, fine_tune, args, log))

        heads = args['num_att_heads']
        self.out_feats_dim = hid
        if isinstance(heads, bool) or not isinstance(heads, numbers.Integral) or not 1 <= heads <= nat.MAX_HEADS:
            raise NotImplementedError(f'CUDA engine: num_att_heads must be an integer from 1 to {nat.MAX_HEADS} '
                                      f'(the exact-EMD solver takes at most {nat.MAX_HEADS} keypoints), got {heads!r}')
        self.num_att_heads = int(heads)
        self.att_mlp_key_ROT = nn.Sequential(nn.Linear(hid, self.num_att_heads * hid, bias=False))
        self.att_mlp_query_ROT = nn.Sequential(nn.Linear(hid, self.num_att_heads * hid, bias=False))
        self.mlp_h_mean_ROT = nn.Sequential(nn.Linear(hid, hid), nn.Dropout(args['dropout']),
                                            get_non_lin(args['nonlin'], args['leakyrelu_neg_slope']))
        self._head, self._head_key = None, None
        self.last_outputs = None
        self._precision = 'fp32'

    @property
    def precision(self) -> str:
        """Arithmetic of the tensor-core GEMMs of layers 1..L-1 at inference: ``'fp32'`` (default; bf16x6, fp32-level
        agreement with an fp64 evaluation) or ``'bf16x3'`` (three products on two-term bf16 splits, about 2^-16 relative
        error per product, half the tensor-core work).  Layer 0, the keypoint head and Kabsch are the same in both.  The
        autograd paths refuse ``'bf16x3'``."""
        return self._precision

    @precision.setter
    def precision(self, value: str):
        self._precision = check_precision(value)

    reset_parameters = _reset_parameters

    def packed_head(self, device) -> PackedHead:
        mods = (self.att_mlp_key_ROT, self.att_mlp_query_ROT, self.mlp_h_mean_ROT)
        key = (tuple(_version_key(m) for m in mods), str(device))
        if self._head is None or self._head_key != key:
            self._head = PackedHead(self.mlp_h_mean_ROT[0].weight, self.mlp_h_mean_ROT[0].bias,
                                    self.att_mlp_key_ROT[0].weight, self.att_mlp_query_ROT[0].weight, device,
                                    float(self.leakyrelu_neg_slope))
            self._head_key = key
        return self._head

    def run_engine(self, batch_hetero_graph, check_status=True, record_event=True):
        """The whole hot path on the device; returns the engine's raw output dict.  With ``check_status=False`` the
        per-pair status words are left pending (``resolve(out)`` finishes the call).  ``record_event=False`` is for
        CUDA-graph capture (``graphed.GraphedForward``), which records its own completion event per replay.  In
        training mode this forward's dropout is drawn here (engine.draw_dropout)."""
        dev = self.residue_emb_layer.weight.device
        dropout = self.iegmn_layers[0].dropout_now() if self.training else None
        return retry_sorted(batch_hetero_graph, plan_for(batch_hetero_graph, dev, self.graph_max_neighbor),
                            lambda plan: self._launch(batch_hetero_graph, plan, check_status, record_event, dropout))

    def _launch(self, batch_hetero_graph, plan, check_status, record_event, dropout):
        emb = self.residue_emb_layer.weight
        dev = emb.device
        eng = IEGMNEngine(dev)
        layers = [lay.packed(dev) for lay in self.iegmn_layers]
        nl, nr = batch_hetero_graph.nodes[LIGAND].data, batch_hetero_graph.nodes[RECEPTOR].data
        out = eng.forward(plan, emb.detach().to(torch.float32).contiguous(), layers, self.packed_head(dev), nl['res_feat'],
                          nr['res_feat'], nl['mu_r_norm'], nr['mu_r_norm'], nl['new_x'], nr['x'], check_status, self.log,
                          record_event=record_event, mma_products=PRECISIONS[self.precision], dropout=dropout)
        out['plan'], out['engine'], out['graph'], out['dropout'] = plan, eng, batch_hetero_graph, dropout
        return out

    def resolve(self, out):
        """Finishes a ``run_engine(..., check_status=False)`` call: waits for its status words and replays the
        reference's host-side control flow for flagged pairs (:570-584).  Unsorted edge lists are re-run sorted."""
        def finish(plan):
            if plan is not out['plan']:     # re-run sorted: the same forward, so the same dropout seed
                return self._launch(out['graph'], plan, True, True, out['dropout'])
            out['engine'].resolve_status(plan, out, out['kabsch'], self.log)
            return out
        return retry_sorted(out['graph'], out['plan'], finish)

    def forward(self, batch_hetero_graph, epoch):
        """Returns ``[T list, b list, Y_ligand list, Y_receptor list]`` like the reference (:602) and
        writes ``x_iegmn_out`` / ``hv_iegmn_out`` into the graph (:507-510).  Under the condition of
        ``Rigid_Body_Docking_Net.forward`` the whole stack is the same single autograd node (``training._HotPath``)."""
        if _wants_autograd(self, graph_inputs(batch_hetero_graph)):
            from .training import autograd_forward
            fwd, outs = autograd_forward(self, batch_hetero_graph, self.log)
            return self.package(fwd, batch_hetero_graph, outs[1:])
        return self.package(self.run_engine(batch_hetero_graph), batch_hetero_graph)

    def package(self, out, batch_hetero_graph, tensors=None):
        """The reference's return value from a forward's raw output dict ``out``; ``tensors`` = (keypoints, rotations,
        translations, last-layer coordinates, last-layer features) are used in place of the dict's (the differentiable
        outputs of an autograd node)."""
        keypts, rot, trans, x_fin, h_fin = tensors if tensors is not None else (
            out['keypts'], out['rotation'], out['translation'], out['x64'], out['h'])
        B, N_l = out['plan'].n_pairs, out['plan'].N_l
        nl, nr = batch_hetero_graph.nodes[LIGAND].data, batch_hetero_graph.nodes[RECEPTOR].data
        dt = nl['new_x'].dtype
        x_fin = x_fin.to(dt)
        nl['x_iegmn_out'], nr['x_iegmn_out'] = x_fin[:N_l], x_fin[N_l:]
        nl['hv_iegmn_out'], nr['hv_iegmn_out'] = h_fin[:N_l], h_fin[N_l:]
        keyp = keypts.to(dt)
        self.last_outputs = out
        return [list(rot.unbind(0)), list(trans.unbind(0)), list(keyp[:B].unbind(0)), list(keyp[B:].unbind(0))]

    def __repr__(self):
        return 'IEGMN (H100 engine) ' + str({k: v for k, v in self.__dict__.items() if not k.startswith('_')})


class Rigid_Body_Docking_Net(nn.Module):
    """``model(batch_hetero_graph, epoch)`` -> (ligand coords list, ligand keypoints list, receptor
    keypoints list, rotations list, translations list), reference :611-696."""

    def __init__(self, args, log=None):
        super().__init__()
        self.debug, self.log, self.device = args['debug'], log, args['device']
        if args['fine_tune']:
            raise NotImplementedError("fine_tune=True is outside the CUDA engine's scope (both checkpoints: fine_F)")
        self.iegmn_original = IEGMN(args, n_lays=args['iegmn_n_lays'], fine_tune=False, log=log)
        self.list_iegmns = [('finetune', self.iegmn_original)]

    @property
    def precision(self) -> str:
        """``IEGMN.precision`` of the model's IEGMN: ``'fp32'`` (default) or ``'bf16x3'``."""
        return self.iegmn_original.precision

    @precision.setter
    def precision(self, value: str):
        self.iegmn_original.precision = value

    reset_parameters = _reset_parameters

    def forward_async(self, batch_hetero_graph, epoch=0):
        """Launches the whole forward without waiting for its status words; ``.result()`` of the returned handle
        completes it and returns the reference's 5-tuple.  Lets a serving loop keep several batches in flight."""
        net, raw = self, self.iegmn_original.run_engine(batch_hetero_graph, check_status=False)

        class Pending:
            def raw_result(self_inner):
                """The engine's batched output dict (``ligand_coors`` (sum N_l, 3), ``rotation`` (B, 3, 3),
                ``translation`` (B, 1, 3), ``keypts`` (2B, K, 3), ...) once the status words are resolved."""
                return net.iegmn_original.resolve(raw)

            def result(self_inner):
                out = net.iegmn_original.resolve(raw)
                return net._assemble(net.iegmn_original.package(out, batch_hetero_graph))
        return Pending()

    def graphed(self, device_batch):
        """A CUDA-graph capture of this model's forward for one fixed-shape device batch (``graphed.GraphedForward``):
        ``.launch().result()`` returns what ``model(batch, epoch)`` returns at the host cost of one graph launch."""
        from .graphed import GraphedForward
        return GraphedForward(self, device_batch)

    def forward(self, batch_hetero_graph, epoch):
        """Training mode (``model.train()``, src/train.py:64), or any mode when a graph input tensor requires grad: the
        whole hot path is ONE autograd node whose backward is the hand-written CUDA backward (``training.TrainEngine``), so
        ``loss.backward()`` (train.py:154) fills ``param.grad`` of every parameter and ``.grad`` of the graph's ``new_x`` /
        ``x`` / ``mu_r_norm`` / ``he`` exactly like the reference's autograd graph does.  Outputs, and ``x_iegmn_out`` /
        ``hv_iegmn_out`` in the graph, are autograd-connected views of the node's outputs.  Evaluation under
        ``torch.no_grad()``, or in ``model.eval()`` with no input requiring grad, keeps the inference path."""
        if _wants_autograd(self, graph_inputs(batch_hetero_graph)):
            from .training import autograd_forward
            fwd, outs = autograd_forward(self, batch_hetero_graph, self.log)
            return self._assemble(self.iegmn_original.package(fwd, batch_hetero_graph, outs[1:]), outs[0])
        return self._assemble(self.iegmn_original(batch_hetero_graph, epoch))

    def _assemble(self, outputs, ligand_coors=None):
        """The 5-tuple from IEGMN's four lists and the batched ligand coordinates (default: the last forward's)."""
        assert len(outputs) == 4
        raw = self.iegmn_original.last_outputs
        if ligand_coors is None:
            ligand_coors = raw['ligand_coors']
        # T new_x + b of every ligand node was applied by the Kabsch kernel (:665)
        ligand_coors = list(torch.split(ligand_coors, raw['plan'].n_lig_list, dim=0))
        for b_align in outputs[1]:
            assert b_align.shape[0] == 1 and b_align.shape[1] == 3
        return ligand_coors, outputs[2], outputs[3], outputs[0], outputs[1]

    def __repr__(self):
        return 'Rigid_Body_Docking_Net (H100 engine) ' + str({k: v for k, v in self.__dict__.items()
                                                              if not k.startswith('_')})
