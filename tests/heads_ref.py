"""Models with num_att_heads = K keypoints per protein and the fp64 batch restatement the keypoint-count tests compare
against.  The restatement is tests/dropout_masks.py's model_forward (same inputs, same masks, same layers) with a K-head
keypoint read-out in place of its fixed 50 heads, and the reference's SVD degeneracy loop in front of Kabsch (its noise
replayed from the engine's torch seed by replay_draws)."""
import contextlib
import math

import numpy as np
import torch
import torch.nn.functional as F

import dropout_masks as dm
import golden_io as gio
import iegmn_oracle as orc


def args_with(ds, K, dropout=0.0):
    a = gio.load_args(ds)
    a['num_att_heads'], a['dropout'] = K, dropout
    return a


def head_weights(sd, K, rng):
    """att_mlp_key_ROT / att_mlp_query_ROT weights (64K, 64) for K heads: the shipped 50 heads in a seeded order (the
    first K of them, or all 50 and K - 50 drawn again), each head perturbed by 0.2 x the weights' standard deviation, so
    that the keypoints spread like a trained model's and no two heads are equal."""
    idx = rng.permutation(50)
    if K > 50:
        idx = np.concatenate([idx, rng.choice(50, K - 50)])
    out = {}
    for key in ('att_mlp_key_ROT.0.weight', 'att_mlp_query_ROT.0.weight'):
        w = np.asarray(sd['iegmn_original.' + key], np.float64).reshape(50, 64, 64)[idx[:K]]
        w = w + 0.2 * w.std() * rng.standard_normal(w.shape)
        out['iegmn_original.' + key] = torch.from_numpy(w.reshape(64 * K, 64).astype(np.float32))
    return out


def build_model(ds, device, K, seed=0, dropout=0.0):
    """The shipped checkpoint of ``ds`` with K-head key / query projections from head_weights, loaded with
    strict=True."""
    from equidock_public_b200.rigid_docking_model import Rigid_Body_Docking_Net
    args = dict(args_with(ds, K, dropout), device=device)
    model = Rigid_Body_Docking_Net(args)
    ck = gio.load_checkpoint(ds)
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in ck.items()}
    sd.update(head_weights(ck, K, np.random.default_rng(seed)))
    model.load_state_dict(sd, strict=True)
    return model.to(device).eval()


def model_forward(sd, args, inp, masks=None, rand_diag=None):
    """dropout_masks.model_forward (same arguments) with K = args['num_att_heads'] keypoints and the reference's SVD
    guard (keypoint_tail; ``rand_diag`` is its noise source): (ligand coordinates (N_l,3), keypoints (2B,K,3), rotations
    (B,3,3), translations (B,3), guard draws per pair [B])."""
    h0 = torch.cat([sd['iegmn_original.residue_emb_layer.weight'][inp['res']], torch.log(inp['mu_r_norm'])], dim=1)
    x0 = inp['x']
    x, h = x0, h0
    L = int(args['iegmn_n_lays'])
    slope = float(args['leakyrelu_neg_slope'])
    for li in range(L):
        pre = f'iegmn_original.iegmn_layers.{li}.'
        p = {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}
        x, h = dm.layer_forward(p, x, h, x0, h0, inp['src'], inp['dst'], inp['he'], inp['seg'], inp['B'], slope,
                                float(args['skip_weight_h']), float(args['x_connection_init']), masks, li)
    return keypoint_tail(sd, h, x, x0[:inp['seg'][inp['B']]], inp['seg'], inp['B'], int(args['num_att_heads']), slope,
                         masks(L, 3) if masks is not None else None, rand_diag)


GUARD_EXIT = 'SVD consistently numerically unstable! Exitting ... '      # rigid_docking_model.py:583


def guarded_kabsch(A, rand_diag=None):
    """Kabsch on one 3x3 keypoint covariance A (fp64, may require grad) behind the reference's degeneracy loop
    (rigid_docking_model.py:570-587): while iegmn_oracle.svd_guard_flags fires on the fp32-rounded singular values (the
    rule of kabsch_apply_kernel), A += diag(rand_diag()), a constant; after the 11th draw SystemExit without a re-test,
    as the reference does.  The guard firing with no ``rand_diag`` raises RuntimeError.  Returns (T = U corr Vt of the
    perturbed A, corr = diag(1, 1, sign det A), number of draws, the perturbed A)."""
    draws = 0
    while orc.svd_guard_flags(torch.linalg.svdvals(A.detach()).float().numpy()):
        if rand_diag is None:
            raise RuntimeError('heads_ref: the SVD guard fired and no noise source was given')
        A = A + torch.diag(torch.as_tensor(rand_diag(), dtype=A.dtype))
        draws += 1
        if draws > 10:
            raise SystemExit(GUARD_EXIT)
    U, _, Vt = torch.linalg.svd(A)
    corr = torch.diag(torch.tensor([1., 1., float(torch.sign(torch.det(A.detach())))], dtype=A.dtype))
    return (U @ corr) @ Vt, draws, A


def keypoint_tail(sd, h, x, x_lig, seg, B, K, slope, pre_mask=None, rand_diag=None, qbar_value=None, trace=None):
    """The keypoint head and Kabsch (rigid_docking_model.py:521-600, 665) over a batch in engine numbering from the last
    layer's h (N,64) / x (N,3): K-head keypoints, the guarded Kabsch of every pair (pairs in order, so ``rand_diag`` is
    called in the order the engine draws), the rigid transform of the input ligand coordinates ``x_lig`` (N_l,3).
    ``pre_mask``: the dropout factor of mlp_h_mean_ROT's output (site 3).  ``qbar_value`` (2B,64): the value the segment
    means of the head's activations take (their gradient stays that of the fp64 means), to evaluate the tail at a
    kernel's own fp32 means.  ``trace`` (dict) receives 'pre' (mlp_h_mean_ROT's output, grad retained) and the perturbed
    covariances 'A' (B,3,3).  Returns (ligand coordinates, keypoints (2B,K,3), rotations (B,3,3), translations (B,3),
    draws per pair)."""
    g = lambda k: sd['iegmn_original.' + k]
    pre = F.linear(h, g('mlp_h_mean_ROT.0.weight'), g('mlp_h_mean_ROT.0.bias'))
    if trace is not None:
        if pre.requires_grad:
            pre.retain_grad()
        trace['pre'] = pre
    act = F.leaky_relu(pre * pre_mask if pre_mask is not None else pre, slope)
    d = h.shape[1]
    qbar = torch.cat([act[seg[s]:seg[s + 1]].mean(0, keepdim=True) for s in range(2 * B)])
    if qbar_value is not None:
        qbar = qbar_value.to(qbar.dtype) + (qbar - qbar.detach())
    Y = []
    for s in range(2 * B):
        o = s + B if s < B else s - B
        hk, z = h[seg[s]:seg[s + 1]], x[seg[s]:seg[s + 1]]
        keys = F.linear(hk, g('att_mlp_key_ROT.0.weight')).view(-1, K, d).transpose(0, 1)
        qry = F.linear(qbar[o:o + 1], g('att_mlp_query_ROT.0.weight')).view(1, K, d).transpose(0, 1).transpose(1, 2)
        att = torch.softmax(keys @ qry / math.sqrt(d), dim=1).view(K, -1)
        Y.append(att @ z)
    coors, rots, trans, draws, covs = [], [], [], [], []
    for b in range(B):
        y_l, y_r = Y[b], Y[B + b]
        yr_m, yl_m = y_r.mean(0, keepdim=True), y_l.mean(0, keepdim=True)
        T, n, A = guarded_kabsch((y_r - yr_m).t() @ (y_l - yl_m), rand_diag)
        t = yr_m - (T @ yl_m.t()).t()
        coors.append((T @ x_lig[seg[b]:seg[b + 1]].t()).t() + t)
        rots.append(T)
        trans.append(t)
        draws.append(n)
        covs.append(A.detach())
    if trace is not None:
        trace['A'] = torch.stack(covs)
    return torch.cat(coors), torch.stack(Y), torch.stack(rots), torch.cat(trans), draws


def replay_draws(seed, p=0.0, training=True, rank=0):
    """``torch.manual_seed(seed)`` and the CPU-generator draws of one engine forward from there, in the engine's order:
    first the dropout seed (engine.draw_dropout; training mode with p > 0 only), then, through the returned callable,
    the diagonal of one ``torch.rand(3, 3)`` per guard retry, flagged pairs in pair order (IEGMNEngine._resolve_status).
    Returns (draw_dropout's tuple or None, rand_diag for keypoint_tail / guarded_kabsch)."""
    from equidock_public_b200.engine import draw_dropout
    torch.manual_seed(seed)
    dropout = draw_dropout(p, rank) if training else None
    return dropout, lambda: torch.rand(3, 3).diagonal().double()


@contextlib.contextmanager
def kink_branch(band, positive):
    """Within the block, every LeakyReLU (torch.nn.functional.leaky_relu) whose input lies within ``band`` x its row's
    max |input| of the kink keeps its value but takes the derivative of the ``positive`` (1) or the negative (slope)
    side.  An fp32 evaluation resolves such inputs only to about 1e-6 of the row's scale and may take either side there,
    so two fp64 evaluations, one per side, bound what the choice alone can change in a gradient."""
    orig = F.leaky_relu

    def leaky(t, negative_slope=0.01, inplace=False):
        y = orig(t, negative_slope)
        z = t.detach().abs()
        near = (z <= band * z.amax(dim=-1, keepdim=True)) & (z > 0)
        d = 1.0 if positive else negative_slope
        return torch.where(near, y.detach() + (t - t.detach()) * d, y)
    F.leaky_relu = leaky
    try:
        yield
    finally:
        F.leaky_relu = orig
