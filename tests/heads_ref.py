"""Models with num_att_heads = K keypoints per protein and the fp64 batch restatement the keypoint-count tests compare
against.  The restatement is tests/dropout_masks.py's model_forward (same inputs, same masks, same layers) with a K-head
keypoint read-out in place of its fixed 50 heads."""
import math

import numpy as np
import torch
import torch.nn.functional as F

import dropout_masks as dm
import golden_io as gio


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


def model_forward(sd, args, inp, masks=None):
    """dropout_masks.model_forward (same arguments and return value) with K = args['num_att_heads'] keypoints:
    (ligand coordinates (N_l,3), keypoints (2B,K,3), rotations (B,3,3), translations (B,3))."""
    B, seg = inp['B'], inp['seg']
    K = int(args['num_att_heads'])
    g = lambda k: sd['iegmn_original.' + k]
    h0 = torch.cat([g('residue_emb_layer.weight')[inp['res']], torch.log(inp['mu_r_norm'])], dim=1)
    x0 = inp['x']
    x, h = x0, h0
    L = int(args['iegmn_n_lays'])
    slope = float(args['leakyrelu_neg_slope'])
    for li in range(L):
        pre = f'iegmn_original.iegmn_layers.{li}.'
        p = {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}
        x, h = dm.layer_forward(p, x, h, x0, h0, inp['src'], inp['dst'], inp['he'], seg, B, slope,
                                float(args['skip_weight_h']), float(args['x_connection_init']), masks, li)
    pre = F.linear(h, g('mlp_h_mean_ROT.0.weight'), g('mlp_h_mean_ROT.0.bias'))
    if masks is not None:
        pre = pre * masks(L, 3)
    act = F.leaky_relu(pre, slope)
    d = h.shape[1]
    qbar = [act[seg[s]:seg[s + 1]].mean(0, keepdim=True) for s in range(2 * B)]
    Y = []
    for s in range(2 * B):
        o = s + B if s < B else s - B
        hk, z = h[seg[s]:seg[s + 1]], x[seg[s]:seg[s + 1]]
        keys = F.linear(hk, g('att_mlp_key_ROT.0.weight')).view(-1, K, d).transpose(0, 1)
        qry = F.linear(qbar[o], g('att_mlp_query_ROT.0.weight')).view(1, K, d).transpose(0, 1).transpose(1, 2)
        att = torch.softmax(keys @ qry / math.sqrt(d), dim=1).view(K, -1)
        Y.append(att @ z)
    coors, rots, trans = [], [], []
    for b in range(B):
        y_l, y_r = Y[b], Y[B + b]
        yr_m, yl_m = y_r.mean(0, keepdim=True), y_l.mean(0, keepdim=True)
        A = (y_r - yr_m).t() @ (y_l - yl_m)
        U, S, Vt = torch.linalg.svd(A)
        corr = torch.diag(torch.tensor([1., 1., float(torch.sign(torch.det(A.detach())))], dtype=A.dtype))
        T = (U @ corr) @ Vt
        t = yr_m - (T @ yl_m.t()).t()
        coors.append((T @ x0[seg[b]:seg[b + 1]].t()).t() + t)
        rots.append(T)
        trans.append(t)
    return torch.cat(coors), torch.stack(Y), torch.stack(rots), torch.cat(trans)
