"""fp64 batch restatement of the IEGMN layer with the reference's coordinate LayerNorm (layer_norm_coors='LN') and final
feature LayerNorm (final_h_layer_norm='LN'), and the models the layer-norm-option tests run.  The restatement is tests/dropout_masks.py's (same masks, same engine
numbering) with the one extra step of the reference's coors_mlp = Sequential(Linear, Dropout, LeakyReLU, LayerNorm,
Linear) (rigid_docking_model.py:199-201; the reference applies it to msg at :263):
    phi = coors_mlp.4(LayerNorm_c(LeakyReLU(coors_mlp.0(msg))))
and of the reference's apply_final_h_layer_norm (:349) after the skip combination:  h' = LayerNorm_f(skip(node_mlp(.))).
A layer whose parameters hold neither coors_mlp.3.* nor final_h_layernorm_layer.* is restated exactly as
tests/dropout_masks.py does."""
import numpy as np
import torch
import torch.nn.functional as F

import dropout_masks as dm
import golden_io as gio


def layer_forward(p, x, h, x0, h0, src, dst, he, seg, B, slope, skip, eta, masks=None, li=0):
    """dropout_masks.layer_forward with the coordinate LayerNorm when p has coors_mlp.3.weight."""
    lr = lambda t: F.leaky_relu(t, slope)
    N = x.shape[0]
    m = (lambda site, dh=64: masks(li, site, dh)) if masks is not None else (lambda site, dh=64: 1.0)
    x_rel = x[src] - x[dst]
    d2 = (x_rel ** 2).sum(1, keepdim=True)
    rbf = torch.cat([torch.exp(-d2 / sg) for sg in dm.SIGMAS], dim=-1)
    z1 = F.linear(torch.cat([h[src], h[dst], he, rbf], dim=-1), p['edge_mlp.0.weight'], p['edge_mlp.0.bias'])
    a = F.layer_norm(lr(z1 * m(0)), (z1.shape[1],), p['edge_mlp.3.weight'], p['edge_mlp.3.bias'])
    msg = F.linear(a, p['edge_mlp.4.weight'], p['edge_mlp.4.bias'])
    q = lr(F.linear(h, p['att_mlp_Q.0.weight']))
    k = lr(F.linear(h, p['att_mlp_K.0.weight']))
    v = F.linear(h, p['att_mlp_V.0.weight'])
    mu = []
    for s in range(2 * B):
        o = s + B if s < B else s - B
        a_, b_ = slice(seg[s], seg[s + 1]), slice(seg[o], seg[o + 1])
        mu.append(torch.softmax(q[a_] @ k[b_].t(), dim=1) @ v[b_])
    mu = torch.cat(mu)
    c3 = lr(F.linear(msg, p['coors_mlp.0.weight'], p['coors_mlp.0.bias']) * m(1))
    if 'coors_mlp.3.weight' in p:                                       # coors_mlp.3 = nn.LayerNorm(64)
        c3 = F.layer_norm(c3, (c3.shape[1],), p['coors_mlp.3.weight'], p['coors_mlp.3.bias'])
    coef = F.linear(c3, p['coors_mlp.4.weight'], p['coors_mlp.4.bias'])
    x_new = eta * x0 + (1. - eta) * x + dm._segmean(x_rel * coef, dst, N)
    u5 = F.linear(torch.cat([h, dm._segmean(msg, dst, N), mu, h0], dim=-1), p['node_mlp.0.weight'], p['node_mlp.0.bias'])
    hid = F.layer_norm(lr(u5 * m(2, u5.shape[1])), (u5.shape[1],), p['node_mlp.3.weight'], p['node_mlp.3.bias'])
    h_new = F.linear(hid, p['node_mlp.4.weight'], p['node_mlp.4.bias'])
    if h_new.shape[1] == h.shape[1]:
        h_new = skip * h_new + (1. - skip) * h
    if 'final_h_layernorm_layer.weight' in p:                           # apply_final_h_layer_norm (:349)
        h_new = F.layer_norm(h_new, (h_new.shape[1],), p['final_h_layernorm_layer.weight'],
                             p['final_h_layernorm_layer.bias'])
    return x_new, h_new


def model_forward(sd, args, inp, masks=None):
    """dropout_masks.model_forward (same arguments and return value) over layers restated by layer_forward above."""
    saved = dm.layer_forward
    dm.layer_forward = layer_forward
    try:
        return dm.model_forward(sd, args, inp, masks)
    finally:
        dm.layer_forward = saved


def args_with(ds, layer_norm_coors='LN', dropout=0.0, final_h_layer_norm='0'):
    a = gio.load_args(ds)
    a['layer_norm_coors'], a['dropout'], a['final_h_layer_norm'] = layer_norm_coors, dropout, final_h_layer_norm
    return a


def build_model(ds, device, args, seed=0, gamma_zero=False):
    """The shipped checkpoint of ``ds`` in a model built with ``args``; the optional LayerNorms the checkpoint lacks get
    seeded gamma ~ 1 + U(-0.5, 0.5) (gamma_zero: the coordinate LayerNorm's gamma is 0, what reset_parameters leaves; a
    final LayerNorm with gamma 0 would give every node the same features and a degenerate keypoint covariance) and
    beta ~ U(-0.2, 0.2), one draw per
    layer module (weight-shared layers share it).  Loads the completed state dict with strict=True."""
    from equidock_public_b200.rigid_docking_model import Rigid_Body_Docking_Net
    args = dict(args, device=device)
    model = Rigid_Body_Docking_Net(args)
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in gio.load_checkpoint(ds).items()}
    rng = np.random.default_rng(seed)
    drawn = {}
    for li, lay in enumerate(model.iegmn_original.iegmn_layers):
        for key, mod in (('coors_mlp.3', 'layer_norm_coors'), ('final_h_layernorm_layer', 'final_h_layer_norm')):
            if args[mod] != 'LN':
                continue
            if (id(lay), key) not in drawn:
                g = np.zeros(64) if gamma_zero and key == 'coors_mlp.3' else 1.0 + rng.uniform(-0.5, 0.5, 64)
                drawn[(id(lay), key)] = (torch.from_numpy(g.astype(np.float32)),
                                         torch.from_numpy(rng.uniform(-0.2, 0.2, 64).astype(np.float32)))
            pre = f'iegmn_original.iegmn_layers.{li}.{key}.'
            sd[pre + 'weight'], sd[pre + 'bias'] = drawn[(id(lay), key)]
    model.load_state_dict(sd, strict=True)
    return model.to(device).eval()
