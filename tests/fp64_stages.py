"""Torch fp64 evaluations of the forward stage formulas of one IEGMN_Layer (rigid_docking_model.py line numbers), from an
engine layer module's weights.  Used by the per-kernel forward tests and the backward attention test; every function
takes and returns fp64 tensors on the device and works under autograd."""
import torch
import torch.nn.functional as F

F64 = torch.float64
SIGMAS = [1.5 ** s for s in range(15)]      # all_sigmas_dist (:116)


def _w(lin):
    return lin.weight.detach().to(F64)


def _b(lin):
    return lin.bias.detach().to(F64)


def projections(mod, h):
    """Psrc, Pdst (+ edge_mlp.0.bias), Q, K, V of h [n][dh] (:130-140, 229-231): the groups of eqd_layer_params.w_proj."""
    dh, slope = h.shape[1], float(mod.leakyrelu_neg_slope)
    w1 = _w(mod.edge_mlp[0])
    return {'Psrc': h @ w1[:, :dh].t(), 'Pdst': h @ w1[:, dh:2 * dh].t() + _b(mod.edge_mlp[0]),
            'Q': F.leaky_relu(h @ _w(mod.att_mlp_Q[0]).t(), slope), 'K': F.leaky_relu(h @ _w(mod.att_mlp_K[0]).t(), slope),
            'V': h @ _w(mod.att_mlp_V[0]).t()}


def attention(seg, q, k, v):
    """mu = softmax(q k^T) v of every protein over its partner's nodes (:46-64, 247-256); seg = host seg_ptr [2B+1]."""
    B = (len(seg) - 1) // 2
    parts = []
    for s in range(2 * B):
        p = s + B if s < B else s - B
        a, b, c, d = int(seg[s]), int(seg[s + 1]), int(seg[p]), int(seg[p + 1])
        parts.append(torch.softmax(q[a:b] @ k[c:d].t(), 1) @ v[c:d])
    return torch.cat(parts, 0)


def edge_stage(mod, plan, proj, x_in):
    """Edge stage (:204-237, 263-283) from this layer's projections P [n][pw] (Psrc at 0, Pdst at 64) and coordinates
    x_in: returns aggr [n][64] = mean of msg over in-edges and xupd [n][3] = mean of x_rel * phi (0 without in-edges)."""
    slope, dh = float(mod.leakyrelu_neg_slope), int(mod.att_mlp_Q[0].weight.shape[0])
    lin1, ln, lin2 = mod.edge_mlp[0], mod.edge_mlp[3], mod.edge_mlp[4]
    lin3, lin4 = mod.coors_mlp[0], mod.coors_mlp[4]
    N, dev = plan.N, x_in.device
    src, dst = plan.col_src.long(), plan.edge_dst.long()
    he = torch.cat([plan.he_l, plan.he_r]).to(F64)
    xrel = x_in[src] - x_in[dst]
    d2 = (xrel ** 2).sum(1, keepdim=True)
    ein = torch.cat([he] + [torch.exp(-d2 / sg) for sg in SIGMAS], 1)
    z1 = proj[src, 0:64] + proj[dst, 64:128] + ein @ _w(lin1)[:, 2 * dh:].t()
    n1 = F.layer_norm(F.leaky_relu(z1, slope), (64,), _w(ln), _b(ln), ln.eps)
    msg = n1 @ _w(lin2).t() + _b(lin2)
    phi = F.leaky_relu(msg @ _w(lin3).t() + _b(lin3), slope) @ _w(lin4).t() + _b(lin4)
    deg = (plan.row_ptr[1:] - plan.row_ptr[:-1]).to(dev, F64).clamp(min=1)[:, None]
    aggr = torch.zeros(N, 64, dtype=F64, device=dev).index_add_(0, dst, msg) / deg
    xupd = torch.zeros(N, 3, dtype=F64, device=dev).index_add_(0, dst, xrel * phi) / deg
    return aggr, xupd


def node_mlp(mod, h, aggr, mu, h0):
    """node_mlp([h | aggr | mu | h0]) (:319-329) and the skip connection of the 64-wide layers (:332-337)."""
    slope, sk = float(mod.leakyrelu_neg_slope), float(mod.skip_weight_h)
    lin0, ln, lin4 = mod.node_mlp[0], mod.node_mlp[3], mod.node_mlp[4]
    u5 = torch.cat([h, aggr, mu, h0], 1) @ _w(lin0).t() + _b(lin0)
    o = F.layer_norm(F.leaky_relu(u5, slope), (u5.shape[1],), _w(ln), _b(ln), ln.eps) @ _w(lin4).t() + _b(lin4)
    return sk * o + (1.0 - sk) * h if h.shape[1] == o.shape[1] else o
