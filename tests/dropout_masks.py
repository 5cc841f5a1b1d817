"""The training-mode dropout masks of the engine (eqd_dropout, include/eqd_iegmn.h; csrc/philox.cuh) restated in numpy,
and an fp64 torch restatement of the model's forward in the engine's batch numbering that applies them, so that the
CUDA forward and backward under dropout can be checked against torch.autograd on the same masks.

keep(seed, rank, layer, site, row, col) = philox4x32_10(counter = (row, col >> 2, (layer << 2) | site, rank),
                                                        key = (lo32(seed), hi32(seed)))[col & 3] >= round(p * 2^32)
"""
from __future__ import annotations

import functools
import math

import numpy as np
import torch
import torch.nn.functional as F

_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on uint32 arrays (broadcast); returns the four output words as uint32 arrays."""
    c = [np.asarray(v, np.uint64) & _M32 for v in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(int(k0) & 0xFFFFFFFF), np.uint64(int(k1) & 0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M32]
        k0 = (k0 + np.uint64(0x9E3779B9)) & _M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & _M32
    return [v.astype(np.uint32) for v in c]


def threshold(p):
    return min(int(round(float(p) * 2.0 ** 32)), 0xFFFFFFFF)


def scale(p):
    return 0.0 if p >= 1.0 else float(np.float32(1.0 / (1.0 - float(p))))


def keep(seed, rank, layer, site, rows, cols, p):
    """Boolean [len(rows)][len(cols)]: which elements of a dropout site the engine keeps."""
    if p >= 1.0:
        return np.zeros((len(rows), len(cols)), bool)
    r = np.asarray(rows, np.uint64)[:, None]
    c = np.asarray(cols, np.uint64)[None, :]
    w = philox4x32_10(r, c >> np.uint64(2), (int(layer) << 2) | int(site), int(rank), int(seed) & 0xFFFFFFFF,
                      (int(seed) >> 32) & 0xFFFFFFFF)
    word = np.choose((c & np.uint64(3)).astype(np.int64), w)
    return word >= np.uint32(threshold(p))


@functools.lru_cache(maxsize=64)
def _keep_all(seed, rank, layer, site, n_rows, n_cols, p):
    """keep over every row and column, cached: the masks of a 400 k-edge batch take seconds in numpy, and the forward
    and backward tests of a stage draw the same ones."""
    k = keep(seed, rank, layer, site, np.arange(n_rows), np.arange(n_cols), p)
    k.setflags(write=False)
    return k


def mask(seed, rank, layer, site, n_rows, n_cols, p):
    """keep * scale as an fp64 torch tensor [n_rows][n_cols] (the factor the engine multiplies the site by)."""
    k = _keep_all(int(seed), int(rank), int(layer), int(site), int(n_rows), int(n_cols), float(p))
    return torch.from_numpy(k.astype(np.float64) * scale(p))


class BatchMasks:
    """The masks of one forward over a batch of N nodes / E edges and L layers (None = dropout off)."""

    def __init__(self, p, seed, rank, N, E, L, dh0=69):
        self.p, self.seed, self.rank, self.N, self.E, self.L, self.dh0 = p, seed, rank, N, E, L, dh0

    def __call__(self, layer, site, dh=64):
        rows = self.E if site < 2 else self.N
        return mask(self.seed, self.rank, layer, site, rows, dh if site == 2 else 64, self.p)


SIGMAS = [1.5 ** s for s in range(15)]


def _segmean(v, idx, n):
    out = torch.zeros((n,) + tuple(v.shape[1:]), dtype=v.dtype, device=v.device).index_add_(0, idx, v)
    deg = torch.zeros(n, dtype=v.dtype, device=v.device).index_add_(0, idx, torch.ones(idx.shape[0], dtype=v.dtype,
                                                                                      device=v.device))
    return out / deg.clamp(min=1).unsqueeze(1)


def layer_forward(p, x, h, x0, h0, src, dst, he, seg, B, slope, skip, eta, masks=None, li=0):
    """One IEGMN layer over the whole batch in engine numbering (p: name -> tensor of the layer's parameters; seg:
    node offsets of the 2B segments).  Returns (x_new, h_new)."""
    lr = lambda t: F.leaky_relu(t, slope)
    N = x.shape[0]
    m = (lambda site, dh=64: masks(li, site, dh)) if masks is not None else (lambda site, dh=64: 1.0)
    x_rel = x[src] - x[dst]
    d2 = (x_rel ** 2).sum(1, keepdim=True)
    rbf = torch.cat([torch.exp(-d2 / sg) for sg in SIGMAS], dim=-1)
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
    z3 = F.linear(msg, p['coors_mlp.0.weight'], p['coors_mlp.0.bias'])
    coef = F.linear(lr(z3 * m(1)), p['coors_mlp.4.weight'], p['coors_mlp.4.bias'])
    x_new = eta * x0 + (1. - eta) * x + _segmean(x_rel * coef, dst, N)
    u5 = F.linear(torch.cat([h, _segmean(msg, dst, N), mu, h0], dim=-1), p['node_mlp.0.weight'], p['node_mlp.0.bias'])
    hid = F.layer_norm(lr(u5 * m(2, u5.shape[1])), (u5.shape[1],), p['node_mlp.3.weight'], p['node_mlp.3.bias'])
    h_new = F.linear(hid, p['node_mlp.4.weight'], p['node_mlp.4.bias'])
    if h_new.shape[1] == h.shape[1]:
        h_new = skip * h_new + (1. - skip) * h
    return x_new, h_new


def model_forward(sd, args, inp, masks=None):
    """Rigid_Body_Docking_Net's forward over a batch in engine numbering, fp64.  sd: name -> tensor (leaves may require
    grad); inp: dict of res (N,), mu_r_norm (N,5), x (N,3) (ligand new_x, receptor x), src / dst (E,), he (E,27),
    seg (2B+1,), B.  Returns (ligand coordinates (N_l,3), keypoints (2B,50,3), rotations (B,3,3), translations (B,3))."""
    B, seg = inp['B'], inp['seg']
    g = lambda k: sd['iegmn_original.' + k]
    h0 = torch.cat([g('residue_emb_layer.weight')[inp['res']], torch.log(inp['mu_r_norm'])], dim=1)
    x0 = inp['x']
    x, h = x0, h0
    L = int(args['iegmn_n_lays'])
    slope = float(args['leakyrelu_neg_slope'])
    for li in range(L):
        pre = f'iegmn_original.iegmn_layers.{li}.'
        p = {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}
        x, h = layer_forward(p, x, h, x0, h0, inp['src'], inp['dst'], inp['he'], seg, B, slope,
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
        keys = F.linear(hk, g('att_mlp_key_ROT.0.weight')).view(-1, 50, d).transpose(0, 1)
        qry = F.linear(qbar[o], g('att_mlp_query_ROT.0.weight')).view(1, 50, d).transpose(0, 1).transpose(1, 2)
        att = torch.softmax(keys @ qry / math.sqrt(d), dim=1).view(50, -1)
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
