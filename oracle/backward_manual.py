"""TEST INFRASTRUCTURE -- hand-derived BACKWARD of the IEGMN hot path in numpy fp64, stage by stage with the same stage
boundaries as the CUDA backward kernels (csrc/bwd_*.cu), so that a GPU test can compare every kernel's outputs with the
corresponding arrays here and a wrong gradient is localised to one kernel in one run.

The reference has no backward code of its own: its gradients are whatever ``loss.backward()`` (src/train.py:154) makes of
the forward in src/model/rigid_docking_model.py.  This file restates the chain rule of that forward (line numbers cite
it); it is pinned by tests/test_backward_manual.py against ``torch.autograd`` on the torch restatement
(``iegmn_oracle_torch.TorchOracle``, itself pinned against the unmodified reference's autograd by
tests/golden/*_grads.npz).

Layout: ONE pair, ``sides`` = [ligand, receptor]; every stage function takes / returns per-side arrays.
"""
from __future__ import annotations

import math
from typing import Dict, List

import numpy as np

from iegmn_oracle import SIGMAS, LayerParams, OracleConfig, leaky_relu, linear

EPS = 1e-5


def lrelu_grad(pre, slope):
    """d leaky_relu / d pre, PyTorch convention (pre > 0 ? 1 : slope)."""
    return np.where(pre > 0, 1.0, slope)


def ln_forward(a, g, b):
    mean = a.mean(-1, keepdims=True)
    var = ((a - mean) ** 2).mean(-1, keepdims=True)
    rstd = 1.0 / np.sqrt(var + EPS)
    nhat = (a - mean) * rstd
    return nhat * g + b, nhat, rstd


def ln_backward(dn, nhat, rstd, g):
    """-> (da, dgamma, dbeta) for n = nhat * g + b."""
    dg, db = (dn * nhat).sum(0), dn.sum(0)
    dnh = dn * g
    da = rstd * (dnh - dnh.mean(-1, keepdims=True) - nhat * (dnh * nhat).mean(-1, keepdims=True))
    return da, dg, db


def seg_mean(values, dst, n):
    out = np.zeros((n,) + values.shape[1:])
    np.add.at(out, dst, values)
    deg = np.bincount(dst, minlength=n).astype(np.float64)
    return out / np.maximum(deg, 1).reshape((n,) + (1,) * (values.ndim - 1)), deg


# ---- forward of one layer with everything the backward needs -------------------------------------------------------

def layer_forward(p: LayerParams, cfg: OracleConfig, sides) -> List[Dict]:
    """IEGMN_Layer.forward (:189-352) keeping the intermediates.  Returns one cache dict per side."""
    slope, dh = cfg.slope, p.h_dim
    caches = []
    for s in sides:
        h = s['h']
        c = {'h': h, 'x': s['x'], 'h0': s['h0'], 'he': s['he'], 'src': s['src'], 'dst': s['dst'], 'x_orig': s['x_orig']}
        c['qpre'], c['kpre'] = linear(h, p.wq), linear(h, p.wk)
        c['q'], c['k'], c['v'] = leaky_relu(c['qpre'], slope), leaky_relu(c['kpre'], slope), linear(h, p.wv)
        c['psrc'] = linear(h, p.edge_w1[:, 0:dh])                    # per-node split of edge_mlp.0 (:186, 229-231)
        c['pdst'] = linear(h, p.edge_w1[:, dh:2 * dh], p.edge_b1)
        caches.append(c)
    for i, c in enumerate(caches):
        o = caches[1 - i]
        src, dst, n = c['src'], c['dst'], c['x'].shape[0]
        c['xrel'] = c['x'][src] - c['x'][dst]                        # :204-205
        d2 = (c['xrel'] ** 2).sum(1, keepdims=True)
        c['rbf'] = np.concatenate([np.exp(-d2 / sg) for sg in SIGMAS], 1)   # :208-214
        c['ein'] = np.concatenate([c['he'], c['rbf']], 1)            # (E, 42)
        c['z1'] = c['psrc'][src] + c['pdst'][dst] + c['ein'] @ p.edge_w1[:, 2 * dh:].T
        a1 = leaky_relu(c['z1'], slope)
        c['n1'], c['nhat1'], c['rstd1'] = ln_forward(a1, p.edge_ln_g, p.edge_ln_b)
        c['msg'] = linear(c['n1'], p.edge_w2, p.edge_b2)             # :236
        c['z3'] = linear(c['msg'], p.coor_w1, p.coor_b1)
        c['c3'] = leaky_relu(c['z3'], slope)
        c['phi'] = linear(c['c3'], p.coor_w2, p.coor_b2)             # (E,1) :263
        c['aggr'], c['deg'] = seg_mean(c['msg'], dst, n)             # :280-283
        xupd, _ = seg_mean(c['xrel'] * c['phi'], dst, n)             # :264, 274-277
        c['x_new'] = cfg.x_connection_init * c['x_orig'] + (1 - cfg.x_connection_init) * c['x'] + xupd
        S = c['q'] @ o['k'].T                                        # :61-63 pair block, no 1/sqrt(d)
        S = S - S.max(1, keepdims=True)
        P = np.exp(S)
        c['P'] = P / P.sum(1, keepdims=True)
        c['mu'] = c['P'] @ o['v']
        c['inp'] = np.concatenate([c['h'], c['aggr'], c['mu'], c['h0']], 1)   # :319-329
        c['u5'] = linear(c['inp'], p.node_w1, p.node_b1)
        a5 = leaky_relu(c['u5'], slope)
        c['n5'], c['nhat5'], c['rstd5'] = ln_forward(a5, p.node_ln_g, p.node_ln_b)
        o6 = linear(c['n5'], p.node_w2, p.node_b2)
        c['skip'] = p.h_dim == p.out_dim
        c['h_new'] = cfg.skip_weight_h * o6 + (1 - cfg.skip_weight_h) * c['h'] if c['skip'] else o6
    return caches


def zero_layer_grads(p: LayerParams):
    return {k: np.zeros_like(getattr(p, k)) for k in ('edge_w1', 'edge_b1', 'edge_ln_g', 'edge_ln_b', 'edge_w2', 'edge_b2',
                                                     'wq', 'wk', 'wv', 'node_w1', 'node_b1', 'node_ln_g', 'node_ln_b',
                                                     'node_w2', 'node_b2', 'coor_w1', 'coor_b1', 'coor_w2', 'coor_b2')}


# ---- stage 1: node MLP backward (kernel bwd_node_mlp) --------------------------------------------------------------

def node_mlp_bwd(p, cfg, c, dh_new, G):
    """d h_new (N,64) -> contributions to dh (skip + W5's h block), daggr, dmu, dh0; accumulates weight grads in G."""
    dh_, slope = p.h_dim, cfg.slope
    do = cfg.skip_weight_h * dh_new if c['skip'] else dh_new
    dh = (1 - cfg.skip_weight_h) * dh_new if c['skip'] else np.zeros_like(c['h'])
    G['node_w2'] += do.T @ c['n5']
    G['node_b2'] += do.sum(0)
    dn = do @ p.node_w2
    da, dg, db = ln_backward(dn, c['nhat5'], c['rstd5'], p.node_ln_g)
    G['node_ln_g'] += dg
    G['node_ln_b'] += db
    du = da * lrelu_grad(c['u5'], slope)
    G['node_w1'] += du.T @ c['inp']
    G['node_b1'] += du.sum(0)
    dinp = du @ p.node_w1
    dh = dh + dinp[:, 0:dh_]
    return dh, dinp[:, dh_:dh_ + 64], dinp[:, dh_ + 64:2 * dh_ + 64], dinp[:, 2 * dh_ + 64:]


# ---- stage 2: cross attention backward (kernels bwd_attn_dq / bwd_attn_dkv) ----------------------------------------

def attn_bwd(cfg, caches, dmu):
    """dmu per side -> (dqpre, dkpre, dv) per side (pre-activation grads of Q, K; V is linear)."""
    dq = [None, None]
    dk = [np.zeros_like(c['k']) for c in caches]
    dv = [np.zeros_like(c['v']) for c in caches]
    for i, c in enumerate(caches):
        o = caches[1 - i]
        D = (dmu[i] * c['mu']).sum(1, keepdims=True)
        dP = dmu[i] @ o['v'].T
        dS = c['P'] * (dP - D)
        dq[i] = dS @ o['k']
        dk[1 - i] += dS.T @ c['q']
        dv[1 - i] += c['P'].T @ dmu[i]
    out = []
    for i, c in enumerate(caches):
        out.append((dq[i] * lrelu_grad(c['qpre'], cfg.slope), dk[i] * lrelu_grad(c['kpre'], cfg.slope), dv[i]))
    return out


# ---- stage 3: edge backward (kernel bwd_edge) + stage 4: gather (kernel bwd_edge_gather) ----------------------------

def edge_bwd(p, cfg, c, daggr, dx_new, G):
    """-> per-edge dz1 (E,64), dxrel (E,3); accumulates the edge / coordinate MLP weight grads."""
    slope, dh_ = cfg.slope, p.h_dim
    dst = c['dst']
    deg = np.maximum(c['deg'], 1)[dst][:, None]
    dmsg = daggr[dst] / deg
    dxm = dx_new[dst] / deg                                          # d (xrel * phi) per edge
    dphi = (c['xrel'] * dxm).sum(1, keepdims=True)
    dxrel = c['phi'] * dxm
    G['coor_w2'] += dphi.T @ c['c3']
    G['coor_b2'] += dphi.sum(0)
    dz3 = (dphi @ p.coor_w2) * lrelu_grad(c['z3'], slope)
    G['coor_w1'] += dz3.T @ c['msg']
    G['coor_b1'] += dz3.sum(0)
    dmsg = dmsg + dz3 @ p.coor_w1
    G['edge_w2'] += dmsg.T @ c['n1']
    G['edge_b2'] += dmsg.sum(0)
    dn = dmsg @ p.edge_w2
    da, dg, db = ln_backward(dn, c['nhat1'], c['rstd1'], p.edge_ln_g)
    G['edge_ln_g'] += dg
    G['edge_ln_b'] += db
    dz1 = da * lrelu_grad(c['z1'], slope)
    G['edge_w1'][:, 2 * dh_:] += dz1.T @ c['ein']
    drbf = dz1 @ p.edge_w1[:, 2 * dh_ + 27:]                         # (E,15)
    dd2 = (drbf * c['rbf'] * (-1.0 / np.asarray(SIGMAS))).sum(1, keepdims=True)
    dxrel = dxrel + 2.0 * c['xrel'] * dd2
    return dz1, dxrel


def edge_gather(cfg, c, dz1, dxrel, dx_new):
    """Per node: dPsrc = sum over OUT-edges of dz1, dPdst = sum over IN-edges, dx = (1-eta) dx_new + sum_out dxrel - sum_in."""
    n = c['x'].shape[0]
    dpsrc, dpdst = np.zeros((n, 64)), np.zeros((n, 64))
    np.add.at(dpsrc, c['src'], dz1)
    np.add.at(dpdst, c['dst'], dz1)
    dx = (1 - cfg.x_connection_init) * dx_new
    np.add.at(dx, c['src'], dxrel)
    np.add.at(dx, c['dst'], -dxrel)
    return dpsrc, dpdst, dx


# ---- stage 5: projection backward (kernel bwd_proj) ----------------------------------------------------------------

def proj_bwd(p, c, dpsrc, dpdst, dqpre, dkpre, dv, G):
    dh_ = p.h_dim
    h = c['h']
    G['edge_w1'][:, 0:dh_] += dpsrc.T @ h
    G['edge_w1'][:, dh_:2 * dh_] += dpdst.T @ h
    G['edge_b1'] += dpdst.sum(0)
    G['wq'] += dqpre.T @ h
    G['wk'] += dkpre.T @ h
    G['wv'] += dv.T @ h
    return (dpsrc @ p.edge_w1[:, 0:dh_] + dpdst @ p.edge_w1[:, dh_:2 * dh_] + dqpre @ p.wq + dkpre @ p.wk + dv @ p.wv)


def layer_backward(p, cfg, caches, dh_new, dx_new, G, stages=None):
    """Whole-layer backward for one pair: (dh_new, dx_new per side) -> (dh, dx, dh0 per side)."""
    nm = [node_mlp_bwd(p, cfg, c, dh_new[i], G) for i, c in enumerate(caches)]
    att = attn_bwd(cfg, caches, [m[2] for m in nm])
    out = []
    for i, c in enumerate(caches):
        dh_part, daggr, dmu, dh0 = nm[i]
        dz1, dxrel = edge_bwd(p, cfg, c, daggr, dx_new[i], G)
        dpsrc, dpdst, dx = edge_gather(cfg, c, dz1, dxrel, dx_new[i])
        dqpre, dkpre, dv = att[i]
        dh = dh_part + proj_bwd(p, c, dpsrc, dpdst, dqpre, dkpre, dv, G)
        out.append((dh, dx, dh0))
        if stages is not None:
            stages.append({'side': i, 'dh_part': dh_part, 'daggr': daggr, 'dmu': dmu, 'dh0': dh0, 'dz1': dz1, 'dxrel': dxrel,
                           'dpsrc': dpsrc, 'dpdst': dpdst, 'dx': dx, 'dqpre': dqpre, 'dkpre': dkpre, 'dv': dv, 'dh': dh,
                           'z1': c['z1'], 'z3': c['z3'], 'u5': c['u5']})
    return out


# ---- head: keypoints + Kabsch ---------------------------------------------------------------------------------------

def head_forward(sd, cfg, h_l, x_l, h_r, x_r):
    """IEGMN.forward :521-589 with the intermediates (folded form u_k = W_K,k^T (W_Q,k qbar) / 8)."""
    g = lambda k: np.asarray(sd['iegmn_original.' + k], np.float64)
    c = {'wm': g('mlp_h_mean_ROT.0.weight'), 'bm': g('mlp_h_mean_ROT.0.bias'),
         'wk': g('att_mlp_key_ROT.0.weight').reshape(cfg.num_att_heads, 64, 64),      # [k][e][d]
         'wq': g('att_mlp_query_ROT.0.weight').reshape(cfg.num_att_heads, 64, 64)}     # [k][e][d']
    H, X = [h_l, h_r], [x_l, x_r]
    c['H'], c['X'] = H, X
    c['pre'] = [linear(h, c['wm'], c['bm']) for h in H]
    c['qbar'] = [leaky_relu(pr, cfg.slope).mean(0) for pr in c['pre']]                 # :525, :529
    c['r'], c['u'], c['att'], c['Y'] = [None, None], [None, None], [None, None], [None, None]
    for i in range(2):                    # keypoints of side i use the OTHER side's mean-pooled query (:544, :555)
        qb = c['qbar'][1 - i]
        c['r'][i] = np.einsum('ked,d->ke', c['wq'], qb)                                # W_Q,k qbar
        c['u'][i] = np.einsum('ked,ke->kd', c['wk'], c['r'][i]) / math.sqrt(64)        # (K, 64)
        lg = c['u'][i] @ H[i].T                                                        # (K, n)
        lg = lg - lg.max(1, keepdims=True)
        e = np.exp(lg)
        c['att'][i] = e / e.sum(1, keepdims=True)
        c['Y'][i] = c['att'][i] @ X[i]
    y_l, y_r = c['Y']
    c['ym'] = [y_l.mean(0), y_r.mean(0)]
    A = (y_r - c['ym'][1]).T @ (y_l - c['ym'][0])                                      # :567
    U, S, Vt = np.linalg.svd(A)
    D = np.diag([1., 1., np.sign(np.linalg.det(A))])                                   # constant (:586)
    c.update(A=A, U=U, S=S, Vt=Vt, D=D)
    c['T'] = U @ D @ Vt
    c['b'] = c['ym'][1] - c['T'] @ c['ym'][0]
    return c


def svd_rotation_backward(U, S, Vt, D, gT):
    """dL/dA for T = U D Vt (D constant): torch's svd_backward with gU = gT V D, gV = gT^T U D, gS = 0:
    gA = U [ (skew(U^T gU) / E) S + S (skew(V^T gV) / E) ] V^T,  E_jk = S_k^2 - S_j^2 (1 on the diagonal), skew(X) = X - X^T.
    The guard's second condition (:574) bounds |E| from below."""
    V = Vt.T
    gU, gV = gT @ V @ D, gT.T @ U @ D
    s2 = S ** 2
    E = s2[None, :] - s2[:, None]
    np.fill_diagonal(E, 1.0)
    sk = lambda X: X - X.T
    inner = (sk(U.T @ gU) / E) * S[None, :] + S[:, None] * (sk(V.T @ gV) / E)
    return U @ inner @ Vt


def kabsch_bwd(c, x_lig_in, dcoors, dY_direct=(None, None), dT_direct=None, db_direct=None):
    """coords = T new_x + b (:665), b = ym_r - T ym_l (:589), T = U D Vt (:586-587), A = Yc_r^T Yc_l (:567)
    -> dY per side (ligand, receptor)."""
    T = c['T']
    dT = dcoors.T @ x_lig_in
    db = dcoors.sum(0)
    if dT_direct is not None:
        dT = dT + dT_direct
    if db_direct is not None:
        db = db + db_direct.reshape(3)
    dym_r = db.copy()
    dT = dT - np.outer(db, c['ym'][0])
    dym_l = -T.T @ db
    dA = svd_rotation_backward(c['U'], c['S'], c['Vt'], c['D'], dT)
    yc_l, yc_r = c['Y'][0] - c['ym'][0], c['Y'][1] - c['ym'][1]
    dyc_r, dyc_l = yc_l @ dA.T, yc_r @ dA
    K = yc_l.shape[0]
    dY_l = dyc_l - dyc_l.mean(0) + dym_l / K
    dY_r = dyc_r - dyc_r.mean(0) + dym_r / K
    if dY_direct[0] is not None:
        dY_l = dY_l + dY_direct[0]
    if dY_direct[1] is not None:
        dY_r = dY_r + dY_direct[1]
    return dY_l, dY_r


def keypoints_bwd(cfg, c, dY, G):
    """dY per side -> (dh per side, dx per side); accumulates head weight grads in G (keys: wm, bm, wk, wq)."""
    H, X = c['H'], c['X']
    dh = [np.zeros_like(H[0]), np.zeros_like(H[1])]
    dx = [None, None]
    dqbar = [np.zeros(64), np.zeros(64)]
    for i in range(2):
        att, Y = c['att'][i], c['Y'][i]
        dx[i] = att.T @ dY[i]
        datt = dY[i] @ X[i].T                                   # (K, n)
        dlog = att * (datt - (dY[i] * Y).sum(1, keepdims=True))
        dh[i] += dlog.T @ c['u'][i]
        du = dlog @ H[i]                                        # (K, 64)
        a = np.einsum('ked,kd->ke', c['wk'], du) / math.sqrt(64)
        G['wk'] += np.einsum('ke,kd->ked', c['r'][i], du) / math.sqrt(64)
        G['wq'] += np.einsum('ke,d->ked', a, c['qbar'][1 - i])
        dqbar[1 - i] += np.einsum('ked,ke->d', c['wq'], a)
    for i in range(2):
        n = H[i].shape[0]
        dpre = (dqbar[i] / n)[None, :] * np.where(c['pre'][i] > 0, 1.0, cfg.slope)
        G['wm'] += dpre.T @ H[i]
        G['bm'] += dpre.sum(0)
        dh[i] += dpre @ c['wm']
    return dh, dx


# ---- whole model ----------------------------------------------------------------------------------------------------

def full_backward(sd, cfg: OracleConfig, ligand, receptor, loss_grads, shared_layers: bool, stages=None):
    """Forward + manual backward for ONE pair.  ``loss_grads(out) -> (dcoors, dY_l, dY_r)`` given the forward outputs
    {'ligand_coors', 'keypts_ligand', 'keypts_receptor', ...}.  Returns ({state_dict name: gradient}, outputs)."""
    f = lambda a: np.asarray(a, np.float64)
    emb = f(sd['iegmn_original.residue_emb_layer.weight'])
    sides, idxs = [], []
    for s, ck in ((ligand, 'new_x'), (receptor, 'x')):
        idx = np.asarray(s['res_feat']).reshape(-1).astype(np.int64)
        idxs.append(idx)
        h0 = np.concatenate([emb[idx], np.log(f(s['mu_r_norm']))], 1)
        x0 = f(s[ck])
        sides.append({'x': x0, 'x_orig': x0, 'h': h0, 'h0': h0, 'he': f(s['he']),
                      'src': np.asarray(s['src']).astype(np.int64), 'dst': np.asarray(s['dst']).astype(np.int64)})
    params, all_caches = [], []
    for li in range(cfg.n_layers):
        p = LayerParams(sd, f'iegmn_original.iegmn_layers.{li}.', np.float64)
        caches = layer_forward(p, cfg, sides)
        for s, c in zip(sides, caches):
            s['x'], s['h'] = c['x_new'], c['h_new']
        params.append(p)
        all_caches.append(caches)
    hc = head_forward(sd, cfg, sides[0]['h'], sides[0]['x'], sides[1]['h'], sides[1]['x'])
    x_in = sides[0]['x_orig']
    out = {'ligand_coors': (hc['T'] @ x_in.T).T + hc['b'], 'keypts_ligand': hc['Y'][0], 'keypts_receptor': hc['Y'][1],
           'rotation': hc['T'], 'translation': hc['b'].reshape(1, 3)}
    dcoors, dYl, dYr = loss_grads(out)
    GH = {'wm': np.zeros((64, 64)), 'bm': np.zeros(64), 'wk': np.zeros_like(hc['wk']), 'wq': np.zeros_like(hc['wq'])}
    dY = kabsch_bwd(hc, x_in, dcoors, (dYl, dYr))
    dh, dx = keypoints_bwd(cfg, hc, dY, GH)
    if stages is not None:
        stages.append({'head': True, 'dY': dY, 'dh': dh, 'dx': dx})
    grads = {'iegmn_original.mlp_h_mean_ROT.0.weight': GH['wm'], 'iegmn_original.mlp_h_mean_ROT.0.bias': GH['bm'],
             'iegmn_original.att_mlp_key_ROT.0.weight': GH['wk'].reshape(-1, 64),
             'iegmn_original.att_mlp_query_ROT.0.weight': GH['wq'].reshape(-1, 64)}
    dh0 = [np.zeros_like(s['h0']) for s in sides]
    names = {'edge_w1': 'edge_mlp.0.weight', 'edge_b1': 'edge_mlp.0.bias', 'edge_ln_g': 'edge_mlp.3.weight',
             'edge_ln_b': 'edge_mlp.3.bias', 'edge_w2': 'edge_mlp.4.weight', 'edge_b2': 'edge_mlp.4.bias',
             'wq': 'att_mlp_Q.0.weight', 'wk': 'att_mlp_K.0.weight', 'wv': 'att_mlp_V.0.weight',
             'node_w1': 'node_mlp.0.weight', 'node_b1': 'node_mlp.0.bias', 'node_ln_g': 'node_mlp.3.weight',
             'node_ln_b': 'node_mlp.3.bias', 'node_w2': 'node_mlp.4.weight', 'node_b2': 'node_mlp.4.bias',
             'coor_w1': 'coors_mlp.0.weight', 'coor_b1': 'coors_mlp.0.bias', 'coor_w2': 'coors_mlp.4.weight',
             'coor_b2': 'coors_mlp.4.bias'}
    layer_G = {}
    for li in reversed(range(cfg.n_layers)):
        key = 1 if (shared_layers and li >= 1) else li               # shared layers accumulate into one buffer
        G = layer_G.setdefault(key, zero_layer_grads(params[li]))
        st = [] if stages is not None else None
        res = layer_backward(params[li], cfg, all_caches[li], dh, dx, G, st)
        dh, dx = [r[0] for r in res], [r[1] for r in res]
        for i in range(2):
            dh0[i] += res[i][2]
        if stages is not None:
            stages.append({'layer': li, 'sides': st})
    for i in range(2):
        dh0[i] += dh[i]                                              # layer 0's input h IS h0
    demb = np.zeros_like(emb)
    for i in range(2):
        np.add.at(demb, idxs[i], dh0[i][:, :64])
    grads['iegmn_original.residue_emb_layer.weight'] = demb
    for li in range(cfg.n_layers):
        key = 1 if (shared_layers and li >= 1) else li
        for short, nm in names.items():
            grads[f'iegmn_original.iegmn_layers.{li}.{nm}'] = layer_G[key][short]
    return grads, out
