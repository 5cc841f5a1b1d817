"""TEST INFRASTRUCTURE -- numpy fp64 restatement of the reference's TRAINING LOSSES (SURVEY 8f rank 1; groundwork for
the on-device losses of configs 3-4, not part of the forward hot path).  Cites /root/reference/src/train.py and
/root/reference/src/utils/ot_utils.py.

Pinning: ``sq_dist_mat`` / ``ot_emd`` are checked against the reference's own ``ot_utils`` functions where
``/root/reference`` is mounted (tests/test_loss_oracle.py).  The reference solves the transport LP with POT 0.7.0
``ot.emd`` (network simplex, requirements.txt:7), which is NOT in this image: **the EMD value is therefore parity
unpinned against POT itself**; it is pinned through LP duality instead -- ``ot_emd`` returns a dual certificate and the
test asserts primal feasibility, dual feasibility and a zero duality gap, which characterises THE optimal value any
exact solver (POT included) must return.  ``G_fn`` / ``body_intersection_loss`` live in src/train.py, whose import runs
argparse and file-system side effects (train.py:22-24); they are restated from the source lines cited.
"""
from __future__ import annotations

import numpy as np


def sq_dist_mat(x1, x2):
    """ot_utils.py:5-19: [n, m] squared l2 distances between two point clouds."""
    x1, x2 = np.asarray(x1, np.float64), np.asarray(x2, np.float64)
    return ((x1[:, None, :] - x2[None, :, :]) ** 2).sum(2)


def ot_emd(cost):
    """ot_utils.py:22-29: exact optimal transport between uniform marginals 1/n, 1/m with cost matrix ``cost``.
    Returns (ot_dist, plan, (u, v)): the optimal value sum(plan * cost), an optimal plan and dual potentials with
    u_i + v_j <= cost_ij (a certificate: sum(u)/n + sum(v)/m == ot_dist).  Solved as the transport LP with HiGHS."""
    import scipy.sparse as sp
    from scipy.optimize import linprog
    cost = np.asarray(cost, np.float64)
    n, m = cost.shape
    a, b = np.full(n, 1.0 / n), np.full(m, 1.0 / m)
    # row i sums x[i, :], row n + j sums x[:, j]; sparse: the dense matrix is 440 MB at n = 1024, m = 50
    A = sp.vstack([sp.kron(sp.eye(n), np.ones((1, m))), sp.kron(np.ones((1, n)), sp.eye(m))], format='csr')
    res = linprog(cost.reshape(-1), A_eq=A, b_eq=np.concatenate([a, b]), bounds=(0, None), method='highs')
    assert res.status == 0, res.message
    plan = res.x.reshape(n, m)
    duals = np.asarray(res.eqlin.marginals, np.float64)
    return float((plan * cost).sum()), plan, (duals[:n], duals[n:])


def ot_certify(cost, x):
    """Optimality certificate of an INTEGER transport plan ``x`` (n, m) between uniform marginals in units of 1/(n m)
    (the device solver's output): asserts that every row sums to m, every column to n, x >= 0, and that the residual
    graph has no negative cycle, which holds iff the plan is optimal.  Independent of any LP solver.
    A residual cycle alternates sinks and sources: sink k -> (backward arc, x_ik > 0) source i -> (forward arc) sink k',
    length C_ik' - C_ik.  Contracting the sources leaves the m-node graph W[k][k'] = min over i with x_ik > 0 of
    (C_ik' - C_ik); Floyd-Warshall on W must leave no negative diagonal entry.  Every arc of W gets a slack
    tau = 1e-9 max|C| / m first: tied costs make many cycles of length exactly 0, and without the slack Floyd-Warshall
    would go round them, doubling their rounding error at every pivot.  So the certificate is: no residual cycle is
    shorter than -1e-9 max|C| (rounding of the costs themselves).  Returns min over cycles of (length + arcs * tau),
    clipped at 0 (the empty cycle)."""
    cost, x = np.asarray(cost, np.float64), np.asarray(x)
    n, m = cost.shape
    assert x.shape == (n, m), (x.shape, cost.shape)
    assert np.issubdtype(x.dtype, np.integer), x.dtype
    assert (x >= 0).all(), 'negative flow'
    assert (x.sum(1) == m).all(), ('row sums', np.flatnonzero(x.sum(1) != m)[:8])
    assert (x.sum(0) == n).all(), ('column sums', np.flatnonzero(x.sum(0) != n)[:8])
    W = np.full((m, m), np.inf)
    for k in range(m):
        feeders = np.flatnonzero(x[:, k] > 0)
        if feeders.size:
            W[k] = (cost[feeders] - cost[feeders, k][:, None]).min(0)
    W += 1e-9 * float(np.abs(cost).max()) / m
    np.fill_diagonal(W, 0.0)
    for k in range(m):
        W = np.minimum(W, W[:, k:k + 1] + W[k:k + 1, :])
    worst = float(np.diag(W).min())
    assert worst >= 0.0, f'negative residual cycle: {worst:.6g}'
    return worst


def G_fn(protein_coords, x, sigma):
    """train.py:41-44: G(x) = -sigma * log(1e-3 + sum_i exp(-||x - a_i||^2 / sigma)); protein_coords (n,3), x (m,3) -> (m,)."""
    e = np.exp(-sq_dist_mat(x, protein_coords) / float(sigma))
    return -sigma * np.log(1e-3 + e.sum(1))


def body_intersection_loss(ligand_coors, receptor_coors, sigma, surface_ct):
    """train.py:46-49: mean_j max(0, ct - G_rec(ligand_j)) + mean_i max(0, ct - G_lig(receptor_i))."""
    return float(np.clip(surface_ct - G_fn(receptor_coors, ligand_coors, sigma), 0, None).mean()
                 + np.clip(surface_ct - G_fn(ligand_coors, receptor_coors, sigma), 0, None).mean())


def batch_loss(pred_ligand_coors, bound_ligand_coors, bound_receptor_coors, keypts_ligand, keypts_receptor,
               pocket_ligand, pocket_receptor, pocket_ot_loss_weight=1.0, intersection_loss_weight=10.0,
               intersection_sigma=25.0, intersection_surface_ct=10.0):
    """train.py:104-150 for lists over the pairs of a batch: per-pair MSE of the predicted ligand coordinates (nn.MSELoss
    mean over all 3 n_i entries, :114), the OT loss on cost_ligand + cost_receptor between pocket points and keypoints
    (:125-129), the body-intersection loss (:131-133); each averaged over the pairs (:143-146) and combined with the
    weights of args.py:64-70 (:150).  Returns (loss, parts)."""
    B = len(pred_ligand_coors)
    mse = ot = inter = 0.0
    for i in range(B):
        p = np.asarray(pred_ligand_coors[i], np.float64)
        mse += ((p - np.asarray(bound_ligand_coors[i], np.float64)) ** 2).mean()
        c = sq_dist_mat(pocket_ligand[i], keypts_ligand[i]) + sq_dist_mat(pocket_receptor[i], keypts_receptor[i])
        ot += ot_emd(c)[0]
        inter += body_intersection_loss(p, bound_receptor_coors[i], intersection_sigma, intersection_surface_ct)
    mse, ot, inter = mse / B, ot / B, inter / B
    return mse + pocket_ot_loss_weight * ot + intersection_loss_weight * inter, {'mse': mse, 'ot': ot, 'intersection': inter}
