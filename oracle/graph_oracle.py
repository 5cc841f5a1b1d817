"""TEST INFRASTRUCTURE -- numpy (fp64) restatement of the reference's residue-graph construction
(/root/reference/src/utils/protein_utils.py:212-397 ``protein_to_graph_unbound_bound_residuesonly`` with
``residue_loc_is_alphaC=True``, ``one_hot=False``; ``distance_list_featurizer`` :71-86), working on plain arrays instead of
biopandas data frames.  It is the checker of the GPU graph builder (csrc/graph_build.cu, SURVEY 8f rank 2) and the way the
compact all-atom fixtures of ALL 125 shipped test pairs (tests/golden/*_all.npz) are turned back into model inputs on the
GPU box, where neither the reference nor biopandas exist.

Pinned: ``oracle/make_golden_all.py`` runs the reference's own, unmodified preprocessing on every shipped test pair and
asserts that this restatement reproduces its graphs (identical edge lists; ``he`` / ``mu_r_norm`` / ``x`` to fp32 rounding),
recording the worst deviations in tests/golden/summary_all.json; tests/test_graph_oracle.py re-checks the nine full-graph
fixtures on every run.

Compact protein format (``protein`` dict):
  atoms      (A, 3) f32   all atom coordinates, residue by residue (the reference's per-residue ``df[['x','y','z']]``)
  atom_ptr   (N+1,) i32   residue r owns atoms[atom_ptr[r]:atom_ptr[r+1]]
  nca_c      (N, 3, 3) f32   N, CA, C atom coordinates of every residue
  res_feat   (N, 1) f32   residue-type index (residue_type_one_hot_dips_not_one_hot)
  bound_ca   (N, 3) f32   bound-structure C-alpha coordinates the unbound structure is aligned to (= CA at inference)
"""
from __future__ import annotations

import numpy as np

SIGMAS = [1.5 ** x for x in range(15)]      # protein_utils.py:72
MU_SIGMAS = np.array([1., 2., 5., 10., 30.])  # protein_utils.py:349


def kabsch(A, B):
    """rigid_transform_Kabsch_3D (protein_utils.py:31-64); A, B are 3 x N."""
    ca, cb = A.mean(1, keepdims=True), B.mean(1, keepdims=True)
    H = (A - ca) @ (B - cb).T
    U, _, Vt = np.linalg.svd(H)
    R = Vt.T @ U.T
    if np.linalg.det(R) < 0:
        R = (Vt.T @ np.diag([1., 1., -1.])) @ U.T
    return R, -R @ ca + cb


def local_frames(nca_c):
    """n_i, u_i, v_i of every residue (protein_utils.py:245-249), fp32 inputs -> fp32 arithmetic like the reference."""
    n_loc, ca, c_loc = (nca_c[:, k].astype(np.float32) for k in range(3))
    u = (n_loc - ca) / np.linalg.norm(n_loc - ca, axis=1, keepdims=True)
    t = (c_loc - ca) / np.linalg.norm(c_loc - ca, axis=1, keepdims=True)
    n = np.cross(u, t)
    n = n / np.linalg.norm(n, axis=1, keepdims=True)
    v = np.cross(n, u)
    return n, u, v


def residue_distance_matrix(atoms, atom_ptr):
    """Mean over all atom pairs of the inter-atomic distance (protein_utils.py:324-329), fp64, inf on the diagonal."""
    N = len(atom_ptr) - 1
    a = atoms.astype(np.float64)
    D = np.full((N, N), np.inf)
    # one big pairwise-distance matrix, then block means (same arithmetic as cdist + mean per block, different order)
    d = np.sqrt(((a[:, None, :] - a[None, :, :]) ** 2).sum(-1)) if a.shape[0] <= 6000 else None
    for i in range(N - 1):
        ai = slice(atom_ptr[i], atom_ptr[i + 1])
        for j in range(i + 1, N):
            aj = slice(atom_ptr[j], atom_ptr[j + 1])
            if d is not None:
                m = d[ai, aj].mean()
            else:
                m = np.sqrt(((a[ai][:, None, :] - a[aj][None, :, :]) ** 2).sum(-1)).mean()
            D[i, j] = D[j, i] = m
    return D


def residue_distance_matrix_fast(atoms, atom_ptr):
    """Same values through one dense (A, A) distance matrix reduced by residue blocks (reduceat) -- seconds instead of
    minutes for a 2000-residue protein."""
    a = atoms.astype(np.float64)
    N = len(atom_ptr) - 1
    A = a.shape[0]
    cnt = np.diff(atom_ptr).astype(np.float64)
    out = np.zeros((N, N))
    step = max(1, int(4e7 // max(A, 1)))
    starts = np.asarray(atom_ptr[:-1], dtype=np.int64)
    for r0 in range(0, A, step):
        blk = np.sqrt(((a[r0:r0 + step, None, :] - a[None, :, :]) ** 2).sum(-1))         # (step, A)
        colsum = np.add.reduceat(blk, starts, axis=1)                                     # (step, N)
        # accumulate rows of this block into their residues
        rid = np.searchsorted(atom_ptr, np.arange(r0, min(A, r0 + step)), side='right') - 1
        np.add.at(out, rid, colsum)
    D = out / (cnt[:, None] * cnt[None, :])
    D = 0.5 * (D + D.T)
    np.fill_diagonal(D, np.inf)
    return D


def residue_distance_rows(atoms, atom_ptr, rows):
    """Rows ``rows`` of the residue distance matrix, (len(rows), N) fp64 with inf at each row's own residue: that residue's
    atoms against all atoms, O(rows x A) -- for proteins too large for the dense (A, A) matrix."""
    a = atoms.astype(np.float64)
    atom_ptr = np.asarray(atom_ptr, np.int64)
    cnt = np.diff(atom_ptr).astype(np.float64)
    out = np.empty((len(rows), len(atom_ptr) - 1))
    for k, i in enumerate(rows):
        blk = np.sqrt(((a[atom_ptr[i]:atom_ptr[i + 1], None, :] - a[None, :, :]) ** 2).sum(-1))   # (atoms of i, A)
        out[k] = np.add.reduceat(blk.sum(0), atom_ptr[:-1]) / (cnt[i] * cnt)
        out[k, i] = np.inf
    return out


def _align(protein, kabsch64):
    """x (N,3) and the rotated local frames n, u, v of one protein after the unbound->bound alignment (:279-308)."""
    nca_c = np.asarray(protein['nca_c'], np.float32)
    n_f, u_f, v_f = local_frames(nca_c)
    x = nca_c[:, 1].astype(np.float32)                                  # residue_loc_is_alphaC (:255-256)
    bound = np.asarray(protein['bound_ca'], np.float32)
    if kabsch64:                  # fp64 fit, x and frames rotated in fp64 (the device's arithmetic)
        x, bound = x.astype(np.float64), bound.astype(np.float64)
    R, t = kabsch(x.T, bound.T)                                         # (:284-285)
    x = ((R @ x.T) + t).T                                               # (:286-291)
    return x, ((R @ n_f.T).T, (R @ u_f.T).T, (R @ v_f.T).T)


def _graph_rows(D, rows, x, frames, cutoff, max_neighbor):
    """compute_dig_kNN_graph (protein_utils.py:311-397) for destination rows ``rows``, D[k] = distance row of rows[k]."""
    n_f, u_f, v_f = frames
    src, dst, dist, mu = [], [], [], []
    for k, i in enumerate(rows):
        valid = list(np.where(D[k, :] < cutoff)[0])                     # (:340)
        if len(valid) > max_neighbor:
            valid = list(np.argsort(D[k, :], kind='stable'))[0:max_neighbor]            # (:342-343)
        dst += [i] * len(valid)
        src += valid
        dv = D[k, valid]
        dist += list(dv)
        if not valid:             # degree 0: the reference's w.max raises on the empty row; the device writes 0
            mu.append(np.zeros(len(MU_SIGMAS)))
            continue
        w = -dv.reshape(1, -1) ** 2 / MU_SIGMAS.reshape(-1, 1)          # softmax over the neighbours (:349-351)
        w = np.exp(w - w.max(axis=1, keepdims=True))
        w = w / w.sum(axis=1, keepdims=True)
        diff = x[[i] * len(valid), :] - x[valid, :]
        mean_vec = w.dot(diff)
        den = w.dot(np.linalg.norm(diff, axis=1))
        mu.append(np.linalg.norm(mean_vec, axis=1) / den)                # (:352-356)
    src, dst, dist = np.asarray(src, np.int64), np.asarray(dst, np.int64), np.asarray(dist, np.float64)
    rbf = np.exp(-(dist[:, None] ** 2) / np.asarray(SIGMAS)[None, :]).astype(np.float32)      # (:71-86)
    basis = np.stack([n_f[dst], u_f[dst], v_f[dst]], axis=1)            # (E, 3, 3): rows n, u, v of the destination (:378)
    mm = lambda vec: np.einsum('erc,ec->er', basis, vec)
    ori = np.concatenate([mm(x[src] - x[dst]), mm(n_f[src]), mm(u_f[src]), mm(v_f[src])], axis=1).astype(np.float32)   # (:379-384)
    return {'src': src.astype(np.int32), 'dst': dst.astype(np.int32), 'he': np.concatenate([rbf, ori], axis=1).reshape(-1, 27),
            'mu_r_norm': np.asarray(mu).astype(np.float32).reshape(-1, 5), 'dist': dist}


def build_graph(protein, cutoff=30.0, max_neighbor=10, fast=True, kabsch64=False):
    """-> dict(src, dst int32 (edges grouped by destination), he (E,27) f32, x (N,3) f32, mu_r_norm (N,5) f32,
    res_feat (N,1) f32) for ONE protein: compute_dig_kNN_graph (protein_utils.py:311-397) after the unbound->bound
    alignment (:279-308).

    ``kabsch64=False`` aligns in fp32 like the reference (fp32 x and bound_ca into the SVD; R, t, x stay fp32, ~1e-7 |x|
    from an fp64 fit); ``True`` fits and rotates x and the frames in fp64, the device's arithmetic.
    Among more than ``max_neighbor`` residues inside the cutoff the closest are taken by a STABLE argsort: ascending
    distance, exact ties by ascending index, the device's rule.  The reference's default argsort is not stable, so under
    exact ties its order depends on the platform; without ties both are the same.
    A residue with no neighbour inside the cutoff gets mu_r_norm = 0 (the reference raises on it)."""
    atom_ptr = np.asarray(protein['atom_ptr'], np.int64)
    N = atom_ptr.shape[0] - 1
    x, frames = _align(protein, kabsch64)
    D = (residue_distance_matrix_fast if fast else residue_distance_matrix)(np.asarray(protein['atoms'], np.float32), atom_ptr)
    g = _graph_rows(D, range(N), x, frames, cutoff, max_neighbor)
    g.update(x=x.astype(np.float32), res_feat=np.asarray(protein['res_feat'], np.float32).reshape(-1, 1))
    return g


def build_rows(protein, rows, cutoff=30.0, max_neighbor=10, kabsch64=False):
    """``build_graph`` restricted to the destination residues ``rows`` (edges of each row in the order given; x and
    mu_r_norm of those rows only), with distances computed per row (``residue_distance_rows``): the check of proteins of
    thousands of residues."""
    rows = [int(i) for i in rows]
    x, frames = _align(protein, kabsch64)
    D = residue_distance_rows(np.asarray(protein['atoms'], np.float32), protein['atom_ptr'], rows)
    g = _graph_rows(D, rows, x, frames, cutoff, max_neighbor)
    g['x'] = x[rows].astype(np.float32)
    return g


def build_pair(ligand, receptor, cutoff=30.0, max_neighbor=10):
    """(ligand protein, receptor protein) -> the (lig_dict, rec_dict) input format of the engine / oracle
    (ligand gets new_x = x, inference_rigid.py:186)."""
    gl, gr = build_graph(ligand, cutoff, max_neighbor), build_graph(receptor, cutoff, max_neighbor)
    gl['new_x'] = gl['x'].copy()
    for g in (gl, gr):
        g.pop('dist')
    return gl, gr
