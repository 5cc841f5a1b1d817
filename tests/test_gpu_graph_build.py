"""GPU (H100): the on-device residue k-NN graph builder (csrc/graph_build.cu, through ``build_graphs`` and the C ABI)
against the fp64 graph oracle (oracle/graph_oracle.py, ``kabsch64=True``, stable tie order) on the SAME fp32 inputs, at
the edges of the kernel: real unbound->bound alignments, rigid motions of the bound trace, rank-deficient alignments
(1-3 residues, exactly collinear and coplanar traces), both neighbour-selection rules at their switch, distances exactly
at the cutoff, exact distance ties, residues above the 64 atoms the kernel caches in shared memory, proteins of 3000 to
12 800 residues (past the 48 KB dynamic shared-memory default, up to the 200 KiB row limit), far coordinates, a 256-pair
ragged batch rebuilt three ways, and the ABI's argument checks.  Also the RMSD meter (csrc/head.cu) on rank-deficient
point sets, which shares the 3x3 SVD (svd3.cuh) with the aligner.

Tolerances (per protein, per row):
  edge lists   identical; only where the oracle's distances at the K-th / (K+1)-th boundary, or |D - cutoff|, are within
               1e-12 relative (the device and the oracle sum the all-atom distances in different orders) is either choice
               accepted.  Exact ties and the exact-cutoff cases get no allowance.
  RBFs         <= 2 fp32 ulps of the oracle value
  mu_r_norm    <= 2 fp32 ulps of the oracle value + 1e-12 (fp64 cancellation in |sum_j w_j (x_i - x_j)|)
  x            <= 2 fp32 ulps of the row's max |x| + 1e-12 max |x| (fp64 rounding of R (ca - c) + c', for rows at the origin)
  he[18:27]    <= 1e-6 (frames are fp32 on both sides; the device may contract to FMA)
  p_ij         <= 1e-6 (1 + |x_src - x_dst|)
Largest errors measured over the whole file on an H100 80GB HBM3 (400 W power limit), printed by each test with -s:
RBFs 0 ulp, mu_r_norm 0 ulp, x 0 ulp (x of a rigidly moved bound trace vs R ca + t: 0.58 ulp), he[18:27] 4.5e-7,
p_ij 3.4e-7 (1 + |x_src - x_dst|), RMSD meter 5.2e-15 relative; no row needed the near-tie allowance.  The file runs in
about 17 s there.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import golden_io as gio
import graph_oracle as go
from equidock_public_b200 import _native as nat
from equidock_public_b200.graph_build import GraphBuffers, ResidueBatch, build_graphs, rebuild_in_place
from equidock_public_b200.hetero_graph import LIGAND, RECEPTOR

pytestmark = pytest.mark.gpu

f32, f64 = np.float32, np.float64
_WORST = {}


def _note(key, v):
    _WORST[key] = max(_WORST.get(key, 0.0), float(v))


# ---- inputs ------------------------------------------------------------------------------------------------------------

def _protein(ca, rng, n_atoms=None, spread=1.5):
    """Compact protein around C-alpha positions ``ca``: one atom per residue (the C-alpha itself, so that residue distances
    are exact) or ``n_atoms[r]`` atoms (the C-alpha plus a normal blob); N and C atoms in random directions."""
    ca = np.asarray(ca, f32)
    N = ca.shape[0]
    cnt = np.ones(N, np.int64) if n_atoms is None else np.asarray(n_atoms, np.int64)
    ptr = np.zeros(N + 1, np.int32)
    ptr[1:] = np.cumsum(cnt)
    atoms = np.repeat(ca, cnt, axis=0)
    extra = np.ones(ptr[-1], bool)
    extra[ptr[:-1]] = False
    atoms[extra] += rng.normal(0, spread, (int(extra.sum()), 3))
    d = rng.normal(size=(N, 2, 3))
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    nca_c = np.stack([ca + 1.46 * d[:, 0], ca, ca + 1.52 * d[:, 1]], axis=1)
    return {'atoms': atoms.astype(f32), 'atom_ptr': ptr, 'nca_c': nca_c.astype(f32), 'res_feat': np.zeros((N, 1), f32),
            'bound_ca': ca.copy()}


def _chain(rng, n, step=3.8):
    """Random-walk C-alpha trace."""
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return np.cumsum(step * d, axis=0)


def _rigid(rng, scale=30.0):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q)), rng.normal(0, scale, 3)


def _moved(p, R, t, offset=0.0):
    """Same protein with the bound trace R ca + t (rounded to fp32), and every coordinate shifted by ``offset``."""
    q = dict(p)
    q['bound_ca'] = ((R @ p['nca_c'][:, 1].astype(f64).T).T + t + offset).astype(f32)
    if offset:
        q['atoms'] = (p['atoms'].astype(f64) + offset).astype(f32)
        q['nca_c'] = (p['nca_c'].astype(f64) + offset).astype(f32)
    return q


# ---- device build, split per protein ------------------------------------------------------------------------------------

def _split(g, rb):
    plan = g._eqd_plan
    row_ptr = plan.row_ptr.cpu().numpy().astype(np.int64)
    E = int(row_ptr[-1])
    col = plan.col_src[:E].cpu().numpy().astype(np.int64)
    he = plan.he_l[:E].cpu().numpy()
    x = torch.cat([g._ndata[LIGAND]['x'], g._ndata[RECEPTOR]['x']]).cpu().numpy()
    mu = torch.cat([g._ndata[LIGAND]['mu_r_norm'], g._ndata[RECEPTOR]['mu_r_norm']]).cpu().numpy()
    seg = rb.t['seg_ptr'].numpy().astype(np.int64)
    out = []
    for s in range(len(seg) - 1):
        n0, n1 = seg[s], seg[s + 1]
        e0, e1 = row_ptr[n0], row_ptr[n1]
        out.append({'row_ptr': row_ptr[n0:n1 + 1] - e0, 'src': col[e0:e1] - n0, 'he': he[e0:e1], 'x': x[n0:n1], 'mu': mu[n0:n1]})
    return out


def _build(prots, dev, cutoff=30.0, K=10):
    """build_graphs over proteins in this order (pairs = first half x second half; odd counts get a 1-residue filler)."""
    prots = list(prots)
    if len(prots) % 2:
        prots.append(_protein(np.zeros((1, 3)), np.random.default_rng(0)))
    h = len(prots) // 2
    rb = ResidueBatch(list(zip(prots[:h], prots[h:])))
    g = build_graphs(rb, dev, cutoff=cutoff, max_neighbor=K)
    return _split(g, rb)


# ---- comparison ----------------------------------------------------------------------------------------------------------

def _near_tie_ok(nb, D, cutoff, K, rel=1e-12):
    """Whether ``nb`` is what one of the two selection rules returns for distances within ``rel`` of the oracle's row D."""
    nb = np.asarray(nb, np.int64)
    tol = rel * cutoff
    sure = set(np.nonzero(D < cutoff - tol)[0].tolist())
    maybe = set(np.nonzero(np.abs(D - cutoff) <= tol)[0].tolist())
    if len(set(nb.tolist())) != nb.size or (nb.size and not (D[nb] < cutoff + tol).all()):
        return False
    if nb.size <= K and (np.diff(nb) > 0).all() and sure <= set(nb.tolist()) <= sure | maybe:
        return True                                  # every residue inside the cutoff, ascending index
    if nb.size == K and len(sure | maybe) > K:       # the K closest, ascending distance
        d = D[nb]
        rest = np.asarray(sorted(sure - set(nb.tolist())), np.int64)
        return bool((np.diff(d) >= -rel * d[1:]).all() and (rest.size == 0 or D[rest].min() >= d.max() * (1 - rel)))
    return False


def _compare(dev, p, cutoff, K, rows=None, ties=True, what=''):
    """One protein: device output ``dev`` against build_rows(kabsch64) on ``rows`` (default all)."""
    N = p['nca_c'].shape[0]
    rows = np.arange(N) if rows is None else np.asarray(rows, np.int64)
    ref = go.build_rows(p, rows, f32(cutoff), K, kabsch64=True)
    off_ref = np.concatenate([[0], np.cumsum(np.bincount(np.searchsorted(rows, ref['dst']), minlength=rows.size))])
    rp = dev['row_ptr']
    e_dev, e_ref, near = [], [], 0
    for k, i in enumerate(rows):
        a = dev['src'][rp[i]:rp[i + 1]]
        b = ref['src'][off_ref[k]:off_ref[k + 1]]
        if np.array_equal(a, b):
            e_dev.append(np.arange(rp[i], rp[i + 1]))
            e_ref.append(np.arange(off_ref[k], off_ref[k + 1]))
            continue
        D = go.residue_distance_rows(p['atoms'], p['atom_ptr'], [i])[0]
        assert ties and _near_tie_ok(a, D, float(f32(cutoff)), K), \
            f'{what} row {i}: device {a.tolist()} oracle {b.tolist()} (oracle d {D[b].tolist()}, device d {D[a].tolist()})'
        near += 1
    _note('near-tie rows', near)
    ed, er = np.concatenate(e_dev + [np.zeros(0, np.int64)]), np.concatenate(e_ref + [np.zeros(0, np.int64)])
    hd, hr = dev['he'][ed].astype(f64), ref['he'][er]
    ulp = lambda v: np.spacing(np.abs(v).astype(f32)).astype(f64)
    if ed.size:
        r = (np.abs(hd[:, :15] - hr[:, :15]) / ulp(hr[:, :15])).max()
        _note('rbf ulp', r)
        assert r <= 2, (what, r)
        fr = np.abs(hd[:, 18:] - hr[:, 18:]).max()
        _note('frames abs', fr)
        assert fr <= 1e-6, (what, fr)
        dist = np.linalg.norm(dev['x'][ref['src'][er]].astype(f64) - dev['x'][ref['dst'][er]], axis=1)
        pe =(np.abs(hd[:, 15:18] - hr[:, 15:18]).max(1) / (1 + dist)).max()
        _note('p_ij / (1+|d|)', pe)
        assert pe <= 1e-6, (what, pe)
    mu_d, mu_r = dev['mu'][rows].astype(f64), ref['mu_r_norm'].astype(f64)
    mr = ((np.abs(mu_d - mu_r) - 1e-12).clip(0) / ulp(mu_r)).max()
    _note('mu ulp', mr)
    assert mr <= 2, (what, mr)
    xr = ref['x'].astype(f64)
    xe = (np.abs(dev['x'][rows].astype(f64) - xr) - 1e-12 * np.abs(xr).max()).clip(0)
    xu = (xe / ulp(np.abs(xr).max(1, keepdims=True))).max()
    _note('x ulp', xu)
    assert xu <= 2, (what, xu)


def _report(name):
    print(f'\n[{name}] ' + ', '.join(f'{k} {v:.3g}' for k, v in sorted(_WORST.items())))


# ---- 1. real alignment ---------------------------------------------------------------------------------------------------

REAL = {'db5': ['1QA9', '1NW9', '3SZK', '5JMO', '1N2C'],
        'dips': ['dm_5dm7.pdb1_22.dill', 'p7_2p7v.pdb1_0.dill', 'aq_4aqa.pdb1_0.dill', 'hm_4hm1.pdb1_0.dill',
                 'b2_1b26.pdb1_3.dill', 'a9_1a9x.pdb4_0.dill', 'ww_2ww2.pdb1_2.dill']}


def _sample_rows(N, rng, n=256):
    if N <= n:
        return np.arange(N)
    base = {0, N - 1} | {v for m in range(128, N, 128) for v in (m - 1, m + 1)}
    base = sorted(v for v in base if 0 <= v < N)[:n // 2]
    return np.unique(np.concatenate([base, rng.choice(N, n - len(base), replace=False)]))


def _real_aligned():
    prots = []
    for ds, names in REAL.items():
        _, allp = gio.load_all(ds)
        for n in names:
            e = allp[n]
            for side, key in (('lig', 'ligand_gt'), ('rec', 'receptor_gt')):
                p = dict(e[side])
                assert p['nca_c'].shape[0] == e['ca'][key].shape[0], (n, side)
                p['bound_ca'] = np.asarray(e['ca'][key], f32)
                prots.append((f'{n}/{side}', p))
    return prots


def test_real_unbound_to_bound_alignment(cuda_device):
    """Shipped pairs aligned to their bound C-alpha traces (ligands 31-244 A away): R is far from I."""
    rng = np.random.default_rng(0)
    prots = _real_aligned()
    dev = _build([p for _, p in prots], cuda_device)
    for (name, p), d in zip(prots, dev):
        _compare(d, p, 30.0, 10, rows=_sample_rows(p['nca_c'].shape[0], rng, 400), what=name)
    _report('real alignment')


# ---- 2. rigid invariance -------------------------------------------------------------------------------------------------

def test_rigid_motion_of_the_bound_trace(cuda_device):
    _, allp = gio.load_all('dips')
    rng = np.random.default_rng(1)
    base = [allp[n][s] for n in REAL['dips'][:3] for s in ('lig', 'rec')]
    motions = [_rigid(rng, 50.0) for _ in base]
    moved = [_moved(p, R, t) for p, (R, t) in zip(base, motions)]
    dev = _build(base + moved, cuda_device)
    worst = 0.0
    for k, (p, (R, t)) in enumerate(zip(base, motions)):
        a, b = dev[k], dev[len(base) + k]
        want = (R @ p['nca_c'][:, 1].astype(f64).T).T + t
        u = (np.abs(b['x'] - want) / np.spacing(np.abs(want).max(1, keepdims=True).astype(f32))).max()
        worst = max(worst, u)
        assert u <= 4, u
        assert np.array_equal(a['row_ptr'], b['row_ptr']) and np.array_equal(a['src'], b['src'])
        assert np.array_equal(a['he'][:, :15], b['he'][:, :15])              # distances do not depend on the alignment
        d = np.linalg.norm(want[a['src']] - want[np.repeat(np.arange(len(want)), np.diff(a['row_ptr']))], axis=1)
        assert (np.abs(a['he'][:, 15:18] - b['he'][:, 15:18]).max(1) <= 1e-6 * (1 + d)).all()
        assert np.abs(a['he'][:, 18:] - b['he'][:, 18:]).max() <= 1e-6
        assert (np.abs(a['mu'] - b['mu']) <= 2 * np.spacing(np.abs(a['mu'])) + 1e-12).all()
        _compare(b, moved[k], 30.0, 10, what=f'moved {k}')
    _note('x vs R ca + t ulp', worst)
    _report('rigid motion')


# ---- 3. rank-deficient alignment -----------------------------------------------------------------------------------------

def _degenerate_traces(rng):
    out = []
    for n in (1, 2, 3):
        out.append((f'{n} residues', rng.normal(0, 5, (n, 3))))
    for k in range(5):
        step = rng.integers(-3, 4, 3)
        step[k % 3] = step[k % 3] or 2
        out.append((f'collinear {k}', rng.integers(-40, 40, 3)[None] + np.arange(3 + 7 * k)[:, None] * step[None]))
    for k in range(3):
        P = rng.integers(-15, 15, (10 + 15 * k, 3)).astype(f64)
        P[:, 2] = 7.0
        out.append((f'coplanar z = 7 ({k})', P))
        P = rng.integers(-15, 15, (10 + 15 * k, 3)).astype(f64)
        P[:, 1] = P[:, 0]
        out.append((f'coplanar x = y ({k})', P))
    return out


def test_rank_deficient_alignment(cuda_device):
    """1-3 residues, exactly collinear and coplanar traces, bound = unbound and bound = a rigid motion.  R is not unique
    for collinear sets, but he, mu_r_norm and x are, so they are compared with the oracle as everywhere else."""
    rng = np.random.default_rng(2)
    prots, names = [], []
    for name, ca in _degenerate_traces(rng):
        p = _protein(ca, rng)
        prots += [p, _moved(p, *_rigid(rng, 40.0))]
        names += [name, name + ' moved']
    dev = _build(prots, cuda_device)
    for name, p, d in zip(names, prots, dev):
        _compare(d, p, 30.0, 10, ties=False, what=name)
    _report('rank-deficient alignment')


# ---- 4. selection paths --------------------------------------------------------------------------------------------------

def _star(rng, radii, blobs=(), at=None):
    """Residue 0 at the origin; single-atom residues at ``radii``, indexed by DESCENDING radius (so that index order and
    distance order differ; single atoms make centroid bounds and distances exact); two-atom residues centred at radii
    ``blobs`` (atoms 1 A either side of the centre along the radius: mean distance r, upper bound r + 1); and ``at``: one
    more residue exactly that far away along x."""
    radii = np.sort(np.asarray(radii, f64))[::-1]
    dirs = rng.normal(size=(len(radii) + len(blobs), 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    pos = [np.zeros(3)] + [dirs[k] * r for k, r in enumerate(radii)] + [dirs[len(radii) + k] * r for k, r in enumerate(blobs)]
    cnt = [1] * (1 + len(radii)) + [2] * len(blobs)
    if at is not None:
        pos.append(np.array([at, 0.0, 0.0]))
        cnt.append(1)
    p = _protein(np.asarray(pos), rng, n_atoms=cnt, spread=0.0)
    for k, r in enumerate(blobs):
        u = dirs[len(radii) + k]
        s = p['atom_ptr'][1 + len(radii) + k]
        p['atoms'][s], p['atoms'][s + 1] = (u * (r + 1)).astype(f32), (u * (r - 1)).astype(f32)
    return p


def _selection_cases(rng, K, cutoff):
    rad = lambda n: rng.uniform(2.0, cutoff - 1.5, n)            # certainly inside: upper bound = distance < cutoff
    cases = {
        'K certain': _star(rng, rad(K)),                                     # K valid: ascending index
        'K+1 certain': _star(rng, rad(K + 1)),                               # K+1: the K closest, ascending distance
        'K certain + 1 uncertain valid': _star(rng, rad(K), [cutoff - 0.7]),
        'K-1 certain + 1 uncertain valid': _star(rng, rad(K - 1), [cutoff - 0.7]),
        'K-1 inside + 1 at the cutoff': _star(rng, rad(K - 1), at=cutoff),  # d == cutoff is outside on both rules
        'K inside + 1 at the cutoff': _star(rng, rad(K), at=cutoff),
        'K+1 inside + 1 at the cutoff': _star(rng, rad(K + 1), at=cutoff),
    }
    for d in range(1, K):
        cases[f'degree {d}'] = _star(rng, rad(d))
    cases['isolated'] = _protein(np.array([[0, 0, 0], [1000, 0, 0], [0, 1000, 0], [0, 0, 3.0]]), rng)   # 1, 2: degree 0
    return cases


@pytest.mark.parametrize('K,cutoff', [(10, 8.0), (3, 6.0), (16, 12.0)])
def test_selection_rules_at_their_switch(K, cutoff, cuda_device):
    rng = np.random.default_rng(K)
    cases = _selection_cases(rng, K, cutoff)
    names = list(cases)
    dev = _build([cases[n] for n in names], cuda_device, cutoff, K)
    for n, d in zip(names, dev):
        _compare(d, cases[n], cutoff, K, ties=False, what=n)
    assert int(dev[names.index('isolated')]['row_ptr'][2] - dev[names.index('isolated')]['row_ptr'][1]) == 0
    assert (dev[names.index('isolated')]['mu'][1:3] == 0).all()
    _report(f'selection K={K}')


@pytest.mark.parametrize('K', [10, 16])
def test_tau_histogram_over_a_sweep_of_cutoffs(K, cuda_device):
    """Dense blobs of multi-atom residues, cutoffs swept so that the K-th upper bound falls into many of the 64 bins."""
    rng = np.random.default_rng(10 + K)
    prots = [_protein(rng.uniform(0, 22, (150, 3)), rng, n_atoms=rng.integers(1, 15, 150), spread=1.2) for _ in range(2)]
    for cutoff in np.linspace(5.0, 40.0, 9):
        dev = _build(prots, cuda_device, float(cutoff), K)
        for k, (p, d) in enumerate(zip(prots, dev)):
            _compare(d, p, float(cutoff), K, what=f'blob {k} cutoff {cutoff}')
    _report(f'tau sweep K={K}')


# ---- 5. parameters ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('K', [1, 2, 10, 15, 16])
def test_max_neighbor_and_cutoff_grid(K, cuda_device):
    _, allp = gio.load_all('dips')
    prots = [allp[n][s] for n in REAL['dips'][:2] for s in ('lig', 'rec')]
    for cutoff in (6.0, 7.3, 8.5, 30.0, 1e4):
        dev = _build(prots, cuda_device, cutoff, K)
        for k, (p, d) in enumerate(zip(prots, dev)):
            _compare(d, p, cutoff, K, what=f'{k} K={K} cutoff={cutoff}')
    _report(f'grid K={K}')


# ---- 6. exact ties -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('K,cutoff', [(10, 30.0), (10, 2.9), (16, 3.0), (1, 30.0)])
def test_exact_ties_on_a_lattice(K, cutoff, cuda_device):
    """7 x 7 x 7 single-atom residues 2 A apart: interior residues have 6 neighbours at 2 A and 12 at 2 sqrt(2) A, so the
    K-th neighbour is tied; ties go by ascending index, with no allowance."""
    rng = np.random.default_rng(6)
    g = np.stack(np.meshgrid(*[np.arange(7)] * 3, indexing='ij'), -1).reshape(-1, 3) * 2.0
    perm = rng.permutation(g.shape[0])            # index order unrelated to the geometry
    p = _protein(g[perm] + 5.0, rng)
    dev = _build([p], cuda_device, cutoff, K)
    _compare(dev[0], p, cutoff, K, ties=False, what='lattice')
    _report(f'lattice K={K} cutoff={cutoff}')


# ---- 7. residues above the shared-memory cache ---------------------------------------------------------------------------

def test_large_residues(cuda_device):
    rng = np.random.default_rng(7)
    N = 80
    cnt = rng.integers(1, 15, N)
    cnt[[0, 5, 6, 33, 34, 60, 79]] = [300, 65, 100, 64, 65, 100, 300]
    prots = [_protein(_chain(rng, N, 2.5), rng, n_atoms=cnt, spread=2.0) for _ in range(2)]
    dev = _build(prots, cuda_device, 30.0, 10)
    for k, (p, d) in enumerate(zip(prots, dev)):
        _compare(d, p, 30.0, 10, what=f'large residues {k}')
        dst = np.repeat(np.arange(N), np.diff(d['row_ptr']))
        edge = {(int(s), int(t)): e for e, (s, t) in enumerate(zip(d['src'], dst))}
        pairs = [(e, edge[(t, s)]) for (s, t), e in edge.items() if (t, s) in edge]
        assert len(pairs) > N
        a, b = zip(*pairs)
        assert np.array_equal(d['he'][list(a), :15], d['he'][list(b), :15])      # d(i,j) == d(j,i) bitwise
    _report('large residues')


# ---- 8. large proteins ---------------------------------------------------------------------------------------------------

def test_large_proteins_and_the_row_limit(cuda_device):
    """3000 / 3100 residues (either side of the 48 KB default dynamic shared memory at 16 B per residue) and 12 800 (the
    200 KiB limit) in one batch with small proteins, after a smaller build in the same process; 12 801 is refused."""
    rng = np.random.default_rng(8)
    _build([_protein(_chain(rng, 50), rng)], cuda_device)
    sizes = [5, 3000, 3100, 12800, 40, 1]
    prots = [_protein(_chain(rng, n), rng, n_atoms=rng.integers(1, 5, n), spread=1.0) for n in sizes]
    dev = _build(prots, cuda_device)
    for n, p, d in zip(sizes, prots, dev):
        _compare(d, p, 30.0, 10, rows=_sample_rows(n, rng), what=f'{n} residues')
    with pytest.raises(nat.NativeLibraryError, match='EQD_ERR_UNSUPPORTED'):
        _build([_protein(_chain(rng, 12801), rng), _protein(_chain(rng, 3), rng)], cuda_device)
    _report('large proteins')


# ---- 9. far coordinates --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('offset', [1e3, 1e4])
def test_far_coordinates(offset, cuda_device):
    _, allp = gio.load_all('dips')
    rng = np.random.default_rng(9)
    prots = [_moved(allp[n][s], *_rigid(rng, 20.0), offset=offset) for n in REAL['dips'][:2] for s in ('lig', 'rec')]
    dev = _build(prots, cuda_device)
    for k, (p, d) in enumerate(zip(prots, dev)):
        _compare(d, p, 30.0, 10, what=f'offset {offset} {k}')
    _report(f'offset {offset}')


# ---- 10. batch plumbing --------------------------------------------------------------------------------------------------

def test_ragged_batch_and_rebuilds_are_bitwise_identical(cuda_device):
    rng = np.random.default_rng(10)
    n = rng.integers(1, 401, 512)
    n[:4] = [1, 400, 2, 399]
    prots = [_protein(_chain(rng, k), rng, n_atoms=rng.integers(1, 9, k)) for k in n]
    rb = ResidueBatch(list(zip(prots[:256], prots[256:])))
    g1 = build_graphs(rb, cuda_device)
    split = _split(g1, rb)
    for s in [0, 1, 2, 3, 100, 255, 256, 300, 511]:
        _compare(split[s], prots[s], 30.0, 10, what=f'batch protein {s}')
    p1 = g1._eqd_plan
    E = int(p1.row_ptr[-1].item())
    ref = [p1.row_ptr.clone(), p1.col_src[:E].clone(), p1.he_l[:E].clone(),
           torch.cat([g1._ndata[LIGAND]['x'], g1._ndata[RECEPTOR]['x']]), torch.cat([g1._ndata[LIGAND]['mu_r_norm'], g1._ndata[RECEPTOR]['mu_r_norm']])]

    def same(row_ptr, col, he, x, mu, what):
        for a, b, nm in zip(ref, (row_ptr, col[:E], he[:E], x, mu), ('row_ptr', 'col_src', 'he', 'x', 'mu_r_norm')):
            assert torch.equal(a, b), (what, nm)

    g2 = build_graphs(rb, cuda_device, sync_sizes=False)
    p2 = g2._eqd_plan
    same(p2.row_ptr, p2.col_src, p2.he_l, torch.cat([g2._ndata[LIGAND]['x'], g2._ndata[RECEPTOR]['x']]),
         torch.cat([g2._ndata[LIGAND]['mu_r_norm'], g2._ndata[RECEPTOR]['mu_r_norm']]), 'sync_sizes=False')
    buf = GraphBuffers(rb, cuda_device)
    buf.upload(rb)
    rebuild_in_place(rb, buf)
    same(buf.row_ptr, buf.col_src, buf.he, buf.x, buf.mu, 'rebuild_in_place')
    g3 = build_graphs(rb, cuda_device)
    p3 = g3._eqd_plan
    same(p3.row_ptr, p3.col_src, p3.he_l, torch.cat([g3._ndata[LIGAND]['x'], g3._ndata[RECEPTOR]['x']]),
         torch.cat([g3._ndata[LIGAND]['mu_r_norm'], g3._ndata[RECEPTOR]['mu_r_norm']]), 'second build')
    _report('ragged batch')


# ---- 11. ABI -------------------------------------------------------------------------------------------------------------

def test_graph_build_abi_checks_return_before_any_launch(cuda_device):
    lib = nat.load()
    rng = np.random.default_rng(11)
    rb = ResidueBatch([(_protein(_chain(rng, 30), rng), _protein(_chain(rng, 20), rng))])
    d = {k: v.to(cuda_device) for k, v in rb.t.items()}
    N = rb.N
    ws_bytes = int(lib.eqd_graph_build_workspace_bytes(N))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=cuda_device)
    deg = torch.full((N,), -7, dtype=torch.int32, device=cuda_device)
    x = torch.full((N, 3), -7.0, device=cuda_device)
    mu = torch.full((N, 5), -7.0, device=cuda_device)
    st = C.c_void_p(torch.cuda.current_stream(cuda_device).cuda_stream)
    args = [nat.ptr(d[k]) for k in ('seg_ptr', 'atom_ptr', 'atoms', 'nca_c', 'bound_ca')]

    def knn(n_nodes=N, max_nodes=rb.max_protein_nodes, K=10, ws_n=ws_bytes, ptrs=None, n_prot=2):
        p = list(args) if ptrs is None else ptrs
        return lib.eqd_graph_build_knn(n_prot, n_nodes, max_nodes, *p, 30.0, K, nat.ptr(ws), ws_n, nat.ptr(deg), nat.ptr(x),
                                       nat.ptr(mu), st)

    assert knn(K=0) == -2 and knn(K=17) == -2 and knn(max_nodes=0) == -2
    assert knn(max_nodes=12801) == -2
    assert knn(ws_n=ws_bytes - 1) == -3
    for k in range(len(args)):
        p = list(args)
        p[k] = None
        assert knn(ptrs=p) == -1, k
    assert lib.eqd_graph_build_knn(2, N, rb.max_protein_nodes, *args, 30.0, 10, None, ws_bytes, nat.ptr(deg), nat.ptr(x),
                                   nat.ptr(mu), st) == -1
    for k in range(3):
        o = [nat.ptr(deg), nat.ptr(x), nat.ptr(mu)]
        o[k] = None
        assert lib.eqd_graph_build_knn(2, N, rb.max_protein_nodes, *args, 30.0, 10, nat.ptr(ws), ws_bytes, *o, st) == -1
    assert knn(n_nodes=0) == 0
    torch.cuda.synchronize()
    assert (deg == -7).all() and (x == -7).all() and (mu == -7).all()       # nothing was launched
    row_ptr = torch.zeros(N + 1, dtype=torch.int32, device=cuda_device)
    col = torch.full((N * 16,), -7, dtype=torch.int32, device=cuda_device)
    he = torch.full((N * 16, 27), -7.0, device=cuda_device)
    o = [nat.ptr(row_ptr), nat.ptr(deg), nat.ptr(ws), nat.ptr(col), nat.ptr(col), nat.ptr(he)]
    for k in range(len(o)):
        q = list(o)
        q[k] = None
        assert lib.eqd_graph_build_edges(N, *q, st) == -1, k
    assert lib.eqd_graph_build_edges(0, *o, st) == 0
    torch.cuda.synchronize()
    assert (col == -7).all() and (he == -7).all()


# ---- RMSD meter on rank-deficient sets ------------------------------------------------------------------------------------

def test_rmsd_meter_on_rank_deficient_sets(cuda_device):
    """eqd_rmsd_meter against the fp64 oracle complex_rmsd: the minimum RMSD is unique even where the rotation is not."""
    import iegmn_oracle as orc
    from equidock_public_b200.engine import GraphPlan
    from equidock_public_b200.eval import Meter_Unbound_Bound
    rng = np.random.default_rng(12)

    def collinear(n):
        step = rng.integers(-3, 4, 3)
        step[0] = step[0] or 1
        return (rng.integers(-30, 30, 3)[None] + np.arange(n)[:, None] * step[None]).astype(f64)

    def coplanar(n, xy=False):
        P = rng.integers(-20, 20, (n, 3)).astype(f64)
        if xy:
            P[:, 1] = P[:, 0]
        else:
            P[:, 2] = -4.0
        return P

    cases = []            # (name, true (n, 3), pred (n, 3), n_lig)

    def moved(Q, noise):
        R, t = _rigid(rng, 25.0)
        return (R @ Q.T).T + t + rng.normal(0, noise, Q.shape)

    sets = [('generic 2000+2000', rng.normal(0, 20, (4000, 3)), 2000)]
    for k in range(4):
        sets += [(f'1+1 ({k})', rng.normal(0, 5, (2, 3)), 1), (f'2+1 ({k})', rng.normal(0, 5, (3, 3)), 2),
                 (f'collinear ({k})', collinear(6 + 5 * k), 3 + k), (f'coplanar z ({k})', coplanar(8 + 8 * k), 4 + k),
                 (f'coplanar x=y ({k})', coplanar(8 + 8 * k, True), 4 + 2 * k)]
    for name, Q, nl in sets:
        for noise in (0.0, 0.5):
            cases.append((f'{name} noise {noise}', Q, moved(Q, noise), nl))
    M = coplanar(25)
    cases.append(('mirrored coplanar', M, moved(M * np.array([-1.0, 1.0, 1.0]), 0.0), 10))
    cases.append(('mirrored coplanar, noisy', M, moved(M * np.array([-1.0, 1.0, 1.0]), 0.3), 10))
    for name, Q, nl in [('identical collinear', collinear(15), 5), ('identical coplanar', coplanar(20), 8),
                        ('identical generic', rng.normal(0, 10, (50, 3)), 20), ('identical 1+1', rng.normal(0, 5, (2, 3)), 1)]:
        cases.append((name, Q, Q.copy(), nl))
    cases = [(n, Q.astype(f32), P.astype(f32), nl) for n, Q, P, nl in cases]
    lt = [Q[:nl] for _, Q, _, nl in cases]
    rt = [Q[nl:] for _, Q, _, nl in cases]
    lp = [P[:nl] for _, _, P, nl in cases]
    rp = [P[nl:] for _, _, P, nl in cases]
    z = torch.zeros(0, dtype=torch.int32, device=cuda_device)
    he = torch.zeros(0, 27, device=cuda_device)
    plan = GraphPlan([a.shape[0] for a in lt], [a.shape[0] for a in rt], z, z, z, z, he, he, cuda_device)
    tt = lambda L: torch.from_numpy(np.concatenate(L)).to(cuda_device)
    out = Meter_Unbound_Bound().update_rmsd_batch(plan, tt(lp), tt(rp), tt(lt), tt(rt)).cpu().numpy()
    worst = 0.0
    for k, (name, Q, P, nl) in enumerate(cases):
        f = lambda a: a.astype(f64)
        ref = orc.complex_rmsd(f(P[:nl]), f(P[nl:]), f(Q[:nl]), f(Q[nl:]))
        if name.startswith('identical'):
            assert out[k, 0] <= 1e-12, (name, out[k, 0])
        err = abs(out[k, 0] - ref) / max(1.0, ref)
        worst = max(worst, err)
        assert err <= 1e-9, (name, out[k, 0], ref)
    _note('rmsd meter rel', worst)
    _report('rmsd meter')
