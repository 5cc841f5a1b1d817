"""CPU: the graph oracle's options used by the device graph-build tests (tests/test_gpu_graph_build.py) -- per-row
distances (``build_rows``), the fp64 alignment (``kabsch64``), the stable tie order and degree-0 residues."""
import numpy as np

import golden_io as gio
import graph_oracle as go


def _single_atoms(ca, rng):
    ca = np.asarray(ca, np.float32)
    n = ca.shape[0]
    d = rng.normal(size=(n, 2, 3))
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    return {'atoms': ca.copy(), 'atom_ptr': np.arange(n + 1, dtype=np.int32),
            'nca_c': np.stack([ca + 1.46 * d[:, 0], ca, ca + 1.52 * d[:, 1]], 1).astype(np.float32),
            'res_feat': np.zeros((n, 1), np.float32), 'bound_ca': ca.copy()}


def test_build_rows_equals_build_graph_on_sampled_rows():
    _, allp = gio.load_all('dips')
    rng = np.random.default_rng(0)
    for name in ('dm_5dm7.pdb1_22.dill', 'aq_4aqa.pdb1_0.dill'):
        p = dict(allp[name]['lig'])
        p['bound_ca'] = allp[name]['ca']['ligand_gt'].astype(np.float32)      # a real rotation
        n = p['nca_c'].shape[0]
        rows = np.unique(np.concatenate([[0, n - 1], rng.choice(n, 40, replace=False)]))
        for cutoff, K in ((30.0, 10), (np.float32(7.3), 16), (6.0, 1)):
            for k64 in (False, True):
                full = go.build_graph(p, cutoff, K, kabsch64=k64)
                part = go.build_rows(p, rows, cutoff, K, kabsch64=k64)
                sel = np.concatenate([np.nonzero(full['dst'] == i)[0] for i in rows])
                assert np.array_equal(part['src'], full['src'][sel]) and np.array_equal(part['dst'], full['dst'][sel])
                assert np.abs(part['dist'] - full['dist'][sel]).max(initial=0) <= 1e-13 * 30
                assert np.abs(part['he'] - full['he'][sel]).max(initial=0) <= 1e-6
                assert np.array_equal(part['x'], full['x'][rows])
                assert np.abs(part['mu_r_norm'] - full['mu_r_norm'][rows]).max() <= 1e-6


def test_kabsch64_is_a_proper_rotation_and_matches_the_fp32_fit():
    _, allp = gio.load_all('db5')
    e = allp['1QA9']
    p = dict(e['lig'])
    p['bound_ca'] = e['ca']['ligand_gt'].astype(np.float32)
    x64, frames64 = go._align(p, True)
    x32, _ = go._align(p, False)
    assert x64.dtype == np.float64 and frames64[0].dtype == np.float64
    ca = p['nca_c'][:, 1].astype(np.float64)
    R, t = go.kabsch(ca.T, p['bound_ca'].astype(np.float64).T)
    assert np.abs(R @ R.T - np.eye(3)).max() < 1e-14 and abs(np.linalg.det(R) - 1) < 1e-14
    assert np.abs((R @ ca.T + t).T - x64).max() < 1e-12
    assert np.abs(x32 - x64).max() < 1e-6 * np.abs(x64).max() + 1e-4       # the fp32 fit is ~1e-7 |x| away
    # rank-deficient fits (collinear, coplanar, 2 points) still give proper rotations
    rng = np.random.default_rng(1)
    for P in (np.arange(9)[:, None] * np.array([[1.0, 2.0, -1.0]]), np.c_[rng.integers(-9, 9, (12, 2)), np.full(12, 3.0)],
              rng.normal(size=(2, 3))):
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        R, _ = go.kabsch(P.T, (q @ P.T).astype(np.float32).astype(np.float64))
        assert np.abs(R @ R.T - np.eye(3)).max() < 1e-12 and abs(np.linalg.det(R) - 1) < 1e-12


def test_degree_zero_residues_and_stable_tie_order():
    rng = np.random.default_rng(2)
    # residue 0 with 12 neighbours at exactly 2 A (ties), residues far away with degree 0
    dirs = np.array([[2, 0, 0], [-2, 0, 0], [0, 2, 0], [0, -2, 0], [0, 0, 2], [0, 0, -2]], np.float64)
    ca = np.concatenate([[[0, 0, 0]], dirs[::-1], dirs * 1.0 + 100.0, [[500, 0, 0], [0, 500, 0]]])
    p = _single_atoms(ca, rng)
    g = go.build_graph(p, cutoff=8.0, max_neighbor=3, kabsch64=True)
    nb0 = g['src'][g['dst'] == 0]
    assert nb0.tolist() == [1, 2, 3]                                    # 6 tied at 2 A: the three lowest indices
    for i in (13, 14):
        assert not (g['dst'] == i).any()
        assert (g['mu_r_norm'][i] == 0).all()
    r = go.build_rows(p, [0, 13, 14], cutoff=8.0, max_neighbor=3, kabsch64=True)
    assert r['src'].tolist() == [1, 2, 3] and (r['mu_r_norm'][1:] == 0).all() and r['he'].shape == (3, 27)
