"""CPU: the dropout mask function (tests/dropout_masks.py, the numpy restatement of csrc/philox.cuh) and the fp64 batch
restatement the GPU dropout tests compare against."""
import numpy as np
import pytest
import torch

import dropout_masks as dm
import golden_io as gio
from equidock_public_b200 import _native as nat


def test_philox_known_answers():
    """Known-answer vectors of Philox4x32-10 (Random123's kat_vectors)."""
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
              (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for c, k, want in cases:
        got = dm.philox4x32_10(*c, *k)
        assert [int(w) for w in got] == list(want)


@pytest.mark.parametrize('p', [0.1, 0.25, 0.5])
def test_keep_rate_within_five_sigma(p):
    rows, cols = np.arange(40000), np.arange(256)      # 1.02e7 draws
    k = dm.keep(0x123456789abcdef, 0, 3, 1, rows, cols, p)
    n = k.size
    sigma = np.sqrt(p * (1 - p) / n)
    assert abs(k.mean() - (1 - p)) < 5 * sigma


def test_masks_of_different_sites_layers_ranks_are_uncorrelated():
    rows, cols, p = np.arange(4000), np.arange(64), 0.25
    seed = 987654321987
    base = dm.keep(seed, 0, 1, 0, rows, cols, p).ravel().astype(np.float64)
    n = base.size
    for rank, layer, site in ((0, 1, 1), (0, 2, 0), (1, 1, 0), (0, 5, 3)):
        other = dm.keep(seed, rank, layer, site, rows, cols, p).ravel().astype(np.float64)
        r = np.corrcoef(base, other)[0, 1]
        assert abs(r) < 5 / np.sqrt(n), (rank, layer, site, r)
    assert abs(np.corrcoef(base, dm.keep(seed + 1, 0, 1, 0, rows, cols, p).ravel())[0, 1]) < 5 / np.sqrt(n)


def test_p_one_drops_everything_and_descriptor_matches():
    assert not dm.keep(5, 0, 0, 0, np.arange(100), np.arange(64), 1.0).any()
    d = nat.dropout_descriptor(1.0, 5, 0)
    assert d.scale == 0.0
    for p in (0.1, 0.25, 0.5, 1.0):
        d = nat.dropout_descriptor(p, (1 << 64) - 3, 7, 2)
        assert d.threshold == dm.threshold(p) and np.float32(d.scale) == np.float32(dm.scale(p))
        assert (d.seed, d.layer, d.rank) == ((1 << 64) - 3, 7, 2)


def test_dropout_struct_layout():
    import ctypes
    assert ctypes.sizeof(nat.EqdDropout) == 32 and nat.EqdDropout.p.offset == 8 and nat.EqdDropout.layer.offset == 20
    assert nat.EqdLayer.dropout.offset == ctypes.sizeof(nat.EqdLayerParams) + ctypes.sizeof(nat.EqdLayerConsts)


def batch_inputs(pairs):
    """Engine-numbered fp64 inputs of dropout_masks.model_forward for a list of (lig, rec) numpy pairs."""
    B = len(pairs)
    sides = [p[0] for p in pairs] + [p[1] for p in pairs]
    n = [len(s['res_feat']) for s in sides]
    seg = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    src = np.concatenate([s['src'].astype(np.int64) + seg[i] for i, s in enumerate(sides)])
    dst = np.concatenate([s['dst'].astype(np.int64) + seg[i] for i, s in enumerate(sides)])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64))
    return {'B': B, 'seg': seg.tolist(), 'src': torch.from_numpy(src), 'dst': torch.from_numpy(dst),
            'res': torch.from_numpy(np.concatenate([s['res_feat'].reshape(-1) for s in sides]).astype(np.int64)),
            'mu_r_norm': t(np.concatenate([s['mu_r_norm'] for s in sides])),
            'x': t(np.concatenate([p[0]['new_x'] for p in pairs] + [p[1]['x'] for p in pairs])),
            'he': t(np.concatenate([s['he'] for s in sides]))}


@pytest.mark.parametrize('ds', ['db5', 'dips'])
def test_batch_restatement_without_masks_matches_the_golden_fp64_outputs(ds):
    names, pairs, outs, _ = gio.load_pairs(ds)
    name = names[0]
    sd = {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in gio.load_checkpoint(ds).items()}
    coors, Y, rot, trans = dm.model_forward(sd, gio.load_args(ds), batch_inputs([pairs[name]]))
    ref = outs[name]['ref64']
    scale_ = max(1.0, np.abs(ref['ligand_coors']).max())
    assert np.abs(coors.numpy() - ref['ligand_coors']).max() < 1e-6 * scale_
    assert np.abs(Y[0].numpy() - ref['keypts_ligand']).max() < 1e-6 * scale_
    assert np.abs(Y[1].numpy() - ref['keypts_receptor']).max() < 1e-6 * scale_
    assert np.abs(rot[0].numpy() - ref['rotation'].reshape(3, 3)).max() < 1e-7
