"""CPU: the host side of DevicePairDataset -- batch offsets computed from the per-pair sizes against the archive's own
batching, epoch schedules (determinism, rank shares), and the ctypes mirror of the new ABI structs."""
import numpy as np
import pytest

from bench_train import make_targets
from equidock_public_b200 import _native as nat
from equidock_public_b200 import synthetic
from equidock_public_b200.datasets import PairSizes
from equidock_public_b200.formats import PairArchive, save_pairs
from equidock_public_b200.hetero_graph import LIGAND, LL, RECEPTOR, RR
from test_abi_and_host import _header_struct_fields

SIZES = [(1, 129, 10), (127, 128, 10), (128, 1, 10), (129, 127, 7), (40, 300, 3), (2, 5, 10), (200, 61, 10)]


@pytest.fixture(scope='module')
def archive(tmp_path_factory):
    rng = np.random.default_rng(4)
    pairs, labels = [], []
    for n_l, n_r, k in SIZES:
        p = (synthetic.synthetic_protein(rng, n_l, k), synthetic.synthetic_protein(rng, n_r, k))
        tg = make_targets(p, rng)
        pairs.append(p)
        labels.append({'pocket_coors': tg['pocket_lig'], 'bound_lig': tg['bound_lig'], 'bound_rec': tg['bound_rec']})
    path = tmp_path_factory.mktemp('ds') / 'a.eqd'
    save_pairs(str(path), pairs, labels)
    return PairArchive(str(path))


@pytest.mark.parametrize('idx', [[0], [3, 3, 0, 6], list(range(7)), [6, 5, 4, 3, 2, 1, 0, 1]])
def test_offsets_match_the_archive(archive, idx):
    o = PairSizes.from_archive(archive).offsets(idx)
    g = archive.batch(idx)
    B = len(idx)
    nodes = g.batch_num_nodes(LIGAND).tolist() + g.batch_num_nodes(RECEPTOR).tolist()
    edges = g.batch_num_edges(LL).tolist() + g.batch_num_edges(RR).tolist()
    assert o['node'].tolist() == np.concatenate([[0], np.cumsum(nodes)]).tolist()
    assert o['edge'].tolist() == np.concatenate([[0], np.cumsum(edges)]).tolist()
    assert o['edge'][B] == g.num_edges(LL) and o['edge'][-1] == g.num_edges(LL) + g.num_edges(RR)
    pockets = [archive.labels(i)['pocket_coors'].shape[0] for i in idx]
    assert o['pocket'].tolist() == np.concatenate([[0], np.cumsum(pockets)]).tolist()
    tiles = [len(range(0, n, nat.TILE_ROWS)) for n in nodes]        # GraphPlan's (segment, first node) tiles
    assert o['tile'].tolist() == np.concatenate([[0], np.cumsum(tiles)]).tolist()
    assert o['packed'].dtype == np.int32 and o['packed'].size == 8 * B + 4
    assert o['packed'].tolist() == o['index'].tolist() + o['node'].tolist() + o['edge'].tolist() + o['pocket'].tolist() + o['tile'].tolist()


def test_offsets_reject_bad_indices(archive):
    s = PairSizes.from_archive(archive)
    for bad in ([], [7], [-1]):
        with pytest.raises(IndexError):
            s.offsets(bad)


def test_epoch_schedule_is_deterministic_and_covers_every_pair():
    s = PairSizes(*(np.ones(103, np.int64),) * 5)
    a = s.epoch_schedule(16, seed=9, epoch=2)
    b = s.epoch_schedule(16, seed=9, epoch=2)
    c = s.epoch_schedule(16, seed=9, epoch=3)
    assert all(np.array_equal(x[0], y[0]) and x[1:] == y[1:] for x, y in zip(a, b)) and len(a) == len(b) == 7
    assert not all(np.array_equal(x[0], y[0]) for x, y in zip(a, c))
    assert sorted(np.concatenate([x[0] for x in a]).tolist()) == list(range(103))
    assert [x[1] for x in a] == list(range(14, 21)) and all(x[2] == 0 for x in a)
    assert len(s.epoch_schedule(16, seed=9, epoch=2, drop_last=True)) == 6


@pytest.mark.parametrize('world', [2, 3, 4])
def test_epoch_ranks_are_disjoint_shares_of_each_global_batch(world):
    s = PairSizes(*(np.ones(50, np.int64),) * 5)
    glob = s.epoch_schedule(12, seed=1, epoch=0)
    per_rank = [s.epoch_schedule(12, seed=1, epoch=0, rank=r, world=world) for r in range(world)]
    n = len(per_rank[0])
    assert all(len(p) == n for p in per_rank)
    assert n == len(glob) - (1 if glob[-1][0].size < world else 0)
    for j in range(n):
        parts = [p[j] for p in per_rank]
        assert np.array_equal(np.concatenate([q[0] for q in parts]), glob[j][0])      # disjoint, in global order
        assert all(q[1] == glob[j][1] for q in parts)
        assert [q[2] for q in parts] == np.concatenate([[0], np.cumsum([q[0].size for q in parts])[:-1]]).tolist()
    with pytest.raises(ValueError):
        s.epoch_schedule(12, seed=1, epoch=0, rank=world, world=world)


@pytest.mark.parametrize('cname,ctype', [('eqd_pair_archive', nat.EqdPairArchive), ('eqd_batch_out', nat.EqdBatchOut)])
def test_batch_assembly_structs_list_the_header_fields_in_order(cname, ctype):
    assert _header_struct_fields(cname) == [f[0] for f in ctype._fields_]
