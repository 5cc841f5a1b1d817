"""Device-resident training data: a whole pair archive (formats.save_pairs with labels) uploaded to one GPU once, and
minibatches assembled there by one kernel (csrc/batch_assemble.cu, ``eqd_assemble_batch``).

Per batch the host only picks pair indices and adds up sizes it keeps from the archive's offsets; the gather of the
pairs, the renumbering of edges, the plan's index arrays (``row_ptr``, ``seg_ptr``, node tiles), the training targets and
the reference's random re-posing of every ligand (``UniformRotation_Translation`` in its data set's ``__getitem__``,
src/utils/protein_utils.py:15-23, ``translation_interval`` 5 A for training, args.py:55) all happen on the device.
``DevicePairDataset.batch`` returns what ``DataParallelTrainer.step`` takes: a ``PairGraphBatch`` with its ``GraphPlan``
attached, and a ``PocketBatch``.

Re-posing: for batch slot b, a Philox4x32-10 stream with key = seed and counter = (slot, draw, step) gives R (unit
quaternion of four normals) and t (unit normal direction x U(0, translation_interval)), the law of
``synthetic.random_rigid``; then ``new_x = R (x - mean(x)) + t`` and ``pocket_lig = R (pocket - mean(x)) + t`` in fp64,
with ``x`` the ligand's unbound coordinates (ndata['x']) and the mean over its residues.  The receptor, ``x`` itself, the
bound coordinates and the receptor-side pocket points are not moved.
"""
from __future__ import annotations

import ctypes as C
from typing import Iterator, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _native as nat
from .engine import GraphPlan
from .formats import PairArchive
from .graph_build import _edge_counts
from .hetero_graph import LIGAND, LL, RECEPTOR, RR, PairGraphBatch
from .losses import PocketBatch

MAX_POCKET = 1024      # largest pocket eqd_losses solves (include/eqd_iegmn.h)


class DatasetError(ValueError):
    """An archive this data set cannot serve."""


class UnsortedEdgesError(DatasetError):
    """A protein's edges are not grouped by ascending destination, or name a node outside the protein."""


class InDegreeOverflowError(DatasetError):
    """A node has more in-edges than ``max_neighbor``."""


class BadResidueError(DatasetError):
    """A ``res_feat`` value outside [0, 21)."""


class MissingLabelsError(DatasetError):
    """The archive has no training labels (pocket points, bound coordinates)."""


class PocketTooLargeError(DatasetError):
    """A pocket larger than the loss kernel solves."""


class DeviceMemoryError(DatasetError):
    """The archive does not fit in the device's free memory."""


def _padded(a: np.ndarray, dtype) -> np.ndarray:
    """Contiguous copy with a 16-byte readable tail (the kernel reads `he` in aligned 16-byte vectors)."""
    a = np.ascontiguousarray(a, dtype=dtype).reshape(-1)
    out = np.zeros(a.size + 16 // a.itemsize, dtype=dtype)
    out[:a.size] = a
    return out


def _check_edges(side: str, node_ptr, edge_ptr, src, dst, max_neighbor: int):
    n_nodes = np.diff(node_ptr)
    prot = np.repeat(np.arange(n_nodes.size), np.diff(edge_ptr))
    n_of_edge = n_nodes[prot]
    bad = (src < 0) | (src >= n_of_edge) | (dst < 0) | (dst >= n_of_edge)
    if bad.any():
        p = int(prot[np.argmax(bad)])
        raise UnsortedEdgesError(f'{side} protein of pair {p}: an edge names a node outside the protein')
    g = dst.astype(np.int64) + node_ptr[:-1][prot]          # global destination: sorted iff every protein is
    if g.size > 1 and (np.diff(g) < 0).any():
        p = int(prot[1 + np.argmax(np.diff(g) < 0)])
        raise UnsortedEdgesError(f'{side} protein of pair {p}: edges are not grouped by ascending destination')
    deg = np.bincount(g, minlength=int(node_ptr[-1]))
    if deg.size and int(deg.max()) > max_neighbor:
        node = int(np.argmax(deg))
        p = int(np.searchsorted(node_ptr, node, side='right') - 1)
        raise InDegreeOverflowError(f'{side} protein of pair {p}: in-degree {int(deg.max())} > max_neighbor {max_neighbor}')


class PairSizes:
    """Per-pair node, edge and pocket counts of an archive, on the host: everything a batch's layout and an epoch's
    schedule are computed from."""

    def __init__(self, n_lig, n_rec, e_lig, e_rec, n_pocket):
        self.n_lig, self.n_rec, self.e_lig, self.e_rec, self.n_pocket = (np.asarray(v, np.int64) for v in
                                                                          (n_lig, n_rec, e_lig, e_rec, n_pocket))
        self.n_pairs = int(self.n_lig.size)

    @classmethod
    def from_archive(cls, archive: PairArchive) -> 'PairSizes':
        a = archive.a
        d = lambda k: np.diff(np.asarray(a[k], np.int64))
        return cls(d('lig/node_ptr'), d('rec/node_ptr'), d('lig/edge_ptr'), d('rec/edge_ptr'), d('label/pocket_ptr'))

    def offsets(self, indices: Sequence[int]) -> dict:
        """Layout of the batch ``indices``: 'index' [B], 'node' / 'edge' [2B+1] (segments in engine order: ligands of
        the batch, then receptors), 'pocket' [B+1], 'tile' [2B+1] offsets, all int64, and 'packed' = their int32
        concatenation in that order, the ``offsets`` argument of eqd_assemble_batch."""
        idx = np.asarray(indices, dtype=np.int64).reshape(-1)
        if idx.size == 0 or idx.min() < 0 or idx.max() >= self.n_pairs:
            raise IndexError(f'pair indices must be a non-empty list in [0, {self.n_pairs})')
        cum = lambda v: np.concatenate([[0], np.cumsum(v)]).astype(np.int64)
        nodes = np.concatenate([self.n_lig[idx], self.n_rec[idx]])
        o = {'index': idx, 'node': cum(nodes), 'edge': cum(np.concatenate([self.e_lig[idx], self.e_rec[idx]])),
             'pocket': cum(self.n_pocket[idx]), 'tile': cum((nodes + nat.TILE_ROWS - 1) // nat.TILE_ROWS)}
        if o['edge'][-1] >= 2 ** 31 or o['node'][-1] >= 2 ** 31:
            raise ValueError('batch too large for int32 node / edge ids')
        o['packed'] = np.concatenate([o[k] for k in ('index', 'node', 'edge', 'pocket', 'tile')]).astype(np.int32)
        return o

    def epoch_schedule(self, batch_size: int, seed: int, epoch: int, rank: int = 0, world: int = 1,
                       drop_last: bool = False):
        """[(pair indices, step, first slot)] of this rank in one epoch.  The epoch is a permutation of all pairs,
        deterministic in (seed, epoch), cut into global batches of ``batch_size`` (the last one shorter unless
        ``drop_last``); rank r takes its contiguous share of every global batch (``np.array_split`` over ``world``), and
        a final global batch with fewer pairs than ranks is skipped by every rank.  ``step`` = epoch * batches per epoch
        + global batch number, ``first slot`` = position of the rank's first pair in its global batch."""
        if batch_size < 1 or world < 1 or not 0 <= rank < world:
            raise ValueError('need batch_size >= 1 and 0 <= rank < world')
        perm = np.random.default_rng([int(seed), int(epoch)]).permutation(self.n_pairs)
        n = self.n_pairs // batch_size if drop_last else -(-self.n_pairs // batch_size)
        out = []
        for j in range(n):
            gb = perm[j * batch_size:(j + 1) * batch_size]
            if gb.size < world:
                continue
            parts = np.array_split(gb, world)
            out.append((parts[rank], epoch * n + j, sum(p.size for p in parts[:rank])))
        return out


class DevicePairDataset:
    """A labelled ``PairArchive`` held in device memory.  ``nbytes`` is what it occupies there."""

    def __init__(self, archive: PairArchive, device, max_neighbor: int = 10):
        a = archive.a
        dev = torch.device(device)
        if dev.type == 'cuda' and dev.index is None:
            dev = torch.device('cuda', torch.cuda.current_device())
        self.device, self.max_neighbor, self.n_pairs = dev, int(max_neighbor), len(archive)
        for key in ('label/pocket_ptr', 'label/pocket_coors', 'label/bound_lig', 'label/bound_rec'):
            if key not in a:
                raise MissingLabelsError(f'archive {archive.a.path} has no {key}: save_pairs(..., labels=...) writes them')
        host = {}
        for side in ('lig', 'rec'):
            node_ptr, edge_ptr = np.asarray(a[f'{side}/node_ptr'], np.int64), np.asarray(a[f'{side}/edge_ptr'], np.int64)
            if (np.diff(node_ptr) < 1).any():
                raise DatasetError(f'{side}: a protein without residues')
            src, dst = np.asarray(a[f'{side}/src'], np.int32), np.asarray(a[f'{side}/dst'], np.int32)
            _check_edges(side, node_ptr, edge_ptr, src, dst, self.max_neighbor)
            res = np.asarray(a[f'{side}/res_feat'])
            if res.size and int(res.max()) >= nat.N_RES_TYPES:
                raise BadResidueError(f'{side}: res_feat value {int(res.max())} outside [0, {nat.N_RES_TYPES})')
            host.update({f'{side}_node_ptr': node_ptr, f'{side}_edge_ptr': edge_ptr, f'{side}_src': src, f'{side}_dst': dst,
                         f'{side}_res_feat': np.ascontiguousarray(res, np.uint8).reshape(-1),
                         f'{side}_x': a[f'{side}/x'], f'{side}_mu_r_norm': a[f'{side}/mu_r_norm'],
                         f'{side}_he': _padded(a[f'{side}/he'], np.float32)})
        pocket_ptr = np.asarray(a['label/pocket_ptr'], np.int64)
        n_pocket = np.diff(pocket_ptr)
        if n_pocket.size and int(n_pocket.max()) > MAX_POCKET:
            raise PocketTooLargeError(f'pair {int(np.argmax(n_pocket))}: pocket of {int(n_pocket.max())} points > {MAX_POCKET}')
        x_lig = np.asarray(a['lig/x'], np.float64).reshape(-1, 3)
        n_lig = np.diff(host['lig_node_ptr'])
        centroid = np.add.reduceat(x_lig, host['lig_node_ptr'][:-1], axis=0) / n_lig[:, None]
        host.update({'pocket_ptr': pocket_ptr, 'pocket_coors': a['label/pocket_coors'], 'bound_lig': a['label/bound_lig'],
                     'bound_rec': a['label/bound_rec'], 'lig_new_x': a['lig/new_x'], 'lig_centroid': centroid})
        need = sum(int(np.asarray(v).nbytes) for v in host.values())
        if dev.type == 'cuda':
            free, _ = torch.cuda.mem_get_info(dev)
            if need > free:
                raise DeviceMemoryError(f'the archive needs {need} bytes of device memory; {dev} has {free} free')
        self.nbytes = need
        self._dev = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in host.items()}
        self._struct = nat.EqdPairArchive()
        self._struct.n_pairs = self.n_pairs
        for k, t in self._dev.items():
            setattr(self._struct, k, t.data_ptr())
        self.sizes = PairSizes(n_lig, np.diff(host['rec_node_ptr']), np.diff(host['lig_edge_ptr']),
                               np.diff(host['rec_edge_ptr']), n_pocket)

    def __len__(self):
        return self.n_pairs

    def batch(self, indices: Sequence[int], seed: Optional[int] = None, step: int = 0, translation_interval: float = 5.0,
              first_slot: int = 0) -> Tuple[PairGraphBatch, PocketBatch]:
        """The pairs ``indices`` (repeats allowed) as (PairGraphBatch with its GraphPlan attached, PocketBatch) on the
        device.  ``seed=None``: ligands as stored; otherwise every ligand is re-posed with the motion of Philox
        counter (first_slot + its position, step).  ``first_slot`` lets the ranks of a data-parallel step draw the poses
        of their share of one global batch.  The applied motions are ``graph.rigid`` = (R (B,3,3), t (B,3)) fp64.
        No host sync: the only transfer is the offsets (host to device)."""
        lay = self.sizes.offsets(indices)
        idx, node_off, edge_off, pocket_off, tile_off = (lay[k] for k in ('index', 'node', 'edge', 'pocket', 'tile'))
        B = int(idx.size)
        N, N_l, E, E_l = int(node_off[-1]), int(node_off[B]), int(edge_off[-1]), int(edge_off[B])
        P, T = int(pocket_off[-1]), int(tile_off[-1])
        dev = self.device
        i32, f32, f64 = (dict(dtype=t, device=dev) for t in (torch.int32, torch.float32, torch.float64))
        # ligand and receptor edge features in one allocation, each part 16-byte aligned with a readable row past its end
        F = nat.EDGE_FEATS
        r0 = ((E_l + 1) * F + 3) // 4 * 4
        he_buf = torch.empty(r0 + (E - E_l + 1) * F, **f32)
        he_l, he_r = he_buf[:(E_l + 1) * F].view(E_l + 1, F), he_buf[r0:].view(E - E_l + 1, F)
        out = {'res_feat': torch.empty(N, 1, **f32), 'x': torch.empty(N, 3, **f32), 'new_x': torch.empty(N_l, 3, **f32),
               'mu_r_norm': torch.empty(N, 5, **f32), 'row_ptr': torch.empty(N + 1, **i32), 'col_src': torch.empty(E, **i32),
               'edge_dst': torch.empty(E, **i32), 'he_lig': he_l, 'he_rec': he_r, 'seg_ptr': torch.empty(2 * B + 1, **i32),
               'node_tiles': torch.empty(2 * T, **i32), 'pocket_ptr': torch.empty(B + 1, **i32),
               'pocket_lig': torch.empty(P, 3, **f32), 'pocket_rec': torch.empty(P, 3, **f32),
               'bound_lig': torch.empty(N_l, 3, **f32), 'bound_rec': torch.empty(N - N_l, 3, **f32),
               'rot': torch.empty(B, 3, 3, **f64), 'trans': torch.empty(B, 3, **f64)}
        ob = nat.EqdBatchOut()
        for k, t in out.items():
            setattr(ob, k, t.data_ptr())
        max_seg_edges = int(np.diff(edge_off).max())
        lib = nat.load()
        with torch.cuda.device(dev):
            offs = torch.from_numpy(lay['packed']).pin_memory().to(dev, non_blocking=True)
            st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            nat.check(lib.eqd_assemble_batch(C.byref(self._struct), B, nat.ptr(offs), max_seg_edges,
                                             0 if seed is None else int(seed) & (2 ** 64 - 1), int(step), int(first_slot),
                                             float(translation_interval), 0 if seed is None else 1, C.byref(ob), st),
                      'eqd_assemble_batch')
            col_src, edge_dst = out['col_src'], out['edge_dst']
            n_lig, n_rec = self.sizes.n_lig[idx].tolist(), self.sizes.n_rec[idx].tolist()
            g = PairGraphBatch({LIGAND: N_l, RECEPTOR: N - N_l},
                               {LL: (col_src[:E_l], edge_dst[:E_l]), RR: (col_src[E_l:] - N_l, edge_dst[E_l:] - N_l)},
                               {LIGAND: torch.tensor(n_lig, dtype=torch.int64), RECEPTOR: torch.tensor(n_rec, dtype=torch.int64)},
                               _edge_counts(np.diff(edge_off[:B + 1]).tolist(), np.diff(edge_off[B:]).tolist(), B))
        g._ndata[LIGAND] = {'res_feat': out['res_feat'][:N_l], 'x': out['x'][:N_l], 'new_x': out['new_x'],
                            'mu_r_norm': out['mu_r_norm'][:N_l]}
        g._ndata[RECEPTOR] = {'res_feat': out['res_feat'][N_l:], 'x': out['x'][N_l:], 'mu_r_norm': out['mu_r_norm'][N_l:]}
        g._edata[LL]['he'], g._edata[RR]['he'] = he_l[:E_l], he_r[:E - E_l]
        g._eqd_plan = GraphPlan.from_device_arrays(n_lig, n_rec, E_l, E, col_src, edge_dst, out['row_ptr'], he_l[:E_l], he_r[:E - E_l],
                                                   out['seg_ptr'],
                                                   out['node_tiles'], node_off, dev, self.max_neighbor, keep=(offs,))
        g.rigid = (out['rot'], out['trans'])
        tgt = PocketBatch.from_device_arrays(out['bound_lig'], out['bound_rec'], out['pocket_lig'], out['pocket_rec'],
                                             out['pocket_ptr'], self.sizes.n_pocket[idx].tolist())
        return g, tgt

    def epoch(self, batch_size: int, seed: int, epoch: int, rank: int = 0, world: int = 1, drop_last: bool = False,
              repose: bool = True, translation_interval: float = 5.0) -> Iterator[Tuple[PairGraphBatch, PocketBatch]]:
        """Yields this rank's batches of one shuffled epoch (``PairSizes.epoch_schedule``): ``batch_size`` is the global
        batch (the reference's ``bs``), so the ranks of a ``DataParallelTrainer`` together step on the reference's global
        batches.  With ``repose`` (under key ``seed``), the pose of a pair depends only on its global batch and its
        position there, not on the number of ranks."""
        for idx, step, first in self.sizes.epoch_schedule(batch_size, seed, epoch, rank, world, drop_last):
            yield self.batch(idx, seed if repose else None, step, translation_interval, first)
