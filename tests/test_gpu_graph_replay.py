"""GPU (H100): the CUDA-graph replay paths that serve inference -- ``model.graphed(batch)`` (graphed.GraphedForward),
serving.PipelinedInference and graph_build.ResidueGraphedForward -- against the eager forward, bit for bit (a replay
runs the eager path's kernels on the eager path's buffers), and the eager forward against the fp64 restatement
(fp64_ref.model_forward) at gpu_harness._coord_bound:

  - after every route by which the weights change: DataParallelTrainer.step (its fused Adam writes the parameters
    through a raw pointer), loss.backward() + torch.optim.Adam, load_state_dict, and in-place changes of one layer's
    coors_mlp.4.bias (a value the layer descriptor carries by value) or of one head weight;
  - at the benchmark's shapes: 330 x (200+200) (the resident attention), the 25 ragged db5-testset pairs and
    2 x (2000+2000) (the streamed attention);
  - over a stream of batches of changing shapes through PipelinedInference's three slots, with and without graphs,
    including two batches of one slot signature whose per-protein edge counts differ;
  - for flagged batches inside a graphed stream: unsorted edges, then the SVD guard, then an ordinary batch."""
import numpy as np
import pytest
import torch

import bench
import fp64_ref as fr
import golden_io as gio
from equidock_public_b200 import graphed
from equidock_public_b200 import hetero_graph as hg
from equidock_public_b200 import synthetic
from equidock_public_b200.engine import GraphPlan
from equidock_public_b200.graph_build import ResidueBatch, ResidueGraphedForward, build_graphs
from equidock_public_b200.serving import PipelinedInference, _tensors
from equidock_public_b200.training import DataParallelTrainer
from gpu_harness import _coord_bound, _device_batch, _model_pairs, _model_targets, _pair_loss, _shard

pytestmark = pytest.mark.gpu

KEYS = ('ligand_coors', 'rotation', 'translation')       # what PipelinedInference returns
RES_MAX_NODES = 248      # the largest protein the resident attention of the 64-wide layers serves (csrc/attn_tc.cu)
GUARD_SEED = 1234        # torch.manual_seed of every forward whose SVD guard may draw


@pytest.fixture(scope='module')
def dips(cuda_device):
    return gio.build_model('dips', cuda_device), gio.load_args('dips')


def _outs(raw, keys=KEYS + ('keypts',)):
    return {k: raw[k].detach().clone() for k in keys}


def _eager(model, g, seed=GUARD_SEED):
    """The eager forward of a graph object: its raw outputs (cloned), the plan it ran on and the guard's draws."""
    torch.manual_seed(seed)
    raw = model.iegmn_original.run_engine(g)
    return dict(_outs(raw), plan=raw['plan'], draws=list(raw['guard_draws']))


def _same(tag, got, ref, keys=KEYS + ('keypts',)):
    for k in keys:
        a, b = got[k].cpu(), ref[k].cpu()
        assert a.shape == b.shape, (tag, k, a.shape, b.shape)
        assert torch.equal(a, b), \
            f'{tag}: {k} differs from the eager forward, max |diff| = {float((a.double() - b.double()).abs().max()):.3e}'


def _vs_fp64(model, args, g, eager, tag):
    """The eager forward's coordinates and rotations against fp64_ref.model_forward on the model's current weights,
    with the guard's draws replayed from GUARD_SEED."""
    _, rand_diag = fr.replay_draws(GUARD_SEED)
    co, _, rot, _, draws = fr.model_forward(fr.fp64_state(model), args, fr.inputs_of(g, eager['plan']), rand_diag=rand_diag)
    assert list(draws) == eager['draws'], (tag, draws, eager['draws'])
    cr = co.numpy()
    err = float(np.abs(eager['ligand_coors'].cpu().double().numpy() - cr).max())
    err_r = float(np.abs(eager['rotation'].cpu().double().numpy() - rot.numpy()).max())
    print(f'\n{tag}: max |coors - fp64| = {err:.3e} (bound {_coord_bound(cr):.3e}), max |R - fp64| = {err_r:.3e}')
    assert err <= _coord_bound(cr), tag
    assert err_r <= 2e-4, tag


def _host(pairs):
    return hg.batch_pairs(synthetic.to_torch_pairs(pairs)).pin_memory()


def _stream(pipe, hosts):
    out = []
    for res in pipe.run(iter(hosts)):
        res['_event'].synchronize()
        out.append({k: res[k].clone() for k in KEYS})
    return out


# ---- 1. weight updates ------------------------------------------------------------------------------------------------

VAL = [(70, 55), (129, 20), (40, 131), (64, 64)]
RESIDUES = [(60, 80), (100, 50)]
ROUTES = [('trainer', 'db5'), ('trainer', 'dips'), ('adam', 'dips'), ('load_state_dict', 'dips'),
          ('coors_bias', 'dips'), ('head_weight', 'dips')]


@pytest.fixture(scope='module')
def train_batch(cuda_device):
    """The benchmark's 32-pair training batch and its targets."""
    return _device_batch(_shard(0, 1)[0], cuda_device)


def _update(route, model, trainer, train_batch, dev):
    iegmn = model.iegmn_original
    if route == 'trainer':
        model.train()
        for seed in (5, 6):
            torch.manual_seed(seed)
            trainer.step(*train_batch)
    elif route == 'adam':
        pairs = _model_pairs('dips', 'ragged')
        model.train()
        opt = torch.optim.Adam(model.parameters(), lr=1e-3)
        coors, kp_l, kp_r, _, _ = model(gio.make_batch(pairs, dev), epoch=0)
        _pair_loss(coors, (kp_l, kp_r), _model_targets(pairs), [len(l['res_feat']) for l, _ in pairs]).backward()
        opt.step()
    elif route == 'load_state_dict':
        gen = torch.Generator().manual_seed(7)
        model.load_state_dict({k: v + 0.05 * v.abs().mean() * torch.randn(v.shape, generator=gen).to(v.device)
                               for k, v in model.state_dict().items()})
    elif route == 'coors_bias':
        with torch.no_grad():
            iegmn.iegmn_layers[3].coors_mlp[4].bias.add_(0.25)
    else:
        with torch.no_grad():
            iegmn.att_mlp_key_ROT[0].weight.mul_(1.25)
    torch.cuda.synchronize()
    model.eval()


@pytest.mark.parametrize('route,ds', ROUTES)
def test_every_replay_path_follows_a_weight_update(route, ds, train_batch, cuda_device):
    """Captured in eval mode before the update: model.graphed, a PipelinedInference whose three slots hold graphs, and a
    ResidueGraphedForward.  After the update (and back in eval mode) each of them replays the post-update eager forward
    bit for bit; the pre-update replay differs from it (the update is visible), and the post-update eager forward agrees
    with fp64 on the updated weights.  The trainer is built before the captures: it re-points the parameters at its
    flat buffer, and the captures must see the pointers the updates then write through."""
    dev = cuda_device
    model, args = gio.build_model(ds, dev), gio.load_args(ds)
    trainer = DataParallelTrainer(model, lr=1e-3) if route == 'trainer' else None
    model.eval()
    rng = np.random.default_rng(61)
    pairs = [synthetic.synthetic_pair(rng, a, b, 10) for a, b in VAL]
    rb = ResidueBatch([synthetic.synthetic_residue_pair(rng, a, b) for a, b in RESIDUES])
    host = _host(pairs)
    gf = model.graphed(gio.make_batch(pairs, dev))
    pipe = PipelinedInference(model, dev, use_cuda_graph=True)
    _stream(pipe, [host] * 3)
    assert all(s.graphed is not None for s in pipe.slots)
    rgf = ResidueGraphedForward(model, rb, dev)
    pre = _outs(gf.launch().raw_result())
    pre_res = _outs(rgf.launch().raw_result())

    _update(route, model, trainer, train_batch, dev)
    g = gio.make_batch(pairs, dev)
    eager = _eager(model, g)
    eager_res = _eager(model, build_graphs(rb, dev))
    assert not torch.equal(pre['ligand_coors'], eager['ligand_coors']), f'{route}: the update left the forward as it was'
    assert not torch.equal(pre_res['ligand_coors'], eager_res['ligand_coors'])
    _same(f'{route}: model.graphed', _outs(gf.launch().raw_result()), eager)
    for i, res in enumerate(_stream(pipe, [host] * 3)):
        _same(f'{route}: PipelinedInference slot {i}', res, eager, KEYS)
    rgf.upload(rb)
    _same(f'{route}: ResidueGraphedForward', _outs(rgf.launch().raw_result()), eager_res)
    _vs_fp64(model, args, g, eager, f'{route} {ds}')


# ---- 2. the benchmark's shapes ----------------------------------------------------------------------------------------

BENCH_PAIRS = {'db5-shaped': 330, 'db5-testset': 25, 'large': 2}


def _bench_pairs(workload, seed):
    sizes = bench.pair_sizes(workload, BENCH_PAIRS[workload])
    return [synthetic.synthetic_pair(np.random.default_rng([seed, i]), a, b, bench.KNN) for i, (a, b) in enumerate(sizes)]


@pytest.mark.parametrize('workload', list(BENCH_PAIRS))
def test_replay_at_the_benchmark_shapes(workload, dips, cuda_device):
    """The benchmark's batches with the DIPS checkpoint: two replays == the eager forward, a second same-shaped batch
    written in place and refreshed == its own eager forward, and the first, the last and the largest pair of the
    eager forward == fp64 (pairs are independent: the reference runs each alone).  330 x (200+200) is a batch the
    resident attention serves, 2000+2000 one it does not."""
    dev = cuda_device
    model, args = dips
    pa, pb = _bench_pairs(workload, 1), _bench_pairs(workload, 2)
    ea, eb = _eager(model, gio.make_batch(pa, dev)), _eager(model, gio.make_batch(pb, dev))
    static = gio.make_batch(pa, dev)
    gf = model.graphed(static)
    biggest = gf.plan.struct.max_segment_nodes
    if workload == 'db5-shaped':
        assert biggest <= RES_MAX_NODES
    if workload == 'large':
        assert biggest > RES_MAX_NODES
    for rep in range(2):
        _same(f'{workload} replay {rep}', _outs(gf.launch().raw_result()), ea)
    dst = dict(_tensors(static))
    for key, t in _tensors(gio.make_batch(pb, dev)):
        dst[key].copy_(t)
    assert gf.refresh()
    _same(f'{workload} refreshed batch', _outs(gf.launch().raw_result()), eb)

    sd = fr.fp64_state(model)
    n_lig = [len(l['res_feat']) for l, _ in pa]
    off = np.concatenate([[0], np.cumsum(n_lig)])
    sizes = [len(l['res_feat']) + len(r['res_feat']) for l, r in pa]
    for i in sorted({0, len(pa) - 1, int(np.argmax(sizes))}):
        g1 = gio.make_batch([pa[i]], dev)
        co, _, rot, _, _ = fr.model_forward(sd, args, fr.inputs_of(g1, GraphPlan.from_graph(g1, dev, bench.KNN)))
        cr = co.numpy()
        err = float(np.abs(ea['ligand_coors'][off[i]:off[i + 1]].cpu().double().numpy() - cr).max())
        err_r = float(np.abs(ea['rotation'][i].cpu().double().numpy() - rot[0].numpy()).max())
        print(f'\n{workload} pair {i} ({pa[i][0]["x"].shape[0]}+{pa[i][1]["x"].shape[0]}): max |coors - fp64| = '
              f'{err:.3e} (bound {_coord_bound(cr):.3e}), max |R - fp64| = {err_r:.3e}')
        assert err <= _coord_bound(cr), (workload, i)
        assert err_r <= 2e-4, (workload, i)


# ---- 3. a stream of mixed shapes --------------------------------------------------------------------------------------

A_SIZES = [(60, 45), (33, 70), (90, 20)]


def _in_degrees(prot, want):
    """The protein with only the first want[d] in-edges of every node d (edges stay grouped by destination)."""
    first = np.searchsorted(prot['dst'], prot['dst'])
    keep = (np.arange(prot['dst'].shape[0]) - first) < want[prot['dst']]
    return dict(prot, **{k: prot[k][keep] for k in ('src', 'dst', 'he')})


def _stream_pairs(kind, seed):
    """'A': 6 in-edges per node on 8-NN graphs.  "A'": the same node counts and edge totals, but 20 nodes of each protein
    of pair 0 keep 5 in-edges and 20 of pair 1 keep 7, so the per-protein edge counts differ from A's while the slot
    signature and GraphPlan.refresh's check do not.  'B' and 'C': other shapes, k = 10."""
    rng = np.random.default_rng(seed)
    if kind == 'B':
        return [synthetic.synthetic_pair(rng, 50, 64, 10) for _ in range(4)]
    if kind == 'C':
        return [synthetic.synthetic_pair(rng, a, b, 10) for a, b in ((129, 8), (8, 129))]
    pairs = []
    for i, (a, b) in enumerate(A_SIZES):
        sides = []
        for prot in synthetic.synthetic_pair(rng, a, b, 8):
            want = np.full(prot['x'].shape[0], 6)
            if kind == "A'" and i < 2:
                want[:20] = 5 if i == 0 else 7
            sides.append(_in_degrees(prot, want))
        pairs.append(tuple(sides))
    return pairs


# every slot (batch k goes to slot k % 3) sees same-shape refills and shape changes; A and A' share a signature
STREAM = ['A', 'C', 'B', "A'", 'C', 'C', 'B', 'A', 'C', 'B', "A'", 'A']


def _shape(kind):
    return kind.rstrip("'")


@pytest.mark.parametrize('use_graph', [True, False])
def test_pipelined_stream_of_mixed_shapes(use_graph, dips, cuda_device, monkeypatch):
    """12 batches of three shapes over the three slots: every result == the eager forward of its batch bit for bit, and
    stays intact while the next two are produced (its pinned buffers are reused three batches later); with graphs, a
    slot captures once per shape change and never on a same-shape refill."""
    dev = cuda_device
    model, _ = dips
    batches = [_stream_pairs(kind, 100 + k) for k, kind in enumerate(STREAM)]
    a, a2 = batches[STREAM.index('A')], batches[STREAM.index("A'")]
    assert [len(l['dst']) for l, _ in a] != [len(l['dst']) for l, _ in a2]
    assert sum(len(l['dst']) for l, _ in a) == sum(len(l['dst']) for l, _ in a2)
    assert sum(len(r['dst']) for _, r in a) == sum(len(r['dst']) for _, r in a2)
    eager = [_eager(model, gio.make_batch(p, dev)) for p in batches]

    made, captured = [], []

    class Counting(graphed.GraphedForward):
        def __init__(self, *a, **k):
            made.append(1)
            super().__init__(*a, **k)

        def _capture(self):
            captured.append(1)
            super()._capture()

    monkeypatch.setattr(graphed, 'GraphedForward', Counting)
    pipe = PipelinedInference(model, dev, use_cuda_graph=use_graph)
    live = []
    for j, res in enumerate(pipe.run(iter([_host(p) for p in batches]))):
        res['_event'].synchronize()
        _same(f'batch {j} ({STREAM[j]})', res, eager[j], KEYS)
        live.append(res)
        for i in range(max(0, j - 2), j):
            _same(f'batch {i} ({STREAM[i]}) read back while batch {j} is served', live[i], eager[i], KEYS)
    assert len(live) == len(STREAM)
    changes = sum(1 for k in range(len(STREAM)) if k < 3 or _shape(STREAM[k]) != _shape(STREAM[k - 3]))
    print(f'\nuse_cuda_graph={use_graph}: {len(made)} GraphedForward constructions, {len(captured)} captures, '
          f'{changes} shape changes in the slots')
    assert len(made) == (changes if use_graph else 0)
    assert len(captured) == len(made)


# ---- 4. flagged batches inside a graphed stream -----------------------------------------------------------------------

F_SIZES = [(61, 47), (40, 33)]


def _flagged_pairs(kind, seed):
    """'U': pair 0's ligand edges in a random order (not grouped by destination); 'S': all receptor residues of pair 1 at
    one point, so that its receptor keypoints coincide and the SVD guard fires; else an ordinary batch."""
    rng = np.random.default_rng(seed)
    pairs = [tuple(dict(p) for p in synthetic.synthetic_pair(rng, a, b, 10)) for a, b in F_SIZES]
    if kind == 'U':
        lig = pairs[0][0]
        perm = rng.permutation(lig['dst'].shape[0])
        for key in ('src', 'dst', 'he'):
            lig[key] = lig[key][perm]
    if kind == 'S':
        rec = pairs[1][1]
        rec['x'] = np.tile(rec['x'][:1], (rec['x'].shape[0], 1))
    return pairs


def test_flagged_batches_in_a_graphed_stream(dips, cuda_device):
    """Slot 0 of a graphed PipelinedInference captures an ordinary batch, then serves a batch with unsorted edges
    (replay flagged: the eager fallback re-runs it on a destination-sorted plan), a same-shaped batch whose SVD guard
    fires (the fallback replays the reference's host loop) and an ordinary batch.  Every result == the eager forward of
    its batch, the guard's batch under the same CPU-generator state: the fallback must run on the batch's own topology,
    not on the sorted plan the previous fallback left on the slot's graph object."""
    dev = cuda_device
    model, _ = dips
    kinds = ['O', 'P', 'P', 'U', 'P', 'P', 'S', 'P', 'P', 'O']
    batches = [_flagged_pairs(kind, 200 + k) for k, kind in enumerate(kinds)]
    eager = [_eager(model, gio.make_batch(p, dev)) for p in batches]
    assert eager[3]['plan'].edge_perm is not None, 'the unsorted batch did not take the sorting path'
    assert eager[6]['draws'][1] > 0 and all(max(e['draws']) == 0 for k, e in zip(kinds, eager) if k != 'S')
    pipe = PipelinedInference(model, dev, use_cuda_graph=True)
    torch.manual_seed(GUARD_SEED)     # only the guard's batch draws, as its eager forward did from GUARD_SEED
    got = _stream(pipe, [_host(p) for p in batches])
    for k, (res, ref) in enumerate(zip(got, eager)):
        _same(f'batch {k} ({kinds[k]})', res, ref, KEYS)
