"""GPU (H100): every public path of the package called outside the plain context (the default stream of cuda:0, one
host thread) against the same call in the plain context, bit for bit -- the kernels have a fixed reduction order
(DESIGN.md §4.2), so where a call runs must not change a single bit of what it returns:

  1. on a side stream: each path under ``with torch.cuda.stream(s)``, s a new stream;
  2. launched on one stream and resolved on another, busy one: the SVD guard's host loop (IEGMNEngine.resolve_status)
     relaunches the Kabsch kernel and must stay ordered with it;
  3. on a second device: the model and the batch on cuda:1 while cuda:0 stays the current device, with no allocation on
     cuda:0 during the call (skipped with one device);
  4. from two host threads at once, each with its own model, batch and stream (ctypes releases the GIL in the native
     calls, so they really run concurrently), on one device and on two.

A launch on the wrong stream or device raises nothing: it reads inputs that are not written yet and returns a quiet wrong
answer.  So the inputs of every case are late: each is a copy first filled with a poison (v / 2 + 1 for floating-point
values), then overwritten on the stream under test behind a bounded spin of ~30 ms (torch.cuda._sleep).  A kernel queued on that stream reads the real inputs; one queued anywhere else reads the poison, and
the outputs differ.  Each case runs once: the spin makes the ordering deterministic."""
import contextlib
import threading

import numpy as np
import pytest
import torch

import bench
import golden_io as gio
from bench_train import make_targets
from equidock_public_b200 import hetero_graph as hg
from equidock_public_b200 import synthetic
from equidock_public_b200.datasets import DevicePairDataset
from equidock_public_b200.engine import GraphPlan
from equidock_public_b200.eval import Meter_Unbound_Bound
from equidock_public_b200.formats import PairArchive, save_pairs
from equidock_public_b200.graph_build import ResidueBatch, build_graphs
from equidock_public_b200.hetero_graph import CANONICAL_ETYPES, LIGAND, LL, RECEPTOR, RR
from equidock_public_b200.losses import PocketBatch, device_losses
from equidock_public_b200.rigid_docking_model import graph_inputs
from equidock_public_b200.serving import PipelinedInference, _tensors
from equidock_public_b200.training import DataParallelTrainer
from gpu_harness import _device_batch, _model_pairs, _model_targets, _pair_loss, _shard

pytestmark = pytest.mark.gpu

SPIN = 60_000_000        # cycles of torch.cuda._sleep: 30-40 ms at the H100's clocks, far longer than any call's launches
GUARD_SEED = 1234        # torch.manual_seed of every forward whose SVD guard may draw
JOIN_S = 600             # seconds a worker thread may take before the test fails as hung

# proteins of 20 to 200 residues, across the 64- and 128-row tile edges (no 1- or 2-residue protein: their degenerate
# Kabsch is not reproducible from run to run)
RAGGED = [(40, 131), (129, 20), (64, 64), (200, 63), (65, 128), (127, 33)]
RESIDUES = [(60, 80), (100, 50), (129, 64)]
ARCHIVE = [(40, 131, 10), (129, 20, 10), (64, 64, 7), (200, 63, 10), (65, 128, 9)]
DATASET_IDX = [3, 0, 4, 1, 3, 2]


# ---- where a call runs ------------------------------------------------------------------------------------------------

class Ctx:
    """Where a path runs.  'plain': cuda:0 and its default stream.  'side': cuda:0 under ``with torch.cuda.stream(s)``,
    s a new stream.  'cuda1': cuda:1 and its current stream, while cuda:0 stays the current device."""

    def __init__(self, kind):
        self.kind = kind
        self.dev = torch.device('cuda:1' if kind == 'cuda1' else 'cuda:0')
        self.stream = torch.cuda.Stream(self.dev) if kind == 'side' else None

    def scope(self):
        return torch.cuda.stream(self.stream) if self.stream is not None else contextlib.nullcontext()

    def spin(self):
        """Keeps the stream under test busy for ~30 ms."""
        if self.kind != 'plain':
            with self.scope(), torch.cuda.device(self.dev):
                torch.cuda._sleep(SPIN)

    def late(self, *tensors):
        """Copies of device tensors of ``self.dev`` written on the stream under test behind a spin, over a poison
        written before on the current stream: floating-point values v / 2 + 1 (finite, different, residue types still
        in range), integers as they are (an index stays valid).  In the plain context: plain copies."""
        if self.kind == 'plain':
            return [t.clone() for t in tensors]
        poisoned_on = torch.cuda.current_stream(self.dev)
        out = [t * 0.5 + 1 if t.is_floating_point() else t.clone() for t in tensors]
        with self.scope(), torch.cuda.device(self.dev), torch.no_grad():
            s = torch.cuda.current_stream(self.dev)
            s.wait_stream(poisoned_on)
            torch.cuda._sleep(SPIN)
            for o, t in zip(out, tensors):
                o.copy_(t)
                if t.is_cuda:         # both were allocated on another stream: neither may be reused before s is
                    o.record_stream(s)      # past the copy (the caller may drop the source right away)
                    t.record_stream(s)
        return out

    def late_graph(self, g):
        """A PairGraphBatch like the device graph ``g`` whose every tensor is ``late``."""
        new = iter(self.late(*[t for _, t in _tensors(g)]))
        c = hg.PairGraphBatch(g._num_nodes, {et: (next(new), next(new)) for et in CANONICAL_ETYPES},
                              g._batch_num_nodes, g._batch_num_edges)
        for nt in g.ntypes:
            c._ndata[nt] = {k: next(new) for k in g._ndata[nt]}
        for et in CANONICAL_ETYPES:
            c._edata[et] = {k: next(new) for k in g._edata[et]}
        return c

    def fetch(self, outs):
        """The outputs on the host, once everything queued on the device is done (a gradient that is None is left
        out: the key sets are compared)."""
        torch.cuda.synchronize(self.dev)
        return {k: v.detach().cpu().clone() for k, v in outs.items() if v is not None}


def _bits(t):
    t = t.contiguous()
    return t.view({8: torch.int64, 4: torch.int32, 2: torch.int16}[t.element_size()]) if t.is_floating_point() else t


def _same(tag, got, ref):
    assert got.keys() == ref.keys(), (tag, sorted(got), sorted(ref))
    for k in ref:
        a, b = got[k], ref[k]
        assert a.shape == b.shape and a.dtype == b.dtype, (tag, k, a.shape, b.shape, a.dtype, b.dtype)
        if not torch.equal(_bits(a), _bits(b)):
            d = (a.double() - b.double()).abs()
            pytest.fail(f'{tag}: {k} differs from the plain context in {int((_bits(a) != _bits(b)).sum())} of '
                        f'{a.numel()} values, max |diff| = {float(d.nan_to_num(float("inf")).max()):.3e}')


# ---- inputs -----------------------------------------------------------------------------------------------------------

_CACHE = {}


def _cached(key, make):
    if key not in _CACHE:
        _CACHE[key] = make()
    return _CACHE[key]


def _pairs(batch):
    """'ragged': RAGGED with k = 10; 'bench': the benchmark's 330 x (200+200) db5-shaped batch."""
    if batch == 'ragged':
        return _cached('ragged', lambda: [synthetic.synthetic_pair(np.random.default_rng([71, i]), a, b, 10)
                                          for i, (a, b) in enumerate(RAGGED)])
    return _cached('bench', lambda: [synthetic.synthetic_pair(np.random.default_rng([72, i]), a, b, bench.KNN)
                                     for i, (a, b) in enumerate(bench.pair_sizes('db5-shaped', 330))])


def _eval_model(ds, dev):
    return _cached(('model', ds, str(dev)), lambda: gio.build_model(ds, dev))


def _train_batch(dev):
    """The benchmark's 32-pair training batch and its targets on ``dev``."""
    triples = _cached('train', lambda: _shard(0, 1)[0])
    return _device_batch(triples, dev)


def _late_targets(ctx, tgt):
    arrays = ctx.late(tgt.bound_lig, tgt.bound_rec, tgt.pocket_lig, tgt.pocket_rec, tgt.pocket_ptr)
    return PocketBatch.from_device_arrays(*arrays, np.diff(tgt.pocket_ptr.cpu().numpy()).tolist())


def _flagged_pairs(kind, seed):
    """'S': all receptor residues of pair 1 at one point, so that its receptor keypoints coincide and the SVD guard
    fires; else an ordinary batch."""
    rng = np.random.default_rng(seed)
    pairs = [tuple(dict(p) for p in synthetic.synthetic_pair(rng, a, b, 10)) for a, b in [(61, 47), (40, 33)]]
    if kind == 'S':
        rec = pairs[1][1]
        rec['x'] = np.tile(rec['x'][:1], (rec['x'].shape[0], 1))
    return pairs


def _result(res, g=None):
    """The reference's 5-tuple (and the graph's last-layer outputs) as one dict of batched tensors."""
    coors, kp_l, kp_r, rot, trans = res
    out = {'ligand_coors': torch.cat(coors), 'keypts_ligand': torch.stack(kp_l), 'keypts_receptor': torch.stack(kp_r),
           'rotation': torch.stack(rot), 'translation': torch.stack(trans)}
    if g is not None:
        for nt in (LIGAND, RECEPTOR):
            out[f'x_iegmn_out {nt}'] = g.nodes[nt].data['x_iegmn_out']
            out[f'hv_iegmn_out {nt}'] = g.nodes[nt].data['hv_iegmn_out']
    return {k: v.detach().clone() for k, v in out.items()}


# ---- the paths: run(ctx) -> {name: host tensor} -----------------------------------------------------------------------

def _eval_forward(ds, batch):
    def run(ctx):
        model = _eval_model(ds, ctx.dev)
        g = ctx.late_graph(gio.make_batch(_pairs(batch), ctx.dev))
        with ctx.scope(), torch.no_grad():
            out = _result(model(g, 0), g)
        return ctx.fetch(out)
    return run


def _forward_async(ctx):
    model = _eval_model('dips', ctx.dev)
    g = ctx.late_graph(gio.make_batch(_pairs('ragged'), ctx.dev))
    with ctx.scope(), torch.no_grad():
        out = _result(model.forward_async(g).result(), g)
    return ctx.fetch(out)


def _bf16x3(ctx):
    model = _eval_model('dips', ctx.dev)
    g = ctx.late_graph(gio.make_batch(_pairs('ragged'), ctx.dev))
    model.precision = 'bf16x3'
    try:
        with ctx.scope(), torch.no_grad():
            out = _result(model(g, 0), g)
    finally:
        model.precision = 'fp32'
    return ctx.fetch(out)


def _graphed(ctx):
    """Capture and two replays under the stream under test."""
    model = _eval_model('dips', ctx.dev)
    g = ctx.late_graph(gio.make_batch(_pairs('ragged'), ctx.dev))
    out = {}
    with ctx.scope():
        gf = model.graphed(g)
        for rep in range(2):
            out.update({f'{k} replay {rep}': v for k, v in _result(gf.launch().result()).items()})
    return ctx.fetch(out)


def _pipelined(use_cuda_graph):
    def run(ctx):
        model = _eval_model('dips', ctx.dev)
        rng = np.random.default_rng(73)
        shapes = [[(60, 45), (33, 70)], [(90, 20)], [(60, 45), (33, 70)], [(90, 20)], [(60, 45), (33, 70)]]
        hosts = [hg.batch_pairs(synthetic.to_torch_pairs([synthetic.synthetic_pair(rng, a, b, 10) for a, b in s]))
                 .pin_memory() for s in shapes]
        pipe = PipelinedInference(model, ctx.dev, use_cuda_graph=use_cuda_graph)
        out = {}
        ctx.spin()
        with ctx.scope():
            for j, res in enumerate(pipe.run(iter(hosts))):
                res['_event'].synchronize()
                out.update({f'{k} batch {j}': res[k].clone() for k in ('ligand_coors', 'rotation', 'translation')})
        return ctx.fetch(out)
    return run


def _layer_autograd(ctx):
    """IEGMN_Layer.forward of a 64-wide layer as an autograd node (eval mode, inputs requiring grad) and its backward."""
    model = _eval_model('dips', ctx.dev)
    lay = model.iegmn_original.iegmn_layers[1]
    base = gio.make_batch(_pairs('ragged'), ctx.dev)
    N_l, N_r = base.num_nodes(LIGAND), base.num_nodes(RECEPTOR)
    rng = np.random.default_rng(74)
    T = lambda *shape, s=1.0: torch.from_numpy((s * rng.standard_normal(shape)).astype(np.float32)).to(ctx.dev)
    side = lambda n: [T(n, 3, s=10.0), T(n, 64), T(n, 69), None, T(n, 3, s=10.0)]
    ins = side(N_l) + side(N_r)
    ws = [T(N_l, 3), T(N_l, 64), T(N_r, 3), T(N_r, 64)]
    g = ctx.late_graph(base)
    ins[3], ins[8] = g.edges[LL].data['he'], g.edges[RR].data['he']
    late = ctx.late(*[t for i, t in enumerate(ins) if i not in (3, 8)])
    for i in (3, 8):
        late.insert(i, ins[i])
    ins = [t.requires_grad_(True) for t in late]
    lay.zero_grad(set_to_none=True)
    with ctx.scope():
        outs = lay(g, *ins)
        sum((o.double() * w.double()).sum() for o, w in zip(outs, ws)).backward()
    res = {f'out {i}': o.detach() for i, o in enumerate(outs)}
    res.update({f'd input {i}': t.grad for i, t in enumerate(ins)})
    res.update({f'd {n}': p.grad for n, p in lay.named_parameters()})
    out = ctx.fetch(res)
    lay.zero_grad(set_to_none=True)
    return out


def _train_backward(other_stream):
    """Rigid_Body_Docking_Net in training mode with the graph's inputs requiring grad: forward and loss on the stream
    under test, loss.backward() there too, or -- ``other_stream`` -- from another stream while the forward's is busy
    (autograd runs the backward on the forward's stream).  In the plain context both run on the default stream."""
    def run(ctx):
        model = gio.build_model('db5', ctx.dev).train()
        pairs = _model_pairs('db5', 'ragged')
        g = ctx.late_graph(gio.make_batch(pairs, ctx.dev))
        leaves = [t.requires_grad_(True) for t in graph_inputs(g)]
        torch.manual_seed(GUARD_SEED)
        with ctx.scope():
            coors, kp_l, kp_r, rot, trans = model(g, 0)
            loss = _pair_loss(coors, (kp_l, kp_r), _model_targets(pairs), [len(l['res_feat']) for l, _ in pairs])
        if other_stream and ctx.kind != 'plain':
            ctx.spin()
            with torch.cuda.stream(torch.cuda.Stream(ctx.dev)):
                loss.backward()
        else:
            with ctx.scope():
                loss.backward()
        torch.cuda.synchronize(ctx.dev)
        res = _result((coors, kp_l, kp_r, rot, trans))
        res['loss'] = loss.detach()
        res.update({f'd input {i}': t.grad for i, t in enumerate(leaves)})
        res.update({f'd {n}': p.grad for n, p in model.named_parameters()})
        return ctx.fetch(res)
    return run


def _trainer(ctx):
    """Two DataParallelTrainer.steps (world = 1) on the benchmark's 32-pair training batch."""
    model = gio.build_model('db5', ctx.dev)
    trainer = DataParallelTrainer(model, lr=1e-3)
    g0, tgt0 = _train_batch(ctx.dev)
    g, tgt = ctx.late_graph(g0), _late_targets(ctx, tgt0)
    res = {}
    with ctx.scope():
        for step in range(2):
            r = trainer.step(g, tgt)
            res.update({f'loss {step}': r['loss'].clone(), f'grad_norm {step}': r['grad_norm'].clone(),
                        f'err {step}': r['err'].clone()})
    res.update(flat_w=trainer.flat_w, m=trainer.m, v=trainer.v)
    return ctx.fetch(res)


def _losses(ctx):
    g0, tgt0 = _train_batch(ctx.dev)
    plan = GraphPlan.from_graph(g0, ctx.dev, 10)
    rng = np.random.default_rng(75)
    pred = tgt0.bound_lig + torch.from_numpy(rng.normal(0, 2, (plan.N_l, 3)).astype(np.float32)).to(ctx.dev)
    kp = torch.from_numpy(rng.normal(0, 10, (2 * plan.n_pairs, 50, 3))).to(ctx.dev)
    pred, kp = ctx.late(pred, kp)
    tgt = _late_targets(ctx, tgt0)
    with ctx.scope():
        r = device_losses(plan, pred, kp, tgt, 1.0, 10.0, 25.0, 10.0)
    return ctx.fetch({k: r[k] for k in ('total', 'parts', 'dcoors', 'dkeypts', 'err')})


def _meter(ctx):
    g0, _ = _train_batch(ctx.dev)
    plan = GraphPlan.from_graph(g0, ctx.dev, 10)
    rng = np.random.default_rng(76)
    T = lambda n: torch.from_numpy(rng.normal(0, 20, (n, 3)).astype(np.float32)).to(ctx.dev)
    coords = ctx.late(T(plan.N_l), T(plan.N_r), T(plan.N_l), T(plan.N_r))
    meter = Meter_Unbound_Bound()
    with ctx.scope():
        out = meter.update_rmsd_batch(plan, *coords)
    return ctx.fetch({'rmsd': out, 'lists': torch.tensor([meter.complex_rmsd_list, meter.ligand_rmsd_list,
                                                          meter.receptor_rmsd_list], dtype=torch.float64)})


def _graph_build(ctx):
    rng = np.random.default_rng(77)
    rb = ResidueBatch([synthetic.synthetic_residue_pair(rng, a, b) for a, b in RESIDUES])
    keys = list(rb.t)
    inputs = dict(zip(keys, ctx.late(*[rb.t[k].to(ctx.dev) for k in keys])))
    with ctx.scope():
        g = build_graphs(rb, ctx.dev, dev_inputs=inputs)
    plan = g._eqd_plan
    res = {f'graph {k}': t for k, t in _tensors(g)}
    res.update({f'plan {k}': getattr(plan, k) for k in ('row_ptr', 'col_src', 'edge_dst', 'seg_ptr', 'node_tiles')})
    return ctx.fetch(res)


@pytest.fixture(scope='module', autouse=True)
def _archive(tmp_path_factory):
    """The pair archive of the DevicePairDataset cases, written once for the module."""
    rng = np.random.default_rng(78)
    pairs, labels = [], []
    for n_l, n_r, k in ARCHIVE:
        lig, rec = synthetic.synthetic_protein(rng, n_l, k), synthetic.synthetic_protein(rng, n_r, k)
        R, t = synthetic.random_rigid(rng)
        lig['new_x'] = ((R @ lig['x'].T).T + t).astype(np.float32)
        tg = make_targets((lig, rec), rng)
        pairs.append((lig, rec))
        labels.append({'pocket_coors': tg['pocket_lig'], 'bound_lig': tg['bound_lig'], 'bound_rec': tg['bound_rec']})
    path = tmp_path_factory.mktemp('streams') / 'pairs.eqd'
    save_pairs(str(path), pairs, labels)
    _CACHE['archive'] = PairArchive(str(path))
    yield
    _CACHE.clear()


def _dataset(repose):
    """DevicePairDataset.batch with the stream under test busy: the batch's offsets are uploaded and assembled there."""
    def run(ctx):
        ds = _cached(('dataset', str(ctx.dev)), lambda: DevicePairDataset(_CACHE['archive'], ctx.dev))
        torch.cuda.synchronize(ctx.dev)
        ctx.spin()
        with ctx.scope():
            g, tgt = ds.batch(DATASET_IDX, seed=9 if repose else None, step=2)
        plan = g._eqd_plan
        res = {f'graph {k}': t for k, t in _tensors(g)}
        res.update({f'plan {k}': getattr(plan, k) for k in ('row_ptr', 'col_src', 'edge_dst', 'seg_ptr', 'node_tiles',
                                                              'he_l', 'he_r')})
        res.update({f'target {k}': getattr(tgt, k) for k in ('bound_lig', 'bound_rec', 'pocket_lig', 'pocket_rec',
                                                               'pocket_ptr')})
        res.update({'rigid R': g.rigid[0], 'rigid t': g.rigid[1]})
        return ctx.fetch(res)
    return run


PATHS = {
    'eval-db5-ragged': _eval_forward('db5', 'ragged'),
    'eval-db5-bench': _eval_forward('db5', 'bench'),
    'eval-dips-ragged': _eval_forward('dips', 'ragged'),
    'eval-dips-bench': _eval_forward('dips', 'bench'),
    'forward_async': _forward_async,
    'bf16x3': _bf16x3,
    'graphed': _graphed,
    'pipelined-graphs': _pipelined(True),
    'pipelined-eager': _pipelined(False),
    'layer-autograd': _layer_autograd,
    'train-backward': _train_backward(False),
    'train-backward-other-stream': _train_backward(True),
    'trainer-two-steps': _trainer,
    'device_losses': _losses,
    'rmsd-meter': _meter,
    'build_graphs': _graph_build,
    'dataset-reposed': _dataset(True),
    'dataset-as-stored': _dataset(False),
}
_REF = {}


def _reference(name):
    """The path in the plain context, once per module."""
    if name not in _REF:
        _REF[name] = PATHS[name](Ctx('plain'))
    return _REF[name]


# ---- 1. side stream ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('name', list(PATHS))
def test_side_stream_matches_plain_context(name, cuda_device):
    ref = _reference(name)
    _same(f'{name} on a side stream', PATHS[name](Ctx('side')), ref)


# ---- 2. launch and resolve on different streams -----------------------------------------------------------------------

@pytest.mark.parametrize('kind,busy', [('guard', 'resolve'), ('guard', 'launch'), ('ordinary', 'resolve'),
                                       ('graphed guard', 'resolve')])
def test_resolve_on_another_stream(kind, busy, cuda_device):
    """forward_async (or a graphed launch) under stream A, .result() under stream B, with B ('resolve') or A ('launch')
    spinning meanwhile: the SVD guard's loop must perturb the covariance, relaunch the Kabsch kernel and read its status
    in one order whichever stream is busy.  Rotations, translations, ligand coordinates, keypoints and the guard's draws
    == the eager forward from the same torch.manual_seed."""
    dev = cuda_device
    model = _eval_model('dips', dev)
    pairs = _flagged_pairs('O' if kind == 'ordinary' else 'S', 301)
    torch.manual_seed(GUARD_SEED)
    with torch.no_grad():
        ref = _result(model(gio.make_batch(pairs, dev), 0))
    ref_draws = list(model.iegmn_original.last_outputs['guard_draws'])
    assert (ref_draws[1] > 0) == (kind != 'ordinary') and ref_draws[0] == 0, ref_draws
    g = gio.make_batch(pairs, dev)
    a, b = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
    if kind == 'graphed guard':
        with torch.cuda.stream(a):
            gf = model.graphed(g)
    torch.cuda.synchronize()
    torch.manual_seed(GUARD_SEED)
    with torch.cuda.stream(a), torch.no_grad():
        pending = gf.launch() if kind == 'graphed guard' else model.forward_async(g)
        if busy == 'launch':
            torch.cuda._sleep(SPIN)
    with torch.cuda.stream(b):
        if busy == 'resolve':
            torch.cuda._sleep(SPIN)
        got = _result(pending.result())
    draws = list(model.iegmn_original.last_outputs['guard_draws'])
    torch.cuda.synchronize()
    print(f'\n{kind}: guard draws {draws} (eager {ref_draws})')
    assert draws == ref_draws, (kind, draws, ref_draws)
    _same(f'{kind}: resolved on another stream', {k: v.cpu() for k, v in got.items()},
          {k: v.cpu() for k, v in ref.items()})


# ---- 3. second device -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('name', list(PATHS))
def test_second_device_matches_cuda0(name, cuda_device):
    """The path on cuda:1 while cuda:0 is the current device: the same bits as on cuda:0 (the same hardware), and not one
    byte allocated on cuda:0 meanwhile (peak of torch's allocator over the call)."""
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two CUDA devices')
    ref = _reference(name)
    torch.cuda.synchronize(0)
    torch.cuda.reset_peak_memory_stats(0)
    before = torch.cuda.memory_allocated(0)
    got = PATHS[name](Ctx('cuda1'))
    assert torch.cuda.current_device() == 0
    assert torch.cuda.max_memory_allocated(0) <= before, \
        f'{name}: {torch.cuda.max_memory_allocated(0) - before} bytes allocated on cuda:0 by a call on cuda:1'
    _same(f'{name} on cuda:1', got, ref)


# ---- 4. concurrent host threads ---------------------------------------------------------------------------------------

def _thread_work(model, g, stream):
    """3 eager forwards and 2 forward_async round trips of one model on ``stream``."""
    out = {}
    with torch.cuda.stream(stream), torch.no_grad():
        for i in range(3):
            out.update({f'{k} eager {i}': v for k, v in _result(model(g, 0)).items()})
        for i in range(2):
            out.update({f'{k} async {i}': v for k, v in _result(model.forward_async(g).result()).items()})
        stream.synchronize()
    return {k: v.cpu() for k, v in out.items()}


@pytest.mark.parametrize('devices', ['cuda0-twice', 'cuda0-and-cuda1'])
def test_concurrent_threads_match_serial(devices, cuda_device):
    """Two host threads, each with its own model (packed on first use, inside the thread), batch and stream, start
    together at a barrier: every output == the same work run serially on the devices' default streams."""
    devs = [torch.device('cuda:0'), torch.device('cuda:0' if devices == 'cuda0-twice' else 'cuda:1')]
    if devs[1].index >= torch.cuda.device_count():
        pytest.skip('needs two CUDA devices')
    rng = np.random.default_rng(79)
    pairs = [[synthetic.synthetic_pair(rng, a, b, 10) for a, b in sizes]
             for sizes in ([(120, 90), (64, 130), (200, 45)], [(77, 150), (129, 64)])]
    serial = [_thread_work(gio.build_model('dips', d), gio.make_batch(p, d), torch.cuda.default_stream(d))
              for d, p in zip(devs, pairs)]
    models = [gio.build_model('dips', d) for d in devs]
    graphs = [gio.make_batch(p, d) for d, p in zip(devs, pairs)]
    streams = [torch.cuda.Stream(d) for d in devs]
    torch.cuda.synchronize()
    barrier = threading.Barrier(2, timeout=JOIN_S)
    got, errors = [None, None], []

    def worker(i):
        try:
            barrier.wait()
            got[i] = _thread_work(models[i], graphs[i], streams[i])
        except BaseException as e:       # reported by the main thread
            errors.append((i, e))
            barrier.abort()

    threads = [threading.Thread(target=worker, args=(i,), daemon=True) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(JOIN_S)
    assert not any(t.is_alive() for t in threads), f'a worker thread did not finish within {JOIN_S} s'
    assert not errors, errors
    for i in range(2):
        _same(f'thread {i} on {devs[i]}', got[i], serial[i])
