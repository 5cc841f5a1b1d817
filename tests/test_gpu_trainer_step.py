"""GPU (H100): the fused training step DataParallelTrainer.step -- forward with stash, device losses, CUDA backward into
one flat gradient, per-bucket all-reduce on a side stream, eqd_sqnorm_partials + eqd_clip_adam; what
``bench.py --workload train`` times -- against fp64, at the benchmark's own training batch: 32 DIPS-shaped pairs
(bench.make_pairs, seed 0; 17 407 nodes, most proteins past the resident-attention bound) on the 5-layer weight-shared
DB5 model with the benchmark's hyperparameters.

  - test_trainer_steps_match_fp64: 3 steps on one rank, clipping inactive and active.  Each step is compared with an fp64
    restatement evaluated at the weights the step started from (heads_ref.model_forward with the engine's guard draws,
    the losses of loss_oracle.batch_loss with the device's certified transport plans held constant); Adam is checked per
    element from the kernel's own inputs; the alignment padding stays 0; the step's forward equals, bit for bit, a fresh
    model's forward at the same weights (no stale packed weights).
  - test_buckets_are_final_when_reported: TrainEngine.backward's on_bucket_done contract, which the all-reduce overlap
    relies on.
  - test_two_ranks_match_fp64: world = 2 (NCCL with two devices, else gloo with both ranks on one device).
  - test_clip_adam_kernels_vs_fp64: eqd_sqnorm_partials + eqd_clip_adam per element against fp64 from their own inputs.

Bounds.  Model-level comparisons use those of tests/test_gpu_layer_norm_options.py: _grad_mismatches for the gradients and
the gradient norm, _coord_bound for coordinates, 1e-3 relative for the loss and its parts.  The optimizer kernels are held
per element to bounds counted from their fp32 operations (_adam_ref)."""
import ctypes as C
import datetime
import math
import os
import socket
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import bench
import bench_train
import golden_io as gio
import heads_ref as hr
import loss_oracle as lo
from equidock_public_b200 import _native as nat
from equidock_public_b200 import hetero_graph as hg
from equidock_public_b200 import synthetic
from equidock_public_b200.losses import PocketBatch, check_loss_status, device_losses
from equidock_public_b200.training import DataParallelTrainer, ParamLayout, TrainEngine
from test_gpu_dropout import _oracle_inputs, _pairs
from test_gpu_layer_norm_options import _coord_bound, _fp64_state, _grad_mismatches

pytestmark = pytest.mark.gpu
U = 2.0 ** -24                         # unit roundoff of fp32
LR, WD, BETAS, EPS = 1e-4, 1e-4, (0.9, 0.999), 1e-8     # bench_train.run's hyperparameters
SEEDS = (31, 32, 33)                   # torch.manual_seed before each step (the SVD guard draws from the CPU generator)
OUT_KEYS = ('ligand_coors', 'keypts', 'rotation', 'translation', 'h', 'x64')


# ---- the benchmark's batch ----------------------------------------------------------------------------------------------

def _shard(rank, world):
    """This rank's shard of the benchmark's 32-pair training batch with its targets: (triples, (lo, hi))."""
    args = types.SimpleNamespace(workload='train', pairs_per_gpu=32 // world, seed=0)
    triples, shard, sizes = bench_train.make_train_pairs(args, rank, world, bench)
    assert sizes == bench.pair_sizes('train', 32)
    return triples, shard


def _device_batch(triples, dev):
    g = hg.batch_pairs(synthetic.to_torch_pairs([(t[0], t[1]) for t in triples])).to(dev)
    tl = lambda key: [torch.from_numpy(t[2][key]) for t in triples]
    return g, PocketBatch(tl('bound_lig'), tl('bound_rec'), tl('pocket_lig'), tl('pocket_rec'), dev)


def _loss_args(margs):
    return (float(margs.get('pocket_ot_loss_weight', 1.0)), float(margs.get('intersection_loss_weight', 10.0)),
            float(margs.get('intersection_sigma', 25.0)), float(margs.get('intersection_surface_ct', 10.0)))


def _trainer(model, clip, margs, world=1):
    la = _loss_args(margs)
    return DataParallelTrainer(model, lr=LR, weight_decay=WD, clip=clip, betas=BETAS, eps=EPS, world=world,
                               pocket_ot_loss_weight=la[0], intersection_loss_weight=la[1], intersection_sigma=la[2],
                               intersection_surface_ct=la[3])


def _model_at(w, dev):
    """A fresh DB5 model in training mode whose parameters are the flat weights ``w`` (a ParamLayout buffer)."""
    model = gio.build_model('db5', dev).train()
    layout = ParamLayout(model)
    with torch.no_grad():
        for p, v in zip(layout.params, layout.views(w.to(dev))):
            p.copy_(v)
    return model


def _padding(layout, dev):
    """Boolean mask of the flat layout's alignment padding."""
    pad = torch.ones(layout.total, dtype=torch.bool)
    for p in layout.params:
        pad[layout.offset[id(p)]:layout.offset[id(p)] + p.numel()] = False
    return pad.to(dev)


# ---- fp64 restatement of one step --------------------------------------------------------------------------------------

def _flows(res, triples):
    """The device's integer transport plans of a device_losses result, one (N_pocket, K) array per pair."""
    x, out, p0 = res['plan'].cpu().numpy(), [], 0
    for t in triples:
        n = len(t[2]['pocket_lig'])
        out.append(x[p0:p0 + n])
        p0 += n
    return out


def _certify(flows, keypts, triples):
    """loss_oracle.ot_certify on every pair's plan against the cost of the keypoints the device solved for."""
    Y = keypts.detach().cpu().numpy()
    B = len(triples)
    for b, t in enumerate(triples):
        cost = lo.sq_dist_mat(t[2]['pocket_lig'], Y[b]) + lo.sq_dist_mat(t[2]['pocket_rec'], Y[B + b])
        lo.ot_certify(cost, flows[b])


def _fp64_loss(co, Y, flows, triples, n_lig, la):
    """loss_oracle.batch_loss in torch fp64 with the transport plans ``flows`` held constant (src/utils/ot_utils.py:27):
    per-pair MSE, OT and intersection losses, each averaged over the pairs.  Returns (total, (mse, ot, inter))."""
    w_ot, w_int, sigma, ct = la
    B, K = len(triples), Y.shape[1]
    T64 = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    G = lambda prot, x: -sigma * torch.log(1e-3 + torch.exp(-((prot[None] - x[:, None]) ** 2).sum(2) / sigma).sum(1))
    mse = ot = inter = 0.0
    off = 0
    for b, (_, _, t) in enumerate(triples):
        p = co[off:off + n_lig[b]]
        off += n_lig[b]
        mse = mse + ((p - T64(t['bound_lig'])) ** 2).mean()
        pl, pr = T64(t['pocket_lig']), T64(t['pocket_rec'])
        cost = ((pl[:, None] - Y[b][None]) ** 2).sum(2) + ((pr[:, None] - Y[B + b][None]) ** 2).sum(2)
        ot = ot + (T64(flows[b].astype(np.float64) / (len(pl) * K)) * cost).sum()
        rec = T64(t['bound_rec'])
        inter = inter + torch.clamp(ct - G(rec, p), min=0).mean() + torch.clamp(ct - G(p, rec), min=0).mean()
    mse, ot, inter = mse / B, ot / B, inter / B
    return mse + w_ot * ot + w_int * inter, (mse, ot, inter)


def _fp64_step(model_t, inp, n_lig, draws, flows, triples, seed, margs):
    """Loss, coordinates and gradients of one step in fp64 at the parameters of ``model_t``, the guard's noise replayed
    from torch.manual_seed(seed) with the engine's draw count per pair asserted.  Gradients by parameter name
    (model.named_parameters: weight-shared layers once, summed)."""
    sd = _fp64_state(model_t, requires_grad=True)
    _, rand_diag = hr.replay_draws(seed)
    co, Y, _, _, d = hr.model_forward(sd, margs, inp, None, rand_diag)
    assert list(d) == list(draws), (d, draws)
    total, parts = _fp64_loss(co, Y, flows, triples, n_lig, _loss_args(margs))
    total.backward()
    grads = {}
    for n, q in model_t.named_parameters():
        gr = sd[n].grad
        grads[n] = gr.numpy() if gr is not None else np.zeros(tuple(q.shape))
    norm = math.sqrt(sum(float((v ** 2).sum()) for v in grads.values()))
    return {'loss': total.item(), 'parts': [float(x.detach()) for x in parts], 'coors': co.detach().numpy(), 'grads': grads,
            'norm': norm}


def _clip_factor(clip, norm):
    return min(1.0, float(np.float32(clip)) / (norm + float(np.float32(1e-6))))


def _flat_by_name(model, layout, flat):
    by_id = {id(p): v for p, v in zip(layout.params, layout.views(flat))}
    return {n: by_id[id(q)].double().cpu().numpy() for n, q in model.named_parameters()}


def _short(n):
    return n.replace('iegmn_original.', '').replace('iegmn_layers.', 'L')


def _check_model_level(tag, got_loss, got_norm, got_coors, got_grads, ref, clip):
    """loss, its parts, the gradient norm, the coordinates and every clipped gradient against the fp64 step ``ref``;
    prints each as a fraction of its bound (per tensor for the gradients)."""
    c = _clip_factor(clip, ref['norm'])
    refs = [ref['loss']] + ref['parts']
    names = ('loss', 'mse', 'ot', 'inter')
    frac = {k: abs(float(got_loss[i]) - refs[i]) / (1e-3 * abs(refs[i])) if refs[i] else abs(float(got_loss[i]))
            for i, k in enumerate(names)}
    nbad = _grad_mismatches({'norm': np.array([got_norm])}, {'norm': np.array([ref['norm']])})
    frac['norm'] = abs(got_norm - ref['norm']) / ((3e-3 + 2e-6) * ref['norm'])
    if got_coors is not None:
        frac['coors'] = float(np.abs(got_coors - ref['coors']).max()) / _coord_bound(ref['coors'])
    rg = {n: v * c for n, v in ref['grads'].items()}
    gmax = max(np.abs(v).max() for v in rg.values())
    per = {n: float(np.abs(got_grads[n] - rg[n]).max()) / (3e-3 * np.abs(rg[n]).max() + 2e-6 * gmax) for n in rg}
    print(f'\n{tag}: loss {float(got_loss[0]):.6g} (fp64 {ref["loss"]:.6g}), |g| {got_norm:.6g} (fp64 {ref["norm"]:.6g}), '
          f'clip factor {c:.4g}; fractions of the bounds: ' + ', '.join(f'{k} {v:.2e}' for k, v in frac.items()))
    print(f'{tag}: gradients, fractions of the bounds: '
          + ', '.join(f'{_short(n)} {v:.1e}' for n, v in sorted(per.items(), key=lambda kv: -kv[1])))
    bad = {k: v for k, v in frac.items() if not v <= 1}
    assert not bad and not nbad, (bad, nbad)
    gbad = _grad_mismatches(got_grads, rg)
    assert not gbad, gbad
    return c


# ---- Adam from the kernel's own inputs ------------------------------------------------------------------------------

def _adam_ref(w0, m0, v0, g, step, lr=LR, betas=BETAS, eps=EPS, wd=WD):
    """torch.optim.Adam's L2 step (weight decay added to the gradient) in fp64 from the kernel's inputs, with the fp32
    values of the hyperparameters the kernel receives; ``g`` is the clipped, scaled gradient the kernel left in its g.
    Returns (w, m, v) and per-element bounds on the kernel's error, counted from its fp32 operations to first order:
      gi = fmaf(wd, w, g)                        1 rounding
      m  = b1 m0 + (1 - b1) gi                   3 more (1 - b1 is exact)     -> 4u (b1 |m0| + (1 - b1) |gi|)
      v  = b2 v0 + (1 - b2) gi gi                2 from gi, 4 more           -> 6u v (all terms positive)
      bc = 1 - powf(b, step) on the host         powf within 1 ulp, amplified by b^t / (1 - b^t) in the difference
      w -= (lr / bc1) (m / (sqrt(v) / sqrt(bc2) + eps))
           denominator: 3u from v, 4 roundings, half of bc2's error; lr / bc1, the quotient and the product 3u;
           m's absolute error over the denominator; the final subtraction u |w|.
    1 % on top of every bound covers the second-order terms."""
    f32 = lambda x: float(np.float32(x))
    b1, b2, lr, eps, wd = f32(betas[0]), f32(betas[1]), f32(lr), f32(eps), f32(wd)
    w0, m0, v0, g = (t.double() for t in (w0, m0, v0, g))
    gi = g + wd * w0
    m = b1 * m0 + (1 - b1) * gi
    v = b2 * v0 + (1 - b2) * gi * gi
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    denom = v.sqrt() / math.sqrt(bc2) + eps
    upd = (lr / bc1) * m / denom
    w = w0 - upd
    rbc = lambda b: U * (2 * b ** step / (1 - b ** step) + 1)
    e_m = 4 * U * (b1 * m0.abs() + (1 - b1) * gi.abs())
    e_v = 6 * U * v
    r_den = 7 * U + 0.5 * rbc(b2)
    e_w = U * w.abs() + (lr / bc1) * e_m / denom + upd.abs() * (r_den + rbc(b1) + 3 * U)
    return (w, m, v), tuple(1.01 * e for e in (e_w, e_m, e_v))


def _worst_fraction(got, ref, bound):
    """max over elements of |got - ref| / bound; an element with a zero bound must be exact (else inf)."""
    err = (got.double() - ref).abs()
    frac = torch.where(bound > 0, err / bound.clamp(min=1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(frac.max())


def _adam_fractions(w0, m0, v0, g, w1, m1, v1, step, **hp):
    """Worst |kernel - fp64| / bound of w, m and v (see _adam_ref)."""
    refs, bounds = _adam_ref(w0, m0, v0, g, step, **hp)
    return {k: _worst_fraction(got, ref, b) for k, got, ref, b in zip('wmv', (w1, m1, v1), refs, bounds)}


# ---- 1. several steps on one rank ---------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def bench_batch(cuda_device):
    """The benchmark's batch, and step 1 of the fp64 restatement at the checkpoint weights (its norm sets the active
    clip; both clip variants start from it)."""
    triples, shard = _shard(0, 1)
    assert shard == (0, 32)
    g, tgt = _device_batch(triples, cuda_device)
    margs = gio.load_args('db5')
    model = gio.build_model('db5', cuda_device).train()
    torch.manual_seed(SEEDS[0])
    fwd = TrainEngine(model).forward(g)
    plan = fwd['plan']
    assert plan.N == 17407 and plan.n_pairs == 32 and plan.edge_perm is None, (plan.N, plan.n_pairs)
    res = device_losses(plan, fwd['ligand_coors'], fwd['keypts'], tgt, *_loss_args(margs))
    check_loss_status(res)
    flows = _flows(res, triples)
    _certify(flows, fwd['keypts'], triples)
    ref = _fp64_step(model, _oracle_inputs(g, plan), plan.n_lig_list, fwd['guard_draws'], flows, triples, SEEDS[0], margs)
    out = {k: fwd[k].clone() for k in OUT_KEYS}
    return {'triples': triples, 'g': g, 'tgt': tgt, 'margs': margs, 'fwd1': out, 'flows1': flows, 'ref1': ref}


@pytest.mark.parametrize('clipping', ['inactive', 'active'])
def test_trainer_steps_match_fp64(clipping, bench_batch, cuda_device):
    """3 steps of DataParallelTrainer.step (world 1) on the benchmark's batch: loss and parts, grad_norm, coordinates and
    the clipped gradient in flat_g against the fp64 step at the step's starting weights W_t; the transport plan of
    device_losses re-run on the step's outputs reproduces the step's loss bit for bit and is certified optimal; Adam per
    element from the kernel's inputs; the padding of flat_w, flat_g, m and v stays 0; the step's forward equals a fresh
    model's forward at W_t bit for bit.  clip: 1e30 (inactive), or half the fp64 norm of step 1 (active)."""
    bb, dev = bench_batch, cuda_device
    triples, g, tgt, margs = bb['triples'], bb['g'], bb['tgt'], bb['margs']
    clip = 1e30 if clipping == 'inactive' else 0.5 * bb['ref1']['norm']
    tr = _trainer(gio.build_model('db5', dev), clip, margs)
    pad = _padding(tr.layout, dev)
    assert int(pad.sum()) == tr.layout.total - tr.layout.n_param_elements > 0
    for t, seed in enumerate(SEEDS):
        w0, m0, v0 = tr.flat_w.clone(), tr.m.clone(), tr.v.clone()
        torch.manual_seed(seed)
        r = tr.step(g, tgt)
        check_loss_status(r)
        loss, norm = r['loss'].clone(), float(r['grad_norm'][0])     # grad_norm: the next step overwrites it
        g1, w1, m1, v1 = tr.flat_g.clone(), tr.flat_w.clone(), tr.m.clone(), tr.v.clone()
        fwd = r['fwd']
        plan = fwd['plan']
        again = device_losses(plan, fwd['ligand_coors'], fwd['keypts'], tgt, *_loss_args(margs))
        assert torch.equal(again['total'], loss)
        flows = _flows(again, triples)
        _certify(flows, fwd['keypts'], triples)
        if t == 0:
            other, ref = bb['fwd1'], bb['ref1']
            assert all(np.array_equal(a, b) for a, b in zip(flows, bb['flows1']))
        else:
            fresh = _model_at(w0, dev)
            torch.manual_seed(seed)
            other = TrainEngine(fresh).forward(g)
            ref = _fp64_step(fresh, _oracle_inputs(g, plan), plan.n_lig_list, fwd['guard_draws'], flows, triples, seed,
                             margs)
        stale = [k for k in OUT_KEYS if not torch.equal(fwd[k], other[k])]
        assert not stale, f'step {t + 1}: the step\'s forward differs from a fresh model at W_t in {stale}'
        tag = f'clip {clipping} step {t + 1}'
        got = _flat_by_name(tr.model, tr.layout, g1)
        c = _check_model_level(tag, loss.cpu().numpy(), norm, fwd['ligand_coors'].double().cpu().numpy(), got, ref, clip)
        assert (c < 1) == (clipping == 'active')
        fr = _adam_fractions(w0, m0, v0, g1, w1, m1, v1, t + 1)
        print(f'{tag}: Adam per element, fractions of the bounds: ' + ', '.join(f'{k} {v:.2e}' for k, v in fr.items()))
        assert all(v <= 1 for v in fr.values()), fr
        for name, buf in (('flat_w', w1), ('flat_g', g1), ('m', m1), ('v', v1)):
            assert not bool(buf[pad].any()), f'{tag}: padding of {name} is not 0'


# ---- 2. buckets are final when reported --------------------------------------------------------------------------------

BUCKET_CASES = [('db5', 'bench', False, 0.0), ('dips', 'bench', False, 0.0), ('db5', 'ragged3', True, 0.0),
                ('dips', 'ragged3', True, 0.0), ('dips', 'ragged3', False, 0.25)]


@pytest.mark.parametrize('ds,batch,inputs,p', BUCKET_CASES)
def test_buckets_are_final_when_reported(ds, batch, inputs, p, cuda_device):
    """TrainEngine.backward(on_bucket_done=...): a copy of flat[lo:hi] taken on the compute stream when a bucket is
    reported equals the final buffer bit for bit (no later kernel writes into a reported bucket, which would race with
    its all-reduce); every bucket is reported once, in layout.buckets order, and the buckets tile [0, total).  DB5's
    shared layers report at their first forward use; inputs: the input-gradient kernels run after the buckets are
    reported; p > 0: the dropout head backward."""
    dev = cuda_device
    args = gio.load_args(ds)
    args['dropout'] = p
    model = gio.build_model(ds, dev, args=args).train()
    if batch == 'bench':
        g = _device_batch(_shard(0, 1)[0], dev)[0]
    else:
        g = gio.make_batch(_pairs(ds, batch), dev)
    eng = TrainEngine(model)
    torch.manual_seed(5)
    fwd = eng.forward(g)
    assert (fwd.get('dropout_head') is not None) == (p > 0)
    gen = torch.Generator(device=dev).manual_seed(6)
    d_coors = torch.randn(fwd['ligand_coors'].shape, device=dev, generator=gen)
    d_keypts = torch.randn(fwd['keypts'].shape, device=dev, generator=gen, dtype=torch.float64)
    flat = torch.zeros(eng.layout.total, device=dev)
    seen = []
    ins = {} if inputs else None
    eng.backward(fwd, d_coors, d_keypts, flat=flat,
                 on_bucket_done=lambda lab, lo_, hi: seen.append((lab, lo_, hi, flat[lo_:hi].clone())), inputs_out=ins)
    torch.cuda.synchronize()
    assert [s[:3] for s in seen] == list(eng.layout.buckets)
    bk = eng.layout.buckets
    assert bk[0][1] == 0 and bk[-1][2] == eng.layout.total and all(bk[i][2] == bk[i + 1][1] for i in range(len(bk) - 1))
    if inputs:
        assert set(ins) == {'x_lig', 'x_rec', 'mu_lig', 'mu_rec', 'he_lig', 'he_rec'}
    changed = {lab: int((c != flat[lo_:hi]).sum()) for lab, lo_, hi, c in seen}
    print(f'\nbuckets {ds} {batch} inputs={inputs} p={p}: ' + ', '.join(f'{lab} [{lo_}, {hi})' for lab, lo_, hi, _ in seen)
          + f'; elements changed after their report: {changed}')
    assert all(v == 0 for v in changed.values()), changed
    assert all(bool(c.abs().sum() > 0) for _, _, _, c in seen)


# ---- 3. two ranks -------------------------------------------------------------------------------------------------------

TWO_RANK_STEPS = 2
TWO_RANK_CLIP = 100.0                  # bench_train.run's clip


def _rank_worker(rank, world, port, out_dir, backend):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dev = torch.device('cuda', rank if backend == 'nccl' else 0)
    torch.cuda.set_device(dev)
    kw = {'device_id': dev} if backend == 'nccl' else {}
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300), **kw)
    try:
        triples, shard = _shard(rank, world)
        g, tgt = _device_batch(triples, dev)
        margs = gio.load_args('db5')
        tr = _trainer(gio.build_model('db5', dev), TWO_RANK_CLIP, margs, world)
        assert tr.engine.rank == rank
        out = {'shard': shard, 'steps': []}
        for seed in SEEDS[:TWO_RANK_STEPS]:
            w0 = tr.flat_w.clone()
            torch.manual_seed(seed)
            r = tr.step(g, tgt)
            check_loss_status(r)
            fwd = r['fwd']
            plan = fwd['plan']
            assert plan.edge_perm is None
            again = device_losses(plan, fwd['ligand_coors'], fwd['keypts'], tgt, *_loss_args(margs))
            assert torch.equal(again['total'], r['loss'])
            out['steps'].append({'w0': w0.cpu(), 'w1': tr.flat_w.cpu(), 'g1': tr.flat_g.cpu(),
                                 'norm': float(r['grad_norm'][0]), 'loss': r['loss'].cpu().numpy(),
                                 'inp': _oracle_inputs(g, plan), 'n_lig': list(plan.n_lig_list),
                                 'draws': list(fwd['guard_draws']), 'flows': _flows(again, triples),
                                 'keypts': fwd['keypts'].cpu(), 'coors': fwd['ligand_coors'].double().cpu().numpy()})
        torch.save(out, os.path.join(out_dir, f'rank{rank}.pt'))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_two_ranks_match_fp64(cuda_device, tmp_path):
    """DataParallelTrainer(world=2) over the benchmark's 32 pairs sharded as bench.make_pairs shards them (15 and 17
    pairs), 2 steps: flat_w (padding included) bitwise equal across ranks after each step; grad_norm and the clipped
    gradient against the fp64 reference, which with unequal shards is the mean over ranks of each rank's mean-loss
    gradient (training.py: each rank normalises by its own pair count).  Two devices: NCCL, one device per rank; one
    device: gloo with both ranks on it.  A rank that fails ends the other (mp.spawn), and both have exited on return."""
    world = 2
    backend = 'nccl' if torch.cuda.device_count() >= world else 'gloo'
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    mp.spawn(_rank_worker, args=(world, port, str(tmp_path), backend), nprocs=world, join=True)
    outs = [torch.load(os.path.join(str(tmp_path), f'rank{r}.pt'), weights_only=False) for r in range(world)]
    assert [o['shard'][1] - o['shard'][0] for o in outs] == [15, 17], [o['shard'] for o in outs]
    triples = [_shard(r, world)[0] for r in range(world)]
    margs = gio.load_args('db5')
    cpu = torch.device('cpu')
    for t in range(TWO_RANK_STEPS):
        st = [o['steps'][t] for o in outs]
        assert torch.equal(st[0]['w0'], st[1]['w0'])
        assert torch.equal(st[0]['w1'], st[1]['w1']), f'step {t + 1}: flat_w differs between the ranks'
        model_t = _model_at(st[0]['w0'], cpu)
        layout = ParamLayout(model_t)
        refs = []
        for r in range(world):
            _certify(st[r]['flows'], st[r]['keypts'], triples[r])
            refs.append(_fp64_step(model_t, st[r]['inp'], st[r]['n_lig'], st[r]['draws'], st[r]['flows'], triples[r],
                                   SEEDS[t], margs))
        mean = {n: sum(rf['grads'][n] for rf in refs) / world for n in refs[0]['grads']}
        ref = {'grads': mean, 'norm': math.sqrt(sum(float((v ** 2).sum()) for v in mean.values()))}
        for r in range(world):
            ref_r = dict(ref, loss=refs[r]['loss'], parts=refs[r]['parts'], coors=refs[r]['coors'])
            got = _flat_by_name(model_t, layout, st[r]['g1'])
            _check_model_level(f'world {world} ({backend}) step {t + 1} rank {r}', st[r]['loss'], st[r]['norm'],
                               st[r]['coors'], got, ref_r, TWO_RANK_CLIP)


# ---- 4. the optimizer kernels -------------------------------------------------------------------------------------------

def _layout_totals():
    from equidock_public_b200.rigid_docking_model import Rigid_Body_Docking_Net
    out = []
    for ds in ('db5', 'dips'):
        a = dict(gio.load_args(ds), device='cpu')
        out.append(ParamLayout(Rigid_Body_Docking_Net(a)).total)
    return out


KERNEL_N = [1, 255, 257, 'db5', 'dips']       # 1 and 255: fewer elements than 256 or 1024 partials


@pytest.mark.parametrize('n', KERNEL_N)
def test_clip_adam_kernels_vs_fp64(n, cuda_device):
    """eqd_sqnorm_partials (1, 64, 256, 1024 partials; 0 and 1025 refused, also by eqd_clip_adam) and eqd_clip_adam
    (scale_extra 1, 1/2, 1/8; weight decay 0 and 1e-4; steps 1, 2, 3, 10 000; max_norm above the norm, half of it and
    equal to it) per element against fp64 from their own inputs: each partial against the fp64 sum of squares of its
    slice, norm_out within 3u, g (= g scale_extra clip) within 6u, and w, m, v within _adam_ref's bounds."""
    dev, lib = cuda_device, nat.load()
    if isinstance(n, str):
        n = _layout_totals()[('db5', 'dips').index(n)]
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    gen = torch.Generator(device=dev).manual_seed(n)
    rnd = lambda scale: torch.randn(n, device=dev, generator=gen) * scale
    g_in, w_in = rnd(0.05), rnd(0.1)
    m_in, v_in = rnd(1e-3), rnd(1e-3) ** 2
    worst = {}
    upd = lambda k, x: worst.__setitem__(k, max(worst.get(k, 0.0), x))
    for P in (0, 1025):
        part = torch.zeros(1025, dtype=torch.float64, device=dev)
        assert lib.eqd_sqnorm_partials(nat.ptr(g_in), n, nat.ptr(part), P, st) != 0
        g = g_in.clone()
        assert lib.eqd_clip_adam(nat.ptr(w_in.clone()), nat.ptr(g), nat.ptr(m_in.clone()), nat.ptr(v_in.clone()), n,
                                 nat.ptr(part), P, 1.0, LR, 0.9, 0.999, EPS, WD, 1, 1.0, None, st) != 0
        assert torch.equal(g, g_in)
    g64 = g_in.double()
    for P in (1, 64, 256, 1024):
        part = torch.full((P,), float('nan'), dtype=torch.float64, device=dev)
        nat.check(lib.eqd_sqnorm_partials(nat.ptr(g_in), n, nat.ptr(part), P, st), 'eqd_sqnorm_partials')
        per = -(-n // P)
        sl = torch.zeros(P * per, dtype=torch.float64, device=dev)
        sl[:n] = g64 ** 2
        ref_part = sl.view(P, per).sum(1)
        upd('partials', float(((part - ref_part).abs() / (1e-12 * ref_part.sum())).max()))
        norm64 = float(ref_part.sum().sqrt())
        for s in (1.0, 0.5, 0.125):
            for mx_name, mx in (('above', 2 * norm64 * s), ('half', 0.5 * norm64 * s), ('equal', norm64 * s)):
                c = _clip_factor(mx, norm64 * s)
                for wd in (0.0, WD):
                    for step in (1, 2, 3, 10000):
                        w, g, m, v = w_in.clone(), g_in.clone(), m_in.clone(), v_in.clone()
                        norm_out = torch.full((1,), float('nan'), device=dev)
                        nat.check(lib.eqd_clip_adam(nat.ptr(w), nat.ptr(g), nat.ptr(m), nat.ptr(v), n, nat.ptr(part), P,
                                                    mx, LR, BETAS[0], BETAS[1], EPS, wd, step, s, nat.ptr(norm_out), st),
                                  'eqd_clip_adam')
                        upd('norm_out', abs(float(norm_out[0]) - norm64 * s) / (3 * U * norm64 * s))
                        g_ref = g64 * (float(np.float32(s)) * c)
                        upd('g', _worst_fraction(g, g_ref, 6 * U * g_ref.abs()))
                        fr = _adam_fractions(w_in, m_in, v_in, g, w, m, v, step, wd=wd)
                        for k, x in fr.items():
                            upd(k, x)
                        if mx_name == 'above':
                            assert torch.equal(g, g_in * float(np.float32(s)))
    print(f'\nclip_adam n={n}: worst fractions of the bounds: ' + ', '.join(f'{k} {v:.2e}' for k, v in worst.items()))
    assert all(v <= 1 for v in worst.values()), worst
