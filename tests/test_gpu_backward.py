"""GPU (H100): the hand-written CUDA backward (csrc/bwd_*.cu, head.cu) and the device losses / optimiser kernels against
the fp64 oracles.  Stage by stage against oracle/backward_manual.py (itself == torch.autograd == the reference's golden
gradients, tests/test_backward_manual.py), then end to end through ``loss.backward()`` on the drop-in module.
Tolerance: the backward runs in fp32 (coordinates / head in fp64); gradients are compared relative to the largest entry of
the tensor: 2e-3 (stage outputs) / 3e-3 (parameter gradients after 5-8 layers), measured values are ~1e-5 .. 3e-4."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import backward_manual as bm
import golden_io as gio
import iegmn_oracle as orc
from equidock_public_b200 import _native as nat
from equidock_public_b200 import synthetic
from equidock_public_b200.training import TrainEngine

pytestmark = pytest.mark.gpu
PAIR = {'db5': '1QA9', 'dips': 'kq_1kq1.pdb1_2.dill'}
KINK_MAX_FRACTION = 1e-2   # of the edge / node rows of a layer (see _stage_report's kink_band)


def _np(t):
    if isinstance(t, np.ndarray):
        return t.astype(np.float64)
    return t.detach().cpu().numpy().astype(np.float64)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _targets(ds):
    z = np.load(gio.GOLDEN + f'/{ds}_grads.npz')
    return z, {k[len('target/'):]: z[k] for k in z.files if k.startswith('target/')}


def _loss_grads(tgt):
    def f(out):
        n = out['ligand_coors'].shape[0]
        return (2.0 * (out['ligand_coors'] - tgt['coors']) / (3 * n),
                2.0 * tgt['w_l'][:, None] * (out['keypts_ligand'] - tgt['p_l']) / 50,
                2.0 * tgt['w_r'][:, None] * (out['keypts_receptor'] - tgt['p_r']) / 50)
    return f


def _stage_report(model, args, pairs, grad_fns, cuda_device, kink_band=0.0):
    """Runs forward + CUDA backward with stage capture on a batch and compares every stage output and every parameter
    gradient with the per-pair manual oracle (concatenated in engine order: ligand nodes / edges of all pairs, then the
    receptor ones).  An entry passes if max|got - ref| <= tol * max|ref| + 2e-6 * G, G = the largest reference magnitude
    of the same group (all stage tensors / all parameter gradients): fp32 cancellation noise on a tensor whose true
    gradient is orders of magnitude below its neighbours' (a saturated attention layer) is not an error.
    kink_band > 0 leaves out the rows of a layer with an fp64 pre-activation (z1, z3 of an edge, u5 of a node) within
    kink_band x (the row's max|z|) of the LeakyReLU kink: the engine's fp32 activations after several layers need not
    resolve its sign there, and the derivative differs by (1 - slope) x the upstream gradient.  Such edges, such nodes and
    the nodes such edges gather into are left out of the per-row stage comparisons (at most KINK_MAX_FRACTION of a
    layer's rows)."""
    sd = {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}
    cfg = orc.OracleConfig.from_args(args)
    shared = bool(args['shared_layers'])
    per_pair, grads_ref = [], None
    for (lig, rec), f in zip(pairs, grad_fns):
        st = []
        gr, out = bm.full_backward(sd, cfg, lig, rec, f, shared, st)
        per_pair.append((st, out, f(out)))
        grads_ref = gr if grads_ref is None else {k: grads_ref[k] + gr[k] for k in gr}
    eng = TrainEngine(model)
    g = gio.make_batch(pairs, cuda_device)
    fwd = eng.forward(g)
    B = len(pairs)
    # the random perturbation branch of the SVD guard (:574-584) is not part of the manual oracle: inputs must not reach it
    assert not bool(fwd['status_host'][:B].any()), ('status flags (SVD guard / NaN / bad residue) on a stage-by-stage case',
                                                    fwd['status_host'][:B].tolist())
    co_ref = np.concatenate([pp[1]['ligand_coors'] for pp in per_pair])
    assert np.abs(_np(fwd['ligand_coors']) - co_ref).max() < 2e-3 * max(1.0, np.abs(co_ref).max() / 100)
    dco = np.concatenate([pp[2][0] for pp in per_pair])
    dky = np.stack([pp[2][1] for pp in per_pair] + [pp[2][2] for pp in per_pair])
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device, dt)
    cap = []
    flat = eng.backward(fwd, t(dco, torch.float32), t(dky, torch.float64), capture=cap)
    torch.cuda.synchronize()
    rows = []          # (group, tag, err, refmax, tol)

    def chk(group, tag, got, ref, tol, keep=None):
        got, ref = _np(got), np.asarray(ref, np.float64)
        d = np.abs(got - ref) if keep is None else np.abs(got - ref)[keep]
        rows.append((group, tag, float(d.max()), float(np.abs(ref).max()), tol))

    def cat(key, li=None, head=False):
        sides = [[], []]
        for stg, _, _ in per_pair:
            if head:
                h = [s_ for s_ in stg if s_.get('head')][0]
                sides[0].append(h[key][0]); sides[1].append(h[key][1])
            else:
                sl, sr = [s_ for s_ in stg if s_.get('layer') == li][0]['sides']
                sides[0].append(sl[key]); sides[1].append(sr[key])
        return np.concatenate(sides[0] + sides[1])

    chk('stage', 'head dh', cap[0]['dh'], cat('dh', head=True), 2e-3)
    chk('stage', 'head dx', cap[0]['dx'], cat('dx', head=True), 2e-3)
    plan = fwd['plan']
    src, dst = plan.col_src.cpu().numpy(), plan.edge_dst.cpu().numpy()
    near = lambda z: (np.abs(z) < kink_band * np.abs(z).max(1, keepdims=True)).any(1)
    for c in cap[1:]:
        li = c['layer']
        dh_w = cat('dh', li).shape[1]
        dhp = c['dmu'].shape[1]
        e_ok, n_ok = ~(near(cat('z1', li)) | near(cat('z3', li))), ~near(cat('u5', li))
        g_ok = np.ones(plan.N, bool)
        g_ok[src[~e_ok]] = g_ok[dst[~e_ok]] = False
        assert (~e_ok).mean() <= KINK_MAX_FRACTION and (~n_ok).mean() <= KINK_MAX_FRACTION
        if not (e_ok.all() and n_ok.all()):
            print(f'L{li}: {(~e_ok).sum()} edge rows, {(~n_ok).sum()} node rows within the kink band')
        chk('stage', f'L{li} node: dh (skip + W5 h block)', c['dh_part'][:, :dh_w], cat('dh_part', li), 2e-3, n_ok)
        chk('stage', f'L{li} node: daggr', c['daggr'], cat('daggr', li), 2e-3, n_ok)
        chk('stage', f'L{li} node: dmu', c['dmu'][:, :dh_w], cat('dmu', li), 2e-3, n_ok)
        chk('stage', f'L{li} edge: dz1', c['dz1'], cat('dz1', li), 2e-3, e_ok)
        chk('stage', f'L{li} edge: dxrel', c['dxrel'], cat('dxrel', li), 2e-3, e_ok)
        chk('stage', f'L{li} gather: dPsrc', c['dP'][:, 0:64], cat('dpsrc', li), 2e-3, g_ok)
        chk('stage', f'L{li} gather: dPdst', c['dP'][:, 64:128], cat('dpdst', li), 2e-3, g_ok)
        chk('stage', f'L{li} attn: dQpre', c['dP'][:, 128:128 + dh_w], cat('dqpre', li), 2e-3)
        chk('stage', f'L{li} attn: dKpre', c['dP'][:, 128 + dhp:128 + dhp + dh_w], cat('dkpre', li), 2e-3)
        chk('stage', f'L{li} attn: dV', c['dP'][:, 128 + 2 * dhp:128 + 2 * dhp + dh_w], cat('dv', li), 2e-3)
        chk('stage', f'L{li} gather: dx', c['dx'], cat('dx', li), 2e-3, g_ok)
        chk('stage', f'L{li} proj: dh', c['dh'][:, :dh_w], cat('dh', li), 2e-3)
    flat_np = _np(flat)
    lo = eng.layout
    for (name, p) in lo.entries:
        ref = grads_ref[name]
        got = flat_np[lo.offset[id(p)]:lo.offset[id(p)] + p.numel()].reshape(ref.shape)
        chk('grad', f'grad {name.replace("iegmn_original.", "")}', got, ref, 3e-3)
    G = {grp: max(r[3] for r in rows if r[0] == grp) for grp in ('stage', 'grad')}
    report, bad = [], []
    for grp, tag, err, refmax, tol in rows:
        ok = err <= tol * refmax + 2e-6 * G[grp]
        report.append(f'{"ok  " if ok else "BAD "}{tag:44s} abs {err:.2e}  rel {err / max(refmax, 1e-30):.2e}  max|ref| {refmax:.3e}')
        if not ok:
            bad.append(report[-1])
    print('\n'.join(report))
    return bad


@pytest.mark.parametrize('ds', ['db5', 'dips'])
def test_backward_stage_by_stage_vs_manual_oracle(ds, cuda_device):
    names, pairs, outs, _ = gio.load_pairs(ds)
    z, tgt = _targets(ds)
    model = gio.build_model(ds, cuda_device).train()
    bad = _stage_report(model, gio.load_args(ds), [pairs[PAIR[ds]]], [_loss_grads(tgt)], cuda_device)
    assert not bad, '\n'.join(bad)


@pytest.mark.parametrize('kind', ['db5', 'dips', 'random', 'bulk', 'k70'])
def test_backward_stage_by_stage_ragged_batch(kind, cuda_device):
    """B = 3 ragged pairs incl. tile boundaries (129 = 128 + 1, 131 = 128 + 3): both checkpoints (5 shared layers / 8
    layers) and a random-init 3-layer unshared model with non-trivial biases / LayerNorm affine parameters.  The random
    model's keypoint attention is sharpened: at default init it is nearly uniform, every keypoint sits at the centroid and
    the reference's SVD guard (:574) fires on all three pairs (the fp64 oracle's own verdict).  Its seed keeps every edge
    pre-activation of the fp64 oracle >= 1.5e-6 away from the LeakyReLU kink: closer than fp32 resolves, the engine may take
    the other branch and the derivative there differs by 0.99 x the upstream gradient (seed 5 has one at 1.4e-8).
    `bulk` (DIPS checkpoint) adds 168 pairs of 200 + 200 nodes: 67 648 nodes, so every persistent backward kernel runs at
    least two tiles per CTA (529 node tiles on the 264 CTAs of the projection backward and the 132 of the others, 680
    attention tiles, about 5 300 edge tiles); of its 90 M pre-activations per layer some lie closer to the kink than
    fp32 resolves, so its rows within 1e-5 x (the row's max|z|) of it are left out (see _stage_report).  `k70`: the DIPS
    checkpoint with graph_max_neighbor = 70 on pairs built with 70 in-edges per node, above the 64 of the forward's
    tensor-core edge tile."""
    from test_gpu_parity import _random_model
    k = 10
    if kind == 'random':
        model, args = _random_model(cuda_device, 3, False, seed=7)
        with torch.no_grad():
            for name, p in model.named_parameters():
                if name.startswith(('iegmn_original.att_mlp_key_ROT.', 'iegmn_original.att_mlp_query_ROT.')):
                    p.mul_(8.0)
    elif kind == 'k70':
        k, args = 70, dict(gio.load_args('dips'), graph_max_neighbor=70)
        model = gio.build_model('dips', cuda_device, args=args)
    else:
        ds = 'dips' if kind == 'bulk' else kind
        model, args = gio.build_model(ds, cuda_device), gio.load_args(ds)
    model.train()
    rng = np.random.default_rng(9)
    sizes = [(100, 131), (129, 90), (75, 80)] if kind == 'k70' else [(40, 131), (129, 20), (64, 64)]
    if kind == 'bulk':
        sizes += [(200, 200)] * 168
        assert -(-sum(a + b for a, b in sizes) // 128) >= 2 * 264
    pairs = [synthetic.synthetic_pair(rng, a, b, k) for a, b in sizes]
    tg = [{'c': rng.normal(0, 5, (a, 3)), 'yl': rng.normal(0, 10, (50, 3)), 'yr': rng.normal(0, 10, (50, 3))} for a, b in sizes]
    fns = [(lambda out, t=t: (2 * (out['ligand_coors'] - t['c']), 2 * (out['keypts_ligand'] - t['yl']),
                              2 * (out['keypts_receptor'] - t['yr']))) for t in tg]
    bad = _stage_report(model, args, pairs, fns, cuda_device, kink_band=1e-5 if kind == 'bulk' else 0.0)
    assert not bad, '\n'.join(bad)


@pytest.mark.parametrize('ds', ['db5', 'dips'])
def test_loss_backward_through_the_module_matches_golden_gradients(ds, cuda_device):
    """The reference's training step shape (src/train.py:98-154): model.train(); outputs -> torch loss -> loss.backward();
    every param.grad against the golden gradients of the UNMODIFIED reference (norm + seeded projection + full tensors)."""
    import iegmn_oracle_torch as ot
    names, pairs, outs, _ = gio.load_pairs(ds)
    lig, rec = pairs[PAIR[ds]]
    z, tgt = _targets(ds)
    model = gio.build_model(ds, cuda_device).train()
    g = gio.make_batch([(lig, rec)], cuda_device)
    coors, kp_l, kp_r, rot, trans = model(g, epoch=0)
    assert coors[0].requires_grad and kp_l[0].requires_grad
    tg = {k: torch.from_numpy(v).to(cuda_device) for k, v in tgt.items()}
    loss = ot.probe_loss(coors[0].double(), kp_l[0].double(), kp_r[0].double(), tg)
    assert abs(loss.item() - float(z['loss'])) < 1e-4 * max(1.0, abs(float(z['loss'])))
    loss.backward()
    bad = []
    gmax = max(float(z[k]) for k in z.files if k.startswith('norm/'))     # largest gradient norm of the model
    for pname, p in model.named_parameters():
        gnp = _np(p.grad)
        nrm = float(z['norm/' + pname])
        floor = 2e-6 * gmax          # fp32 cancellation noise on parameters whose gradient is 1e-5 of their neighbours'
        if abs(np.linalg.norm(gnp) - nrm) > 3e-3 * nrm + floor:
            bad.append((pname, 'norm', np.linalg.norm(gnp), nrm))
        d = np.random.default_rng(zlib.crc32(pname.encode())).standard_normal(gnp.shape)
        if abs((gnp * d).sum() - float(z['proj/' + pname])) > 3 * (3e-3 * nrm + floor):
            bad.append((pname, 'proj', (gnp * d).sum(), float(z['proj/' + pname])))
        if 'full/' + pname in z.files:
            ref = z['full/' + pname].astype(np.float64)
            if np.abs(gnp - ref).max() > 3e-3 * np.abs(ref).max() + floor:
                bad.append((pname, 'full', _rel(gnp, ref)))
    assert not bad, bad


def test_ragged_batch_gradient_is_the_sum_of_pair_gradients(cuda_device):
    """B = 3 ragged pairs incl. tile boundaries through loss.backward() on the module (DIPS checkpoint, 8 layers)."""
    model, args = gio.build_model('dips', cuda_device), gio.load_args('dips')
    model.train()
    rng = np.random.default_rng(9)
    sizes = [(40, 131), (129, 20), (64, 64)]
    pairs = [synthetic.synthetic_pair(rng, a, b, 10) for a, b in sizes]
    sd = {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}
    cfg = orc.OracleConfig.from_args(args)
    tg = [{'c': rng.normal(0, 5, (a, 3)), 'yl': rng.normal(0, 10, (50, 3)), 'yr': rng.normal(0, 10, (50, 3))} for a, b in sizes]
    total = None
    for (lig, rec), t in zip(pairs, tg):
        f = lambda out, t=t: (2 * (out['ligand_coors'] - t['c']), 2 * (out['keypts_ligand'] - t['yl']), 2 * (out['keypts_receptor'] - t['yr']))
        gr, _ = bm.full_backward(sd, cfg, lig, rec, f, bool(args['shared_layers']))
        total = gr if total is None else {k: total[k] + gr[k] for k in gr}
    coors, kp_l, kp_r, _, _ = model(gio.make_batch(pairs, cuda_device), epoch=0)
    dev = cuda_device
    loss = sum(((coors[i].double() - torch.from_numpy(tg[i]['c']).to(dev)) ** 2).sum()
               + ((kp_l[i].double() - torch.from_numpy(tg[i]['yl']).to(dev)) ** 2).sum()
               + ((kp_r[i].double() - torch.from_numpy(tg[i]['yr']).to(dev)) ** 2).sum() for i in range(3))
    loss.backward()
    gmax = max(np.abs(v).max() for v in total.values())
    bad = [(n, _rel(_np(p.grad), total[n])) for n, p in model.named_parameters()
           if np.abs(_np(p.grad) - total[n]).max() > 3e-3 * np.abs(total[n]).max() + 2e-6 * gmax]
    assert not bad, bad


def test_clip_adam_kernel_vs_torch_adam(cuda_device):
    lib = nat.load()
    torch.manual_seed(1)
    n = 100003
    w0 = torch.randn(n, device=cuda_device)
    w_t = torch.nn.Parameter(w0.clone())
    opt = torch.optim.Adam([w_t], lr=2e-4, weight_decay=1e-4)
    w, m, v = w0.clone(), torch.zeros(n, device=cuda_device), torch.zeros(n, device=cuda_device)
    part = torch.empty(64, dtype=torch.float64, device=cuda_device)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for step in range(1, 4):
        gr = torch.randn(n, device=cuda_device) * (3.0 if step == 2 else 0.1)
        w_t.grad = gr.clone()
        torch.nn.utils.clip_grad_norm_([w_t], max_norm=100.0)
        opt.step()
        g2 = gr.clone()
        nat.check(lib.eqd_sqnorm_partials(nat.ptr(g2), n, nat.ptr(part), 64, st), 'sq')
        nat.check(lib.eqd_clip_adam(nat.ptr(w), nat.ptr(g2), nat.ptr(m), nat.ptr(v), n, nat.ptr(part), 64, 100.0, 2e-4, 0.9, 0.999,
                                    1e-8, 1e-4, step, 1.0, None, st), 'adam')
        assert (w - w_t.detach()).abs().max().item() < 2e-6


@pytest.mark.parametrize('n_pocket', [[7], [48, 4, 133], [398]])
def test_device_losses_vs_oracle(n_pocket, cuda_device):
    """MSE, exact EMD (must hit the LP optimum certified by duality in oracle/loss_oracle.py) and the body-intersection
    loss, values and gradients (the OT plan is a constant: ot_utils.py:27), N_pocket in {7, 48, 398} (SURVEY 8f)."""
    import loss_oracle as lo
    from equidock_public_b200.engine import GraphPlan
    from equidock_public_b200.losses import PocketBatch, device_losses, check_loss_status
    rng = np.random.default_rng(sum(n_pocket))
    B = len(n_pocket)
    pairs = [synthetic.synthetic_pair(rng, 30 + 17 * i, 41 + 9 * i, 10) for i in range(B)]
    g = gio.make_batch(pairs, cuda_device)
    plan = GraphPlan.from_graph(g, cuda_device)
    pred = [p[0]['new_x'].astype(np.float64) + rng.normal(0, 2, p[0]['new_x'].shape) for p in pairs]
    bl = [p[0]['x'].astype(np.float64) for p in pairs]
    br = [(p[1]['x'].astype(np.float64) + 12.0) for p in pairs]
    kl = [rng.normal(0, 15, (50, 3)) for _ in range(B)]
    kr = [rng.normal(0, 15, (50, 3)) for _ in range(B)]
    pl = [rng.normal(0, 12, (n, 3)) for n in n_pocket]
    pr = [rng.normal(0, 12, (n, 3)) for n in n_pocket]
    f32 = lambda a: np.asarray(a, np.float32)
    pred32, bl32, br32, pl32, pr32 = ([f32(a) for a in L] for L in (pred, bl, br, pl, pr))
    t = lambda L: [torch.from_numpy(a) for a in L]
    tgt = PocketBatch(t(bl32), t(br32), t(pl32), t(pr32), cuda_device)
    res = device_losses(plan, torch.from_numpy(np.concatenate(pred32)).to(cuda_device),
                        torch.from_numpy(np.stack(kl + kr)).to(cuda_device), tgt, 1.0, 10.0, 25.0, 10.0)
    check_loss_status(res)
    ref_loss, parts = lo.batch_loss(pred32, bl32, br32, kl, kr, pl32, pr32, 1.0, 10.0, 25.0, 10.0)
    tot = _np(res['total'])
    assert abs(tot[0] - ref_loss) < 1e-8 * max(1.0, abs(ref_loss)), (tot, ref_loss, parts)
    assert abs(tot[1] - parts['mse']) < 1e-9 * max(1, parts['mse']) and abs(tot[2] - parts['ot']) < 1e-9 * max(1, parts['ot'])
    assert abs(tot[3] - parts['intersection']) < 1e-9 * max(1, parts['intersection'])
    # gradients by torch autograd on the oracle's formulas with the kernel's plan as a constant: the optimal plan need not
    # be unique, so the plan is certified optimal (lo.ot_certify) and both keypoint gradients are checked against it
    flows = res['plan'].cpu().numpy()
    for i in range(B):
        p = torch.tensor(pred32[i].astype(np.float64), requires_grad=True)
        yl = torch.tensor(kl[i], requires_grad=True)
        yr = torch.tensor(kr[i], requires_grad=True)
        cost = lo.sq_dist_mat(pl32[i], kl[i]) + lo.sq_dist_mat(pr32[i], kr[i])
        p0, n = sum(n_pocket[:i]), n_pocket[i]
        x = flows[p0:p0 + n]
        lo.ot_certify(cost, x)
        T = torch.from_numpy(x.astype(np.float64) / (50 * n))
        c_t = ((torch.tensor(pl32[i].astype(np.float64))[:, None] - yl[None]) ** 2).sum(2) + \
              ((torch.tensor(pr32[i].astype(np.float64))[:, None] - yr[None]) ** 2).sum(2)
        G = lambda prot, x: -25.0 * torch.log(1e-3 + torch.exp(-((prot[None] - x[:, None]) ** 2).sum(2) / 25.0).sum(1))
        rec_t = torch.tensor(br32[i].astype(np.float64))
        inter = torch.clamp(10.0 - G(rec_t, p), min=0).mean() + torch.clamp(10.0 - G(p, rec_t), min=0).mean()
        loss = (((p - torch.tensor(bl32[i].astype(np.float64))) ** 2).mean() + (T * c_t).sum() + 10.0 * inter) / B
        loss.backward()
        lo_, hi_ = plan.seg_ptr_host[i], plan.seg_ptr_host[i + 1]
        assert _rel(_np(res['dcoors'][lo_:hi_]), p.grad.numpy()) < 1e-5
        # both halves; the bound is relative to sum_i T_ik |Y_k - P_i| (the signed sum can cancel)
        for ours, ref, P, Y in ((_np(res['dkeypts'][i]), yl.grad.numpy(), pl32[i], kl[i]),
                                (_np(res['dkeypts'][B + i]), yr.grad.numpy(), pr32[i], kr[i])):
            mag = 2.0 / B * (T.numpy()[:, :, None] * np.abs(Y[None] - P.astype(np.float64)[:, None])).sum(0)
            assert (np.abs(ours - ref) <= 1e-12 * mag).all(), float((np.abs(ours - ref) - 1e-12 * mag).max())


def test_rmsd_meter_kernel_vs_reference_definition(cuda_device):
    """eval.Meter_Unbound_Bound (batched kernel) == the numpy restatement of src/utils/eval.py:19-42 (oracle complex_rmsd),
    incl. a pair whose best superposition is a reflection before the fix (:56-59)."""
    from equidock_public_b200.eval import Meter_Unbound_Bound
    from equidock_public_b200.engine import GraphPlan
    rng = np.random.default_rng(3)
    sizes = [(30, 41), (128, 7), (5, 300)]
    pairs = [synthetic.synthetic_pair(rng, a, b, 4) for a, b in sizes]
    plan = GraphPlan.from_graph(gio.make_batch(pairs, cuda_device), cuda_device)
    lt = [rng.normal(0, 10, (a, 3)).astype(np.float32) for a, b in sizes]
    rt = [rng.normal(0, 10, (b, 3)).astype(np.float32) for a, b in sizes]
    lp, rp = [], []
    for i, (a, b) in enumerate(sizes):
        R, tv = synthetic.random_rigid(rng, 30.0)
        if i == 1:
            R = R @ np.diag([1, 1, -1]).astype(np.float32)       # mirrored prediction
        lp.append(((R @ lt[i].T).T + tv + rng.normal(0, 0.7, (a, 3))).astype(np.float32))
        rp.append(((R @ rt[i].T).T + tv + rng.normal(0, 0.7, (b, 3))).astype(np.float32))
    tt = lambda L: [torch.from_numpy(x).to(cuda_device) for x in L]
    meter = Meter_Unbound_Bound()
    out = meter.update_rmsd_batch(plan, tt(lp), tt(rp), tt(lt), tt(rt)).cpu().numpy()
    for i in range(3):
        f = lambda a: a.astype(np.float64)
        ref = orc.complex_rmsd(f(lp[i]), f(rp[i]), f(lt[i]), f(rt[i]))
        assert abs(out[i, 0] - ref) < 1e-9 * max(1, ref)
        assert abs(out[i, 1] - np.sqrt(((f(lp[i]) - f(lt[i])) ** 2).sum(1).mean())) < 1e-9 * max(1.0, out[i, 1])
    single = Meter_Unbound_Bound().update_rmsd(tt(lp)[0], tt(rp)[0], tt(lt)[0], tt(rt)[0])
    assert abs(single - out[0, 0]) < 1e-12


def test_fused_trainer_step_equals_autograd_plus_torch_adam(cuda_device):
    """DataParallelTrainer.step (device losses, CUDA backward into the flat buffer, fused clip + Adam) == the reference's
    loop shape: model.train(); outputs -> the same losses through torch autograd on our outputs -> loss.backward() ->
    clip_grad_norm_ -> torch.optim.Adam.step(), for two consecutive steps."""
    from equidock_public_b200.losses import PocketBatch, device_losses
    from equidock_public_b200.training import DataParallelTrainer
    import copy
    rng = np.random.default_rng(12)
    sizes = [(60, 75), (90, 50)]
    pairs = [synthetic.synthetic_pair(rng, a, b, 10) for a, b in sizes]
    m1 = gio.build_model('db5', cuda_device).train()
    m2 = gio.build_model('db5', cuda_device).train()
    g = gio.make_batch(pairs, cuda_device)
    bl = [torch.from_numpy(p[0]['x']) for p in pairs]
    br = [torch.from_numpy(p[1]['x'] + 8.0) for p in pairs]
    pk = [torch.from_numpy((0.5 * (p[0]['x'][:9] + p[1]['x'][:9] + 8.0)).astype(np.float32)) for p in pairs]
    tgt = PocketBatch(bl, br, pk, pk, cuda_device)
    tr = DataParallelTrainer(m1, lr=1e-3, weight_decay=1e-4, clip=100.0)
    opt = torch.optim.Adam(m2.parameters(), lr=1e-3, weight_decay=1e-4)
    for step in range(2):
        r1 = tr.step(g, tgt)
        opt.zero_grad()
        coors, kl, kr, _, _ = m2(g, epoch=0)
        plan = m2.iegmn_original.last_outputs['plan']
        res = device_losses(plan, torch.cat(coors), torch.cat([torch.stack(kl), torch.stack(kr)]).double(), tgt, 1.0, 10.0, 25.0, 10.0)
        # route the device-loss gradients through autograd: loss surrogate = <outputs, dloss/doutputs>
        sur = (torch.cat(coors) * res['dcoors']).sum() + (torch.cat([torch.stack(kl), torch.stack(kr)]).double() * res['dkeypts']).sum()
        sur.backward()
        torch.nn.utils.clip_grad_norm_(m2.parameters(), max_norm=100.0)
        opt.step()
        assert abs(float(r1['loss'][0]) - float(res['total'][0])) < 1e-6 * max(1.0, abs(float(res['total'][0])))
    for (n1, p1), (n2, p2) in zip(m1.named_parameters(), m2.named_parameters()):
        assert (p1 - p2).abs().max().item() < 5e-6, n1
