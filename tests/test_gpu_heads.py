"""GPU (H100): models with num_att_heads = K keypoints per protein (K = 4, 25, 32, 33, 64 at the kernels; 25 and 64 end to
end) against fp64.

  - eqd_head_fold, eqd_keypoints and eqd_kabsch_apply: every fp64 stage from the kernel's own inputs, at the bounds of
    tests/test_gpu_forward_kernels.py, then the keypoints and the rigid transform against oracle/iegmn_oracle.py.  K = 32 /
    33 end the last warp's heads at a lane boundary / one past it, 33 and 64 leave a partial last group of 25 heads.
  - eqd_bwd_head against oracle/backward_manual.py at the 1e-5 of tests/test_gpu_backward_kernels.py.
  - eqd_losses_k: the exact-EMD value against the HiGHS optimum (1e-9), every plan certified optimal by
    loss_oracle.ot_certify, at pocket sizes 4 .. 398 and one past the largest pocket whose cost matrix still fits in
    shared memory for that K (1024, the solver's capacity, where it always fits).
  - Whole models (5 shared / 8 layers): forward, CUDA-graph replay, loss.backward() and DataParallelTrainer.step against
    torch.autograd on the fp64 restatement of tests/heads_ref.py, at the bounds of tests/test_gpu_dropout.py; once with
    dropout 0.25.
Every kernel launch runs twice and must be bitwise equal.  Models: the shipped checkpoints with seeded K-head key / query
projections (heads_ref.build_model)."""
import ctypes as C

import numpy as np
import pytest
import torch

import backward_manual as bm
import dropout_masks as dm
import golden_io as gio
import heads_ref as hr
import iegmn_oracle as orc
import loss_oracle as lo
from equidock_public_b200 import _native as nat
from equidock_public_b200 import synthetic
from equidock_public_b200.engine import GraphPlan
from equidock_public_b200.losses import PocketBatch, check_loss_status, device_losses
from equidock_public_b200.training import TrainEngine
from test_gpu_dropout import _loss, _oracle_inputs, _run_module
from test_gpu_dropout import _pairs as _model_pairs
from test_gpu_layer_norm_options import _fp64_state, _grad_mismatches
from test_gpu_losses import _plan

pytestmark = pytest.mark.gpu
F64 = torch.float64
KS = [4, 25, 32, 33, 64]


def _pairs(kind):
    if kind == 'single':
        _, pairs, _, _ = gio.load_pairs('dips')
        return [pairs['kq_1kq1.pdb1_2.dill']]
    rng = np.random.default_rng(31)
    sizes = {'ragged3': [(40, 131), (129, 20), (64, 64)], 'sizes': [(1, 63), (64, 65), (65, 1), (63, 64)]}[kind]
    return [synthetic.synthetic_pair(rng, a, b, min(10, a - 1, b - 1) if min(a, b) > 1 else 0) for a, b in sizes]


def _rel(got, ref):
    got, ref = torch.as_tensor(got).to(F64).cpu(), torch.as_tensor(ref).to(F64).cpu()
    assert torch.isfinite(got).all()
    return float((got - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)


def _twice(run):
    a, b = run(), run()
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    return a


def _sd_np(model):
    return {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}


def _cfg(args):
    return orc.OracleConfig(args['iegmn_n_lays'], args['skip_weight_h'], args['x_connection_init'],
                            args['leakyrelu_neg_slope'], args['num_att_heads'])


# ---- forward kernels --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('kind', ['single', 'ragged3', 'sizes'])
@pytest.mark.parametrize('K', KS)
def test_head_forward_kernels_vs_fp64(K, kind, cuda_device):
    dev, lib = cuda_device, nat.load()
    g = gio.make_batch(_pairs(kind), dev)
    plan = GraphPlan.from_graph(g, dev, 10)
    model = hr.build_model('dips', dev, K, seed=K)
    net = model.iegmn_original
    head = net.packed_head(dev)
    assert head.struct.n_heads == K and head.m_qk.shape == (K, 64, 64)
    B, N, NL = plan.n_pairs, plan.N, plan.N_l
    gen = torch.Generator(device=dev).manual_seed(100 + K)
    h = torch.randn(N, 64, generator=gen, device=dev) * 0.7
    x = (torch.randn(N, 3, generator=gen, device=dev, dtype=F64) * 8.0).contiguous()
    xl = x[:NL].float().contiguous()
    ws_bytes = int(lib.eqd_workspace_bytes_k(N, plan.n_node_tiles, B, K))
    a256 = lambda v: (v + 255) // 256 * 256
    q_off = a256(max(plan.n_node_tiles, 1) * 256) + a256((2 * B + 1) * 4)
    u_off = q_off + a256(2 * B * 64 * 8)
    assert ws_bytes == u_off + a256(2 * B * K * 64 * 8)

    def run():
        ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device=dev)
        m = torch.full((K, 64, 64), float('nan'), dtype=F64, device=dev)
        nat.check(lib.eqd_head_fold(C.byref(head.struct), nat.ptr(m), None), 'eqd_head_fold')
        kp = torch.full((2 * B, K, 3), float('nan'), dtype=F64, device=dev)
        ym = torch.full((2 * B, 3), float('nan'), dtype=F64, device=dev)
        cov = torch.full((B, 9), float('nan'), dtype=F64, device=dev)
        nat.check(lib.eqd_keypoints(C.byref(plan.struct), C.byref(head.struct), nat.ptr(h), nat.ptr(x), nat.ptr(ws),
                                    ws_bytes, nat.ptr(kp), nat.ptr(ym), nat.ptr(cov), None), 'eqd_keypoints')
        rot, trans = torch.full((B, 9), float('nan'), device=dev), torch.full((B, 3), float('nan'), device=dev)
        lig = torch.full((NL, 3), float('nan'), device=dev)
        sing = torch.full((B, 3), float('nan'), dtype=F64, device=dev)
        status = torch.zeros(B, dtype=torch.int32, device=dev)
        nat.check(lib.eqd_kabsch_apply(C.byref(plan.struct), nat.ptr(cov), nat.ptr(ym), nat.ptr(xl), None, nat.ptr(rot),
                                       nat.ptr(trans), nat.ptr(lig), nat.ptr(sing), nat.ptr(status), None),
                  'eqd_kabsch_apply')
        qbar = ws[q_off:q_off + 2 * B * 512].view(F64).view(2 * B, 64).clone()
        u = ws[u_off:u_off + 2 * B * K * 512].view(F64).view(2 * B, K, 64).clone()
        return m, qbar, u, kp, ym, cov, rot, trans, lig, sing, status

    m, qbar, u, kp, ym, cov, rot, trans, lig, sing, status = _twice(run)
    wq = net.att_mlp_query_ROT[0].weight.detach().to(F64).view(K, 64, 64)
    wk = net.att_mlp_key_ROT[0].weight.detach().to(F64).view(K, 64, 64)
    seg = [int(v) for v in plan.seg_ptr_host]
    part = [s + B if s < B else s - B for s in range(2 * B)]
    h64 = h.to(F64)
    kp_ref = torch.stack([torch.softmax(h64[seg[s]:seg[s + 1]] @ u[s].t(), 0).t() @ x[seg[s]:seg[s + 1]]
                          for s in range(2 * B)])
    yc = kp - kp.mean(1)[:, None]
    errs = {'m_qk': (_rel(m, torch.einsum('kec,ked->kcd', wq, wk) / 8.0), 1e-14),
            'u': (_rel(u, torch.einsum('kcd,sc->skd', m, qbar[part])), 1e-13),
            'keypts': (_rel(kp, kp_ref), 1e-12), 'ymean': (_rel(ym, kp.mean(1)), 1e-14),
            'cov': (_rel(cov, torch.einsum('bkr,bkc->brc', yc[B:], yc[:B]).reshape(B, 9)), 1e-14)}
    print(f'\nhead K={K} {kind}: ' + ', '.join(f'{k} {e:.1e}' for k, (e, _) in errs.items()))
    assert all(e <= tol for e, tol in errs.values()), errs
    # end to end against the numpy fp64 oracle (iegmn_oracle.keypoints_and_kabsch): keypoints from the fp32 qbar GEMM
    # (1e-5), the rotation within 2e-4 and the ligand within the coordinate bound where the oracle's guard does not fire
    sd, cfg = _sd_np(model), _cfg(hr.args_with('dips', K))
    hn, xn = h64.cpu().numpy(), x.cpu().numpy()
    for b in range(B):
        (la, lb), (ra, rb) = (seg[b], seg[b + 1]), (seg[B + b], seg[B + b + 1])
        c = bm.head_forward(sd, cfg, hn[la:lb], xn[la:lb], hn[ra:rb], xn[ra:rb])
        assert _rel(kp[b], c['Y'][0]) <= 1e-5 and _rel(kp[B + b], c['Y'][1]) <= 1e-5, b
        try:
            T, t, _, _, info = orc.keypoints_and_kabsch(sd, cfg, hn[la:lb], xn[la:lb], hn[ra:rb], xn[ra:rb], np.float64)
        except RuntimeError:                   # the guard fired (a one-node protein: all K keypoints coincide)
            assert int(status[b]) & nat.STATUS_SVD_DEGENERATE, b
            continue
        assert not int(status[b]) & nat.STATUS_SVD_DEGENERATE, (b, info['S'])
        assert float(np.abs(rot[b].cpu().numpy().reshape(3, 3) - T).max()) <= 2e-4, b
        ref = xl[la:lb].double().cpu().numpy() @ T.T + t
        assert float(np.abs(lig[la:lb].cpu().numpy() - ref).max()) <= 2e-3 * max(1.0, np.abs(ref).max() / 100), b
    if kind == 'sizes':
        assert int(status[0]) & nat.STATUS_SVD_DEGENERATE and int(status[2]) & nat.STATUS_SVD_DEGENERATE


def test_head_entry_points_refuse_keypoint_counts_out_of_range(cuda_device):
    dev, lib = cuda_device, nat.load()
    head = hr.build_model('dips', dev, 4).iegmn_original.packed_head(dev)
    m = torch.empty(64, 64, 64, dtype=F64, device=dev)
    for K in (65, -1):
        s = nat.EqdHeadParams.from_buffer_copy(head.struct)
        s.n_heads = K
        assert lib.eqd_head_fold(C.byref(s), nat.ptr(m), None) == -2          # EQD_ERR_UNSUPPORTED


# ---- backward kernel --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('K', KS)
def test_bwd_head_vs_manual_oracle(K, cuda_device):
    dev, lib = cuda_device, nat.load()
    model = hr.build_model('dips', dev, K, seed=K)
    eng = TrainEngine(model)
    g = gio.make_batch(_pairs('ragged3') + _pairs('sizes'), dev)
    fwd = eng.forward(g)
    torch.cuda.synchronize()
    plan = fwd['plan']
    B, N, NL = plan.n_pairs, plan.N, plan.N_l
    gen = torch.Generator(device=dev).manual_seed(700 + K)
    dcoors = (torch.randn(NL, 3, generator=gen, device=dev) * 0.05).contiguous()
    dkp = (torch.randn(2 * B, K, 3, generator=gen, device=dev) * 0.05).double().contiguous()
    ws_bytes = int(lib.eqd_bwd_head_workspace_bytes_k(N, plan.n_node_tiles, B, K))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)

    def run():
        dh = torch.full((N, 64), float('nan'), device=dev)
        dx = torch.full((N, 3), float('nan'), dtype=F64, device=dev)
        dpre = torch.full((N, 64), float('nan'), device=dev)
        gk, gq = torch.zeros(K * 64, 64, device=dev), torch.zeros(K * 64, 64, device=dev)
        nat.check(lib.eqd_bwd_head(C.byref(plan.struct), C.byref(fwd['head'].struct), nat.ptr(fwd['h']), nat.ptr(fwd['x64']),
                                   nat.ptr(fwd['cov']), nat.ptr(fwd['x_lig_in']), nat.ptr(dcoors), nat.ptr(dkp), None, None,
                                   nat.ptr(ws), ws_bytes, nat.ptr(dh), nat.ptr(dx), nat.ptr(dpre), nat.ptr(gk), nat.ptr(gq),
                                   None), 'eqd_bwd_head')
        return dh, dx, dpre, gk, gq

    dh, dx, _, gk, gq = _twice(run)
    assert torch.isfinite(dh).all() and torch.isfinite(dx).all()
    status = fwd['status_host'][:B].numpy()
    clean = [b for b in range(B) if status[b] == 0]
    assert len(clean) >= B - 2, status                       # the two pairs with a one-node protein may be flagged
    sd, cfg = _sd_np(model), _cfg(hr.args_with('dips', K))
    seg = [int(v) for v in plan.seg_ptr_host]
    h64, x64, xin = fwd['h'].double().cpu().numpy(), fwd['x64'].cpu().numpy(), fwd['x_lig_in'].double().cpu().numpy()
    dco, dk = dcoors.double().cpu().numpy(), dkp.cpu().numpy()
    G = {'wm': np.zeros((64, 64)), 'bm': np.zeros(64), 'wk': np.zeros((K, 64, 64)), 'wq': np.zeros((K, 64, 64))}
    worst = 0.0
    for b in clean:
        (la, lb), (ra, rb) = (seg[b], seg[b + 1]), (seg[B + b], seg[B + b + 1])
        c = bm.head_forward(sd, cfg, h64[la:lb], x64[la:lb], h64[ra:rb], x64[ra:rb])
        dY = bm.kabsch_bwd(c, xin[la:lb], dco[la:lb], (dk[b], dk[B + b]))
        dh_ref, dx_ref = bm.keypoints_bwd(cfg, c, dY, G)
        for side, (a, z) in enumerate(((la, lb), (ra, rb))):
            worst = max(worst, _rel(dh[a:z], dh_ref[side]), _rel(dx[a:z], dx_ref[side]))
    print(f'\nbwd head K={K}: worst dh / dx error {worst:.2e}')
    assert worst <= 1e-5
    if len(clean) == B:
        assert _rel(gk, G['wk'].reshape(K * 64, 64)) <= 1e-5 and _rel(gq, G['wq'].reshape(K * 64, 64)) <= 1e-5


# ---- exact EMD --------------------------------------------------------------------------------------------------------

def _c_smem_cap(M):
    """Largest pocket whose fp64 cost matrix the transport solver keeps in shared memory for M keypoints (ot_layout in
    csrc/losses.cu)."""
    fixed = lambda c: (c * 6 + M * 6 + c + 2 * M + M * 64 + 64) * 8 + (4 * c + 5 * M + 64) * 4 + M * 64 * 2 + c * M + 256
    c = 1
    while fixed(c + 1) + (c + 1) * M * 8 <= 227 * 1024 - 2048:
        c += 1
    return c


def test_shared_memory_cap_at_50_keypoints():
    assert _c_smem_cap(50) == 370          # the layout of the shipped K (tests/test_gpu_losses.py LAYOUT_BATCHES)


@pytest.mark.parametrize('K', KS)
def test_emd_vs_highs(K, cuda_device):
    dev = cuda_device
    cap = min(_c_smem_cap(K) + 1, 1024)
    W = dict(w_ot=float(np.float32(0.37)), w_int=float(np.float32(3.1)), sigma=17.0, ct=6.5)
    for pockets in ([4, 48, 133, 398], [cap, 7]):
        rng = np.random.default_rng([K, len(pockets)])
        B = len(pockets)
        sizes = [(20 + 3 * b, 25 + 2 * b) for b in range(B)]
        pl = [rng.normal(0, 12, (n, 3)).astype(np.float32) for n in pockets]
        pr = [rng.normal(0, 12, (n, 3)).astype(np.float32) for n in pockets]
        kp = rng.normal(0, 15, (2 * B, K, 3))
        pred = np.concatenate([rng.normal(0, 6, (a, 3)) for a, _ in sizes]).astype(np.float32)
        bl = [rng.normal(0, 6, (a, 3)).astype(np.float32) for a, _ in sizes]
        br = [rng.normal(2, 6, (r, 3)).astype(np.float32) for _, r in sizes]
        plan = _plan(sizes, dev)
        t = lambda L: [torch.from_numpy(a) for a in L]
        tgt = PocketBatch(t(bl), t(br), t(pl), t(pr), dev)

        def run():
            res = device_losses(plan, torch.from_numpy(pred).to(dev), torch.from_numpy(kp).to(dev), tgt, W['w_ot'],
                                W['w_int'], W['sigma'], W['ct'])
            return res['parts'].clone(), res['plan'].clone(), res['dkeypts'], res['dcoors'], res['total'], res['err']

        parts, flow, dk, _, _, err = _twice(run)
        check_loss_status({'err': err})
        assert dk.shape == (2 * B, K, 3) and flow.shape == (sum(pockets), K)
        parts, flow, dk = parts.cpu().numpy(), flow.cpu().numpy(), dk.cpu().numpy()
        p0 = 0
        for b, n in enumerate(pockets):
            cost = lo.sq_dist_mat(pl[b], kp[b]) + lo.sq_dist_mat(pr[b], kp[B + b])
            x = flow[p0:p0 + n]
            p0 += n
            lo.ot_certify(cost, x)
            opt = lo.ot_emd(cost)[0]
            assert abs(parts[b, 1] - opt) <= 1e-9 * max(abs(opt), 1.0), (K, n, parts[b, 1], opt)
            T = x.astype(np.float64) / (K * n)
            gsc = 2.0 * W['w_ot'] / B
            for row, P in ((b, pl[b]), (B + b, pr[b])):
                diff = kp[row][None, :, :] - P.astype(np.float64)[:, None, :]
                ref = gsc * (T[:, :, None] * diff).sum(0)
                assert (np.abs(dk[row] - ref) <= 1e-12 * gsc * (T[:, :, None] * np.abs(diff)).sum(0)).all(), (K, n, row)


# ---- whole models -----------------------------------------------------------------------------------------------------

def _targets(pairs, K, seed=3):
    rng = np.random.default_rng(seed)
    return [{'c': rng.normal(0, 5, (len(l['res_feat']), 3)), 'yl': rng.normal(0, 10, (K, 3)),
             'yr': rng.normal(0, 10, (K, 3))} for l, r in pairs]


def _coord_bound(ref):
    return 2e-3 * max(1.0, float(np.abs(ref).max()) / 100)


@pytest.mark.parametrize('K', [25, 64])
@pytest.mark.parametrize('ds', ['db5', 'dips'])
def test_module_forward_graph_replay_and_training_vs_fp64(ds, K, cuda_device):
    dev = cuda_device
    args = hr.args_with(ds, K)
    model = hr.build_model(ds, dev, K, seed=K)
    pairs = _model_pairs(ds, 'ragged3')
    g = gio.make_batch(pairs, dev)
    with torch.no_grad():
        coors, kp_l, kp_r, rot, trans = model(g, epoch=0)
    assert kp_l[0].shape == (K, 3) and kp_r[-1].shape == (K, 3)
    got = torch.cat(coors)
    plan = model.iegmn_original.last_outputs['plan']
    co_ref, Y, R, _ = hr.model_forward(_fp64_state(model), args, _oracle_inputs(g, plan))
    cr = co_ref.numpy()
    err = float(np.abs(got.cpu().double().numpy() - cr).max())
    print(f'\nforward {ds} K={K}: max |coors - fp64| = {err:.3e}')
    assert err <= _coord_bound(cr)
    assert float(np.abs(torch.stack(rot).cpu().double().numpy() - R.numpy()).max()) <= 2e-4
    kp = torch.cat([torch.stack(kp_l), torch.stack(kp_r)]).cpu().double().numpy()
    assert float(np.abs(kp - Y.numpy()).max()) <= _coord_bound(Y.numpy())
    res = model.graphed(g).launch().result()
    assert torch.equal(torch.cat(res[0]), got)
    assert all(torch.equal(a, b) for a, b in zip(res[1] + res[2], kp_l + kp_r))
    # training: loss.backward() through the module, twice (bitwise), against torch.autograd on the fp64 restatement
    model.train()
    tg = _targets(pairs, K)
    g, fwd, loss, coors, grads = _run_module(model, pairs, tg, dev, 11)
    _, _, loss2, coors2, grads2 = _run_module(model, pairs, tg, dev, 11)
    assert torch.equal(loss, loss2) and torch.equal(coors, coors2) and all(torch.equal(grads[n], grads2[n]) for n in grads)
    sd = _fp64_state(model, requires_grad=True)
    co_ref, Y, _, _ = hr.model_forward(sd, args, _oracle_inputs(g, fwd['plan']))
    B = fwd['plan'].n_pairs
    loss_ref = _loss(co_ref, (Y[:B], Y[B:]), tg, fwd['plan'].n_lig_list)
    loss_ref.backward()
    assert abs(loss.item() - loss_ref.item()) < 1e-3 * abs(loss_ref.item())
    got = {n: q.cpu().double().numpy() for n, q in grads.items()}
    assert got['iegmn_original.att_mlp_key_ROT.0.weight'].shape == (64 * K, 64)
    bad = _grad_mismatches(got, {k: v.grad.numpy() for k, v in sd.items()})
    assert not bad, bad


@pytest.mark.parametrize('K', [25, 64])
@pytest.mark.parametrize('ds', ['db5', 'dips'])
def test_fused_trainer_step_matches_the_module_path(ds, K, cuda_device):
    from equidock_public_b200.training import DataParallelTrainer
    dev = cuda_device
    rng = np.random.default_rng(12)
    pairs = [synthetic.synthetic_pair(rng, a, b, 10) for a, b in [(60, 75), (90, 50)]]
    g = gio.make_batch(pairs, dev)
    bl = [torch.from_numpy(p[0]['x']) for p in pairs]
    br = [torch.from_numpy(p[1]['x'] + 8.0) for p in pairs]
    pk = [torch.from_numpy((0.5 * (p[0]['x'][:9] + p[1]['x'][:9] + 8.0)).astype(np.float32)) for p in pairs]
    tgt = PocketBatch(bl, br, pk, pk, dev)
    m1 = hr.build_model(ds, dev, K, seed=4).train()
    m2 = hr.build_model(ds, dev, K, seed=4).train()
    tr = DataParallelTrainer(m1, lr=1e-3, weight_decay=1e-4, clip=1e30)
    r1 = tr.step(g, tgt)
    coors, kl, kr, _, _ = m2(g, epoch=0)
    plan = m2.iegmn_original.last_outputs['plan']
    kp = torch.cat([torch.stack(kl), torch.stack(kr)]).double()
    res = device_losses(plan, torch.cat(coors), kp, tgt, 1.0, 10.0, 25.0, 10.0)
    assert res['dkeypts'].shape == (4, K, 3) and res['plan'].shape == (18, K)
    ((torch.cat(coors) * res['dcoors']).sum() + (kp * res['dkeypts']).sum()).backward()
    assert abs(float(r1['loss'][0]) - float(res['total'][0])) < 1e-6 * max(1.0, abs(float(res['total'][0])))
    by_param = {id(q): v for q, v in zip(tr.layout.params, tr.layout.views(tr.flat_g))}
    flat = {n: by_param[id(q)].double().cpu().numpy() for n, q in m1.named_parameters()}
    ref = {n: q.grad.detach().double().cpu().numpy() for n, q in m2.named_parameters()}
    bad = _grad_mismatches(flat, ref)
    assert not bad, bad


def test_training_with_dropout_vs_fp64_under_the_same_masks(cuda_device):
    dev, K, p = cuda_device, 25, 0.25
    args = hr.args_with('dips', K, dropout=p)
    model = hr.build_model('dips', dev, K, seed=5, dropout=p).train()
    pairs = _model_pairs('dips', 'ragged3')
    tg = _targets(pairs, K)
    g, fwd, loss, coors, grads = _run_module(model, pairs, tg, dev, 11)
    _, _, loss2, coors2, grads2 = _run_module(model, pairs, tg, dev, 11)
    assert torch.equal(loss, loss2) and torch.equal(coors, coors2) and all(torch.equal(grads[n], grads2[n]) for n in grads)
    _, _, loss3, _, _ = _run_module(model, pairs, tg, dev, 12)
    assert not torch.equal(loss, loss3)
    plan, d0 = fwd['plan'], fwd['dropout_layers'][0].dropout
    masks = dm.BatchMasks(p, d0.seed, 0, plan.N, plan.E, int(args['iegmn_n_lays']))
    sd = _fp64_state(model, requires_grad=True)
    co_ref, Y, _, _ = hr.model_forward(sd, args, _oracle_inputs(g, plan), masks)
    B = plan.n_pairs
    loss_ref = _loss(co_ref, (Y[:B], Y[B:]), tg, plan.n_lig_list)
    loss_ref.backward()
    cr = co_ref.detach().numpy()
    assert np.abs(coors.cpu().numpy() - cr).max() < _coord_bound(cr)
    assert abs(loss.item() - loss_ref.item()) < 1e-3 * abs(loss_ref.item())
    bad = _grad_mismatches({n: q.cpu().double().numpy() for n, q in grads.items()}, {k: v.grad.numpy() for k, v in sd.items()})
    assert not bad, bad
