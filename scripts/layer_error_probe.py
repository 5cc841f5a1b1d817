"""GPU: single-layer error of the FFMA vs tensor-core node stage, starting every layer from the oracle's exact inputs."""
import os, sys, ctypes as C
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')): sys.path.insert(0, p)
import numpy as np, torch
import golden_io as gio, iegmn_oracle as orc
from equidock_public_b200 import _native as nat
from equidock_public_b200.engine import GraphPlan
dev = torch.device('cuda:0'); lib = nat.load()
ds, name = sys.argv[1], sys.argv[2]
names, pairs, outs, _ = gio.load_pairs(ds)
sd = gio.load_checkpoint(ds); args = gio.load_args(ds); cfg = orc.OracleConfig.from_args(args)
model = gio.build_model(ds, dev)
lig, rec = pairs[name]
trace = []
orc.forward_pair(sd, cfg, lig, rec, trace=trace)          # trace[li] = [ {side0...}, {side1...} ]
g = gio.make_batch([pairs[name]], dev); plan = GraphPlan.from_graph(g, dev, 10); G = C.byref(plan.struct)
N, Nl = plan.N, plan.N_l
f64 = lambda a: np.asarray(a, dtype=np.float64)
emb = f64(sd['iegmn_original.residue_emb_layer.weight'])
h0 = np.concatenate([np.concatenate([emb[np.asarray(s['res_feat']).reshape(-1).astype(int)], np.log(f64(s['mu_r_norm']))], 1) for s in (lig, rec)], 0)
x_orig = np.concatenate([f64(lig['new_x']), f64(rec['x'])], 0)
T = lambda a, dt=torch.float32: torch.from_numpy(np.ascontiguousarray(a)).to(dev, dt)
h0p = torch.zeros(N, 72, device=dev); h0p[:, :69] = T(h0)
x0 = T(x_orig, torch.float64)
h_prev, x_prev = h0, x_orig
for li in range(cfg.n_layers):
    lay = model.iegmn_original.iegmn_layers[li].packed(dev); L = C.byref(lay.struct)
    want_h = np.concatenate([trace[li][0]['h_new'], trace[li][1]['h_new']], 0)
    want_mu = np.concatenate([trace[li][0]['mu'], trace[li][1]['mu']], 0)
    want_ag = np.concatenate([trace[li][0]['msg_aggr'], trace[li][1]['msg_aggr']], 0)
    dhp = lay.dhp
    hin = torch.zeros(N, dhp, device=dev); hin[:, :lay.dh] = T(h_prev)
    xin = T(x_prev, torch.float64)
    proj = torch.zeros(N, 128 + 3 * dhp, device=dev)
    lib.eqd_project(G, L, nat.ptr(hin), dhp, nat.ptr(proj), None)
    aggr = torch.zeros(N, 64, device=dev); xo = torch.zeros(N, 3, device=dev, dtype=torch.float64)
    st = torch.zeros(plan.n_pairs + 1, dtype=torch.int32, device=dev)
    lib.eqd_edge_stage(G, L, nat.ptr(proj), nat.ptr(xin), nat.ptr(x0), nat.ptr(aggr), nat.ptr(xo), nat.ptr(st), None)
    hf = torch.zeros(N, 64, device=dev)
    lib.eqd_node_stage(G, L, None, nat.ptr(hin), dhp, nat.ptr(h0p), nat.ptr(proj), nat.ptr(aggr), None, nat.ptr(hf), None,
                       None)
    torch.cuda.synchronize()
    msg = f'layer {li}: aggr err {np.abs(aggr.cpu().numpy() - want_ag).max():.2e}  FFMA node h err {np.abs(hf.cpu().numpy() - want_h).max():.2e}'
    if lay.dh == 64:
        projt = torch.zeros(N, 320, device=dev)
        kv = torch.zeros(lib.eqd_kv_blocks_bytes(N), dtype=torch.uint8, device=dev)
        lib.eqd_project_tc(G, L, nat.ptr(hin), nat.ptr(projt), nat.ptr(kv), None)
        mu = torch.zeros(N, 64, device=dev); ht = torch.zeros(N, 64, device=dev)
        lib.eqd_attention_tc(G, nat.ptr(projt), nat.ptr(kv), nat.ptr(mu), None)
        lib.eqd_node_mlp_tc(G, L, nat.ptr(hin), nat.ptr(aggr), nat.ptr(mu), nat.ptr(h0p), nat.ptr(ht), None)
        torch.cuda.synchronize()
        msg += f' | TC: proj diff {(projt - proj).abs().max().item():.2e} mu err {np.abs(mu.cpu().numpy() - want_mu).max():.2e} h err {np.abs(ht.cpu().numpy() - want_h).max():.2e} (max|mu| {np.abs(want_mu).max():.2f} max|h| {np.abs(want_h).max():.2f} max|q.k| {float((projt[:, 128:192].double() @ projt[:, 192:256].double().t()).abs().max()):.0f})'
    print(msg, flush=True)
    h_prev = want_h
    x_prev = np.concatenate([trace[li][0]['x_new'], trace[li][1]['x_new']], 0)
