"""GPU: per-kernel times of the 64-wide tensor-core node stage at the bench shape (330 pairs of 200 + 200 nodes, k = 10,
DIPS layer-1 weights): eqd_attention_tc, eqd_node_mlp_tc, eqd_project_tc and the whole eqd_node_stage_tc, each timed with
CUDA events around back-to-back launches after a warm-up.  EQD_LIB_PATH selects the build (A/B of two builds).
usage: node_stage_times.py [launches per kernel, default 300]"""
import ctypes as C, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import torch
import golden_io as gio
from equidock_public_b200 import _native as nat, hetero_graph as hg, synthetic
from equidock_public_b200.engine import GraphPlan

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 300
dev = torch.device('cuda:0')
lib = nat.load()
smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                     capture_output=True, text=True).stdout.strip()
print(f'GPU: {torch.cuda.get_device_name(dev)} | nvidia-smi: {smi} | lib: {nat.LIB_PATH}', flush=True)

net = gio.build_model('dips', dev).iegmn_original
batch = hg.batch_pairs(synthetic.to_torch_pairs(synthetic.synthetic_batch(330, 200, 200, 10, seed=0))).to(dev)
plan = GraphPlan.from_graph(batch, dev, 10)
N = plan.N
G = C.byref(plan.struct)
L1 = net.iegmn_layers[1].packed(dev); L2 = net.iegmn_layers[2].packed(dev)
l1, l2 = C.byref(L1.struct), C.byref(L2.struct)
f32 = dict(dtype=torch.float32, device=dev)
torch.manual_seed(0)
h = torch.randn(N, 64, **f32) * 0.5
h0 = torch.zeros(N, 72, **f32); h0[:, :69] = torch.randn(N, 69, **f32) * 0.5
aggr = torch.randn(N, 64, **f32) * 0.5
proj = torch.zeros(N, 320, **f32); projn = torch.zeros(N, 320, **f32)
kv = torch.zeros(lib.eqd_kv_blocks_bytes(N), dtype=torch.uint8, device=dev)
mu = torch.zeros(N, 64, **f32); hout = torch.zeros(N, 64, **f32)
P = nat.ptr
st = None
assert lib.eqd_project_tc(G, l1, P(h), P(proj), P(kv), st) == 0
# eqd_project_tc overwrites kv, which the attention reads: it projects into the second buffer, from the same h
kvn = kv.clone()

kernels = {
    'eqd_attention_tc': lambda: lib.eqd_attention_tc(G, P(proj), P(kv), P(mu), st),
    'eqd_node_mlp_tc': lambda: lib.eqd_node_mlp_tc(G, l1, P(h), P(aggr), P(mu), P(h0), P(hout), st),
    'eqd_project_tc': lambda: lib.eqd_project_tc(G, l2, P(h), P(projn), P(kvn), st),
    'eqd_node_stage_tc': lambda: lib.eqd_node_stage_tc(G, l1, l2, P(h), P(h0), P(proj), P(aggr), P(kv), P(mu), P(hout),
                                                       P(projn), st),
}
print(f'N = {N} nodes, {plan.n_node_tiles} node tiles, {reps} launches per kernel', flush=True)
for name, fn in kernels.items():
    for _ in range(20):
        assert fn() == 0, name
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record(); b.synchronize()
    print(f'{name:20s} {a.elapsed_time(b) / reps * 1e3:8.1f} us', flush=True)
