"""Cost of the keypoint count num_att_heads = K (25, 50, 64), the models alternated in one process:
  - inference: pairs/s of bench.py's `db5-shaped` batch (330 pairs of 200 + 200 residues, k = 10, the 8-layer DIPS
    checkpoint) under CUDA-graph replay, and the keypoint head alone on that batch (eqd_keypoints + eqd_kabsch_apply on
    the last layer's outputs, CUDA events);
  - training: one fused DataParallelTrainer step on the shape of bench.py's `train` workload (32 ragged DIPS-shaped pairs,
    the 5-layer shared DB5 model).
The K-head key / query projections are seeded (tests/heads_ref.build_model).  The card name and power limit are read in
the same run.

    python scripts/heads_cost.py [--reps 6] [--replays 20] [--steps 10]
"""
import argparse
import ctypes as C
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), HERE]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
import bench_train  # noqa: E402
import heads_ref as hr  # noqa: E402
from dropout_cost import card  # noqa: E402
from equidock_public_b200 import _native as nat  # noqa: E402
from equidock_public_b200 import hetero_graph as hg  # noqa: E402
from equidock_public_b200 import synthetic  # noqa: E402
from equidock_public_b200.losses import PocketBatch  # noqa: E402
from equidock_public_b200.training import DataParallelTrainer  # noqa: E402
from norm_options_cost import timed  # noqa: E402

KS = (25, 50, 64)


def head_call(model, batch, dev):
    """A closure that runs the keypoint head (eqd_keypoints + eqd_kabsch_apply) on the last-layer outputs of one eager
    forward of ``batch``."""
    lib = nat.load()
    net = model.iegmn_original
    with torch.no_grad():
        model(batch, epoch=0)
    out = net.last_outputs
    plan, head = out['plan'], net.packed_head(dev)
    B, N, K = plan.n_pairs, plan.N, head.n_heads
    ws_bytes = int(lib.eqd_workspace_bytes_k(N, plan.n_node_tiles, B, K))
    f64 = dict(dtype=torch.float64, device=dev)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    kp, ym, cov = torch.empty(2 * B, K, 3, **f64), torch.empty(2 * B, 3, **f64), torch.empty(B, 9, **f64)
    rot, trans = torch.empty(B, 9, device=dev), torch.empty(B, 3, device=dev)
    lig, sing = torch.empty(plan.N_l, 3, device=dev), torch.empty(B, 3, **f64)
    status = torch.zeros(B, dtype=torch.int32, device=dev)
    xl = out['x64'][:plan.N_l].float().contiguous()
    st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    g, hp = C.byref(plan.struct), C.byref(head.struct)

    def run():
        nat.check(lib.eqd_keypoints(g, hp, nat.ptr(out['h']), nat.ptr(out['x64']), nat.ptr(ws), ws_bytes, nat.ptr(kp),
                                    nat.ptr(ym), nat.ptr(cov), st), 'eqd_keypoints')
        nat.check(lib.eqd_kabsch_apply(g, nat.ptr(cov), nat.ptr(ym), nat.ptr(xl), None, nat.ptr(rot), nat.ptr(trans),
                                       nat.ptr(lig), nat.ptr(sing), nat.ptr(status), st), 'eqd_kabsch_apply')
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=6)
    ap.add_argument('--replays', type=int, default=20)
    ap.add_argument('--steps', type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('heads_cost.py measures on a CUDA device only')
    dev = torch.device('cuda', 0)
    n_inf = 330
    pairs = [synthetic.synthetic_pair(np.random.default_rng([0, i]), n_l, n_r, 10)
             for i, (n_l, n_r) in enumerate(bench.pair_sizes('db5-shaped', n_inf))]
    batch = hg.batch_pairs(synthetic.to_torch_pairs(pairs)).to(dev)
    graphs, heads = {}, {}
    for K in KS:
        model = hr.build_model('dips', dev, K, seed=0)
        heads[K] = head_call(model, batch, dev)
        graphs[K] = model.graphed(batch)
    tpairs = [synthetic.synthetic_pair(np.random.default_rng([1, i]), n_l, n_r, 10)
              for i, (n_l, n_r) in enumerate(bench.pair_sizes('train', 32))]
    tg = [bench_train.make_targets(p, np.random.default_rng([0, 7, i])) for i, p in enumerate(tpairs)]
    tbatch = hg.batch_pairs(synthetic.to_torch_pairs(tpairs)).to(dev)
    tl = lambda key: [torch.from_numpy(t[key]) for t in tg]
    targets = PocketBatch(tl('bound_lig'), tl('bound_rec'), tl('pocket_lig'), tl('pocket_rec'), dev)
    trainers = {K: DataParallelTrainer(hr.build_model('db5', dev, K, seed=0).train(), lr=1e-4, weight_decay=1e-4,
                                       clip=100.0) for K in KS}
    for K in KS:                                 # warm-up: module loads, workspaces, packed weights
        for _ in range(3):
            graphs[K].launch().result()
            heads[K]()
            trainers[K].step(tbatch, targets)
    torch.cuda.synchronize()
    inf, head, step = ({K: [] for K in KS} for _ in range(3))
    for _ in range(a.reps):
        for K in KS:                             # alternated: every K sees the same clocks and neighbours
            inf[K].append(n_inf / (timed(lambda: graphs[K].launch().result(), a.replays) / 1e3))
            head[K].append(timed(heads[K], 10 * a.replays))
            step[K].append(timed(lambda: trainers[K].step(tbatch, targets), a.steps))
    med = lambda d: {f'K={K}': float(np.median(v)) for K, v in d.items()}
    reps = lambda d: {f'K={K}': v for K, v in d.items()}
    print(json.dumps({'card': card(), 'db5_shaped_pairs_per_s': med(inf), 'db5_shaped_head_ms': med(head),
                      'train_ms_per_step': med(step), 'db5_shaped_pairs_per_s_reps': reps(inf),
                      'db5_shaped_head_ms_reps': reps(head), 'train_ms_per_step_reps': reps(step)}))


if __name__ == '__main__':
    main()
