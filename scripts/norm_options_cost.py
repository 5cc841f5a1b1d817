"""Cost of the coordinate LayerNorm (layer_norm_coors='LN', coors_mlp.3), its two modes alternated in one process:
  - inference: pairs/s of bench.py's `db5-shaped` batch (330 pairs of 200 + 200 residues, k = 10, the 8-layer DIPS
    checkpoint) under CUDA-graph replay;
  - training: one fused DataParallelTrainer step on the shape of bench.py's `train` workload (32 ragged DIPS-shaped pairs,
    the 5-layer shared DB5 model).
The LN models carry seeded gamma / beta (tests/layer_norm_ref.build_model).  The card name and power limit are read in the
same run.

    python scripts/norm_options_cost.py [--reps 6] [--replays 20] [--steps 10]
"""
import argparse
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
import layer_norm_ref as nr  # noqa: E402
from dropout_cost import card  # noqa: E402
from equidock_public_b200 import hetero_graph as hg  # noqa: E402
from equidock_public_b200 import synthetic  # noqa: E402
from equidock_public_b200.losses import PocketBatch  # noqa: E402
from equidock_public_b200.training import DataParallelTrainer  # noqa: E402

MODES = ('0', 'LN')


def timed(fn, n):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(n):
        fn()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=6)
    ap.add_argument('--replays', type=int, default=20)
    ap.add_argument('--steps', type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('norm_options_cost.py measures on a CUDA device only')
    dev = torch.device('cuda', 0)
    n_inf = 330
    pairs = [synthetic.synthetic_pair(np.random.default_rng([0, i]), n_l, n_r, 10)
             for i, (n_l, n_r) in enumerate(bench.pair_sizes('db5-shaped', n_inf))]
    batch = hg.batch_pairs(synthetic.to_torch_pairs(pairs)).to(dev)
    graphs = {}
    for m in MODES:
        model = nr.build_model('dips', dev, nr.args_with('dips', m), seed=0)
        graphs[m] = model.graphed(batch)
    tpairs = [synthetic.synthetic_pair(np.random.default_rng([1, i]), n_l, n_r, 10)
              for i, (n_l, n_r) in enumerate(bench.pair_sizes('train', 32))]
    tg = [bench_train.make_targets(p, np.random.default_rng([0, 7, i])) for i, p in enumerate(tpairs)]
    tbatch = hg.batch_pairs(synthetic.to_torch_pairs(tpairs)).to(dev)
    tl = lambda key: [torch.from_numpy(t[key]) for t in tg]
    targets = PocketBatch(tl('bound_lig'), tl('bound_rec'), tl('pocket_lig'), tl('pocket_rec'), dev)
    trainers = {m: DataParallelTrainer(nr.build_model('db5', dev, nr.args_with('db5', m), seed=0).train(), lr=1e-4,
                                       weight_decay=1e-4, clip=100.0) for m in MODES}
    for m in MODES:                              # warm-up: module loads, workspaces, packed weights
        for _ in range(3):
            graphs[m].launch().result()
            trainers[m].step(tbatch, targets)
    torch.cuda.synchronize()
    inf = {m: [] for m in MODES}
    step = {m: [] for m in MODES}
    for _ in range(a.reps):
        for m in MODES:                          # alternated: both see the same clocks and neighbours
            inf[m].append(n_inf / (timed(lambda: graphs[m].launch().result(), a.replays) / 1e3))
            step[m].append(timed(lambda: trainers[m].step(tbatch, targets), a.steps))
    med = lambda d: {f'layer_norm_coors={m}': float(np.median(v)) for m, v in d.items()}
    print(json.dumps({'card': card(), 'db5_shaped_pairs_per_s': med(inf), 'train_ms_per_step': med(step),
                      'db5_shaped_pairs_per_s_reps': {m: v for m, v in inf.items()},
                      'train_ms_per_step_reps': {m: v for m, v in step.items()},
                      'inference_cost': float(np.median(inf['0']) / np.median(inf['LN']) - 1.0),
                      'train_cost': float(np.median(step['LN']) / np.median(step['0']) - 1.0)}))


if __name__ == '__main__':
    main()
