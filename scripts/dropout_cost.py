"""Training-step time with dropout off (p = 0) and on (p = 0.25), alternated in one process, on the shape of bench.py's
`train` workload: 32 ragged DIPS-shaped pairs, the 5-layer shared IEGMN of the DB5 checkpoint, one fused
DataParallelTrainer step (forward with stash, device losses, CUDA backward, clip + Adam).  With dropout on, the forward
runs every layer on the fp32 CUDA-core kernels and the fp32 kernels of both directions draw Philox masks; this prints
what that costs.  The card name and power limit are read in the same run.

    python scripts/dropout_cost.py [--steps 20] [--reps 6]
"""
import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
import bench_train  # noqa: E402
import golden_io as gio  # noqa: E402
from equidock_public_b200 import hetero_graph as hg  # noqa: E402
from equidock_public_b200 import synthetic  # noqa: E402
from equidock_public_b200.losses import PocketBatch  # noqa: E402
from equidock_public_b200.training import DataParallelTrainer  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--reps', type=int, default=6)
    ap.add_argument('--pairs', type=int, default=32)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('dropout_cost.py measures on a CUDA device only')
    dev = torch.device('cuda', 0)
    sizes = bench.pair_sizes('train', a.pairs)
    pairs = [synthetic.synthetic_pair(np.random.default_rng([0, i]), n_l, n_r, 10) for i, (n_l, n_r) in enumerate(sizes)]
    tg = [bench_train.make_targets(p, np.random.default_rng([0, 7, i])) for i, p in enumerate(pairs)]
    batch = hg.batch_pairs(synthetic.to_torch_pairs(pairs)).to(dev)
    tl = lambda key: [torch.from_numpy(t[key]) for t in tg]
    targets = PocketBatch(tl('bound_lig'), tl('bound_rec'), tl('pocket_lig'), tl('pocket_rec'), dev)
    trainers = {}
    for p in (0.0, 0.25):
        args = gio.load_args('db5')
        args['dropout'] = p
        model = gio.build_model('db5', dev, args=args)
        trainers[p] = DataParallelTrainer(model, lr=1e-4, weight_decay=1e-4, clip=100.0)
    torch.manual_seed(0)
    for tr in trainers.values():                 # warm-up: module loads, workspaces, packed weights
        for _ in range(3):
            tr.step(batch, targets)
    torch.cuda.synchronize()
    times = {p: [] for p in trainers}
    for _ in range(a.reps):
        for p, tr in trainers.items():          # alternated: both see the same clocks and neighbours
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(a.steps):
                tr.step(batch, targets)
            t1.record()
            t1.synchronize()
            times[p].append(t0.elapsed_time(t1) / a.steps)
    med = {p: float(np.median(v)) for p, v in times.items()}
    print(json.dumps({'card': card(), 'pairs_per_step': a.pairs, 'layers': 5, 'steps_per_rep': a.steps,
                      'ms_per_step': {f'p={p}': v for p, v in med.items()},
                      'ms_per_step_reps': {f'p={p}': v for p, v in times.items()},
                      'dropout_cost': med[0.25] / med[0.0] - 1.0}))


if __name__ == '__main__':
    main()
