"""GPU: throughput of the two inference precisions (IEGMN.precision 'fp32' = bf16x6, 'bf16x3') in ONE process.

For each of bench.py's inference workloads (db5-shaped, db5-testset, large) two models with the same DIPS weights, one
per precision, each replay CUDA graphs of the same seeded batch (two graphs in flight, as bench.py's timed loop).  The
modes alternate repetition by repetition (the first mode swaps every repetition), each repetition K steps timed with
CUDA events.  Then one eager pass per mode with the engine's stage events gives the mean edge / node stage time of
layer 0 and of the 64-wide layers.  Prints the card, its power limit and max SM clock, one line per workload and a
final JSON line; `nvidia-smi -q` (read-only query) goes to OUT/nvidia-smi-q.txt.

usage: precision_ab.py [--steps K] [--reps R] [--workloads a,b] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np

MODES = ('fp32', 'bf16x3')


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip()


def stage_means(lib, timer, n_layers):
    """{edge_l0, node_l0, edge_l64, node_l64}: mean ms per forward of layer 0's stages and per 64-wide layer."""
    acc = {k: [] for k in ('edge_l0', 'node_l0', 'edge_l64', 'node_l64')}
    for arr in timer.sets:
        for li in range(n_layers):
            e = lib.eqd_event_elapsed_ms(arr[4 * li], arr[4 * li + 1])
            n = lib.eqd_event_elapsed_ms(arr[4 * li + 2], arr[4 * li + 3])
            acc['edge_l0' if li == 0 else 'edge_l64'].append(e)
            acc['node_l0' if li == 0 else 'node_l64'].append(n)
    return {k: float(np.mean(v)) for k, v in acc.items()}


def run_workload(name, steps, reps, dev):
    import torch
    import bench
    import golden_io as gio
    from equidock_public_b200 import engine as engine_mod
    from equidock_public_b200 import hetero_graph as hg
    from equidock_public_b200 import synthetic
    from equidock_public_b200.engine import IEGMNEngine
    wl = bench.WORKLOADS[name]
    sizes = bench.pair_sizes(name, wl['pairs_per_gpu'])
    pairs = [synthetic.synthetic_pair(np.random.default_rng([0, i]), a, b, bench.KNN) for i, (a, b) in enumerate(sizes)]
    host = hg.batch_pairs(synthetic.to_torch_pairs(pairs)).pin_memory()
    sd = gio.load_checkpoint(wl['ckpt'])
    models, graphs = {}, {}
    for mode in MODES:
        m = gio.build_model(wl['ckpt'], dev, sd=sd)
        m.precision = mode
        models[mode] = m
        graphs[mode] = [m.graphed(host.to(dev)) for _ in range(2)]

    def body(mode):
        g = graphs[mode]
        pending = None
        for i in range(steps):
            nxt = g[i & 1].launch()
            if pending is not None:
                pending.raw_result()
            pending = nxt
        return pending.raw_result()

    outs = {}
    for mode in MODES:                      # warm-up; also keeps each mode's outputs of the seeded batch
        for _ in range(3):
            outs[mode] = body(mode)
        outs[mode] = {k: outs[mode][k].clone() for k in ('ligand_coors', 'rotation', 'translation')}
    t_lead = time.perf_counter()
    while time.perf_counter() - t_lead < 1.0:   # clocks ramped before the first timed repetition
        body('fp32')
    ms = {m: [] for m in MODES}
    for r in range(reps):
        order = MODES if r % 2 == 0 else MODES[::-1]
        for mode in order:
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            body(mode)
            e1.record()
            e1.synchronize()
            ms[mode].append(e0.elapsed_time(e1))
    B = len(sizes)
    rate = {m: [B * steps / (t * 1e-3) for t in ms[m]] for m in MODES}
    # per-stage times: one eager pass of `steps` forwards per mode with the engine's stage events
    stages = {}
    orig_forward = IEGMNEngine.forward
    try:
        for mode in MODES:
            timer = engine_mod.NativeStageTimer()
            timer.reserve(steps, wl['n_layers'])
            IEGMNEngine.forward = lambda self, *a, _t=timer, **k: orig_forward(self, *a, stage_timer=_t, **k)
            b = host.to(dev)
            for _ in range(steps):
                models[mode](b, 0)
            torch.cuda.synchronize()
            stages[mode] = stage_means(timer.lib, timer, wl['n_layers'])
            timer.close()
    finally:
        IEGMNEngine.forward = orig_forward
    d = {k: float((outs['bf16x3'][k].double() - outs['fp32'][k].double()).abs().max()) for k in outs['fp32']}
    med = {m: float(np.median(rate[m])) for m in MODES}
    return {'workload': name, 'pairs': B, 'steps': steps, 'reps': reps,
            'pairs_per_s': {m: [round(v, 1) for v in rate[m]] for m in MODES},
            'median_pairs_per_s': med, 'gain': med['bf16x3'] / med['fp32'] - 1.0,
            'stage_ms': stages, 'max_abs_diff_bf16x3_vs_fp32': d}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--reps', type=int, default=6)
    ap.add_argument('--workloads', default='db5-shaped,db5-testset,large')
    ap.add_argument('--out', default=None, help='directory for nvidia-smi-q.txt and precision_ab.json')
    a = ap.parse_args()
    import torch
    dev = torch.device('cuda:0')
    torch.cuda.set_device(dev)
    print(f'card (name, power limit, max SM clock): {card()}', flush=True)
    res = []
    for name in a.workloads.split(','):
        r = run_workload(name, a.steps, a.reps, dev)
        res.append(r)
        s = r['stage_ms']
        print(f"{name}: {r['pairs']} pairs, pairs/s fp32 {r['pairs_per_s']['fp32']} bf16x3 {r['pairs_per_s']['bf16x3']}; "
              f"median {r['median_pairs_per_s']['fp32']:.0f} -> {r['median_pairs_per_s']['bf16x3']:.0f} "
              f"({100 * r['gain']:+.1f} %)", flush=True)
        for m in MODES:
            print(f"  {m:7s} stage ms/forward: layer 0 edge {s[m]['edge_l0']:.3f} node {s[m]['node_l0']:.3f}; "
                  f"64-wide layer edge {s[m]['edge_l64']:.3f} node {s[m]['node_l64']:.3f}", flush=True)
        print(f"  max |bf16x3 - fp32|: {r['max_abs_diff_bf16x3_vs_fp32']}", flush=True)
    summary = {'card': card(), 'results': res}
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        q = subprocess.run(['nvidia-smi', '-q'], capture_output=True, text=True)
        with open(os.path.join(a.out, 'nvidia-smi-q.txt'), 'w') as f:
            f.write(q.stdout)
        with open(os.path.join(a.out, 'precision_ab.json'), 'w') as f:
            json.dump(summary, f, indent=1)
    print(json.dumps({'card': summary['card'], **{r['workload']: {'gain': round(r['gain'], 4), **r['median_pairs_per_s']}
                                                   for r in res}}))


if __name__ == '__main__':
    main()
