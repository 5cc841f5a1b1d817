"""GPU: what asking for the graph's input gradients adds to ``loss.backward()`` through the drop-in module, at the shape
of bench.py's ``train`` workload (32 DIPS-shaped ragged pairs, k = 10, 5-layer shared IEGMN, DB5 checkpoint).

Per step: one forward in training mode (not timed), then ``loss.backward()`` timed with CUDA events; the two modes
(no input requires grad / new_x, x, mu_r_norm and he of both sides require grad) alternate step by step so that both
see the same machine state.  Prints the card, its power limit and, per mode, the median and min..max backward time.

    python scripts/input_grad_cost.py [--steps 40] [--warmup 5] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import numpy as np
import torch

import bench
import golden_io as gio
from equidock_public_b200 import synthetic
from equidock_public_b200.rigid_docking_model import graph_inputs


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ''
    return q or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=40, help='timed steps per mode')
    ap.add_argument('--warmup', type=int, default=5, help='untimed steps per mode')
    ap.add_argument('--pairs', type=int, default=bench.WORKLOADS['train']['pairs_per_gpu'])
    ap.add_argument('--out', default=None, help='also write the result as DIR/input_grad_cost.json')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('input_grad_cost.py measures on a CUDA device; none is visible')
    dev = torch.device('cuda:0')
    wl = bench.WORKLOADS['train']
    model = gio.build_model(wl['ckpt'], dev).train()
    rng = np.random.default_rng(0)
    sizes = bench.pair_sizes('train', args.pairs)
    pairs = [synthetic.synthetic_pair(rng, a, b, 10) for a, b in sizes]
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    times = {False: [], True: []}
    g = gio.make_batch(pairs, dev)
    for step in range(args.warmup + args.steps):
        for want in (False, True):
            for t in graph_inputs(g):
                t.grad = None
                t.requires_grad_(want)
            model.zero_grad(set_to_none=True)
            coors, kp_l, kp_r, rot, trans = model(g, epoch=0)
            loss = sum((c.double() ** 2).mean() for c in coors) + sum((k.double() ** 2).mean() for k in kp_l + kp_r)
            torch.cuda.synchronize()
            ev[0].record()
            loss.backward()
            ev[1].record()
            torch.cuda.synchronize()
            if step >= args.warmup:
                times[want].append(ev[0].elapsed_time(ev[1]))
    res = {'card': card(), 'pairs': len(sizes), 'nodes': int(sum(a + b for a, b in sizes)), 'steps_per_mode': args.steps}
    for want, tag in ((False, 'params_only_ms'), (True, 'with_input_grads_ms')):
        v = np.asarray(times[want])
        res[tag] = {'median': float(np.median(v)), 'min': float(v.min()), 'max': float(v.max())}
    res['added_ms_median'] = res['with_input_grads_ms']['median'] - res['params_only_ms']['median']
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'input_grad_cost.json'), 'w') as fh:
            json.dump(res, fh, indent=1)


if __name__ == '__main__':
    main()
