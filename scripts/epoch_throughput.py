"""Training epochs from the host data path vs the device-resident data set (equidock_public_b200/datasets.py).

Builds a seeded archive of DIPS-shaped pairs (bench.py's size distribution, k = 10) with bench_train.make_targets labels,
then times whole shuffled epochs of DataParallelTrainer steps at --batch pairs per step, two ways, alternated in one
process on one GPU:
  host:   PairArchive pairs -> numpy re-posing of every ligand as the reference's data set does it (random_rigid about the
          ligand's mean) -> hetero_graph.batch_pairs -> .to(dev) -> PocketBatch (the plan is derived in trainer.step)
  device: DevicePairDataset.epoch (one gather kernel per batch, re-posing on the device)
Also: the host share of a host-path step (assembly + upload, timed on the host), and the assembly kernel alone
(torch.profiler device time, in a separate profiled pass) with its compulsory bytes over that time.
Prints the card name and power limit with the numbers, and one JSON line.

  python scripts/epoch_throughput.py [--pairs 2048] [--unique 256] [--batch 32] [--reps 3] [--out results/epoch_throughput.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)


def make_archive(path, n_pairs, n_unique, seed):
    """n_pairs entries cycling through n_unique distinct pairs (generating a pair costs far more than storing it)."""
    import bench
    from bench_train import make_targets
    from equidock_public_b200 import synthetic
    from equidock_public_b200.formats import save_pairs
    pairs, labels = [], []
    for i, (n_l, n_r) in enumerate(bench.pair_sizes('train', min(n_unique, n_pairs), seed)):
        rng = np.random.default_rng([seed, i])
        p = synthetic.synthetic_pair(rng, n_l, n_r, 10)
        tg = make_targets(p, rng)
        pairs.append(p)
        labels.append({'pocket_coors': tg['pocket_lig'], 'bound_lig': tg['bound_lig'], 'bound_rec': tg['bound_rec']})
    k = [i % len(pairs) for i in range(n_pairs)]
    save_pairs(path, [pairs[i] for i in k], [labels[i] for i in k])


def host_batch(arch, idx, rng, interval, dev):
    """The host data path of one step, re-posing included (numpy, per pair, as the reference's __getitem__)."""
    import torch
    from equidock_public_b200 import hetero_graph as hg
    from equidock_public_b200 import synthetic
    from equidock_public_b200.losses import PocketBatch
    pairs, bl, br, pl, pr = [], [], [], [], []
    for i in idx:
        lig, rec = arch.pair(int(i))
        lab = arch.labels(int(i))
        R, t = synthetic.random_rigid(rng, interval, np.float64)
        c = lig['x'].astype(np.float64).mean(0, keepdims=True)
        lig = dict(lig, new_x=((lig['x'] - c) @ R.T + t).astype(np.float32))
        pk = np.asarray(lab['pocket_coors'])
        pairs.append(tuple({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in d.items()} for d in (lig, rec)))
        bl.append(torch.from_numpy(np.ascontiguousarray(lab['bound_lig'])))
        br.append(torch.from_numpy(np.ascontiguousarray(lab['bound_rec'])))
        pl.append(torch.from_numpy(((pk - c) @ R.T + t).astype(np.float32)))
        pr.append(torch.from_numpy(np.ascontiguousarray(pk)))
    g = hg.batch_pairs(pairs).to(dev)
    return g, PocketBatch(bl, br, pl, pr, dev)


def assembly_bytes(ds, idx):
    """Compulsory device-memory bytes of one eqd_assemble_batch call (every input byte read once, every output byte
    written once; the binary searches of row_ptr hit cache and are not counted)."""
    o = ds.sizes.offsets(idx)
    B = len(idx)
    N, N_l, E, P, T = int(o['node'][-1]), int(o['node'][B]), int(o['edge'][-1]), int(o['pocket'][-1]), int(o['tile'][-1])
    rd = N * (1 + 12 + 20) + N_l * (12 + 12) + (N - N_l) * 12 + E * (108 + 8) + P * 12 + 4 * o['packed'].size
    wr = N * (4 + 12 + 20 + 4) + N_l * (12 + 12) + (N - N_l) * 12 + E * (108 + 8) + P * 24 + 4 * (2 * B + 1 + 2 * T + B + 1) + B * 96
    return rd + wr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pairs', type=int, default=2048)
    ap.add_argument('--unique', type=int, default=256, help='distinct pairs the archive cycles through')
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--reps', type=int, default=3, help='epochs per path (alternated)')
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--interval', type=float, default=5.0)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    import golden_io as gio
    from equidock_public_b200.datasets import DevicePairDataset
    from equidock_public_b200.formats import PairArchive
    from equidock_public_b200.losses import check_loss_status
    from equidock_public_b200.training import DataParallelTrainer
    if not torch.cuda.is_available():
        raise SystemExit('epoch_throughput: needs a CUDA device')
    dev = torch.device('cuda', 0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = f'{torch.cuda.get_device_name(dev)}, power limit not readable'
    print(f'card: {q}', flush=True)
    tmp = tempfile.mkdtemp(prefix='eqd_epoch_')
    path = os.path.join(tmp, 'pairs.eqd')
    t0 = time.perf_counter()
    make_archive(path, args.pairs, args.unique, args.seed)
    print(f'archive: {args.pairs} DIPS-shaped pairs ({min(args.unique, args.pairs)} distinct), {os.path.getsize(path) / 1e6:.1f} MB, built in {time.perf_counter() - t0:.1f} s', flush=True)
    arch = PairArchive(path)
    t0 = time.perf_counter()
    ds = DevicePairDataset(arch, dev)
    torch.cuda.synchronize()
    upload_s = time.perf_counter() - t0
    print(f'device data set: {ds.nbytes / 1e6:.1f} MB, uploaded (with checks) in {upload_s:.2f} s', flush=True)

    margs = gio.load_args('db5')
    model = gio.build_model('db5', dev, args=margs)
    trainer = DataParallelTrainer(model, lr=1e-4, weight_decay=1e-4, clip=100.0,
                                  pocket_ot_loss_weight=float(margs.get('pocket_ot_loss_weight', 1.0)),
                                  intersection_loss_weight=float(margs.get('intersection_loss_weight', 10.0)),
                                  intersection_sigma=float(margs.get('intersection_sigma', 25.0)),
                                  intersection_surface_ct=float(margs.get('intersection_surface_ct', 10.0)))

    def epoch_host(e):
        rng = np.random.default_rng([args.seed, 99, e])
        host_s, last = 0.0, None
        for idx, _, _ in ds.sizes.epoch_schedule(args.batch, args.seed, e):
            h0 = time.perf_counter()
            g, tgt = host_batch(arch, idx, rng, args.interval, dev)
            host_s += time.perf_counter() - h0
            last = trainer.step(g, tgt)
        return last, host_s

    def epoch_device(e):
        last = None
        for g, tgt in ds.epoch(args.batch, args.seed, e, translation_interval=args.interval):
            last = trainer.step(g, tgt)
        return last, 0.0

    n_steps = len(ds.sizes.epoch_schedule(args.batch, args.seed, 0))
    res = {'host': [], 'device': []}
    host_share = []
    for e, fn in enumerate([epoch_host, epoch_device]):          # warm-up: every shape class, allocator, module loads
        check_loss_status(fn(1000 + e)[0])
    for r in range(args.reps):
        for name, fn in (('host', epoch_host), ('device', epoch_device)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            last, hs = fn(r)
            float(last['loss'][0].item())
            dt = time.perf_counter() - t0
            check_loss_status(last)
            res[name].append(dt)
            if name == 'host':
                host_share.append(hs / dt)
            print(f'rep {r} {name:6s}: epoch {dt:.3f} s = {1e3 * dt / n_steps:.2f} ms/step, '
                  f'{args.pairs / dt:.1f} pairs/s' + (f', host assembly + upload {1e3 * hs / n_steps:.2f} ms/step' if name == 'host' else ''),
                  flush=True)

    # the assembly kernel alone: device time from the profiler, over a fixed set of batches
    from torch.profiler import ProfilerActivity, profile
    sched = ds.sizes.epoch_schedule(args.batch, args.seed, 0)
    for idx, step, first in sched[:4]:
        ds.batch(idx, args.seed, step, args.interval, first)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for idx, step, first in sched:
            ds.batch(idx, args.seed, step, args.interval, first)
        torch.cuda.synchronize()
    kern = [ev for ev in prof.events() if 'assemble_batch_kernel' in ev.name]
    dev_us = sum(ev.device_time for ev in kern)
    nbytes = sum(assembly_bytes(ds, idx) for idx, _, _ in sched)
    kernel = {'launches': len(kern), 'mean_us': dev_us / max(len(kern), 1), 'bytes_per_launch': nbytes / len(sched),
              'GB_per_s': nbytes / (dev_us * 1e-6) / 1e9 if dev_us else None}
    print(f"assembly kernel: {kernel['launches']} launches, mean {kernel['mean_us']:.1f} us, "
          f"{kernel['bytes_per_launch'] / 1e6:.2f} MB moved per launch, {kernel['GB_per_s']:.0f} GB/s "
          f"(data sheet HBM3 peak 3350 GB/s for a 700 W H100 SXM)", flush=True)
    med = {k: float(np.median(v)) for k, v in res.items()}
    line = {'card': q, 'pairs': args.pairs, 'batch': args.batch, 'steps_per_epoch': n_steps, 'reps': args.reps,
            'epoch_s': res, 'median_epoch_s': med, 'pairs_per_s': {k: args.pairs / v for k, v in med.items()},
            'speedup_device_over_host': med['host'] / med['device'], 'host_path_host_share': host_share,
            'dataset_device_bytes': ds.nbytes, 'upload_s': upload_s, 'assembly_kernel': kernel}
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as fh:
            json.dump(line, fh, indent=1)


if __name__ == '__main__':
    main()
