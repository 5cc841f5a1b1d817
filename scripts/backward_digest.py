"""Flat parameter gradient and graph-input gradients of the whole-model backward (TrainEngine.backward) on fixed seeded
batches of both checkpoints, saved as .npy and printed as sha256.  Run it at two commits (each tree with its own built
library) and compare the files to check that a change leaves the whole-model backward bitwise unchanged.

    python scripts/backward_digest.py OUT_DIR
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)

import golden_io as gio  # noqa: E402
from equidock_public_b200 import synthetic  # noqa: E402
from equidock_public_b200.training import TrainEngine  # noqa: E402


def digest(ds, dev, out_dir):
    args = dict(gio.load_args(ds), x_connection_init=0.3)
    model = gio.build_model(ds, dev, args=args).train()
    rng = np.random.default_rng(5)
    pairs = [synthetic.synthetic_pair(rng, a, b, 10) for a, b in [(40, 131), (129, 20), (64, 64), (300, 257)]]
    g = gio.make_batch(pairs, dev)
    eng = TrainEngine(model)
    fwd = eng.forward(g)
    t = lambda ref, dt: torch.from_numpy(rng.normal(0, 1, tuple(ref.shape))).to(dev, dt)
    inputs = {}
    flat = eng.backward(fwd, t(fwd['ligand_coors'], torch.float32), t(fwd['keypts'], torch.float64),
                        t(fwd['rotation'], torch.float32), t(fwd['translation'], torch.float32),
                        d_x_out=t(fwd['x64'], torch.float64), d_h_out=t(fwd['h'], torch.float32), inputs_out=inputs)
    torch.cuda.synchronize()
    res = {}
    for name, v in [('flat', flat)] + sorted(inputs.items()):
        a = v.detach().cpu().numpy()
        np.save(os.path.join(out_dir, f'{ds}_{name}.npy'), a)
        res[name] = hashlib.sha256(a.tobytes()).hexdigest()
    return res


def main():
    out_dir = sys.argv[1]
    os.makedirs(out_dir, exist_ok=True)
    dev = torch.device('cuda:0')
    res = {ds: digest(ds, dev, out_dir) for ds in ('db5', 'dips')}
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
