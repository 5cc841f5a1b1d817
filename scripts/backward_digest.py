"""Forward outputs and gradients of the CUDA training path on fixed seeded batches, saved as .npy and printed as sha256.
Run it at two commits (each tree with its own built library) and compare the files to check that a change leaves the
forward and backward bitwise unchanged.

Each configuration runs the whole-model backward (TrainEngine.backward: flat parameter gradient and graph-input
gradients) on both checkpoints, and one IEGMN_Layer autograd call each of the 69-wide layer 0 and a 64-wide layer of
the DIPS checkpoint (outputs, gradients of the ten inputs and of the layer's parameters).  Besides the shipped
configuration they are dropout 0.25 under a fixed torch.manual_seed, layer_norm_coors='LN' and final_h_layer_norm='LN',
which run the fp32 forward kernels and their backward recomputes.

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
from equidock_public_b200.hetero_graph import LIGAND, LL, RECEPTOR, RR  # noqa: E402
from equidock_public_b200.training import TrainEngine  # noqa: E402

CONFIGS = {'default': {}, 'dropout': {'dropout': 0.25}, 'coors_ln': {'layer_norm_coors': 'LN'},
           'final_ln': {'final_h_layer_norm': 'LN'}}
FWD_KEYS = ('ligand_coors', 'keypts', 'rotation', 'translation', 'x64', 'h')


def _save(out_dir, tag, tensors):
    res = {}
    for name, v in tensors:
        a = v.detach().cpu().numpy()
        np.save(os.path.join(out_dir, f'{tag}_{name}.npy'), a)
        res[name] = hashlib.sha256(a.tobytes()).hexdigest()
    return res


def _model(ds, dev, cfg):
    args = dict(gio.args_with(ds, **CONFIGS[cfg]), x_connection_init=0.3)
    return gio.build_model(ds, dev, args=args).train()


def model_digest(ds, cfg, dev, out_dir):
    model = _model(ds, dev, cfg)
    rng = np.random.default_rng(5)
    pairs = [synthetic.synthetic_pair(rng, a, b, 10) for a, b in [(40, 131), (129, 20), (64, 64), (300, 257)]]
    g = gio.make_batch(pairs, dev)
    eng = TrainEngine(model)
    torch.manual_seed(11)
    fwd = eng.forward(g)
    t = lambda ref, dt: torch.from_numpy(rng.normal(0, 1, tuple(ref.shape))).to(dev, dt)
    inputs = {}
    flat = eng.backward(fwd, t(fwd['ligand_coors'], torch.float32), t(fwd['keypts'], torch.float64),
                        t(fwd['rotation'], torch.float32), t(fwd['translation'], torch.float32),
                        d_x_out=t(fwd['x64'], torch.float64), d_h_out=t(fwd['h'], torch.float32), inputs_out=inputs)
    torch.cuda.synchronize()
    return _save(out_dir, f'{cfg}_{ds}', [(f'fwd_{k}', fwd[k]) for k in FWD_KEYS] + [('flat', flat)]
                 + sorted(inputs.items()))


def layer_digest(li, cfg, dev, out_dir):
    """One IEGMN_Layer call under autograd on layer li of the DIPS checkpoint with seeded inputs and a seeded linear loss
    of its four outputs."""
    lay = _model('dips', dev, cfg).iegmn_original.iegmn_layers[li]
    rng = np.random.default_rng(7)
    pairs = [synthetic.synthetic_pair(rng, a, b, 10) for a, b in [(40, 131), (129, 20), (64, 64)]]
    g = gio.make_batch(pairs, dev)
    rnd = lambda *shape: torch.from_numpy(rng.normal(0, 1, shape)).to(dev, torch.float32)
    ins = []
    for nt, xk, et in ((LIGAND, 'new_x', LL), (RECEPTOR, 'x', RR)):
        x = g.nodes[nt].data[xk].to(torch.float32)
        n = x.shape[0]
        ins += [x.clone(), rnd(n, lay.h_feats_dim), rnd(n, 69), g.edges[et].data['he'], x.clone()]
    for v in ins:
        v.requires_grad_(True)
    torch.manual_seed(13)
    outs = lay(g, *ins)
    loss = sum((o.double() * torch.from_numpy(rng.normal(0, 1, tuple(o.shape))).to(dev)).sum() for o in outs)
    loss.backward()
    torch.cuda.synchronize()
    return _save(out_dir, f'{cfg}_layer{li}', [(f'out{i}', o) for i, o in enumerate(outs)]
                 + [(f'd_in{i}', v.grad) for i, v in enumerate(ins)]
                 + [(f'd_{n}', p.grad) for n, p in lay.named_parameters() if p.grad is not None])


def main():
    out_dir = sys.argv[1]
    os.makedirs(out_dir, exist_ok=True)
    dev = torch.device('cuda:0')
    res = {}
    for cfg in CONFIGS:
        for ds in ('db5', 'dips'):
            res[f'{cfg}/{ds}'] = model_digest(ds, cfg, dev, out_dir)
        for li in (0, 1):
            res[f'{cfg}/layer{li}'] = layer_digest(li, cfg, dev, out_dir)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
