"""GPU: the tensor-core node MLP of a 64-wide layer (eqd_node_mlp_tc, warpgroup tile chains of 64 rows) against a torch
fp64 restatement of node_mlp, at the tile boundaries and past one round of the resident chains, plus a bit pin at a size
where every chain runs several tiles and prefetches across them."""
import ctypes as C
import hashlib

import numpy as np
import pytest
import torch

import golden_io as gio
from equidock_public_b200 import _native as nat

pytestmark = pytest.mark.gpu

# 100 pairs of 200 + 200 nodes plus the ragged pairs of test_gpu_node_stage.py (785 + 725 nodes): 649 tiles of 64 rows,
# the last one 38 rows long, on 264 resident chains (132 SMs x 2)
N_PIN = 100 * 400 + 785 + 725


def _layer(dev):
    mod = gio.build_model('dips', dev).iegmn_original.iegmn_layers[1]
    return mod, mod.packed(dev)


def _inputs(n, seed, dev):
    rng = np.random.default_rng(seed)
    f = lambda *shape: torch.from_numpy(rng.standard_normal(shape).astype(np.float32)).to(dev)
    h, aggr, mu = f(n, 64) * 0.7, f(n, 64) * 0.3, f(n, 64) * 0.5
    h0 = torch.zeros(n, 72, device=dev)
    h0[:, :69] = f(n, 69)
    return h, aggr, mu, h0


def _node_mlp_tc(lay, n, h, aggr, mu, h0):
    """eqd_node_mlp_tc over n nodes (the kernel reads only n_nodes of the graph)."""
    lib = nat.load()
    g = nat.EqdGraph()
    g.n_nodes = n
    h_out = torch.full((n, 64), float('nan'), device=h.device)
    assert lib.eqd_node_mlp_tc(C.byref(g), C.byref(lay.struct), nat.ptr(h), nat.ptr(aggr), nat.ptr(mu), nat.ptr(h0),
                               nat.ptr(h_out), None) == 0
    torch.cuda.synchronize()
    return h_out


def _node_mlp_bits(dev):
    _, lay = _layer(dev)
    return hashlib.sha256(_node_mlp_tc(lay, N_PIN, *_inputs(N_PIN, 7, dev)).cpu().numpy().tobytes()).hexdigest()


# h' of the 128-row shared-memory kernel that the chain kernel replaced (computed with both builds: equal).  Each
# element keeps its splits, products, piece-wise round-to-nearest sums and LayerNorm chain order, so a change shows here
# even where it stays inside the 1e-5 tolerance below.
NODE_MLP_SHA256 = '56ebe0cebc83f08fa40e4bbdb3697811b5e1af0c8b7417aec17de04e779e6294'


def test_node_mlp_bits_pinned(cuda_device):
    assert _node_mlp_bits(cuda_device) == NODE_MLP_SHA256


@pytest.mark.parametrize('n', [1, 63, 64, 65, 264 * 64 + 4])
def test_node_mlp_vs_fp64(n, cuda_device):
    """264 * 64 + 4 nodes: 265 tiles, so exactly one resident chain runs a second (4-row) tile."""
    dev = cuda_device
    mod, lay = _layer(dev)
    h, aggr, mu, h0 = _inputs(n, 100 + n, dev)
    out = _node_mlp_tc(lay, n, h, aggr, mu, h0)

    d = lambda t: t.detach().double()
    lin0, ln, lin4 = mod.node_mlp[0], mod.node_mlp[3], mod.node_mlp[4]
    x = torch.cat([d(h), d(aggr), d(mu), d(h0[:, :69])], 1)
    z = torch.nn.functional.leaky_relu(x @ d(lin0.weight).t() + d(lin0.bias), float(mod.leakyrelu_neg_slope))
    z = torch.nn.functional.layer_norm(z, (64,), d(ln.weight), d(ln.bias), ln.eps)
    z = z @ d(lin4.weight).t() + d(lin4.bias)
    sk = float(mod.skip_weight_h)
    ref = sk * z + (1.0 - sk) * d(h)

    assert torch.isfinite(out).all()
    err = float((out.double() - ref).abs().max()) / max(1.0, float(ref.abs().max()))
    assert err <= 1e-5
