"""Host side of the keypoint count num_att_heads = K (1..64): which values the module accepts, its state dict and
checkpoints, the eqd_head_params layout, the K-sized workspace entry points and the weight-gradient index maps.  Needs no
GPU; the layout and sizing tests load the native library."""
import ctypes

import numpy as np
import pytest
import torch

import golden_io as gio
import heads_ref as hr
from equidock_public_b200 import _native as nat
from equidock_public_b200 import formats
from equidock_public_b200.training import HEAD_REDUCTION, ParamLayout, reduction_maps
from test_weight_grad_maps import _check_maps

CPU = torch.device('cpu')


def _net(K, ds='db5'):
    from equidock_public_b200.rigid_docking_model import Rigid_Body_Docking_Net
    return Rigid_Body_Docking_Net(dict(hr.args_with(ds, K), device='cpu'))


@pytest.mark.parametrize('K', [1, 4, 25, 50, 64, np.int64(33)])
def test_accepted_keypoint_counts(K):
    net = _net(K).iegmn_original
    assert net.num_att_heads == int(K)
    assert net.att_mlp_key_ROT[0].weight.shape == net.att_mlp_query_ROT[0].weight.shape == (64 * int(K), 64)


@pytest.mark.parametrize('K', [0, 65, 100, -1, 50.0, True, '50', None])
def test_refused_keypoint_counts(K):
    with pytest.raises(NotImplementedError, match='1 to 64'):
        _net(K)


@pytest.mark.parametrize('ds', ['db5', 'dips'])
@pytest.mark.parametrize('K', [1, 4, 25, 64])
def test_state_dict_and_checkpoint_round_trip(ds, K, tmp_path):
    model = hr.build_model(ds, CPU, K, seed=K)
    sd = model.state_dict()
    assert set(sd) == set(gio.load_checkpoint(ds))                       # the reference's keys
    for key in ('att_mlp_key_ROT.0.weight', 'att_mlp_query_ROT.0.weight'):
        assert sd['iegmn_original.' + key].shape == (64 * K, 64)
    path = str(tmp_path / 'ck.pth')
    formats.save_checkpoint(path, model, {}, 2, hr.args_with(ds, K))
    args, sd2, _, _ = formats.load_checkpoint(path)
    assert args['num_att_heads'] == K
    from equidock_public_b200.rigid_docking_model import Rigid_Body_Docking_Net
    m2 = Rigid_Body_Docking_Net(dict(args, device='cpu', debug=False))
    m2.load_state_dict(sd2, strict=True)
    assert all(torch.equal(a, b) for a, b in zip(model.state_dict().values(), m2.state_dict().values()))
    with pytest.raises(RuntimeError):                                     # a K-head checkpoint does not fit another K
        _net(K + 1 if K < 64 else 63, ds).load_state_dict(sd2, strict=True)


def test_head_params_layout():
    assert ctypes.sizeof(nat.EqdHeadParams) == 48
    assert nat.EqdHeadParams.leaky_slope.offset == 40 and nat.EqdHeadParams.n_heads.offset == 44
    assert nat.MAX_HEADS == 64 and nat.HEADS == 50


def test_sizing_entry_points():
    lib = nat.load()
    g = nat.EqdGraph()
    for n_nodes, tiles, B, n_rec, n_pocket in ((1, 1, 1, 1, 1), (2601, 24, 3, 1300, 300), (132000, 1100, 330, 66000, 9000)):
        g.n_nodes, g.n_pairs, g.n_node_tiles, g.n_lig_nodes = n_nodes, B, tiles, n_nodes - n_rec
        # K = 50 (and the 0 = 50 of eqd_head_params) are the sizes of the entry points without K
        assert lib.eqd_workspace_bytes_k(n_nodes, tiles, B, 50) == lib.eqd_workspace_bytes(n_nodes, tiles, B)
        assert lib.eqd_bwd_head_workspace_bytes_k(n_nodes, tiles, B, 50) == lib.eqd_bwd_head_workspace_bytes(n_nodes, tiles, B)
        assert lib.eqd_forward_workspace_bytes_k(ctypes.byref(g), 50) == lib.eqd_forward_workspace_bytes(ctypes.byref(g))
        assert lib.eqd_losses_workspace_bytes_k(n_rec, n_pocket, 50) == lib.eqd_losses_workspace_bytes(n_rec, n_pocket)
        for K in (0, 65, -3):
            assert lib.eqd_workspace_bytes_k(n_nodes, tiles, B, K) == 0
            assert lib.eqd_bwd_head_workspace_bytes_k(n_nodes, tiles, B, K) == 0
            assert lib.eqd_forward_workspace_bytes_k(ctypes.byref(g), K) == 0
            assert lib.eqd_losses_workspace_bytes_k(n_rec, n_pocket, K) == 0
        a256 = lambda v: (v + 255) // 256 * 256
        prev = None
        for K in (1, 4, 25, 33, 64):
            w = lib.eqd_workspace_bytes_k(n_nodes, tiles, B, K)
            # u [2B][K][64] fp64 is the only K-sized array of the head workspace (eqd_iegmn.h)
            assert w - lib.eqd_workspace_bytes_k(n_nodes, tiles, B, 1) == a256(2 * B * K * 512) - a256(2 * B * 512)
            sizes = (w, lib.eqd_bwd_head_workspace_bytes_k(n_nodes, tiles, B, K),
                     lib.eqd_forward_workspace_bytes_k(ctypes.byref(g), K), lib.eqd_losses_workspace_bytes_k(n_rec, n_pocket, K))
            assert prev is None or all(a >= b for a, b in zip(sizes, prev))
            prev = sizes


@pytest.mark.parametrize('ds', ['db5', 'dips'])
@pytest.mark.parametrize('K', [1, 25, 64])
def test_head_gradient_layout_covers_every_head_parameter_once(ds, K):
    """The head's reduction maps cover mlp_h_mean_ROT.0 once; the key / query gradients, which eqd_bwd_head writes in
    their state-dict layout straight into the flat buffer, own disjoint 64K x 64 slices of it."""
    model = hr.build_model(ds, CPU, K)
    layout = ParamLayout(model)
    maps = reduction_maps((HEAD_REDUCTION,), layout.entries, layout, CPU)
    net = model.iegmn_original
    _check_maps((HEAD_REDUCTION,), maps, list(net.mlp_h_mean_ROT[0].parameters()), layout)
    spans = sorted((layout.offset[id(p)], layout.offset[id(p)] + p.numel()) for p in layout.params)
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))
    for mod in (net.att_mlp_key_ROT, net.att_mlp_query_ROT):
        p = mod[0].weight
        assert p.numel() == 64 * K * 64 and layout.offset[id(p)] % 64 == 0
    assert sum(p.numel() for p in layout.params) == sum(p.numel() for p in {id(q): q for q in model.parameters()}.values())
