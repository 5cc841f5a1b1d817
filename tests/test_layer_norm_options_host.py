"""Host side of the reference's coordinate LayerNorm option (layer_norm_coors='LN', coors_mlp.3): which args values the
module accepts, its state dict and checkpoints, the ABI descriptor, the packing, the weight-gradient index maps and the
fp64 restatement the GPU tests compare against (tests/layer_norm_ref.py).  Needs neither a GPU nor, except for the
descriptor layout, the native library."""
import ctypes

import numpy as np
import pytest
import torch

import golden_io as gio
import layer_norm_ref as nr
from equidock_public_b200 import _native as nat
from equidock_public_b200 import formats
from equidock_public_b200.engine import PackedLayer
from equidock_public_b200.training import LayerLayout, LayerTrainPack, ParamLayout, layer_reductions
from test_weight_grad_maps import _check_maps

CPU = torch.device('cpu')


def _args(ds, **kw):
    a = dict(gio.load_args(ds), device='cpu')
    a.update(kw)
    return a


def test_accepted_and_refused_values():
    from equidock_public_b200.rigid_docking_model import Rigid_Body_Docking_Net
    for c in ('0', 'LN'):
        for f in ('0', 'LN'):
            Rigid_Body_Docking_Net(_args('db5', layer_norm_coors=c, final_h_layer_norm=f))
    for k, v in (('layer_norm_coors', 'BN'), ('layer_norm_coors', 'GN'), ('layer_norm_coors', 'ln'),
                 ('final_h_layer_norm', 'BN'), ('final_h_layer_norm', 'GN'), ('final_h_layer_norm', 'ln')):
        with pytest.raises(NotImplementedError):
            Rigid_Body_Docking_Net(_args('db5', **{k: v}))
    for kw in ({'layer_norm_coors': 'BN'}, {'final_h_layer_norm': 'GN'}):
        with pytest.raises(ValueError):
            PackedLayer(gio.load_checkpoint('db5'), CPU, 0.5, 0.0, 0.01, **kw)


@pytest.mark.parametrize('ds', ['db5', 'dips'])
@pytest.mark.parametrize('coors,final', [('0', '0'), ('LN', '0'), ('0', 'LN'), ('LN', 'LN')])
def test_state_dict_keys_and_checkpoint_round_trip(ds, coors, final, tmp_path):
    model = nr.build_model(ds, CPU, nr.args_with(ds, coors, final_h_layer_norm=final), seed=5)
    sd = model.state_dict()
    base = set(gio.load_checkpoint(ds))
    extra = set(sd) - base
    n = int(gio.load_args(ds)['iegmn_n_lays'])
    assert set(sd) >= base
    want = set()
    for key, on in (('coors_mlp.3', coors == 'LN'), ('final_h_layernorm_layer', final == 'LN')):
        if on:
            want |= {f'iegmn_original.iegmn_layers.{li}.{key}.{w}' for li in range(n) for w in ('weight', 'bias')}
    assert extra == want
    assert all(sd[k].shape == (64,) for k in extra)
    path = str(tmp_path / 'ck.pth')
    formats.save_checkpoint(path, model, {}, 3, nr.args_with(ds, coors, final_h_layer_norm=final))
    args, sd2, _, _ = formats.load_checkpoint(path)
    assert args['layer_norm_coors'] == coors and args['final_h_layer_norm'] == final
    from equidock_public_b200.rigid_docking_model import Rigid_Body_Docking_Net
    m2 = Rigid_Body_Docking_Net(dict(args, device='cpu', debug=False))
    m2.load_state_dict(sd2, strict=True)
    assert all(torch.equal(a, b) for a, b in zip(model.state_dict().values(), m2.state_dict().values()))


def test_descriptor_layout():
    assert ctypes.sizeof(nat.EqdLayerParams) == 184
    assert ctypes.sizeof(nat.EqdLayerNorms) == 32
    assert nat.EqdLayerNorms.coors_ln_g.offset == 0 and nat.EqdLayerNorms.coors_ln_b.offset == 8
    assert nat.EqdLayerNorms.final_ln_g.offset == 16 and nat.EqdLayerNorms.final_ln_b.offset == 24
    d = 184 + ctypes.sizeof(nat.EqdLayerConsts)
    assert nat.EqdLayer.dropout.offset == d
    assert nat.EqdLayer.norms.offset == d + ctypes.sizeof(nat.EqdDropout)
    assert ctypes.sizeof(nat.EqdLayer) == d + ctypes.sizeof(nat.EqdDropout) + 32
    assert nat.load().eqd_abi_version() == nat.ABI_VERSION == 15


def _layer_sd(model, li):
    pre = f'iegmn_original.iegmn_layers.{li}.'
    return {k[len(pre):]: v for k, v in model.state_dict().items() if k.startswith(pre)}


@pytest.mark.parametrize('li', [0, 3])
def test_packing(li):
    """Off: the packing is byte for byte the default one and the descriptor's norms are NULL.  On: the same blob plus
    gamma / beta of coors_mlp.3 as they are in the state dict, pointed to by the descriptor."""
    model = nr.build_model('dips', CPU, nr.args_with('dips', final_h_layer_norm='LN'), seed=6)
    lsd = _layer_sd(model, li)
    a = PackedLayer(lsd, CPU, 0.5, 0.1, 0.01)
    b = PackedLayer(lsd, CPU, 0.5, 0.1, 0.01, layer_norm_coors='0', final_h_layer_norm='0')
    c = PackedLayer(lsd, CPU, 0.5, 0.1, 0.01, layer_norm_coors='LN', final_h_layer_norm='LN')
    assert torch.equal(a.t['_blob'], b.t['_blob'])
    assert bytes(a.struct.consts) == bytes(b.struct.consts) and bytes(a.struct.dropout) == bytes(b.struct.dropout)
    assert not any(getattr(a.struct.norms, k) for k, _ in nat.EqdLayerNorms._fields_)
    n = a.t['_blob'].numel()
    assert torch.equal(c.t['_blob'][:n], a.t['_blob'])
    assert bytes(a.struct.consts) == bytes(c.struct.consts)
    for k, name in (('coors_ln_g', 'coors_mlp.3.weight'), ('coors_ln_b', 'coors_mlp.3.bias'),
                    ('final_ln_g', 'final_h_layernorm_layer.weight'), ('final_ln_b', 'final_h_layernorm_layer.bias')):
        t = c.t['_' + k]
        assert getattr(c.struct.norms, k) == t.data_ptr()
        assert np.array_equal(t.numpy(), lsd[name].numpy().astype(np.float32))
    assert not np.array_equal(c.t['_coors_ln_g'].numpy(), np.ones(64, np.float32))     # seeded, not the default 1


@pytest.mark.parametrize('ds', ['db5', 'dips'])
@pytest.mark.parametrize('whole_model', [True, False], ids=['ParamLayout', 'LayerLayout'])
def test_weight_grad_maps_cover_every_parameter_once(ds, whole_model):
    """With both LayerNorms on, the reductions' index maps (coors_mlp.3.* in the edge stage's per-CTA sums, 384 floats
    per CTA; final_h_layernorm_layer.* in the node stage's, 272 floats) hit every element of every parameter of every layer module exactly once."""
    model = nr.build_model(ds, CPU, nr.args_with(ds, final_h_layer_norm='LN'), seed=7)
    layers = {id(m): m for m in model.iegmn_original.iegmn_layers}.values()
    whole = ParamLayout(model)
    for lm in layers:
        layout = whole if whole_model else LayerLayout(lm)
        tp = LayerTrainPack(lm, lm.packed(CPU), layout, CPU)
        vec = [r for r in tp.reductions if r.name == 'edgevec'][0]
        assert vec.ncols == 384 and ('coors_mlp.3.weight', 256) in vec.sums and ('coors_mlp.3.bias', 320) in vec.sums
        nvec = [r for r in tp.reductions if r.name == 'nodevec'][0]
        assert nvec.ncols == 272 and ('final_h_layernorm_layer.weight', 144) in nvec.sums
        _check_maps(tp.reductions, tp.maps, list(lm.parameters()), layout)
    assert [r.ncols for r in layer_reductions(64, 64) if r.name == 'edgevec'] == [256]


def test_restatement_follows_the_module_sequentials():
    """tests/layer_norm_ref.layer_forward against the layer module's own nn.Sequential submodules in fp64 (edge_mlp,
    coors_mlp, att_mlp_*, node_mlp, final_h_layernorm_layer) on a small pair: pins the coordinate LayerNorm to coors_mlp's
    structure Linear -> Dropout -> LeakyReLU -> LayerNorm -> Linear, and the final LayerNorm to the skip combination."""
    from equidock_public_b200 import synthetic
    model = nr.build_model('dips', CPU, nr.args_with('dips', final_h_layer_norm='LN'), seed=8)
    mod = model.iegmn_original.iegmn_layers[2].double().eval()
    lig, rec = synthetic.synthetic_pair(np.random.default_rng(4), 12, 9, 4)
    rng = np.random.default_rng(1)
    sides = []
    off = 0
    for s in (lig, rec):
        n = len(s['x'])
        sides.append({'x': torch.from_numpy(s['x']).double(), 'h': torch.from_numpy(rng.normal(0, 1, (n, 64))),
                      'h0': torch.from_numpy(rng.normal(0, 1, (n, 69))), 'he': torch.from_numpy(s['he']).double(),
                      'src': torch.from_numpy(s['src']).long(), 'dst': torch.from_numpy(s['dst']).long(), 'off': off})
        off += n
    with torch.no_grad():
        outs = []
        for i, s in enumerate(sides):
            o = sides[1 - i]
            x, h, src, dst = s['x'], s['h'], s['src'], s['dst']
            x_rel = x[src] - x[dst]
            d2 = (x_rel ** 2).sum(1, keepdim=True)
            rbf = torch.cat([torch.exp(-d2 / sg) for sg in nr.dm.SIGMAS], -1)
            msg = mod.edge_mlp(torch.cat([h[src], h[dst], s['he'], rbf], -1))
            mu = torch.softmax(mod.att_mlp_Q(h) @ mod.att_mlp_K(o['h']).t(), 1) @ mod.att_mlp_V(o['h'])
            n = len(x)
            x_new = mod.x_connection_init * x + (1 - mod.x_connection_init) * x + nr.dm._segmean(x_rel * mod.coors_mlp(msg), dst, n)
            h_new = mod.node_mlp(torch.cat([h, nr.dm._segmean(msg, dst, n), mu, s['h0']], -1))
            outs.append((x_new, mod.final_h_layernorm_layer(mod.skip_weight_h * h_new + (1 - mod.skip_weight_h) * h)))
        cat = lambda k: torch.cat([sides[0][k], sides[1][k]])
        p = {k: v for k, v in mod.state_dict().items()}
        x_ref, h_ref = nr.layer_forward(p, cat('x'), cat('h'), cat('x'), cat('h0'),
                                        torch.cat([sides[0]['src'], sides[1]['src'] + 12]),
                                        torch.cat([sides[0]['dst'], sides[1]['dst'] + 12]), cat('he'), [0, 12, 21], 1,
                                        float(mod.leakyrelu_neg_slope), float(mod.skip_weight_h),
                                        float(mod.x_connection_init))
    assert torch.allclose(torch.cat([outs[0][0], outs[1][0]]), x_ref, rtol=0, atol=1e-12)
    assert torch.allclose(torch.cat([outs[0][1], outs[1][1]]), h_ref, rtol=0, atol=1e-12)
    # the coordinate LayerNorm changes phi: without it the restatement lands elsewhere
    p0 = {k: v for k, v in p.items() if not k.startswith('coors_mlp.3')}
    x0_ref, _ = nr.layer_forward(p0, cat('x'), cat('h'), cat('x'), cat('h0'),
                                 torch.cat([sides[0]['src'], sides[1]['src'] + 12]),
                                 torch.cat([sides[0]['dst'], sides[1]['dst'] + 12]), cat('he'), [0, 12, 21], 1,
                                 float(mod.leakyrelu_neg_slope), float(mod.skip_weight_h), float(mod.x_connection_init))
    assert float((x0_ref - x_ref).abs().max()) > 1e-3
