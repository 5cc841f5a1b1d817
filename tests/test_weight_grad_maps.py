"""Index maps of the backward's weight-gradient reductions (training.layer_reductions and HEAD_REDUCTION), for both
shipped checkpoints and both flat gradient layouts: every parameter element receives exactly one gradient entry, and
every source index lies inside the buffer its reduction reads.  Host only: needs neither a GPU nor the native
library."""
import numpy as np
import pytest
import torch

import golden_io as gio
from equidock_public_b200.training import HEAD_REDUCTION, LayerLayout, LayerTrainPack, ParamLayout, reduction_maps

CPU = torch.device('cpu')


def _check_maps(table, maps, params, layout):
    """The destination indices of ``maps`` hit every element of ``params`` in ``layout`` once and nothing else; the
    source indices of each map are distinct and lie inside the partial [K][ncols] of its reduction, or inside one row of
    the colsum / per-CTA vec sums (``ncols`` floats)."""
    dst = []
    for r in table:
        blocks, sums = maps[r.name]
        assert (blocks is not None) == bool(r.blocks) and (sums is not None) == bool(r.sums), r.name
        for mp, extent in ((blocks, r.K * r.ncols), (sums, r.ncols)):
            if mp is None:
                continue
            src = mp[0].numpy()
            assert len(src) == len(mp[1]), r.name
            assert 0 <= src.min() and src.max() < extent, (r.name, src.min(), src.max(), extent)
            assert len(np.unique(src)) == len(src), r.name
            dst.append(mp[1].numpy())
    want = np.concatenate([layout.offset[id(p)] + np.arange(p.numel()) for p in params])
    assert np.array_equal(np.sort(np.concatenate(dst)), np.sort(want))


@pytest.mark.parametrize('ds', ['db5', 'dips'])
@pytest.mark.parametrize('whole_model', [True, False], ids=['ParamLayout', 'LayerLayout'])
def test_layer_maps_cover_every_parameter_once(ds, whole_model):
    model = gio.build_model(ds, CPU)
    layers = {id(m): m for m in model.iegmn_original.iegmn_layers}.values()    # a shared layer module once
    whole = ParamLayout(model)
    for lm in layers:
        layout = whole if whole_model else LayerLayout(lm)
        tp = LayerTrainPack(lm, lm.packed(CPU), layout, CPU)
        _check_maps(tp.reductions, tp.maps, list(lm.parameters()), layout)
    assert {lm.packed(CPU).dh for lm in layers} == {64, 69}      # both layer widths are covered


@pytest.mark.parametrize('ds', ['db5', 'dips'])
def test_head_map_covers_mlp_h_mean_once(ds):
    model = gio.build_model(ds, CPU)
    layout = ParamLayout(model)
    maps = reduction_maps((HEAD_REDUCTION,), layout.entries, layout, CPU)
    _check_maps((HEAD_REDUCTION,), maps, list(model.iegmn_original.mlp_h_mean_ROT[0].parameters()), layout)
