"""The precision switch on the host side (no GPU): the attribute, its validation, and the descriptor field it sets."""
import ctypes

import pytest

import golden_io as gio
from equidock_public_b200 import _native as nat
from equidock_public_b200.engine import PRECISIONS


def test_precision_attribute_and_validation():
    m = gio.build_model('dips', 'cpu')
    assert m.precision == 'fp32' and m.iegmn_original.precision == 'fp32'
    m.precision = 'bf16x3'
    assert m.iegmn_original.precision == 'bf16x3'
    m.iegmn_original.precision = 'fp32'
    assert m.precision == 'fp32'
    for bad in ('fp16', 'FP32', 'bf16x6', '', None, 3):
        with pytest.raises(ValueError):
            m.precision = bad
        with pytest.raises(ValueError):
            m.iegmn_original.precision = bad
    assert m.precision == 'fp32'
    assert PRECISIONS == {'fp32': 0, 'bf16x3': 3}


def test_mma_products_fills_the_tail_padding():
    """eqd_layer_params.mma_products sits right after leaky_slope, in what was the struct's tail padding."""
    P = nat.EqdLayerParams
    assert P.mma_products.offset == P.leaky_slope.offset + 4
    assert ctypes.sizeof(P) == P.mma_products.offset + 4 == 184
    assert nat.EqdLayer().dev.mma_products == 0
