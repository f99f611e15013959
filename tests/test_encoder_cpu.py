"""CPU: the RGCA Encoder / GeomDecoder mirrors have the reference's state-dict layout (tests/golden/encoder_ref.npz <-
tests/golden/make_encoder_golden.py), and the stride-2 Conv2dWNUB refuses what its kernels do not cover."""
import json
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "encoder_ref.npz")


def test_state_dict_layouts_match_reference():
    from goliath_b200.rgca import Encoder, GeomDecoder

    ref = json.loads(str(np.load(GOLD)["layouts"]))
    ours = {"Encoder": Encoder(256, 10), "GeomDecoder": GeomDecoder(256, torch.randn(10, 3), 1.0)}
    for name, mod in ours.items():
        got = {k: list(v.shape) for k, v in mod.state_dict().items()}
        assert got == {k: s for k, s in ref[name]}, name


def test_encoder_glorot_scales():
    """rgca.py:322-324: every layer Glorot with a LeakyReLU(0.2) gain, mean / logvar with gain 1; weight == weight_v."""
    from goliath_b200 import nn as gnn
    from goliath_b200.rgca import Encoder

    torch.manual_seed(0)
    enc = Encoder(256, 10)
    for m in enc.modules():
        if isinstance(m, (gnn.Conv2dWNUB, gnn.LinearWN)):
            assert torch.allclose(m.weight, m.weight_v, rtol=1e-5, atol=1e-7)
            assert m.bias is None or not m.bias.any()
    bound = np.sqrt(2.0 / 1.04) * np.sqrt(2.0 / ((3 + 32) * 16)) * np.sqrt(3.0)
    top = float(enc.texmod[0].weight_v.detach().abs().max())
    assert 0.9 * bound < top <= bound
    bound1 = np.sqrt(2.0 / (512 + 256)) * np.sqrt(3.0)
    top1 = float(enc.mean.weight_v.detach().abs().max())
    assert 0.9 * bound1 < top1 <= bound1


def test_stride2_layer_refusals():
    from goliath_b200 import nn as gnn

    layer = gnn.Conv2dWNUB(3, 8, 6, 10, 4, 2, 1)
    assert layer.weight_v.shape == (8, 3, 4, 4) and layer.weight_g.shape == (8, 1, 1, 1) and layer.bias.shape == (8, 6, 10)
    assert gnn.Conv2dWNUB(3, 8, 6, 10, 4, 2, 1, bias=False).bias is None
    with pytest.raises(RuntimeError, match="CUDA"):
        layer(torch.randn(1, 3, 12, 20))
    for bad in ((1, 3, 12, 21), (1, 3, 11, 20), (1, 3, 6, 10), (1, 4, 12, 20), (3, 12, 20)):
        with pytest.raises(RuntimeError):
            layer(torch.randn(*bad))
    with pytest.raises(RuntimeError):
        gnn.Conv2dWNUB(3, 8, 6, 10, 4, 2, 1, bias=False)(torch.randn(1, 3, 12, 22))
    for k, s, p in ((4, 2, 0), (3, 2, 1), (4, 1, 1), (4, 4, 1), (5, 1, 2)):
        with pytest.raises(NotImplementedError):
            gnn.Conv2dWNUB(3, 8, 6, 10, k, s, p)
    with pytest.raises(NotImplementedError):
        gnn.Conv2dWN(3, 8, 4, 2, 1)
