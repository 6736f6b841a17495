"""The NHT decoder's C ABI is declared, exported and bound; configurations that are not built are refused; FeatureDecoder's state dict
has the reference class's keys and shapes.  No GPU needed."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from helpers import ROOT, declared


def test_every_nhtb200_symbol_is_exported_and_bound():
    import b200_native as nat

    names = declared("nht_b200.h")
    assert names == set(nat.NHT_EXPORTS)
    lib = nat.nht_lib()
    for name in names:
        assert hasattr(lib, name) and getattr(lib, name).argtypes is not None, name


@pytest.mark.parametrize("kw", [
    dict(dir_encoding="Frequency"),
    dict(hidden_dim=64),
    dict(dir_encoding_degree=5),
    dict(dir_encoding_degree=0),
    dict(num_layers=0),
    dict(ray_feature_dim=120, dir_encoding_degree=3),
    dict(output_activation="Tanh"),
])
def test_unsupported_configurations_raise(kw):
    import feature_decoder as fd

    args = dict(ray_feature_dim=24, hidden_dim=128, num_layers=3, dir_encoding="SphericalHarmonics", dir_encoding_degree=3, sh_scale=3.0,
                output_activation="Sigmoid")
    args.update(kw)
    with pytest.raises(NotImplementedError):
        fd.FeatureDecoder(**args)


def test_state_dict_matches_the_reference_class():
    import feature_decoder as fd

    z = np.load(os.path.join(ROOT, "tests", "golden", "nht_decoder_tcnn.npz"))
    for num_layers in (3, 4):
        dec = fd.FeatureDecoder(24, 128, num_layers, "SphericalHarmonics", 3, 3.0, "Sigmoid")
        sd = dec.state_dict()
        n_params = [int(r[3]) for r in z["n_params_table"] if tuple(r[:3]) == (24, 3, num_layers)][0]
        assert list(sd) == ["network.params"]
        assert sd["network.params"].shape == (n_params,) and sd["network.params"].dtype == torch.float32
        assert [n for n, _ in dec.named_parameters()] == ["network.params"]
        # tcnn's per-matrix xavier-uniform ranges
        off = 0
        for o, i in fd.matrix_shapes(dec.config):
            blk = sd["network.params"][off:off + o * i]
            assert blk.abs().max() <= np.sqrt(6.0 / (o + i)) and blk.std() > 0.5 * np.sqrt(6.0 / (o + i)) / np.sqrt(3)
            off += o * i
    assert "ray_feature_dim=24" in dec.extra_repr()
    assert C.sizeof(fd.nat.NhtConfig) == 24
