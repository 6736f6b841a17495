"""The C-ABI library loads without a GPU and exports every symbol include/gut_b200.h declares; the product
path fails loudly (no CPU fallback) when no CUDA device is present."""
import ctypes
import os

import pytest

from helpers import ROOT, declared


def test_library_exports_every_declared_symbol():
    import b200_native as nat

    lib = nat.load()
    names = declared("gut_b200.h")
    assert len(names) >= 14
    for name in names:
        assert hasattr(lib, name), f"{name} declared in include/gut_b200.h but not exported"
    assert set(nat.EXPORTS) == set(names)
    assert b"sm_90a" in lib.gutb200_version()
    grt = declared("grt_b200.h")
    assert len(grt) >= 9 and set(nat.GRT_EXPORTS) == set(grt)
    for name in grt:
        assert hasattr(lib, name), f"{name} declared in include/grt_b200.h but not exported"


def test_struct_layouts_match_header():
    import b200_native as nat

    assert ctypes.sizeof(nat.Camera) == 4 * (2 + 2 + 2 + 6 + 2 + 4 + 7 + 7 + 2 + 1 + 6 + 6 + 3 + 1)
    assert ctypes.sizeof(nat.Config) == 4 * 18
    cfg = nat.default_config()
    assert cfg.kernel_degree == 2 and abs(cfg.min_alpha - 1 / 255) < 1e-9 and abs(cfg.ut_delta - 3 ** 0.5) < 1e-6
    assert abs(cfg.min_transmittance - 1e-4) < 1e-10 and cfg.tile_culling == 1 and cfg.global_z_order == 1


def test_no_cpu_fallback_without_gpu():
    torch = pytest.importorskip("torch")
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import b200_native as nat
    import threedgut_tracer

    import threedgrt_tracer

    with pytest.raises(RuntimeError):
        nat.Context(nat.default_config(), 0)
    with pytest.raises(RuntimeError):
        nat.GrtContext(nat.grt_default_config(), 0)
    with pytest.raises(Exception):
        threedgut_tracer.Tracer({})
    with pytest.raises(Exception):
        threedgrt_tracer.Tracer({})


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "3dgrut_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                src = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "oracle" not in src.replace("# oracle", ""), f"{f} references the oracle"
