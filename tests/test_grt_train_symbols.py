"""The entry points the 3DGRT training step adds to the C ABI are declared, exported and bound (no GPU needed)."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared(header):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", header)).read(), flags=re.S)
    return set(re.findall(r"\b((?:gutb200|grtb200)_[a-z_0-9]+)\s*\(", text))


def test_training_step_entry_points_are_exported():
    import b200_native as nat

    lib = nat.load()
    assert "grtb200_build_bvh_packed" in _declared("grt_b200.h") and "grtb200_build_bvh_packed" in nat.GRT_EXPORTS
    assert "gutb200_image_loss_rgb" in _declared("gut_b200.h") and "gutb200_image_loss_rgb" in nat.EXPORTS
    for name in ("grtb200_build_bvh_packed", "gutb200_image_loss_rgb", "grtb200_build_bvh", "gutb200_image_loss"):
        assert hasattr(lib, name), name
    assert hasattr(nat.GrtContext, "build_bvh_packed")


def test_training_step_module_imports_without_a_gpu():
    import losses
    import train_step_grt
    from threedgrt_tracer.tracer import OptixTracer

    assert set(train_step_grt.PHASES) >= {"build", "trace", "loss", "backward", "exchange", "adam"}
    assert callable(losses.image_loss_rgb) and callable(OptixTracer.build_bvh_packed)
    assert "out" in OptixTracer.trace_bwd.__code__.co_varnames
