"""The entry points the composited loss and the regularised Adam step add to the C ABI are declared, exported and bound, and the training
steps' new arguments are there (no GPU needed)."""
import inspect

from helpers import declared

NEW = ("gutb200_image_loss", "gutb200_gaussian_adam_step_reg")
REMOVED = ("gutb200_image_loss_rgb", "gutb200_image_loss_composited", "gutb200_image_loss_postprocessed")  # one loss entry takes every case


def test_loss_terms_entry_points_are_exported():
    import b200_native as nat

    lib = nat.load()
    for name in NEW:
        assert name in declared("gut_b200.h") and name in nat.EXPORTS, name
        assert hasattr(lib, name), name
    assert len(lib.gutb200_image_loss.argtypes) == 17  # layout, background, mask and post-processing included
    assert lib.gutb200_gaussian_adam_step_reg.argtypes is not None
    for name in REMOVED:
        assert name not in declared("gut_b200.h") and name not in nat.SIGNATURES and not hasattr(lib, name), name


def test_new_arguments_without_a_gpu():
    import losses
    import optimizers
    import train_step
    import train_step_grt

    for cls in (train_step.GaussianTrainStep, train_step_grt.GaussianTrainStepGRT):
        init = inspect.signature(cls.__init__).parameters
        assert init["background"].default == "black" and init["background_seed"].default == 0
        assert init["lambda_opacity"].default == 0.0 and init["lambda_scale"].default == 0.0
        assert inspect.signature(cls.step).parameters["mask"].default is None
    step = inspect.signature(optimizers.FusedGaussianAdam.step).parameters
    assert step["lambda_opacity"].default == 0.0 and step["lambda_scale"].default == 0.0
    assert inspect.signature(losses.image_loss).parameters["background"].default is None
    assert callable(losses.image_loss_rgb_alpha)
    for name in ("black", "white", (0.2, 0.5, 0.9), (0, 0, 0)):
        bg = losses.Background(name)
        assert bg.black == (name in ("black", (0, 0, 0))) and not bg.random
    for bad in ("grey", (1.0, 1.0)):
        try:
            losses.Background(bad)
        except ValueError:
            pass
        else:
            raise AssertionError(f"Background({bad!r}) was accepted")
