"""The loss dispatch of TrainStep._step on the CPU: a renderer stand-in on the TrainStep hooks and the three losses.image_loss* entries
recorded instead of launched.  For the rgba layout (3DGUT), the split rgb + alpha layout (3DGRT, NHT) and the split layout with a strided
alpha (the hybrid's primary alpha), every background, mask, SSIM and post-processing case picks the entry the GPU steps call, hands it the
step's tensors, and what it returns reaches `_backward`; the L1 shortcut's loss and gradient are the formula."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

H, W = 5, 7
SH = {"positions": 3, "density": 1, "rotation": 4, "scale": 3, "features_albedo": 3, "features_specular": 45}
CASES = {  # name -> TrainStep options; "mask" also passes a mask to step
    "l1": {},
    "ssim": {"lambda_ssim": 0.2},
    "colour": {"background": (0.2, 0.4, 0.6)},
    "random": {"background": "random"},
    "mask": {},
    "srgb": {"post_processing": "linear-to-srgb"},
}
LAYOUTS = ("rgba", "split", "hybrid")


class _Optimizer:
    selective = False

    def __init__(self, lrs):
        self.lrs = dict(lrs)
        self.steps = 0

    def step(self, *args, **kw):
        self.steps += 1


def _step_class():
    import train_step
    import view_parallel

    class FakeRenderer(train_step.TrainStep):
        """view = (rays_o [1,H,W,3], the Frame to hand back)."""

        def _init_renderer(self, conf):
            self.backward_calls = []

        def _new_exchange(self):
            return view_parallel.FlatGradientExchange(self.n, self.device, group=self.group)

        def _new_optimizer(self, lrs, eps, selective):
            return _Optimizer(lrs)

        def _forward(self, view, particles, features, train):
            assert train and particles.shape == (self.n, 12) and features.shape == (self.n, 48)
            return view[1]

        def _backward(self, frame, d_pred, d_alpha):
            self.backward_calls.append((frame, d_pred, d_alpha))
            return ()

        def _sensor_position(self, frame):
            return np.zeros(3, np.float32)

    return FakeRenderer


def _frame(layout, g):
    import train_step

    rgba = torch.rand((H, W, 4), generator=g)
    hits, vis = torch.ones((H, W, 1)), torch.ones((10, 1))
    if layout == "rgba":
        return train_step.Frame(rgba, 4, rgba[..., :3], None, hits, vis, ())
    rgb = torch.rand((H, W, 3), generator=g)
    alpha = rgba[..., 3:] if layout == "hybrid" else rgba[..., 3:].contiguous()  # the hybrid's is a strided view of the primary rgba
    return train_step.Frame(rgb, 3, rgb, alpha, hits, vis, ())


@pytest.fixture
def recorded(monkeypatch):
    """The image_loss* calls as (name, args, kwargs, returned gradients)."""
    import losses

    calls = []

    def entry(name, n_grads):
        def fake(*args, **kw):
            grads = tuple(torch.full((H, W, 1), float(i + 1)) for i in range(n_grads))
            calls.append((name, args, kw, grads))
            return (torch.tensor(0.5), torch.tensor(0.25), torch.tensor(0.75), *grads)
        return fake

    monkeypatch.setattr(losses, "image_loss", entry("image_loss", 1))
    monkeypatch.setattr(losses, "image_loss_rgb", entry("image_loss_rgb", 1))
    monkeypatch.setattr(losses, "image_loss_rgb_alpha", entry("image_loss_rgb_alpha", 2))
    monkeypatch.setattr(losses, "mask_hw", lambda m, h, w: m.reshape(h, w).to(torch.float32).contiguous())  # the CUDA check aside
    return calls


def _run(layout, case):
    g = torch.Generator().manual_seed(3)
    params = {k: torch.randn(10, w, generator=g) for k, w in SH.items()}
    step = _step_class()(params, {k: 1e-3 for k in SH}, lambda_l1=0.8, **CASES[case])
    frame, target = _frame(layout, g), torch.rand((H, W, 3), generator=g)
    mask = (torch.rand((1, H, W, 1), generator=g) > 0.5).float() if case == "mask" else None
    loss = step._step((torch.zeros((1, H, W, 3)), frame), target, None, mask)
    (seen, d_pred, d_alpha), = step.backward_calls
    assert seen is frame
    return step, frame, target, mask, loss, d_pred, d_alpha


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("layout", LAYOUTS)
def test_the_loss_entry_its_tensors_and_what_reaches_the_backward(layout, case, recorded):
    step, frame, target, mask, loss, d_pred, d_alpha = _run(layout, case)
    if case == "l1":  # black, unmasked, no SSIM, no post-processing: the torch shortcut, no entry
        assert recorded == []
        diff = frame.rgb - target
        assert torch.equal(loss, 0.8 * diff.abs().mean())
        d_rgb = 0.8 * torch.sign(diff) / diff.numel()
        if layout == "rgba":
            assert d_pred.shape == (H, W, 4) and torch.equal(d_pred[..., :3], d_rgb) and not d_pred[..., 3].any()
        else:
            assert torch.equal(d_pred, d_rgb)
        assert d_alpha is None
        return
    (name, args, kw, grads), = recorded
    background = {"colour": step.background.color, "random": step.background.image}.get(case)  # as Background.draw hands them out
    post = "linear-to-srgb" if case == "srgb" else None
    lambdas = (0.8, 0.2 if case == "ssim" else 0.0)
    assert torch.equal(args[1 if layout == "rgba" or case == "ssim" else 2], target)
    if case == "random":
        assert background.shape == (H, W, 3)
    if case == "colour":
        assert background == (0.2, 0.4, 0.6)
    if layout == "rgba":
        assert name == "image_loss" and args[0] is frame.pred and args[2:] == lambdas
        assert kw["background"] is background and kw["post_processing"] == post
        assert (kw["mask"] is None) == (mask is None) and (mask is None or torch.equal(kw["mask"], mask.reshape(H, W)))
        assert d_pred is grads[0] and d_alpha is None  # the alpha gradient is d_rgba's channel 3
    elif case == "ssim":  # black and unmasked: the rgb loss, no alpha gradient
        assert name == "image_loss_rgb" and args[0] is frame.pred and args[2:] == lambdas and kw == {}
        assert d_pred is grads[0] and d_alpha is None
    else:  # composited, masked or post-processed: rgb and the (primary) alpha, contiguous
        assert name == "image_loss_rgb_alpha" and args[0] is frame.pred and args[3:] == lambdas
        assert args[1].is_contiguous() and torch.equal(args[1], frame.alpha)
        if layout == "split":
            assert args[1] is frame.alpha  # already contiguous: not copied
        assert kw["background"] is background and kw["post_processing"] == post
        assert (kw["mask"] is None) == (mask is None) and (mask is None or torch.equal(kw["mask"], mask.reshape(H, W)))
        assert d_pred is grads[0] and d_alpha is grads[1]
    assert torch.equal(loss, torch.tensor(0.5))  # world 1: the entry's loss, no regularisers


def test_metrics_inputs_reads_the_frame(recorded):
    for layout in LAYOUTS:
        g = torch.Generator().manual_seed(1)
        step = _step_class()({k: torch.randn(10, w, generator=g) for k, w in SH.items()}, {k: 1e-3 for k in SH})
        frame = _frame(layout, g)
        step._forward = lambda view, particles, features, train, frame=frame: frame if not train else None
        got = step.metrics_inputs(torch.zeros((1, H, W, 3)))
        assert got["pred"] is frame.pred and got["hits"] is frame.hits
        if layout == "rgba":
            assert got["alpha"] is None
        else:
            assert got["alpha"].is_contiguous() and torch.equal(got["alpha"], frame.alpha)
