"""base_model.FusedStep, the autograd bridge of the NICE-SLAM, Vox-Fusion and Point-SLAM fused
steps, driven by a fake launch that returns known gradients: input-order routing, total-loss
scaling, the NaN on unequal per-term scales, ``n_live`` and the forward-only error."""
import pytest
import torch

from xrdslam_b200.base_model import FusedStep


def _inputs(pattern):
    """One input per flag, each of its own length, requires_grad as the flag says."""
    return [torch.zeros(k + 2, requires_grad=r) for k, r in enumerate(pattern)]


def _fake(inputs, missing=(), forward_only=False):
    """A launch that records the flags it gets and returns gradient k + 1 for input k where it
    is needed, None for the inputs in ``missing``; (losses[2], (rgb, mask), grads)."""
    seen = []

    def launch(needs):
        seen.append(tuple(needs))
        grads = None if forward_only else [
            torch.full_like(t, k + 1.) if need and k not in missing else None
            for k, (t, need) in enumerate(zip(inputs, needs))]
        return torch.ones(2), (torch.ones(4, 3), torch.ones(4, dtype=torch.bool)), grads
    return launch, seen


def _expected(inputs, k, scale=1.):
    return torch.full_like(inputs[k], (k + 1.) * scale)


@pytest.mark.parametrize('pattern', [(True, False, True), (False, True, False, False),
                                     (True, True), (False, False, True)])
def test_launch_gets_the_requires_grad_pattern(pattern):
    inputs = _inputs(pattern)
    launch, seen = _fake(inputs)
    FusedStep.apply(launch, None, *inputs)
    assert seen == [pattern]


def test_each_gradient_reaches_its_own_input():
    inputs = _inputs((True, False, True, True, True))
    launch, _ = _fake(inputs, missing={3})
    losses, rgb, mask = FusedStep.apply(launch, None, *inputs)
    assert not rgb.requires_grad and not mask.requires_grad
    (losses[0] + losses[1]).backward()
    for k in (0, 2, 4):
        assert torch.equal(inputs[k].grad, _expected(inputs, k))
    assert inputs[1].grad is None  # does not require grad
    assert inputs[3].grad is None  # requires grad, but the launch has no gradient for it


@pytest.mark.parametrize('c', [1., 0.25, -3.])
def test_total_loss_scale_scales_every_gradient(c):
    inputs = _inputs((True, True, False, True))
    launch, _ = _fake(inputs)
    losses, _, _ = FusedStep.apply(launch, 2, *inputs)
    (c * (losses[0] + losses[1])).backward()
    for k in (0, 1, 3):
        assert torch.equal(inputs[k].grad, _expected(inputs, k, c))


@pytest.mark.parametrize('n_live,nan', [(None, True), (2, True), (1, False)])
def test_unequal_term_scales_give_nan_unless_the_term_is_dead(n_live, nan):
    """Only losses[0] enters the loss, so the terms' upstream gradients are (1, 0)."""
    inputs = _inputs((True, True))
    launch, _ = _fake(inputs)
    losses, _, _ = FusedStep.apply(launch, n_live, *inputs)
    losses[0].backward()
    for k, t in enumerate(inputs):
        if nan:
            assert torch.isnan(t.grad).all()
        else:
            assert torch.equal(t.grad, _expected(inputs, k))


def test_forward_only_launch_refuses_backward():
    inputs = _inputs((True, False))
    launch, _ = _fake(inputs, forward_only=True)
    losses, rgb, mask = FusedStep.apply(launch, None, *inputs)
    assert losses.requires_grad
    for out in (rgb, mask):
        assert not out.requires_grad and out.grad_fn is None
    with pytest.raises(RuntimeError, match='forward-only'):
        losses.sum().backward()
