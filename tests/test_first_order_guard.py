"""CPU: the guard that the engine's autograd Functions put on their kernel gradients (engine.first_order_only), on a plain
torch stand-in for a kernel backward: a Function whose backward computes its gradient outside autograd, as the ctypes
launches do.  Without the guard torch treats that gradient as a constant: a Hessian comes back all zero and a gradient
penalty loses its term.  With it both raise, and first-order gradients, with or without create_graph, are unchanged."""
import pytest
import torch

from differentiable_robot_model_b200 import engine


class _SinKernel(torch.autograd.Function):
    """y = sin(x) * w, with a backward that builds its gradients from detached values."""
    guarded = False

    @staticmethod
    def forward(ctx, x, w):
        ctx.primals = (x, w)
        ctx.save_for_backward(x, w)
        return x.detach().sin() * w.detach()

    @staticmethod
    def backward(ctx, g):
        x, w = (t.detach() for t in ctx.saved_tensors)
        gx = g.detach() * x.cos() * w if ctx.needs_input_grad[0] else None
        gw = (g.detach() * x.sin()).sum(0) if ctx.needs_input_grad[1] else None
        if _SinKernel.guarded:
            return engine.first_order_only((gx, gw), ctx.primals + (g,))
        return gx, gw


@pytest.fixture(params=[False, True], ids=["unguarded", "guarded"])
def guarded(request):
    _SinKernel.guarded = request.param
    yield request.param
    _SinKernel.guarded = False


def _inputs():
    x = torch.tensor([[0.3, 1.1], [-0.7, 2.0]], dtype=torch.float64, requires_grad=True)
    w = torch.tensor([1.5, -0.5], dtype=torch.float64, requires_grad=True)
    return x, w


def test_hessian_raises_instead_of_returning_zeros(guarded):
    x, w = _inputs()
    fn = lambda xx: _SinKernel.apply(xx, w).sum()
    if not guarded:     # what torch does with an unguarded kernel backward: a silent all-zero Hessian
        assert torch.count_nonzero(torch.autograd.functional.hessian(fn, x)) == 0
        return
    with pytest.raises(RuntimeError, match="second-order derivatives"):
        torch.autograd.functional.hessian(fn, x)


def test_gradient_penalty_raises_instead_of_dropping_its_term(guarded):
    x, w = _inputs()
    y = _SinKernel.apply(x, w)
    (g,) = torch.autograd.grad(y.square().sum(), x, create_graph=True)
    loss = y.sum() + g.square().sum()
    if not guarded:
        loss.backward()
        assert torch.allclose(x.grad, (w * x.cos()).detach())     # d(y.sum())/dx only: the penalty's term is gone
        return
    with pytest.raises(RuntimeError, match="compute_inverse_dynamics_derivatives"):
        loss.backward()


def test_inner_step_on_parameters_raises(guarded):
    """MAML-style: the outer loss depends on w - lr * dL/dw, so its gradient needs d(dL/dw)/dw."""
    x, w = _inputs()
    (gw,) = torch.autograd.grad(_SinKernel.apply(x, w).square().sum(), w, create_graph=True)
    outer = _SinKernel.apply(x.detach(), w - 0.1 * gw).sum()
    if guarded:
        with pytest.raises(RuntimeError, match="second-order"):
            outer.backward()
    else:
        outer.backward()


@pytest.mark.filterwarnings("ignore:Using backward\\(\\) with create_graph=True")
def test_first_order_gradients_are_unchanged(guarded):
    x, w = _inputs()
    G = torch.tensor([[0.2, -1.0], [3.0, 0.5]], dtype=torch.float64)
    plain = torch.autograd.grad((G * _SinKernel.apply(x, w)).sum(), (x, w))
    graphed = torch.autograd.grad((G * _SinKernel.apply(x, w)).sum(), (x, w), create_graph=True)
    for a, b in zip(plain, graphed):
        assert torch.equal(a, b)
        assert not a.requires_grad
        assert b.requires_grad == guarded
    assert torch.equal(plain[0], (G * x.cos() * w).detach())
    assert torch.equal(plain[1], (G * x.sin()).sum(0).detach())
    # two create_graph backwards accumulate into .grad; an optimiser step then reads it
    for _ in range(2):
        (G * _SinKernel.apply(x, w)).sum().backward(create_graph=True)
    assert torch.equal(x.grad.detach(), 2 * plain[0])
    opt = torch.optim.SGD([x, w], lr=0.1, momentum=0.9)
    opt.step()
    assert torch.isfinite(x).all()


def test_no_wrapping_when_nothing_requires_grad():
    g = torch.ones(3)
    with torch.enable_grad():
        out = engine.first_order_only((g, None), (torch.zeros(3), None))
    assert out[0] is g and out[1] is None
    x = torch.zeros(3, requires_grad=True)
    with torch.no_grad():
        assert engine.first_order_only((g,), (x,))[0] is g
    with torch.enable_grad():
        wrapped = engine.first_order_only((g, None), (x,))
    assert wrapped[1] is None and wrapped[0].requires_grad and torch.equal(wrapped[0], g)
