"""Round-2 layer kernels (sigmoid / tanh / absval / bnll / power / threshold, eltwise, channel softmax, MVN, within-channel
LRN, stochastic pooling) against the fp32 oracle in ops/reference.py — forward and backward, on an H100."""
import pytest
import torch

from poseidon_b200.ops import reference as R

pytestmark = pytest.mark.gpu
CL = torch.channels_last


def _x(shape, seed=0, scale=1.0, positive=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.randn(shape, generator=g, device="cuda") * scale
    if positive:
        t = t.abs() + 0.05
    t = t.to(torch.bfloat16)
    return t.contiguous(memory_format=CL) if t.dim() == 4 else t


def _close(got, ref, rel=2e-2, what=""):
    err = (got.float() - ref.float()).abs().max().item()
    mag = ref.float().abs().max().item() + 1e-6
    assert err <= rel * mag, f"{what}: max err {err} vs magnitude {mag}"


def _check(fn_sm, fn_ref, xs, rel=2e-2, grad=True):
    """Run the engine function on bf16 inputs and the oracle on their fp32 copies; compare outputs and input gradients."""
    a = [x.clone().requires_grad_(grad) for x in xs]
    b = [x.float().requires_grad_(grad) for x in xs]
    y, yr = fn_sm(*a), fn_ref(*b)
    assert y.dtype == torch.bfloat16 and tuple(y.shape) == tuple(yr.shape)
    _close(y, yr, rel, "forward")
    if grad:
        dy = _x(tuple(yr.shape), 99)
        if dy.dim() == 4 and y.dim() == 4:
            dy = dy.contiguous(memory_format=CL)
        y.backward(dy)
        yr.backward(dy.float())
        for i, (p, q) in enumerate(zip(a, b)):
            _close(p.grad, q.grad, rel * 1.5, f"grad of input {i}")


@pytest.mark.parametrize("shape", [(4, 64, 9, 7), (32, 1000), (3, 24, 5, 5)])
@pytest.mark.parametrize("op", ["sigmoid", "tanh", "absval", "bnll", "power2", "power_half", "power1"])
def test_unary_neurons(ext, op, shape):
    from poseidon_b200.ops import sm100
    sm = {"sigmoid": sm100.sigmoid, "tanh": sm100.tanh, "absval": sm100.absval, "bnll": sm100.bnll,
          "power2": lambda t: sm100.power(t, 2.0, 0.5, 1.0), "power1": lambda t: sm100.power(t, 1.0, -2.0, 0.25),
          "power_half": lambda t: sm100.power(t, 0.5, 1.0, 0.1)}[op]
    ref = {"sigmoid": torch.sigmoid, "tanh": torch.tanh, "absval": torch.abs, "bnll": R.bnll,
           "power2": lambda t: R.power(t, 2.0, 0.5, 1.0), "power1": lambda t: R.power(t, 1.0, -2.0, 0.25),
           "power_half": lambda t: R.power(t, 0.5, 1.0, 0.1)}[op]
    x = _x(shape, 1, 2.0, positive=(op == "power_half"))
    _check(sm, ref, [x])


def test_threshold(ext):
    from poseidon_b200.ops import sm100
    x = _x((4, 32, 6, 6), 2)
    y = sm100.threshold(x, 0.25)
    assert torch.equal(y.float(), (x.float() > 0.25).float())


@pytest.mark.parametrize("op,coeffs", [("PROD", None), ("SUM", None), ("SUM", [0.5, -2.0, 1.5]), ("MAX", None)])
@pytest.mark.parametrize("shape", [(4, 64, 9, 7), (16, 256)])
def test_eltwise(ext, op, coeffs, shape):
    from poseidon_b200.ops import sm100
    xs = [_x(shape, 10 + i) for i in range(3)]

    def ref(*t):
        if op != "MAX":
            return R.eltwise(t, op, coeffs)
        # the reference routes the gradient of a tie to the EARLIER bottom (eltwise_layer.cu:11-34: strict '>' against the
        # running maximum); torch.maximum would split it, and bf16 inputs do tie
        st = torch.stack(t)
        arg = st.argmax(0)              # first maximal index
        return st.gather(0, arg.unsqueeze(0)).squeeze(0)
    _check(lambda *t: sm100.eltwise(t, op, coeffs), ref, xs)


@pytest.mark.parametrize("shape", [(64, 1000), (4, 21, 13, 11), (2, 1000, 1, 1), (8, 2048)])
def test_softmax(ext, shape):
    from poseidon_b200.ops import sm100
    x = _x(shape, 3, 3.0)
    _check(sm100.softmax, lambda t: torch.softmax(t, 1), [x])


@pytest.mark.parametrize("nv,ac", [(True, False), (True, True), (False, False), (False, True)])
def test_mvn(ext, nv, ac):
    from poseidon_b200.ops import sm100
    x = _x((3, 72, 9, 11), 4, 2.0) + 0.5
    _check(lambda t: sm100.mvn(t, nv, ac), lambda t: R.mvn(t, nv, ac), [x], rel=3e-2)


@pytest.mark.parametrize("size", [3, 5])
def test_lrn_within_channel(ext, size):
    from poseidon_b200.ops import sm100
    x = _x((2, 32, 12, 10), 5, 2.0)
    # the oracle runs on the CPU: torch's CUDA avg_pool2d backward (ceil_mode + padding, channels-last) disagrees with its
    # own CPU implementation and with the closed form (scripts/debug/lrn_within_dbg.py) — the kernel matches the latter
    a = x.clone().requires_grad_(True)
    b = x.float().cpu().contiguous().requires_grad_(True)
    y, yr = sm100.lrn_within(a, size, 0.5, 0.75), R.lrn_within(b, size, 0.5, 0.75)
    _close(y.cpu(), yr, 3e-2, "forward")
    dy = _x(tuple(yr.shape), 99)
    y.backward(dy)
    yr.backward(dy.float().cpu())
    _close(a.grad.cpu(), b.grad, 4.5e-2, "grad")


def test_stochastic_pool_test_phase_and_train_statistics(ext):
    from poseidon_b200.ops import sm100
    x = _x((2, 16, 12, 12), 6, 1.0, positive=True)
    y = sm100.stochastic_pool(x, (3, 3), (2, 2), False)
    _close(y, R.stochastic_pool(x.float(), (3, 3), (2, 2), False), 2e-2, "test phase")
    # training: every output is one of its window's elements, the gradient lands on exactly that element, and over many
    # draws the pick frequency follows the activations
    xs = x.clone().requires_grad_(True)
    yt = sm100.stochastic_pool(xs, (3, 3), (2, 2), True)
    cols, oh, ow = R._pool_windows(x.float(), (3, 3), (2, 2))
    assert ((cols - yt.detach().float().unsqueeze(-1)).abs().min(-1).values < 1e-6).all()
    yt.backward(torch.ones_like(yt))
    assert abs(xs.grad.float().sum().item() - yt.numel()) < 1e-3          # each output routes its gradient to one input
    base = torch.zeros(4096, 16, 2, 2, device="cuda")
    base[:, :, 0, 0], base[:, :, 1, 1] = 1.0, 3.0                             # windows hold (1, 0, 0, 3)
    picked = sm100.stochastic_pool(base.to(torch.bfloat16).contiguous(memory_format=CL), (2, 2), (2, 2), True)
    frac3 = (picked.float() == 3).float().mean().item()
    assert 0.70 < frac3 < 0.80, frac3                                          # P(pick 3) = 3 / 4
