"""Nets whose channel counts are not multiples of 8 (LeNet: 1 -> 20 -> 50, inner-product K = 500) on the sm100 engine.

The engine zero-pads such layers to multiples of 8 around the kernels (ops/sm100.py: ConvState.Coutp / Cp, IPState.Kp);
the Python side of that is covered on the CPU by tests/test_sm100_emulated.py.  These are the same comparisons against the
fp32 engine on the real kernels.  (File name: collected last, after the other GPU suites.)"""
import numpy as np
import pytest
import torch

from smallnet import feed, make_data, small_solver_param
from test_sm100_emulated import _odd_channel_net

pytestmark = [pytest.mark.gpu]


def _run(engine, net_fn, steps, batch, hw, classes):
    from poseidon_b200 import get_solver
    sp = small_solver_param(net_fn(), max_iter=steps)
    s = get_solver(sp, engine=engine, dtype=torch.float32 if engine == "torch" else None)
    x, y = make_data(batch * steps, hw=hw, classes=classes)
    feed(s, x, y)
    losses = []
    for _ in range(steps):
        s.step(1)
        losses.append(float(s.last_loss))
    torch.cuda.synchronize()
    weights = {f"{n}.{j}": l.export_blob(j) for n, l in zip(s.net.layer_names, s.net.layers)
               for j in range(len(l.blobs))}
    s.close()
    return losses, weights


def test_odd_channel_net_matches_fp32_engine(ext):
    l_ref, w_ref = _run("torch", _odd_channel_net, 3, 4, 12, 10)
    l_sm, w_sm = _run("sm100", _odd_channel_net, 3, 4, 12, 10)
    for a, b in zip(l_ref, l_sm):
        assert abs(a - b) < 0.05 * max(1.0, abs(a)), (l_ref, l_sm)
    for name in w_ref:
        d = np.abs(w_ref[name] - w_sm[name]).max()
        mm = np.abs(w_ref[name] - 0.1).max() if name.endswith(".1") else np.abs(w_ref[name]).max()
        assert d <= 0.08 * mm + 3e-4, f"{name}: max diff {d} vs magnitude {mm}"


@pytest.mark.parametrize("name", ["lenet", "cifar10_quick"])
def test_small_zoo_models_train_on_sm100(ext, name):
    from poseidon_b200 import get_solver
    from poseidon_b200.models import zoo

    def run(engine):
        net = getattr(zoo, name)(batch=64)
        sp = zoo.get_solver_param(name, net=net, display=0, snapshot=0, snapshot_after_train=False, test_interval=0,
                                  max_iter=4, random_seed=3)
        sp.clear("test_iter")
        s = get_solver(sp, engine=engine, dtype=torch.float32 if engine == "torch" else None)
        out = []
        for _ in range(4):
            s.step(1)
            out.append(float(s.last_loss))
        s.close()
        return out

    l_sm, l_ref = run("sm100"), run("torch")
    for a, b in zip(l_ref, l_sm):
        assert abs(a - b) < 0.03 * max(1.0, abs(a)), (l_ref, l_sm)
