"""The wgmma weight gradient of blocks l >= 1 (`wgrad_tc_row_kernel`, 3xTF32) against the exact-fp32 FFMA kernel
(`wgrad_row_kernel`, MAML_B200_WGRAD_TC=0), each on a model whose operator handles are created with the switch set.

Compared through the functional operator rather than a meta-gradient: the gradient of one backward pass (one operand
pair) and the Hessian-vector product of one tangent pass (two operand pairs: A (x) dz-dot + A-dot (x) dz).  Nothing
else in those passes depends on the weight gradient, so the two builds see the same activations and the same leaky-ReLU
and max-pool decisions, and the results differ by the weight gradient's rounding alone.  Every golden case, and every
filter count the engine admits.  Every case also runs a partial last stage (grid row counts such as 5 x 225 are not
multiples of 32) and windows that start on the guard rows."""
import pytest
import torch
import torch.nn.functional as Fnn

import functional_cases as fc
from conftest import ALL_CASES
from engine_layout import rel_err
from oracle import maml_oracle as O

pytestmark = pytest.mark.gpu

PREFIX = "classifier."


def _grad_and_hvp(a, state, x, y, device, monkeypatch, wgrad_tc):
    inner = O.inner_param_names(a)
    gen = torch.Generator().manual_seed(11)
    v = {n: torch.randn(state[n].shape, generator=gen) for n in inner}
    step = int(a.number_of_training_steps_per_iter) - 1
    with monkeypatch.context() as env:
        env.setenv("MAML_B200_WGRAD_TC", wgrad_tc)
        m = fc.model(a, state, device)                     # operator handles are created (and read the switch) on use
        named = dict(m.named_parameters())
        params = {n[len(PREFIX):]: named[n].detach().clone().unsqueeze(0).requires_grad_(True) for n in inner}
        loss = Fnn.cross_entropy(m.classifier.forward(x.to(device), num_step=step, params=params, training=True), y.to(device))
        g = torch.autograd.grad(loss, list(params.values()), create_graph=True)
        z = sum((gi * v[n].to(device).reshape(gi.shape)).sum() for gi, n in zip(g, inner))
        hv = torch.autograd.grad(z, list(params.values()))
    return inner, [t.detach() for t in g], [t.detach() for t in hv]


def _compare(a, state, x, y, device, monkeypatch):
    names, g0, h0 = _grad_and_hvp(a, state, x, y, device, monkeypatch, "0")
    _, g1, h1 = _grad_and_hvp(a, state, x, y, device, monkeypatch, "1")
    bad = []
    for what, r0, r1 in (("grad", g0, g1), ("hvp", h0, h1)):
        for n, want, got in zip(names, r0, r1):
            if "conv.bias" in n:
                err, ok = float((got - want).abs().max()), float((got - want).abs().max()) <= 1e-5
            else:
                err = rel_err(got, want)
                ok = err <= 2e-5
            if not ok:
                bad.append((what, n, err))
    assert not bad, bad


@pytest.mark.parametrize("case", ALL_CASES)
def test_wgrad_tc_matches_ffma_on_golden_cases(case, cuda_device, monkeypatch):
    a, state, batch = fc.case(case)
    x, y = fc.images(batch, "support")
    _compare(a, state, x, y, cuda_device, monkeypatch)


@pytest.mark.parametrize("filters", [16, 32, 48, 64])
def test_wgrad_tc_matches_ffma_for_every_filter_count(filters, cuda_device, monkeypatch):
    """Omniglot 5-way 1-shot geometry (block 1: 14 x 14 on a 15-wide grid) on the 5 support and 15 target images."""
    from howtotrainyourmamlpytorch_b200 import make_args
    a = make_args("omniglot_mamlpp_5w1s", batch_size=2, cnn_num_filters=filters, num_target_samples=3)
    state = O.init_state(a)
    batch = O.synthetic_batch(a, iteration=3, kind="normal")
    for which in ("support", "target"):
        x, y = fc.images(batch, which)
        _compare(a, state, x, y, cuda_device, monkeypatch)
