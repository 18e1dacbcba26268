"""Gradients with respect to the images through the functional-network operator (level B1): ``VGGReLUNormNetwork.forward``
differentiated w.r.t. ``x`` (``maml_b200_net_input_grad``: adversarial queries need dL/dx_target at the adapted weights)
and the mixed second-order term d/dx <grad_theta L, v> (``maml_b200_net_hvp_input_grad``: an outer loss reaches support
images only through the inner gradients, e.g. learned support sets)."""
import pytest
import torch
import torch.nn.functional as Fnn

from conftest import load_golden, grad_tolerance
from engine_layout import rel_err
import functional_cases as fc
from oracle import maml_oracle as O

pytestmark = pytest.mark.gpu

PREFIX = "classifier."
# synthetic_c4_f48: the C0 = 4 weight gradient's stream reduction needs more than the default 48 KB of shared memory
TINY = ["tiny_pp", "tiny_maml", "tiny_bern", "synthetic_c2", "synthetic_c4", "synthetic_c4_f48", "tiny_pp_moved"]
# B1 backward policy (DESIGN.md section 6): 5e-5 of the fp64 reference's max-norm
B1_REL = 5e-5


def _direction(a, state, seed=11):
    gen = torch.Generator().manual_seed(seed)
    return {n: torch.randn(state[n].shape, generator=gen, dtype=torch.float64) for n in O.inner_param_names(a)}


def _oracle_dx(a, state, x, y, step, v, device, dtype=torch.float64):
    """Autograd through the oracle network (fp64 unless asked): dL/dx (v None) or d/dx <grad_theta L, v>."""
    inner = O.inner_param_names(a)
    st64 = {k: t.to(device, dtype) for k, t in state.items()}
    fast = {n: st64[n].clone().requires_grad_(v is not None) for n in inner}
    x64 = x.to(device, dtype).requires_grad_(True)
    loss = Fnn.cross_entropy(O._net_forward(x64, fast, st64, a, step), y.to(device))
    if v is None:
        return torch.autograd.grad(loss, x64)[0].cpu()
    g = torch.autograd.grad(loss, [fast[n] for n in inner], create_graph=True)
    z = sum((gi * v[n].to(device)).sum() for gi, n in zip(g, inner))
    return torch.autograd.grad(z, x64)[0].cpu()


def _op_dx(m, a, x, y, step, v, device):
    inner = O.inner_param_names(a)
    named = dict(m.named_parameters())
    params = {n[len(PREFIX):]: named[n].detach().clone().unsqueeze(0).requires_grad_(v is not None) for n in inner}
    xd = x.to(device).requires_grad_(True)
    loss = Fnn.cross_entropy(m.classifier.forward(xd, num_step=step, params=params, training=True), y.to(device))
    if v is None:
        return torch.autograd.grad(loss, xd)[0].cpu()
    g = torch.autograd.grad(loss, list(params.values()), create_graph=True)
    z = sum((gi * v[n].to(device, torch.float32).reshape(gi.shape)).sum() for gi, n in zip(g, inner))
    return torch.autograd.grad(z, xd)[0].cpu()


def _per_call(case, order, device):
    a, state, batch = fc.case(case)
    m = fc.model(a, state, device)
    v = _direction(a, state) if order == 2 else None
    S = int(a.number_of_training_steps_per_iter)
    rows, worst = [], 0.0
    for which in ("target", "support"):
        x, y = fc.images(batch, which)
        for step in sorted({0, S - 1}):
            got = _op_dx(m, a, x, y, step, v, device)
            want = _oracle_dx(a, state, x, y, step, v, device)
            assert got.shape == x.shape and got.dtype == x.dtype
            e = rel_err(got.double(), want)
            worst = max(worst, e)
            rows.append("%-7s step %d  rel %.2e" % (which, step, e))
    print("\n[%s %s vs fp64 autograd]\n   " % (case, "dL/dx" if order == 1 else "d/dx <grad L, v>") + "\n   ".join(rows))
    return worst


@pytest.mark.parametrize("case", TINY + fc.ENVELOPE)
def test_input_grad_matches_fp64_autograd(case, cuda_device):
    """dL/dx of CE(op(x, fast)) against float64 autograd through the oracle's F.conv2d / F.batch_norm / ... network, at the
    first and last step, on the target and the support batch shape."""
    assert _per_call(case, 1, cuda_device) <= B1_REL


@pytest.mark.parametrize("case", TINY + fc.ENVELOPE)
def test_mixed_second_order_input_grad_matches_fp64_autograd(case, cuda_device):
    """d/dx <grad_theta L, v> for a random direction v over the conv / linear fast weights (the backward of the operator's
    backward, taken w.r.t. the images) against float64 autograd."""
    assert _per_call(case, 2, cuda_device) <= B1_REL


# Full size.  Two checks per step:
#  * the kernel: dx against an fp64 transposed convolution of the engine's OWN first-block output gradient (debug tap):
#    1e-6 of max-norm (measured 1.5e-7 on an H100), i.e. the data-gradient kernel is exact to fp32 summation noise;
#  * end to end against fp64 autograd: max(3 x |oracle32 - oracle64|, 5e-5) of max-norm.  dx is linear in the first
#    block's output gradient, so a pooling arg-max or leaky-ReLU branch that flips between any two fp32 evaluations
#    (DESIGN.md section 6, noise floor) moves a few pixels by an O(1) fraction of max-norm: on the Mini-ImageNet target
#    batch (75 images of 84x84x3) the fp32 oracle itself lands 5e-2 away from fp64 and this operator 4.8e-2, with 309 of
#    1.6e6 values off by more than 1e-4.  On Omniglot both sit near 3e-7.
@pytest.mark.parametrize("case", ["omniglot_mamlpp_5w1s", "mini_imagenet_mamlpp_5w1s"])
def test_input_grad_full_size_vs_own_dz0_and_oracle(case, cuda_device):
    a, state, batch = fc.case(case)
    m = fc.model(a, state, cuda_device)
    x, y = fc.images(batch, "target")
    rows, bad = [], []
    n, C, H, W = x.shape
    w0 = state["classifier.layer_dict.conv0.conv.weight"].double().to(cuda_device)
    tf32 = torch.backends.cudnn.allow_tf32
    for step in (0, int(a.number_of_training_steps_per_iter) - 1):
        got = _op_dx(m, a, x, y, step, None, cuda_device)
        eng = m.classifier._operator_handles[(n, cuda_device.index)].first_order
        dz0 = torch.from_numpy(eng.debug_read("tgt_dz", 0, 0, 0)).to(cuda_device, torch.float64)
        dz0 = dz0.view(n, H + 1, W + 1, -1)[:, 1:, 1:, :].permute(0, 3, 1, 2)      # padded grid -> NCHW
        own = Fnn.conv_transpose2d(dz0, w0, padding=1).cpu()
        want = _oracle_dx(a, state, x, y, step, None, cuda_device)
        torch.backends.cudnn.allow_tf32 = False
        try:
            want32 = _oracle_dx(a, state, x, y, step, None, cuda_device, torch.float32)
        finally:
            torch.backends.cudnn.allow_tf32 = tf32
        e, ek, e32 = rel_err(got.double(), want), rel_err(got.double(), own), rel_err(want32.double(), want)
        tol = max(3 * e32, B1_REL)
        rows.append("step %d  kernel vs fp64 of its own dz0 %.2e  end to end %.2e  oracle32 %.2e  tol %.2e" % (step, ek, e, e32, tol))
        if ek > 1e-6 or e > tol:
            bad.append(step)
    print("\n[%s dL/dx_target]\n   " % case + "\n   ".join(rows))
    assert not bad, rows


def _meta_loop(net, params, a, xs, xt, ys, yt, epoch):
    """The reference's inner loop (oracle.autograd_train_iter), always second order, with a pluggable network; returns the
    outer loss.  Support and target images are whatever the caller passes (leaves here)."""
    S = int(a.number_of_training_steps_per_iter)
    sched = O.target_pass_schedule(a, epoch, True, S)
    w_msl = torch.from_numpy(O.msl_weights(a, epoch)).to(xs.device, xs.dtype)
    inner = O.inner_param_names(a)
    total = []
    for b in range(xs.shape[0]):
        fast = {n: params[n] for n in inner}
        x_s, y_s = xs[b].reshape(-1, *xs.shape[-3:]), ys[b].reshape(-1).long()
        x_t, y_t = xt[b].reshape(-1, *xt.shape[-3:]), yt[b].reshape(-1).long()
        losses = []
        for s in range(S):
            g = torch.autograd.grad(Fnn.cross_entropy(net(x_s, fast, s), y_s), [fast[n] for n in inner], create_graph=True)
            fast = {n: fast[n] - params[O.lslr_name(n)][s] * gi for n, gi in zip(inner, g)}
            if sched[s] is not None:
                loss_t = Fnn.cross_entropy(net(x_t, fast, s), y_t)
                losses.append(w_msl[s] * loss_t if sched[s] == "msl" else loss_t)
        total.append(torch.stack(losses).sum())
    return torch.stack(total).mean()


def _oracle_loop_grads(a, state, batch, epoch, dtype):
    params = {k: v.to(dtype).clone().requires_grad_(k in O.inner_param_names(a)) for k, v in state.items()}
    xs, xt = (t.to(dtype).clone().requires_grad_(True) for t in batch[:2])
    loss = _meta_loop(lambda x, fast, s: O._net_forward(x, fast, params, a, s), params, a, xs, xt, batch[2], batch[3], epoch)
    return [gi.double() for gi in torch.autograd.grad(loss, [xs, xt])]


@pytest.mark.parametrize("case", ["tiny_pp", "tiny_maml", "tiny_bern", "omniglot_mamlpp_5w1s"])
def test_meta_loop_image_gradients_match_oracle(case, cuda_device):
    """The reference's second-order loop on the operator with x_support and x_target as leaves: d(outer loss)/d(x_support)
    (only through the inner gradients, i.e. the mixed term) and d(outer loss)/d(x_target) against the same loop on the
    oracle.  Bound: max(3 x |oracle32 - oracle64|, 2e-5 x max-norm) on the tiny cases, the chaos bound of DESIGN.md
    section 6 (5x the oracle's own fp32-vs-fp64 distance, floored at 2e-2 of max-norm) at full size."""
    g = load_golden(case)
    a, state, batch = g.args, g.state(), g.batch(0)
    epoch = g.iters[0][0]
    m = fc.model(a, state, cuda_device)
    named = dict(m.named_parameters())

    def op(x, fast, s):
        return m.classifier.forward(x, num_step=s, training=True, params={n[len(PREFIX):]: w.unsqueeze(0) for n, w in fast.items()})

    xs, xt = (t.float().to(cuda_device).requires_grad_(True) for t in batch[:2])
    loss = _meta_loop(op, named, a, xs, xt, batch[2].to(cuda_device), batch[3].to(cuda_device), epoch)
    got = [gi.detach().cpu().double() for gi in torch.autograd.grad(loss, [xs, xt])]
    o64 = _oracle_loop_grads(a, state, batch, epoch, torch.float64)
    o32 = _oracle_loop_grads(a, state, batch, epoch, torch.float32)
    big = case == "omniglot_mamlpp_5w1s"
    rows, bad = [], []
    for name, gt, w64, w32 in zip(("x_support", "x_target"), got, o64, o32):
        tol = grad_tolerance(name, w32, w64, big=big)
        err = float((gt - w64).abs().max())
        rows.append("%-10s err %.2e  oracle32 %.2e  tol %.2e  max-norm %.2e" %
                    (name, err, float((w32 - w64).abs().max()), tol, float(w64.abs().max())))
        if err > tol or not float(w64.abs().max()) > 0:
            bad.append(name)
    print("\n[%s meta loop image gradients]\n   " % case + "\n   ".join(rows))
    assert not bad, rows


def test_c_abi_tasks_and_call_order(cuda_device):
    """n_tasks = 2 gives the two n_tasks = 1 results bit for bit (both entries), and an entry that does not follow the call
    whose buffers it reads fails and writes nothing: the image-gradient entries after net_forward, after the other kind or
    with another n_tasks; net_backward and net_running_update on a fresh handle, after a net_hvp or with another n_tasks /
    num_step.  A repeated net_backward of one forward is accepted."""
    a, state, batch = fc.case("tiny_pp")
    m = fc.model(a, state, cuda_device)
    xs, xt = batch[0].float(), batch[1].float()
    x2 = torch.stack([xt[0].reshape(-1, *xt.shape[-3:]), xt[1 % xt.shape[0]].reshape(-1, *xt.shape[-3:]) * 0.5 + 0.1]).to(cuda_device)
    n, N, step = x2.shape[1], int(a.num_classes_per_set), int(a.number_of_training_steps_per_iter) - 1
    fwd, hvp = fc.engine(a, 1, n // N, 2, cuda_device), fc.engine(a, n // N, 1, 2, cuda_device)
    meta = fc.meta_like(m, fwd, cuda_device)
    gen = torch.Generator().manual_seed(3)
    dl = torch.randn(2, n, N, generator=gen).to(cuda_device)
    v = torch.randn(fwd.meta_size, generator=gen).to(cuda_device)
    logits = torch.empty(2, n, N, device=cuda_device)
    grad = torch.empty(fwd.result_size, device=cuda_device)
    jv, hv = torch.empty(2, n, N, device=cuda_device), torch.empty(hvp.result_size, device=cuda_device)

    def first(T, x, d):
        out = torch.empty(T, *x.shape[1:], device=cuda_device)
        fwd.net_forward(T, step, meta, x, logits)
        fwd.net_backward(T, step, meta, d, grad)
        fwd.net_input_grad(T, out)
        return out

    def mixed(T, x, d):
        out = torch.empty(T, *x.shape[1:], device=cuda_device)
        hvp.net_hvp(T, step, meta, x, d, v, jv, hv)
        hvp.net_hvp_input_grad(T, out)
        return out

    for f in (first, mixed):
        both = f(2, x2, dl)
        for t in range(2):
            one = f(1, x2[t:t + 1].contiguous(), dl[t:t + 1].contiguous())
            assert torch.equal(both[t], one[0]), (f.__name__, t)
        assert float(both.abs().max()) > 0

    sentinel = torch.full((2, n) + tuple(x2.shape[2:]), float("nan"), device=cuda_device)
    grad_sentinel = torch.full((fwd.result_size,), float("nan"), device=cuda_device)
    # running statistics: an EMA of NaN stays NaN, so these are finite and must keep their bits
    S, F = int(a.number_of_training_steps_per_iter), int(a.cnn_num_filters)
    run_mean = torch.zeros(int(a.num_stages), S, F, device=cuda_device)
    run_var = torch.ones_like(run_mean)

    def refused(call, match, *outs):
        outs = outs or (sentinel,)
        before = [o.clone() for o in outs]
        with pytest.raises(RuntimeError, match=match):
            call()
        torch.cuda.synchronize()
        for o, b in zip(outs, before):
            assert torch.equal(o.view(torch.int32), b.view(torch.int32)), "a refused call wrote its output"

    fresh = fc.engine(a, 1, n // N, 2, cuda_device)
    order = "must immediately follow maml_b200_net_forward or maml_b200_net_backward"
    refused(lambda: fresh.net_backward(2, step, meta, dl, grad_sentinel), order, grad_sentinel)
    refused(lambda: fresh.net_running_update(2, step, run_mean, run_var), order, run_mean, run_var)
    fresh.close()
    fwd.net_forward(2, step, meta, x2, logits)
    refused(lambda: fwd.net_input_grad(2, sentinel), "must immediately follow maml_b200_net_backward")
    refused(lambda: fwd.net_hvp_input_grad(2, sentinel), "must immediately follow maml_b200_net_hvp")
    refused(lambda: fwd.net_backward(2, (step + 1) % S, meta, dl, grad_sentinel), "num_step differs", grad_sentinel)
    refused(lambda: fwd.net_backward(1, step, meta, dl[:1].contiguous(), grad_sentinel), "n_tasks differs", grad_sentinel)
    fwd.net_backward(2, step, meta, dl, grad)
    again = torch.empty_like(grad)
    fwd.net_backward(2, step, meta, dl, again)       # a repeated backward of one forward is accepted and gives the same
    assert torch.equal(grad, again)
    refused(lambda: fwd.net_hvp_input_grad(2, sentinel), "must immediately follow maml_b200_net_hvp")
    refused(lambda: fwd.net_input_grad(1, sentinel), "n_tasks differs")
    # a net_hvp on the first-order handle (support shape: N images per batch) overwrites the forward's weights and statistics
    fwd.net_hvp(2, step, meta, x2[:, :N].contiguous(), dl[:, :N].contiguous(), v, torch.empty(2, N, N, device=cuda_device),
                torch.empty(fwd.result_size, device=cuda_device))
    refused(lambda: fwd.net_backward(2, step, meta, dl, grad_sentinel), order, grad_sentinel)
    refused(lambda: fwd.net_running_update(2, step, run_mean, run_var), order, run_mean, run_var)
    hvp.net_hvp(2, step, meta, x2, dl, v, jv, hv)
    refused(lambda: hvp.net_input_grad(2, sentinel), "must immediately follow maml_b200_net_backward")
    refused(lambda: hvp.net_hvp_input_grad(1, sentinel), "n_tasks differs")
    fwd.close()
    hvp.close()


def _weight_quantities(m, a, x, y, step, v, cvec, device):
    """First-order weight gradients, Hv and J v of the operator -- everything it produced before image gradients
    existed."""
    inner = O.inner_param_names(a)
    named = dict(m.named_parameters())
    params = {n[len(PREFIX):]: named[n].detach().clone().unsqueeze(0).requires_grad_(True) for n in inner}
    loss = Fnn.cross_entropy(m.classifier.forward(x, num_step=step, params=params), y)
    g = torch.autograd.grad(loss, list(params.values()), create_graph=True)
    z = sum((gi * v[n].to(device, torch.float32).reshape(gi.shape)).sum() for gi, n in zip(g, inner))
    hv = torch.autograd.grad(z, list(params.values()))
    cv = cvec.clone().requires_grad_(True)
    jt = torch.autograd.grad(m.classifier.forward(x, num_step=step, params=params), list(params.values()), grad_outputs=cv,
                             create_graph=True)
    jv, = torch.autograd.grad(sum((gi * v[n].to(device, torch.float32).reshape(gi.shape)).sum() for gi, n in zip(jt, inner)), cv)
    return [t.detach().clone() for t in list(g) + list(hv) + [jv]]


def test_weight_derivatives_unchanged_by_image_gradients(cuda_device, monkeypatch):
    """With x not requiring grad the operator never calls the image-gradient entries, and its weight gradients, Hv and
    J v are bit-identical to those computed with x requiring grad."""
    from howtotrainyourmamlpytorch_b200 import _native
    a, state, batch = fc.case("tiny_pp")
    m = fc.model(a, state, cuda_device)
    x, y = fc.images(batch, "support")
    x, y = x.to(cuda_device), y.to(cuda_device)
    v = _direction(a, state)
    cvec = torch.randn(x.shape[0], int(a.num_classes_per_set), generator=torch.Generator().manual_seed(5)).to(cuda_device)
    with_x = _weight_quantities(m, a, x.clone().requires_grad_(True), y, 1, v, cvec, cuda_device)

    def boom(*args, **kw):
        raise AssertionError("image-gradient entry called although x does not require grad")

    monkeypatch.setattr(_native.Engine, "net_input_grad", boom)
    monkeypatch.setattr(_native.Engine, "net_hvp_input_grad", boom)
    without_x = _weight_quantities(m, a, x, y, 1, v, cvec, cuda_device)
    assert len(with_x) == len(without_x)
    for i, (p, q) in enumerate(zip(with_x, without_x)):
        assert torch.equal(p, q), i


def test_image_gradient_output_is_not_differentiable(cuda_device):
    """A cotangent on the image gradient (e.g. a penalty on |dL/dx| differentiated again) needs image tangent directions,
    which the engine does not have: NotImplementedError, not a wrong number."""
    a, state, batch = fc.case("tiny_pp")
    m = fc.model(a, state, cuda_device)
    named = dict(m.named_parameters())
    x, y = fc.images(batch, "target")
    x = x.to(cuda_device).requires_grad_(True)
    params = {n[len(PREFIX):]: named[n].detach().clone().unsqueeze(0).requires_grad_(True) for n in O.inner_param_names(a)}
    loss = Fnn.cross_entropy(m.classifier.forward(x, num_step=0, params=params), y.to(cuda_device))
    dx, = torch.autograd.grad(loss, [x], create_graph=True)
    with pytest.raises(NotImplementedError, match="images"):
        torch.autograd.grad(dx.square().sum(), list(params.values()))
