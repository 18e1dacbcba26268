"""Second-order MAML through the functional-network operator (level B1): ``VGGReLUNormNetwork.forward`` differentiated
twice, the way the reference's training loop does it (``torch.autograd.grad(support_loss, fast_weights,
create_graph=True)`` in apply_inner_loop_update, few_shot_learning_system.py:138-139, then ``loss.backward()``).
The backward of the operator's backward runs on the engine (``maml_b200_net_hvp``)."""
import os
import sys

import pytest
import torch
import torch.nn.functional as Fnn

from conftest import BIG_CASES, TINY_CASES, load_golden, grad_tolerance
from engine_layout import rel_err
import functional_cases as fc
from oracle import maml_oracle as O

pytestmark = pytest.mark.gpu

PREFIX = "classifier."


def _check(rows, name, got, want, conv_bias_abs):
    """B1 backward policy: 5e-5 of the reference's max-norm; conv biases (dead parameters: BatchNorm removes them, every
    derivative w.r.t. them is 0) get an absolute bound on rounding noise."""
    got, want = got.detach().cpu().double().reshape(want.shape), want.detach().double()
    if "conv.bias" in name:
        e = float((got - want).abs().max())
        rows.append("%-62s abs %.2e" % (name, e))
        return e <= conv_bias_abs
    e = rel_err(got, want)
    rows.append("%-62s rel %.2e" % (name, e))
    return e <= 5e-5


@pytest.mark.parametrize("case", ["tiny_pp", "tiny_maml", "tiny_bern", "tiny_pp_moved"] + fc.ENVELOPE)
def test_double_backward_matches_fp64_autograd(case, cuda_device):
    """g = autograd.grad(CE(op(x, fast)), fast, create_graph=True), then autograd.grad(sum <g_i, v_i>) w.r.t. the fast
    weights AND the BatchNorm gamma / beta the module owns, against the same expression through the oracle's
    F.conv2d / F.batch_norm / ... network in float64.  The logits tangent J v reaches the weights through the
    cross-entropy's Hessian, so this exercises both outputs of the engine's pass; it is also compared on its own against
    torch.func.jvp of the oracle logits.  The gamma / beta rows pin the sign (+H_gamma v).  ``tiny_pp_moved``: distinct
    gamma / beta per step, nonzero biases."""
    a, state, batch = fc.case(case)
    m = fc.model(a, state, cuda_device)
    named = dict(m.named_parameters())
    xs, xt, ys, yt = batch
    x = xs[0].reshape(-1, *xs.shape[-3:])
    y = ys[0].reshape(-1).long()
    inner, bn = O.inner_param_names(a), fc.bn_names(state)
    gen = torch.Generator().manual_seed(7)
    v = {n: torch.randn(state[n].shape, generator=gen, dtype=torch.float64) for n in inner}
    c = torch.randn(x.shape[0], int(a.num_classes_per_set), generator=gen, dtype=torch.float64)
    S = int(a.number_of_training_steps_per_iter)
    rows, bad = [], []
    for step in sorted({0, S - 1}):
        # oracle, float64
        st64 = {k: t.double().clone().requires_grad_(k in bn) for k, t in state.items()}
        fast64 = {n: state[n].double().clone().requires_grad_(True) for n in inner}
        x64 = x.double()
        ref_loss = Fnn.cross_entropy(O._net_forward(x64, fast64, st64, a, step), y)
        ref_g = torch.autograd.grad(ref_loss, [fast64[n] for n in inner], create_graph=True)
        ref_hv = torch.autograd.grad(sum((gi * v[n]).sum() for gi, n in zip(ref_g, inner)),
                                     [fast64[n] for n in inner] + [st64[n] for n in bn])
        _, ref_jv = torch.func.jvp(lambda *w: O._net_forward(x64, dict(zip(inner, w)), st64, a, step),
                                   tuple(fast64[n].detach() for n in inner), tuple(v[n] for n in inner))
        # engine operator (fast weights with the reference's leading replica dim)
        params = {n[len(PREFIX):]: named[n].detach().clone().unsqueeze(0).requires_grad_(True) for n in inner}
        xd = x.to(cuda_device)
        loss = Fnn.cross_entropy(m.classifier.forward(xd, num_step=step, params=params, training=True), y.to(cuda_device))
        gr = torch.autograd.grad(loss, list(params.values()), create_graph=True)
        z = sum((gi * v[n].to(cuda_device, torch.float32).reshape(gi.shape)).sum() for gi, n in zip(gr, inner))
        hv = torch.autograd.grad(z, list(params.values()) + [named[n] for n in bn])
        scale = max(float(t.abs().max()) for t in ref_hv)
        for n, got, want in zip(inner + bn, hv, ref_hv):
            if not _check(rows, "s%d hv %s" % (step, n), got, want, 1e-4 + 5e-5 * scale):
                bad.append((step, n))
        # J v on its own: logits under fast weights with upstream cotangent cvec (requires grad) -> J^T cvec;
        # d/dcvec <J^T cvec, v> = J v
        cvec = c.to(cuda_device, torch.float32).requires_grad_(True)
        logits = m.classifier.forward(xd, num_step=step, params=params)
        jt = torch.autograd.grad(logits, list(params.values()), grad_outputs=cvec, create_graph=True)
        jv, = torch.autograd.grad(sum((gi * v[n].to(cuda_device, torch.float32).reshape(gi.shape)).sum()
                                      for gi, n in zip(jt, inner)), cvec)
        if not _check(rows, "s%d J v (logits tangent)" % step, jv, ref_jv, 0.0):
            bad.append((step, "jv"))
    print("\n[%s double backward vs fp64 autograd]\n   " % case + "\n   ".join(rows))
    assert not bad, bad


def _reference_loop_on_operator(m, a, batch, epoch, device):
    """oracle.autograd_train_iter's loop restated on the operator: the reference's fast weights (leading replica dim)
    through m.classifier.forward, torch.autograd.grad(create_graph=second_order), LSLR update, MSL-weighted target
    losses, then the outer gradient.  Also returns the oracle's running-statistics sequence, recomputed in float64 from
    the same fast weights."""
    named = dict(m.named_parameters())
    state64 = {k: v.detach().cpu().double() for k, v in m.state_dict().items()}
    S = int(a.number_of_training_steps_per_iter)
    second_order = bool(a.second_order) and epoch > a.first_order_to_second_order_epoch
    sched = O.target_pass_schedule(a, epoch, True, S)
    w_msl = torch.from_numpy(O.msl_weights(a, epoch)).to(device)
    inner = O.inner_param_names(a)
    xs, xt, ys, yt = batch
    stats, total, logits_out = [], [], []
    for b in range(xs.shape[0]):
        fast = {n: named[n] for n in inner}
        x_s, y_s = xs[b].reshape(-1, *xs.shape[-3:]), ys[b].reshape(-1).long()
        x_t, y_t = xt[b].reshape(-1, *xt.shape[-3:]), yt[b].reshape(-1).long()
        task_losses, last = [], None
        for s in range(S):
            def run(x, s=s):
                with torch.no_grad():
                    O._net_forward(x.double(), {n: fast[n].detach().cpu().double() for n in inner}, state64, a, s, stats)
                return m.classifier.forward(x.to(device), num_step=s, training=True,
                                            params={n[len(PREFIX):]: fast[n].unsqueeze(0) for n in inner})
            loss_s = Fnn.cross_entropy(run(x_s), y_s.to(device))
            grads = torch.autograd.grad(loss_s, [fast[n] for n in inner], create_graph=second_order)
            fast = {n: fast[n] - named[O.lslr_name(n)][s] * gr for n, gr in zip(inner, grads)}
            if sched[s] is not None:
                last = run(x_t)
                loss_t = Fnn.cross_entropy(last, y_t.to(device))
                task_losses.append(w_msl[s] * loss_t if sched[s] == "msl" else loss_t)
        logits_out.append(last.detach().cpu())
        total.append(torch.stack(task_losses).sum())
    loss = torch.stack(total).mean()
    names = O.trainable_names(a)
    gr = torch.autograd.grad(loss, [named[n] for n in names], allow_unused=True)
    grads = {n: (gi if gi is not None else torch.zeros_like(named[n])).detach().cpu() for n, gi in zip(names, gr)}
    return float(loss.detach()), torch.stack(logits_out), grads, stats


@pytest.mark.parametrize("case", TINY_CASES + ["omniglot_mamlpp_5w1s"] + fc.ENVELOPE)
def test_reference_loop_on_operator_matches_goldens(case, cuda_device):
    """The reference's training loop, second order where the config says so, with the network replaced by this
    operator: loss, last-step logits and every meta-gradient (LSLR included) vs the golden fixtures of the unmodified
    reference (tolerances of test_golden_reference_parity), the running statistics vs oracle.apply_running_stats, and
    the meta-gradient vs the fused iteration on the same batch.  tiny_pp_first pins the first-order route."""
    g = load_golden(case)
    a = g.args
    m = fc.model(a, g.state(), cuda_device)
    batch, epoch = g.batch(0), g.iters[0][0]
    state = g.state()
    loss, logits, grads, stats = _reference_loop_on_operator(m, a, batch, epoch, cuda_device)
    big = case in BIG_CASES
    flip_rel = 5e-4 if case == "tiny_odd" else None     # one pooling near-tie below an fp32 ulp (test_golden_reference_parity)
    ref_loss32, ref_loss64 = g.scalar("loss"), g.scalar("loss64")
    assert abs(loss - ref_loss64) <= max(3 * abs(ref_loss32 - ref_loss64), (5e-3 if big else 2e-5) * abs(ref_loss64))
    ref_logits = torch.from_numpy(g.array("logits"))
    assert logits.shape == ref_logits.shape
    assert float((logits - ref_logits).abs().max()) <= (0.25 if big else 1e-3) * float(ref_logits.abs().max())
    run = {k: v.detach().cpu() for k, v in m.state_dict().items() if "running" in k}
    ref_run = O.apply_running_stats(state, a, stats)
    for k in run:
        assert torch.allclose(run[k], ref_run[k].float(), rtol=5e-5, atol=5e-6), k
    g32, g64 = g.grads(0, ""), g.grads(0, "64")
    _, _, fused = fc.model(a, g.state(), cuda_device).meta_gradient(batch, epoch)
    rows, bad = [], []
    for n in g64:
        got = grads[n].double()
        if g.kind == "bernoulli" and not big and not ("conv.bias" in n or "conv-bias" in n):
            e32 = float((got - g32[n].double()).abs().max())
            own = float((g32[n].double() - g64[n].double()).abs().max())
            if e32 > max(3.0 * own, 2e-5 * float(g32[n].abs().max())) + 1e-7:
                bad.append(("fp32-anchored (near-ties)", n))
        tol = grad_tolerance(n, g32[n], g64[n], big=big)
        scale = max(float(g64[n].abs().max()), 1e-30)
        if flip_rel is not None and not ("conv.bias" in n or "conv-bias" in n):
            tol = max(tol, flip_rel * scale)
        err = float((got - g64[n].double()).abs().max())
        err_fused = float((got - fused[n].cpu().double()).abs().max())
        rows.append("%-78s err %.2e  vs fused %.2e  tol %.2e" % (n, err, err_fused, tol))
        if err > tol:
            bad.append(("golden", n))
        if err_fused > tol:
            bad.append(("fused", n))
    print("\n[%s reference loop on the operator (loss %.7f, ref64 %.7f)]\n   " % (case, loss, ref_loss64) + "\n   ".join(rows))
    assert not bad, bad


def test_unmodified_reference_class_trains_on_the_operator(cuda_device, monkeypatch):
    """The UNMODIFIED reference MAMLFewShotClassifier (staged under oracle/_ref) with its VGGReLUNormNetwork replaced by
    this repository's: train_forward_prop + backward (second order, tiny_pp) leaves the golden meta-gradients in .grad."""
    ref_dir = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")
    if not os.path.exists(os.path.join(ref_dir, "few_shot_learning_system.py")):
        pytest.skip("oracle/_ref is not staged (needs a reference checkout at build time)")
    from howtotrainyourmamlpytorch_b200.meta_neural_network_architectures import VGGReLUNormNetwork
    g = load_golden("tiny_pp")
    a = g.args
    assert a.second_order
    mods = ("few_shot_learning_system", "meta_neural_network_architectures", "inner_loop_optimizers")
    saved = {k: sys.modules.pop(k) for k in mods if k in sys.modules}
    sys.path.insert(0, ref_dir)
    try:
        import few_shot_learning_system as ref_fsl        # the reference, unmodified
        monkeypatch.setattr(ref_fsl, "VGGReLUNormNetwork", VGGReLUNormNetwork)
        monkeypatch.setattr(torch.cuda, "device_count", lambda: 1)      # no nn.DataParallel
        monkeypatch.setattr(a, "use_cuda", True)
        model = ref_fsl.MAMLFewShotClassifier(im_shape=(2, a.image_channels, a.image_height, a.image_width),
                                              device=cuda_device, args=a)
        model.load_state_dict({k: v.to(cuda_device) for k, v in g.state().items()})
        xs, xt, ys, yt = g.batch(0)
        batch = (xs.float().to(cuda_device), xt.float().to(cuda_device), ys.long().to(cuda_device), yt.long().to(cuda_device))
        losses, _ = model.train_forward_prop(data_batch=batch, epoch=g.iters[0][0])
        model.optimizer.zero_grad()
        losses["loss"].backward()
        g32, g64 = g.grads(0, ""), g.grads(0, "64")
        named = dict(model.named_parameters())
        assert abs(float(losses["loss"].detach()) - g.scalar("loss64")) <= max(3 * abs(g.scalar("loss") - g.scalar("loss64")),
                                                                      2e-5 * abs(g.scalar("loss64")))
        for n in g64:
            got = named[n].grad.detach().cpu().double()
            err = float((got - g64[n].double()).abs().max())
            assert err <= grad_tolerance(n, g32[n], g64[n]), (n, err)
    finally:
        sys.path.remove(ref_dir)
        for k in mods:
            sys.modules.pop(k, None)
        sys.modules.update(saved)


def test_batchnorm_gradient_output_is_not_differentiable(cuda_device):
    """A cotangent on the gradient of a BatchNorm gamma / beta needs gamma / beta tangent directions, which the engine
    does not have: NotImplementedError, not a wrong number."""
    g = load_golden("tiny_pp")
    a = g.args
    m = fc.model(a, g.state(), cuda_device)
    named = dict(m.named_parameters())
    xs, xt, ys, yt = g.batch(0)
    x = xs[0].reshape(-1, *xs.shape[-3:]).to(cuda_device)
    y = ys[0].reshape(-1).long().to(cuda_device)
    inner = O.inner_param_names(a)
    params = {n[len(PREFIX):]: named[n].detach().clone().unsqueeze(0).requires_grad_(True) for n in inner}
    gamma = named[fc.bn_names(g.state())[-1]]
    loss = Fnn.cross_entropy(m.classifier.forward(x, num_step=0, params=params), y)
    g_gamma, = torch.autograd.grad(loss, [gamma], create_graph=True)
    with pytest.raises(NotImplementedError, match="gamma / beta"):
        torch.autograd.grad(g_gamma.sum(), list(params.values()))
