"""Forward-mode differentiation (``torch.autograd.forward_ad``) of the functional-network operator (level B1):
``VGGReLUNormNetwork.forward``'s logits tangent J_theta t + J_x x_dot (``maml_b200_net_jvp``), the tangent of its gradients
(forward-over-reverse, ``maml_b200_net_hvp_image``), and forward-mode hypergradients of the reference's second-order loop."""
import pytest
import torch
import torch.autograd.forward_ad as fwAD
import torch.nn.functional as Fnn

from conftest import load_golden
from engine_layout import rel_err
import functional_cases as fc
from oracle import maml_oracle as O

pytestmark = pytest.mark.gpu

PREFIX = "classifier."
# tiny_pp_moved: distinct gamma / beta per step (the gamma / beta tangent directions scale with the primal gamma)
TINY = ["tiny_pp", "tiny_maml", "tiny_bern", "synthetic_c2", "synthetic_c3", "synthetic_c4", "tiny_pp_moved"]
# odd image width: the first block's padded grid rows have an odd length, so every shared-memory tile staged behind an
# image window must be re-aligned (the two-pair weight-gradient kernels read their second dz tile as float4)
ODD_WIDTH = ["synthetic_c1_w15", "synthetic_c3_w15"]
DIRECTIONS = ["weights", "gamma_beta", "images", "all"]
B1_REL = 5e-5          # B1 policy (DESIGN.md section 6): 5e-5 of the fp64 reference's max-norm


def _tangents(a, state, x, direction, seed=7):
    """(weight tangents, gamma / beta tangents, image tangent) in fp64 on the CPU; the parts `direction` leaves out are {} /
    None."""
    gen = torch.Generator().manual_seed(seed)
    rnd = lambda t: torch.randn(t.shape, generator=gen, dtype=torch.float64)   # noqa: E731
    w = {n: rnd(state[n]) for n in O.inner_param_names(a)} if direction in ("weights", "all") else {}
    gb = {n: rnd(state[n]) for n in fc.bn_names(state)} if direction in ("gamma_beta", "all") else {}
    xd = rnd(x) if direction in ("images", "all") else None
    return w, gb, xd


def _oracle_jt(a, state, x, step, w, gb, xd, device, dtype=torch.float64):
    """J t through the oracle network with torch.func.jvp."""
    st = {k: t.to(device, dtype) for k, t in state.items()}
    inner, bn = O.inner_param_names(a), fc.bn_names(state)

    def f(x_, fast, bnp):
        return O._net_forward(x_, fast, {**st, **bnp}, a, step)
    prim = (x.to(device, dtype), {n: st[n] for n in inner}, {n: st[n] for n in bn})
    zero = lambda t: torch.zeros_like(t)   # noqa: E731
    tan = (xd.to(device, dtype) if xd is not None else zero(prim[0]),
           {n: (w[n].to(device, dtype) if n in w else zero(st[n])) for n in inner},
           {n: (gb[n].to(device, dtype) if n in gb else zero(st[n])) for n in bn})
    return torch.func.jvp(f, prim, tan)[1].cpu()


def _op_jt(m, a, x, step, w, gb, xd, device):
    named = dict(m.named_parameters())
    with fwAD.dual_level():
        params = {}
        for n in O.inner_param_names(a):
            p = named[n].detach().clone().unsqueeze(0)
            params[n[len(PREFIX):]] = fwAD.make_dual(p, w[n].to(device, torch.float32).unsqueeze(0)) if n in w else p
        for n in fc.bn_names(dict(m.state_dict())):
            p = named[n].detach().clone()
            params[n[len(PREFIX):]] = fwAD.make_dual(p, gb[n].to(device, torch.float32)) if n in gb else p
        xin = x.to(device)
        if xd is not None:
            xin = fwAD.make_dual(xin, xd.to(device, torch.float32))
        out = m.classifier.forward(xin, num_step=step, params=params, training=True)
        return fwAD.unpack_dual(out).tangent.cpu()


@pytest.mark.parametrize("direction", DIRECTIONS)
@pytest.mark.parametrize("case", TINY + fc.ENVELOPE)
def test_jvp_matches_fp64_autograd(case, direction, cuda_device):
    """J t (logits tangent) against torch.func.jvp in float64 through the oracle's network, at the first and last step, on
    the support and the target batch shape."""
    a, state, batch = fc.case(case)
    m = fc.model(a, state, cuda_device)
    S = int(a.number_of_training_steps_per_iter)
    rows, worst = [], 0.0
    for which in ("support", "target"):
        x, _ = fc.images(batch, which)
        w, gb, xd = _tangents(a, state, x, direction)
        for step in sorted({0, S - 1}):
            got = _op_jt(m, a, x, step, w, gb, xd, cuda_device)
            want = _oracle_jt(a, state, x, step, w, gb, xd, cuda_device)
            e = rel_err(got.double(), want)
            worst = max(worst, e)
            rows.append("%-7s step %d  rel %.2e" % (which, step, e))
    print("\n[%s J t along %s vs fp64]\n   " % (case, direction) + "\n   ".join(rows))
    assert worst <= B1_REL, rows


@pytest.mark.parametrize("case", TINY + ODD_WIDTH + fc.ENVELOPE)
def test_forward_over_reverse_matches_fp64_autograd(case, cuda_device):
    """Tangents of the weight gradients and of dx of CE(op(x, fast)) along (x_dot, theta_dot) -- with the d(logits) tangent
    that cross-entropy's backward produces -- against torch.func.jvp(torch.func.grad(...)) in float64."""
    a, state, batch = fc.case(case)
    m = fc.model(a, state, cuda_device)
    inner = O.inner_param_names(a)
    named = dict(m.named_parameters())
    S = int(a.number_of_training_steps_per_iter)
    rows, bad = [], []
    for which in ("support", "target"):
        x, y = fc.images(batch, which)
        w, _, xd = _tangents(a, state, x, "all")
        for step in sorted({0, S - 1}):
            with fwAD.dual_level():
                params = {n[len(PREFIX):]: fwAD.make_dual(named[n].detach().clone().unsqueeze(0).requires_grad_(True),
                                                          w[n].to(cuda_device, torch.float32).unsqueeze(0)) for n in inner}
                xin = fwAD.make_dual(x.to(cuda_device).requires_grad_(True), xd.to(cuda_device, torch.float32))
                loss = Fnn.cross_entropy(m.classifier.forward(xin, num_step=step, params=params, training=True),
                                         y.to(cuda_device))
                g = torch.autograd.grad(loss, list(params.values()) + [xin], create_graph=True)
                got = [fwAD.unpack_dual(gi).tangent.detach().cpu().double() for gi in g]
            st = {k: t.to(cuda_device, torch.float64) for k, t in state.items()}

            def loss64(x_, fast):
                return Fnn.cross_entropy(O._net_forward(x_, fast, st, a, step), y.to(cuda_device))
            prim = (x.to(cuda_device, torch.float64), {n: st[n] for n in inner})
            tan = (xd.to(cuda_device), {n: w[n].to(cuda_device) for n in inner})
            _, want = torch.func.jvp(lambda x_, f_: torch.func.grad(loss64, argnums=(0, 1))(x_, f_), prim, tan)
            wants = [want[1][n].cpu().reshape(gi.shape) for n, gi in zip(inner, got)] + [want[0].cpu()]
            for name, gt, wt in zip([n[len(PREFIX):] for n in inner] + ["x"], got, wants):
                err = float((gt.reshape(wt.shape) - wt).abs().max())
                scale = float(wt.abs().max())
                # conv biases are dead parameters (BatchNorm removes them): their exact tangent is 0, judged absolutely
                tol = 1e-4 + B1_REL * scale if name.endswith("conv.bias") else B1_REL * scale
                rows.append("%-7s s%d %-40s err %.2e  tol %.2e" % (which, step, name, err, tol))
                if err > tol:
                    bad.append(rows[-1])
    print("\n[%s forward-over-reverse vs fp64]\n   " % case + "\n   ".join(rows))
    assert not bad, bad


def _meta_loss(net, params, a, batch, epoch, device, dtype):
    """The reference's second-order inner loop (oracle.autograd_train_iter) with a pluggable network; the outer loss."""
    S = int(a.number_of_training_steps_per_iter)
    sched = O.target_pass_schedule(a, epoch, True, S)
    w_msl = torch.from_numpy(O.msl_weights(a, epoch)).to(device, dtype)
    inner = O.inner_param_names(a)
    xs, xt, ys, yt = (t.to(device) for t in batch)
    total = []
    for b in range(xs.shape[0]):
        fast = {n: params[n] for n in inner}
        x_s, y_s = xs[b].reshape(-1, *xs.shape[-3:]).to(dtype), ys[b].reshape(-1).long()
        x_t, y_t = xt[b].reshape(-1, *xt.shape[-3:]).to(dtype), yt[b].reshape(-1).long()
        losses = []
        for s in range(S):
            g = torch.autograd.grad(Fnn.cross_entropy(net(x_s, fast, s), y_s), [fast[n] for n in inner], create_graph=True)
            fast = {n: fast[n] - params[O.lslr_name(n)][s] * gi for n, gi in zip(inner, g)}
            if sched[s] is not None:
                loss_t = Fnn.cross_entropy(net(x_t, fast, s), y_t)
                losses.append(w_msl[s] * loss_t if sched[s] == "msl" else loss_t)
        total.append(torch.stack(losses).sum())
    return torch.stack(total).mean()


def _lslr_names(a):
    return [O.lslr_name(n) for n in O.inner_param_names(a)]


def _oracle_hypergrad(a, state, batch, epoch, alpha_dot, device, dtype):
    params = {k: v.to(device, dtype).clone().requires_grad_(k in O.inner_param_names(a) or k in alpha_dot)
              for k, v in state.items()}
    loss = _meta_loss(lambda x, fast, s: O._net_forward(x, fast, params, a, s), params, a, batch, epoch, device, dtype)
    g = torch.autograd.grad(loss, [params[n] for n in alpha_dot])
    return float(sum((gi.double() * alpha_dot[n].to(device)).sum() for gi, n in zip(g, alpha_dot)))


@pytest.mark.parametrize("case", ["tiny_pp", "tiny_maml"])
def test_forward_mode_hypergradient_of_meta_loop(case, cuda_device):
    """The reference's second-order loop on the operator with the LSLR vectors dual: the forward-mode d(meta-loss) . alpha_dot
    against reverse mode <grad_alpha L, alpha_dot> on the same operator, and against the fp64 oracle (bound of
    test_functional_second_order: max(3 x |oracle32 - oracle64|, 2e-5 x |oracle64|))."""
    g = load_golden(case)
    a, state, batch = g.args, g.state(), g.batch(0)
    epoch = g.iters[0][0]
    m = fc.model(a, state, cuda_device)
    named = dict(m.named_parameters())
    gen = torch.Generator().manual_seed(5)
    alpha_dot = {n: torch.randn(state[n].shape, generator=gen, dtype=torch.float64) for n in _lslr_names(a)}

    def op(x, fast, s):
        return m.classifier.forward(x, num_step=s, training=True, params={n[len(PREFIX):]: w.unsqueeze(0) for n, w in fast.items()})

    with fwAD.dual_level():
        params = {k: (fwAD.make_dual(v.detach().clone(), alpha_dot[k].to(cuda_device, torch.float32)) if k in alpha_dot
                      else v) for k, v in named.items()}
        loss = _meta_loss(op, params, a, batch, epoch, cuda_device, torch.float32)
        fwd = float(fwAD.unpack_dual(loss).tangent)
    rev_params = dict(named)          # the LSLR vectors as leaves (MAML's are not trainable parameters)
    rev_params.update({n: named[n].detach().clone().requires_grad_(True) for n in alpha_dot})
    loss = _meta_loss(op, rev_params, a, batch, epoch, cuda_device, torch.float32)
    grads = torch.autograd.grad(loss, [rev_params[n] for n in alpha_dot])
    rev = float(sum((gi.double().cpu() * alpha_dot[n]).sum() for gi, n in zip(grads, alpha_dot)))
    o64 = _oracle_hypergrad(a, state, batch, epoch, alpha_dot, cuda_device, torch.float64)
    o32 = _oracle_hypergrad(a, state, batch, epoch, alpha_dot, cuda_device, torch.float32)
    tol = max(3 * abs(o32 - o64), 2e-5 * abs(o64))
    print("\n[%s d(meta loss) . alpha_dot]  forward %.9e  reverse %.9e  oracle64 %.9e  oracle32 %.9e  tol %.2e" %
          (case, fwd, rev, o64, o32, tol))
    assert abs(fwd - rev) <= tol and abs(fwd - o64) <= tol and abs(rev - o64) <= tol


@pytest.mark.parametrize("case", ["omniglot_mamlpp_5w1s", "mini_imagenet_mamlpp_5w1s"])
def test_jvp_full_size(case, cuda_device):
    """J t along (weights, gamma / beta, images) on the full-size target batch: max(3 x |oracle32 - oracle64|, 5e-5) of
    max-norm, as the full-size image-gradient test bounds it (pooling / leaky-ReLU flips between fp32 evaluations)."""
    a, state, batch = fc.case(case)
    m = fc.model(a, state, cuda_device)
    x, _ = fc.images(batch, "target")
    w, gb, xd = _tangents(a, state, x, "all")
    tf32 = torch.backends.cudnn.allow_tf32
    rows, bad = [], []
    for step in (0, int(a.number_of_training_steps_per_iter) - 1):
        got = _op_jt(m, a, x, step, w, gb, xd, cuda_device)
        want = _oracle_jt(a, state, x, step, w, gb, xd, cuda_device)
        torch.backends.cudnn.allow_tf32 = False
        try:
            want32 = _oracle_jt(a, state, x, step, w, gb, xd, cuda_device, torch.float32)
        finally:
            torch.backends.cudnn.allow_tf32 = tf32
        e, e32 = rel_err(got.double(), want), rel_err(want32.double(), want)
        tol = max(3 * e32, B1_REL)
        rows.append("step %d  rel %.2e  oracle32 %.2e  tol %.2e" % (step, e, e32, tol))
        if e > tol:
            bad.append(step)
    print("\n[%s J t]\n   " % case + "\n   ".join(rows))
    assert not bad, rows


def test_c_abi_tasks_and_zero_image_tangent(cuda_device):
    """Through the C ABI: n_tasks = 2 gives the two n_tasks = 1 per-batch results bit for bit (net_jvp's J t; net_hvp_image's
    J v and, through net_hvp_input_grad, its image part), and net_hvp_image with x_dot = 0 gives net_hvp's J v and H v bit
    for bit.  H v is summed over the batches, so its n_tasks = 2 form is compared to the sum of the two to fp32 rounding."""
    a, state, batch = fc.case("tiny_pp")
    m = fc.model(a, state, cuda_device)
    xt = batch[1].float()
    x2 = torch.stack([xt[0].reshape(-1, *xt.shape[-3:]), xt[1 % xt.shape[0]].reshape(-1, *xt.shape[-3:]) * 0.5 + 0.1]).to(cuda_device)
    n, N, step = x2.shape[1], int(a.num_classes_per_set), int(a.number_of_training_steps_per_iter) - 1
    eng = fc.engine(a, n // N, 1, 2, cuda_device)
    meta = fc.meta_like(m, eng, cuda_device)
    gen = torch.Generator().manual_seed(3)
    t_like = torch.randn(eng.meta_size, generator=gen).to(cuda_device)
    xdot = torch.randn(x2.shape, generator=gen).to(cuda_device)
    dl = torch.randn(2, n, N, generator=gen).to(cuda_device)

    def jvp(T, x, xd, _dl):
        jv = torch.empty(T, n, N, device=cuda_device)
        eng.net_jvp(T, step, meta, x, t_like, xd, jv)
        return [jv.clone()], None

    def hvp_image(T, x, xd, d):
        jv, hv = torch.empty(T, n, N, device=cuda_device), torch.empty(eng.result_size, device=cuda_device)
        dxdot = torch.empty(T, *x.shape[1:], device=cuda_device)
        eng.net_hvp_image(T, step, meta, x, xd, d, t_like, jv, hv)
        eng.net_hvp_input_grad(T, dxdot)
        return [jv.clone(), dxdot], hv.clone()

    for f in (jvp, hvp_image):
        both = f(2, x2, xdot, dl)
        ones = [f(1, x2[t:t + 1].contiguous(), xdot[t:t + 1].contiguous(), dl[t:t + 1].contiguous()) for t in range(2)]
        for k, out in enumerate(both[0]):
            for t in range(2):
                assert torch.equal(out[t], ones[t][0][k][0]), (f.__name__, k, t)
            assert float(out.abs().max()) > 0
        if both[1] is not None:           # the meta-layout part (the first meta_size values) is the sum over the batches
            P = eng.meta_size
            summed = ones[0][1][:P] + ones[1][1][:P]
            assert float((both[1][:P] - summed).abs().max()) <= 1e-6 * float(summed.abs().max())

    jv_a, hv_a = torch.empty(2, n, N, device=cuda_device), torch.empty(eng.result_size, device=cuda_device)
    jv_b, hv_b = torch.empty_like(jv_a), torch.empty_like(hv_a)
    eng.net_hvp(2, step, meta, x2, dl, t_like, jv_a, hv_a)
    eng.net_hvp_image(2, step, meta, x2, torch.zeros_like(x2), dl, t_like, jv_b, hv_b)
    assert torch.equal(jv_a, jv_b) and torch.equal(hv_a, hv_b)


# kernel ids of the device trace (scripts/trace_kernel_ids.json)
K_CONV0, K_WGRAD0, K_INPUT_GRAD0, K_BNACT_TAN_GB = 2, 4, 31, 32


@pytest.mark.parametrize("case, call", [("env_c4_two_stages", "hvp_image"), ("env_ring_edge", "hvp_image"),
                                        ("env_one_stage", "jvp")])
def test_envelope_calls_reach_their_kernels(case, call, cuda_device):
    """The device trace of one call at the shapes the envelope parametrizations above exist for: net_hvp_image with
    x_dot != 0 and then net_hvp_input_grad run the first-block convolution and weight gradient and the image-gradient
    kernel, here in their two-pair forms (C0 = 4 with F = 64; C0 = 3 with F = 64 on 124-wide images, where the image
    gradient needs more than 48 KB of shared memory); net_jvp at L = 1 runs the gamma / beta-tangent BatchNorm kernel on
    block 0, whose pooled tangent is the head's input."""
    a, state, batch = fc.case(case)
    m = fc.model(a, state, cuda_device)
    x, _ = fc.images(batch, "support")
    x = x.unsqueeze(0).contiguous().to(cuda_device)
    n, N, step = x.shape[1], int(a.num_classes_per_set), int(a.number_of_training_steps_per_iter) - 1
    eng = fc.engine(a, n // N, 1, 1, cuda_device)
    meta = fc.meta_like(m, eng, cuda_device)
    gen = torch.Generator().manual_seed(3)
    t_like = torch.randn(eng.meta_size, generator=gen).to(cuda_device)
    xdot = torch.randn(x.shape, generator=gen).to(cuda_device)
    dl = torch.randn(1, n, N, generator=gen).to(cuda_device)
    jv = torch.empty(1, n, N, device=cuda_device)
    eng.trace(True)
    if call == "jvp":
        eng.net_jvp(1, step, meta, x, t_like, None, jv)
        want = {K_BNACT_TAN_GB}
    else:
        eng.net_hvp_image(1, step, meta, x, xdot, dl, t_like, jv, torch.empty(eng.result_size, device=cuda_device))
        eng.net_hvp_input_grad(1, torch.empty_like(x))
        want = {K_CONV0, K_WGRAD0, K_INPUT_GRAD0}
    torch.cuda.synchronize()
    ids = {k for _, k, _ in eng.trace_read(capacity=1 << 14) if not (k & 0x80)}
    eng.trace(False)
    eng.close()
    print("\n[%s %s] kernel ids %s" % (case, call, sorted(ids)))
    assert want <= ids, sorted(ids)
    assert float(jv.abs().max()) > 0


def test_gamma_beta_tangent_through_the_gradient_is_refused_before_any_launch(cuda_device):
    """A forward-mode tangent on a BatchNorm gamma / beta that reaches the operator's BACKWARD (forward-over-reverse) needs
    gamma / beta tangent directions in the backward tangent: refused before any launch.  (J t along gamma / beta itself,
    without the backward, is supported: test_jvp_matches_fp64_autograd.)"""
    a, state, batch = fc.case("tiny_pp")
    m = fc.model(a, state, cuda_device)
    x, y = fc.images(batch, "support")
    named = dict(m.named_parameters())
    bn = fc.bn_names(state)[0]
    with fwAD.dual_level():
        params = {n[len(PREFIX):]: named[n].detach().clone().unsqueeze(0).requires_grad_(True) for n in O.inner_param_names(a)}
        params[bn[len(PREFIX):]] = fwAD.make_dual(named[bn].detach().clone(), torch.ones_like(named[bn]))
        loss = Fnn.cross_entropy(m.classifier.forward(x.to(cuda_device), num_step=0, params=params, training=True),
                                 y.to(cuda_device))
        ops = m.classifier._operator_handles[(x.shape[0], cuda_device.index)]
        second_before = ops.second_order is not None
        gen_before = ops.gen
        torch.cuda.synchronize()
        with pytest.raises(NotImplementedError, match="gamma / beta"):
            torch.autograd.grad(loss, list(params.values())[:1], create_graph=True)
    # the refusal comes before the operator's handles are touched: no replayed forward, no second-order handle created by it
    assert ops.gen == gen_before and (ops.second_order is not None) == second_before
