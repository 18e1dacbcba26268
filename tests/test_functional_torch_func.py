"""The functional-network operator under ``torch.func``: ``vmap`` over tasks as ONE engine call (the per-task C-ABI
entries ``maml_b200_net_*_tasks``), ``grad`` / ``vjp`` / ``jacrev`` up to second order, and the functorch-style MAML loop
(``vmap`` over the meta-batch, inner ``torch.func.grad`` steps, outer ``torch.autograd.grad``)."""
import pytest
import torch
import torch.nn.functional as Fnn
from torch.func import grad, jacrev, vmap

from conftest import BIG_CASES, TINY_CASES, grad_tolerance, load_golden
from engine_layout import rel_err
import functional_cases as fc
from oracle import maml_oracle as O

pytestmark = pytest.mark.gpu

PREFIX = "classifier."


@pytest.fixture(scope="module")
def tiny_pp(cuda_device):
    a, state, batch = fc.case("tiny_pp")
    return a, state, batch, fc.model(a, state, cuda_device)


def _tasks(batch, which, device):
    """[B, n, C, H, W] images and [B, n] labels of every task of a golden batch."""
    xs, xt, ys, yt = batch
    x, y = (xs, ys) if which == "support" else (xt, yt)
    B = x.shape[0]
    return x.reshape(B, -1, *x.shape[-3:]).float().to(device), y.reshape(B, -1).long().to(device)


def _per_task_weights(m, a, B, device):
    """B distinct copies of the fast weights (task b scaled by 1 + 0.05 b), without the replica dim."""
    named = dict(m.named_parameters())
    scale = 1.0 + 0.05 * torch.arange(B, dtype=torch.float32, device=device)
    return {n[len(PREFIX):]: named[n].detach() * scale.view(-1, *[1] * named[n].dim()) for n in O.inner_param_names(a)}


def _oracle_logits(x, fast, state, a, step):
    """fp64 oracle logits of one task; `fast` without the classifier prefix."""
    st64 = {k: t.detach().cpu().double() for k, t in state.items()}
    f64 = {PREFIX + k: t.detach().cpu().double() for k, t in fast.items()}
    return O._net_forward(x.detach().cpu().double(), f64, st64, a, step)


# ---- 1. the per-task entries at the C ABI -------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["tiny_pp", "tiny_maml"] + fc.ENVELOPE)
def test_per_task_entries_at_the_c_abi(case, cuda_device):
    """Stride 0 + summing mode reproduces net_forward / net_backward / net_hvp_image bit for bit; B distinct weight vectors
    (and directions) with per-task results match B separate n_tasks = 1 calls to 1e-5 of max-norm.  B >= 3
    (functional_cases.widen)."""
    a, state, batch = fc.case(case)
    batch = fc.widen(batch)
    m = fc.model(a, state, cuda_device)
    xt, _ = _tasks(batch, "target", cuda_device)
    xs, _ = _tasks(batch, "support", cuda_device)
    B, N = xt.shape[0], int(a.num_classes_per_set)
    step = int(a.number_of_training_steps_per_iter) - 1
    gen = torch.Generator().manual_seed(3)
    fwd = fc.engine(a, 1, xt.shape[1] // N, B, cuda_device)
    meta = fc.meta_like(m, fwd, cuda_device)
    dl = torch.randn(B, xt.shape[1], N, generator=gen).to(cuda_device)
    out = {k: torch.zeros(B, fwd.result_size, device=cuda_device) for k in ("old", "new", "tasks")}
    lg = {k: torch.zeros(B, xt.shape[1], N, device=cuda_device) for k in ("old", "new")}
    fwd.net_forward(B, step, meta, xt, lg["old"])
    fwd.net_backward(B, step, meta, dl, out["old"][0])
    fwd.net_forward_tasks(B, step, meta, 0, xt, lg["new"])
    fwd.net_backward_tasks(B, step, meta, 0, dl, out["new"][0], sum_tasks=True)
    assert torch.equal(lg["old"], lg["new"]) and torch.equal(out["old"][0], out["new"][0])
    worst = {}

    def close(what, b, got, want):
        e = rel_err(got.cpu().double(), want.cpu().double())
        worst[what] = max(worst.get(what, 0.0), e)
        assert e <= 1e-5, (what, b, e)

    # B distinct weight vectors
    metas = torch.stack([meta * (1.0 + 0.05 * b) for b in range(B)])
    # BatchNorm gamma / beta are shared: every row carries task 0's
    logits = torch.zeros(B, xt.shape[1], N, device=cuda_device)
    fwd.net_forward_tasks(B, step, metas, fwd.meta_size, xt, logits)
    fwd.net_backward_tasks(B, step, metas, fwd.meta_size, dl, out["tasks"])
    for b in range(B):
        mb = metas[b].clone()
        for l in range(int(a.num_stages)):
            for seg in (4 * l + 2, 4 * l + 3):
                off, size = fwd.segments[seg]
                mb[off:off + size] = metas[0, off:off + size]
        one_l = torch.zeros(1, xt.shape[1], N, device=cuda_device)
        one_g = torch.zeros(fwd.result_size, device=cuda_device)
        fwd.net_forward(1, step, mb, xt[b:b + 1].contiguous(), one_l)
        fwd.net_backward(1, step, mb, dl[b:b + 1].contiguous(), one_g)
        close("logits", b, logits[b], one_l[0])
        close("grad", b, out["tasks"][b, :fwd.meta_size], one_g[:fwd.meta_size])

    # hvp on the support shape
    sec = fc.engine(a, xs.shape[1] // N, 1, B, cuda_device)
    meta2 = fc.meta_like(m, sec, cuda_device)
    dls = torch.randn(B, xs.shape[1], N, generator=gen).to(cuda_device)
    v = torch.randn(sec.meta_size, generator=gen).to(cuda_device)
    jv = {k: torch.zeros(B, xs.shape[1], N, device=cuda_device) for k in ("old", "new")}
    hv = {k: torch.zeros(B, sec.result_size, device=cuda_device) for k in ("old", "new", "tasks")}
    sec.net_hvp_image(B, step, meta2, xs, None, dls, v, jv["old"], hv["old"][0])
    sec.net_hvp_image_tasks(B, step, meta2, 0, xs, None, dls, v, 0, jv["new"], hv["new"][0], sum_tasks=True)
    assert torch.equal(jv["old"], jv["new"]) and torch.equal(hv["old"][0], hv["new"][0])
    metas2 = torch.stack([meta2 * (1.0 + 0.05 * b) for b in range(B)])
    vs = torch.stack([v * (1.0 - 0.1 * b) for b in range(B)])
    jvt = torch.zeros(B, xs.shape[1], N, device=cuda_device)
    sec.net_hvp_image_tasks(B, step, metas2, sec.meta_size, xs, None, dls, vs, sec.meta_size, jvt, hv["tasks"])
    for b in range(B):
        mb = metas2[b].clone()
        for l in range(int(a.num_stages)):
            for seg in (4 * l + 2, 4 * l + 3):
                off, size = sec.segments[seg]
                mb[off:off + size] = metas2[0, off:off + size]
        one_jv = torch.zeros(1, xs.shape[1], N, device=cuda_device)
        one_hv = torch.zeros(sec.result_size, device=cuda_device)
        sec.net_hvp_image(1, step, mb, xs[b:b + 1].contiguous(), None, dls[b:b + 1].contiguous(), vs[b].contiguous(), one_jv,
                          one_hv)
        close("jv", b, jvt[b], one_jv[0])
        close("hv", b, hv["tasks"][b, :sec.meta_size], one_hv[:sec.meta_size])
    print("\n[%s per-task entries vs n_tasks = 1, B = %d] worst rel %s" %
          (case, B, " ".join("%s %.2e" % kv for kv in worst.items())))


# ---- 2. vmap of the forward ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["tiny_pp", "tiny_maml", "tiny_bern", "tiny_pp_moved"] + fc.ENVELOPE)
def test_vmap_forward_matches_fp64_oracle(case, cuda_device):
    """vmap over B >= 3 tasks (functional_cases.widen) with the weights batched or shared and x batched or shared, against
    the fp64 oracle per task at the B1 policy (5e-5 of max-norm)."""
    a, state, batch = fc.case(case)
    batch = fc.widen(batch)
    m = fc.model(a, state, cuda_device)
    net = m.classifier
    x, _ = _tasks(batch, "target", cuda_device)
    B = x.shape[0]
    step = int(a.number_of_training_steps_per_iter) - 1
    shared = {n[len(PREFIX):]: p.detach() for n, p in m.named_parameters() if n in O.inner_param_names(a)}
    per = _per_task_weights(m, a, B, cuda_device)
    runs = {
        "x batched, weights shared": (vmap(lambda xb: net(xb, step, params=shared))(x), lambda b: (x[b], shared)),
        "x batched, weights batched": (vmap(lambda xb, p: net(xb, step, params=p))(x, per),
                                       lambda b: (x[b], {k: v[b] for k, v in per.items()})),
        "x shared, weights batched": (vmap(lambda p: net(x[0], step, params=p))(per),
                                      lambda b: (x[0], {k: v[b] for k, v in per.items()})),
    }
    bad, worst = [], 0.0
    for what, (got, task) in runs.items():
        assert got.shape[0] == B
        for b in range(B):
            xb, fast = task(b)
            e = rel_err(got[b].cpu().double(), _oracle_logits(xb, fast, state, a, step))
            worst = max(worst, e)
            if e > 5e-5:
                bad.append((what, b, e))
    print("\n[%s vmap forward vs fp64, B = %d] worst rel %.2e" % (case, B, worst))
    assert not bad, bad


# ---- 3. vmap(grad), grad of a summed vmap, jacrev --------------------------------------------------------------------------
def _fp64_task_grads(a, state, x, y, fast, step):
    """fp64 autograd of CE(oracle(x, fast)) w.r.t. the fast weights, BatchNorm gamma / beta and x."""
    st64 = {k: t.detach().cpu().double().clone().requires_grad_(k in fc.bn_names(state)) for k, t in state.items()}
    f64 = {k: t.detach().cpu().double().clone().requires_grad_(True) for k, t in fast.items()}
    x64 = x.detach().cpu().double().clone().requires_grad_(True)
    loss = Fnn.cross_entropy(O._net_forward(x64, {PREFIX + k: v for k, v in f64.items()}, st64, a, step), y.cpu())
    bn = fc.bn_names(state)
    gr = torch.autograd.grad(loss, list(f64.values()) + [st64[n] for n in bn] + [x64])
    k = len(f64)
    return dict(zip(f64, gr[:k])), dict(zip(bn, gr[k:-1])), gr[-1]


def _close(rows, name, got, want):
    got, want = got.detach().cpu().double().reshape(want.shape), want.double()
    if "conv.bias" in name:
        e = float((got - want).abs().max())
        rows.append("%-56s abs %.2e" % (name, e))
        return e <= 1e-5
    e = rel_err(got, want)
    rows.append("%-56s rel %.2e" % (name, e))
    return e <= 5e-5


@pytest.mark.parametrize("case", ["tiny_pp", "tiny_maml", "tiny_pp_moved"] + fc.ENVELOPE)
def test_vmap_grad_and_grad_of_summed_vmap(case, cuda_device):
    """Per-task gradients of the fast weights, of the module's BatchNorm gamma / beta (shared, passed unbatched) and of x
    (batched), through vmap(grad(loss)) and through grad of the summed vmap, against fp64 autograd per task.  B >= 3
    tasks (functional_cases.widen)."""
    a, state, batch = fc.case(case)
    batch = fc.widen(batch)
    m = fc.model(a, state, cuda_device)
    net = m.classifier
    named = dict(m.named_parameters())
    x, y = _tasks(batch, "support", cuda_device)
    B = x.shape[0]
    step = 0
    per = _per_task_weights(m, a, B, cuda_device)
    bn = {n[len(PREFIX):]: named[n].detach() for n in fc.bn_names(state)}

    def loss(fast, bnp, xb, yb):
        return Fnn.cross_entropy(net(xb, step, params={**fast, **bnp}), yb)

    g_fast, g_bn, g_x = vmap(grad(loss, argnums=(0, 1, 2)), in_dims=(0, None, 0, 0))(per, bn, x, y)
    s_fast, s_bn, s_x = grad(lambda f, p, xb: vmap(loss, in_dims=(0, None, 0, 0))(f, p, xb, y).sum(),
                             argnums=(0, 1, 2))(per, bn, x)
    rows, bad = [], []
    sum_bn = {}
    for b in range(B):
        rf, rbn, rx = _fp64_task_grads(a, state, x[b], y[b], {k: v[b] for k, v in per.items()}, step)
        for k in rf:
            for tag, got in (("vmap(grad)", g_fast[k][b]), ("grad(sum vmap)", s_fast[k][b])):
                if not _close(rows, "t%d %s %s" % (b, tag, k), got, rf[k]):
                    bad.append((b, tag, k))
        for n in rbn:
            sum_bn[n] = sum_bn.get(n, 0) + rbn[n]
            if not _close(rows, "t%d vmap(grad) %s" % (b, n), g_bn[n[len(PREFIX):]][b], rbn[n]):
                bad.append((b, "bn", n))
        for tag, got in (("vmap(grad)", g_x[b]), ("grad(sum vmap)", s_x[b])):
            if not _close(rows, "t%d %s x" % (b, tag), got, rx):
                bad.append((b, tag, "x"))
    for n, want in sum_bn.items():
        if not _close(rows, "grad(sum vmap) %s" % n, s_bn[n[len(PREFIX):]], want):
            bad.append(("sum", n))
    print("\n[%s torch.func gradients vs fp64]\n   " % case + "\n   ".join(rows))
    assert not bad, bad


def test_jacrev_of_logits(tiny_pp, cuda_device):
    """jacrev of the logits w.r.t. one conv weight (one batched backward: shared weights, batched cotangents) vs fp64."""
    a, state, batch, m = tiny_pp
    net = m.classifier
    x, _ = _tasks(batch, "support", cuda_device)
    x = x[0]
    fast = {n[len(PREFIX):]: p.detach() for n, p in m.named_parameters() if n in O.inner_param_names(a)}
    k = "layer_dict.conv1.conv.weight"
    J = jacrev(lambda w: net(x, 0, params={**fast, k: w}))(fast[k])
    st64 = {kk: t.double() for kk, t in state.items()}
    f64 = {PREFIX + kk: v.cpu().double() for kk, v in fast.items()}
    J64 = jacrev(lambda w: O._net_forward(x.cpu().double(), {**f64, PREFIX + k: w}, st64, a, 0))(f64[PREFIX + k])
    assert J.shape == J64.shape
    assert rel_err(J.cpu().double(), J64) <= 5e-5


# ---- 4./5. the functorch MAML loop -------------------------------------------------------------------------------------------
_ENGINE_CALLS = ("net_forward", "net_backward", "net_hvp", "net_hvp_image", "net_jvp", "net_forward_tasks",
                 "net_backward_tasks", "net_hvp_image_tasks", "net_input_grad", "net_hvp_input_grad", "net_running_update")


def _functorch_loop(m, a, batch, epoch, device):
    """PyTorch's functorch MAML recipe on the operator: vmap over the meta-batch, S inner torch.func.grad steps with the LSLR
    update (the gradient detached for first order), MSL-weighted target losses, outer torch.autograd.grad.  Returns the
    loss, last-step logits, meta-gradients and every task's fast weights before / after each step."""
    net = m.classifier
    named = dict(m.named_parameters())
    S = int(a.number_of_training_steps_per_iter)
    second_order = bool(a.second_order) and epoch > a.first_order_to_second_order_epoch
    sched = O.target_pass_schedule(a, epoch, True, S)
    w_msl = torch.from_numpy(O.msl_weights(a, epoch)).to(device)
    inner = O.inner_param_names(a)
    xs, ys = _tasks(batch, "support", device)
    xt, yt = _tasks(batch, "target", device)

    def task(fast, x_s, y_s, x_t, y_t):
        fasts, losses, last = [fast], [], None
        for s in range(S):
            g = grad(lambda p: Fnn.cross_entropy(net(x_s, s, params=p), y_s))(fast)
            if not second_order:
                g = {k: v.detach() for k, v in g.items()}
            fast = {k: fast[k] - named[O.lslr_name(PREFIX + k)][s] * g[k] for k in fast}
            fasts.append(fast)
            if sched[s] is not None:
                last = net(x_t, s, params=fast)
                loss_t = Fnn.cross_entropy(last, y_t)
                losses.append(w_msl[s] * loss_t if sched[s] == "msl" else loss_t)
        return torch.stack(losses).sum(), last, fasts

    fast0 = {n[len(PREFIX):]: named[n] for n in inner}
    task_losses, logits, fasts = vmap(task, in_dims=(None, 0, 0, 0, 0))(fast0, xs, ys, xt, yt)
    loss = task_losses.mean()
    names = O.trainable_names(a)
    gr = torch.autograd.grad(loss, [named[n] for n in names], allow_unused=True)
    grads = {n: (gi if gi is not None else torch.zeros_like(named[n])).detach().cpu() for n, gi in zip(names, gr)}
    fasts = [{k: v.detach().cpu().double() for k, v in f.items()} for f in fasts]
    return float(loss.detach()), logits.detach().cpu(), grads, fasts, sched


@pytest.mark.parametrize("case", TINY_CASES + ["omniglot_mamlpp_5w1s"] + fc.ENVELOPE)
def test_functorch_maml_loop_matches_goldens(case, cuda_device, monkeypatch):
    """The functorch MAML loop on the operator: loss, last-step logits and every meta-gradient (LSLR included) vs the
    golden fixtures (policy of test_reference_loop_on_operator_matches_goldens), the meta-gradient vs the fused iteration,
    the running statistics vs oracle.apply_running_stats fed in step-major order -- and every engine call of the loop ran
    with n_tasks = B (one call per mapped operator call, not B)."""
    from howtotrainyourmamlpytorch_b200 import _native
    g = load_golden(case)
    a = g.args
    state = g.state()
    m = fc.model(a, state, cuda_device)
    batch, epoch = g.batch(0), g.iters[0][0]
    B = batch[0].shape[0]
    calls = []
    for name in _ENGINE_CALLS:
        orig = getattr(_native.Engine, name)
        monkeypatch.setattr(_native.Engine, name,
                            lambda self, n_tasks, *rest, _o=orig, _n=name, **kw: (calls.append((_n, n_tasks)),
                                                                                   _o(self, n_tasks, *rest, **kw))[1])
    loss, logits, grads, fasts, sched = _functorch_loop(m, a, batch, epoch, cuda_device)
    monkeypatch.undo()
    assert calls and {n for n, _ in calls} >= {"net_forward_tasks", "net_backward_tasks"}
    assert all(t == B for _, t in calls), sorted(set(calls))
    if bool(a.second_order) and epoch > a.first_order_to_second_order_epoch:
        assert "net_hvp_image_tasks" in {n for n, _ in calls}

    big = case in BIG_CASES
    flip_rel = 5e-4 if case == "tiny_odd" else None
    ref_loss32, ref_loss64 = g.scalar("loss"), g.scalar("loss64")
    assert abs(loss - ref_loss64) <= max(3 * abs(ref_loss32 - ref_loss64), (5e-3 if big else 2e-5) * abs(ref_loss64))
    ref_logits = torch.from_numpy(g.array("logits"))
    assert logits.shape == ref_logits.shape
    assert float((logits - ref_logits).abs().max()) <= (0.25 if big else 1e-3) * float(ref_logits.abs().max())

    # running statistics: the oracle's EMA fed step-major (all support passes of step s, then all target passes)
    state64 = {k: v.double() for k, v in state.items()}
    xs, _ = _tasks(batch, "support", "cpu")
    xt, _ = _tasks(batch, "target", "cpu")
    stats = []
    with torch.no_grad():
        for s in range(int(a.number_of_training_steps_per_iter)):
            for b in range(B):
                O._net_forward(xs[b].double(), {PREFIX + k: v[b] for k, v in fasts[s].items()}, state64, a, s, stats)
            if sched[s] is not None:
                for b in range(B):
                    O._net_forward(xt[b].double(), {PREFIX + k: v[b] for k, v in fasts[s + 1].items()}, state64, a, s, stats)
    run = {k: v.detach().cpu() for k, v in m.state_dict().items() if "running" in k}
    ref_run = O.apply_running_stats(state, a, stats)
    for k in run:
        assert torch.allclose(run[k], ref_run[k].float(), rtol=5e-5, atol=5e-6), k

    g32, g64 = g.grads(0, ""), g.grads(0, "64")
    _, _, fused = fc.model(a, state, cuda_device).meta_gradient(batch, epoch)
    rows, bad = [], []
    for n in g64:
        got = grads[n].double()
        if g.kind == "bernoulli" and not big and not ("conv.bias" in n or "conv-bias" in n):
            e32 = float((got - g32[n].double()).abs().max())
            own = float((g32[n].double() - g64[n].double()).abs().max())
            if e32 > max(3.0 * own, 2e-5 * float(g32[n].abs().max())) + 1e-7:
                bad.append(("fp32-anchored (near-ties)", n))
        tol = grad_tolerance(n, g32[n], g64[n], big=big)
        if flip_rel is not None and not ("conv.bias" in n or "conv-bias" in n):
            tol = max(tol, flip_rel * max(float(g64[n].abs().max()), 1e-30))
        err = float((got - g64[n].double()).abs().max())
        err_fused = float((got - fused[n].cpu().double()).abs().max())
        rows.append("%-78s err %.2e  vs fused %.2e  tol %.2e" % (n, err, err_fused, tol))
        if err > tol:
            bad.append(("golden", n))
        if err_fused > tol:
            bad.append(("fused", n))
    print("\n[%s functorch loop on the operator (loss %.7f, ref64 %.7f)]\n   " % (case, loss, ref_loss64) + "\n   ".join(rows))
    assert not bad, bad


# ---- 6. refusals ---------------------------------------------------------------------------------------------------------------
def test_refusals_under_torch_func(tiny_pp, cuda_device):
    """A BatchNorm gamma / beta batched under vmap, torch.func.jvp / jacfwd through the operator and third order (under
    torch.func and under torch.autograd) raise NotImplementedError."""
    a, state, batch, m = tiny_pp
    net = m.classifier
    named = dict(m.named_parameters())
    x, y = _tasks(batch, "support", cuda_device)
    B = x.shape[0]
    fast = {n[len(PREFIX):]: p.detach() for n, p in m.named_parameters() if n in O.inner_param_names(a)}
    gname = fc.bn_names(state)[-1][len(PREFIX):]
    gamma = named[PREFIX + gname].detach()
    with pytest.raises(NotImplementedError, match="gamma / beta"):
        vmap(lambda gm: net(x[0], 0, params={**fast, gname: gm}))(gamma.unsqueeze(0).expand(B, *gamma.shape))
    k = "layer_dict.conv0.conv.weight"
    with pytest.raises(NotImplementedError, match="jvp"):
        torch.func.jvp(lambda w: net(x[0], 0, params={**fast, k: w}), (fast[k],), (torch.ones_like(fast[k]),))
    with pytest.raises(NotImplementedError, match="jvp"):
        torch.func.jacfwd(lambda w: net(x[0], 0, params={**fast, k: w}))(fast[k])

    def loss(w):
        return Fnn.cross_entropy(net(x[0], 0, params={**fast, k: w}), y[0])
    with pytest.raises(NotImplementedError, match="third"):
        grad(lambda w: grad(lambda u: grad(loss)(u).pow(2).sum())(w).sum())(fast[k])
    w0 = fast[k].clone().requires_grad_(True)
    g1, = torch.autograd.grad(loss(w0), w0, create_graph=True)
    g2, = torch.autograd.grad(g1.pow(2).sum(), w0, create_graph=True)
    with pytest.raises(NotImplementedError, match="third"):
        torch.autograd.grad(g2.sum(), w0)
