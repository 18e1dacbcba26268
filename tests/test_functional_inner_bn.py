"""Inner-loop BatchNorm gamma / beta (``enable_inner_loop_optimizable_bn_params``) through the functional network operator
``VGGReLUNormNetwork.forward`` (level B1): logits, first- and second-order reverse mode with cotangents on the gamma /
beta gradients, the mixed image term, forward mode along gamma / beta tangents (through the gradient too), the per-task
entries and ``torch.func`` with per-task gamma / beta, the running-statistics EMA, the reference's and the functorch
MAML loops, and the C entries.

Every fp64 reference is torch autograd / ``torch.func`` through ``maml_oracle._net_forward`` with beta / gamma as leaves in
``fast`` (with the flag the oracle reads them from there, without a step index).  Cases: the nine ``ibn_*`` fixtures;
every ``functional_cases.ENVELOPE`` shape as ``<case>_ibn`` (the fixture's args with the flag, the module's own
initialisation moved by ``maml_oracle.moved_state``: distinct gamma / beta per block and channel, the fixture's batch);
and two full-size configs on their target batches, Omniglot MAML++ 5w1s at 8 tasks and Mini-ImageNet MAML++ 5w1s at 2,
where the operator's own handles run the capped inner-BN grids (``engine_layout.norm_grid_regimes``).  Each compared
point prints its smallest fp64 margin (|pre-activation| and the gap between a pooling window's two largest activations);
below ``PIN_MARGIN`` the fp64 reference takes the GPU's leaky-ReLU branches and pooling arg-maxes (rebuilt from the
operator's handle) instead of its own.

Every tensor, beta / gamma included, is compared at the B1 policy: 5e-5 of the fp64 reference's max-norm.  The conv
biases are dead under BatchNorm (every derivative w.r.t. them is 0 in exact arithmetic): theirs is 5e-5 of the largest
max-norm of the tensors compared with them."""
import pytest
import torch
import torch.autograd.forward_ad as fwAD
import torch.nn.functional as Fnn
from torch.func import grad, jacrev, vjp, vmap

from conftest import grad_tolerance, load_golden
from engine_layout import geometry, grid_to_nchw, norm_grid_regimes, rel_err
import functional_cases as fc
from oracle import maml_oracle as O

PREFIX = "classifier."
FLAG = "enable_inner_loop_optimizable_bn_params"
IBN_CASES = ["ibn_tiny_pp", "ibn_tiny_pp_moved", "ibn_tiny_first", "ibn_tiny_maml", "ibn_one_stage", "ibn_ffma_wide",
             "ibn_bern", "ibn_eight_moved", "ibn_many_tasks"]
# full-size configs (target batch, the task count of test_inner_loop_bn's full-size cases): Omniglot at 8 tasks, and
# Mini-ImageNet at 2, whose 75-image batches run the capped inner-BN grids
FULL = {"ibn_full_omniglot_mamlpp_5w1s": ("omniglot_mamlpp_5w1s", 8),
        "ibn_full_mini_imagenet_mamlpp_5w1s": ("mini_imagenet_mamlpp_5w1s", 2)}
CAPPED = ["ibn_full_mini_imagenet_mamlpp_5w1s"]
CASES = IBN_CASES + [n + "_ibn" for n in fc.ENVELOPE] + list(FULL)
MOVED_SEED = 13
B1_REL = 5e-5          # B1 policy: 5e-5 of the fp64 reference's max-norm
PIN_MARGIN = 1e-6      # below this fp64 margin the reference takes the GPU's decisions


# ------------------------------------------------------------------------------------------------ helpers
def ibn_case(name):
    """(args, fp32 state, batch, which images the point uses) of an inner-BN fixture, of an envelope fixture run with the
    flag (``<case>_ibn``), or of a full-size config (seeded N(0, 1) episodes).  Full-size points use the target batch."""
    if name in IBN_CASES:
        g = load_golden(name)
        return g.args, g.state(), g.batch(0), "support"
    from howtotrainyourmamlpytorch_b200 import MAMLFewShotClassifier
    from howtotrainyourmamlpytorch_b200.configs import CONFIGS
    from howtotrainyourmamlpytorch_b200.utils.parser_utils import args_from_json
    if name in FULL:
        config, tasks = FULL[name]
        a = args_from_json(None, **dict(CONFIGS[config], batch_size=tasks, **{FLAG: True}))
        batch, which = O.synthetic_batch(a, iteration=0, kind="normal"), "target"
    else:
        g = load_golden(name[:-len("_ibn")])
        a = args_from_json(None, **dict(g.argdict, **{FLAG: True}))
        batch, which = g.batch(0), "support"
    torch.manual_seed(0)
    m = MAMLFewShotClassifier(im_shape=(2, a.image_channels, a.image_height, a.image_width), device="cpu", args=a)
    state = {k: v.detach().clone() for k, v in O.moved_state(m.state_dict(), a, MOVED_SEED).items()}
    return a, state, batch, which


def is_dead(n):
    return n.endswith("conv.bias")


def ref_logits(a, x, fast, forced=None):
    """fp64 logits: ``maml_oracle._net_forward`` with gamma / beta read from ``fast``; with ``forced`` (per-block (slope,
    idx)) the same network with those decisions pinned (``maml_oracle.block_forward``)."""
    if forced is None:
        return O._net_forward(x, fast, {}, a, 0)
    out = x
    for l in range(O.num_stages(a)):
        wn, bn_, gn, btn, _, _ = O.conv_names(l)
        out = O.block_forward(out, fast[wn], fast[bn_], fast[gn], fast[btn], forced[l])["p"]
    return Fnn.linear(out.reshape(out.shape[0], -1), fast[O.LIN_W], fast[O.LIN_B])


def fp64_margin(a, x, fast):
    """The smallest |pre-activation| and pooling-window gap (largest minus second largest activation) of the fp64 forward
    over the positions that reach the output."""
    out, worst = x.double(), float("inf")
    for l in range(O.num_stages(a)):
        wn, bn_, gn, btn, _, _ = O.conv_names(l)
        z = Fnn.conv2d(out, fast[wn].double(), fast[bn_].double(), padding=1)
        y = Fnn.batch_norm(z, None, None, fast[gn].double(), fast[btn].double(), training=True, eps=O.BN_EPS)
        n, c, h, w = y.shape
        yc = y[:, :, :h // 2 * 2, :w // 2 * 2]
        win = Fnn.leaky_relu(yc).reshape(n, c, h // 2, 2, w // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(n, c, h // 2, w // 2, 4)
        top = win.sort(dim=-1, descending=True).values
        worst = min(worst, float(yc.abs().min()), float((top[..., 0] - top[..., 1]).min()))
        out = Fnn.max_pool2d(Fnn.leaky_relu(y), 2, 2)
    return worst


def gpu_decisions(net, a, x, params):
    """The leaky-ReLU branches and pooling arg-maxes the GPU took in the operator's forward of x under params (one batch):
    its normalised activations read back from the first-order handle, y = fmaf(gamma, zh, beta) with params' own gamma /
    beta (the fp64 value rounded once to fp32), first max wins."""
    with torch.no_grad():
        net(x, 0, params=params)
    eng = net._handles(x).first_order
    geo, _ = geometry(a)
    F, n = int(a.cnn_num_filters), int(x.shape[-4])
    out = []
    for l, gl in enumerate(geo):
        zh = grid_to_nchw(eng.debug_read("tgt_zh", 0, 0, l), n, gl["h"], gl["w"], F)
        _, _, gn, btn, _, _ = O.conv_names(l)
        gam, bet = (params[k[len(PREFIX):]].detach().reshape(-1).cpu().double()[None, :, None, None] for k in (gn, btn))
        y = (gam * zh.double() + bet).float()
        slope = torch.where(y > 0, torch.ones_like(y), torch.full_like(y, 0.01))
        act = torch.where(y > 0, y, torch.tensor(0.01, dtype=torch.float32) * y)
        _, idx = Fnn.max_pool2d(act, 2, 2, return_indices=True)
        out.append((slope.double(), idx))
    return out


def point(tag, net, a, x, fast32, device):
    """Prints the fp64 margin of the forward at (x, fast32) and returns the decisions the fp64 reference uses there: None
    (its own) or the GPU's (on ``device``) when the margin is below PIN_MARGIN."""
    margin = fp64_margin(a, x.to(device), {k: v.to(device) for k, v in fast32.items()})
    pinned = margin < PIN_MARGIN
    print("[%s] smallest fp64 margin %.2e%s" % (tag, margin, " -> GPU decisions pinned" if pinned else ""))
    if not pinned:
        return None
    dec = gpu_decisions(net, a, x.to(device), {k[len(PREFIX):]: v.to(device) for k, v in fast32.items()})
    return [(s.to(device), i.to(device)) for s, i in dec]


def leaves64(a, state, x, device):
    """fp64 leaves on ``device``: the fast weights (gamma / beta included) and x, all requiring grad."""
    fast = {n: state[n].to(device, torch.float64).clone().requires_grad_(True) for n in O.inner_param_names(a)}
    return fast, x.to(device, torch.float64).clone().requires_grad_(True)


def op_params(m, a):
    """Fresh fp32 fast-weight leaves (requiring grad) for the operator, gamma / beta included, keyed as the reference passes
    them."""
    named = dict(m.named_parameters())
    return {n[len(PREFIX):]: named[n].detach().clone().requires_grad_(True) for n in O.inner_param_names(a)}


def check(rows, name, got, want, floor=0.0, rel=B1_REL):
    """|got - want|_inf within rel of max(|want|_inf, floor)."""
    got, want = got.detach().cpu().double().reshape(want.shape), want.detach().cpu().double()
    e = float((got - want).abs().max()) / max(float(want.abs().max()), floor, 1e-30)
    rows.append("%-64s rel %.2e%s" % (name, e, "" if e <= rel else "   <-- FAIL"))
    return e / rel


def check_all(rows, tag, names, got, want):
    """check() of every tensor of a set; the dead conv biases against the set's largest max-norm."""
    scale = max(float(w.detach().abs().max()) for w in want)
    return max(check(rows, "%s %s" % (tag, n), g_, w_, scale if is_dead(n) else 0.0) for n, g_, w_ in zip(names, got, want))


def report(case, what, rows, worst):
    print("\n[%s %s] worst %.2f x tolerance\n   " % (case, what, worst) + "\n   ".join(rows))
    assert not any(r.endswith("FAIL") for r in rows), "see the report above"


def ibn_engine(a, n, max_tasks, device, support, **kw):
    """A stand-alone engine handle of a's network for batches of n images (support or target shape)."""
    from howtotrainyourmamlpytorch_b200 import _native
    N = int(a.num_classes_per_set)
    with torch.cuda.device(device):
        return _native.Engine(n_way=N, k_shot=n // N if support else 1, t_target=1 if support else n // N,
                              channels=int(a.image_channels), height=int(a.image_height), width=int(a.image_width),
                              filters=int(a.cnn_num_filters), num_stages=int(a.num_stages),
                              inner_steps=int(a.number_of_training_steps_per_iter),
                              per_step_bn=bool(a.per_step_bn_statistics), max_tasks=max_tasks, **kw)


_ENGINE_CALLS = ("net_forward", "net_backward", "net_hvp", "net_hvp_image", "net_jvp", "net_forward_tasks",
                 "net_backward_tasks", "net_hvp_image_tasks", "net_jvp_tasks", "net_input_grad", "net_hvp_input_grad",
                 "net_running_update")


def _record_calls(monkeypatch, calls):
    from howtotrainyourmamlpytorch_b200 import _native
    for name in _ENGINE_CALLS:
        orig = getattr(_native.Engine, name)
        monkeypatch.setattr(_native.Engine, name,
                            lambda self, n_tasks, *rest, _o=orig, _n=name, **kw: (calls.append((_n, n_tasks)),
                                                                                   _o(self, n_tasks, *rest, **kw))[1])


# ------------------------------------------------------------------------------------------------ CPU
def test_operator_layout_and_cpu_refusal():
    """The operator's segments of an inner-BN network are its inner-loop tensors (gamma / beta [F] included), which are the
    engine's inner_bn meta layout minus LSLR; gamma / beta take tangent directions and may be batched under vmap there (a
    plain BatchNorm network's do neither); a CPU input raises NotImplementedError naming the flag."""
    from howtotrainyourmamlpytorch_b200.meta_neural_network_architectures import _refuse_batched_norm
    a, state, _, _ = ibn_case("ibn_tiny_pp")
    net = fc.model(a, state, "cpu").classifier
    assert [PREFIX + n for n in net._segment_names()] == O.inner_param_names(a)
    norm, directions = net._norm_segments()
    assert len(norm) == 2 * net.num_stages and directions
    _refuse_batched_norm(net, [0] * len(net._segment_names()))
    bn = fc.model(*fc.case("tiny_pp")[:2], "cpu").classifier
    norm, directions = bn._norm_segments()
    assert len(norm) == 2 * bn.num_stages and not directions
    with pytest.raises(NotImplementedError, match="batched"):
        _refuse_batched_norm(bn, [0] * len(bn._segment_names()))
    x = torch.zeros(int(a.num_classes_per_set), a.image_channels, a.image_height, a.image_width)
    with pytest.raises(NotImplementedError, match=FLAG):
        net(x, 0)


@pytest.mark.parametrize("case", CAPPED)
def test_full_size_cases_reach_the_capped_grids(case):
    """bn_grid and the backward reduce's cap restated on an H100's 132 SMs: the Mini-ImageNet case's target batch at its
    task count runs the capped inner-BN forward / apply and reduce grids, so a case whose shape drifts out of them fails
    here."""
    a, _, batch, _ = ibn_case(case)
    reached = norm_grid_regimes(a, int(batch[0].shape[0]))
    assert {"ibn_reduce_capped", "ibn_apply_capped"} <= reached, sorted(reached)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_logits_and_first_order_gradients(case, cuda_device):
    """(1) Logits against fp64, bit-identical at steps 0 and S - 1 (gamma / beta have no step index with the flag); the
    gradients of a cross-entropy w.r.t. every inner tensor (beta / gamma included) and the images against fp64 autograd."""
    a, state, batch, which = ibn_case(case)
    m = fc.model(a, state, cuda_device)
    net = m.classifier
    x, y = fc.images(batch, which)
    inner = O.inner_param_names(a)
    forced = point(case, net, a, x, {n: state[n] for n in inner}, cuda_device)
    fast, x64 = leaves64(a, state, x, cuda_device)
    logits64 = ref_logits(a, x64, fast, forced)
    g64 = torch.autograd.grad(Fnn.cross_entropy(logits64, y.to(cuda_device)), list(fast.values()) + [x64])
    S = int(a.number_of_training_steps_per_iter)
    outs = {}
    for step in sorted({0, S - 1}):
        params = op_params(m, a)
        xd = x.to(cuda_device).requires_grad_(True)
        logits = net(xd, step, params=params)
        gr = torch.autograd.grad(Fnn.cross_entropy(logits, y.to(cuda_device)), list(params.values()) + [xd])
        outs[step] = [logits.detach()] + [g_.detach() for g_ in gr]
    for o0, o1 in zip(outs[0], outs[S - 1]):
        assert torch.equal(o0, o1)
    rows = []
    worst = check(rows, "logits", outs[0][0], logits64)
    worst = max(worst, check_all(rows, "grad", inner + ["x"], outs[0][1:], g64))
    report(case, "logits and first-order gradients vs fp64", rows, worst)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_double_backward_and_mixed_image_term(case, cuda_device):
    """(2) g = grad(CE(op), fast weights incl. gamma / beta, create_graph=True), then the gradient of sum <g_i, v_i> w.r.t.
    every inner tensor and the images (x a leaf: the mixed term), with cotangents on the beta / gamma gradients alone and on
    all gradients, against fp64 autograd."""
    a, state, batch, which = ibn_case(case)
    m = fc.model(a, state, cuda_device)
    net = m.classifier
    x, y = fc.images(batch, which)
    inner = O.inner_param_names(a)
    gb = [n for n in inner if ".norm_layer." in n]
    forced = point(case, net, a, x, {n: state[n] for n in inner}, cuda_device)
    gen = torch.Generator().manual_seed(7)
    v = {n: torch.randn(state[n].shape, generator=gen, dtype=torch.float64).to(cuda_device) for n in inner}
    fast, x64 = leaves64(a, state, x, cuda_device)
    wrt64 = list(fast.values()) + [x64]
    yd = y.to(cuda_device)
    g = torch.autograd.grad(Fnn.cross_entropy(ref_logits(a, x64, fast, forced), yd), list(fast.values()), create_graph=True)
    selections = (("gamma / beta cotangents", gb), ("all cotangents", inner))
    ref = {what: torch.autograd.grad(sum((gi * v[n]).sum() for gi, n in zip(g, inner) if n in names), wrt64,
                                     retain_graph=True) for what, names in selections}
    rows, worst = [], 0.0
    params = op_params(m, a)
    xd = x.to(cuda_device).requires_grad_(True)
    wrt = list(params.values())
    gr = torch.autograd.grad(Fnn.cross_entropy(net(xd, 0, params=params), yd), wrt, create_graph=True)
    for what, names in selections:
        z = sum((gi * v[n].float().reshape(gi.shape)).sum() for gi, n in zip(gr, inner) if n in names)
        got = torch.autograd.grad(z, wrt + [xd], retain_graph=True)
        worst = max(worst, check_all(rows, what + ": d/d", inner + ["x (mixed term)"], got, ref[what]))
    report(case, "double backward vs fp64", rows, worst)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_forward_mode(case, cuda_device):
    """(3) J t (``forward_ad``) along the gamma / beta tangents alone and along every inner tensor and the images against
    torch.func.jvp in fp64; forward-over-reverse with a gamma / beta tangent reaching the backward (the tangent of every
    inner gradient) against fp64 autograd."""
    a, state, batch, which = ibn_case(case)
    m = fc.model(a, state, cuda_device)
    net = m.classifier
    named = dict(m.named_parameters())
    x, y = fc.images(batch, which)
    inner = O.inner_param_names(a)
    gb = [n for n in inner if ".norm_layer." in n]
    forced = point(case, net, a, x, {n: state[n] for n in inner}, cuda_device)
    gen = torch.Generator().manual_seed(9)
    t = {n: torch.randn(state[n].shape, generator=gen, dtype=torch.float64).to(cuda_device) for n in inner}
    xt = torch.randn(x.shape, generator=gen, dtype=torch.float64).to(cuda_device)
    fast, x64 = leaves64(a, state, x, cuda_device)
    prim = ({n: v_.detach() for n, v_ in fast.items()}, x64.detach())
    rows, worst = [], 0.0
    for direction in ("gamma / beta", "all"):
        tan = ({n: t[n] if direction == "all" or n in gb else torch.zeros_like(t[n]) for n in inner},
               xt if direction == "all" else torch.zeros_like(xt))
        _, want = torch.func.jvp(lambda f, xx: ref_logits(a, xx, f, forced), prim, tan)
        with fwAD.dual_level():
            params = {}
            for n in inner:
                p = named[n].detach().clone()
                params[n[len(PREFIX):]] = fwAD.make_dual(p, t[n].float()) if direction == "all" or n in gb else p
            xin = fwAD.make_dual(x.to(cuda_device), xt.float()) if direction == "all" else x.to(cuda_device)
            got = fwAD.unpack_dual(net(xin, 0, params=params)).tangent
        worst = max(worst, check(rows, "J t along %s" % direction, got, want))
    # forward-over-reverse along a gamma / beta tangent: d/de grad L(theta + e t_gb) = grad <grad_gb L, t_gb>
    yd = y.to(cuda_device)
    g = torch.autograd.grad(Fnn.cross_entropy(ref_logits(a, x64.detach(), fast, forced), yd), [fast[n] for n in gb],
                            create_graph=True)
    want = torch.autograd.grad(sum((g_ * t[n]).sum() for g_, n in zip(g, gb)), list(fast.values()))
    with fwAD.dual_level():
        leaves = op_params(m, a)
        params = dict(leaves)
        for n in gb:                                   # gamma / beta: dual views of their leaves
            params[n[len(PREFIX):]] = fwAD.make_dual(leaves[n[len(PREFIX):]], t[n].float())
        gr = torch.autograd.grad(Fnn.cross_entropy(net(x.to(cuda_device), 0, params=params), yd), list(leaves.values()),
                                 create_graph=True)
        got = [fwAD.unpack_dual(g_).tangent for g_ in gr]
    worst = max(worst, check_all(rows, "forward-over-reverse (gamma / beta tangent):", inner, got, want))
    report(case, "forward mode", rows, worst)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_per_task_entries_and_torch_func(case, cuda_device, monkeypatch):
    """(4) On inner_bn handles, B tasks with their own weights and gamma / beta (and their own directions): the per-task
    results (sum_tasks 0) of net_forward_tasks / net_backward_tasks / net_hvp_image_tasks / net_jvp_tasks match B
    one-task calls to 1e-5 of max-norm, each task's beta / gamma rows in its own result vector, and the summed result
    (sum_tasks 1) is their sum.  vmap of the operator with batched gamma / beta runs as one engine call per entry (n_tasks
    = B), and vmap(grad) matches per-task fp64 autograd at each task's own gamma / beta.  On the fixtures: jacrev of
    grad, and vjp of grad, w.r.t. a gamma, against fp64 (second order)."""
    a, state, batch, which = ibn_case(case)
    batch = fc.widen(batch)
    m = fc.model(a, state, cuda_device)
    net = m.classifier
    N, S = int(a.num_classes_per_set), int(a.number_of_training_steps_per_iter)
    xs_all, ys_all = (batch[0], batch[2]) if which == "support" else (batch[1], batch[3])
    B = xs_all.shape[0]
    x = xs_all.reshape(B, -1, *xs_all.shape[-3:]).float().to(cuda_device)
    y = ys_all.reshape(B, -1).long().to(cuda_device)
    n = x.shape[1]
    step = S - 1
    gen = torch.Generator().manual_seed(3)
    worst = {}

    def close(what, got, want, tol=1e-5):
        e = rel_err(got.cpu().double(), want.cpu().double())
        worst[what] = max(worst.get(what, 0.0), e / tol)
        assert e <= tol, (what, e)

    # ---- the C ABI (forward / backward on a target-shape handle, hvp / jvp on a support-shape one)
    fwd, sec = ibn_engine(a, n, B, cuda_device, False, inner_bn=True), ibn_engine(a, n, B, cuda_device, True, inner_bn=True)
    gb_segs = list(net._norm_segments()[0])
    scale = torch.tensor([1.0 + 0.05 * b for b in range(B)], device=cuda_device)
    metas = torch.stack([fc.meta_like(m, fwd, cuda_device)] * B) * scale[:, None]   # gamma / beta differ per task too
    dl = torch.randn(B, n, N, generator=gen).to(cuda_device)
    logits = torch.zeros(B, n, N, device=cuda_device)
    res, summed = torch.zeros(B, fwd.result_size, device=cuda_device), torch.zeros(fwd.result_size, device=cuda_device)
    fwd.net_forward_tasks(B, step, metas, fwd.meta_size, x, logits)
    fwd.net_backward_tasks(B, step, metas, fwd.meta_size, dl, res)
    fwd.net_backward_tasks(B, step, metas, fwd.meta_size, dl, summed, sum_tasks=True)
    P = fwd.meta_size
    close("summed grad", summed[:P], res[:, :P].sum(0))
    singles = []
    for b in range(B):
        one_l, one_g = torch.zeros(1, n, N, device=cuda_device), torch.zeros(fwd.result_size, device=cuda_device)
        fwd.net_forward_tasks(1, step, metas[b].contiguous(), 0, x[b:b + 1].contiguous(), one_l)
        fwd.net_backward_tasks(1, step, metas[b].contiguous(), 0, dl[b:b + 1].contiguous(), one_g, sum_tasks=True)
        close("logits", logits[b], one_l[0])
        close("grad", res[b, :P], one_g[:P])
        singles.append(one_g)
    for i in gb_segs:                                   # task b's beta / gamma rows are task b's, not another task's
        off, size = fwd.segments[i]
        for b in range(B):
            close("gamma / beta rows", res[b, off:off + size], singles[b][off:off + size])
            assert not torch.equal(res[b, off:off + size], res[(b + 1) % B, off:off + size])
    metas2 = torch.stack([fc.meta_like(m, sec, cuda_device)] * B) * scale[:, None]
    vs = torch.randn(B, sec.meta_size, generator=gen).to(cuda_device)     # per-task directions, gamma / beta included
    jvt, hvt = torch.zeros(B, n, N, device=cuda_device), torch.zeros(B, sec.result_size, device=cuda_device)
    jt = torch.zeros(B, n, N, device=cuda_device)
    sec.net_hvp_image_tasks(B, step, metas2, sec.meta_size, x, None, dl, vs, sec.meta_size, jvt, hvt)
    sec.net_jvp_tasks(B, step, metas2, sec.meta_size, x, vs, sec.meta_size, None, jt)
    for b in range(B):
        one_jv, one_hv = torch.zeros(1, n, N, device=cuda_device), torch.zeros(sec.result_size, device=cuda_device)
        one_jt = torch.zeros(1, n, N, device=cuda_device)
        args1 = (metas2[b].contiguous(), 0, x[b:b + 1].contiguous())
        sec.net_hvp_image_tasks(1, step, *args1, None, dl[b:b + 1].contiguous(), vs[b].contiguous(), 0, one_jv, one_hv,
                                sum_tasks=True)
        sec.net_jvp_tasks(1, step, *args1, vs[b].contiguous(), 0, None, one_jt)
        close("jv", jvt[b], one_jv[0])
        close("hv", hvt[b, :sec.meta_size], one_hv[:sec.meta_size])
        close("jvp_tasks", jt[b], one_jt[0])
        close("jvp_tasks = hvp's J v", jt[b], jvt[b])
    fwd.close()
    sec.close()

    # ---- torch.func: vmap with batched gamma / beta as one engine call; vmap(grad) against per-task fp64
    named = dict(m.named_parameters())
    inner = O.inner_param_names(a)
    per = {k[len(PREFIX):]: named[k].detach() * scale.view(-1, *[1] * named[k].dim()) for k in inner}
    calls = []
    _record_calls(monkeypatch, calls)
    got = vmap(lambda xb, p: net(xb, step, params=p))(x, per)

    def loss(p, xb, yb):
        return Fnn.cross_entropy(net(xb, step, params=p), yb)
    g_fast, g_x = vmap(grad(loss, argnums=(0, 1)))(per, x, y)
    monkeypatch.undo()
    assert [c for c in calls if c[0] == "net_forward_tasks"] == [("net_forward_tasks", B)] * 2, calls
    assert calls and all(t_ == B for _, t_ in calls), sorted(set(calls))
    rows, worst64 = [], 0.0
    for b in range(B):
        fast32 = {k: per[k[len(PREFIX):]][b] for k in inner}
        forced = point("%s task %d" % (case, b), net, a, x[b], fast32, cuda_device)
        f64 = {k: v_.double().clone().requires_grad_(True) for k, v_ in fast32.items()}
        x64 = x[b].double().clone().requires_grad_(True)
        l64 = ref_logits(a, x64, f64, forced)
        want = torch.autograd.grad(Fnn.cross_entropy(l64, y[b]), list(f64.values()) + [x64])
        worst64 = max(worst64, check(rows, "vmap logits, task %d" % b, got[b], l64))
        worst64 = max(worst64, check_all(rows, "vmap(grad) task %d" % b, inner + ["x"],
                                         [g_fast[k[len(PREFIX):]][b] for k in inner] + [g_x[b]], want))
    if case in IBN_CASES:
        # second order through torch.func: jacrev(grad) and vjp(grad) w.r.t. the last block's gamma, task 0
        kg = O.conv_names(O.num_stages(a) - 1)[2]
        x0, y0 = x[0], y[0]
        base = {k: per[k[len(PREFIX):]][0] for k in inner}
        forced = point(case + " jacrev", net, a, x0, base, cuda_device)

        def g_op(gam):
            return grad(lambda gg: loss({**{k[len(PREFIX):]: v_ for k, v_ in base.items()}, kg[len(PREFIX):]: gg}, x0, y0))(gam)

        def g_ref(gam):
            return torch.autograd.grad(Fnn.cross_entropy(ref_logits(a, x0.double(), {**{k: v_.double() for k, v_ in base.items()},
                                                                                     kg: gam}, forced), y0), gam,
                                       create_graph=True)[0]
        gam32 = base[kg]
        H = jacrev(g_op)(gam32)
        H64 = torch.autograd.functional.jacobian(g_ref, gam32.double())
        worst64 = max(worst64, check(rows, "jacrev(grad) w.r.t. %s" % kg[len(PREFIX):], H, H64))
        c = torch.randn(gam32.shape, generator=gen).to(cuda_device)
        _, pull = vjp(g_op, gam32)
        worst64 = max(worst64, check(rows, "vjp(grad) w.r.t. %s" % kg[len(PREFIX):], pull(c)[0], H64.t() @ c.double()))
    print("\n[%s per-task entries, B = %d] worst %s" % (case, B, " ".join("%s %.2f" % kv for kv in worst.items())))
    report(case, "torch.func vs per-task fp64", rows, worst64)


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in IBN_CASES if load_golden(c).args.per_step_bn_statistics] +
                         ["env_moved_pp_ibn", "ibn_full_mini_imagenet_mamlpp_5w1s"])
def test_running_statistics_ema(case, cuda_device):
    """(5) The operator's forward on a per-step inner-BN network leaves F.batch_norm's EMA of the batch statistics in
    running_mean / running_var[num_step] (each task's batch in order under vmap), against the fp64 reference's F.batch_norm
    with the same running statistics; the other steps' rows stay as they were."""
    a, state, batch, which = ibn_case(case)
    m = fc.model(a, state, cuda_device)
    net = m.classifier
    inner = O.inner_param_names(a)
    S = int(a.number_of_training_steps_per_iter)
    step = S - 1
    xs_all = batch[0] if which == "support" else batch[1]
    B = min(int(xs_all.shape[0]), 2)
    x = xs_all[:B].reshape(B, -1, *xs_all.shape[-3:]).float().to(cuda_device)
    st64 = {k: v_.to(cuda_device, torch.float64) for k, v_ in state.items()}
    stats = []
    with torch.no_grad():
        for b in range(B):
            O._net_forward(x[b].double(), {n: st64[n] for n in inner}, st64, a, step, stats_out=stats)
        vmap(lambda xb: net(xb, step))(x) if B > 1 else net(x[0], step)
    want = O.apply_running_stats(st64, a, stats)
    got = {k: v_.detach() for k, v_ in m.state_dict().items() if "running" in k}
    rows = []
    worst = 0.0
    for k, w_ in want.items():
        worst = max(worst, check(rows, k[len(PREFIX):], got[k][step], w_[step], rel=1e-5))
        others = [s for s in range(S) if s != step]
        assert torch.equal(got[k][others].cpu(), state[k][others]), k
    report(case, "running-statistics EMA vs F.batch_norm", rows, worst)


# ---- (6) the reference's second-order loop and the functorch loop on the operator ------------------------------------
def _reference_loop(m, a, batch, epoch, device):
    named = dict(m.named_parameters())
    net = m.classifier
    S = int(a.number_of_training_steps_per_iter)
    second_order = bool(a.second_order) and epoch > a.first_order_to_second_order_epoch
    sched = O.target_pass_schedule(a, epoch, True, S)
    w_msl = torch.from_numpy(O.msl_weights(a, epoch)).to(device)
    inner = O.inner_param_names(a)
    xs, xt, ys, yt = batch
    total, logits_out = [], []
    for b in range(xs.shape[0]):
        fast = {n: named[n] for n in inner}
        x_s, y_s = xs[b].reshape(-1, *xs.shape[-3:]).float().to(device), ys[b].reshape(-1).long().to(device)
        x_t, y_t = xt[b].reshape(-1, *xt.shape[-3:]).float().to(device), yt[b].reshape(-1).long().to(device)
        losses, last = [], None
        for s in range(S):
            params = {n[len(PREFIX):]: fast[n].unsqueeze(0) for n in inner}
            gr = torch.autograd.grad(Fnn.cross_entropy(net(x_s, s, params=params, training=True), y_s),
                                     [fast[n] for n in inner], create_graph=second_order)
            fast = {n: fast[n] - named[O.lslr_name(n)][s] * g_ for n, g_ in zip(inner, gr)}
            if sched[s] is not None:
                last = net(x_t, s, params={n[len(PREFIX):]: fast[n].unsqueeze(0) for n in inner}, training=True)
                lt = Fnn.cross_entropy(last, y_t)
                losses.append(w_msl[s] * lt if sched[s] == "msl" else lt)
        logits_out.append(last.detach().cpu())
        total.append(torch.stack(losses).sum())
    return torch.stack(total).mean(), torch.stack(logits_out)


def _functorch_loop(m, a, batch, epoch, device):
    """vmap over the meta-batch: gamma / beta enter shared and are per task (batched) after the first inner step."""
    named = dict(m.named_parameters())
    net = m.classifier
    S = int(a.number_of_training_steps_per_iter)
    second_order = bool(a.second_order) and epoch > a.first_order_to_second_order_epoch
    sched = O.target_pass_schedule(a, epoch, True, S)
    w_msl = torch.from_numpy(O.msl_weights(a, epoch)).to(device)
    inner = O.inner_param_names(a)
    xs, xt, ys, yt = batch
    B = xs.shape[0]
    xs, xt = (t_.reshape(B, -1, *t_.shape[-3:]).float().to(device) for t_ in (xs, xt))
    ys, yt = (t_.reshape(B, -1).long().to(device) for t_ in (ys, yt))

    def task(fast, x_s, y_s, x_t, y_t):
        losses, last = [], None
        for s in range(S):
            g_ = grad(lambda p: Fnn.cross_entropy(net(x_s, s, params=p), y_s))(fast)
            if not second_order:
                g_ = {k: v_.detach() for k, v_ in g_.items()}
            fast = {k: fast[k] - named[O.lslr_name(PREFIX + k)][s] * g_[k] for k in fast}
            if sched[s] is not None:
                last = net(x_t, s, params=fast)
                lt = Fnn.cross_entropy(last, y_t)
                losses.append(w_msl[s] * lt if sched[s] == "msl" else lt)
        return torch.stack(losses).sum(), last
    task_losses, logits = vmap(task, in_dims=(None, 0, 0, 0, 0))({n[len(PREFIX):]: named[n] for n in inner}, xs, ys, xt, yt)
    return task_losses.mean(), logits.detach().cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("loop", ["reference", "functorch"])
@pytest.mark.parametrize("case", IBN_CASES)
def test_maml_loops_on_operator_match_goldens(case, loop, cuda_device, monkeypatch):
    """(6) The reference's training loop (second order where the config says so) and the functorch loop (vmap over the
    meta-batch, every engine call at n_tasks = B) on the operator: loss, last-step logits and every outer gradient (gamma /
    beta and their LSLR rates included) against the unmodified reference's goldens at test_inner_loop_bn's tolerances,
    and against run_train_iter's fused iteration on the same model and batch."""
    g = load_golden(case)
    a, state = g.args, g.state()
    m = fc.model(a, state, cuda_device)
    batch, epoch = g.batch(0), g.iters[0][0]
    B = batch[0].shape[0]
    calls = []
    _record_calls(monkeypatch, calls)
    loss, logits = (_reference_loop if loop == "reference" else _functorch_loop)(m, a, batch, epoch, cuda_device)
    named = dict(m.named_parameters())
    names = O.trainable_names(a)
    gr = torch.autograd.grad(loss, [named[n] for n in names], allow_unused=True)
    monkeypatch.undo()
    grads = {n: (g_ if g_ is not None else torch.zeros_like(named[n])).detach().cpu() for n, g_ in zip(names, gr)}
    if loop == "functorch":
        assert calls and all(t_ == B for _, t_ in calls), sorted(set(calls))
    ref32, ref64 = g.scalar("loss"), g.scalar("loss64")
    assert abs(float(loss.detach()) - ref64) <= max(3 * abs(ref32 - ref64), 2e-5 * abs(ref64))
    ref_logits_ = torch.from_numpy(g.array("logits"))
    assert float((logits - ref_logits_).abs().max()) <= 1e-3 * float(ref_logits_.abs().max())
    _, _, fused = fc.model(a, state, cuda_device).meta_gradient(batch, epoch)
    g32, g64 = g.grads(0, ""), g.grads(0, "64")
    rows, bad, worst = [], [], 0.0
    for n in g64:
        tol = grad_tolerance(n, g32[n], g64[n])
        err = float((grads[n].double() - g64[n].double()).abs().max())
        err_fused = float((grads[n].double() - fused[n].cpu().double()).abs().max())
        worst = max(worst, err / tol, err_fused / tol)
        rows.append("%-74s err %.2e  vs fused %.2e  tol %.2e" % (n, err, err_fused, tol))
        if err > tol or err_fused > tol:
            bad.append(n)
    print("\n[%s %s loop on the operator] worst %.2f x tolerance\n   " % (case, loop, worst) + "\n   ".join(rows))
    assert not bad, bad


# ---- (7) the C entries ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_c_entries(cuda_device):
    """The five shared-weight entries refuse an inner_bn handle, naming inner_bn and the per-task entry; net_jvp_tasks at
    strides 0 is net_jvp bit for bit on a BatchNorm and a layer-norm handle (the operator's forward mode runs through it);
    a stride that is neither 0 nor >= meta_size fails."""
    a, state, batch, _ = ibn_case("ibn_tiny_pp")
    m = fc.model(a, state, cuda_device)
    x, _ = fc.images(batch, "support")
    n, N = x.shape[0], int(a.num_classes_per_set)
    x = x.unsqueeze(0).expand(2, *x.shape).contiguous().to(cuda_device)
    eng = ibn_engine(a, n, 2, cuda_device, True, inner_bn=True)
    meta = fc.meta_like(m, eng, cuda_device)
    dl = torch.zeros(2, n, N, device=cuda_device)
    out, res = torch.zeros(2, n, N, device=cuda_device), torch.zeros(eng.result_size, device=cuda_device)
    for name, call in (("net_forward", lambda: eng.net_forward(2, 0, meta, x, out)),
                       ("net_backward", lambda: eng.net_backward(2, 0, meta, dl, res)),
                       ("net_hvp_image", lambda: eng.net_hvp(2, 0, meta, x, dl, meta, out, res)),
                       ("net_hvp_image", lambda: eng.net_hvp_image(2, 0, meta, x, None, dl, meta, out, res)),
                       ("net_jvp", lambda: eng.net_jvp(2, 0, meta, x, meta, None, out))):
        with pytest.raises(RuntimeError, match="inner_bn.*maml_b200_%s_tasks" % name):
            call()
    for bad in (1, eng.meta_size - 1):
        with pytest.raises(RuntimeError, match="stride"):
            eng.net_jvp_tasks(2, 0, meta, bad, x, meta, 0, None, out)
        with pytest.raises(RuntimeError, match="stride"):
            eng.net_jvp_tasks(2, 0, meta, 0, x, meta, bad, None, out)
        with pytest.raises(RuntimeError, match="stride"):
            eng.net_forward_tasks(2, 0, meta, bad, x, out)
    eng.net_jvp_tasks(2, 0, meta, 0, x, meta, 0, None, out)          # strides 0: accepted
    assert float(out.abs().max()) > 0
    eng.close()
    gen = torch.Generator().manual_seed(5)
    for base, layer_norm in (("tiny_pp", False), ("ln_tiny_pp", True)):
        g = load_golden(base)
        mb = fc.model(g.args, g.state(), cuda_device)
        xb, _ = fc.images(g.batch(0), "support")
        xb = torch.stack([xb, xb * 0.5 + 0.1]).to(cuda_device)
        e = ibn_engine(g.args, xb.shape[1], 2, cuda_device, True, layer_norm=layer_norm)
        mt = fc.meta_like(mb, e, cuda_device)
        t_like = torch.randn(e.meta_size, generator=gen).to(cuda_device)
        xdot = torch.randn(xb.shape, generator=gen).to(cuda_device)
        for xd in (None, xdot):
            jv_a = torch.zeros(2, xb.shape[1], int(g.args.num_classes_per_set), device=cuda_device)
            jv_b = torch.ones_like(jv_a)
            e.net_jvp(2, 0, mt, xb, t_like, xd, jv_a)
            e.net_jvp_tasks(2, 0, mt, 0, xb, t_like, 0, xd, jv_b)
            assert torch.equal(jv_a, jv_b), (base, xd is None)
        e.close()
