"""The layer-norm network (``norm_layer: "layer_norm"``, reference MetaLayerNormLayer) through the functional network
operator ``VGGReLUNormNetwork.forward`` (level B1): logits, first- and second-order reverse mode, the mixed image term,
forward mode, the per-task entries and ``torch.func``, the reference's and the functorch MAML loops, and the refusals.

Every fp64 reference is torch autograd / ``torch.func`` through ``oracle.ln_oracle``'s network with the layer-norm bias as
a leaf.  Cases: the five layer-norm fixtures, and every ``functional_cases.ENVELOPE`` shape as a layer-norm case (the
fixture's args with ``norm_layer="layer_norm"``, the module's own initialisation moved by ``ln_oracle.moved_state``, the
fixture's batch).  Each compared point prints its smallest fp64 margin (|pre-activation| and the gap between a pooling
window's two largest activations); below ``PIN_MARGIN`` the fp64 reference takes the GPU's leaky-ReLU branches and pooling
arg-maxes (read from the operator's handle) instead of its own, as ``test_layer_norm`` does for the fused iteration.

Layer norm subtracts one mean over F*h*w, not one per channel, so the conv biases are live: every tensor, the conv biases
included, is compared at the B1 policy (5e-5 of the fp64 reference's max-norm)."""
import pytest
import torch
import torch.autograd.forward_ad as fwAD
import torch.nn.functional as Fnn
from torch.func import grad, jacrev, vmap

from conftest import load_golden
from engine_layout import geometry, grid_to_nchw, rel_err
import functional_cases as fc
from oracle import ln_oracle as LN
from oracle import maml_oracle as O

PREFIX = "classifier."
LN_CASES = ["ln_tiny_pp", "ln_tiny_pp_moved", "ln_tiny_maml", "ln_nonsquare_odd", "ln_bern"]
CASES = LN_CASES + [n + "_ln" for n in fc.ENVELOPE]
MOVED_SEED = 11
B1_REL = 5e-5          # B1 policy: 5e-5 of the fp64 reference's max-norm
PIN_MARGIN = 1e-6      # below this fp64 margin the reference takes the GPU's decisions


# ------------------------------------------------------------------------------------------------ helpers
def ln_case(name):
    """(args, fp32 state, batch) of a layer-norm fixture, or of an envelope fixture run with layer norm (``<case>_ln``)."""
    if not name.endswith("_ln"):
        g = load_golden(name)
        return g.args, g.state(), g.batch(0)
    from howtotrainyourmamlpytorch_b200 import MAMLFewShotClassifier
    from howtotrainyourmamlpytorch_b200.utils.parser_utils import args_from_json
    g = load_golden(name[:-len("_ln")])
    a = args_from_json(None, **dict(g.argdict, norm_layer="layer_norm"))
    torch.manual_seed(0)
    m = MAMLFewShotClassifier(im_shape=(2, a.image_channels, a.image_height, a.image_width), device="cpu", args=a)
    state = {k: v.detach().clone() for k, v in m.state_dict().items()}
    return a, LN.moved_state(state, a, MOVED_SEED), g.batch(0)


def bias_names(a):
    return [O.conv_names(l)[3] for l in range(O.num_stages(a))]


def ref_logits(a, x, fast, biases, forced=None):
    """fp64 logits: ``ln_oracle._net_forward`` with the layer-norm biases as given (leaves); with ``forced`` (per-block
    (slope, idx)) the same network with those decisions pinned (``ln_oracle.block_forward``)."""
    ones = {O.conv_names(l)[2]: torch.ones_like(biases[O.conv_names(l)[3]]).detach() for l in range(O.num_stages(a))}
    if forced is None:
        return LN._net_forward(x, fast, {**ones, **biases}, a)
    out = x
    for l in range(O.num_stages(a)):
        wn, bn_, gn, btn, _, _ = O.conv_names(l)
        out = LN.block_forward(out, fast[wn], fast[bn_], ones[gn], biases[btn], forced[l])["p"]
    return Fnn.linear(out.reshape(out.shape[0], -1), fast[O.LIN_W], fast[O.LIN_B])


def fp64_margin(a, x, fast, biases):
    """The smallest |pre-activation| and pooling-window gap (largest minus second largest activation) of the fp64 forward
    over the positions that reach the output."""
    out, worst = x.double(), float("inf")
    for l in range(O.num_stages(a)):
        wn, bn_, gn, btn, _, _ = O.conv_names(l)
        z = Fnn.conv2d(out, fast[wn].double(), fast[bn_].double(), padding=1)
        y = Fnn.layer_norm(z, z.shape[1:], None, biases[btn].double(), LN.LN_EPS)
        n, c, h, w = y.shape
        yc = y[:, :, :h // 2 * 2, :w // 2 * 2]
        win = Fnn.leaky_relu(yc).reshape(n, c, h // 2, 2, w // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(n, c, h // 2, w // 2, 4)
        top = win.sort(dim=-1, descending=True).values
        worst = min(worst, float(yc.abs().min()), float((top[..., 0] - top[..., 1]).min()))
        out = Fnn.max_pool2d(Fnn.leaky_relu(y), 2, 2)
    return worst


def gpu_decisions(net, a, x, params, task=0, tasks=1):
    """The leaky-ReLU branches and pooling arg-maxes the GPU took in the operator's forward of x under params: its
    normalised activations read back from the first-order handle, y = zh + b rounded once to fp32, first max wins."""
    with torch.no_grad():
        net(x, 0, params=params)
    eng = net._handles(x).first_order if tasks == 1 else net.__dict__["_operator_handles"][
        (int(x.shape[-4]), x.device.index, tasks)].first_order
    geo, _ = geometry(a)
    F, n = int(a.cnn_num_filters), int(x.shape[-4])
    own = dict(net.named_parameters())
    out = []
    for l, gl in enumerate(geo):
        zh = grid_to_nchw(eng.debug_read("tgt_zh", task, 0, l), n, gl["h"], gl["w"], F)
        b = own["layer_dict.conv%d.norm_layer.bias" % l].detach().cpu()
        y = (zh.double() + b.double()[None]).float()
        slope = torch.where(y > 0, torch.ones_like(y), torch.full_like(y, 0.01))
        act = torch.where(y > 0, y, torch.tensor(0.01, dtype=torch.float32) * y)
        _, idx = Fnn.max_pool2d(act, 2, 2, return_indices=True)
        out.append((slope.double(), idx))
    return out


def point(tag, m, a, state, x, device):
    """Prints the fp64 margin of the forward at (x, the module's weights) and returns the decisions the fp64 reference
    uses there: None (its own) or the GPU's when the margin is below PIN_MARGIN."""
    st = {k: v.double() for k, v in state.items()}
    margin = fp64_margin(a, x, st, st)
    pinned = margin < PIN_MARGIN
    print("[%s] smallest fp64 margin %.2e%s" % (tag, margin, " -> GPU decisions pinned" if pinned else ""))
    return gpu_decisions(m.classifier, a, x.to(device), None) if pinned else None


def leaves64(a, state, x):
    """fp64 leaves: the fast weights, the layer-norm biases and x, all requiring grad."""
    fast = {n: state[n].double().clone().requires_grad_(True) for n in O.inner_param_names(a)}
    biases = {n: state[n].double().clone().requires_grad_(True) for n in bias_names(a)}
    return fast, biases, x.double().clone().requires_grad_(True)


def op_params(m, a, with_biases=False):
    """Fresh fp32 fast-weight leaves (requiring grad) for the operator, keyed as the reference passes them; the module's
    own layer-norm bias Parameters (leaves requiring grad) with ``with_biases``."""
    named = dict(m.named_parameters())
    p = {n[len(PREFIX):]: named[n].detach().clone().requires_grad_(True) for n in O.inner_param_names(a)}
    b = {n[len(PREFIX):]: named[n] for n in bias_names(a)}
    return (p, b) if with_biases else p


def check(rows, name, got, want, rel=B1_REL):
    got, want = got.detach().cpu().double().reshape(want.shape), want.detach().cpu().double()
    e = rel_err(got, want)
    rows.append("%-64s rel %.2e%s" % (name, e, "" if e <= rel else "   <-- FAIL"))
    return e <= rel


def report(case, what, rows):
    print("\n[%s %s]\n   " % (case, what) + "\n   ".join(rows))
    assert not any(r.endswith("FAIL") for r in rows), "see the report above"


def ln_engine(a, n, max_tasks, device, support):
    """A stand-alone layer-norm handle for batches of n images (support or target shape)."""
    from howtotrainyourmamlpytorch_b200 import _native
    N = int(a.num_classes_per_set)
    with torch.cuda.device(device):
        return _native.Engine(n_way=N, k_shot=n // N if support else 1, t_target=1 if support else n // N,
                              channels=int(a.image_channels), height=int(a.image_height), width=int(a.image_width),
                              filters=int(a.cnn_num_filters), num_stages=int(a.num_stages),
                              inner_steps=int(a.number_of_training_steps_per_iter), per_step_bn=False,
                              max_tasks=max_tasks, layer_norm=True)


def _golden_tol(g32, g64, rel=2e-5):
    """test_layer_norm's golden policy: 3x the reference's own fp32-vs-fp64 distance, at least `rel` of its max-norm."""
    own = float((g32.double() - g64.double()).abs().max())
    return max(3 * own, rel * float(g64.abs().max()) + 1e-7)


# ------------------------------------------------------------------------------------------------ CPU
def test_operator_layout_and_cpu_refusal():
    """The operator's segments of a layer-norm network are the reference's outer parameters minus LSLR (conv.weight,
    conv.bias, norm_layer.bias per block: the frozen weight is not one); its norm tensors take tangent directions,
    BatchNorm's do not; a CPU input raises NotImplementedError naming the layer-norm operator."""
    a, state, _ = ln_case("ln_tiny_pp")
    m = fc.model(a, state, "cpu")
    net = m.classifier
    assert [PREFIX + n for n in net._segment_names()] == [n for n in LN.trainable_names(a) if "inner_loop" not in n]
    norm, directions = net._norm_segments()
    assert [net._segment_names()[i] for i in norm] == [n[len(PREFIX):] for n in bias_names(a)] and directions
    bn = fc.model(*fc.case("tiny_pp")[:2], "cpu").classifier
    norm, directions = bn._norm_segments()
    assert len(norm) == 2 * bn.num_stages and not directions
    x = torch.zeros(int(a.num_classes_per_set), a.image_channels, a.image_height, a.image_width)
    with pytest.raises(NotImplementedError, match="layer-norm"):
        net(x, 0)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_logits_and_first_order_gradients(case, cuda_device):
    """(1) Logits against fp64; bit-identical at steps 0 and S - 1 (the layer norm has no per-step rows); a query image's
    logits bit-identical when the other images of its batch change.  (2) The gradients of a cross-entropy w.r.t. the fast
    weights, the conv biases, the layer-norm biases and the images against fp64 autograd."""
    a, state, batch = ln_case(case)
    m = fc.model(a, state, cuda_device)
    net = m.classifier
    x, y = fc.images(batch, "support")
    forced = point(case, m, a, state, x, cuda_device)
    fast, biases, x64 = leaves64(a, state, x)
    logits64 = ref_logits(a, x64, fast, biases, forced)
    g64 = torch.autograd.grad(Fnn.cross_entropy(logits64, y), list(fast.values()) + list(biases.values()) + [x64])
    S = int(a.number_of_training_steps_per_iter)
    outs = {}
    for step in sorted({0, S - 1}):
        params, own_b = op_params(m, a, with_biases=True)
        xd = x.to(cuda_device).requires_grad_(True)
        logits = net(xd, step, params=params)
        gr = torch.autograd.grad(Fnn.cross_entropy(logits, y.to(cuda_device)),
                                 list(params.values()) + list(own_b.values()) + [xd])
        outs[step] = [logits.detach()] + [g.detach() for g in gr]
    for o0, o1 in zip(outs[0], outs[S - 1]):
        assert torch.equal(o0, o1)
    rows = []
    check(rows, "logits", outs[0][0], logits64.detach())
    for n, got, want in zip(list(fast) + list(biases) + ["x"], outs[0][1:], g64):
        check(rows, "grad " + n, got, want)
    # non-transductivity: image 0's logits do not depend on the other images of the batch
    gen = torch.Generator().manual_seed(5)
    x2 = x.clone()
    x2[1:] = torch.randn(x2[1:].shape, generator=gen) * 3.0
    with torch.no_grad():
        l2 = net(x2.to(cuda_device), 0)
        l1 = net(x.to(cuda_device), 0)
    assert torch.equal(l1[0], l2[0])
    report(case, "logits and first-order gradients vs fp64", rows)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_double_backward_and_mixed_image_term(case, cuda_device):
    """(3) g = grad(CE(op), fast weights + layer-norm biases, create_graph=True), then the gradient of sum <g_i, v_i>
    w.r.t. the weights, the biases and (4) the images -- with cotangents on the weight gradients, and separately on the
    bias gradients (bias directions of the engine's tangent pass) -- against fp64 autograd; J v along weights and biases on
    its own against torch.func.jvp."""
    a, state, batch = ln_case(case)
    m = fc.model(a, state, cuda_device)
    net = m.classifier
    x, y = fc.images(batch, "support")
    forced = point(case, m, a, state, x, cuda_device)
    inner, bns = O.inner_param_names(a), bias_names(a)
    gen = torch.Generator().manual_seed(7)
    v = {n: torch.randn(state[n].shape, generator=gen, dtype=torch.float64) for n in inner + bns}
    c = torch.randn(x.shape[0], int(a.num_classes_per_set), generator=gen, dtype=torch.float64)
    fast, biases, x64 = leaves64(a, state, x)
    wrt64 = list(fast.values()) + list(biases.values()) + [x64]
    g = torch.autograd.grad(Fnn.cross_entropy(ref_logits(a, x64, fast, biases, forced), y),
                            list(fast.values()) + list(biases.values()), create_graph=True)
    ref = {}
    for what, names in (("weight cotangents", inner), ("bias cotangents", bns)):
        z = sum((gi * v[n]).sum() for gi, n in zip(g, inner + bns) if n in names)
        ref[what] = torch.autograd.grad(z, wrt64, retain_graph=True)
    _, ref_jv = torch.func.jvp(lambda f, b: ref_logits(a, x64.detach(), f, b, forced),
                               ({n: t.detach() for n, t in fast.items()}, {n: t.detach() for n, t in biases.items()}),
                               ({n: v[n] for n in inner}, {n: v[n] for n in bns}))
    S = int(a.number_of_training_steps_per_iter)
    rows, outs = [], {}
    for step in sorted({0, S - 1}):
        params, own_b = op_params(m, a, with_biases=True)
        xd = x.to(cuda_device).requires_grad_(True)
        wrt = list(params.values()) + list(own_b.values())
        gr = torch.autograd.grad(Fnn.cross_entropy(net(xd, step, params=params), y.to(cuda_device)), wrt, create_graph=True)
        got = {}
        for what, names in (("weight cotangents", inner), ("bias cotangents", bns)):
            z = sum((gi * v[n].to(cuda_device, torch.float32).reshape(gi.shape)).sum()
                    for gi, n in zip(gr, inner + bns) if n in names)
            got[what] = [t.detach() for t in torch.autograd.grad(z, wrt + [xd], retain_graph=True)]
        # J v on its own: d/dc <J^T c, v> = J v
        cvec = c.to(cuda_device, torch.float32).requires_grad_(True)
        jt = torch.autograd.grad(net(x.to(cuda_device), step, params=params), wrt, grad_outputs=cvec, create_graph=True)
        jv, = torch.autograd.grad(sum((gi * v[n].to(cuda_device, torch.float32).reshape(gi.shape)).sum()
                                      for gi, n in zip(jt, inner + bns)), cvec)
        outs[step] = got["weight cotangents"] + got["bias cotangents"] + [jv.detach()]
        if step == 0:
            for what in got:
                for n, gt, want in zip(inner + bns + ["x (mixed term)"], got[what], ref[what]):
                    check(rows, "%s: d/d %s" % (what, n), gt, want)
            check(rows, "J v (weights + biases)", jv, ref_jv)
    for o0, o1 in zip(outs[0], outs[S - 1]):
        assert torch.equal(o0, o1)
    report(case, "double backward vs fp64", rows)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_forward_mode(case, cuda_device):
    """(5) J t along the weights, the layer-norm biases, the images and all three (``forward_ad``) against torch.func.jvp in
    fp64; forward-over-reverse along a bias tangent (the tangent of the weight gradients) against fp64 autograd; and the
    forward-mode LSLR hypergradient of the reference's second-order loop (task 0) against reverse mode."""
    a, state, batch = ln_case(case)
    m = fc.model(a, state, cuda_device)
    net = m.classifier
    named = dict(m.named_parameters())
    x, y = fc.images(batch, "support")
    forced = point(case, m, a, state, x, cuda_device)
    inner, bns = O.inner_param_names(a), bias_names(a)
    gen = torch.Generator().manual_seed(9)
    t = {n: torch.randn(state[n].shape, generator=gen, dtype=torch.float64) for n in inner + bns}
    xt = torch.randn(x.shape, generator=gen, dtype=torch.float64)
    fast, biases, x64 = leaves64(a, state, x)
    prim = ({n: v.detach() for n, v in fast.items()}, {n: v.detach() for n, v in biases.items()}, x64.detach())
    rows = []
    for direction in ("weights", "biases", "images", "all"):
        use = lambda kind: direction in (kind, "all")    # noqa: E731
        tan = ({n: t[n] if use("weights") else torch.zeros_like(t[n]) for n in inner},
               {n: t[n] if use("biases") else torch.zeros_like(t[n]) for n in bns},
               xt if use("images") else torch.zeros_like(xt))
        _, want = torch.func.jvp(lambda f, b, xx: ref_logits(a, xx, f, b, forced), prim, tan)
        with fwAD.dual_level():
            params = {}
            for n in inner + bns:
                p = named[n].detach().clone()
                params[n[len(PREFIX):]] = fwAD.make_dual(p, t[n].to(cuda_device, torch.float32)) \
                    if use("biases" if n in bns else "weights") else p
            xin = x.to(cuda_device)
            if use("images"):
                xin = fwAD.make_dual(xin, xt.to(cuda_device, torch.float32))
            got = fwAD.unpack_dual(net(xin, 0, params=params)).tangent
        check(rows, "J t along %s" % direction, got, want)
    # forward-over-reverse along a bias tangent: d/de grad_theta L(theta, b + e t_b) = grad_theta <grad_b L, t_b>
    gb = torch.autograd.grad(Fnn.cross_entropy(ref_logits(a, x64.detach(), fast, biases, forced), y),
                             list(biases.values()), create_graph=True)
    want = torch.autograd.grad(sum((g_ * t[n]).sum() for g_, n in zip(gb, bns)), list(fast.values()))
    with fwAD.dual_level():
        params = op_params(m, a)
        for n in bns:
            params[n[len(PREFIX):]] = fwAD.make_dual(named[n].detach().clone(), t[n].to(cuda_device, torch.float32))
        gr = torch.autograd.grad(Fnn.cross_entropy(net(x.to(cuda_device), 0, params=params), y.to(cuda_device)),
                                 [params[n[len(PREFIX):]] for n in inner], create_graph=True)
        got = [fwAD.unpack_dual(g_).tangent for g_ in gr]
    for n, g_, w_ in zip(inner, got, want):
        check(rows, "forward-over-reverse (bias tangent): %s" % n, g_, w_)
    # LSLR hypergradient of task 0's second-order loop: forward mode vs reverse mode
    xs_, ys_ = (v_.to(cuda_device) for v_ in fc.images(batch, "support"))
    xq, yq = (v_.to(cuda_device) for v_ in fc.images(batch, "target"))
    S = int(a.number_of_training_steps_per_iter)
    lslr_t = {n: torch.randn(S + 1, generator=gen).to(cuda_device) for n in inner}

    def loop(lr):
        fw = {n: named[n] for n in inner}
        for s in range(S):
            gs = torch.autograd.grad(Fnn.cross_entropy(net(xs_, s, params={n[len(PREFIX):]: fw[n] for n in inner}), ys_),
                                     [fw[n] for n in inner], create_graph=True)
            fw = {n: fw[n] - lr[n][s] * g_ for n, g_ in zip(inner, gs)}
        return Fnn.cross_entropy(net(xq, S - 1, params={n[len(PREFIX):]: fw[n] for n in inner}), yq)
    lr = {n: named[O.lslr_name(n)].detach().clone().requires_grad_(True) for n in inner}   # leaves (MAML: not learnable)
    rev = torch.autograd.grad(loop(lr), list(lr.values()))
    rev = float(sum((g_ * lslr_t[n]).sum() for g_, n in zip(rev, inner)))
    with fwAD.dual_level():
        fwd = float(fwAD.unpack_dual(loop({n: fwAD.make_dual(lr[n].detach(), lslr_t[n]) for n in inner})).tangent)
    e = abs(fwd - rev) / max(abs(rev), 1e-30)
    rows.append("%-64s rel %.2e%s" % ("LSLR hypergradient, forward vs reverse (%.6e)" % rev, e, "" if e <= B1_REL else
                                      "   <-- FAIL"))
    report(case, "forward mode", rows)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_per_task_entries_and_torch_func(case, cuda_device):
    """(6) On a layer-norm handle: stride 0 + summing mode reproduces net_forward / net_backward / net_hvp_image bit for
    bit; B distinct weight vectors and directions (bias directions included, per task) with per-task results match B
    n_tasks = 1 calls to 1e-5 of max-norm, each task's bias rows in its own result vector.  vmap forward and vmap(grad)
    (biases shared, their per-task gradients summed) against per-task operator calls; jacrev w.r.t. a bias vs fp64."""
    a, state, batch = ln_case(case)
    batch = fc.widen(batch)
    m = fc.model(a, state, cuda_device)
    net = m.classifier
    N, S = int(a.num_classes_per_set), int(a.number_of_training_steps_per_iter)
    xs_all, ys_all = batch[0], batch[2]
    B = xs_all.shape[0]
    x = xs_all.reshape(B, -1, *xs_all.shape[-3:]).float().to(cuda_device)
    y = ys_all.reshape(B, -1).long().to(cuda_device)
    n = x.shape[1]
    step = S - 1
    gen = torch.Generator().manual_seed(3)
    worst = {}

    def close(what, got, want, tol=1e-5):
        e = rel_err(got.cpu().double(), want.cpu().double())
        worst[what] = max(worst.get(what, 0.0), e)
        assert e <= tol, (what, e)

    # ---- the C ABI, on the support shape (forward / backward and hvp on one handle each)
    fwd, sec = ln_engine(a, n, B, cuda_device, False), ln_engine(a, n, B, cuda_device, True)
    meta = fc.meta_like(m, fwd, cuda_device)
    bias_segs = [i for i in net._norm_segments()[0]]
    dl = torch.randn(B, n, N, generator=gen).to(cuda_device)
    res = {k: torch.zeros(B, fwd.result_size, device=cuda_device) for k in ("old", "new", "tasks")}
    lg = {k: torch.zeros(B, n, N, device=cuda_device) for k in ("old", "new")}
    fwd.net_forward(B, step, meta, x, lg["old"])
    fwd.net_backward(B, step, meta, dl, res["old"][0])
    fwd.net_backward(B, step, meta, dl, res["new"][1])          # a second backward of the same forward: the same
    assert torch.equal(res["old"][0], res["new"][1])
    fwd.net_forward_tasks(B, step, meta, 0, x, lg["new"])
    fwd.net_backward_tasks(B, step, meta, 0, dl, res["new"][0], sum_tasks=True)
    assert torch.equal(lg["old"], lg["new"]) and torch.equal(res["old"][0], res["new"][0])
    metas = torch.stack([meta * (1.0 + 0.05 * b) for b in range(B)])
    for b in range(1, B):                                     # the biases are shared: every row carries task 0's
        for i in bias_segs:
            off, size = fwd.segments[i]
            metas[b, off:off + size] = metas[0, off:off + size]
    logits = torch.zeros(B, n, N, device=cuda_device)
    fwd.net_forward_tasks(B, step, metas, fwd.meta_size, x, logits)
    fwd.net_backward_tasks(B, step, metas, fwd.meta_size, dl, res["tasks"])
    singles = []
    for b in range(B):
        one_l = torch.zeros(1, n, N, device=cuda_device)
        one_g = torch.zeros(fwd.result_size, device=cuda_device)
        fwd.net_forward(1, step, metas[b].contiguous(), x[b:b + 1].contiguous(), one_l)
        fwd.net_backward(1, step, metas[b].contiguous(), dl[b:b + 1].contiguous(), one_g)
        close("logits", logits[b], one_l[0])
        close("grad", res["tasks"][b, :fwd.meta_size], one_g[:fwd.meta_size])
        singles.append(one_g)
    for i in bias_segs:                                       # task b's bias rows are task b's, not another task's
        off, size = fwd.segments[i]
        for b in range(B):
            close("bias rows", res["tasks"][b, off:off + size], singles[b][off:off + size])
            assert not torch.equal(res["tasks"][b, off:off + size], res["tasks"][(b + 1) % B, off:off + size])
    meta2 = fc.meta_like(m, sec, cuda_device)
    v = torch.randn(sec.meta_size, generator=gen).to(cuda_device)
    jv = {k: torch.zeros(B, n, N, device=cuda_device) for k in ("old", "new")}
    hv = {k: torch.zeros(B, sec.result_size, device=cuda_device) for k in ("old", "new", "tasks")}
    sec.net_hvp_image(B, step, meta2, x, None, dl, v, jv["old"], hv["old"][0])
    sec.net_hvp_image_tasks(B, step, meta2, 0, x, None, dl, v, 0, jv["new"], hv["new"][0], sum_tasks=True)
    assert torch.equal(jv["old"], jv["new"]) and torch.equal(hv["old"][0], hv["new"][0])
    metas2 = torch.stack([meta2 * (1.0 + 0.05 * b) for b in range(B)])
    for b in range(1, B):
        for i in bias_segs:
            off, size = sec.segments[i]
            metas2[b, off:off + size] = metas2[0, off:off + size]
    vs = torch.stack([v * (1.0 - 0.1 * b) for b in range(B)])    # per-task directions, the bias ones included
    jvt = torch.zeros(B, n, N, device=cuda_device)
    sec.net_hvp_image_tasks(B, step, metas2, sec.meta_size, x, None, dl, vs, sec.meta_size, jvt, hv["tasks"])
    for b in range(B):
        one_jv = torch.zeros(1, n, N, device=cuda_device)
        one_hv = torch.zeros(sec.result_size, device=cuda_device)
        sec.net_hvp_image(1, step, metas2[b].contiguous(), x[b:b + 1].contiguous(), None, dl[b:b + 1].contiguous(),
                          vs[b].contiguous(), one_jv, one_hv)
        close("jv", jvt[b], one_jv[0])
        close("hv", hv["tasks"][b, :sec.meta_size], one_hv[:sec.meta_size])

    # ---- torch.func: vmap forward, vmap(grad) against per-task operator calls
    named = dict(m.named_parameters())
    scale = 1.0 + 0.05 * torch.arange(B, dtype=torch.float32, device=cuda_device)
    per = {k[len(PREFIX):]: named[k].detach() * scale.view(-1, *[1] * named[k].dim()) for k in O.inner_param_names(a)}
    bia = {k[len(PREFIX):]: named[k].detach() for k in bias_names(a)}
    got = vmap(lambda xb, p: net(xb, step, params=p))(x, per)

    def loss(p, bp, xb, yb):
        return Fnn.cross_entropy(net(xb, step, params={**p, **bp}), yb)
    g_fast, g_b, g_x = vmap(grad(loss, argnums=(0, 1, 2)), in_dims=(0, None, 0, 0))(per, bia, x, y)
    for b in range(B):
        pb = {k: v_[b] for k, v_ in per.items()}
        close("vmap logits", got[b], net(x[b], step, params=pb).detach())
        one = grad(loss, argnums=(0, 1, 2))(pb, bia, x[b], y[b])
        for k in pb:
            close("vmap(grad) weights", g_fast[k][b], one[0][k])
        for k in bia:
            close("vmap(grad) biases", g_b[k][b], one[1][k])
        close("vmap(grad) x", g_x[b], one[2])
    print("\n[%s per-task entries and torch.func, B = %d] worst rel %s" %
          (case, B, " ".join("%s %.2e" % kv for kv in worst.items())))
    if case not in LN_CASES:
        return
    # jacrev of task 0's logits w.r.t. the last block's layer-norm bias (fixture shapes: the fp64 Jacobian is small)
    k = bias_names(a)[-1][len(PREFIX):]
    x0 = x[0]
    xs0, _ = fc.images(batch, "support")
    forced = point(case + " jacrev", m, a, state, xs0, cuda_device)
    J = jacrev(lambda bb: net(x0, 0, params={k: bb}))(bia[k])
    st64 = {kk: t_.double() for kk, t_ in state.items()}
    J64 = jacrev(lambda bb: ref_logits(a, xs0.double(), {nn: st64[nn] for nn in O.inner_param_names(a)},
                                       {**{nn: st64[nn] for nn in bias_names(a)}, PREFIX + k: bb}, forced))(st64[PREFIX + k])
    close("jacrev bias (vs fp64)", J, J64, B1_REL)
    print("[%s] jacrev w.r.t. %s vs fp64: rel %.2e" % (case, k, worst["jacrev bias (vs fp64)"]))


# ---- (7) the reference's second-order loop and the functorch loop on the operator ------------------------------------
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


_ENGINE_CALLS = ("net_forward", "net_backward", "net_hvp", "net_hvp_image", "net_jvp", "net_forward_tasks",
                 "net_backward_tasks", "net_hvp_image_tasks", "net_input_grad", "net_hvp_input_grad", "net_running_update")


def _record_calls(monkeypatch, calls):
    from howtotrainyourmamlpytorch_b200 import _native
    for name in _ENGINE_CALLS:
        orig = getattr(_native.Engine, name)
        monkeypatch.setattr(_native.Engine, name,
                            lambda self, n_tasks, *rest, _o=orig, _n=name, **kw: (calls.append((_n, n_tasks)),
                                                                                   _o(self, n_tasks, *rest, **kw))[1])


@pytest.mark.gpu
@pytest.mark.parametrize("loop", ["reference", "functorch"])
@pytest.mark.parametrize("case", LN_CASES)
def test_maml_loops_on_operator_match_goldens(case, loop, cuda_device, monkeypatch):
    """(7) The reference's training loop (second order where the config says so) and the functorch loop (vmap over the
    meta-batch: every engine call at n_tasks = B) on the operator: loss, last-step logits and every outer gradient (the
    layer-norm biases and LSLR included) against the unmodified reference's goldens (test_layer_norm's policy) and the
    meta-gradient against run_train_iter's fused iteration on the same model and batch."""
    g = load_golden(case)
    a, state = g.args, g.state()
    m = fc.model(a, state, cuda_device)
    batch, epoch = g.batch(0), g.iters[0][0]
    B = batch[0].shape[0]
    calls = []
    _record_calls(monkeypatch, calls)
    loss, logits = (_reference_loop if loop == "reference" else _functorch_loop)(m, a, batch, epoch, cuda_device)
    named = dict(m.named_parameters())
    names = LN.trainable_names(a)
    gr = torch.autograd.grad(loss, [named[n] for n in names], allow_unused=True)
    monkeypatch.undo()
    grads = {n: (g_ if g_ is not None else torch.zeros_like(named[n])).detach().cpu() for n, g_ in zip(names, gr)}
    if loop == "functorch":
        assert calls and all(t == B for _, t in calls), sorted(set(calls))
    ref32, ref64 = g.scalar("loss"), g.scalar("loss64")
    assert abs(float(loss.detach()) - ref64) <= max(3 * abs(ref32 - ref64), 2e-5 * abs(ref64))
    ref_logits = torch.from_numpy(g.array("logits"))
    assert float((logits - ref_logits).abs().max()) <= 1e-3 * float(ref_logits.abs().max())
    _, _, fused = fc.model(a, state, cuda_device).meta_gradient(batch, epoch)
    g32, g64 = g.grads(0, ""), g.grads(0, "64")
    rows, bad = [], []
    for n in g64:
        tol = _golden_tol(g32[n], g64[n])
        err = float((grads[n].double() - g64[n].double()).abs().max())
        err_fused = float((grads[n].double() - fused[n].cpu().double()).abs().max())
        rows.append("%-70s err %.2e  vs fused %.2e  tol %.2e" % (n, err, err_fused, tol))
        if err > tol or err_fused > tol:
            bad.append(n)
    print("\n[%s %s loop on the operator]\n   " % (case, loop) + "\n   ".join(rows))
    assert not bad, bad


@pytest.mark.gpu
def test_refusals(cuda_device, monkeypatch):
    """(8) Refused before any engine launch: a layer-norm bias batched under vmap, a frozen weight that is not all ones (in
    params or in the module), nested vmap.  Refused too: torch.func.jvp, third order (w.r.t. a bias), a cotangent on the
    image gradient."""
    a, state, batch = ln_case("ln_tiny_pp")
    m = fc.model(a, state, cuda_device)
    net = m.classifier
    named = dict(m.named_parameters())
    x, y = fc.images(batch, "support")
    x, y = x.to(cuda_device), y.to(cuda_device)
    fast = {n[len(PREFIX):]: named[n].detach() for n in O.inner_param_names(a)}
    k = bias_names(a)[1][len(PREFIX):]
    w = "layer_dict.conv1.norm_layer.weight"
    calls = []
    _record_calls(monkeypatch, calls)
    with pytest.raises(NotImplementedError, match="layer-norm bias batched"):
        vmap(lambda bb: net(x, 0, params={**fast, k: bb}))(named[PREFIX + k].detach().unsqueeze(0).expand(3, -1, -1, -1))
    with pytest.raises(ValueError, match="conv1.norm_layer.weight is not all ones"):
        net(x, 0, params={**fast, w: torch.full_like(named[PREFIX + w], 2.0)})
    with pytest.raises(NotImplementedError, match="nested"):
        vmap(vmap(lambda xx: net(xx, 0, params=fast)))(x.unsqueeze(0).unsqueeze(0).expand(2, 2, *x.shape))
    assert calls == [], calls
    with torch.no_grad():
        named[PREFIX + w].fill_(2.0)
    with pytest.raises(ValueError, match="conv1.norm_layer.weight is not all ones"):
        net(x, 0, params=fast)
    assert calls == [], calls
    with torch.no_grad():
        named[PREFIX + w].fill_(1.0)
    monkeypatch.undo()
    kw = "layer_dict.conv0.conv.weight"
    with pytest.raises(NotImplementedError, match="jvp"):
        torch.func.jvp(lambda ww: net(x, 0, params={**fast, kw: ww}), (fast[kw],), (torch.ones_like(fast[kw]),))

    def loss(bb):
        return Fnn.cross_entropy(net(x, 0, params={**fast, k: bb}), y)
    b0 = named[PREFIX + k].detach().clone()
    with pytest.raises(NotImplementedError, match="third"):
        grad(lambda bb: grad(lambda u: grad(loss)(u).pow(2).sum())(bb).sum())(b0)
    xr = x.clone().requires_grad_(True)
    gx, = torch.autograd.grad(Fnn.cross_entropy(net(xr, 0, params=fast), y), xr, create_graph=True)
    with pytest.raises(NotImplementedError, match="images"):
        torch.autograd.grad(gx.pow(2).sum(), xr)
