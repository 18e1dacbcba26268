"""The layer-norm network (``norm_layer: "layer_norm"``, reference MetaLayerNormLayer) on the fused training and
validation iteration, against golden vectors of the unmodified reference (``oracle/gen_golden_ln.py``) and the fp64
oracles (``oracle/ln_oracle.py``: autograd, and the autograd-free restatement of the kernels' formulas).  CPU tests: both
oracles reproduce each fixture's fp64 reference run, the module's state_dict / Adam order match the reference's, the
refusals, and the grid regime each full-size case exists for.  GPU tests: every stage of the iteration against the
autograd-free oracle, decision-forced parity, the iteration against the goldens (meta-gradient, validation leg, post-Adam
state), tensor cores against FFMA, rank r of G, the kernels each handle launches, and non-transductivity.

Besides the fixtures, two kinds of case have no fixture of their own:
  * ``<case>_ln``: every envelope and moved-state fixture of the BatchNorm network (``gen_golden.ENVELOPE_CASES`` and
    ``MOVED_CASES``) run with layer norm: the fixture's args with ``norm_layer="layer_norm"``, its batch and epoch, and the
    module's own initialisation moved by ``ln_oracle.moved_state`` (as ``test_functional_layer_norm`` does);
  * ``FULL``: seeded full-size cases on the benchmark's configs.  There the layer-norm kernels run on a capped grid
    (several pooling windows per thread, many CTAs adding to each image's fp64 sums), down to one CTA per image.

Unlike BatchNorm, layer norm does not remove the conv bias (it subtracts one mean over F*h*w, not one per channel), so
the conv biases are live parameters here and are compared like every other tensor."""
import numpy as np
import pytest
import torch

import functional_cases as fc
from conftest import load_golden
from engine_layout import (check_norm_path, device_sms, flat_to_nchw, geometry, gpu_decisions, grid_to_nchw,
                           host_plan, norm_grid_regimes, rel_err, theta_to_ref, traced_kernel_ids)
from oracle import ln_oracle as LN
from oracle import maml_oracle as O

LN_CASES = ["ln_tiny_pp", "ln_tiny_pp_moved", "ln_tiny_maml", "ln_nonsquare_odd", "ln_bern", "ln_eight_moved",
            "ln_one_stage"]
ENV = [n + "_ln" for n in fc.ENVELOPE]
MOVED_SEED = 11

# seeded full-size cases: name -> (config, tasks, ln_oracle.moved_state seed or None, the ln_grid regime it exists for)
FULL = {
    "ln_full_omniglot_mamlpp_5w1s": ("omniglot_mamlpp_5w1s", 16, None, "ln_capped"),
    "ln_full_mini_imagenet_mamlpp_5w1s": ("mini_imagenet_mamlpp_5w1s", 2, MOVED_SEED, "ln_capped"),
    "ln_full_mini_imagenet_mamlpp_5w5s": ("mini_imagenet_mamlpp_5w5s", 1, MOVED_SEED, "ln_capped"),
    # 100 support images x 3 tasks > 4 * 132: one CTA per image
    "ln_full_omniglot_mamlpp_20w5s": ("omniglot_mamlpp_20w5s", 3, MOVED_SEED, "ln_one_cta"),
}
STAGE_CASES = LN_CASES + ENV + list(FULL)
# Stage tolerances widened by a factor, each from a measurement on an H100 (700 W): the worst stage error as a multiple of
# the base tolerance.
#   env_maml_shared_bn_ln: plain MAML at F = 48 from a moved state, four inner steps and one target pass at the last.
#     Measured 1.20: task 1's target-pass gradient at the last step is 3e-5 to 6e-5 of max-norm away on every tensor
#     alike, i.e. in the loss gradient softmax - onehot itself, which cancels on a nearly fitted task.  The pinned
#     meta-gradient of the case agrees to 0.14 of its tolerance.
STAGE_SCALE = {"env_maml_shared_bn_ln": 2.0}


def _module_state(a):
    from howtotrainyourmamlpytorch_b200 import MAMLFewShotClassifier
    torch.manual_seed(0)
    m = MAMLFewShotClassifier(im_shape=(2, a.image_channels, a.image_height, a.image_width), device="cpu", args=a)
    return {k: v.detach().clone() for k, v in m.state_dict().items()}


class _Seeded(object):
    """A case without a fixture of its own: args, a state (the module's own initialisation, moved when a seed is given)
    and episodes -- a full-size case's seeded synthetic ones (Bernoulli images for Omniglot, N(0, 1) for Mini-ImageNet),
    or an envelope fixture's."""

    def __init__(self, argdict, iters, moved, batch=None):
        from howtotrainyourmamlpytorch_b200.utils.parser_utils import args_from_json
        self.argdict = dict(argdict, norm_layer="layer_norm")
        self.args = args_from_json(None, **self.argdict)
        self.iters = iters
        self._state = _module_state(self.args)
        if moved is not None:
            self._state = LN.moved_state(self._state, self.args, moved)
        self._batch = batch

    def state(self, dtype=torch.float32):
        return {k: v.detach().clone().to(dtype) for k, v in self._state.items()}

    def batch(self, it=0):
        return self._batch if self._batch is not None else O.synthetic_batch(self.args, iteration=self.iters[it][1])


def _case(case):
    from howtotrainyourmamlpytorch_b200.configs import CONFIGS
    if case in FULL:
        config, tasks, moved, _ = FULL[case]
        return _Seeded(dict(CONFIGS[config], batch_size=tasks), [(0, 0)], moved)
    if case in ENV:
        g = load_golden(case[:-len("_ln")])
        return _Seeded(g.argdict, g.iters[:1], MOVED_SEED, g.batch(0))
    return load_golden(case)


def _tol(g32, g64, rel=2e-5):
    """Golden tolerance of one tensor: 3x the reference's own fp32-vs-fp64 distance, at least `rel` of its max-norm."""
    own = float((g32.double() - g64.double()).abs().max())
    return max(3 * own, rel * float(g64.abs().max()) + 1e-7)


def _model(g, device, **debug):
    from howtotrainyourmamlpytorch_b200 import MAMLFewShotClassifier
    a = g.args
    m = MAMLFewShotClassifier(im_shape=(2, a.image_channels, a.image_height, a.image_width), device=device, args=a)
    for k, v in debug.items():
        setattr(m, k, v)
    m.load_state_dict(g.state())
    return m


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("oracle", ["autograd", "manual"])
@pytest.mark.parametrize("case", LN_CASES)
def test_oracle_reproduces_fp64_reference(case, oracle):
    g = load_golden(case)
    state = {k: v.double() for k, v in g.state(torch.float64).items()}
    fn = LN.autograd_train_iter if oracle == "autograd" else LN.manual_train_iter
    res = fn(state, g.args, g.batch(0), g.iters[0][0])
    assert abs(float(res["loss"]) - g.scalar("loss64")) <= 1e-12 * abs(g.scalar("loss64"))
    ref = g.grads(0, "64")
    assert list(res["grads"].keys()) == list(ref.keys())
    for n, got in res["grads"].items():
        assert float((got - ref[n].double()).abs().max()) <= 1e-12 * max(float(ref[n].abs().max()), 1e-30), n


@pytest.mark.parametrize("case", LN_CASES)
def test_state_dict_and_adam_order_match_the_reference(case):
    g = load_golden(case)
    m = _model(g, "cpu")
    sd = m.state_dict()
    ref = g.state()
    assert list(sd.keys()) == list(ref.keys()) == LN.state_keys(g.args)
    for k in ref:
        assert tuple(sd[k].shape) == tuple(ref[k].shape), k
        assert torch.equal(sd[k], ref[k]), k
    # Adam sees the trainable parameters only, in the reference's order; the frozen weight is not one of them
    assert [n for n, _ in m._trainable_param_list()] == LN.trainable_names(g.args) == list(g.grads(0).keys())
    assert [n for n in m._order if "inner_loop" not in n] == \
        [n for n in LN.trainable_names(g.args) if "inner_loop" not in n]
    group = m.optimizer.state_dict()["param_groups"][0]
    assert group["params"] == list(range(len(LN.trainable_names(g.args))))
    for l in range(int(g.args.num_stages)):
        w = dict(m.named_parameters())["classifier.layer_dict.conv%d.norm_layer.weight" % l]
        assert not w.requires_grad and bool(torch.all(w == 1))


def test_refusals():
    from howtotrainyourmamlpytorch_b200 import MAMLFewShotClassifier
    from howtotrainyourmamlpytorch_b200.utils.parser_utils import args_from_json
    g = load_golden("ln_tiny_pp")
    a = g.args
    m = MAMLFewShotClassifier(im_shape=(2, a.image_channels, a.image_height, a.image_width), device="cpu", args=a)
    x = torch.zeros(a.num_classes_per_set, a.image_channels, a.image_height, a.image_width)
    with pytest.raises(NotImplementedError, match="layer-norm"):
        m.classifier(x, 0)
    d = dict(g.argdict, enable_inner_loop_optimizable_bn_params=True)
    with pytest.raises(NotImplementedError, match="layer_norm"):
        MAMLFewShotClassifier(im_shape=(2, a.image_channels, a.image_height, a.image_width), device="cpu",
                              args=args_from_json(None, **d))
    m.classifier._check_layer_norm_weights()           # all ones: accepted
    sd = m.state_dict()
    sd["classifier.layer_dict.conv1.norm_layer.weight"] = torch.full_like(sd["classifier.layer_dict.conv1.norm_layer.weight"], 2.0)
    m.load_state_dict(sd)
    with pytest.raises(ValueError, match="conv1.norm_layer.weight is not all ones"):
        m.classifier._check_layer_norm_weights()


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", LN_CASES)
def test_golden_reference_parity(case, cuda_device):
    """Loss, logits, accuracy and every outer gradient (the layer-norm biases included) vs the unmodified reference."""
    g = load_golden(case)
    m = _model(g, cuda_device)
    losses, preds, grads = m.meta_gradient(g.batch(0), g.iters[0][0])
    ref32, ref64 = g.scalar("loss"), g.scalar("loss64")
    assert abs(float(losses["loss"]) - ref64) <= max(3 * abs(ref32 - ref64), 2e-5 * abs(ref64))
    ref_logits = torch.from_numpy(g.array("logits"))
    assert float((torch.from_numpy(np.stack(preds)) - ref_logits).abs().max()) <= 1e-3 * float(ref_logits.abs().max())
    assert abs(losses["accuracy"] - g.scalar("accuracy")) <= 1e-6
    g32, g64 = g.grads(0, ""), g.grads(0, "64")
    assert set(grads) >= set(g64)
    bad = []
    for n in g64:
        got = grads[n].cpu().double()
        err = float((got - g64[n].double()).abs().max())
        tol = _tol(g32[n], g64[n])
        print("%-70s err %.2e tol %.2e" % (n, err, tol))
        if err > tol:
            bad.append((n, err, tol))
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("case", LN_CASES)
def test_validation_iter(case, cuda_device):
    """run_validation_iter against the reference's: loss, accuracy, logits; nothing in the state changes (layer norm has
    no running statistics)."""
    g = load_golden(case)
    m = _model(g, cuda_device)
    m.current_epoch = g.iters[0][0]
    before = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    losses, preds = m.run_validation_iter(g.batch(0))
    ref_loss = float(g.val("loss"))
    assert abs(float(losses["loss"]) - ref_loss) <= 2e-5 * abs(ref_loss)
    ref_logits = torch.from_numpy(g.val("logits"))
    assert float((torch.from_numpy(np.stack(preds)) - ref_logits).abs().max()) <= 2e-4 * float(ref_logits.abs().max())
    assert abs(float(losses["accuracy"]) - float(g.val("accuracy"))) <= 1e-6
    for k, v in m.state_dict().items():
        assert torch.equal(before[k], v.detach().cpu()), k


@pytest.mark.gpu
@pytest.mark.parametrize("case", LN_CASES)
def test_train_iterations_post_state(case, cuda_device):
    """run_train_iter (fwd/bwd, clamp + Adam) over the recorded iterations: the post-step state_dict must match."""
    g = load_golden(case)
    m = _model(g, cuda_device)
    for it, (epoch, _) in enumerate(g.iters):
        losses, _ = m.run_train_iter(g.batch(it), epoch)
        assert abs(float(losses["loss"]) - g.scalar("loss", it)) <= 1e-4 * abs(g.scalar("loss", it))
        post = g.post(it)
        sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
        assert list(sd.keys()) == list(post.keys())
        for k in post:
            # Adam's first steps move every weight by ~lr * g / (|g| + 1e-8): an element whose gradient is at noise level
            # may move differently; everything else must agree
            diff = (sd[k] - post[k]).abs()
            assert float((diff > 2e-5).float().mean()) <= 2e-3 and float(diff.max()) <= 2.5e-3, (it, k, float(diff.max()))


@pytest.mark.gpu
@pytest.mark.parametrize("case", LN_CASES + [c for c in ENV if host_plan(load_golden(c[:-len("_ln")]).args, 1)["tc"]])
def test_tensor_core_convs_match_fp32_ffma_convs(case, cuda_device):
    """The wgmma 3xTF32 path against the exact-fp32 FFMA kernels (`reserved` bit 1) on a layer-norm handle: every
    intermediate of the first support pass and its gradient g[0] to 2e-5 of max-norm (the envelope cases' policy), and on
    the fixtures the whole meta-gradient within 3x the reference's own fp32-vs-fp64 distance of each tensor (floor 2e-5):
    ln_tiny_pp at epoch 0 runs its inner loop far out (that distance is 4e-2 of max-norm there), elsewhere it is about
    1e-6."""
    g = _case(case)
    g32, g64 = (g.grads(0, ""), g.grads(0, "64")) if case in LN_CASES else ({}, {})
    outs = []
    for force in (False, True):
        m = _model(g, cuda_device, _debug_force_fp32_convs=force)
        _, _, grads = m.meta_gradient(g.batch(0), g.iters[0][0])
        eng = m._engine
        taps = {"g0": torch.from_numpy(eng.debug_read("g", 0, 0, 0))}
        for l in range(int(g.args.num_stages)):
            taps["zh%d" % l] = torch.from_numpy(eng.debug_read("sup_zh", 0, 0, l))
            taps["dz%d" % l] = torch.from_numpy(eng.debug_read("sup_dz", 0, 0, l))
        taps.update({n: v.cpu() for n, v in grads.items() if n in g64})
        outs.append(taps)
    for k in outs[0]:
        tol = 2e-5
        if k in g64:
            tol = max(tol, 3 * rel_err(g32[k].double(), g64[k].double()))
        assert rel_err(outs[0][k], outs[1][k]) <= tol, (k, rel_err(outs[0][k], outs[1][k]))


@pytest.mark.gpu
@pytest.mark.parametrize("case,G", [("ln_tiny_pp", 3), ("ln_tiny_pp_moved", 3), ("env_many_tasks_ln", 4)])
def test_engine_as_rank_r_of_G_sums_to_single_call(case, G, cuda_device):
    """Rank r of G, one rank after the other on one GPU: the G result vectors sum to the single call's (the layer-norm
    bias segments included; the vector has no running-statistics part)."""
    g = _case(case)
    batch, epoch = g.batch(0), g.iters[0][0]
    B = batch[0].shape[0]
    Bl = B // G
    m = _model(g, cuda_device)
    m.meta_gradient(batch, epoch)
    full = m._result.detach().double().cpu().clone()
    assert full.numel() == m._engine.meta_size + 2
    acc = torch.zeros_like(full)
    for r in range(G):
        mr = _model(g, cuda_device)
        mr._ensure_engine(B)
        mr._shard_override = (r, G)
        mr.meta_gradient(tuple(t[r * Bl:(r + 1) * Bl].contiguous() for t in batch), epoch)
        acc += mr._result.detach().double().cpu()
    for (off, size), name in zip(m._engine.segments, m._order):
        a, b = acc[off:off + size], full[off:off + size]
        assert float((a - b).abs().max()) <= 2e-6 * float(b.abs().max()) + 1e-9, name
    ms = m._engine.meta_size
    assert abs(float(acc[ms] - full[ms])) <= 1e-6 * abs(float(full[ms]))
    assert float(acc[ms + 1]) == float(full[ms + 1])


@pytest.mark.gpu
@pytest.mark.parametrize("case", ENV)
def test_path_reached(case, cuda_device):
    """The kernels one iteration launches (device trace): the layer-norm kernels, their tangent twins exactly when the
    epoch is second order, no BatchNorm or inner-loop BatchNorm kernel, and the convolutions of the host plan."""
    g = _case(case)
    batch, epoch = g.batch(0), g.iters[0][0]
    ids = traced_kernel_ids(_model(g, cuda_device), batch, epoch)
    plan = check_norm_path(ids, "ln", g.args, epoch, batch[0].shape[0])
    print("\n[%s] kernel ids %s, host plan %s" % (case, sorted(ids), plan))


@pytest.mark.parametrize("case", list(FULL))
def test_full_size_cases_reach_their_grid_regime(case):
    """ln_grid (kernels_bn.cu) restated on the GPU's SM count (an H100's 132 without one): each full-size case reaches
    the regime it is declared for, so a case whose shape drifts out of it fails here."""
    config, tasks, _, regime = FULL[case]
    from howtotrainyourmamlpytorch_b200.configs import CONFIGS
    from howtotrainyourmamlpytorch_b200.utils.parser_utils import args_from_json
    a = args_from_json(None, **dict(CONFIGS[config], batch_size=tasks, norm_layer="layer_norm"))
    reached = norm_grid_regimes(a, tasks, device_sms())
    assert regime in reached, (case, regime, sorted(reached))


def _query_logits(m, batch, change_others):
    xs, xt, ys, yt = (t.clone() for t in batch)
    if change_others:
        # every query image of the episode but the first one of each task is replaced
        flat = xt.view(xt.shape[0], -1, *xt.shape[-3:])
        flat[:, 1:] = torch.randn_like(flat[:, 1:]) * 3.0
    _, preds = m.run_validation_iter((xs, xt, ys, yt))
    return torch.from_numpy(np.stack(preds))[:, 0]


@pytest.mark.gpu
def test_layer_norm_is_not_transductive(cuda_device):
    """A query image's logits do not depend on the other query images of its episode with layer norm (per-image
    statistics: bit-identical), and do with BatchNorm (batch statistics) -- the reason to choose layer norm."""
    g = load_golden("ln_tiny_pp")
    torch.manual_seed(0)
    a = _query_logits(_model(g, cuda_device), g.batch(0), False)
    b = _query_logits(_model(g, cuda_device), g.batch(0), True)
    assert float((a - b).abs().max()) <= 1e-6 * float(a.abs().max()), float((a - b).abs().max())
    print("layer norm: max |change| of the first query's logits", float((a - b).abs().max()))
    gb = load_golden("tiny_pp")                 # the same shape with BatchNorm
    torch.manual_seed(0)
    a = _query_logits(_model(gb, cuda_device), gb.batch(0), False)
    b = _query_logits(_model(gb, cuda_device), gb.batch(0), True)
    assert float((a - b).abs().max()) > 1e-6 * float(a.abs().max())


# ------------------------------------------------------------------------------------------------ stages and decisions
def _decision_flips(intermediates):
    """(#decisions differing from fp64, worst fp64 margin at one) of a pinned run: leaky-ReLU branches and pooling
    arg-maxes."""
    import torch.nn.functional as Fnn
    n_flip, worst_margin = 0, 0.0
    for x in [i for i in intermediates if "theta" in i]:
        for f in list(x["sup_f"]) + [t[0] for t in x["tgt_f"] if t is not None]:
            for blk in f["blocks"]:
                y = blk["y"]
                flip = (y > 0) != (blk["slope"] > 0.5)
                if flip.any():
                    n_flip += int(flip.sum())
                    worst_margin = max(worst_margin, float(y[flip].abs().max()))
                act = y * O._slope(y)
                n_, c_ = act.shape[:2]
                gap = Fnn.max_pool2d(act, 2, 2) - act.view(n_, c_, -1).gather(2, blk["idx"].view(n_, c_, -1)).view(n_, c_, *blk["idx"].shape[2:])
                if (gap > 0).any():
                    n_flip += int((gap > 0).sum())
                    worst_margin = max(worst_margin, float(gap.max()))
    return n_flip, worst_margin


def _stage_report(a, eng, ref, B):
    """Every materialised intermediate of tasks 0 and B-1 against the pinned oracle's: (report rows, worst error as a
    multiple of its tolerance)."""
    geo, (ph, pw) = geometry(a)
    F = int(a.cnn_num_filters)
    N, K, T = int(a.num_classes_per_set), int(a.num_samples_per_class), int(a.num_target_samples)
    S, L = int(a.number_of_training_steps_per_iter), len(geo)
    rows, worst = [], 0.0

    def chk(name, got, want, tol):
        nonlocal worst
        e = rel_err(got, want)
        rows.append("%-44s %.2e%s" % (name, e, "" if e <= tol else "   <-- FAIL"))
        worst = max(worst, e / tol)

    def chk_vec(tag, vec, want, tol=5e-5):
        got = theta_to_ref(vec, a)
        for n, v in want.items():
            chk("%s %s" % (tag, n[-26:]), got[n], v, 2e-4 if n == O.LIN_B and tol > 1e-5 else tol)

    for t in sorted({0, B - 1}):
        inter = [x for x in ref["intermediates"] if "theta" in x and x["task"] == t][0]
        tan0 = [x for x in ref["intermediates"] if x.get("step") == 0 and x["task"] == t]
        for s in range(S):
            chk_vec("t%d theta[%d]" % (t, s), eng.debug_read("theta", t, s, 0), inter["theta"][s], tol=1e-5)
            for l in range(L):
                gl = geo[l]
                chk("t%d sup zh   s%d l%d" % (t, s, l), grid_to_nchw(eng.debug_read("sup_zh", t, s, l), N * K, gl["h"], gl["w"], F),
                    inter["sup_f"][s]["blocks"][l]["zh"], 2e-5)
                p = (grid_to_nchw(eng.debug_read("sup_ain", t, s, l + 1), N * K, gl["h"] // 2, gl["w"] // 2, F) if l + 1 < L
                     else flat_to_nchw(eng.debug_read("sup_ain", t, s, L), N * K, ph, pw, F))
                chk("t%d sup pool s%d l%d" % (t, s, l), p, inter["sup_f"][s]["blocks"][l]["p"], 2e-5)
                dp = (grid_to_nchw(eng.debug_read("sup_dp", t, s, l), N * K, gl["h"] // 2, gl["w"] // 2, F) if l + 1 < L
                      else flat_to_nchw(eng.debug_read("sup_dp", t, s, l), N * K, ph, pw, F))
                chk("t%d sup dp   s%d l%d" % (t, s, l), dp, inter["sup_b"][s]["blocks"][l]["dp"], 5e-5)
                chk("t%d sup dz   s%d l%d" % (t, s, l), grid_to_nchw(eng.debug_read("sup_dz", t, s, l), N * K, gl["h"], gl["w"], F),
                    inter["sup_b"][s]["blocks"][l]["dz"], 5e-5)
            chk_vec("t%d g[%d]" % (t, s), eng.debug_read("g", t, s, 0), inter["sup_g"][s])
            if inter["tgt_f"][s] is not None:
                for l in range(L):
                    gl = geo[l]
                    chk("t%d tgt zh   s%d l%d" % (t, s, l),
                        grid_to_nchw(eng.debug_read("tgt_zh", t, s, l), N * T, gl["h"], gl["w"], F),
                        inter["tgt_f"][s][0]["blocks"][l]["zh"], 2e-5)
                    chk("t%d tgt dz   s%d l%d" % (t, s, l),
                        grid_to_nchw(eng.debug_read("tgt_dz", t, s, l), N * T, gl["h"], gl["w"], F),
                        inter["tgt_b"][s]["blocks"][l]["dz"], 5e-5)
                chk_vec("t%d tgrad[%d]" % (t, s), eng.debug_read("tgrad", t, s, 0), inter["tgt_g"][s])
        chk_vec("t%d tbar" % t, eng.debug_read("tbar", t, 0, 0), inter["tbar"])
        if tan0:
            chk_vec("t%d u[0]" % t, eng.debug_read("u", t, 0, 0), tan0[0]["u"])
            for l in range(L):
                gl = geo[l]
                chk("t%d tan zh-dot l%d" % (t, l), grid_to_nchw(eng.debug_read("tan_zh", t, 0, l), N * K, gl["h"], gl["w"], F),
                    tan0[0]["tangent"]["fwd"][l]["zh_dot"], 5e-5)
                chk("t%d tan dz-dot l%d" % (t, l), grid_to_nchw(eng.debug_read("tan_dz", t, 0, l), N * K, gl["h"], gl["w"], F),
                    tan0[0]["tangent"]["bwd"][l]["dz_dot"], 5e-5)
    return rows, worst


_RUNS = {}


def _forced_run(case, device):
    """One GPU iteration (every target pass kept) and one fp64 autograd-free oracle run with the GPU's decisions pinned
    per case, shared by the stage-wise and the decision-forced test.  Kept as what those tests compare (the stage-wise
    report, the decision statistics, loss, logits and meta-gradients), not as the runs' intermediates: at full size those
    take gigabytes."""
    if case not in _RUNS:
        g = _case(case)
        m = _model(g, device, _debug_keep_target_passes=True)
        batch, epoch = g.batch(0), g.iters[0][0]
        losses, preds, grads = m.meta_gradient(batch, epoch)
        dec = gpu_decisions(m, g.args, batch, epoch)
        ref = LN.manual_train_iter(g.state(torch.float64), g.args, batch, epoch, decisions=dec, keep_intermediates=True)
        rows, worst = _stage_report(g.args, m._engine, ref, batch[0].shape[0])
        _RUNS[case] = dict(rows=rows, worst=worst, flips=_decision_flips(ref["intermediates"]), loss=float(losses["loss"]),
                           logits=np.stack(preds), grads={n: v.detach().cpu() for n, v in grads.items()},
                           ref_loss=float(ref["loss"]), ref_grads=ref["grads"], ref_logits=ref["logits"])
        del m, ref, dec
    return _RUNS[case]


@pytest.mark.gpu
@pytest.mark.parametrize("case", STAGE_CASES)
def test_stagewise_against_oracle(case, cuda_device):
    """Every materialised intermediate of tasks 0 and B-1 against the fp64 autograd-free oracle with the GPU's decisions
    pinned (so near-ties cannot move the comparison): theta^s, every support pass (zh, pooled output, dp, dz) and its
    gradient, every target pass (zh, dz) and tgrad[s], theta-bar and u after the reverse sweep, and step 0's tangent pass
    (zh-dot, dz-dot of every block)."""
    run = _forced_run(case, cuda_device)
    print("\n[%s stagewise] worst %.2f x tolerance\n   " % (case, run["worst"]) + "\n   ".join(run["rows"]))
    assert run["worst"] <= STAGE_SCALE.get(case, 1.0), "stage mismatch (see report above): worst = %.2f x tolerance" % run["worst"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", STAGE_CASES)
def test_decision_forced_parity(case, cuda_device):
    """(1) Every discrete decision the GPU took (leaky-ReLU branch, pooling arg-max) is consistent with fp64 arithmetic
    except at margins below 1e-4; (2) with those decisions pinned the fp64 oracle's loss, logits and every meta-gradient
    tensor (layer-norm biases and conv biases included) agree with the GPU's to 1e-4 of the tensor's max-norm.  Mini-ImageNet
    5-way 5-shot takes the bounds test_gpu_parity sets for that shape (its inner loop amplifies fp32 rounding): margins
    below 1e-3, 3e-4 of max-norm (3e-3 on the LSLR rates)."""
    run = _forced_run(case, cuda_device)
    n_flip, worst_margin = run["flips"]
    wide = case in FULL and FULL[case][0] == "mini_imagenet_mamlpp_5w5s"
    print("\n[%s] decisions differing from fp64: %d, worst fp64 margin at one: %.2e" % (case, n_flip, worst_margin))
    assert worst_margin <= (1e-3 if wide else 1e-4), worst_margin
    assert abs(run["loss"] - run["ref_loss"]) <= 1e-5 * abs(run["ref_loss"])
    bad, worst = [], 0.0
    for n, v in run["ref_grads"].items():
        err = float((run["grads"][n].double() - v).abs().max())
        scale = max(float(v.abs().max()), 1e-30)
        rel = (3e-3 if "names_learning_rates" in n else 3e-4) if wide else 1e-4
        worst = max(worst, err / (rel * scale + 1e-7))
        print("%-70s err %.2e (%.1e of max)" % (n, err, err / scale))
        if err > rel * scale + 1e-7:
            bad.append((n, err, scale))
    print("[%s] worst meta-gradient error: %.2f x tolerance" % (case, worst))
    assert not bad, bad
    got_logits = torch.from_numpy(run["logits"]).double()
    assert float((got_logits - run["ref_logits"]).abs().max()) <= 1e-4 * float(run["ref_logits"].abs().max())
