"""The engine across the configurations ``maml_b200_create`` admits (filters 16..64, 1..4 stages, 1..8 inner steps,
1..4 input channels, 2..32 ways, batches of up to 128 images, any H x W that survives the halvings).

Every envelope case (``oracle/gen_golden.py`` ENVELOPE_CASES and, at moved states, MOVED_CASES; fixtures generated from
the unmodified reference) names the axis it exists for and the engine paths it has to reach.  Per case:
  * CPU: the fp64 oracle (autograd and manual) reproduces the reference's fp64 run to 1e-12, and the validation leg;
    on the moved-state cases, the fp64 oracle with a gamma / beta / alpha indexing bug lands far from the reference;
  * GPU: the path the handle takes (device trace of one iteration), every intermediate of task 0 (support and target
    passes at every inner step, the reverse sweep, step 0's tangent pass) against the fp64 oracle with the GPU's
    decisions pinned, the decision-forced meta-gradient, the direct golden comparison, the validation leg, the post-Adam
    state, the functional operator and tensor cores vs FFMA.
Tolerances are those of the tiny cases in test_gpu_parity.py / test_oracle_golden.py and of the functional-operator
tests (DESIGN.md section 6)."""
import json

import numpy as np
import pytest
import torch
import torch.nn.functional as Fnn

import functional_cases as fc
from conftest import load_golden, grad_tolerance
from engine_layout import (geometry, grid_to_nchw, flat_to_nchw, theta_to_ref, rel_err, gpu_decisions, host_plan,
                           traced_kernel_ids)
from oracle import maml_oracle as O

gpu = pytest.mark.gpu

# case -> (the axis it exists for, the engine paths it must reach).  Path keys:
#   tc:    blocks l >= 1 run the tensor-core convolution / weight gradient (else the FFMA kernels, or no such block)
#   tail:  the support pass runs the fused last block + head (tail_fused / tail_onchip) instead of head_kernel
#   ring:  depth of the tensor-core conv's B ring next to split-K 2 in tangent mode (only where it is the point)
#   chunks: weight-gradient chunks per block l >= 1 on an H100 (132 SMs) (only where it is the point)
ENVELOPE = {
    "env_nonsquare_odd": ("H != W, odd H at block 0, odd W at block 1", dict(tc=True, tail=True)),
    "env_tall_c2": ("C0 = 2, pooled 5 x 1, MSL between its extremes", dict(tc=True, tail=True)),
    "env_c4_two_stages": ("L = 2, C0 = 4 in the fused iteration", dict(tc=True, tail=False)),
    "env_one_stage": ("L = 1: first block = last block, no tensor-core block", dict(tc=False, tail=True)),
    "env_eight_steps": ("S = 8 = MAML_MAX_STEPS, MSL on", dict(tc=True, tail=True)),
    "env_one_step": ("S = 1, second order, one target slot", dict(tc=True, tail=True)),
    "env_way32": ("N*K = 128 (the cap), 32 head groups", dict(tc=True, tail=False)),
    "env_way17": ("17 support rows: head kernel", dict(tc=True, tail=False)),
    "env_way16": ("16 support rows: fused tail; 24 target rows", dict(tc=True, tail=True)),
    "env_way2": ("2-way 1-shot: last-block BatchNorm over 18 values", dict(tc=True, tail=True)),
    "env_ffma_wide": ("block 1 65 wide: the handle turns the tensor cores off", dict(tc=False, tail=True)),
    "env_ring_edge": ("block 1 62 wide: largest halo, ring depth 2", dict(tc=True, tail=False, ring=2)),
    "env_many_tasks": ("48 tasks: one weight-gradient chunk per block", dict(tc=True, tail=True, chunks=1)),
    "env_bern_nonsquare": ("Bernoulli images, exact ties next to the dropped row", dict(tc=True, tail=True)),
    "env_maml_shared_bn": ("plain MAML: shared BatchNorm, no LSLR, non-square, F = 48",
                           dict(tc=True, tail=False)),
    # moved states (oracle.maml_oracle.moved_state): per-step gamma / beta, per-(tensor, step) LSLR rates, nonzero biases
    "env_moved_pp": ("moved state: MAML++ second order, MSL between its extremes", dict(tc=True, tail=True)),
    "env_moved_first": ("moved state: first order, MSL off", dict(tc=True, tail=True)),
    "env_moved_maml": ("moved state: plain MAML, shared BatchNorm, head kernel", dict(tc=True, tail=False)),
    "env_moved_one_stage": ("moved state: L = 1, fused tail on block 0", dict(tc=False, tail=True)),
    "env_moved_ffma": ("moved state: block 1 65 wide, FFMA convolutions", dict(tc=False, tail=True)),
    "env_moved_eight": ("moved state: S = 8, the largest step and LSLR index space", dict(tc=True, tail=True)),
}
CASES = list(ENVELOPE)
MOVED = [c for c in CASES if c.startswith("env_moved_")]
BERNOULLI = ["env_bern_nonsquare"]
SWEEP_TOL = 5e-5       # reverse sweep and tangent pass taps, of max-norm (test_stagewise_with_gpu_decisions)

# kernel ids of the device trace (scripts/trace_kernel_ids.json)
K_CONV_ROWS, K_CONV0, K_WGRAD_ROW, K_WGRAD0 = 1, 2, 3, 4
K_HEAD, K_CONV_TC, K_TAIL, K_TAIL_TAN, K_TAIL_ONCHIP, K_WGRAD_TC = 14, 22, 23, 24, 25, 27


def _tasks(g):
    return int(g.batch(0)[0].shape[0])


def _model(g, device, keep_targets=False, force_fp32=False):
    from howtotrainyourmamlpytorch_b200 import MAMLFewShotClassifier
    a = g.args
    m = MAMLFewShotClassifier(im_shape=(2, a.image_channels, a.image_height, a.image_width), device=device, args=a)
    m._debug_keep_target_passes = keep_targets
    m._debug_force_fp32_convs = force_fp32
    m.load_state_dict(g.state())
    return m


def _dead(n):
    return "conv.bias" in n or "conv-bias" in n


# ----------------------------------------------------------------------------------------------------------------------
# CPU
# ----------------------------------------------------------------------------------------------------------------------
def test_case_table_matches_the_generator():
    """This module's list, the functional-operator tests' list (functional_cases.ENVELOPE) and the generator's tables name
    the same cases, and every fixture carries its case's args (and the moved-state cases their moved state)."""
    from oracle import gen_golden
    assert sorted(c for c in CASES if c not in MOVED) == sorted(gen_golden.ENVELOPE_CASES)
    assert sorted(MOVED) == sorted(gen_golden.MOVED_CASES)
    assert fc.ENVELOPE == list(gen_golden.ENVELOPE_CASES) + list(gen_golden.MOVED_CASES)
    assert sorted(fc.ENVELOPE) == sorted(CASES)
    for case in CASES:
        _, argdict, iters = gen_golden.make_args(case)
        g = load_golden(case)
        assert g.argdict == json.loads(json.dumps(argdict)), case
        assert [list(i) for i in iters] == g.iters, case
        assert g.kind == gen_golden.case_kind(case), case
        assert "it0/xs" in g.blob.files and g.blob["it0/grad64/" + O.LIN_W].dtype == np.float64, case
        moved = int(g.blob["moved"]) if "moved" in g.blob.files else None
        assert moved == gen_golden.case_moved(case) and (moved is not None) == (case in MOVED), case
        if moved is not None:
            init = O.init_state(g.args)
            want = O.moved_state(init, g.args, moved)
            st = g.state()
            assert list(st) == list(want), case
            for k in want:
                assert torch.equal(st[k], want[k]), (case, k)


def _mutants(state, args):
    """The moved state with one indexing bug each, as the engine would see it: gamma / beta of step 0 at every step
    (per-step BatchNorm only), alpha of step 0 at every step, alpha of the first tensor for every tensor, gamma = 1 and
    beta = 0."""
    out = {}
    bn = [k for k in state if k.endswith("norm_layer.weight") or k.endswith("norm_layer.bias")]
    lslr = [O.lslr_name(n) for n in O.inner_param_names(args)]
    if args.per_step_bn_statistics:
        out["gamma/beta of step 0"] = dict(state, **{k: state[k][:1].expand_as(state[k]).clone() for k in bn})
    out["alpha of step 0"] = dict(state, **{k: state[k][:1].expand_as(state[k]).clone() for k in lslr})
    out["alpha of tensor 0"] = dict(state, **{k: state[lslr[0]].clone() for k in lslr})
    out["gamma = 1, beta = 0"] = dict(state, **{k: (torch.ones_like(state[k]) if k.endswith("weight")
                                                   else torch.zeros_like(state[k])) for k in bn})
    return out


@pytest.mark.parametrize("case", MOVED)
def test_moved_state_tells_indexing_bugs_apart(case):
    """At a moved state, the fp64 oracle with any one of the indexing bugs above lands >= 1e-3 of max-norm away from the
    reference's fp64 meta-gradient on some live tensor (at the reference's initialisation the same bugs agree to ~1e-14):
    a regenerated fixture that drifts back to an uninformative state fails here."""
    g = load_golden(case)
    state, ref = g.state(torch.float64), g.grads(0, "64")
    rows = []
    for name, st in _mutants(state, g.args).items():
        res = O.autograd_train_iter(st, g.args, g.batch(0), g.iters[0][0])
        dist = max(float((res["grads"][n] - ref[n]).abs().max()) / float(ref[n].abs().max())
                   for n in ref if not _dead(n))
        rows.append((name, dist))
    print("\n[%s] mutant distance to the reference (of max-norm): %s" % (case, ", ".join("%s %.2e" % r for r in rows)))
    assert all(d >= 1e-3 for _, d in rows), rows


@pytest.mark.parametrize("case", CASES)
def test_host_rules_reach_the_declared_paths(case):
    """The host rules the handle applies put each case on the path it exists for (checked against the device trace on
    the GPU): a case whose shape drifts off its path fails here."""
    g = load_golden(case)
    plan = host_plan(g.args, _tasks(g))
    for k, want in ENVELOPE[case][1].items():
        assert plan[k] == want, (case, k, plan[k], want)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("impl", ["autograd", "manual"])
def test_envelope_fp64_exact(case, impl):
    """Both oracle restatements in fp64 reproduce the reference's fp64 loss and every outer gradient to 1e-12 of the
    tensor's max-norm (dead conv biases: 1e-12 of the largest live gradient, absolute)."""
    g = load_golden(case)
    fn = O.autograd_train_iter if impl == "autograd" else O.manual_train_iter
    res = fn(g.state(torch.float64), g.args, g.batch(0), g.iters[0][0])
    ref_loss = g.scalar("loss64")
    assert abs(float(res["loss"]) - ref_loss) <= 1e-12 * abs(ref_loss)
    ref = g.grads(0, "64")
    assert list(res["grads"].keys()) == list(ref.keys())
    live = max(float(v.abs().max()) for n, v in ref.items() if not _dead(n))
    for n, v in res["grads"].items():
        tol = 1e-12 * (live if _dead(n) else float(ref[n].abs().max()))
        err = float((v.double() - ref[n].double()).abs().max())
        assert err <= tol, (case, n, err, tol)


@pytest.mark.parametrize("case", CASES)
def test_envelope_validation_leg_matches_reference(case):
    """The oracle's evaluation pass (fp32, autograd restatement) against the reference's run_validation_iter: loss,
    logits, accuracy and the running statistics it leaves behind (same bounds as the tiny cases)."""
    g = load_golden(case)
    res = O.autograd_train_iter(g.state(), g.args, g.batch(0), g.iters[0][0], training_phase=False,
                                current_epoch=g.iters[0][0])
    ref_loss = float(g.val("loss"))
    assert abs(float(res["loss"]) - ref_loss) <= 2e-6 * abs(ref_loss)
    ref_logits = torch.from_numpy(g.val("logits"))
    assert float((res["logits"].float() - ref_logits).abs().max()) <= 1e-5 * float(ref_logits.abs().max())
    assert abs(res["accuracy"] - float(g.val("accuracy"))) < 1e-9
    post = g.val_post()
    assert set(post.keys()) == set(res["running"].keys())
    for k, v in res["running"].items():
        assert torch.allclose(v.float(), post[k], rtol=5e-5, atol=5e-6), k


# ----------------------------------------------------------------------------------------------------------------------
# GPU
# ----------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("case", CASES)
def test_path_reached(case, cuda_device):
    """The kernels one iteration actually launches (device trace) are those of the case's declared path."""
    g = load_golden(case)
    a = g.args
    batch, epoch = g.batch(0), g.iters[0][0]
    ids = traced_kernel_ids(_model(g, cuda_device), batch, epoch)
    want = ENVELOPE[case][1]
    plan = host_plan(a, _tasks(g), torch.cuda.get_device_properties(cuda_device).multi_processor_count)
    L = int(a.num_stages)
    print("\n[%s] %s: kernel ids %s, host plan %s" % (case, ENVELOPE[case][0], sorted(ids), plan))
    assert {K_CONV0, K_WGRAD0, K_HEAD} <= ids
    if want["tc"]:
        assert {K_CONV_TC, K_WGRAD_TC} <= ids and not ids & {K_CONV_ROWS, K_WGRAD_ROW}, sorted(ids)
    elif L > 1:
        assert {K_CONV_ROWS, K_WGRAD_ROW} <= ids and not ids & {K_CONV_TC, K_WGRAD_TC}, sorted(ids)
    else:
        assert not ids & {K_CONV_ROWS, K_WGRAD_ROW, K_CONV_TC, K_WGRAD_TC}, sorted(ids)
    second_order = bool(a.second_order) and epoch > a.first_order_to_second_order_epoch
    if want["tail"]:
        # support passes through tail_fused or tail_onchip, tangent passes through tail_tan_fused (second order only:
        # a first-order iteration runs no tangent pass)
        assert ids & {K_TAIL, K_TAIL_ONCHIP} and (K_TAIL_TAN in ids) == second_order, sorted(ids)
    else:
        assert not ids & {K_TAIL, K_TAIL_ONCHIP, K_TAIL_TAN}, sorted(ids)
    # the ring depth and the chunk count have no kernel id: the host rule stands in for them
    for k in ("ring", "chunks"):
        if k in want:
            assert plan[k] == want[k], (k, plan[k], want[k])


_RUNS = {}


def _decision_flips(intermediates):
    """(#decisions, #leaky-branch flips vs fp64, #arg-max flips vs fp64, worst fp64 margin at a flip) of a pinned run."""
    n_slope_flip, n_arg_flip, worst_margin, n_dec = 0, 0, 0.0, 0
    for x in [i for i in intermediates if "theta" in i]:
        for f in list(x["sup_f"]) + [t[0] for t in x["tgt_f"] if t is not None]:
            for blk in f["blocks"]:
                y = blk["y"]
                nat_pos = y > 0
                flip = nat_pos != (blk["slope"] > 0.5)
                n_dec += y.numel()
                if flip.any():
                    n_slope_flip += int(flip.sum())
                    worst_margin = max(worst_margin, float(y[flip].abs().max()))
                act = y * torch.where(nat_pos, torch.ones_like(y), torch.full_like(y, 0.01))
                pmax = Fnn.max_pool2d(act, 2, 2)
                n_, c_ = act.shape[:2]
                gap = pmax - act.view(n_, c_, -1).gather(2, blk["idx"].view(n_, c_, -1)).view(pmax.shape)
                if (gap > 0).any():
                    n_arg_flip += int((gap > 0).sum())
                    worst_margin = max(worst_margin, float(gap.max()))
    return n_dec, n_slope_flip, n_arg_flip, worst_margin


def _forced_run(case, device):
    """One meta_gradient with every target pass kept, the GPU's decisions, and the fp64 oracle with them pinned.  Kept
    per case for the stage-wise and the decision-forced test: the engine's task-0 taps (every support and target pass,
    every tgrad[s], u and theta-bar after the reverse sweep, the tangent pass of step 0), the oracle's task-0
    intermediates, the decision statistics and both results."""
    if case not in _RUNS:
        g = load_golden(case)
        a = g.args
        m = _model(g, device, keep_targets=True)
        batch, epoch = g.batch(0), g.iters[0][0]
        losses, preds, grads = m.meta_gradient(batch, epoch)
        dec = gpu_decisions(m, a, batch, epoch)
        ref = O.manual_train_iter(g.state(torch.float64), a, batch, epoch, decisions=dec, keep_intermediates=True)
        eng, L, S = m._engine, int(a.num_stages), int(a.number_of_training_steps_per_iter)
        sched = O.target_pass_schedule(a, epoch, True, S)
        taps = {}
        for s in range(S):
            taps[("theta", s, 0)] = eng.debug_read("theta", 0, s, 0)
            taps[("g", s, 0)] = eng.debug_read("g", 0, s, 0)
            passes = ("sup", "tgt") if sched[s] is not None else ("sup",)
            if sched[s] is not None:
                taps[("tgrad", s, 0)] = eng.debug_read("tgrad", 0, s, 0)
            for p in passes:
                for l in range(L):
                    for name in ("_zh", "_dp", "_dz"):
                        taps[(p + name, s, l)] = eng.debug_read(p + name, 0, s, l)
                    taps[(p + "_ain", s, l + 1)] = eng.debug_read(p + "_ain", 0, s, l + 1)
        taps[("u", 0, 0)] = eng.debug_read("u", 0, 0, 0)
        taps[("tbar", 0, 0)] = eng.debug_read("tbar", 0, 0, 0)
        for l in range(L):                          # the tangent pass buffers hold step 0's, the last one run
            for name in ("tan_zh", "tan_dp", "tan_dz"):
                taps[(name, 0, l)] = eng.debug_read(name, 0, 0, l)
            taps[("tan_ain", 0, l + 1)] = eng.debug_read("tan_ain", 0, 0, l + 1)
        tang0 = [x for x in ref["intermediates"] if "Hu" in x and x["task"] == 0 and x["step"] == 0]
        _RUNS[case] = dict(taps=taps, inter0=[x for x in ref["intermediates"] if "theta" in x and x["task"] == 0][0],
                           tang0=tang0[0] if tang0 else None, sched=sched,
                           flips=_decision_flips(ref["intermediates"]), loss=float(losses["loss"]),
                           logits=np.stack(preds), grads={n: t.detach().cpu() for n, t in grads.items()},
                           ref_loss=float(ref["loss"]), ref_grads=ref["grads"], ref_logits=ref["logits"])
        del m, ref, dec
    return _RUNS[case]


@gpu
@pytest.mark.parametrize("case", CASES)
def test_stagewise_with_gpu_decisions(case, cuda_device):
    """Every materialised intermediate of task 0 against the fp64 oracle with the GPU's decisions pinned: what locates a
    fault.  Phase A: theta, zh, pool, dp, dz and g of every block at every inner step, and the same of every target pass
    with its weighted gradient tgrad[s].  Phase B: u = alpha[.][0] * theta-bar and theta-bar after the sweep, H u of step
    0 (= u / alpha[.][0] - theta-bar), and the tangent pass of step 0 (zh-dot, p-dot, dz-dot, dp-dot).  Tolerances of
    test_stagewise_against_oracle for the passes; the reverse sweep's are set from measured errors (see below)."""
    g = load_golden(case)
    a = g.args
    run = _forced_run(case, cuda_device)
    taps, inter, tang0 = run["taps"], run["inter0"], run["tang0"]
    geo, (ph, pw) = geometry(a)
    F = int(a.cnn_num_filters)
    n_of = {"sup": int(a.num_classes_per_set) * int(a.num_samples_per_class),
            "tgt": int(a.num_classes_per_set) * int(a.num_target_samples)}
    S = int(a.number_of_training_steps_per_iter)
    L = len(geo)
    rows, worst, worst_name = [], 0.0, ""

    def chk(name, got, want, tol=1e-5, absolute=None):
        nonlocal worst, worst_name
        e = rel_err(got, want) if absolute is None else float((got.double() - want.double()).abs().max())
        r = e / (tol if absolute is None else absolute)
        rows.append("%-34s %.2e%s" % (name, e, "" if r <= 1.0 else "   <-- FAIL"))
        if r > worst:
            worst, worst_name = r, name

    def chk_params(what, got, want, tol, bias_tol, dead_abs):
        """One parameter-shaped vector: conv biases (dead) absolutely, the linear bias (a sum of softmax - onehot rows
        that cancels to ~1e-2 of its terms) at bias_tol."""
        for n, v in want.items():
            if "conv.bias" in n:
                chk("%s %s" % (what, n[-22:]), got[n], v, absolute=dead_abs)
            else:
                chk("%s %s" % (what, n[-22:]), got[n], v, tol=bias_tol if "linear.bias" in n else tol)

    def grid(buf, n, l, pooled):
        """A tap of block l (pooled: its output / its dp) in NCHW: padded grid, or the flat features after the last."""
        gl = geo[l]
        if not pooled:
            return grid_to_nchw(buf, n, gl["h"], gl["w"], F)
        if l + 1 < L:
            return grid_to_nchw(buf, n, gl["h"] // 2, gl["w"] // 2, F)
        return flat_to_nchw(buf, n, ph, pw, F)

    def chk_pass(p, s, fwd, bwd):
        n = n_of[p]
        for l in range(L):
            chk("%s zh   s%d l%d" % (p, s, l), grid(taps[(p + "_zh", s, l)], n, l, False), fwd["blocks"][l]["zh"], tol=2e-5)
            chk("%s pool s%d l%d" % (p, s, l), grid(taps[(p + "_ain", s, l + 1)], n, l, True), fwd["blocks"][l]["p"],
                tol=2e-5)
        for l in reversed(range(L)):
            chk("%s dp   s%d l%d" % (p, s, l), grid(taps[(p + "_dp", s, l)], n, l, True), bwd["blocks"][l]["dp"], tol=5e-5)
            chk("%s dz   s%d l%d" % (p, s, l), grid(taps[(p + "_dz", s, l)], n, l, False), bwd["blocks"][l]["dz"], tol=5e-5)

    for s in range(S):
        chk_params("theta[%d]" % s, theta_to_ref(taps[("theta", s, 0)], a), inter["theta"][s], 1e-5, 1e-5, 1e-5)
        chk_pass("sup", s, inter["sup_f"][s], inter["sup_b"][s])
        chk_params("g[%d]" % s, theta_to_ref(taps[("g", s, 0)], a), inter["sup_g"][s], 5e-5, 2e-4, 1e-5)
        if run["sched"][s] is not None:
            chk_pass("tgt", s, inter["tgt_f"][s][0], inter["tgt_b"][s])
            chk_params("tgrad[%d]" % s, theta_to_ref(taps[("tgrad", s, 0)], a), inter["tgt_g"][s], 5e-5, 2e-4, 1e-5)

    # reverse sweep: u and theta-bar after it, H u of step 0 = u / alpha - theta-bar (theta-bar's own error cancels
    # there: what is left is the tangent pass's error and one rounding of theta-bar), and step 0's tangent pass.
    # Measured on an H100 over every envelope case: <= 6.6e-6 of max-norm -> SWEEP_TOL = 5e-5, a margin of 7x or more
    state64 = g.state(torch.float64)
    alpha0 = {n: float(state64[O.lslr_name(n)][0]) for n in inter["tbar"]}
    u = theta_to_ref(taps[("u", 0, 0)], a)
    tbar = theta_to_ref(taps[("tbar", 0, 0)], a)
    dead = 1e-5 * max(1.0, max(float(v.abs().max()) for n, v in inter["tbar"].items() if "conv.bias" not in n))
    chk_params("u", u, {n: alpha0[n] * v for n, v in inter["tbar0"].items()}, SWEEP_TOL, SWEEP_TOL, dead)
    chk_params("tbar", tbar, inter["tbar"], SWEEP_TOL, SWEEP_TOL, dead)
    if tang0 is not None:
        chk_params("Hu[0]", {n: u[n].double() / alpha0[n] - tbar[n].double() for n in u}, tang0["Hu"], SWEEP_TOL,
                   SWEEP_TOL, dead / min(alpha0.values()))
        # with the tensor cores, dp-dot of the blocks below the last holds only the addend dgrad(W, dz-dot); the other,
        # dgrad(u_W, dz), is computed on a side stream into a buffer of its own
        tf, tb, theta0, n = tang0["tangent"]["fwd"], tang0["tangent"]["bwd"], inter["theta"][0], n_of["sup"]
        for l in range(L):
            chk("tan zh   l%d" % l, grid(taps[("tan_zh", 0, l)], n, l, False), tf[l]["zh_dot"], tol=SWEEP_TOL)
            chk("tan pool l%d" % l, grid(taps[("tan_ain", 0, l + 1)], n, l, True), tf[l]["p_dot"], tol=SWEEP_TOL)
        for l in reversed(range(L)):
            want = tb[l]["dp_dot"]
            if ENVELOPE[case][1]["tc"] and l + 1 < L:
                want = Fnn.conv_transpose2d(tb[l + 1]["dz_dot"], theta0[O.conv_names(l + 1)[0]], stride=1, padding=1)
            chk("tan dp   l%d" % l, grid(taps[("tan_dp", 0, l)], n, l, True), want, tol=SWEEP_TOL)
            chk("tan dz   l%d" % l, grid(taps[("tan_dz", 0, l)], n, l, False), tb[l]["dz_dot"], tol=SWEEP_TOL)
    print("\n[%s stagewise, GPU decisions pinned] worst %.2f x tolerance at %s\n   %s"
          % (case, worst, worst_name, "\n   ".join(rows)))
    assert worst <= 1.0, "stage mismatch (see report above): worst = %.2f x tolerance at %s" % (worst, worst_name)


@gpu
@pytest.mark.parametrize("case", CASES)
def test_decision_forced_parity(case, cuda_device):
    """Every decision the GPU took agrees with fp64 except at margins <= 1e-4; with them pinned the loss agrees to
    1e-5, every meta-gradient tensor to 1e-4 of its max-norm, and the logits."""
    run = _forced_run(case, cuda_device)
    n_dec, n_slope_flip, n_arg_flip, worst_margin = run["flips"]
    ref_loss, grads = run["ref_loss"], run["grads"]
    rows, bad, worst = [], [], 0.0
    live = max(float(v.abs().max()) for v in run["ref_grads"].values())
    for n, v in run["ref_grads"].items():
        err = float((grads[n].double() - v).abs().max())
        scale = max(float(v.abs().max()), 1e-30)
        tol = 1e-5 * max(1.0, live) if _dead(n) else 1e-4 * scale + 1e-7
        if not _dead(n):
            worst = max(worst, err / scale)
        rows.append("%-78s err %.2e (%.1e of max)" % (n, err, err / scale))
        if err > tol:
            bad.append((n, err, tol))
    print("\n[%s] decisions %d, leaky-branch flips %d, arg-max flips %d, worst fp64 margin at a flip %.2e; "
          "loss %.7f vs %.7f; worst meta-gradient error %.2e of max-norm\n   %s"
          % (case, n_dec, n_slope_flip, n_arg_flip, worst_margin, run["loss"], ref_loss, worst, "\n   ".join(rows)))
    assert worst_margin <= 1e-4, worst_margin
    assert abs(run["loss"] - ref_loss) <= 1e-5 * abs(ref_loss), (run["loss"], ref_loss)
    assert not bad, bad
    got_logits = torch.from_numpy(run["logits"]).double()
    assert float((got_logits - run["ref_logits"]).abs().max()) <= 1e-4 * float(run["ref_logits"].abs().max())


@gpu
@pytest.mark.parametrize("case", CASES)
def test_golden_reference_parity(case, cuda_device):
    """Loss, logits, accuracy, MSL weights and every outer gradient against the unmodified reference, on the tiny-case
    policy (conftest.grad_tolerance)."""
    g = load_golden(case)
    m = _model(g, cuda_device)
    losses, preds, grads = m.meta_gradient(g.batch(0), g.iters[0][0])
    ref_loss32, ref_loss64 = g.scalar("loss"), g.scalar("loss64")
    assert abs(float(losses["loss"]) - ref_loss64) <= max(3 * abs(ref_loss32 - ref_loss64), 2e-5 * abs(ref_loss64))
    ref_logits = torch.from_numpy(g.array("logits"))
    got_logits = torch.from_numpy(np.stack(preds))
    assert got_logits.shape == ref_logits.shape
    assert float((got_logits - ref_logits).abs().max()) <= 1e-3 * float(ref_logits.abs().max())
    g32, g64 = g.grads(0, ""), g.grads(0, "64")
    if case in BERNOULLI:
        for n in g32:
            if _dead(n):
                continue
            e32 = float((grads[n].cpu().double() - g32[n].double()).abs().max())
            own = float((g32[n].double() - g64[n].double()).abs().max())
            assert e32 <= max(3.0 * own, 2e-5 * float(g32[n].abs().max())) + 1e-7, ("fp32-anchored (near-ties)", n, e32, own)
    bad = []
    for n in g64:
        err = float((grads[n].cpu().double() - g64[n].double()).abs().max())
        tol = grad_tolerance(n, g32[n], g64[n], big=False)
        if err > tol:
            bad.append((n, err, tol))
    assert not bad, bad
    assert abs(losses["accuracy"] - g.scalar("accuracy")) <= 1e-6
    w = g.array("msl")
    for i in range(len(w)):
        assert abs(float(losses["loss_importance_vector_%d" % i]) - w[i]) < 1e-7


@gpu
@pytest.mark.parametrize("case", CASES)
def test_validation_iter(case, cuda_device):
    """run_validation_iter against the reference's: loss, accuracy, last-step logits, parameters untouched, running
    statistics mutated like the reference's."""
    g = load_golden(case)
    m = _model(g, cuda_device)
    m.current_epoch = g.iters[0][0]
    before = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    losses, preds = m.run_validation_iter(g.batch(0))
    tol = 2e-5
    ref_loss = float(g.val("loss"))
    assert abs(float(losses["loss"]) - ref_loss) <= tol * abs(ref_loss), (float(losses["loss"]), ref_loss)
    ref_logits = torch.from_numpy(g.val("logits"))
    got = torch.from_numpy(np.stack(preds))
    assert got.shape == ref_logits.shape
    assert float((got - ref_logits).abs().max()) <= 10 * tol * float(ref_logits.abs().max())
    assert abs(float(losses["accuracy"]) - float(g.val("accuracy"))) <= 1e-6
    after = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    post = g.val_post()
    for k in before:
        if "running" in k:
            assert torch.allclose(after[k], post[k], rtol=1e-4, atol=1e-5), (k, float((after[k] - post[k]).abs().max()))
        else:
            assert torch.equal(before[k], after[k]), "validation must not change %s" % k


@gpu
@pytest.mark.parametrize("case", CASES)
def test_train_iterations_post_state(case, cuda_device):
    """run_train_iter over the recorded iterations (two where the case records two; clamp, Adam, running-statistics
    EMA): the post-step state_dict against the reference's, on the criteria of
    test_gpu_parity.test_train_iterations_post_state."""
    g = load_golden(case)
    m = _model(g, cuda_device)
    for it, (epoch, _) in enumerate(g.iters):
        losses, preds = m.run_train_iter(g.batch(it), epoch)
        assert abs(float(losses["loss"]) - g.scalar("loss", it)) <= 1e-4 * abs(g.scalar("loss", it)), it
        assert abs(float(losses["learning_rate"]) - g.scalar("learning_rate", it)) <= 1e-9
        post = g.post(it)
        sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
        assert list(sd.keys()) == list(post.keys())
        for k in post:
            if _dead(k):
                continue
            if "running" in k:
                assert torch.allclose(sd[k], post[k], rtol=1e-4, atol=1e-5), (it, k, float((sd[k] - post[k]).abs().max()))
            else:
                diff = (sd[k] - post[k]).abs()
                frac_bad = float((diff > 2e-5).float().mean())
                assert frac_bad <= 2e-3 and float(diff.max()) <= 2.5e-3, (it, k, frac_bad, float(diff.max()))
        with torch.no_grad():
            for k, p in m.named_parameters():
                if "conv.bias" in k:
                    p.copy_(post[k].to(p.device))


@gpu
@pytest.mark.parametrize("case", CASES)
def test_functional_operator(case, cuda_device):
    """VGGReLUNormNetwork.forward at the case's shape, last inner step, on task 0's support batch, against fp64 autograd
    through the oracle network: logits (2e-5), the gradients w.r.t. the fast weights and the BatchNorm gamma / beta, the
    Hessian-vector product along a random direction and the image gradient (5e-5 of max-norm; dead conv biases
    absolute)."""
    a, state, batch = fc.case(case)
    m = fc.model(a, state, cuda_device)
    named = dict(m.named_parameters())
    x, y = fc.images(batch, "support")
    step = int(a.number_of_training_steps_per_iter) - 1
    inner, bn = O.inner_param_names(a), fc.bn_names(state)
    gen = torch.Generator().manual_seed(3)
    v = {n: torch.randn(state[n].shape, generator=gen, dtype=torch.float64) for n in inner}
    # fp64 oracle
    st64 = {k: t.double().clone().requires_grad_(k in bn) for k, t in state.items()}
    fast64 = {n: state[n].double().clone().requires_grad_(True) for n in inner}
    x64 = x.double().requires_grad_(True)
    ref_logits = O._net_forward(x64, fast64, st64, a, step)
    ref_loss = Fnn.cross_entropy(ref_logits, y)
    wrt64 = [fast64[n] for n in inner] + [st64[n] for n in bn]
    ref_g = torch.autograd.grad(ref_loss, wrt64 + [x64], create_graph=True)
    ref_dx = ref_g[-1].detach()
    ref_hv = torch.autograd.grad(sum((gi * v[n]).sum() for gi, n in zip(ref_g, inner)), wrt64)
    # engine operator
    xd = x.to(cuda_device)
    params = {n[len("classifier."):]: named[n].detach().clone().unsqueeze(0).requires_grad_(True) for n in inner}
    wrt = list(params.values()) + [named[n] for n in bn]
    logits = m.classifier.forward(xd, num_step=step, params=params, training=True)
    rows, bad = [], []
    e = rel_err(logits.detach().cpu(), ref_logits.detach())
    rows.append("%-62s rel %.2e" % ("logits", e))
    if e > 2e-5:
        bad.append(("logits", e))
    loss = Fnn.cross_entropy(logits, y.to(cuda_device))
    gr = torch.autograd.grad(loss, wrt, create_graph=True)
    z = sum((gi * v[n].to(cuda_device, torch.float32).reshape(gi.shape)).sum() for gi, n in zip(gr, inner))
    hv = torch.autograd.grad(z, wrt)
    hv_scale = max(float(t.abs().max()) for t in ref_hv)
    for what, got_all, want_all, bias_abs in (("grad", gr, ref_g[:-1], 1e-4), ("hvp", hv, ref_hv, 1e-4 + 5e-5 * hv_scale)):
        for n, got, want in zip(inner + bn, got_all, want_all):
            got, want = got.detach().cpu().double().reshape(want.shape), want.detach()
            if "conv.bias" in n:
                e = float((got - want).abs().max())
                ok = e <= bias_abs
            else:
                e = rel_err(got, want)
                ok = e <= 5e-5
            rows.append("%-62s %.2e" % ("%s %s" % (what, n), e))
            if not ok:
                bad.append((what, n, e))
    # image gradient (fast weights that do not require grad: the first-order input-gradient entry)
    xg = xd.clone().requires_grad_(True)
    plain = {k: t.detach() for k, t in params.items()}
    dx, = torch.autograd.grad(Fnn.cross_entropy(m.classifier.forward(xg, num_step=step, params=plain, training=True),
                                                y.to(cuda_device)), xg)
    e = rel_err(dx.cpu(), ref_dx)
    rows.append("%-62s rel %.2e" % ("dL/dx", e))
    if e > 5e-5:
        bad.append(("dL/dx", e))
    print("\n[%s functional operator vs fp64 autograd, step %d]\n   %s" % (case, step, "\n   ".join(rows)))
    assert not bad, bad


@gpu
@pytest.mark.parametrize("case", [c for c in CASES if ENVELOPE[c][1]["tc"]])
def test_tensor_core_convs_match_fp32_ffma_convs(case, cuda_device):
    """The wgmma 3xTF32 convolutions and weight gradients against their exact-fp32 FFMA twins on the same inputs: every
    intermediate of the first support forward / backward of task 0 to 2e-5."""
    g = load_golden(case)
    L = int(g.args.num_stages)
    outs = []
    for force in (False, True):
        m = _model(g, cuda_device, force_fp32=force)
        m.meta_gradient(g.batch(0), g.iters[0][0])
        eng = m._engine
        taps = {}
        for l in range(L):
            taps["zh%d" % l] = eng.debug_read("sup_zh", 0, 0, l)
            taps["dz%d" % l] = eng.debug_read("sup_dz", 0, 0, l)
            if l < L - 1:
                taps["dp%d" % l] = eng.debug_read("sup_dp", 0, 0, l)
        taps["g0"] = eng.debug_read("g", 0, 0, 0)
        outs.append(taps)
    errs = {k: rel_err(torch.from_numpy(outs[0][k]), torch.from_numpy(outs[1][k])) for k in outs[0]}
    print("\n[%s tensor cores vs FFMA] %s" % (case, " ".join("%s %.1e" % kv for kv in errs.items())))
    assert all(e <= 2e-5 for e in errs.values()), errs
