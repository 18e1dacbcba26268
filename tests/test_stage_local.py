"""Every stage of the benchmarked workloads against fp64 at the task counts bench.py times them at, under every launch
plan the switches select.

The launch plan of a handle depends on its task count (max_tasks) and the SM count: the regime (programmatic dependent
launch and the ring depth of the main-chain tensor-core convolutions), the split-K cluster size of conv_tc_kernel, the
weight-gradient chunk plan and the grid caps of the normalisation kernels.  The full-size goldens run 1 or 2 tasks; bench
runs the Omniglot configs at 8 tasks per GPU, which on an H100 (132 SMs) puts the headline in the throughput regime.

The checker is stage-local: one ``meta_gradient`` with every target pass kept, then each kernel's output against an fp64
evaluation of the oracle's block functions that starts from the GPU's OWN inputs to that stage (debug taps), with the
GPU's own leaky-ReLU branches and pooling arg-maxes.  No error carries over from an earlier stage, no near-tie can flip
between the two sides, and the bounds hold whatever the image size, task count or inner-loop divergence:

  stage       GPU inputs                          fp64 reference                           compared with
  forward     ain[l] (images at l = 0), theta     block_forward, decisions forced          zh[l]
  pool        the GPU's zh[l], gamma / beta       fmaf, leaky-ReLU, first max wins         ain[l+1], to 1 fp32 ulp
  head        ain[L], theta                       head_forward / head_backward             dp[L-1], linear part of g / tgrad
  norm bwd    the GPU's dp[l]                     block_backward                           dz[l] (inner-loop gamma / beta: their g)
  dgrad       the GPU's dz[l]                     conv_transpose2d                         dp[l-1]
  wgrad       ain[l], the GPU's dz[l]             conv2d_weight, bias sum                  block l of g[s] / tgrad[s]
  tangent     tan_ain[l], u, tan_dp[l] (step 0)   torch.func.jvp of the same functions     tan_zh, tan_ain, tan_dz, tan_dp

Every task is checked at steps 0 and S-1, tasks 0 and T-1 at the steps between, support and target passes.

Tolerances (of the compared tensor's max-norm), each at least 5x the worst measured on an H100 over every case below:
see TOL."""
import gc

import numpy as np
import pytest
import torch
import torch.nn.functional as Fnn

from engine_layout import (K_BN, K_CONV_ROWS, K_CONV_TC, K_IBN, K_LN, K_WGRAD_ROW, K_WGRAD_TC, activate_pool,
                           check_norm_path, device_sms, flat_to_nchw, geometry, grid_to_nchw, host_plan,
                           norm_grid_regimes, norm_params, rel_err, theta_to_ref, traced_kernel_ids)
from oracle import ln_oracle as LN
from oracle import maml_oracle as O

EPOCH = 3            # multi-step loss between its extremes: every target pass has a weight of its own
MOVED_SEED = 7
K_BNBWD_FUSED, K_TAIL, K_TAIL_TAN, K_TAIL_ONCHIP = {9, 13}, 23, 24, 25

# the benchmarked workloads at their per-GPU task counts: name -> (config, tasks, input kind, moved-state seed, overrides)
WORKLOADS = {
    "headline": ("omniglot_mamlpp_5w1s", 8, "normal", None, {}),
    "headline_bernoulli": ("omniglot_mamlpp_5w1s", 8, "bernoulli", None, {}),      # what bench feeds: exact pooling ties
    "headline_moved": ("omniglot_mamlpp_5w1s", 8, "normal", MOVED_SEED, {}),
    "maml": ("omniglot_maml_5w1s", 8, "bernoulli", None, {}),
    "omniglot_20w5s": ("omniglot_mamlpp_20w5s", 8, "bernoulli", None, {}),
    "mini_imagenet_5w1s": ("mini_imagenet_mamlpp_5w1s", 2, "normal", None, {}),
    "mini_imagenet_5w5s": ("mini_imagenet_mamlpp_5w5s", 2, "normal", None, {}),
    # the other normalisations at the headline's shape and task count, from moved states
    "headline_layer_norm": ("omniglot_mamlpp_5w1s", 8, "normal", MOVED_SEED, {"norm_layer": "layer_norm"}),
    "headline_inner_bn": ("omniglot_mamlpp_5w1s", 8, "normal", MOVED_SEED,
                          {"enable_inner_loop_optimizable_bn_params": True}),
}

# the plan each workload reaches on an H100 (132 SMs): regime, weight-gradient chunks per block, grid regimes of the
# normalisation kernels (engine_layout.host_plan / norm_grid_regimes).  A change that moves a workload to another plan
# has to update this table, and with it what the matrix below covers.
PLANS = {
    "headline": ("throughput", 5, set()),
    "headline_bernoulli": ("throughput", 5, set()),
    "headline_moved": ("throughput", 5, set()),
    "maml": ("throughput", 5, set()),
    "omniglot_20w5s": ("throughput", 5, {"ibn_reduce_capped", "ibn_apply_capped", "ln_capped", "ln_one_cta"}),
    "mini_imagenet_5w1s": ("throughput", 22, {"ibn_reduce_capped", "ibn_apply_capped", "ln_capped"}),
    "mini_imagenet_5w5s": ("throughput", 22, {"ibn_reduce_capped", "ibn_apply_capped", "ln_capped"}),
    "headline_layer_norm": ("throughput", 5, set()),
    "headline_inner_bn": ("throughput", 5, set()),
}

# the launch-plan matrix on the headline at 8 tasks: name -> (workload, switches read when the handle is created, force
# the fp32 FFMA convolutions).  The split-K cluster size (TC_SPLIT) is requested, not asserted: it is the smaller of the
# request and what the occupancy calculator admits at launch, and no tap shows it.
SWITCHES = {
    "split1": ("headline", {"MAML_B200_TC_SPLIT": "1"}, False),
    "split2": ("headline", {"MAML_B200_TC_SPLIT": "2"}, False),
    "split4": ("headline", {"MAML_B200_TC_SPLIT": "4"}, False),
    "ring2": ("headline", {"MAML_B200_TC_NB": "2"}, False),
    "ring8": ("headline", {"MAML_B200_TC_NB": "8"}, False),
    "pdl_on": ("headline", {"MAML_B200_PDL": "1"}, False),          # the latency regime's feature in the throughput one
    "bn_unfused": ("headline", {"MAML_B200_BN_FUSE": "0"}, False),
    "tail_unfused": ("headline", {"MAML_B200_TAIL_FUSE": "0"}, False),
    "tail_offchip": ("headline", {"MAML_B200_TAIL_ONCHIP": "0"}, False),
    "wgrad_ffma": ("headline", {"MAML_B200_WGRAD_TC": "0"}, False),
    "fp32_convs": ("headline", {}, True),
    "inner_bn_unfused": ("headline_inner_bn", {"MAML_B200_BN_FUSE": "0"}, False),
}
CASES = {**{w: (w, {}, False) for w in WORKLOADS}, **SWITCHES}

# max |GPU - fp64| over the compared tensor's max-norm, per stage kind; the pool is compared in fp32 ulps.  Worst measured
# over every case on an H100 80GB HBM3 (700 W): forward 2.4e-6 (fp32 FFMA convolutions; 5.7e-7 on the tensor cores), pool
# 0 ulps, head 2.3e-5, norm backward 6.3e-7, dgrad 1.1e-6, wgrad 1.24e-5, tangent 3.2e-6.  The head's errors are those of
# softmax - onehot on nearly fitted tasks at the last inner step, where it cancels to a fraction of its terms; the weight
# gradient's are those of its sums over 78 k (Omniglot 20-way support) to 132 k (Mini-ImageNet target) pixel rows -- on the
# 5-way Omniglot passes it sits at 1.4e-6.
TOL = {"forward": 2e-5, "pool": 1.0, "head": 1.5e-4, "norm_bwd": 1e-5, "dgrad": 1e-5, "wgrad": 7e-5, "tangent": 3e-5}
# linear-layer bias gradients: a sum over rows of softmax - onehot, which cancels to ~1e-2 of its terms on a fitted task
HEAD_BIAS_TOL = 2e-4


def _args(workload):
    from howtotrainyourmamlpytorch_b200 import make_args
    config, tasks, _, _, over = WORKLOADS[workload]
    return make_args(config, batch_size=tasks, **over)


def _dead(a, n):
    """Conv biases under BatchNorm: true gradient 0, both sides are rounding noise."""
    return n.endswith("conv.bias") and getattr(a, "norm_layer", "batch_norm") != "layer_norm"


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("workload", list(WORKLOADS))
def test_workload_plan(workload):
    """The host rules put each workload on the plan PLANS declares for an H100."""
    a = _args(workload)
    tasks = WORKLOADS[workload][1]
    plan = host_plan(a, tasks)
    regime, chunks, grids = PLANS[workload]
    assert (plan["regime"], plan["chunks"]) == (regime, chunks), (workload, plan)
    assert plan["pdl"] == (regime == "latency") and plan["nb"] == (8 if regime == "latency" else 4), plan
    assert plan["tc"], plan
    assert norm_grid_regimes(a, tasks) == grids, (workload, norm_grid_regimes(a, tasks))


def test_headline_regime_on_h100():
    """The headline at 8 tasks: (9 + 9) * 8 = 144 block-1 tiles, more than an H100's 132 SMs -- throughput regime."""
    plan = host_plan(_args("headline"), 8)
    assert plan["tiles"] == 144 and plan["regime"] == "throughput"
    assert host_plan(_args("headline"), 8, num_sms=148)["regime"] == "latency"


# ------------------------------------------------------------------------------------------------ GPU
class _Checker(object):
    """Worst error per stage kind, as a multiple of its tolerance, and one report row per comparison."""

    def __init__(self):
        self.rows, self.worst = [], {k: (0.0, "") for k in TOL}

    def rel(self, kind, name, got, want, tol=None):
        e = rel_err(got, want)
        self._add(kind, name, e, tol or TOL[kind])

    def absolute(self, kind, name, got, want, scale):
        e = float((got.double() - want.double()).abs().max()) / max(scale, 1e-30)
        self._add(kind, name, e, TOL[kind])

    def ulps(self, name, got, want):
        got, want = got.float().numpy(), want.float().numpy()
        e = float(np.max(np.abs(got.astype(np.float64) - want) / np.spacing(np.abs(want)))) if want.size else 0.0
        self._add("pool", name, e, TOL["pool"])

    def _add(self, kind, name, e, tol):
        r = e / tol
        self.rows.append("%-9s %-36s %.2e%s" % (kind, name, e, "" if r <= 1.0 else "   <-- FAIL"))
        if r >= self.worst[kind][0]:
            self.worst[kind] = (r, name)


def _check_params(chk, kind, a, tag, got, want, names, dead_scale=None):
    """Parameter-shaped comparisons (blocks of g / tgrad): live tensors of their max-norm, dead conv biases (sums of dz
    that cancel to rounding noise) against ``dead_scale``, the largest per-channel sum of |dz|, linear biases at
    HEAD_BIAS_TOL."""
    for n in names:
        if _dead(a, n):
            chk.absolute(kind, "%s %s" % (tag, n[-24:]), got[n], want[n], dead_scale)
        else:
            chk.rel(kind, "%s %s" % (tag, n[-24:]), got[n], want[n], HEAD_BIAS_TOL if n == O.LIN_B else None)


def _stage_local(m, a, batch, epoch, tc, chk):
    """The checker of the module docstring on one iteration of ``m`` (run with every target pass kept)."""
    eng = m._engine
    ln = getattr(a, "norm_layer", "batch_norm") == "layer_norm"
    ibn = bool(a.enable_inner_loop_optimizable_bn_params)
    M = LN if ln else O
    geo, (ph, pw) = geometry(a)
    F, N, L = int(a.cnn_num_filters), int(a.num_classes_per_set), len(geo)
    K, T, S = int(a.num_samples_per_class), int(a.num_target_samples), int(a.number_of_training_steps_per_iter)
    B = batch[0].shape[0]
    sched = O.target_pass_schedule(a, epoch, True, S)
    w_msl = O.msl_weights(a, epoch)
    sd = {k: v.detach().cpu().double() for k, v in m.state_dict().items()}
    d = torch.float64

    def read(name, b, s, l, n, grid_l, pooled):
        buf = eng.debug_read(name, b, s, l)
        gl = geo[grid_l]
        if not pooled:
            return grid_to_nchw(buf, n, gl["h"], gl["w"], F)
        if grid_l + 1 < L:
            return grid_to_nchw(buf, n, gl["h"] // 2, gl["w"] // 2, F)
        return flat_to_nchw(buf, n, ph, pw, F)

    def wb(l):
        wn, bn_, _, _, _, _ = O.conv_names(l)
        return wn, bn_

    def forward(a_in, th, gb, l, forced):
        wn, bn_ = wb(l)
        return M.block_forward(a_in, th[wn], th[bn_], gb[0], gb[1], forced)

    def backward(fw, th, gb, l, dp):
        return M.block_backward(fw, th[wb(l)[0]], gb[0], dp, need_dgrad=False)

    def one_pass(b, kind, s):
        """forward, pool, head, norm backward, dgrad and wgrad stages of one pass; returns the per-block records."""
        n = N * (K if kind == "sup" else T)
        x = (batch[0] if kind == "sup" else batch[1])[b].reshape(n, *batch[0].shape[-3:]).to(d)
        y = (batch[2] if kind == "sup" else batch[3])[b].reshape(n).long()
        th = {k: v.to(d) for k, v in theta_to_ref(eng.debug_read("theta", b, s + (kind == "tgt"), 0), a).items()}
        scale = float(w_msl[s]) if (kind == "tgt" and sched[s] == "msl") else 1.0
        grad = theta_to_ref(eng.debug_read("g" if kind == "sup" else "tgrad", b, s, 0), a)
        tag = "t%d %s s%d" % (b, kind, s)
        recs = []
        for l in range(L):
            a_in = x if l == 0 else read(kind + "_ain", b, s, l, n, l - 1, True).to(d)
            gb = tuple(v.to(d) for v in norm_params(a, sd, th, l, s))
            zh = read(kind + "_zh", b, s, l, n, l, False)
            slope, idx, p = activate_pool(zh, *gb)
            fw = forward(a_in, th, gb, l, (slope, idx))
            chk.rel("forward", "%s zh l%d" % (tag, l), zh, fw["zh"])
            chk.ulps("%s pool l%d" % (tag, l), read(kind + "_ain", b, s, l + 1, n, l, True), p)
            recs.append(dict(a_in=a_in, gb=gb, fw=fw))
        f = read(kind + "_ain", b, s, L, n, L - 1, True).to(d).reshape(n, -1)
        _, _, prob = O.head_forward(f, th[O.LIN_W], th[O.LIN_B], y)
        hb = O.head_backward(f, th[O.LIN_W], prob, y, scale)
        dp = read(kind + "_dp", b, s, L - 1, n, L - 1, True)
        chk.rel("head", "%s dp l%d" % (tag, L - 1), dp, hb["df"].reshape(dp.shape))
        _check_params(chk, "head", a, tag, grad, {O.LIN_W: hb["dW"], O.LIN_B: hb["db"]}, (O.LIN_W, O.LIN_B))
        for l in reversed(range(L)):
            r = recs[l]
            dp = read(kind + "_dp", b, s, l, n, l, True).to(d)
            bw = backward(r["fw"], th, r["gb"], l, dp)
            dz = read(kind + "_dz", b, s, l, n, l, False)
            chk.rel("norm_bwd", "%s dz l%d" % (tag, l), dz, bw["dz"])
            if ibn:
                _, _, gn, btn, _, _ = O.conv_names(l)
                _check_params(chk, "norm_bwd", a, tag, grad, {gn: bw["dgamma"], btn: bw["dbeta"]}, (gn, btn))
            wn, bn_ = wb(l)
            dz = dz.to(d)
            if l > 0:
                dprev = read(kind + "_dp", b, s, l - 1, n, l - 1, True)
                chk.rel("dgrad", "%s dp l%d" % (tag, l - 1), dprev, Fnn.conv_transpose2d(dz, th[wn], padding=1))
            want = {wn: torch.nn.grad.conv2d_weight(r["a_in"], th[wn].shape, dz, padding=1), bn_: dz.sum(dim=(0, 2, 3))}
            _check_params(chk, "wgrad", a, tag, grad, want, (wn, bn_), float(dz.abs().sum(dim=(0, 2, 3)).max()))
        return recs

    def tangent(b, recs):
        """Step 0's tangent pass of task b (the one its tangent buffers hold) in the direction u the GPU used."""
        n = N * K
        y = batch[2][b].reshape(n).long()
        th = {k: v.to(d) for k, v in theta_to_ref(eng.debug_read("theta", b, 0, 0), a).items()}
        u = {k: v.to(d) for k, v in theta_to_ref(eng.debug_read("u", b, 0, 0), a).items()}
        tag = "t%d tan" % b
        sup_dz = [read("sup_dz", b, 0, l, n, l, False).to(d) for l in range(L)]
        for l in range(L):
            r = recs[l]
            wn, bn_ = wb(l)
            forced = (r["fw"]["slope"], r["fw"]["idx"])
            a_dot = torch.zeros_like(r["a_in"]) if l == 0 else read("tan_ain", b, 0, l, n, l - 1, True).to(d)
            _, _, gn, btn, _, _ = O.conv_names(l)
            gb_dot = (u[gn], u[btn]) if ibn else tuple(torch.zeros_like(v) for v in r["gb"])

            def fwd_fn(a_in, W, bias, gam, bet):
                fw = M.block_forward(a_in, W, bias, gam, bet, forced)
                return fw["zh"], fw["p"]
            _, (zh_dot, p_dot) = torch.func.jvp(fwd_fn, (r["a_in"], th[wn], th[bn_]) + r["gb"],
                                                (a_dot, u[wn], u[bn_]) + gb_dot)
            chk.rel("tangent", "%s zh l%d" % (tag, l), read("tan_zh", b, 0, l, n, l, False), zh_dot)
            chk.rel("tangent", "%s pool l%d" % (tag, l), read("tan_ain", b, 0, l + 1, n, l, True), p_dot)
        f = read("sup_ain", b, 0, L, n, L - 1, True).to(d).reshape(n, -1)
        f_dot = read("tan_ain", b, 0, L, n, L - 1, True).to(d).reshape(n, -1)

        def head_fn(f_, W, bias):
            _, _, prob = O.head_forward(f_, W, bias, y)
            return O.head_backward(f_, W, prob, y)["df"]
        _, df_dot = torch.func.jvp(head_fn, (f, th[O.LIN_W], th[O.LIN_B]), (f_dot, u[O.LIN_W], u[O.LIN_B]))
        dp_dot = read("tan_dp", b, 0, L - 1, n, L - 1, True)
        chk.rel("tangent", "%s dp l%d" % (tag, L - 1), dp_dot, df_dot.reshape(dp_dot.shape))
        for l in reversed(range(L)):
            r = recs[l]
            wn, bn_ = wb(l)
            forced = (r["fw"]["slope"], r["fw"]["idx"])
            a_dot = torch.zeros_like(r["a_in"]) if l == 0 else read("tan_ain", b, 0, l, n, l - 1, True).to(d)
            _, _, gn, btn, _, _ = O.conv_names(l)
            gb_dot = (u[gn], u[btn]) if ibn else tuple(torch.zeros_like(v) for v in r["gb"])
            dp = read("sup_dp", b, 0, l, n, l, True).to(d)
            dp_dot = read("tan_dp", b, 0, l, n, l, True).to(d)
            if tc and l + 1 < L:
                # with the tensor cores, tan_dp below the last block holds only dgrad(W, dz-dot); the other addend,
                # dgrad(u_W, dz), is computed on a side stream into a buffer of its own
                dp_dot = dp_dot + Fnn.conv_transpose2d(sup_dz[l + 1], u[wb(l + 1)[0]], padding=1)

            def bwd_fn(a_in, W, bias, gam, bet, dp_):
                fw = M.block_forward(a_in, W, bias, gam, bet, forced)
                return M.block_backward(fw, W, gam, dp_, need_dgrad=False)["dz"]
            _, dz_dot = torch.func.jvp(bwd_fn, (r["a_in"], th[wn], th[bn_]) + r["gb"] + (dp,),
                                       (a_dot, u[wn], u[bn_]) + gb_dot + (dp_dot,))
            tdz = read("tan_dz", b, 0, l, n, l, False)
            chk.rel("tangent", "%s dz l%d" % (tag, l), tdz, dz_dot)
            if l > 0:
                want = Fnn.conv_transpose2d(tdz.to(d), th[wn], padding=1)
                if not tc:
                    want = want + Fnn.conv_transpose2d(sup_dz[l], u[wn], padding=1)
                chk.rel("tangent", "%s dp l%d" % (tag, l - 1), read("tan_dp", b, 0, l - 1, n, l - 1, True), want)

    second_order = bool(a.second_order) and epoch > a.first_order_to_second_order_epoch
    for b in range(B):
        for s in range(S):
            if s not in (0, S - 1) and b not in (0, B - 1):
                continue
            recs = one_pass(b, "sup", s)
            if sched[s] is not None:
                one_pass(b, "tgt", s)
            if s == 0 and second_order:
                tangent(b, recs)


def _check_kernels(ids, case, a, tasks):
    """The kernels of one traced iteration: those of the handle's norm path and of the plan its switches select."""
    _, switches, fp32 = CASES[case]
    norm = "ln" if a.norm_layer == "layer_norm" else ("ibn" if a.enable_inner_loop_optimizable_bn_params else "bn")
    if norm != "bn":
        check_norm_path(ids, norm, a, EPOCH, tasks)
    else:
        assert K_BN & ids and not ids & (K_LN | K_IBN), sorted(ids)
    conv = {K_CONV_ROWS} if fp32 else {K_CONV_TC}
    wgrad = {K_WGRAD_ROW} if (fp32 or switches.get("MAML_B200_WGRAD_TC") == "0") else {K_WGRAD_TC}
    assert conv | wgrad <= ids and not ids & ({K_CONV_ROWS, K_CONV_TC, K_WGRAD_ROW, K_WGRAD_TC} - conv - wgrad), sorted(ids)
    if switches.get("MAML_B200_BN_FUSE") == "0":
        assert not ids & K_BNBWD_FUSED, sorted(ids)
    # the fused tail runs the last block's BatchNorm backward itself: BN_FUSE=0 turns it off too
    tail = norm == "bn" and host_plan(a, tasks, device_sms())["tail"] and \
        switches.get("MAML_B200_TAIL_FUSE") != "0" and switches.get("MAML_B200_BN_FUSE") != "0"
    if tail:
        assert ids & {K_TAIL, K_TAIL_ONCHIP} and K_TAIL_TAN in ids, sorted(ids)
        if switches.get("MAML_B200_TAIL_ONCHIP") == "0":
            assert K_TAIL in ids and K_TAIL_ONCHIP not in ids, sorted(ids)
    else:
        assert not ids & {K_TAIL, K_TAIL_TAN, K_TAIL_ONCHIP}, sorted(ids)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_stage_local(case, cuda_device, monkeypatch):
    """One iteration of the case against the stage-local fp64 checker, every task at the first and last inner step;
    and the plan it runs: the kernels of a traced iteration, the regime and chunk count of the host rules."""
    from howtotrainyourmamlpytorch_b200 import MAMLFewShotClassifier, synthetic_batch
    workload, switches, fp32 = CASES[case]
    for k, v in switches.items():
        monkeypatch.setenv(k, v)
    a = _args(workload)
    _, tasks, kind, moved, _ = WORKLOADS[workload]
    plan = host_plan(a, tasks, device_sms())
    torch.manual_seed(0)
    m = MAMLFewShotClassifier(im_shape=(2, a.image_channels, a.image_height, a.image_width), device=cuda_device, args=a)
    m._debug_keep_target_passes = True
    m._debug_force_fp32_convs = fp32
    if moved is not None:
        m.load_state_dict((LN if a.norm_layer == "layer_norm" else O).moved_state(m.state_dict(), a, moved))
    batch = synthetic_batch(a, iteration=1, kind=kind)
    ids = traced_kernel_ids(m, batch, EPOCH)          # the taps read below are those of the traced iteration
    _check_kernels(ids, case, a, tasks)
    chk = _Checker()
    _stage_local(m, a, batch, EPOCH, plan["tc"] and not fp32, chk)
    del m
    gc.collect()
    print("\n[%s] plan %s, kernels %s\n   %s\n[%s] worst per stage kind (error, x tolerance, where): %s" % (
        case, {k: plan[k] for k in ("regime", "chunks", "tiles")}, sorted(ids), "\n   ".join(chk.rows), case,
        "; ".join("%s %.2e %.3f %s" % (k, r * TOL[k], r, n) for k, (r, n) in chk.worst.items())))
    assert device_sms() != 132 or (plan["regime"], plan["chunks"]) == PLANS[workload][:2], plan
    bad = {k: v for k, v in chk.worst.items() if v[0] > 1.0}
    assert not bad, "stage mismatch (x tolerance): %s" % bad
