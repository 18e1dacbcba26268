"""ORACLE -- TEST INFRASTRUCTURE ONLY.  Not part of the shipped product.

CPU restatement of the reference's MAML / MAML++ inner-loop hot path
(`MAMLFewShotClassifier.run_train_iter`), used only as the checker for the CUDA path:
only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this module.  The product package
(``howtotrainyourmamlpytorch_b200``) never imports it and fails loudly when its CUDA
library is missing.

Parity status: the reference ships NO tests / golden vectors for this path
(SURVEY.md section 4), so the oracle is pinned the other way round: the unmodified reference
(a pure-Python/PyTorch program) is imported from ``/root/reference`` in the authoring
container by ``oracle/gen_golden.py`` and its outputs (loss, logits, all outer gradients,
post-Adam parameters, running statistics; fp32 and fp64) are committed under
``tests/golden/``.  ``tests/test_oracle_golden.py`` checks both restatements below against
those vectors.

The arithmetic of the path lives in a third-party dependency of the reference that is not
under ``/root/reference``: PyTorch (``torch.nn.functional`` + autograd; the reference pins no
version, this image has torch 2.11.0).  Two restatements are kept:

``autograd_train_iter``  follows the reference call for call (same ``torch.nn.functional``
    ops, ``torch.autograd.grad(create_graph=second_order)``, one reverse sweep) but as a
    flat functional program.  It is the ``"port"`` CPU baseline that ``bench.py`` times.
    Follows reference ``few_shot_learning_system.py:170-263`` (forward), ``:122-161``
    (apply_inner_loop_update), ``:265-286`` (net_forward), ``:83-103`` (MSL weights),
    ``meta_neural_network_architectures.py:620-660, 387-428, 205-247, 68-97, 120-141``
    and ``inner_loop_optimizers.py:99-113``.

``manual_train_iter``  is the autograd-free executable specification that the CUDA kernels
    implement one to one (SURVEY.md appendix A1-A4): explicit block forward, block
    backward, forward-over-reverse tangent (Hessian-vector) pass and the reverse sweep
    over inner steps.  It also returns every intermediate the kernels materialise so the
    GPU tests can bisect a mismatch stage by stage.
"""
from collections import OrderedDict
import math

import numpy as np
import torch
import torch.nn.functional as F

BN_EPS = 1e-5          # reference meta_neural_network_architectures.py:144
BN_MOMENTUM = 0.1      # reference meta_neural_network_architectures.py:144
LEAKY_SLOPE = 0.01     # F.leaky_relu default, reference :426


# ----------------------------------------------------------------------------------------
# configuration helpers
# ----------------------------------------------------------------------------------------
def num_stages(args):
    return int(getattr(args, "num_stages", 4))


def spatial_sizes(args):
    """[(h_l, w_l)] conv-output size of every block and the pooled size after the last."""
    h, w = int(args.image_height), int(args.image_width)
    sizes = []
    for _ in range(num_stages(args)):
        sizes.append((h, w))
        h, w = h // 2, w // 2
    return sizes, (h, w)


def feature_dim(args):
    _, (h, w) = spatial_sizes(args)
    return int(args.cnn_num_filters) * h * w


def conv_names(l):
    p = "classifier.layer_dict.conv%d." % l
    return (p + "conv.weight", p + "conv.bias", p + "norm_layer.weight", p + "norm_layer.bias",
            p + "norm_layer.running_mean", p + "norm_layer.running_var")


LIN_W = "classifier.layer_dict.linear.weights"
LIN_B = "classifier.layer_dict.linear.bias"


def lslr_name(param_name):
    # reference inner_loop_optimizers.py:89 (key.replace(".", "-")) on names without the
    # leading "classifier." (the dict is built from classifier.named_parameters()).
    short = param_name[len("classifier."):]
    return "inner_loop_optimizer.names_learning_rates_dict." + short.replace(".", "-")


def inner_param_names(args):
    """The adaptable tensors, in reference order (few_shot_learning_system.py:105-120): per block conv.weight, conv.bias
    (with ``enable_inner_loop_optimizable_bn_params`` also norm_layer.bias, norm_layer.weight), then the linear layer."""
    names = []
    for l in range(num_stages(args)):
        wn, bn_, gn, btn, _, _ = conv_names(l)
        names += [wn, bn_, btn, gn] if args.enable_inner_loop_optimizable_bn_params else [wn, bn_]
    names += [LIN_W, LIN_B]
    return names


def trainable_names(args):
    """Outer (Adam) parameter order = reference ``trainable_parameters`` (:288-294)."""
    names = []
    for l in range(num_stages(args)):
        wn, bn_, gn, btn, _, _ = conv_names(l)
        names += [wn, bn_]
        if args.learnable_bn_beta:
            names.append(btn)
        if args.learnable_bn_gamma:
            names.append(gn)
    names += [LIN_W, LIN_B]
    if args.learnable_per_layer_per_step_inner_loop_learning_rate:
        names += [lslr_name(n) for n in inner_param_names(args)]
    return names


def init_state(args, dtype=torch.float32):
    """Reference initialisation restated (few_shot_learning_system.py:13-23,42-53;
    meta_neural_network_architectures.py:62-66,114-118,177-192; inner_loop_optimizers.py:86-91).
    Returns an OrderedDict with the reference's ``state_dict`` key names and order."""
    rng = np.random.RandomState(seed=args.seed)
    torch_seed = rng.randint(0, 999999)
    torch.manual_seed(torch_seed)
    S = int(args.number_of_training_steps_per_iter)
    Fn = int(args.cnn_num_filters)
    cin = int(args.image_channels)
    st = OrderedDict()
    for l in range(num_stages(args)):
        wn, bn_, gn, btn, rmn, rvn = conv_names(l)
        w = torch.empty(Fn, cin, 3, 3)
        torch.nn.init.xavier_uniform_(w)
        st[wn] = w
        st[bn_] = torch.zeros(Fn)
        if args.per_step_bn_statistics:
            st[rmn] = torch.zeros(S, Fn)
            st[rvn] = torch.ones(S, Fn)
            # reference quirk: two all-zero dummy forwards at num_step=0 while the network builds itself
            # (meta_neural_network_architectures.py:365 and :603) leave running_var[0] = 0.9*0.9 (fp32)
            st[rvn][0] = st[rvn][0] * (1 - BN_MOMENTUM) * (1 - BN_MOMENTUM)
            st[btn] = torch.zeros(S, Fn)
            st[gn] = torch.ones(S, Fn)
        else:
            st[rmn] = torch.zeros(Fn)
            st[rvn] = torch.zeros(Fn)          # sic: zeros in shared mode (reference :188)
            st[btn] = torch.zeros(Fn)
            st[gn] = torch.ones(Fn)
        cin = Fn
    lw = torch.ones(int(args.num_classes_per_set), feature_dim(args))
    torch.nn.init.xavier_uniform_(lw)
    st[LIN_W] = lw
    st[LIN_B] = torch.zeros(int(args.num_classes_per_set))
    for n in inner_param_names(args):
        st[lslr_name(n)] = torch.ones(S + 1) * float(args.task_learning_rate)
    return OrderedDict((k, v.to(dtype)) for k, v in st.items())


def moved_state(state, args, seed):
    """``state`` moved away from the reference's initialisation, seeded and deterministic: BatchNorm gamma ~ U(0.6, 1.4)
    and beta ~ 0.2 N(0, 1) per (step, channel), one LSLR rate ~ U(0.02, 0.1) per (tensor, step), conv and linear biases
    ~ 0.1 N(0, 1), running means ~ 0.1 N(0, 1) and variances ~ U(0.5, 1.5) per (step, channel).  Weights are kept.
    At the initialisation gamma = 1, beta = 0, the biases are 0 and every rate is equal, so a kernel that reads gamma /
    beta / alpha from the wrong step, block or tensor, or drops a gamma factor or a bias, computes the right numbers
    there; here it does not.  The ranges keep the inner loop tame (the reference's own fp32 run stays 1e-6 to 1.6e-5 of
    max-norm from its fp64 run on the envelope shapes)."""
    gen = torch.Generator().manual_seed(int(seed))
    out = OrderedDict()
    for k, v in state.items():
        shape = v.shape
        if k.endswith("norm_layer.weight"):
            new = 0.6 + 0.8 * torch.rand(shape, generator=gen, dtype=torch.float64)
        elif k.endswith("norm_layer.bias"):
            new = 0.2 * torch.randn(shape, generator=gen, dtype=torch.float64)
        elif k.endswith("running_mean"):
            new = 0.1 * torch.randn(shape, generator=gen, dtype=torch.float64)
        elif k.endswith("running_var"):
            new = 0.5 + torch.rand(shape, generator=gen, dtype=torch.float64)
        elif k.endswith("conv.bias") or k == LIN_B:
            new = 0.1 * torch.randn(shape, generator=gen, dtype=torch.float64)
        elif k.startswith("inner_loop_optimizer."):
            new = 0.02 + 0.08 * torch.rand(shape, generator=gen, dtype=torch.float64)
        else:
            new = v.detach().clone()
        out[k] = new.to(v.dtype)
    return out


def msl_weights(args, current_epoch):
    """Per-step loss importance vector (reference few_shot_learning_system.py:83-103),
    float64 arithmetic then rounded to float32 exactly like ``torch.Tensor(np_array)``."""
    S = int(args.number_of_training_steps_per_iter)
    w = np.ones(shape=(S,)) * (1.0 / S)
    decay = 1.0 / S / args.multi_step_loss_num_epochs
    min_nonfinal = 0.03 / S
    for i in range(S - 1):
        w[i] = np.maximum(w[i] - (current_epoch * decay), min_nonfinal)
    w[-1] = np.minimum(w[-1] + (current_epoch * (S - 1) * decay), 1.0 - ((S - 1) * min_nonfinal))
    return w.astype(np.float32)


def cosine_lr(args, epoch):
    """Closed form used by ``scheduler.step(epoch=epoch)`` (reference :70-71, :346)."""
    base, eta_min, T = float(args.meta_learning_rate), float(args.min_learning_rate), int(args.total_epochs)
    return eta_min + (base - eta_min) * (1.0 + math.cos(math.pi * epoch / T)) / 2.0


def target_pass_schedule(args, epoch, training_phase, num_steps):
    """For every inner step s: None (no target pass) or the loss weight.  Weight ``None``
    inside the list means "un-weighted" (plain loss).  Reference :232-244."""
    S_train = int(args.number_of_training_steps_per_iter)
    use_msl = bool(args.use_multi_step_loss_optimization) if training_phase else True
    sched = []
    for s in range(num_steps):
        if use_msl and training_phase and epoch < args.multi_step_loss_num_epochs:
            sched.append("msl")
        elif s == S_train - 1:
            sched.append("final")
        else:
            sched.append(None)
    return sched


# ----------------------------------------------------------------------------------------
# restatement 1: autograd, call for call
# ----------------------------------------------------------------------------------------
def _bn_params(state, fast, args, l, step):
    """Block l's BatchNorm gamma / beta at inner step ``step``.  With ``enable_inner_loop_optimizable_bn_params`` they are
    fast weights, read from ``fast`` without a step index (reference meta_neural_network_architectures.py:194-198,
    :229-234); otherwise they are ``state``'s, one row per step with per-step statistics."""
    _, _, gn, btn, _, _ = conv_names(l)
    if args.enable_inner_loop_optimizable_bn_params:
        return fast[gn], fast[btn]
    g, b = state[gn], state[btn]
    if args.per_step_bn_statistics:
        return g[step], b[step]
    return g, b


def _net_forward(x, fast, state, args, step, stats_out=None):
    out = x
    for l in range(num_stages(args)):
        wn, bn_, _, _, _, _ = conv_names(l)
        out = F.conv2d(out, fast[wn], fast[bn_], stride=1, padding=1)
        if stats_out is not None:
            with torch.no_grad():
                m = out.numel() // out.shape[1]
                mu = out.mean(dim=(0, 2, 3))
                var_unbiased = out.var(dim=(0, 2, 3), unbiased=True) if m > 1 else out.new_zeros(out.shape[1])
                stats_out.append((l, step, mu, var_unbiased))
        g, b = _bn_params(state, fast, args, l, step)
        out = F.batch_norm(out, None, None, g, b, training=True, momentum=BN_MOMENTUM, eps=BN_EPS)
        out = F.leaky_relu(out)
        out = F.max_pool2d(out, kernel_size=(2, 2), stride=2, padding=0)
    out = out.reshape(out.shape[0], -1)
    return F.linear(out, fast[LIN_W], fast[LIN_B])


def autograd_train_iter(state, args, batch, epoch, training_phase=True, current_epoch=None):
    """One outer iteration (no optimiser step): loss, accuracy, per-task last-step logits,
    outer gradients for ``trainable_names`` and the updated running statistics.

    ``state``: dict name -> tensor (reference state_dict names); its dtype is the compute dtype.
    ``batch``: (x_support [B,N,K,C,H,W], x_target [B,N,T,C,H,W], y_support [B,N,K], y_target [B,N,T]).
    """
    epoch = int(epoch)
    if current_epoch is None:
        current_epoch = epoch
    dtype = state[LIN_W].dtype
    xs, xt, ys, yt = batch
    xs, xt = xs.to(dtype), xt.to(dtype)
    ys, yt = ys.long(), yt.long()
    B = xs.shape[0]
    S_train = int(args.number_of_training_steps_per_iter)
    num_steps = S_train if training_phase else int(args.number_of_evaluation_steps_per_iter)
    second_order = bool(args.second_order) and epoch > args.first_order_to_second_order_epoch and training_phase
    sched = target_pass_schedule(args, epoch, training_phase, num_steps)
    w_msl = torch.from_numpy(msl_weights(args, current_epoch)).to(dtype)

    leaves = OrderedDict()
    for k, v in state.items():
        leaves[k] = v.detach().clone().requires_grad_(k in trainable_names(args))
    inner = inner_param_names(args)
    stats = []
    total_losses, all_correct, logits_out = [], [], []
    for b in range(B):
        fast = {n: leaves[n] for n in inner}
        x_s = xs[b].reshape(-1, *xs.shape[-3:])
        y_s = ys[b].reshape(-1)
        x_t = xt[b].reshape(-1, *xt.shape[-3:])
        y_t = yt[b].reshape(-1)
        task_losses = []
        last_logits = None
        for s in range(num_steps):
            logits_s = _net_forward(x_s, fast, leaves, args, s, stats)
            loss_s = F.cross_entropy(logits_s, y_s)
            grads = torch.autograd.grad(loss_s, [fast[n] for n in inner], create_graph=second_order,
                                        allow_unused=True)
            fast = {n: fast[n] - leaves[lslr_name(n)][s] * g for n, g in zip(inner, grads)}
            if sched[s] is not None:
                logits_t = _net_forward(x_t, fast, leaves, args, s, stats)
                loss_t = F.cross_entropy(logits_t, y_t)
                task_losses.append(w_msl[s] * loss_t if sched[s] == "msl" else loss_t)
                last_logits = logits_t
        logits_out.append(last_logits.detach())
        all_correct.append((last_logits.argmax(dim=1) == y_t).float())
        total_losses.append(torch.stack(task_losses).sum())
    loss = torch.stack(total_losses).mean()
    accuracy = float(torch.cat(all_correct).mean())
    out = {"loss": loss.detach(), "accuracy": accuracy, "logits": torch.stack(logits_out),
           "msl_weights": w_msl}
    if training_phase:
        names = trainable_names(args)
        gr = torch.autograd.grad(loss, [leaves[n] for n in names], allow_unused=True)
        out["grads"] = OrderedDict((n, (g if g is not None else torch.zeros_like(leaves[n])).detach())
                                   for n, g in zip(names, gr))
    # The reference's evaluation "backup" of the running statistics is copy(tensor.data): an ALIAS of the same storage
    # (meta_neural_network_architectures.py:240-242), so restore_backup_stats (:250-255) puts the mutated values back --
    # F.batch_norm's EMA side effect survives run_validation_iter.  Pinned by the val/ entries of the golden fixtures.
    out["running"] = apply_running_stats(state, args, stats)
    return out


def apply_running_stats(state, args, stats):
    """EMA side effect of F.batch_norm on ``running_*[num_step]`` in call order (reference
    meta_neural_network_architectures.py:226-247).  Shared-BN mode passes None => no update."""
    run = {k: v.detach().clone() for k, v in state.items() if "running" in k}
    if not args.per_step_bn_statistics:
        return run
    for (l, step, mu, var_unbiased) in stats:
        _, _, _, _, rmn, rvn = conv_names(l)
        run[rmn][step] = (1 - BN_MOMENTUM) * run[rmn][step] + BN_MOMENTUM * mu
        run[rvn][step] = (1 - BN_MOMENTUM) * run[rvn][step] + BN_MOMENTUM * var_unbiased
    return run


# ----------------------------------------------------------------------------------------
# outer step (clamp + Adam), reference few_shot_learning_system.py:325-336, :69
# ----------------------------------------------------------------------------------------
def adam_step(params, grads, exp_avg, exp_avg_sq, step, lr, clamp=None, betas=(0.9, 0.999), eps=1e-8):
    """torch.optim.Adam (no weight decay, no amsgrad) restated; all dicts name -> tensor.
    ``clamp``: iterable of names to clamp to [-10, 10] first (imagenet quirk :332-335)."""
    step = step + 1
    b1, b2 = betas
    bc1 = 1 - b1 ** step
    bc2 = 1 - b2 ** step
    new_p, new_m, new_v = {}, {}, {}
    for n, g in grads.items():
        g = g.clamp(-10, 10) if (clamp is not None and n in clamp) else g
        m = exp_avg[n] * b1 + (1 - b1) * g
        v = exp_avg_sq[n] * b2 + (1 - b2) * g * g
        denom = v.sqrt() / math.sqrt(bc2) + eps
        new_p[n] = params[n] - (lr / bc1) * m / denom
        new_m[n], new_v[n] = m, v
    return new_p, new_m, new_v, step


# ----------------------------------------------------------------------------------------
# restatement 2: autograd-free executable spec (SURVEY.md appendix A1-A4)
# ----------------------------------------------------------------------------------------
def _slope(y):
    return torch.where(y > 0, torch.ones_like(y), torch.full_like(y, LEAKY_SLOPE))


def block_forward(a_in, W, b, gamma, beta, forced=None):
    """A1.  Returns dict of everything later passes need.

    ``forced``: optional (slope, idx) -- the discrete decisions (leaky-ReLU branch per element, arg-max
    per pooling window) to USE instead of deriving them from y.  The network is piecewise smooth; with
    the decisions pinned, two implementations must agree to rounding error even when a pre-activation
    sits within an ulp of a branch point (tests/test_gpu_parity.py: decision-forced parity)."""
    z = F.conv2d(a_in, W, b, stride=1, padding=1)
    m = z.numel() // z.shape[1]
    mu = z.mean(dim=(0, 2, 3))
    zc = z - mu[None, :, None, None]
    v = (zc * zc).mean(dim=(0, 2, 3))
    r = (v + BN_EPS) ** -0.5
    zh = zc * r[None, :, None, None]
    y = gamma[None, :, None, None] * zh + beta[None, :, None, None]
    if forced is None:
        sl = _slope(y)
        a = y * sl
        p, idx = F.max_pool2d(a, 2, 2, return_indices=True)
    else:
        sl = forced[0].to(y.dtype)
        idx = forced[1]
        a = y * sl
        n, c = a.shape[:2]
        p = a.view(n, c, -1).gather(2, idx.view(n, c, -1)).view(n, c, *idx.shape[2:])
    return {"a_in": a_in, "zh": zh, "r": r, "mu": mu, "v": v, "m": m, "slope": sl, "idx": idx, "p": p, "y": y,
            "var_unbiased": v * (m / max(m - 1, 1))}


def _unpool(dp, idx, like):
    out = torch.zeros_like(like)
    n, c = like.shape[:2]
    out.view(n, c, -1).scatter_(2, idx.view(n, c, -1), dp.reshape(n, c, -1))
    return out


def block_backward(fw, W, gamma, dp, need_dgrad):
    """A2.  dp: grad w.r.t. pooled output.  Returns dW, db, dgamma, dbeta, da_in, + saved."""
    dy = _unpool(dp, fw["idx"], fw["zh"]) * fw["slope"]
    zh, r, m = fw["zh"], fw["r"], fw["m"]
    s1 = dy.sum(dim=(0, 2, 3))                 # = dbeta
    s2 = (dy * zh).sum(dim=(0, 2, 3))          # = dgamma
    g = gamma[None, :, None, None]
    dzh = dy * g
    m1 = (gamma * s1 / m)[None, :, None, None]
    m2 = (gamma * s2 / m)[None, :, None, None]
    dz = r[None, :, None, None] * (dzh - m1 - zh * m2)
    dW = torch.nn.grad.conv2d_weight(fw["a_in"], W.shape, dz, stride=1, padding=1)
    db = dz.sum(dim=(0, 2, 3))
    da_in = F.conv_transpose2d(dz, W, stride=1, padding=1) if need_dgrad else None
    return {"dW": dW, "db": db, "dgamma": s2, "dbeta": s1, "da_in": da_in, "dz": dz, "dy": dy,
            "dzh": dzh, "m1": m1, "m2": m2}


def head_forward(f, Wfc, bfc, y):
    logits = f @ Wfc.t() + bfc
    lse = torch.logsumexp(logits, dim=1)
    loss = (lse - logits.gather(1, y[:, None])[:, 0]).mean()
    prob = torch.softmax(logits, dim=1)
    return logits, loss, prob


def head_backward(f, Wfc, prob, y, scale=1.0):
    n = f.shape[0]
    dl = prob.clone()
    dl[torch.arange(n), y] -= 1.0
    dl = dl * (scale / n)
    return {"dl": dl, "dW": dl.t() @ f, "db": dl.sum(0), "df": dl @ Wfc}


def net_forward_manual(x, theta, state, args, step, y, forced=None):
    """theta: dict name->tensor for the fast tensors.  forced: optional per-block (slope, idx)."""
    fws = []
    a = x
    for l in range(num_stages(args)):
        wn, bn_, _, _, _, _ = conv_names(l)
        g, b = _bn_params(state, theta, args, l, step)
        fw = block_forward(a, theta[wn], theta[bn_], g, b, None if forced is None else forced[l])
        fws.append(fw)
        a = fw["p"]
    f = a.reshape(a.shape[0], -1)
    logits, loss, prob = head_forward(f, theta[LIN_W], theta[LIN_B], y)
    return {"blocks": fws, "f": f, "logits": logits, "loss": loss, "prob": prob}


def net_backward_manual(fwd, theta, state, args, step, y, scale=1.0):
    """Gradient of scale*loss w.r.t. the fast tensors and gamma/beta: beta's is S1 = sum dy, gamma's S2 = sum dy * zh
    per channel, among the fast tensors' with inner-loop gamma / beta, else in ``bn_grads`` (the step's)."""
    hb = head_backward(fwd["f"], theta[LIN_W], fwd["prob"], y, scale)
    grads = {LIN_W: hb["dW"], LIN_B: hb["db"]}
    bn_grads = {}
    saved = [None] * num_stages(args)
    dp = hb["df"].reshape(fwd["blocks"][-1]["p"].shape)
    for l in reversed(range(num_stages(args))):
        wn, bn_, gn, btn, _, _ = conv_names(l)
        g, _ = _bn_params(state, theta, args, l, step)
        bw = block_backward(fwd["blocks"][l], theta[wn], g, dp, need_dgrad=(l > 0))
        grads[wn], grads[bn_] = bw["dW"], bw["db"]
        gb_grads = grads if args.enable_inner_loop_optimizable_bn_params else bn_grads
        gb_grads[gn], gb_grads[btn] = bw["dgamma"], bw["dbeta"]
        saved[l] = dict(bw, dp=dp)
        dp = bw["da_in"]
    return grads, bn_grads, {"head": hb, "blocks": saved}


def tangent_pass(fwd, bwd_saved, theta, u, state, args, step, y):
    """A3: forward-mode derivative of (support forward + support backward) in direction u
    (dict over the fast tensors).  Returns (Hu dict, mixed second-derivative terms on this
    step's gamma / beta, intermediates).  Shared gamma / beta have no tangents.  Inner-loop
    gamma / beta have tangents (gdot, bdot) in u, and with dzh = gamma * dy:
      ydot   = gamma * zhdot + gdot * zh + bdot
      dzhdot = gamma * dydot + gdot * dy
    so dzdot gains r gdot (dy - S1/m - zh S2/m); their sums T1 = sum dydot (beta), T2 =
    sum dydot zh + dy zhdot (gamma) are then Hu's, and there are no mixed terms."""
    inner_bn = args.enable_inner_loop_optimizable_bn_params
    L = num_stages(args)
    tf = []
    a_dot = None
    for l in range(L):
        wn, bn_, gn, btn, _, _ = conv_names(l)
        fw = fwd["blocks"][l]
        g, _ = _bn_params(state, theta, args, l, step)
        z_dot = F.conv2d(fw["a_in"], u[wn], u[bn_], stride=1, padding=1)
        if a_dot is not None:
            z_dot = z_dot + F.conv2d(a_dot, theta[wn], None, stride=1, padding=1)
        zh, r = fw["zh"], fw["r"]
        mu_dot = z_dot.mean(dim=(0, 2, 3))[None, :, None, None]
        q = (zh * z_dot).mean(dim=(0, 2, 3))                      # mean(zh * z_dot)
        zh_dot = r[None, :, None, None] * (z_dot - mu_dot - zh * q[None, :, None, None])
        y_dot = g[None, :, None, None] * zh_dot
        if inner_bn:
            y_dot = y_dot + u[gn][None, :, None, None] * zh + u[btn][None, :, None, None]
        a_dot_full = y_dot * fw["slope"]
        n, c = a_dot_full.shape[:2]
        p_dot = a_dot_full.view(n, c, -1).gather(2, fw["idx"].view(n, c, -1)).view(fw["p"].shape)
        tf.append({"zh_dot": zh_dot, "q": q, "p_dot": p_dot, "a_in_dot": a_dot, "z_dot": z_dot})
        a_dot = p_dot
    f, prob = fwd["f"], fwd["prob"]
    f_dot = a_dot.reshape(f.shape)
    n = f.shape[0]
    l_dot = f_dot @ theta[LIN_W].t() + f @ u[LIN_W].t() + u[LIN_B]
    dl = bwd_saved["head"]["dl"]
    dl_dot = (prob * l_dot - prob * (prob * l_dot).sum(dim=1, keepdim=True)) / n
    Hu = {LIN_W: dl_dot.t() @ f + dl.t() @ f_dot, LIN_B: dl_dot.sum(0)}
    df_dot = dl_dot @ theta[LIN_W] + dl @ u[LIN_W]
    mixed = {}
    tb = [None] * L
    dp_dot = df_dot.reshape(fwd["blocks"][-1]["p"].shape)
    for l in reversed(range(L)):
        wn, bn_, gn, btn, _, _ = conv_names(l)
        fw, bw, t = fwd["blocks"][l], bwd_saved["blocks"][l], tf[l]
        g, _ = _bn_params(state, theta, args, l, step)
        gg = g[None, :, None, None]
        zh, r, m = fw["zh"], fw["r"], fw["m"]
        dy_dot = _unpool(dp_dot, fw["idx"], zh) * fw["slope"]
        dbeta_dot = dy_dot.sum(dim=(0, 2, 3))
        dgamma_dot = (dy_dot * zh + bw["dy"] * t["zh_dot"]).sum(dim=(0, 2, 3))
        dzh_dot = dy_dot * gg
        if inner_bn:
            dzh_dot = dzh_dot + bw["dy"] * u[gn][None, :, None, None]
        m1_dot = dzh_dot.mean(dim=(0, 2, 3))[None, :, None, None]
        m2_dot = (dzh_dot * zh + bw["dzh"] * t["zh_dot"]).mean(dim=(0, 2, 3))[None, :, None, None]
        r_dot_over_r = (-r * t["q"])[None, :, None, None]          # r_dot = -r^2 q
        dz_dot = r_dot_over_r * bw["dz"] + r[None, :, None, None] * (
            dzh_dot - m1_dot - t["zh_dot"] * bw["m2"] - zh * m2_dot)
        W = theta[wn]
        dW_dot = torch.nn.grad.conv2d_weight(fw["a_in"], W.shape, dz_dot, stride=1, padding=1)
        if t["a_in_dot"] is not None:
            dW_dot = dW_dot + torch.nn.grad.conv2d_weight(t["a_in_dot"], W.shape, bw["dz"], stride=1, padding=1)
        Hu[wn] = dW_dot
        Hu[bn_] = dz_dot.sum(dim=(0, 2, 3))
        gb_dot = Hu if inner_bn else mixed
        gb_dot[gn], gb_dot[btn] = dgamma_dot, dbeta_dot
        tb[l] = {"dz_dot": dz_dot, "dp_dot": dp_dot, "dy_dot": dy_dot}
        if l > 0:
            dp_dot = F.conv_transpose2d(dz_dot, W, stride=1, padding=1) + \
                F.conv_transpose2d(bw["dz"], u[wn], stride=1, padding=1)
    return Hu, mixed, {"fwd": tf, "bwd": tb, "l_dot": l_dot, "dl_dot": dl_dot}


def manual_train_iter(state, args, batch, epoch, training_phase=True, current_epoch=None,
                      keep_intermediates=False, decisions=None):
    """A4.  Same contract as ``autograd_train_iter`` (plus ``intermediates`` when asked).
    ``decisions``: optional {(task, "sup"|"tgt", step): [per-block (slope, idx)]} to pin the discrete
    choices of every pass (see ``block_forward``)."""
    epoch = int(epoch)
    if current_epoch is None:
        current_epoch = epoch
    dtype = state[LIN_W].dtype
    xs, xt, ys, yt = batch
    xs, xt = xs.to(dtype), xt.to(dtype)
    ys, yt = ys.long(), yt.long()
    B = xs.shape[0]
    S_train = int(args.number_of_training_steps_per_iter)
    num_steps = S_train if training_phase else int(args.number_of_evaluation_steps_per_iter)
    second_order = bool(args.second_order) and epoch > args.first_order_to_second_order_epoch and training_phase
    sched = target_pass_schedule(args, epoch, training_phase, num_steps)
    w_msl = torch.from_numpy(msl_weights(args, current_epoch)).to(dtype)
    inner = inner_param_names(args)
    per_step = bool(args.per_step_bn_statistics)

    outer = OrderedDict((n, torch.zeros_like(state[n])) for n in state if "running" not in n)
    stats = []
    losses, corrects, logits_out, inter = [], [], [], []
    with torch.no_grad():
        for b in range(B):
            x_s = xs[b].reshape(-1, *xs.shape[-3:]); y_s = ys[b].reshape(-1)
            x_t = xt[b].reshape(-1, *xt.shape[-3:]); y_t = yt[b].reshape(-1)
            theta = [{n: state[n] for n in inner}]
            sup_f, sup_b, sup_g, tgt_f = [], [], [], []
            task_loss = torch.zeros((), dtype=dtype)
            last_logits = None
            # ---- phase A: unroll
            for s in range(num_steps):
                fwd = net_forward_manual(x_s, theta[s], state, args, s, y_s,
                                         None if decisions is None else decisions[(b, "sup", s)])
                for l, fw in enumerate(fwd["blocks"]):
                    stats.append((l, s, fw["mu"], fw["var_unbiased"]))
                g, _, saved = net_backward_manual(fwd, theta[s], state, args, s, y_s)
                sup_f.append(fwd); sup_b.append(saved); sup_g.append(g)
                theta.append({n: theta[s][n] - state[lslr_name(n)][s] * g[n] for n in inner})
                if sched[s] is not None:
                    tf_ = net_forward_manual(x_t, theta[s + 1], state, args, s, y_t,
                                             None if decisions is None else decisions[(b, "tgt", s)])
                    for l, fw in enumerate(tf_["blocks"]):
                        stats.append((l, s, fw["mu"], fw["var_unbiased"]))
                    wgt = w_msl[s] if sched[s] == "msl" else torch.ones((), dtype=dtype)
                    task_loss = task_loss + wgt * tf_["loss"]
                    tgt_f.append((tf_, wgt))
                    last_logits = tf_["logits"]
                else:
                    tgt_f.append(None)
            losses.append(task_loss)
            logits_out.append(last_logits)
            corrects.append((last_logits.argmax(dim=1) == y_t).float())
            if not training_phase:
                continue
            # ---- phase B: reverse sweep
            tbar = {n: torch.zeros_like(state[n]) for n in inner}
            tgt_b, tgt_g = [None] * num_steps, [None] * num_steps
            for s in reversed(range(num_steps)):
                if tgt_f[s] is not None:
                    tf_, wgt = tgt_f[s]
                    tg, tbn, tsaved = net_backward_manual(tf_, theta[s + 1], state, args, s, y_t, scale=float(wgt))
                    tgt_b[s], tgt_g[s] = tsaved, tg
                    for n in inner:
                        tbar[n] = tbar[n] + tg[n]
                    for n, gval in tbn.items():
                        if per_step:
                            outer[n][s] += gval
                        else:
                            outer[n] += gval
                for n in inner:
                    outer[lslr_name(n)][s] += -(tbar[n] * sup_g[s][n]).sum()
                if keep_intermediates and s == 0:
                    tbar_before0 = dict(tbar)
                if second_order:
                    u = {n: state[lslr_name(n)][s] * tbar[n] for n in inner}
                    Hu, mixed, tint = tangent_pass(sup_f[s], sup_b[s], theta[s], u, state, args, s, y_s)
                    for n in inner:
                        tbar[n] = tbar[n] - Hu[n]
                    for n, gval in mixed.items():
                        if per_step:
                            outer[n][s] -= gval
                        else:
                            outer[n] -= gval
                    if keep_intermediates:
                        inter.append({"task": b, "step": s, "u": u, "Hu": Hu, "mixed": mixed, "tangent": tint})
            for n in inner:
                outer[n] += tbar[n]
            if keep_intermediates:
                # tgt_b / tgt_g: the target backward records and the weighted target gradients per step (None where
                # the step has no target pass); tbar0: theta-bar before step 0's Hessian term, tbar: after it
                inter.append({"task": b, "theta": theta, "sup_f": sup_f, "sup_b": sup_b, "sup_g": sup_g,
                              "tgt_f": tgt_f, "tgt_b": tgt_b, "tgt_g": tgt_g, "tbar0": tbar_before0, "tbar": dict(tbar)})
    loss = torch.stack(losses).mean()
    out = {"loss": loss, "accuracy": float(torch.cat(corrects).mean()), "logits": torch.stack(logits_out),
           "msl_weights": w_msl}
    if training_phase:
        names = trainable_names(args)
        out["grads"] = OrderedDict((n, outer[n] / B) for n in names)
    out["running"] = apply_running_stats(state, args, stats)     # evaluation too: see autograd_train_iter
    if keep_intermediates:
        out["intermediates"] = inter
    return out


# ----------------------------------------------------------------------------------------
# synthetic episodes (SURVEY.md section 8d / BASELINE.md section 4)
# ----------------------------------------------------------------------------------------
def synthetic_batch(args, iteration=0, batch_size=None, kind=None):
    """Seeded synthetic episodes with the reference's batch layout.
    Omniglot-shaped (C=1): Bernoulli(0.93) in {0,1}; otherwise N(0,1).  Labels y[b,c,:]=c."""
    B = int(batch_size if batch_size is not None else args.batch_size)
    N, K, T = int(args.num_classes_per_set), int(args.num_samples_per_class), int(args.num_target_samples)
    C, H, W = int(args.image_channels), int(args.image_height), int(args.image_width)
    gen = torch.Generator().manual_seed(1234 + int(iteration))
    if kind is None:
        kind = "bernoulli" if C == 1 else "normal"
    if kind == "bernoulli":
        xs = (torch.rand(B, N, K, C, H, W, generator=gen) < 0.93).float()
        xt = (torch.rand(B, N, T, C, H, W, generator=gen) < 0.93).float()
    else:
        xs = torch.randn(B, N, K, C, H, W, generator=gen)
        xt = torch.randn(B, N, T, C, H, W, generator=gen)
    ys = torch.arange(N).view(1, N, 1).expand(B, N, K).contiguous().float()
    yt = torch.arange(N).view(1, N, 1).expand(B, N, T).contiguous().float()
    return xs, xt, ys, yt
