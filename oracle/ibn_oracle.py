"""ORACLE TOOLING -- TEST INFRASTRUCTURE ONLY.  fp64 restatement of the reference's MAML / MAML++ iteration with
``enable_inner_loop_optimizable_bn_params``: each block's BatchNorm bias (beta) and weight (gamma) are [F] tensors that
join the inner loop (reference meta_neural_network_architectures.py:194-198, few_shot_learning_system.py:105-120).  They
are updated per task by the LSLR rule with their own rate vectors, enter the support gradient of every step (second order
through ``create_graph``), and the network's forward reads them from the fast weights without a step index (:229-234).
The running statistics keep their per-step rows.  Everything else is ``oracle/maml_oracle.py``'s."""
from collections import OrderedDict

import torch
import torch.nn.functional as F

from oracle import maml_oracle as O


def inner_param_names(args):
    """The adaptable tensors in the reference's inner-loop order: per block conv.weight, conv.bias, norm_layer.bias,
    norm_layer.weight; then the linear layer."""
    names = []
    for l in range(O.num_stages(args)):
        wn, bn_, gn, btn, _, _ = O.conv_names(l)
        names += [wn, bn_, btn, gn]
    return names + [O.LIN_W, O.LIN_B]


def trainable_names(args):
    """Outer (Adam) parameter order: the module's trainable parameters, then one LSLR vector per inner tensor."""
    names = list(inner_param_names(args))
    if args.learnable_per_layer_per_step_inner_loop_learning_rate:
        names += [O.lslr_name(n) for n in inner_param_names(args)]
    return names


def _net_forward(x, fast, args, step, stats_out=None):
    out = x
    for l in range(O.num_stages(args)):
        wn, bn_, gn, btn, _, _ = O.conv_names(l)
        out = F.conv2d(out, fast[wn], fast[bn_], stride=1, padding=1)
        if stats_out is not None:
            with torch.no_grad():
                m = out.numel() // out.shape[1]
                mu = out.mean(dim=(0, 2, 3))
                var_unbiased = out.var(dim=(0, 2, 3), unbiased=True) if m > 1 else out.new_zeros(out.shape[1])
                stats_out.append((l, step, mu, var_unbiased))
        out = F.batch_norm(out, None, None, fast[gn], fast[btn], training=True, momentum=O.BN_MOMENTUM, eps=O.BN_EPS)
        out = F.leaky_relu(out)
        out = F.max_pool2d(out, kernel_size=(2, 2), stride=2, padding=0)
    out = out.reshape(out.shape[0], -1)
    return F.linear(out, fast[O.LIN_W], fast[O.LIN_B])


def autograd_train_iter(state, args, batch, epoch, training_phase=True, current_epoch=None):
    """``maml_oracle.autograd_train_iter`` with gamma / beta as fast weights: loss, accuracy, last-step logits, the outer
    gradients of ``trainable_names`` and the updated running statistics."""
    epoch = int(epoch)
    if current_epoch is None:
        current_epoch = epoch
    dtype = state[O.LIN_W].dtype
    xs, xt, ys, yt = batch
    xs, xt = xs.to(dtype), xt.to(dtype)
    ys, yt = ys.long(), yt.long()
    num_steps = int(args.number_of_training_steps_per_iter) if training_phase else int(args.number_of_evaluation_steps_per_iter)
    second_order = bool(args.second_order) and epoch > args.first_order_to_second_order_epoch and training_phase
    sched = O.target_pass_schedule(args, epoch, training_phase, num_steps)
    w_msl = torch.from_numpy(O.msl_weights(args, current_epoch)).to(dtype)
    names = trainable_names(args)
    leaves = OrderedDict((k, v.detach().clone().requires_grad_(k in names)) for k, v in state.items())
    inner = inner_param_names(args)
    stats, total_losses, all_correct, logits_out = [], [], [], []
    for b in range(xs.shape[0]):
        fast = {n: leaves[n] for n in inner}
        x_s, y_s = xs[b].reshape(-1, *xs.shape[-3:]), ys[b].reshape(-1)
        x_t, y_t = xt[b].reshape(-1, *xt.shape[-3:]), yt[b].reshape(-1)
        task_losses, last_logits = [], None
        for s in range(num_steps):
            loss_s = F.cross_entropy(_net_forward(x_s, fast, args, s, stats), y_s)
            grads = torch.autograd.grad(loss_s, [fast[n] for n in inner], create_graph=second_order)
            fast = {n: fast[n] - leaves[O.lslr_name(n)][s] * g for n, g in zip(inner, grads)}
            if sched[s] is not None:
                logits_t = _net_forward(x_t, fast, args, s, stats)
                loss_t = F.cross_entropy(logits_t, y_t)
                task_losses.append(w_msl[s] * loss_t if sched[s] == "msl" else loss_t)
                last_logits = logits_t
        logits_out.append(last_logits.detach())
        all_correct.append((last_logits.argmax(dim=1) == y_t).float())
        total_losses.append(torch.stack(task_losses).sum())
    loss = torch.stack(total_losses).mean()
    out = {"loss": loss.detach(), "accuracy": float(torch.cat(all_correct).mean()), "logits": torch.stack(logits_out),
           "msl_weights": w_msl}
    if training_phase:
        gr = torch.autograd.grad(loss, [leaves[n] for n in names], allow_unused=True)
        out["grads"] = OrderedDict((n, (g if g is not None else torch.zeros_like(leaves[n])).detach())
                                   for n, g in zip(names, gr))
    out["running"] = O.apply_running_stats(state, args, stats)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# Autograd-free restatement (the kernels' formulas, as maml_oracle's manual_train_iter / tangent_pass), with gamma / beta
# read from the fast weights theta of the pass and their tangents from the direction u.
# ----------------------------------------------------------------------------------------------------------------------
def net_forward_manual(x, theta, args, y, forced=None):
    """theta: the fast tensors (gamma / beta included).  forced: optional per-block (slope, idx)."""
    fws, a = [], x
    for l in range(O.num_stages(args)):
        wn, bn_, gn, btn, _, _ = O.conv_names(l)
        fw = O.block_forward(a, theta[wn], theta[bn_], theta[gn], theta[btn], None if forced is None else forced[l])
        fws.append(fw)
        a = fw["p"]
    f = a.reshape(a.shape[0], -1)
    logits, loss, prob = O.head_forward(f, theta[O.LIN_W], theta[O.LIN_B], y)
    return {"blocks": fws, "f": f, "logits": logits, "loss": loss, "prob": prob}


def net_backward_manual(fwd, theta, args, y, scale=1.0):
    """Gradient of scale * loss w.r.t. every fast tensor: conv / linear as usual, beta = S1 = sum dy, gamma = S2 =
    sum dy * zh per channel."""
    hb = O.head_backward(fwd["f"], theta[O.LIN_W], fwd["prob"], y, scale)
    grads = {O.LIN_W: hb["dW"], O.LIN_B: hb["db"]}
    saved = [None] * O.num_stages(args)
    dp = hb["df"].reshape(fwd["blocks"][-1]["p"].shape)
    for l in reversed(range(O.num_stages(args))):
        wn, bn_, gn, btn, _, _ = O.conv_names(l)
        bw = O.block_backward(fwd["blocks"][l], theta[wn], theta[gn], dp, need_dgrad=(l > 0))
        grads[wn], grads[bn_], grads[gn], grads[btn] = bw["dW"], bw["db"], bw["dgamma"], bw["dbeta"]
        saved[l] = dict(bw, dp=dp)
        dp = bw["da_in"]
    return grads, {"head": hb, "blocks": saved}


def tangent_pass(fwd, bwd_saved, theta, u, args, y):
    """Forward-mode derivative of (support forward + support backward) along u, which has gamma / beta directions
    (gdot, bdot) too.  Returns (Hu over every fast tensor, intermediates).  Per block, with dzh = gamma * dy:
      ydot   = gamma * zhdot + gdot * zh + bdot
      dzhdot = gamma * dydot + gdot * dy
      dzdot  = -r q dz + r (dzhdot - mean(dzhdot) - zhdot * mean(dzh * zh) - zh * mean(dzhdot * zh + dzh * zhdot)),
    whose gdot part is r gdot (dy - S1/m - zh S2/m); Hu_beta = T1 = sum dydot, Hu_gamma = T2 = sum dydot zh + dy zhdot."""
    L = O.num_stages(args)
    tf, a_dot = [], None
    for l in range(L):
        wn, bn_, gn, btn, _, _ = O.conv_names(l)
        fw = fwd["blocks"][l]
        z_dot = F.conv2d(fw["a_in"], u[wn], u[bn_], stride=1, padding=1)
        if a_dot is not None:
            z_dot = z_dot + F.conv2d(a_dot, theta[wn], None, stride=1, padding=1)
        zh, r = fw["zh"], fw["r"]
        mu_dot = z_dot.mean(dim=(0, 2, 3))[None, :, None, None]
        q = (zh * z_dot).mean(dim=(0, 2, 3))
        zh_dot = r[None, :, None, None] * (z_dot - mu_dot - zh * q[None, :, None, None])
        y_dot = theta[gn][None, :, None, None] * zh_dot + u[gn][None, :, None, None] * zh + u[btn][None, :, None, None]
        a_dot_full = y_dot * fw["slope"]
        n, c = a_dot_full.shape[:2]
        p_dot = a_dot_full.view(n, c, -1).gather(2, fw["idx"].view(n, c, -1)).view(fw["p"].shape)
        tf.append({"zh_dot": zh_dot, "q": q, "p_dot": p_dot, "a_in_dot": a_dot, "z_dot": z_dot})
        a_dot = p_dot
    f, prob = fwd["f"], fwd["prob"]
    f_dot = a_dot.reshape(f.shape)
    n = f.shape[0]
    l_dot = f_dot @ theta[O.LIN_W].t() + f @ u[O.LIN_W].t() + u[O.LIN_B]
    dl = bwd_saved["head"]["dl"]
    dl_dot = (prob * l_dot - prob * (prob * l_dot).sum(dim=1, keepdim=True)) / n
    Hu = {O.LIN_W: dl_dot.t() @ f + dl.t() @ f_dot, O.LIN_B: dl_dot.sum(0)}
    df_dot = dl_dot @ theta[O.LIN_W] + dl @ u[O.LIN_W]
    tb = [None] * L
    dp_dot = df_dot.reshape(fwd["blocks"][-1]["p"].shape)
    for l in reversed(range(L)):
        wn, bn_, gn, btn, _, _ = O.conv_names(l)
        fw, bw, t = fwd["blocks"][l], bwd_saved["blocks"][l], tf[l]
        gg, gd = theta[gn][None, :, None, None], u[gn][None, :, None, None]
        zh, r = fw["zh"], fw["r"]
        dy_dot = O._unpool(dp_dot, fw["idx"], zh) * fw["slope"]
        dzh_dot = dy_dot * gg + bw["dy"] * gd
        m1_dot = dzh_dot.mean(dim=(0, 2, 3))[None, :, None, None]
        m2_dot = (dzh_dot * zh + bw["dzh"] * t["zh_dot"]).mean(dim=(0, 2, 3))[None, :, None, None]
        dz_dot = (-r * t["q"])[None, :, None, None] * bw["dz"] + r[None, :, None, None] * (
            dzh_dot - m1_dot - t["zh_dot"] * bw["m2"] - zh * m2_dot)
        W = theta[wn]
        dW_dot = torch.nn.grad.conv2d_weight(fw["a_in"], W.shape, dz_dot, stride=1, padding=1)
        if t["a_in_dot"] is not None:
            dW_dot = dW_dot + torch.nn.grad.conv2d_weight(t["a_in_dot"], W.shape, bw["dz"], stride=1, padding=1)
        Hu[wn], Hu[bn_] = dW_dot, dz_dot.sum(dim=(0, 2, 3))
        Hu[btn] = dy_dot.sum(dim=(0, 2, 3))
        Hu[gn] = (dy_dot * zh + bw["dy"] * t["zh_dot"]).sum(dim=(0, 2, 3))
        tb[l] = {"dz_dot": dz_dot, "dp_dot": dp_dot, "dy_dot": dy_dot}
        if l > 0:
            dp_dot = F.conv_transpose2d(dz_dot, W, stride=1, padding=1) + \
                F.conv_transpose2d(bw["dz"], u[wn], stride=1, padding=1)
    return Hu, {"fwd": tf, "bwd": tb, "l_dot": l_dot, "dl_dot": dl_dot}


def manual_train_iter(state, args, batch, epoch, training_phase=True, current_epoch=None, keep_intermediates=False,
                      decisions=None):
    """``autograd_train_iter``'s contract, autograd-free (plus ``intermediates`` when asked).  ``decisions``: optional
    {(task, "sup"|"tgt", step): [per-block (slope, idx)]} pinning the discrete choices of every pass.  Intermediates per
    task: theta^s, the support passes and gradients g_s, the target passes and tgrad[s], theta-bar before / after step 0's
    Hessian term; per (task, step) of the sweep: u and Hu and the tangent pass."""
    epoch = int(epoch)
    if current_epoch is None:
        current_epoch = epoch
    dtype = state[O.LIN_W].dtype
    xs, xt, ys, yt = batch
    xs, xt = xs.to(dtype), xt.to(dtype)
    ys, yt = ys.long(), yt.long()
    B = xs.shape[0]
    num_steps = int(args.number_of_training_steps_per_iter) if training_phase else int(args.number_of_evaluation_steps_per_iter)
    second_order = bool(args.second_order) and epoch > args.first_order_to_second_order_epoch and training_phase
    sched = O.target_pass_schedule(args, epoch, training_phase, num_steps)
    w_msl = torch.from_numpy(O.msl_weights(args, current_epoch)).to(dtype)
    inner = inner_param_names(args)
    outer = OrderedDict((n, torch.zeros_like(state[n])) for n in state if "running" not in n)
    stats, losses, corrects, logits_out, inter = [], [], [], [], []
    with torch.no_grad():
        for b in range(B):
            x_s, y_s = xs[b].reshape(-1, *xs.shape[-3:]), ys[b].reshape(-1)
            x_t, y_t = xt[b].reshape(-1, *xt.shape[-3:]), yt[b].reshape(-1)
            theta = [{n: state[n] for n in inner}]
            sup_f, sup_b, sup_g, tgt_f = [], [], [], []
            task_loss, last_logits = torch.zeros((), dtype=dtype), None
            for s in range(num_steps):
                fwd = net_forward_manual(x_s, theta[s], args, y_s, None if decisions is None else decisions[(b, "sup", s)])
                for l, fw in enumerate(fwd["blocks"]):
                    stats.append((l, s, fw["mu"], fw["var_unbiased"]))
                g, saved = net_backward_manual(fwd, theta[s], args, y_s)
                sup_f.append(fwd); sup_b.append(saved); sup_g.append(g)
                theta.append({n: theta[s][n] - state[O.lslr_name(n)][s] * g[n] for n in inner})
                if sched[s] is not None:
                    tf_ = net_forward_manual(x_t, theta[s + 1], args, y_t,
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
            tbar = {n: torch.zeros_like(state[n]) for n in inner}
            tgt_b, tgt_g, tbar0 = [None] * num_steps, [None] * num_steps, None
            for s in reversed(range(num_steps)):
                if tgt_f[s] is not None:
                    tf_, wgt = tgt_f[s]
                    tg, tsaved = net_backward_manual(tf_, theta[s + 1], args, y_t, scale=float(wgt))
                    tgt_b[s], tgt_g[s] = tsaved, tg
                    for n in inner:
                        tbar[n] = tbar[n] + tg[n]
                for n in inner:
                    outer[O.lslr_name(n)][s] += -(tbar[n] * sup_g[s][n]).sum()
                if s == 0:
                    tbar0 = dict(tbar)
                if second_order:
                    u = {n: state[O.lslr_name(n)][s] * tbar[n] for n in inner}
                    Hu, tint = tangent_pass(sup_f[s], sup_b[s], theta[s], u, args, y_s)
                    for n in inner:
                        tbar[n] = tbar[n] - Hu[n]
                    if keep_intermediates:
                        inter.append({"task": b, "step": s, "u": u, "Hu": Hu, "tangent": tint})
            for n in inner:
                outer[n] += tbar[n]
            if keep_intermediates:
                inter.append({"task": b, "theta": theta, "sup_f": sup_f, "sup_b": sup_b, "sup_g": sup_g, "tgt_f": tgt_f,
                              "tgt_b": tgt_b, "tgt_g": tgt_g, "tbar0": tbar0, "tbar": dict(tbar)})
    out = {"loss": torch.stack(losses).mean(), "accuracy": float(torch.cat(corrects).mean()),
           "logits": torch.stack(logits_out), "msl_weights": w_msl}
    if training_phase:
        out["grads"] = OrderedDict((n, outer[n] / B) for n in trainable_names(args))
    out["running"] = O.apply_running_stats(state, args, stats)
    if keep_intermediates:
        out["intermediates"] = inter
    return out
