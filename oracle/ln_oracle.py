"""fp64 / fp32 restatement of the reference's LAYER-NORM network (``norm_layer: "layer_norm"``) -- test infrastructure.

The reference's ``MetaLayerNormLayer`` (meta_neural_network_architectures.py:261-322) runs ``F.layer_norm`` over the conv
output [F, h, w] of each image (the size before pooling), eps 1e-5, with a frozen all-ones ``weight`` and a learnable
``bias`` [F, h, w].  The layer has no running statistics and ignores ``num_step``; ``get_inner_loop_parameter_dict``
(few_shot_learning_system.py:111-120) leaves it out of the inner loop, so the bias is an outer (Adam) parameter only.
Everything else -- schedules, LSLR, multi-step loss, second order -- is ``maml_oracle``'s, reused here.
"""
from collections import OrderedDict

import torch
import torch.nn.functional as F

from oracle import maml_oracle as O

LN_EPS = 1e-5
_moved_state = O.moved_state


def trainable_names(args):
    """Outer (Adam) parameter order of the layer-norm network: per block conv.weight, conv.bias, norm_layer.bias (the
    frozen weight has requires_grad=False), then the linear layer and the LSLR vectors."""
    names = []
    for l in range(O.num_stages(args)):
        wn, bn_, _, btn, _, _ = O.conv_names(l)
        names += [wn, bn_, btn]
    names += [O.LIN_W, O.LIN_B]
    if args.learnable_per_layer_per_step_inner_loop_learning_rate:
        names += [O.lslr_name(n) for n in O.inner_param_names(args)]
    return names


def state_keys(args):
    """``state_dict`` keys of the layer-norm network in registration order (no running statistics)."""
    keys = []
    for l in range(O.num_stages(args)):
        wn, bn_, gn, btn, _, _ = O.conv_names(l)
        keys += [wn, bn_, gn, btn]
    keys += [O.LIN_W, O.LIN_B]
    keys += [O.lslr_name(n) for n in O.inner_param_names(args)]
    return keys


def moved_state(state, args, seed):
    """``maml_oracle.moved_state`` for the layer-norm network: the bias [F, h, w] ~ 0.2 N(0, 1), conv / linear biases and
    LSLR rates moved as there; the frozen weight stays all ones (the reference never changes it).  At the initial zero
    bias a kernel that drops the bias or reads it at the wrong position computes the right numbers; here it does not."""
    out = _moved_state(state, args, seed)
    for k in out:
        if k.endswith("norm_layer.weight"):
            out[k] = torch.ones_like(state[k])
    return out


def _net_forward(x, fast, state, args):
    out = x
    for l in range(O.num_stages(args)):
        wn, bn_, gn, btn, _, _ = O.conv_names(l)
        out = F.conv2d(out, fast[wn], fast[bn_], stride=1, padding=1)
        out = F.layer_norm(out, out.shape[1:], state[gn], state[btn], LN_EPS)
        out = F.leaky_relu(out)
        out = F.max_pool2d(out, kernel_size=(2, 2), stride=2, padding=0)
    out = out.reshape(out.shape[0], -1)
    return F.linear(out, fast[O.LIN_W], fast[O.LIN_B])


def logits(state, args, x, fast=None):
    """Logits of a batch of images x [n, C, H, W] under ``state`` (``fast``: optional inner-parameter overrides)."""
    fast = dict(fast or {})
    for n in O.inner_param_names(args):
        fast.setdefault(n, state[n])
    return _net_forward(x.to(state[O.LIN_W].dtype), fast, state, args)


def autograd_train_iter(state, args, batch, epoch, training_phase=True, current_epoch=None):
    """``maml_oracle.autograd_train_iter`` with the layer-norm network: loss, accuracy, per-task last-step logits and the
    outer gradients of ``trainable_names`` (training).  No running statistics."""
    epoch = int(epoch)
    if current_epoch is None:
        current_epoch = epoch
    dtype = state[O.LIN_W].dtype
    xs, xt, ys, yt = batch
    xs, xt = xs.to(dtype), xt.to(dtype)
    ys, yt = ys.long(), yt.long()
    S_train = int(args.number_of_training_steps_per_iter)
    num_steps = S_train if training_phase else int(args.number_of_evaluation_steps_per_iter)
    second_order = bool(args.second_order) and epoch > args.first_order_to_second_order_epoch and training_phase
    sched = O.target_pass_schedule(args, epoch, training_phase, num_steps)
    w_msl = torch.from_numpy(O.msl_weights(args, current_epoch)).to(dtype)
    names = trainable_names(args)
    leaves = OrderedDict((k, v.detach().clone().requires_grad_(k in names)) for k, v in state.items())
    inner = O.inner_param_names(args)
    total_losses, all_correct, logits_out = [], [], []
    for b in range(xs.shape[0]):
        fast = {n: leaves[n] for n in inner}
        x_s, y_s = xs[b].reshape(-1, *xs.shape[-3:]), ys[b].reshape(-1)
        x_t, y_t = xt[b].reshape(-1, *xt.shape[-3:]), yt[b].reshape(-1)
        task_losses, last = [], None
        for s in range(num_steps):
            loss_s = F.cross_entropy(_net_forward(x_s, fast, leaves, args), y_s)
            grads = torch.autograd.grad(loss_s, [fast[n] for n in inner], create_graph=second_order, allow_unused=True)
            fast = {n: fast[n] - leaves[O.lslr_name(n)][s] * g for n, g in zip(inner, grads)}
            if sched[s] is not None:
                last = _net_forward(x_t, fast, leaves, args)
                loss_t = F.cross_entropy(last, y_t)
                task_losses.append(w_msl[s] * loss_t if sched[s] == "msl" else loss_t)
        logits_out.append(last.detach())
        all_correct.append((last.argmax(dim=1) == y_t).float())
        total_losses.append(torch.stack(task_losses).sum())
    loss = torch.stack(total_losses).mean()
    out = {"loss": loss.detach(), "accuracy": float(torch.cat(all_correct).mean()), "logits": torch.stack(logits_out)}
    if training_phase:
        gr = torch.autograd.grad(loss, [leaves[n] for n in names], allow_unused=True)
        out["grads"] = OrderedDict((n, (g if g is not None else torch.zeros_like(leaves[n])).detach())
                                   for n, g in zip(names, gr))
    return out


# ----------------------------------------------------------------------------------------
# autograd-free restatement: the formulas the layer-norm kernels compute, stage by stage
# ----------------------------------------------------------------------------------------
def _img(t):
    """per-image scalar [n] -> broadcastable [n, 1, 1, 1]"""
    return t[:, None, None, None]


def block_forward(a_in, W, b, weight, bias, forced=None):
    """conv -> layer norm over [F, h, w] of each image (y = weight * zh + bias) -> leaky-ReLU -> 2x2 max-pool.
    ``forced``: optional (slope, idx), the discrete decisions to use instead of deriving them from y (see
    ``maml_oracle.block_forward``)."""
    z = F.conv2d(a_in, W, b, stride=1, padding=1)
    m = z[0].numel()
    mu = z.mean(dim=(1, 2, 3))
    zc = z - _img(mu)
    v = (zc * zc).mean(dim=(1, 2, 3))
    r = (v + LN_EPS) ** -0.5
    zh = zc * _img(r)
    y = weight[None] * zh + bias[None]
    if forced is None:
        sl = O._slope(y)
        p, idx = F.max_pool2d(y * sl, 2, 2, return_indices=True)
    else:
        sl, idx = forced[0].to(y.dtype), forced[1]
        n, c = y.shape[:2]
        p = (y * sl).view(n, c, -1).gather(2, idx.view(n, c, -1)).view(n, c, *idx.shape[2:])
    return {"a_in": a_in, "zh": zh, "r": r, "m": m, "slope": sl, "idx": idx, "p": p, "y": y}


def block_backward(fw, W, weight, dp, need_dgrad):
    """dp: gradient w.r.t. the pooled output.  dz = r (dzh - S1/m - zh S2/m) with per-image S1 = sum dzh,
    S2 = sum dzh * zh; the bias gradient is the sum over the images of dy at each position."""
    dy = O._unpool(dp, fw["idx"], fw["zh"]) * fw["slope"]
    zh, r, m = fw["zh"], fw["r"], fw["m"]
    dzh = dy * weight[None]
    m1 = _img(dzh.sum(dim=(1, 2, 3)) / m)
    m2 = _img((dzh * zh).sum(dim=(1, 2, 3)) / m)
    dz = _img(r) * (dzh - m1 - zh * m2)
    dW = torch.nn.grad.conv2d_weight(fw["a_in"], W.shape, dz, stride=1, padding=1)
    da_in = F.conv_transpose2d(dz, W, stride=1, padding=1) if need_dgrad else None
    return {"dW": dW, "db": dz.sum(dim=(0, 2, 3)), "dbias": dy.sum(dim=0), "da_in": da_in, "dz": dz, "dy": dy,
            "dzh": dzh, "m2": m2}


def net_forward_manual(x, theta, state, args, y, forced=None):
    fws, a = [], x
    for l in range(O.num_stages(args)):
        wn, bn_, gn, btn, _, _ = O.conv_names(l)
        fw = block_forward(a, theta[wn], theta[bn_], state[gn], state[btn], None if forced is None else forced[l])
        fws.append(fw)
        a = fw["p"]
    f = a.reshape(a.shape[0], -1)
    logits, loss, prob = O.head_forward(f, theta[O.LIN_W], theta[O.LIN_B], y)
    return {"blocks": fws, "f": f, "logits": logits, "loss": loss, "prob": prob}


def net_backward_manual(fwd, theta, state, args, y, scale=1.0):
    """Gradient of scale * loss w.r.t. the inner tensors and the layer-norm biases."""
    hb = O.head_backward(fwd["f"], theta[O.LIN_W], fwd["prob"], y, scale)
    grads, ln_grads = {O.LIN_W: hb["dW"], O.LIN_B: hb["db"]}, {}
    saved = [None] * O.num_stages(args)
    dp = hb["df"].reshape(fwd["blocks"][-1]["p"].shape)
    for l in reversed(range(O.num_stages(args))):
        wn, bn_, gn, btn, _, _ = O.conv_names(l)
        bw = block_backward(fwd["blocks"][l], theta[wn], state[gn], dp, need_dgrad=(l > 0))
        grads[wn], grads[bn_], ln_grads[btn] = bw["dW"], bw["db"], bw["dbias"]
        saved[l] = dict(bw, dp=dp)
        dp = bw["da_in"]
    return grads, ln_grads, {"head": hb, "blocks": saved}


def tangent_pass(fwd, bwd_saved, theta, u, state, args, y):
    """Forward-mode derivative of (support forward + support backward) in direction u (the inner tensors; the
    layer-norm bias carries no tangent).  Returns (Hu, H_b u per layer-norm bias, intermediates)."""
    L = O.num_stages(args)
    tf, a_dot = [], None
    for l in range(L):
        wn, bn_, gn, _, _, _ = O.conv_names(l)
        fw = fwd["blocks"][l]
        z_dot = F.conv2d(fw["a_in"], u[wn], u[bn_], stride=1, padding=1)
        if a_dot is not None:
            z_dot = z_dot + F.conv2d(a_dot, theta[wn], None, stride=1, padding=1)
        zh, r = fw["zh"], fw["r"]
        q = (zh * z_dot).mean(dim=(1, 2, 3))
        zh_dot = _img(r) * (z_dot - _img(z_dot.mean(dim=(1, 2, 3))) - zh * _img(q))
        a_dot_full = state[gn][None] * zh_dot * fw["slope"]
        n, c = a_dot_full.shape[:2]
        p_dot = a_dot_full.view(n, c, -1).gather(2, fw["idx"].view(n, c, -1)).view(fw["p"].shape)
        tf.append({"zh_dot": zh_dot, "q": q, "p_dot": p_dot, "a_in_dot": a_dot})
        a_dot = p_dot
    f, prob = fwd["f"], fwd["prob"]
    f_dot = a_dot.reshape(f.shape)
    n = f.shape[0]
    l_dot = f_dot @ theta[O.LIN_W].t() + f @ u[O.LIN_W].t() + u[O.LIN_B]
    dl = bwd_saved["head"]["dl"]
    dl_dot = (prob * l_dot - prob * (prob * l_dot).sum(dim=1, keepdim=True)) / n
    Hu = {O.LIN_W: dl_dot.t() @ f + dl.t() @ f_dot, O.LIN_B: dl_dot.sum(0)}
    df_dot = dl_dot @ theta[O.LIN_W] + dl @ u[O.LIN_W]
    mixed, tb = {}, [None] * L
    dp_dot = df_dot.reshape(fwd["blocks"][-1]["p"].shape)
    for l in reversed(range(L)):
        wn, bn_, gn, btn, _, _ = O.conv_names(l)
        fw, bw, t = fwd["blocks"][l], bwd_saved["blocks"][l], tf[l]
        zh, r, m = fw["zh"], fw["r"], fw["m"]
        dy_dot = O._unpool(dp_dot, fw["idx"], zh) * fw["slope"]
        dzh_dot = dy_dot * state[gn][None]
        m1_dot = _img(dzh_dot.mean(dim=(1, 2, 3)))
        m2_dot = _img((dzh_dot * zh + bw["dzh"] * t["zh_dot"]).mean(dim=(1, 2, 3)))
        dz_dot = _img(-r * t["q"]) * bw["dz"] + _img(r) * (dzh_dot - m1_dot - t["zh_dot"] * bw["m2"] - zh * m2_dot)
        W = theta[wn]
        dW_dot = torch.nn.grad.conv2d_weight(fw["a_in"], W.shape, dz_dot, stride=1, padding=1)
        if t["a_in_dot"] is not None:
            dW_dot = dW_dot + torch.nn.grad.conv2d_weight(t["a_in_dot"], W.shape, bw["dz"], stride=1, padding=1)
        Hu[wn], Hu[bn_] = dW_dot, dz_dot.sum(dim=(0, 2, 3))
        mixed[btn] = dy_dot.sum(dim=0)
        tb[l] = {"dz_dot": dz_dot, "dp_dot": dp_dot, "dy_dot": dy_dot}
        if l > 0:
            dp_dot = F.conv_transpose2d(dz_dot, W, stride=1, padding=1) + \
                F.conv_transpose2d(bw["dz"], u[wn], stride=1, padding=1)
    return Hu, mixed, {"fwd": tf, "bwd": tb, "l_dot": l_dot}


def manual_train_iter(state, args, batch, epoch, training_phase=True, current_epoch=None, keep_intermediates=False,
                      decisions=None):
    """Same contract as ``autograd_train_iter`` (plus ``intermediates`` when asked, in the form of
    ``maml_oracle.manual_train_iter``'s).  ``decisions``: optional {(task, "sup"|"tgt", step): [per-block (slope, idx)]}."""
    epoch = int(epoch)
    if current_epoch is None:
        current_epoch = epoch
    dtype = state[O.LIN_W].dtype
    xs, xt, ys, yt = batch
    xs, xt = xs.to(dtype), xt.to(dtype)
    ys, yt = ys.long(), yt.long()
    B = xs.shape[0]
    S_train = int(args.number_of_training_steps_per_iter)
    num_steps = S_train if training_phase else int(args.number_of_evaluation_steps_per_iter)
    second_order = bool(args.second_order) and epoch > args.first_order_to_second_order_epoch and training_phase
    sched = O.target_pass_schedule(args, epoch, training_phase, num_steps)
    w_msl = torch.from_numpy(O.msl_weights(args, current_epoch)).to(dtype)
    inner = O.inner_param_names(args)
    outer = OrderedDict((n, torch.zeros_like(state[n])) for n in state)
    losses, corrects, logits_out, inter = [], [], [], []
    with torch.no_grad():
        for b in range(B):
            x_s, y_s = xs[b].reshape(-1, *xs.shape[-3:]), ys[b].reshape(-1)
            x_t, y_t = xt[b].reshape(-1, *xt.shape[-3:]), yt[b].reshape(-1)
            theta = [{n: state[n] for n in inner}]
            sup_f, sup_b, sup_g, tgt_f = [], [], [], []
            task_loss, last_logits = torch.zeros((), dtype=dtype), None
            for s in range(num_steps):
                fwd = net_forward_manual(x_s, theta[s], state, args, y_s,
                                         None if decisions is None else decisions[(b, "sup", s)])
                g, _, saved = net_backward_manual(fwd, theta[s], state, args, y_s)
                sup_f.append(fwd); sup_b.append(saved); sup_g.append(g)
                theta.append({n: theta[s][n] - state[O.lslr_name(n)][s] * g[n] for n in inner})
                if sched[s] is not None:
                    tf_ = net_forward_manual(x_t, theta[s + 1], state, args, y_t,
                                             None if decisions is None else decisions[(b, "tgt", s)])
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
            tgt_b, tgt_g = [None] * num_steps, [None] * num_steps
            tbar_before0 = None
            for s in reversed(range(num_steps)):
                if tgt_f[s] is not None:
                    tf_, wgt = tgt_f[s]
                    tg, tln, tsaved = net_backward_manual(tf_, theta[s + 1], state, args, y_t, scale=float(wgt))
                    tgt_b[s], tgt_g[s] = tsaved, tg
                    for n in inner:
                        tbar[n] = tbar[n] + tg[n]
                    for n, gval in tln.items():
                        outer[n] += gval
                for n in inner:
                    outer[O.lslr_name(n)][s] += -(tbar[n] * sup_g[s][n]).sum()
                if s == 0:
                    tbar_before0 = dict(tbar)
                if second_order:
                    u = {n: state[O.lslr_name(n)][s] * tbar[n] for n in inner}
                    Hu, mixed, tint = tangent_pass(sup_f[s], sup_b[s], theta[s], u, state, args, y_s)
                    for n in inner:
                        tbar[n] = tbar[n] - Hu[n]
                    for n, gval in mixed.items():
                        outer[n] -= gval
                    if keep_intermediates:
                        inter.append({"task": b, "step": s, "u": u, "Hu": Hu, "mixed": mixed, "tangent": tint})
            for n in inner:
                outer[n] += tbar[n]
            if keep_intermediates:
                inter.append({"task": b, "theta": theta, "sup_f": sup_f, "sup_b": sup_b, "sup_g": sup_g,
                              "tgt_f": tgt_f, "tgt_b": tgt_b, "tgt_g": tgt_g, "tbar0": tbar_before0, "tbar": dict(tbar)})
    out = {"loss": torch.stack(losses).mean(), "accuracy": float(torch.cat(corrects).mean()),
           "logits": torch.stack(logits_out)}
    if training_phase:
        out["grads"] = OrderedDict((n, outer[n] / B) for n in trainable_names(args))
    if keep_intermediates:
        out["intermediates"] = inter
    return out
