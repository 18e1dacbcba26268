"""Time one outer training iteration (forward + meta-gradient) of the headline config (Omniglot MAML++ 5-way 1-shot,
meta-batch 8, second order) three ways, on one GPU:

  operator  the reference's training loop (per task, per inner step: torch.autograd.grad(create_graph=True), LSLR
            update, MSL target losses; then the outer backward) on this repository's VGGReLUNormNetwork.forward
            (integration route B1: engine forward / backward / Hessian-vector product);
  torch     the same loop on torch ops on the GPU (oracle._net_forward: F.conv2d / F.batch_norm / ..., fp32, TF32 off);
  fused     MAMLFewShotClassifier.run_train_iter (route B0: the whole iteration as one engine call, Adam step included);
  operator_vmap  the functorch MAML recipe on the operator: torch.func.vmap over the meta-batch, inner torch.func.grad
            steps with the LSLR update, MSL target losses, outer torch.autograd.grad -- every operator call runs the
            meta-batch as one engine call (n_tasks = 8);
  torch_vmap     the same functorch loop on torch ops (oracle._net_forward under vmap); reported as skipped, with the
            error, if torch.func cannot run it.

Warm-up first; every timed iteration ends in a device synchronise; the legs alternate within each repeat.  Prints
one JSON line: per leg the median / min / max milliseconds per iteration, plus the GPU name and power limit read in
the same run.  ``--norm-layer layer_norm`` runs the same config with the layer-norm network (its torch legs on
oracle.ln_oracle._net_forward) and adds "norm_layer" to the line.  ``--inner-bn`` sets
enable_inner_loop_optimizable_bn_params on the BatchNorm network (BatchNorm gamma / beta adapted per task in the inner
loop, and differentiated with the other fast weights in every leg) and adds "inner_bn" to the line.

  python scripts/functional_route_timing.py [--repeats 20] [--warmup 3] [--norm-layer {batch_norm,layer_norm}] [--inner-bn]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch                                         # noqa: E402
import torch.nn.functional as Fnn                    # noqa: E402

CONFIG, META_BATCH = "omniglot_mamlpp_5w1s", 8


def reference_loop(net_forward, params, a, batch, epoch, O, names):
    """oracle.autograd_train_iter's loop with a pluggable network forward; returns the outer gradients."""
    S = int(a.number_of_training_steps_per_iter)
    second_order = bool(a.second_order) and epoch > a.first_order_to_second_order_epoch
    sched = O.target_pass_schedule(a, epoch, True, S)
    w_msl = torch.from_numpy(O.msl_weights(a, epoch)).to(batch[0].device)
    inner = O.inner_param_names(a)
    xs, xt, ys, yt = batch
    total = []
    for b in range(xs.shape[0]):
        fast = {n: params[n] for n in inner}
        x_s, y_s = xs[b].reshape(-1, *xs.shape[-3:]), ys[b].reshape(-1)
        x_t, y_t = xt[b].reshape(-1, *xt.shape[-3:]), yt[b].reshape(-1)
        task_losses = []
        for s in range(S):
            loss_s = Fnn.cross_entropy(net_forward(x_s, fast, s), y_s)
            grads = torch.autograd.grad(loss_s, [fast[n] for n in inner], create_graph=second_order)
            fast = {n: fast[n] - params[O.lslr_name(n)][s] * g for n, g in zip(inner, grads)}
            if sched[s] is not None:
                loss_t = Fnn.cross_entropy(net_forward(x_t, fast, s), y_t)
                task_losses.append(w_msl[s] * loss_t if sched[s] == "msl" else loss_t)
        total.append(torch.stack(task_losses).sum())
    loss = torch.stack(total).mean()
    return torch.autograd.grad(loss, [params[n] for n in names], allow_unused=True)


def functorch_loop(net_forward, params, a, batch, epoch, O, names):
    """The loop above written the torch.func way: vmap over the tasks, torch.func.grad for the inner steps (its result
    detached for first order), the outer gradient through torch.autograd."""
    S = int(a.number_of_training_steps_per_iter)
    second_order = bool(a.second_order) and epoch > a.first_order_to_second_order_epoch
    sched = O.target_pass_schedule(a, epoch, True, S)
    w_msl = torch.from_numpy(O.msl_weights(a, epoch)).to(batch[0].device)
    inner = O.inner_param_names(a)
    xs, xt, ys, yt = batch
    B = xs.shape[0]

    def task(fast, x_s, y_s, x_t, y_t):
        task_losses = []
        for s in range(S):
            g = torch.func.grad(lambda p, s=s: Fnn.cross_entropy(net_forward(x_s, p, s), y_s))(fast)
            if not second_order:
                g = {n: v.detach() for n, v in g.items()}
            fast = {n: fast[n] - params[O.lslr_name(n)][s] * g[n] for n in inner}
            if sched[s] is not None:
                loss_t = Fnn.cross_entropy(net_forward(x_t, fast, s), y_t)
                task_losses.append(w_msl[s] * loss_t if sched[s] == "msl" else loss_t)
        return torch.stack(task_losses).sum()

    per_task = [t.reshape(B, -1, *t.shape[-3:]) for t in (xs, xt)] + [t.reshape(B, -1) for t in (ys, yt)]
    loss = torch.func.vmap(task, in_dims=(None, 0, 0, 0, 0))({n: params[n] for n in inner}, per_task[0], per_task[2],
                                                             per_task[1], per_task[3]).mean()
    return torch.autograd.grad(loss, [params[n] for n in names], allow_unused=True)


def gpu_info():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True).stdout.strip()
    name, _, power = out.partition(",")
    return name.strip() or torch.cuda.get_device_name(0), power.strip() or "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--norm-layer", default="batch_norm", choices=["batch_norm", "layer_norm"])
    ap.add_argument("--inner-bn", action="store_true", help="enable_inner_loop_optimizable_bn_params (batch norm only)")
    cli = ap.parse_args()
    if cli.inner_bn and cli.norm_layer == "layer_norm":
        ap.error("--inner-bn needs --norm-layer batch_norm")
    if not torch.cuda.is_available():
        raise SystemExit("functional_route_timing.py needs a CUDA device")
    from howtotrainyourmamlpytorch_b200 import MAMLFewShotClassifier, make_args, synthetic_batch
    from oracle import ln_oracle as LN
    from oracle import maml_oracle as O
    layer_norm = cli.norm_layer == "layer_norm"
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda", 0)
    extra = {"norm_layer": "layer_norm"} if layer_norm else {}
    if cli.inner_bn:
        extra["enable_inner_loop_optimizable_bn_params"] = True
    a = make_args(CONFIG, batch_size=META_BATCH, **extra)
    names = LN.trainable_names(a) if layer_norm else O.trainable_names(a)
    epoch = 0
    batch = synthetic_batch(a, iteration=0)
    dbatch = tuple(t.to(dev) for t in batch)
    dbatch = (dbatch[0].float(), dbatch[1].float(), dbatch[2].long(), dbatch[3].long())
    m_op = MAMLFewShotClassifier(im_shape=(2, a.image_channels, a.image_height, a.image_width), device=dev, args=a)
    m_fused = MAMLFewShotClassifier(im_shape=(2, a.image_channels, a.image_height, a.image_width), device=dev, args=a)
    m_fused.load_state_dict(m_op.state_dict())
    op_params = dict(m_op.named_parameters())
    t_params = {k: v.detach().clone().to(dev).requires_grad_(v.requires_grad) for k, v in m_op.state_dict().items()}
    t_params.update({k: v.detach().clone().requires_grad_(True) for k, v in op_params.items() if v.requires_grad})
    pre = len("classifier.")

    def op_forward(x, fast, s):
        return m_op.classifier.forward(x, num_step=s, training=True, params={n[pre:]: w.unsqueeze(0) for n, w in fast.items()})

    def torch_forward(x, fast, s):
        return LN._net_forward(x, fast, t_params, a) if layer_norm else O._net_forward(x, fast, t_params, a, s)

    legs = {
        "operator": lambda: reference_loop(op_forward, op_params, a, dbatch, epoch, O, names),
        "torch": lambda: reference_loop(torch_forward, t_params, a, dbatch, epoch, O, names),
        "fused": lambda: m_fused.run_train_iter(batch, epoch),
        "operator_vmap": lambda: functorch_loop(op_forward, op_params, a, dbatch, epoch, O, names),
        "torch_vmap": lambda: functorch_loop(torch_forward, t_params, a, dbatch, epoch, O, names),
    }
    skipped = {}
    try:
        legs["torch_vmap"]()
    except Exception as e:                  # torch.func cannot run the torch-op network: report, do not time
        skipped["torch_vmap"] = "%s: %s" % (type(e).__name__, str(e).splitlines()[0] if str(e) else "")
        del legs["torch_vmap"]
    for _ in range(cli.warmup):
        for f in legs.values():
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in legs}
    for _ in range(cli.repeats):
        for k, f in legs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            times[k].append(1e3 * (time.perf_counter() - t0))
    name, power = gpu_info()

    def summary(v):
        v = sorted(v)
        return {"median_ms": round(v[len(v) // 2], 3), "min_ms": round(v[0], 3), "max_ms": round(v[-1], 3)}

    line = {"config": CONFIG, "meta_batch": META_BATCH, "second_order": True, "gpu": name,
            "power_limit": power, "repeats": cli.repeats, "warmup": cli.warmup,
            "legs": {k: summary(v) for k, v in times.items()}, "skipped": skipped}
    if layer_norm:
        line["norm_layer"] = "layer_norm"
    if cli.inner_bn:
        line["inner_bn"] = True
    print(json.dumps(line))


if __name__ == "__main__":
    main()
