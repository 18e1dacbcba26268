"""Time the image gradients of the functional-network operator (VGGReLUNormNetwork.forward) on one GPU, on the headline
config (Omniglot MAML++ 5-way 1-shot, meta-batch 8) and on mini_imagenet_mamlpp_5w1s (meta-batch 2):

  fgsm      one FGSM step on the target images at adapted weights: per task forward + backward to x_target, then
            x + eps * sign(dL/dx).  The weights are adapted beforehand (all inner steps, untimed).
  outer     one second-order outer iteration of the reference's loop with x_support as a leaf: the outer gradient w.r.t.
            every trainable tensor and x_support (which it reaches only through the inner gradients).

Each on the operator (engine forward / backward / HVP and the image-gradient entries) and on the same loop with torch
ops on the GPU (oracle._net_forward: F.conv2d / F.batch_norm / ..., fp32, TF32 off); the legs alternate within each
repeat, every timed call ends in a device synchronise.  Then the first-block data-gradient kernel alone
(maml_b200_net_input_grad: one launch; maml_b200_net_hvp_input_grad: its two-pair form), timed with CUDA events over
many launches, with the bytes it must move (first-conv output gradient read, first-block weights, image gradient
written; computed from the shapes) against the 3.35 TB/s HBM3 data-sheet bound.  Prints one JSON line with the GPU name
and power limit read in the same run.

  python scripts/input_grad_timing.py [--repeats 10] [--warmup 2] [--launches 200]
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

CONFIGS = [("omniglot_mamlpp_5w1s", 8), ("mini_imagenet_mamlpp_5w1s", 2)]
HBM_BYTES_PER_S = 3.35e12                            # H100 SXM5 80 GB data sheet
FGSM_EPS = 0.03


def gpu_info():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True).stdout.strip()
    name, _, power = out.partition(",")
    return name.strip() or torch.cuda.get_device_name(0), power.strip() or "unknown"


def meta_loop(net, params, a, xs, xt, ys, yt, epoch, O):
    """The reference's second-order loop with a pluggable network forward; returns the outer loss."""
    S = int(a.number_of_training_steps_per_iter)
    sched = O.target_pass_schedule(a, epoch, True, S)
    w_msl = torch.from_numpy(O.msl_weights(a, epoch)).to(xs.device)
    inner = O.inner_param_names(a)
    total = []
    for b in range(xs.shape[0]):
        fast = {n: params[n] for n in inner}
        x_s, y_s = xs[b].reshape(-1, *xs.shape[-3:]), ys[b].reshape(-1)
        x_t, y_t = xt[b].reshape(-1, *xt.shape[-3:]), yt[b].reshape(-1)
        losses = []
        for s in range(S):
            g = torch.autograd.grad(Fnn.cross_entropy(net(x_s, fast, s), y_s), [fast[n] for n in inner], create_graph=True)
            fast = {n: fast[n] - params[O.lslr_name(n)][s] * gi for n, gi in zip(inner, g)}
            if sched[s] is not None:
                loss_t = Fnn.cross_entropy(net(x_t, fast, s), y_t)
                losses.append(w_msl[s] * loss_t if sched[s] == "msl" else loss_t)
        total.append(torch.stack(losses).sum())
    return torch.stack(total).mean()


def adapted(net, params, a, xs, ys, O):
    """Fast weights after all inner steps of every task (first order, detached: the FGSM leg's starting point)."""
    inner = O.inner_param_names(a)
    out = []
    for b in range(xs.shape[0]):
        fast = {n: params[n].detach().requires_grad_(True) for n in inner}
        x_s, y_s = xs[b].reshape(-1, *xs.shape[-3:]), ys[b].reshape(-1)
        for s in range(int(a.number_of_training_steps_per_iter)):
            g = torch.autograd.grad(Fnn.cross_entropy(net(x_s, fast, s), y_s), [fast[n] for n in inner])
            fast = {n: (fast[n] - params[O.lslr_name(n)][s].detach() * gi).detach().requires_grad_(True)
                    for n, gi in zip(inner, g)}
        out.append({n: t.detach() for n, t in fast.items()})
    return out


def fgsm(net, fast_per_task, a, xt, yt):
    S = int(a.number_of_training_steps_per_iter)
    adv = []
    for b in range(xt.shape[0]):
        x = xt[b].reshape(-1, *xt.shape[-3:]).clone().requires_grad_(True)
        dx, = torch.autograd.grad(Fnn.cross_entropy(net(x, fast_per_task[b], S - 1), yt[b].reshape(-1)), x)
        adv.append(x.detach() + FGSM_EPS * dx.sign())
    return adv


def kernel_timing(a, m, xt, launches):
    """The data-gradient kernel alone: net_input_grad (one operand pair) and net_hvp_input_grad (two)."""
    from howtotrainyourmamlpytorch_b200 import _native
    dev = xt.device
    x = xt[0].reshape(1, -1, *xt.shape[-3:]).contiguous()
    n, N = x.shape[1], int(a.num_classes_per_set)
    C, H, W, F = int(a.image_channels), int(a.image_height), int(a.image_width), int(a.cnn_num_filters)
    kw = dict(n_way=N, channels=C, height=H, width=W, filters=F, num_stages=int(a.num_stages),
              inner_steps=int(a.number_of_training_steps_per_iter), per_step_bn=bool(a.per_step_bn_statistics), max_tasks=1)
    fwd = _native.Engine(k_shot=1, t_target=n // N, **kw)
    hvp = _native.Engine(k_shot=n // N, t_target=1, **kw)
    meta = torch.zeros(fwd.meta_size, device=dev)
    for (off, size), t in zip(fwd.segments, m.classifier._segment_tensors(None)):
        meta[off:off + size] = t.detach().reshape(-1)
    gen = torch.Generator().manual_seed(0)
    dl = torch.randn(1, n, N, generator=gen).to(dev)
    v = torch.randn(fwd.meta_size, generator=gen).to(dev)
    dx = torch.empty_like(x)
    fwd.net_forward(1, 0, meta, x, torch.empty(1, n, N, device=dev))
    fwd.net_backward(1, 0, meta, dl, torch.empty(fwd.result_size, device=dev))
    hvp.net_hvp(1, 0, meta, x, dl, v, torch.empty(1, n, N, device=dev), torch.empty(hvp.result_size, device=dev))
    out = {}
    for name, call, nsrc in (("net_input_grad", lambda: fwd.net_input_grad(1, dx), 1),
                             ("net_hvp_input_grad", lambda: hvp.net_hvp_input_grad(1, dx), 2)):
        for _ in range(10):
            call()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            call()
        e1.record()
        torch.cuda.synchronize()
        us = 1e3 * e0.elapsed_time(e1) / launches
        nbytes = 4.0 * (nsrc * (n * H * W * F + 9 * C * F) + n * C * H * W)
        flops = 2.0 * n * H * W * C * 9 * F * nsrc
        out[name] = {"us_per_launch": round(us, 2), "bytes": int(nbytes), "achieved_TBps": round(nbytes / us / 1e6, 3),
                     "fraction_of_3.35TBps": round(nbytes / us / 1e6 / (HBM_BYTES_PER_S / 1e12), 3),
                     "alg_GFLOPs": round(flops / us / 1e3, 1), "images": n}
    fwd.close()
    hvp.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--launches", type=int, default=200)
    cli = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("input_grad_timing.py needs a CUDA device")
    from howtotrainyourmamlpytorch_b200 import MAMLFewShotClassifier, make_args, synthetic_batch
    from oracle import maml_oracle as O
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda", 0)
    name, power = gpu_info()
    results = []
    for config, meta_batch in CONFIGS:
        a = make_args(config, batch_size=meta_batch)
        epoch = 0
        xs, xt, ys, yt = (t.to(dev) for t in synthetic_batch(a, iteration=0))
        xs, xt, ys, yt = xs.float(), xt.float(), ys.long(), yt.long()
        m = MAMLFewShotClassifier(im_shape=(2, a.image_channels, a.image_height, a.image_width), device=dev, args=a)
        op_params = dict(m.named_parameters())
        t_params = {k: v.detach().clone().requires_grad_(v.requires_grad) for k, v in m.state_dict().items()}
        t_params.update({k: v.detach().clone().requires_grad_(True) for k, v in op_params.items() if v.requires_grad})
        pre = len("classifier.")

        def op_net(x, fast, s):
            return m.classifier.forward(x, num_step=s, training=True, params={n[pre:]: w.unsqueeze(0) for n, w in fast.items()})

        def torch_net(x, fast, s):
            return O._net_forward(x, fast, t_params, a, s)

        names = O.trainable_names(a)
        op_fast = adapted(op_net, op_params, a, xs, ys, O)
        t_fast = adapted(torch_net, t_params, a, xs, ys, O)

        def outer(net, params):
            x_s = xs.clone().requires_grad_(True)
            loss = meta_loop(net, params, a, x_s, xt, ys, yt, epoch, O)
            return torch.autograd.grad(loss, [params[n] for n in names] + [x_s], allow_unused=True)

        legs = {
            "fgsm_operator": lambda: fgsm(op_net, op_fast, a, xt, yt),
            "fgsm_torch": lambda: fgsm(torch_net, t_fast, a, xt, yt),
            "outer_operator": lambda: outer(op_net, op_params),
            "outer_torch": lambda: outer(torch_net, t_params),
        }
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

        def summary(v):
            v = sorted(v)
            return {"median_ms": round(v[len(v) // 2], 3), "min_ms": round(v[0], 3), "max_ms": round(v[-1], 3)}

        results.append({"config": config, "meta_batch": meta_batch, "legs": {k: summary(v) for k, v in times.items()},
                        "kernel": kernel_timing(a, m, xt, cli.launches)})
    print(json.dumps({"gpu": name, "power_limit": power, "repeats": cli.repeats, "warmup": cli.warmup,
                      "launches": cli.launches, "results": results}))


if __name__ == "__main__":
    main()
