"""Time forward-mode differentiation of the functional-network operator (VGGReLUNormNetwork.forward) on one GPU, on the
headline config (Omniglot MAML++ 5-way 1-shot, meta-batch 8) and on mini_imagenet_mamlpp_5w1s (meta-batch 2):

  jt        J t for every task's support batch at the meta weights, along a random direction over the conv / linear
            weights (the double-vjp route cannot take an image direction: a cotangent on the operator's image gradient is
            refused in reverse mode):
              jt_operator      torch.autograd.forward_ad on the operator (maml_b200_net_jvp: primal + tangent forward)
              jt_double_vjp    torch.autograd.functional.jvp on the operator (double-vjp: forward, backward, maml_b200_net_hvp)
              jt_torch         torch.autograd.forward_ad over torch ops on the GPU (oracle._net_forward)
  hyper     one second-order outer iteration of the reference's loop with a forward-mode hypergradient: the outer loss and
            its derivative along a random direction of the LSLR vectors
              hyper_operator   forward_ad with the LSLR vectors dual, on the operator
              hyper_reverse    reverse mode on the operator (the outer gradient w.r.t. the LSLR vectors)
              hyper_torch      forward_ad with the LSLR vectors dual, on torch ops on the GPU

Torch ops run in fp32 with TF32 off.  The legs alternate within each repeat and every timed call ends in a device
synchronise; a leg that fails (e.g. an op without a forward-mode formula) is reported with its error instead of a time.
Prints one JSON line with the GPU name and power limit read in the same run.

  python scripts/forward_mode_timing.py [--repeats 5] [--warmup 2]
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
import torch.autograd.forward_ad as fwAD             # noqa: E402
import torch.nn.functional as Fnn                    # noqa: E402

CONFIGS = [("omniglot_mamlpp_5w1s", 8), ("mini_imagenet_mamlpp_5w1s", 2)]


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    cli = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("forward_mode_timing.py needs a CUDA device")
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
        inner = O.inner_param_names(a)
        lslr = [O.lslr_name(n) for n in inner]
        gen = torch.Generator().manual_seed(0)
        w_dot = {n: torch.randn(op_params[n].shape, generator=gen).to(dev) for n in inner}
        a_dot = {n: torch.randn(op_params[n].shape, generator=gen).to(dev) for n in lslr}

        def op_net(x, fast, s):
            return m.classifier.forward(x, num_step=s, training=True, params={n[pre:]: w.unsqueeze(0) for n, w in fast.items()})

        def torch_net(x, fast, s):
            return O._net_forward(x, fast, t_params, a, s)

        def jt_forward_ad(net, params):
            out = []
            with fwAD.dual_level():
                fast = {n: fwAD.make_dual(params[n].detach(), w_dot[n]) for n in inner}
                for b in range(xs.shape[0]):
                    out.append(fwAD.unpack_dual(net(xs[b].reshape(-1, *xs.shape[-3:]), fast, 0)).tangent)
            return out

        def jt_double_vjp():
            out = []
            for b in range(xs.shape[0]):
                x = xs[b].reshape(-1, *xs.shape[-3:])

                def f(*ws):
                    return op_net(x, dict(zip(inner, ws)), 0)
                prim = tuple(op_params[n].detach() for n in inner)
                tan = tuple(w_dot[n] for n in inner)
                out.append(torch.autograd.functional.jvp(f, prim, tan)[1])
            return out

        def hyper_forward_ad(net, params):
            with fwAD.dual_level():
                p = dict(params)
                for n in lslr:
                    p[n] = fwAD.make_dual(params[n].detach(), a_dot[n])
                loss = meta_loop(net, p, a, xs, xt, ys, yt, epoch, O)
                return fwAD.unpack_dual(loss).tangent

        def hyper_reverse():
            loss = meta_loop(op_net, op_params, a, xs, xt, ys, yt, epoch, O)
            g = torch.autograd.grad(loss, [op_params[n] for n in lslr])
            return sum((gi * a_dot[n]).sum() for gi, n in zip(g, lslr))

        legs = {
            "jt_operator": lambda: jt_forward_ad(op_net, op_params),
            "jt_double_vjp": jt_double_vjp,
            "jt_torch": lambda: jt_forward_ad(torch_net, t_params),
            "hyper_operator": lambda: hyper_forward_ad(op_net, op_params),
            "hyper_reverse": hyper_reverse,
            "hyper_torch": lambda: hyper_forward_ad(torch_net, t_params),
        }
        failed = {}
        for _ in range(cli.warmup):
            for k, f in legs.items():
                if k in failed:
                    continue
                try:
                    f()
                except Exception as e:                    # reported, not timed
                    failed[k] = "%s: %s" % (type(e).__name__, str(e).splitlines()[0][:200])
        torch.cuda.synchronize()
        times = {k: [] for k in legs if k not in failed}
        for _ in range(cli.repeats):
            for k in times:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                legs[k]()
                torch.cuda.synchronize()
                times[k].append(1e3 * (time.perf_counter() - t0))

        def summary(v):
            v = sorted(v)
            return {"median_ms": round(v[len(v) // 2], 3), "min_ms": round(v[0], 3), "max_ms": round(v[-1], 3)}

        results.append({"config": config, "meta_batch": meta_batch, "legs": {k: summary(v) for k, v in times.items()},
                        "failed": failed})
    print(json.dumps({"gpu": name, "power_limit": power, "repeats": cli.repeats, "warmup": cli.warmup, "results": results}))


if __name__ == "__main__":
    main()
