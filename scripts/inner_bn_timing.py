"""Step time of the network with inner-loop BatchNorm gamma / beta (enable_inner_loop_optimizable_bn_params) against the
same network without the flag, on the same workload.

  python scripts/inner_bn_timing.py [--steps 30] [--warmup 5] [--rounds 3]

Workloads: Omniglot MAML++ 5-way 1-shot at 8 tasks (the headline shape) and Mini-ImageNet MAML++ 5-way 1-shot at 2 tasks,
seeded synthetic episodes (oracle.maml_oracle.synthetic_batch).  One step = run_train_iter (forward / backward, second
order, Adam), timed with a host clock around `steps` steps that end in a device synchronise; the two networks alternate
over `rounds` rounds and the best round of each is reported, with the GPU name and power limit.  The flag's handles run
the unfused streaming BatchNorm kernels (no cluster, fused-tail or on-chip tail kernels).  One JSON line per workload."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from howtotrainyourmamlpytorch_b200 import MAMLFewShotClassifier  # noqa: E402
from howtotrainyourmamlpytorch_b200.configs import CONFIGS  # noqa: E402
from howtotrainyourmamlpytorch_b200.utils.parser_utils import args_from_json  # noqa: E402
from oracle import maml_oracle as O  # noqa: E402

WORKLOADS = [("omniglot_mamlpp_5w1s", 8), ("mini_imagenet_mamlpp_5w1s", 2)]


def gpu_desc():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def model(config, tasks, inner_bn):
    d = dict(CONFIGS[config], batch_size=tasks, enable_inner_loop_optimizable_bn_params=inner_bn)
    a = args_from_json(None, **d)
    m = MAMLFewShotClassifier(im_shape=(2, a.image_channels, a.image_height, a.image_width), device="cuda", args=a)
    batch = tuple(t.cuda() for t in O.synthetic_batch(a, iteration=0))
    return m, batch


def time_steps(m, batch, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        m.run_train_iter(batch, 20)      # epoch 20: second order, past the multi-step-loss epochs of both configs
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("inner_bn_timing.py needs a CUDA device")
    name, power = gpu_desc()
    for config, tasks in WORKLOADS:
        runs = {flag: model(config, tasks, flag) for flag in (False, True)}
        for m, batch in runs.values():
            time_steps(m, batch, a.warmup)
        best = {flag: float("inf") for flag in runs}
        for _ in range(a.rounds):
            for flag, (m, batch) in runs.items():
                best[flag] = min(best[flag], time_steps(m, batch, a.steps))
        print(json.dumps({"workload": config, "tasks": tasks, "bn_ms_per_step": round(best[False], 3),
                          "inner_bn_ms_per_step": round(best[True], 3),
                          "inner_bn_over_bn": round(best[True] / best[False], 3),
                          "steps": a.steps, "rounds": a.rounds, "gpu": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
