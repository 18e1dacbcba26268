#!/usr/bin/env python
"""Time the UNMODIFIED reference (staged under ``oracle/_ref`` by ``oracle/stage_reference.py``) on the hot path:
``MAMLFewShotClassifier.run_train_iter`` (reference few_shot_learning_system.py:338-369) through the reference's own
public API and stock code path -- none of this repo's kernels, engine or model code runs here.  What this repo
contributes is the workload description only: the args Bunch of a BASELINE configuration (the reference's own JSON
values restated in ``howtotrainyourmamlpytorch_b200/configs.py``) and the seeded synthetic episode tensors.

  python baseline/run_reference.py --config NAME --device cpu|cuda [--batch-size B] [--steps K] [--warmup W]
                                   [--threads T | --tune-threads] [--max-seconds S]

``--device cpu`` hides the GPUs (CUDA_VISIBLE_DEVICES="") before torch is imported, exactly as BASELINE.md section 4
prescribes -- the reference self-selects CUDA otherwise (:73-81).  ``--device cuda`` lets it do that: the reference's
own GPU path (eager PyTorch on cuDNN / ATen), the "library kernels to beat" of SURVEY.md section 8d.
Prints ONE JSON line: per-iteration times, tasks/s (batch / median), threads used, CPU model, reference commit.
"""
import argparse
import contextlib
import io
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "oracle", "_ref")


def cpu_model():
    try:
        for line in open("/proc/cpuinfo"):
            if line.startswith("model name"):
                return line.split(":", 1)[1].strip()
    except Exception:
        pass
    return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="omniglot_mamlpp_5w1s")
    ap.add_argument("--device", default="cpu", choices=["cpu", "cuda"])
    ap.add_argument("--batch-size", type=int, default=None)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--threads", type=int, default=None)
    ap.add_argument("--tune-threads", action="store_true",
                    help="one probe iteration at 8/16/32/64/all host threads, keep the fastest (the reference's ops are "
                         "small: more threads is not faster)")
    ap.add_argument("--max-seconds", type=float, default=240.0, help="stop timing early once this much wall time is spent")
    ap.add_argument("--kind", default=None, help="synthetic input distribution override (bernoulli|normal)")
    cli = ap.parse_args()

    if not os.path.isdir(REF) or not os.path.exists(os.path.join(REF, "few_shot_learning_system.py")):
        print(json.dumps({"unavailable": "oracle/_ref is not staged (run oracle/stage_reference.py)"}))
        return 0
    if cli.device == "cpu":
        os.environ["CUDA_VISIBLE_DEVICES"] = ""
    sys.path.insert(0, ROOT)
    import torch
    import warnings
    warnings.filterwarnings("ignore")
    from howtotrainyourmamlpytorch_b200.configs import make_args          # workload description only
    from howtotrainyourmamlpytorch_b200.synthetic import synthetic_batch
    sys.path.insert(0, REF)
    import few_shot_learning_system as ref_sys                            # the reference, unmodified

    over = {"batch_size": cli.batch_size} if cli.batch_size else {}
    args = make_args(cli.config, **over)
    args.use_cuda = torch.cuda.is_available()
    ncpu = os.cpu_count() or 1
    dev = torch.device("cuda", torch.cuda.current_device()) if (cli.device == "cuda" and torch.cuda.is_available()) else torch.device("cpu")
    if cli.device == "cuda" and dev.type != "cuda":
        print(json.dumps({"unavailable": "no CUDA device visible to the reference"}))
        return 0
    if dev.type == "cuda":
        # fp32 like the CPU path: the reference never enables TF32 itself
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False

    with contextlib.redirect_stdout(io.StringIO()):
        model = ref_sys.MAMLFewShotClassifier(im_shape=(2, args.image_channels, args.image_height, args.image_width),
                                              device=dev, args=args)
    n_pool = 4
    batches = [synthetic_batch(args, iteration=i, kind=cli.kind) for i in range(n_pool)]

    def one(i):
        t0 = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            losses, _ = model.run_train_iter(data_batch=batches[i % n_pool], epoch=0)
        loss = float(losses["loss"])          # the reference's caller does this too (experiment_builder.py:122-126)
        if dev.type == "cuda":
            torch.cuda.synchronize()
        return time.perf_counter() - t0, loss

    threads = cli.threads
    tuned = None
    if dev.type == "cpu":
        if threads is None and cli.tune_threads:
            cands = sorted(set(c for c in (8, 16, 32, 64, ncpu) if c <= ncpu)) or [ncpu]
            tuned, best_t = {}, None
            one(0)                                        # first call: lazy initialisation, never counted
            for c in cands:
                torch.set_num_threads(c)
                t, _ = one(1)
                tuned[c] = t
                if best_t is None or t < best_t:
                    threads, best_t = c, t
                if t > 4.0 * best_t:
                    break
        if threads is None:
            threads = ncpu
        torch.set_num_threads(threads)

    wall0 = time.perf_counter()
    for i in range(max(1, cli.warmup)):
        one(i)
    times, loss = [], None
    for i in range(max(1, cli.steps)):
        t, loss = one(cli.warmup + i)
        times.append(t)
        if time.perf_counter() - wall0 > cli.max_seconds and len(times) >= 2:
            break
    st = sorted(times)
    med = st[len(st) // 2]
    commit = None
    try:
        commit = json.load(open(os.path.join(REF, "MANIFEST.json"))).get("commit")
    except Exception:
        pass
    out = {
        "impl": "reference (unmodified, oracle/_ref)", "commit": commit, "config": cli.config, "device": str(dev),
        "batch_size": int(args.batch_size), "tasks_per_sec": args.batch_size / med, "ms_per_iter": 1e3 * med,
        "times_s": times, "warmup": max(1, cli.warmup), "threads": (threads if dev.type == "cpu" else None),
        "host_threads": ncpu, "cpu_model": cpu_model(), "thread_probe_s": tuned, "last_loss": loss,
        "torch": torch.__version__,
        "gpu": (torch.cuda.get_device_name(dev) if dev.type == "cuda" else None),
    }
    print(json.dumps(out), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
