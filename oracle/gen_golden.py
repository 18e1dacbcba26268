"""ORACLE TOOLING -- TEST INFRASTRUCTURE ONLY.

Generates the golden vectors under ``tests/golden/`` by importing the UNMODIFIED reference
from ``/root/reference`` (a pure-Python/PyTorch program; it runs on CPU in the authoring
container) and running ``MAMLFewShotClassifier.run_train_iter`` on seeded synthetic episodes.

  python oracle/gen_golden.py            # regenerates every case
  python oracle/gen_golden.py tiny_pp    # one case

Each ``tests/golden/<case>.npz`` holds: the args (JSON string), the initial ``state_dict``,
the fp32 reference outputs (loss, accuracy, last-step logits, every outer gradient captured
just before ``optimizer.step``, the post-Adam ``state_dict`` incl. running statistics, the
logged ``learning_rate``), and the fp64 reference loss / gradients (noise-floor anchor for
the tolerance policy, SURVEY.md appendix C).  Inputs are stored only for the tiny and envelope cases; the
full-size ones are regenerated from their seed by ``oracle.maml_oracle.synthetic_batch``.

The reference cannot travel to the GPU box (``/root/reference`` does not exist there), so
nothing under ``tests/`` reads it at run time: tests read these fixtures.
"""
import contextlib
import io
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from howtotrainyourmamlpytorch_b200.configs import CONFIGS  # noqa: E402
from howtotrainyourmamlpytorch_b200.utils.parser_utils import args_from_json  # noqa: E402
from oracle import maml_oracle as O  # noqa: E402

REF = "/root/reference"

_TINY = dict(image_height=20, image_width=20, image_channels=3, cnn_num_filters=16,
             num_classes_per_set=3, num_samples_per_class=2, num_target_samples=2,
             number_of_training_steps_per_iter=3, number_of_evaluation_steps_per_iter=3,
             batch_size=3, total_epochs=100, multi_step_loss_num_epochs=10,
             dataset_name="mini_imagenet_tiny")

# case name -> (base config, overrides, list of (epoch, iteration-seed) train iterations)
# Inputs are N(0,1) unless the case says otherwise (4th tuple entry).  Bernoulli "Omniglot-like" images give
# exact max-pool ties whose resolution is rounding noise, so the reference's own fp32-vs-fp64 gradients differ
# by 10-100 % there (measured; see DESIGN.md "noise floor"): the direct comparison is loose for that case, but
# the decision-forced test (GPU decisions pinned in the fp64 oracle) and the tie statistics ARE meaningful --
# this is the input distribution bench.py runs (BASELINE.md section 4).
KIND = "normal"
CASES = {
    "tiny_pp":        ("mini_imagenet_mamlpp_5w1s", dict(_TINY), [(0, 0), (0, 1)]),
    "tiny_pp_late":   ("mini_imagenet_mamlpp_5w1s", dict(_TINY), [(12, 0)]),
    "tiny_pp_first":  ("mini_imagenet_mamlpp_5w1s", dict(_TINY, second_order=False), [(3, 0)]),
    "tiny_maml":      ("omniglot_maml_5w1s", dict(_TINY, image_channels=1, image_height=16, image_width=16,
                                                  dataset_name="omniglot_tiny"), [(0, 0), (1, 1)]),
    "tiny_odd":       ("omniglot_mamlpp_5w1s", dict(_TINY, image_channels=1, image_height=28, image_width=28,
                                                    cnn_num_filters=32, batch_size=2,
                                                    dataset_name="omniglot_tiny"), [(2, 0)]),
    # Bernoulli(0.93) "Omniglot-like" binary images: exact max-pool ties in every block-0 window whose four receptive
    # fields coincide -- the case first-max-wins exists for (stage-wise GPU test compares dz against the oracle)
    "tiny_bern":      ("omniglot_mamlpp_5w1s", dict(_TINY, image_channels=1, image_height=28, image_width=28,
                                                    cnn_num_filters=32, batch_size=2,
                                                    dataset_name="omniglot_tiny"), [(0, 0), (0, 1)], "bernoulli"),
    "omniglot_mamlpp_5w1s": ("omniglot_mamlpp_5w1s", dict(batch_size=2), [(0, 0)]),
    "omniglot_maml_5w1s":   ("omniglot_maml_5w1s", dict(batch_size=2), [(0, 0)]),
    "mini_imagenet_mamlpp_5w1s": ("mini_imagenet_mamlpp_5w1s", dict(batch_size=1), [(0, 0)]),
    "omniglot_mamlpp_20w5s": ("omniglot_mamlpp_20w5s", dict(batch_size=1), [(0, 0)]),
    # the benchmarked input distribution of BASELINE configs[1] (exact pooling ties)
    "omniglot_mamlpp_5w1s_bernoulli": ("omniglot_mamlpp_5w1s", dict(batch_size=2), [(0, 0)], "bernoulli"),
    # BASELINE configs[3] shape (Mini-ImageNet 5-way 5-shot), one task
    "mini_imagenet_mamlpp_5w5s": ("mini_imagenet_mamlpp_5w5s", dict(batch_size=1), [(0, 0)]),
}


def _envelope(base, hwc, f, l, s, nkt, b, iters, kind=KIND, moved=None, **over):
    """One envelope case: H x W x C images, F filters, L stages, S inner steps, N-way K-shot with T targets, B tasks.
    ``moved``: a seed of ``maml_oracle.moved_state``, applied to the reference model before anything is recorded."""
    (h, w, c), (n, k, t) = hwc, nkt
    d = dict(_TINY, image_height=h, image_width=w, image_channels=c, cnn_num_filters=f, num_stages=l,
             number_of_training_steps_per_iter=s, number_of_evaluation_steps_per_iter=s, num_classes_per_set=n,
             num_samples_per_class=k, num_target_samples=t, batch_size=b)
    if c != 3:
        d["dataset_name"] = "omniglot_tiny"
    d.update(over)
    return (base, d, iters, kind) if moved is None else (base, d, iters, kind, moved)


# Envelope cases: one seeded configuration per corner of what maml_b200_create admits (filters 16..64, 1..4 stages,
# 1..8 inner steps, 1..4 channels, 2..32 ways, batches up to 128 images, any H x W), each named for the axis it exists
# for (DESIGN.md section 6).  Inputs are stored like the tiny cases'.  Most cases record a second iteration, so that
# the post-Adam state is checked after Adam's second step too.  Where the default inner LR of 0.1 throws the inner loop
# far out (the 1-shot cases: losses of 20-60, or the reference's own fp32 run 1e-3 of max-norm away from its fp64 run on
# 2-way), the case uses 0.02, so that the comparison with fp64 stays a statement about rounding.  Every fixture holds
# about eight copies of the weights (state, gradients in fp32 and fp64, post-Adam state per iteration), so wide filter
# banks go with few stages or one iteration: each file stays under 1 MB.
ENVELOPE_CASES = {
    # H != W; odd H at block 0 (21: a pooled row is dropped), odd W at block 1 (15)
    "env_nonsquare_odd": _envelope("mini_imagenet_mamlpp_5w1s", (21, 30, 3), 16, 3, 2, (3, 2, 2), 2, [(0, 0), (0, 1)]),
    # C0 = 2; a tall image pooled down to 5 x 1; MSL weights between the extremes.
    # Episode 6, not 0: episode 0 holds a leaky-ReLU pre-activation and a pooling pair 2e-7 from a tie (fp64), which fp32
    # evaluations resolve either way (the decision-forced test pins it; the direct comparisons cannot)
    "env_tall_c2": _envelope("omniglot_mamlpp_5w1s", (40, 13, 2), 32, 3, 3, (3, 2, 2), 2, [(3, 6), (3, 1)]),
    # L = 2 and C0 = 4 (the widest channel count) in the fused iteration.  One iteration: after
    # a second one, any fp32 restatement (the CPU oracle included) sits up to 1e-4 away from the reference on 0.5-1.5 %
    # of some tensors' elements (Adam's second step divides small, noisy gradient elements by their own magnitude)
    "env_c4_two_stages": _envelope("omniglot_mamlpp_5w1s", (10, 14, 4), 64, 2, 2, (3, 2, 2), 2, [(0, 0)]),
    # L = 1: no tensor-core block, the first block is the last block, the fused tail runs on block 0
    "env_one_stage": _envelope("omniglot_mamlpp_5w1s", (12, 12, 1), 16, 1, 2, (3, 2, 2), 2, [(0, 0), (0, 1)],
                               task_learning_rate=0.02),
    # S = 8 = MAML_MAX_STEPS with the multi-step loss on: eight target passes, LSLR vectors of 9
    "env_eight_steps": _envelope("omniglot_mamlpp_5w1s", (16, 16, 1), 32, 4, 8, (3, 2, 2), 2, [(0, 0), (0, 1)]),
    # S = 1, second order, multi-step loss off: one target slot
    "env_one_step": _envelope("mini_imagenet_mamlpp_5w1s", (14, 18, 3), 32, 3, 1, (3, 2, 2), 2, [(20, 0), (20, 1)]),
    # 32-way 4-shot: a support batch of 128 images (the cap), 32 head row groups
    "env_way32": _envelope("omniglot_mamlpp_5w1s", (8, 8, 1), 16, 3, 2, (32, 4, 1), 1, [(0, 0)]),
    # the two sides of head_rows / tail_fusable: 17 support rows (head kernel) and 16 (fused tail), 24 target rows
    "env_way17": _envelope("omniglot_mamlpp_5w1s", (8, 8, 1), 16, 2, 2, (17, 1, 1), 1, [(0, 0)]),
    "env_way16": _envelope("omniglot_mamlpp_5w1s", (8, 8, 1), 16, 2, 2, (8, 2, 3), 1, [(0, 0), (0, 1)]),
    # 2-way 1-shot: the smallest batches; the last block's BatchNorm sees 2 x 3 x 3 = 18 values per channel
    "env_way2": _envelope("omniglot_mamlpp_5w1s", (28, 28, 1), 16, 4, 2, (2, 1, 1), 2, [(0, 0)], task_learning_rate=0.02),
    # block 1 is 65 wide (grid 66): the halo tile does not fit, so the handle itself runs the FFMA convolutions
    "env_ffma_wide": _envelope("omniglot_mamlpp_5w1s", (8, 130, 1), 16, 2, 2, (3, 1, 1), 1, [(0, 0)], task_learning_rate=0.02),
    # block 1 is 62 wide (grid 63): the largest halo the tensor-core convolution admits, a B ring of exactly 2 stages
    # next to split-K 2 in tangent mode
    "env_ring_edge": _envelope("mini_imagenet_mamlpp_5w1s", (6, 124, 3), 64, 2, 2, (3, 1, 1), 1, [(0, 0)], task_learning_rate=0.02),
    # 48 tasks: one weight-gradient chunk per block (num_sms / (3 * 48) rounds to 0), many tasks in every grid
    "env_many_tasks": _envelope("omniglot_mamlpp_5w1s", (8, 8, 1), 16, 3, 2, (3, 1, 1), 48, [(0, 0)]),
    # Bernoulli(0.93) images on a non-square odd image: exact pooling ties next to the dropped row
    "env_bern_nonsquare": _envelope("omniglot_mamlpp_5w1s", (27, 20, 1), 32, 4, 2, (3, 2, 2), 2, [(0, 0)], "bernoulli"),
    # plain MAML: shared BatchNorm statistics, no LSLR, no multi-step loss, non-square; F = 48 on the tensor cores, and
    # the head kernel after the last block (5 x 7 pooling windows per image are too many for the fused tail)
    "env_maml_shared_bn": _envelope("omniglot_maml_5w1s", (18, 26, 3), 48, 2, 4, (3, 2, 2), 2, [(0, 0)],
                                    dataset_name="omniglot_tiny"),
}

# Moved-state envelope cases (maml_oracle.moved_state, applied to the reference model before anything is recorded):
# distinct gamma / beta per step and block, one LSLR rate per tensor and step, nonzero biases and running statistics.
# At the initialisation every one of these is uniform, so a kernel that reads them from the wrong step, block or tensor
# computes the right numbers there.  Same fixture layout and test battery as ENVELOPE_CASES (which keeps the shape
# corners, all at the initialisation); one case per path that reads gamma / beta / alpha differently:
MOVED_CASES = {
    # MAML++ second order, MSL weights between their extremes, fused tail, tensor cores, two iterations
    "env_moved_pp": _envelope("mini_imagenet_mamlpp_5w1s", (14, 14, 3), 32, 3, 3, (3, 2, 2), 2, [(3, 0), (3, 1)],
                              moved=1),
    # a first-order epoch with the multi-step loss off (one target pass, at the last step).  One iteration: one block-2
    # weight-gradient element is 7e-8 of max-norm and has opposite signs in the reference's fp32 and fp64 runs; Adam's
    # first step turns that into +-lr, which moves a second iteration's loss by 3e-4 (fp64 restatements land where the
    # engine does, the reference's fp32 run does not)
    "env_moved_first": _envelope("mini_imagenet_mamlpp_5w1s", (16, 16, 3), 32, 3, 3, (3, 2, 2), 2, [(12, 0)],
                                 moved=2, second_order=False),
    # plain MAML: shared BatchNorm, the head kernel after the last block (5 x 7 pooling windows per image)
    "env_moved_maml": _envelope("omniglot_maml_5w1s", (18, 26, 3), 32, 2, 3, (3, 2, 2), 2, [(0, 0)], moved=3,
                                dataset_name="omniglot_tiny"),
    # L = 1: the fused tail runs on block 0
    "env_moved_one_stage": _envelope("omniglot_mamlpp_5w1s", (12, 12, 1), 16, 1, 3, (3, 2, 2), 2, [(3, 0), (3, 1)],
                                     moved=4),
    # block 1 65 wide: the handle itself runs the FFMA convolutions
    "env_moved_ffma": _envelope("omniglot_mamlpp_5w1s", (8, 130, 1), 16, 2, 3, (3, 1, 1), 1, [(3, 0)], moved=5),
    # S = 8: the largest step-row and LSLR index space
    "env_moved_eight": _envelope("omniglot_mamlpp_5w1s", (16, 16, 1), 16, 4, 8, (3, 2, 2), 2, [(3, 0), (3, 1)], moved=6),
}
CASES.update(ENVELOPE_CASES)
CASES.update(MOVED_CASES)


def case_kind(case):
    c = CASES[case]
    return c[3] if len(c) > 3 else KIND


def case_moved(case):
    """The ``moved_state`` seed of a case, or None (the reference's initialisation)."""
    c = CASES[case]
    return c[4] if len(c) > 4 else None


def make_args(case):
    base, over, iters = CASES[case][:3]
    d = dict(CONFIGS[base])
    d.update(over)
    d["experiment_name"] = case
    return args_from_json(None, **d), d, iters


def build_reference(args, dtype):
    sys.path.insert(0, REF)
    import few_shot_learning_system as ref_sys  # noqa: the reference, unmodified
    with contextlib.redirect_stdout(io.StringIO()):
        model = ref_sys.MAMLFewShotClassifier(
            im_shape=(2, args.image_channels, args.image_height, args.image_width),
            device=torch.device("cpu"), args=args)
    if dtype == torch.float64:
        model.double()
    return model


def run_reference_fp32(args, iters, store_inputs, kind=KIND, moved=None):
    """fp32 reference run.  The true model gives the losses / logits / post-Adam state.  The outer
    gradients are captured on a twin model whose ``dataset_name`` lacks 'imagenet' -- the reference clamps
    ``param.grad`` in place between ``backward`` and ``optimizer.step`` (:332-335), so the twin is the only
    way to see the UNCLAMPED gradients without editing the reference.  The twin is reloaded from the true
    model's parameters before every iteration.  ``moved``: a ``moved_state`` seed applied to the model first."""
    import copy
    import warnings
    warnings.filterwarnings("ignore")
    model = build_reference(args, torch.float32)
    if moved is not None:
        model.load_state_dict(O.moved_state(model.state_dict(), args, moved))
    args_nc = copy.copy(args)
    args_nc.dataset_name = args.dataset_name.replace("imagenet", "imgnet")
    twin = build_reference(args_nc, torch.float32)
    out = {}
    for k, v in model.state_dict().items():
        out["state/" + k] = v.detach().numpy().copy()
    for it, (epoch, seed_it) in enumerate(iters):
        batch = O.synthetic_batch(args, iteration=seed_it, kind=kind)
        if store_inputs:
            for nm, t in zip(("xs", "xt", "ys", "yt"), batch):
                out["it%d/%s" % (it, nm)] = t.numpy().copy()
        twin.load_state_dict(copy.deepcopy(model.state_dict()))
        captured = {}
        orig_step = twin.optimizer.step

        def step_and_capture(*a, **kw):
            for n, p in twin.named_parameters():
                if p.requires_grad:
                    captured[n] = (p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p))
            return None          # the twin never updates

        twin.optimizer.step = step_and_capture
        with contextlib.redirect_stdout(io.StringIO()):
            twin.run_train_iter(data_batch=batch, epoch=epoch)
        twin.optimizer.step = orig_step
        with contextlib.redirect_stdout(io.StringIO()):
            losses, preds = model.run_train_iter(data_batch=batch, epoch=epoch)
        out["it%d/loss" % it] = np.float64(float(losses["loss"]))
        out["it%d/accuracy" % it] = np.float64(float(losses["accuracy"]))
        out["it%d/learning_rate" % it] = np.float64(float(losses["learning_rate"]))
        S = args.number_of_training_steps_per_iter
        out["it%d/msl" % it] = np.array([float(losses["loss_importance_vector_%d" % i]) for i in range(S)])
        out["it%d/logits" % it] = np.stack(preds).astype(np.float32)
        for n, g in captured.items():
            out["it%d/grad/%s" % (it, n)] = g.numpy().copy()
        for k, v in model.state_dict().items():
            out["it%d/post/%s" % (it, k)] = v.detach().numpy().copy()
    return out


def run_reference_validation(args, iters, state32, kind=KIND):
    """Reference ``run_validation_iter`` (few_shot_learning_system.py:371-397) from the INITIAL state on the first
    recorded batch: loss, accuracy, last-step logits and the running statistics afterwards (the reference's
    backup/restore of them is an alias, meta_neural_network_architectures.py:240-255, so they come out mutated)."""
    model = build_reference(args, torch.float32)
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in state32.items()})
    epoch, seed_it = iters[0]
    model.current_epoch = int(epoch)
    batch = O.synthetic_batch(args, iteration=seed_it, kind=kind)
    with contextlib.redirect_stdout(io.StringIO()):
        losses, preds = model.run_validation_iter(data_batch=batch)
    out = {"val/loss": np.float64(float(losses["loss"])), "val/accuracy": np.float64(float(losses["accuracy"])),
           "val/logits": np.stack(preds).astype(np.float32)}
    for k, v in model.state_dict().items():
        if "running" in k:
            out["val/post/" + k] = v.detach().numpy().copy()
    return out


def run_reference_fp64(args, iters, state32, big, kind=KIND):
    """fp64 reference gradients at the SAME parameters as each fp32 iteration started from
    (iteration 0 only -- later iterations start from fp32-updated parameters)."""
    model = build_reference(args, torch.float64)
    sd = {k: torch.from_numpy(v).double() for k, v in state32.items()}
    model.load_state_dict(sd)
    epoch, seed_it = iters[0]
    batch = O.synthetic_batch(args, iteration=seed_it, kind=kind)
    xs, xt, ys, yt = batch
    model.current_epoch = int(epoch)
    data = (xs.double(), xt.double(), ys.long(), yt.long())
    with contextlib.redirect_stdout(io.StringIO()):
        losses, _ = model.train_forward_prop(data_batch=data, epoch=int(epoch))
        model.optimizer.zero_grad()
        losses["loss"].backward()
    out = {"it0/loss64": np.float64(float(losses["loss"]))}
    for n, p in model.named_parameters():
        if p.requires_grad:
            g = p.grad.detach() if p.grad is not None else torch.zeros_like(p)
            out["it0/grad64/" + n] = g.numpy().astype(np.float32 if big else np.float64)
    return out


def write_reference_checkpoint(case="tiny_pp"):
    """A checkpoint WRITTEN BY THE REFERENCE (its own save_model, few_shot_learning_system.py:399-409) after the recorded
    train iterations of ``case`` -> tests/golden/ref_ckpt_<case>/train_model_latest.  tests/test_host_logic.py loads it
    through this repo's load_model and compares with the post-state fixtures."""
    import warnings
    warnings.filterwarnings("ignore")
    args, argdict, iters = make_args(case)
    model = build_reference(args, torch.float32)
    for epoch, seed_it in iters:
        batch = O.synthetic_batch(args, iteration=seed_it, kind=case_kind(case))
        with contextlib.redirect_stdout(io.StringIO()):
            model.run_train_iter(data_batch=batch, epoch=epoch)
    d = os.path.join(ROOT, "tests", "golden", "ref_ckpt_" + case)
    os.makedirs(d, exist_ok=True)
    state = {"best_val_acc": 0.25, "best_val_iter": 1, "current_iter": len(iters), "best_epoch": 0,
             "train_loss_mean": 1.5, "per_epoch_statistics": {"train_loss_mean": [1.5]}}
    model.save_model(model_save_dir=os.path.join(d, "train_model_latest"), state=state)
    return d


def write_episode_fixture():
    """Episodes drawn by the reference's own ``FewShotLearningDatasetParallel.get_set`` (data.py:478-524) from a small
    synthetic IN-MEMORY dataset (the object is built without its file-scanning __init__) -> tests/golden/episodes.npz:
    for Omniglot-like (1 channel, rot90 train augmentation) and ImageNet-like (3 channels, mean / std normalisation)
    settings, several seeds, augmentation on and off.  The GPU sampler must reproduce them bit for bit."""
    sys.path.insert(0, REF)
    sys.argv = [sys.argv[0]]
    import data as ref_data  # noqa: the reference, unmodified
    from howtotrainyourmamlpytorch_b200.data import synthetic_class_images
    blob = {}
    for tag, dataset_name, C, binary in (("omni", "omniglot_dataset", 1, True), ("imnet", "mini_imagenet_full_size", 3, False)):
        H = W = 8
        classes = synthetic_class_images(12, 7, H, W, C, seed=11 if C == 1 else 12, binary=binary)
        args, _, _ = make_args("tiny_pp")
        args.dataset_name = dataset_name
        args.image_channels, args.image_height, args.image_width = C, H, W
        args.num_classes_per_set, args.num_samples_per_class, args.num_target_samples = 4, 2, 3
        ds = object.__new__(ref_data.FewShotLearningDatasetParallel)
        ds.args = args
        ds.dataset_name = dataset_name
        ds.data_loaded_in_memory = True
        ds.image_channel = C
        ds.num_classes_per_set, ds.num_samples_per_class, ds.num_target_samples = 4, 2, 3
        ds.dataset_size_dict = {"train": {k: len(v) for k, v in classes.items()}}
        ds.datasets = {"train": {k: v for k, v in classes.items()}}
        cases = []
        for seed in (5, 123456, 99):
            for aug in (False, True):
                xs, xt, ys, yt, _ = ds.get_set("train", seed=seed, augment_images=aug)
                key = "%s/seed%d_aug%d" % (tag, seed, int(aug))
                blob[key + "/xs"] = xs.numpy().astype(np.float32); blob[key + "/xt"] = xt.numpy().astype(np.float32)
                blob[key + "/ys"] = np.asarray(ys, dtype=np.float32); blob[key + "/yt"] = np.asarray(yt, dtype=np.float32)
                cases.append((seed, int(aug)))
        blob[tag + "/cases"] = np.array(cases)
        blob[tag + "/meta"] = np.array(json.dumps({"dataset_name": dataset_name, "C": C, "H": H, "W": W, "classes": 12,
                                                   "samples": 7, "seed": 11 if C == 1 else 12, "binary": binary,
                                                   "N": 4, "K": 2, "T": 3}))
    path = os.path.join(ROOT, "tests", "golden", "episodes.npz")
    np.savez_compressed(path, **blob)
    return path


def check_against_oracle(args, blob, iters, kind=KIND):
    """Immediately validate both restatements against what was just generated."""
    state = {k[len("state/"):]: torch.from_numpy(v) for k, v in blob.items() if k.startswith("state/")}
    epoch, seed_it = iters[0]
    batch = O.synthetic_batch(args, iteration=seed_it, kind=kind)
    worst = {}
    for nm, fn in (("autograd", O.autograd_train_iter), ("manual", O.manual_train_iter)):
        for dt, suffix in ((torch.float32, ""), (torch.float64, "64")):
            st = {k: v.to(dt) for k, v in state.items()}
            res = fn(st, args, batch, epoch)
            ref_loss = float(blob["it0/loss" + suffix])
            err = abs(float(res["loss"]) - ref_loss) / max(abs(ref_loss), 1e-30)
            gerr = 0.0
            for n, g in res["grads"].items():
                ref = torch.from_numpy(blob["it0/grad%s/%s" % (suffix, n)]).to(torch.float64)
                denom = float(ref.abs().max())
                if denom < 1e-6:
                    continue  # dead conv-bias gradients: pure noise in the reference
                gerr = max(gerr, float((g.double() - ref).abs().max()) / denom)
            worst[nm + suffix] = (err, gerr)
    # validation leg (fp32): loss, logits and the mutated running statistics
    for nm, fn in (("autograd", O.autograd_train_iter), ("manual", O.manual_train_iter)):
        res = fn(state, args, batch, epoch, training_phase=False, current_epoch=epoch)
        ref_loss = float(blob["val/loss"])
        err = abs(float(res["loss"]) - ref_loss) / max(abs(ref_loss), 1e-30)
        lerr = float((res["logits"].float() - torch.from_numpy(blob["val/logits"])).abs().max())
        rerr = 0.0
        for k, v in res["running"].items():
            rerr = max(rerr, float((v - torch.from_numpy(blob["val/post/" + k])).abs().max()))
        worst[nm + "_val"] = (err, max(lerr, rerr))
    return worst


def main():
    os.makedirs(os.path.join(ROOT, "tests", "golden"), exist_ok=True)
    which = sys.argv[1:] or list(CASES.keys())
    torch.set_num_threads(8)
    if "--episodes" in which:
        print(write_episode_fixture())
        return
    if "--checkpoint" in which:
        print(write_reference_checkpoint("tiny_pp"))
        return
    for case in which:
        args, argdict, iters = make_args(case)
        kind = case_kind(case)
        big = not case.startswith("tiny_") and case not in ENVELOPE_CASES and case not in MOVED_CASES
        moved = case_moved(case)
        blob = run_reference_fp32(args, iters, store_inputs=not big, kind=kind, moved=moved)
        state32 = {k[len("state/"):]: v for k, v in blob.items() if k.startswith("state/")}
        blob.update(run_reference_validation(args, iters, state32, kind))
        blob.update(run_reference_fp64(args, iters, state32, big, kind))
        blob["args_json"] = np.array(json.dumps(argdict))
        blob["iters_json"] = np.array(json.dumps(iters))
        blob["kind"] = np.array(kind)
        if moved is not None:
            blob["moved"] = np.array(moved)
        path = os.path.join(ROOT, "tests", "golden", case + ".npz")
        np.savez_compressed(path, **blob)
        worst = check_against_oracle(args, blob, iters, kind)
        # the reference's own fp32-vs-fp64 distance (live tensors, of max-norm): how tame the inner loop is
        own = max(float(np.abs(blob[k].astype(np.float64) - blob[k.replace("/grad/", "/grad64/")]).max())
                  / max(float(np.abs(blob[k.replace("/grad/", "/grad64/")]).max()), 1e-30)
                  for k in blob if k.startswith("it0/grad/") and "conv.bias" not in k and "conv-bias" not in k)
        print(case, "%.1f KB" % (os.path.getsize(path) / 1024.0), "fp32 vs fp64 %.1e" % own,
              {k: ("%.1e" % a, "%.1e" % b) for k, (a, b) in worst.items()}, flush=True)


if __name__ == "__main__":
    main()
