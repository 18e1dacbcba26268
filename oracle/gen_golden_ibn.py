"""ORACLE TOOLING -- TEST INFRASTRUCTURE ONLY.  Golden vectors of the network with inner-loop BatchNorm gamma / beta
(``enable_inner_loop_optimizable_bn_params``) from the UNMODIFIED reference, in the format of ``oracle/gen_golden.py``
(whose runners it reuses):

  python oracle/gen_golden_ibn.py               # every case
  python oracle/gen_golden_ibn.py ibn_tiny_pp   # one case

Writes ``tests/golden/<case>.npz`` (with the validation leg) and checks ``oracle/maml_oracle.py`` against the fp64
reference run at once."""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import gen_golden as G  # noqa: E402
from oracle import maml_oracle as O  # noqa: E402

_IBN = dict(enable_inner_loop_optimizable_bn_params=True)
_OMNI = dict(image_channels=1, dataset_name="omniglot_tiny")
# case -> (base config, overrides, train iterations [(epoch, seed)], input kind, moved_state seed)
IBN_CASES = {
    # MAML++ second order at the tiny shape (20x20x3, F = 16, 3-way 2-shot, S = 3, 3 tasks), two recorded iterations
    "ibn_tiny_pp": ("mini_imagenet_mamlpp_5w1s", dict(G._TINY, **_IBN), [(0, 0), (0, 1)], "normal", None),
    # the same away from the initialisation: distinct gamma / beta per block, biases and LSLR rates moved
    "ibn_tiny_pp_moved": ("mini_imagenet_mamlpp_5w1s", dict(G._TINY, **_IBN), [(3, 0)], "normal", 7),
    # a first-order epoch.  Moved-state seed 13: every max-pool margin of its fp64 run is >= 6e-7 (seed 11 has one of 4e-8
    # in block 0, inside fp32 rounding, where an fp32 run may pick either position)
    "ibn_tiny_first": ("mini_imagenet_mamlpp_5w1s", dict(G._TINY, second_order=False, **_IBN), [(3, 0)], "normal", 13),
    # plain MAML: shared running statistics (None in F.batch_norm), shared inner learning rates, no multi-step loss
    "ibn_tiny_maml": ("omniglot_maml_5w1s", dict(G._TINY, image_height=16, image_width=16, **dict(_OMNI, **_IBN)),
                      [(0, 0)], "normal", 5),
    # one block (L = 1): the head follows block 0 directly
    "ibn_one_stage": ("omniglot_mamlpp_5w1s", dict(G._TINY, image_height=12, image_width=12, num_stages=1,
                                                   number_of_training_steps_per_iter=2, number_of_evaluation_steps_per_iter=2,
                                                   batch_size=2, **dict(_OMNI, **_IBN)), [(0, 0)], "normal", 3),
    # an 8 x 130 image: too wide for the tensor-core conv's halo box, so blocks >= 1 run on the FFMA kernels
    "ibn_ffma_wide": ("omniglot_mamlpp_5w1s", dict(G._TINY, image_height=8, image_width=130, num_stages=2,
                                                   number_of_training_steps_per_iter=2, number_of_evaluation_steps_per_iter=2,
                                                   num_samples_per_class=1, num_target_samples=1, batch_size=1,
                                                   task_learning_rate=0.02, **dict(_OMNI, **_IBN)), [(0, 0)], "normal", 9),
    # Bernoulli images: exact pooling ties
    "ibn_bern": ("omniglot_mamlpp_5w1s", dict(G._TINY, image_height=28, image_width=28, cnn_num_filters=32, batch_size=2,
                                              task_learning_rate=0.02, **dict(_OMNI, **_IBN)), [(0, 0)], "bernoulli", None),
    # the shape of env_moved_eight: S = 8, so the gamma / beta LSLR vectors (9 entries) and the per-step running-statistics
    # rows are indexed past step 4
    "ibn_eight_moved": G._envelope("omniglot_mamlpp_5w1s", (16, 16, 1), 16, 4, 8, (3, 2, 2), 2, [(3, 0), (3, 1)],
                                   moved=6, **_IBN),
    # the shape of env_many_tasks at a moved state: 48 tasks, so every task's gamma / beta (theta + task * Ppad) past task 7
    # is read
    "ibn_many_tasks": G._envelope("omniglot_mamlpp_5w1s", (8, 8, 1), 16, 3, 2, (3, 1, 1), 48, [(0, 0)], moved=8, **_IBN),
}


def make_args(case):
    base, over, iters = IBN_CASES[case][:3]
    G.CASES[case] = (base, over, iters)
    return G.make_args(case)


def check_against_oracle(args, blob, iters, kind):
    """Relative loss error and worst gradient error (of each tensor's max-norm) of the fp64 oracle against the fp64
    reference run."""
    state = {k[len("state/"):]: torch.from_numpy(v).double() for k, v in blob.items() if k.startswith("state/")}
    epoch, seed_it = iters[0]
    res = O.autograd_train_iter(state, args, O.synthetic_batch(args, iteration=seed_it, kind=kind), epoch)
    err = abs(float(res["loss"]) - float(blob["it0/loss64"])) / abs(float(blob["it0/loss64"]))
    gerr = 0.0
    for n, g in res["grads"].items():
        ref = torch.from_numpy(blob["it0/grad64/" + n]).double()
        gerr = max(gerr, float((g - ref).abs().max()) / max(float(ref.abs().max()), 1e-30))
    return err, gerr


def main():
    torch.set_num_threads(8)
    for case in sys.argv[1:] or list(IBN_CASES):
        args, argdict, iters = make_args(case)
        kind, moved = IBN_CASES[case][3], IBN_CASES[case][4]
        blob = G.run_reference_fp32(args, iters, store_inputs=True, kind=kind, moved=moved)
        state32 = {k[len("state/"):]: v for k, v in blob.items() if k.startswith("state/")}
        blob.update(G.run_reference_validation(args, iters, state32, kind))
        blob.update(G.run_reference_fp64(args, iters, state32, False, kind))
        blob["args_json"] = np.array(json.dumps(argdict))
        blob["iters_json"] = np.array(json.dumps(iters))
        blob["kind"] = np.array(kind)
        if moved is not None:
            blob["moved"] = np.array(moved)
        path = os.path.join(G.ROOT, "tests", "golden", case + ".npz")
        np.savez_compressed(path, **blob)
        print(case, "%.1f KB" % (os.path.getsize(path) / 1024.0), "oracle vs fp64 reference (loss, grads): %.1e %.1e"
              % check_against_oracle(args, blob, iters, kind), flush=True)


if __name__ == "__main__":
    main()
