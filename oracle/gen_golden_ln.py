"""ORACLE TOOLING -- TEST INFRASTRUCTURE ONLY.  Golden vectors of the LAYER-NORM network (``norm_layer: "layer_norm"``)
from the UNMODIFIED reference, in the format of ``oracle/gen_golden.py`` (whose runners it reuses):

  python oracle/gen_golden_ln.py               # every case
  python oracle/gen_golden_ln.py ln_tiny_pp    # one case

Writes ``tests/golden/<case>.npz`` and checks ``oracle/ln_oracle.py`` against the fp64 reference run at once."""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import gen_golden as G  # noqa: E402
from oracle import ln_oracle as LN  # noqa: E402
from oracle import maml_oracle as O  # noqa: E402

_LN = dict(norm_layer="layer_norm")
# case -> (base config, overrides, train iterations [(epoch, seed)], input kind, moved_state seed)
LN_CASES = {
    # MAML++ second order at the tiny shape (20x20x3, F = 16, 3-way 2-shot, S = 3, 3 tasks), two recorded iterations
    "ln_tiny_pp": ("mini_imagenet_mamlpp_5w1s", dict(G._TINY, **_LN), [(0, 0), (0, 1)], "normal", None),
    # the same away from the initialisation: bias [F, h, w], conv / linear biases and LSLR rates moved
    "ln_tiny_pp_moved": ("mini_imagenet_mamlpp_5w1s", dict(G._TINY, **_LN), [(3, 0), (3, 1)], "normal", 7),
    # plain MAML: shared (non-learnable) inner learning rates, no multi-step loss
    "ln_tiny_maml": ("omniglot_maml_5w1s", dict(G._TINY, image_channels=1, image_height=16, image_width=16, **_LN),
                     [(0, 0)], "normal", None),
    # H != W with odd sizes: 21 x 30 -> block 1 is 10 x 15 (odd width), the dropped column still counts in the statistics
    "ln_nonsquare_odd": ("mini_imagenet_mamlpp_5w1s",
                         dict(G._TINY, image_height=21, image_width=30, batch_size=2, **_LN), [(0, 0)], "normal", None),
    # Bernoulli images: exact pooling ties
    "ln_bern": ("omniglot_mamlpp_5w1s", dict(G._TINY, image_channels=1, image_height=28, image_width=28, batch_size=2,
                                             task_learning_rate=0.02, **_LN), [(0, 0)], "bernoulli", None),
    # the shape of env_moved_eight: S = 8, so the LSLR vectors (9 entries) and the per-(pass, step) bias-gradient rows are
    # indexed past step 4
    "ln_eight_moved": G._envelope("omniglot_mamlpp_5w1s", (16, 16, 1), 16, 4, 8, (3, 2, 2), 2, [(3, 0), (3, 1)],
                                  moved=6, **_LN),
    # the shape of env_one_stage: L = 1, the head follows block 0's per-image normalisation
    "ln_one_stage": G._envelope("omniglot_mamlpp_5w1s", (12, 12, 1), 16, 1, 2, (3, 2, 2), 2, [(0, 0), (0, 1)],
                                moved=None, task_learning_rate=0.02, **_LN) + (None,),
}


def make_args(case):
    base, over, iters = LN_CASES[case][:3]
    G.CASES[case] = (base, over, iters)
    return G.make_args(case)


def check_against_oracle(args, blob, iters, kind):
    """Relative loss error and worst gradient error (of each tensor's max-norm) of the fp64 oracle against the fp64
    reference run."""
    state = {k[len("state/"):]: torch.from_numpy(v).double() for k, v in blob.items() if k.startswith("state/")}
    epoch, seed_it = iters[0]
    res = LN.autograd_train_iter(state, args, O.synthetic_batch(args, iteration=seed_it, kind=kind), epoch)
    err = abs(float(res["loss"]) - float(blob["it0/loss64"])) / abs(float(blob["it0/loss64"]))
    gerr = 0.0
    for n, g in res["grads"].items():
        ref = torch.from_numpy(blob["it0/grad64/" + n]).double()
        gerr = max(gerr, float((g - ref).abs().max()) / max(float(ref.abs().max()), 1e-30))
    return err, gerr


def main():
    torch.set_num_threads(8)
    for case in sys.argv[1:] or list(LN_CASES):
        args, argdict, iters = make_args(case)
        kind, moved = LN_CASES[case][3], LN_CASES[case][4]
        big = False                               # every case stores its inputs (each file stays under 1 MB)
        O_moved = O.moved_state
        O.moved_state = LN.moved_state            # the reference's frozen weight stays all ones
        try:
            blob = G.run_reference_fp32(args, iters, store_inputs=not big, kind=kind, moved=moved)
        finally:
            O.moved_state = O_moved
        state32 = {k[len("state/"):]: v for k, v in blob.items() if k.startswith("state/")}
        blob.update(G.run_reference_validation(args, iters, state32, kind))
        blob.update(G.run_reference_fp64(args, iters, state32, big, kind))
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
