"""Test helpers shared by the functional-network operator tests: cases, models, batches and stand-alone engine handles."""
import torch

from conftest import load_golden
from oracle import gen_golden
from oracle import maml_oracle as O


MOVED_SEED = 7
# Every envelope case and every moved-state case of the fused iteration's fixtures, in the generator's order: the
# functional-operator tests run on each, so that the operator's own launch plans (sized for n images and B tasks, not for
# the fused iteration's support + target batch) meet every shape maml_b200_create admits and every moved state
ENVELOPE = list(gen_golden.ENVELOPE_CASES) + list(gen_golden.MOVED_CASES)


def case(name):
    """(args, fp32 state, batch) of a golden case, or of synthetic_c<C>[_w<W>][_f<F>]: a seeded model with C input
    channels, W x W images (14 if not given) and F filters (32 if not given), so that the first-block kernels run at every
    channel count, at even and odd widths and at filter counts where no golden case covers them.  A ``_moved`` suffix
    moves the case's state off the initialisation (``maml_oracle.moved_state``): distinct gamma / beta per step."""
    if name.endswith("_moved"):
        a, state, batch = case(name[:-len("_moved")])
        return a, O.moved_state(state, a, MOVED_SEED), batch
    if name.startswith("synthetic_c"):
        from howtotrainyourmamlpytorch_b200 import make_args
        parts = name.split("_")
        c = int(parts[1][1:])
        opt = {p[0]: int(p[1:]) for p in parts[2:]}
        w, f = opt.pop("w", 14), opt.pop("f", 32)
        assert not opt, name
        a = make_args("omniglot_mamlpp_5w1s", image_channels=c, image_height=w, image_width=w,
                      cnn_num_filters=f, num_stages=3, number_of_training_steps_per_iter=2,
                      number_of_evaluation_steps_per_iter=2, batch_size=2, num_target_samples=3)
        return a, O.init_state(a), O.synthetic_batch(a, iteration=5, kind="normal")
    g = load_golden(name)
    return g.args, g.state(), g.batch(0)


def widen(batch, tasks=3):
    """The batch with at least `tasks` tasks, for the tests of the per-task entries: task b >= B (the fixture's B) is
    task b % B with its images at x * 0.5^k + 0.1 k, k = b - B + 1, and its labels.  A batch of `tasks` or more tasks is
    returned as it is."""
    xs, xt, ys, yt = batch
    B = xs.shape[0]

    def more(t, images):
        rows = [t]
        for b in range(B, tasks):
            k = b - B + 1
            rows.append(t[b % B:b % B + 1] * 0.5 ** k + 0.1 * k if images else t[b % B:b % B + 1])
        return torch.cat(rows)
    return more(xs, True), more(xt, True), more(ys, False), more(yt, False)


def model(a, state, device):
    from howtotrainyourmamlpytorch_b200 import MAMLFewShotClassifier
    m = MAMLFewShotClassifier(im_shape=(2, a.image_channels, a.image_height, a.image_width), device=device, args=a)
    m.load_state_dict(state)
    return m


def images(batch, which, b=0):
    xs, xt, ys, yt = batch
    x, y = (xs, ys) if which == "support" else (xt, yt)
    return x[b].reshape(-1, *x.shape[-3:]).float(), y[b].reshape(-1).long()


def bn_names(state):
    return [k for k in state if k.endswith("norm_layer.weight") or k.endswith("norm_layer.bias")]


def engine(a, k_shot, t_target, max_tasks, device):
    """A stand-alone engine handle for a's network, with batches of N * k_shot support and N * t_target target images."""
    from howtotrainyourmamlpytorch_b200 import _native
    with torch.cuda.device(device):
        return _native.Engine(n_way=int(a.num_classes_per_set), k_shot=k_shot, t_target=t_target, channels=int(a.image_channels),
                              height=int(a.image_height), width=int(a.image_width), filters=int(a.cnn_num_filters),
                              num_stages=int(a.num_stages), inner_steps=int(a.number_of_training_steps_per_iter),
                              per_step_bn=bool(a.per_step_bn_statistics), max_tasks=max_tasks)


def meta_like(m, eng, device):
    """m's own weights in the engine's meta layout."""
    meta = torch.zeros(eng.meta_size, dtype=torch.float32, device=device)
    for (off, size), t in zip(eng.segments, m.classifier._segment_tensors(None)):
        meta[off:off + size] = t.detach().reshape(-1)
    return meta
