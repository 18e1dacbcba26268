"""The five BASELINE.json configurations as args overrides.

Values restate the reference's shipped JSON files (reference
``experiment_config/omniglot_maml++-omniglot_1_8_0.1_64_5_0.json`` etc.; SURVEY.md
section 8d) so that bench / tests do not need ``/root/reference`` at run time.  Anything not
listed keeps the argparse default of ``utils/parser_utils.py`` (notably
``task_learning_rate=0.1`` and ``seed=104``).
"""
from .utils.parser_utils import args_from_json

_COMMON = dict(
    num_stages=4, conv_padding=True, max_pooling=True, norm_layer="batch_norm",
    number_of_training_steps_per_iter=5, number_of_evaluation_steps_per_iter=5,
    second_order=True, first_order_to_second_order_epoch=-1,
    learnable_bn_gamma=True, learnable_bn_beta=True, enable_inner_loop_optimizable_bn_params=False,
    meta_learning_rate=0.001, total_iter_per_epoch=500, num_evaluation_tasks=600,
)

_OMNIGLOT = dict(
    image_height=28, image_width=28, image_channels=1, dataset_name="omniglot_dataset",
    dataset_path="omniglot_dataset", cnn_num_filters=64, num_target_samples=1,
    min_learning_rate=0.00001, total_epochs=100, multi_step_loss_num_epochs=10,
)

_MINI_IMAGENET = dict(
    image_height=84, image_width=84, image_channels=3, dataset_name="mini_imagenet_full_size",
    dataset_path="mini_imagenet_full_size", cnn_num_filters=48, num_target_samples=15,
    min_learning_rate=0.001, total_epochs=100, multi_step_loss_num_epochs=15,
    init_inner_loop_learning_rate=0.01,   # never read (reference quirk), kept for schema fidelity
)

_MAML_PP = dict(per_step_bn_statistics=True, learnable_per_layer_per_step_inner_loop_learning_rate=True,
                use_multi_step_loss_optimization=True)
_MAML = dict(per_step_bn_statistics=False, learnable_per_layer_per_step_inner_loop_learning_rate=False,
             use_multi_step_loss_optimization=False)


def _mk(*parts, **kw):
    d = {}
    for p in (_COMMON,) + parts:
        d.update(p)
    d.update(kw)
    return d


CONFIGS = {
    # configs[0]: Omniglot MAML 5-way 1-shot, meta-batch 8 (the reference's CPU-runnable case)
    "omniglot_maml_5w1s": _mk(_OMNIGLOT, _MAML, batch_size=8, num_classes_per_set=5,
                              num_samples_per_class=1, experiment_name="omniglot_maml_5w1s"),
    # configs[1]: Omniglot MAML++ 5-way 1-shot, meta-batch 8, one GPU (the headline workload)
    "omniglot_mamlpp_5w1s": _mk(_OMNIGLOT, _MAML_PP, batch_size=8, num_classes_per_set=5,
                                num_samples_per_class=1, experiment_name="omniglot_mamlpp_5w1s"),
    # configs[2]: Mini-ImageNet MAML++ 5-way 1-shot, 48 filters, meta-batch 2
    "mini_imagenet_mamlpp_5w1s": _mk(_MINI_IMAGENET, _MAML_PP, batch_size=2, num_classes_per_set=5,
                                     num_samples_per_class=1, experiment_name="mini_imagenet_mamlpp_5w1s"),
    # configs[3]: Mini-ImageNet MAML++ 5-way 5-shot, meta-batch 16 over 8 GPUs
    "mini_imagenet_mamlpp_5w5s": _mk(_MINI_IMAGENET, _MAML_PP, batch_size=16, num_classes_per_set=5,
                                     num_samples_per_class=5, experiment_name="mini_imagenet_mamlpp_5w5s"),
    # configs[4]: Omniglot MAML++ 20-way 5-shot, meta-batch 64 over 8 GPUs
    "omniglot_mamlpp_20w5s": _mk(_OMNIGLOT, _MAML_PP, batch_size=64, num_classes_per_set=20,
                                 num_samples_per_class=5, experiment_name="omniglot_mamlpp_20w5s"),
}


def make_args(name, **overrides):
    """Args Bunch for one of the BASELINE configurations (``CONFIGS`` key) + overrides."""
    d = dict(CONFIGS[name])
    d.update(overrides)
    return args_from_json(None, **d)
