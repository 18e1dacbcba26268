"""Config / flag handling for the H100 MAML hot path.

Mirrors the reference's flag system (``utils/parser_utils.py:4-106`` of the reference):
argparse defaults overridden by the keys of a JSON file (except keys containing
``continue_from`` / ``gpu_to_use``), ``"true"/"false"`` strings turned into bools, and the
result exposed as an attribute bag (``Bunch``).  The JSON schema is kept byte-compatible so
the reference's ``experiment_config/*.json`` files drive this implementation unchanged.

Quirks that are kept on purpose (SURVEY.md section 5):
  * ``init_inner_loop_learning_rate`` in the JSON is never read; the inner LR is
    ``task_learning_rate`` (default 0.1) -- reference ``few_shot_learning_system.py:46``.
  * ``seed`` defaults to 104 and the shipped JSON files never override it.
"""
import argparse
import json
import os

# (name, type, default) -- same names/defaults as the reference's argparse block
# (reference utils/parser_utils.py:11-54).  Strings "True"/"False" become bools later.
_DEFAULTS = [
    ("batch_size", int, 32),
    ("image_height", int, 28),
    ("image_width", int, 28),
    ("image_channels", int, 1),
    ("reset_stored_filepaths", str, "False"),
    ("reverse_channels", str, "False"),
    ("num_of_gpus", int, 1),
    ("samples_per_iter", int, 1),
    ("labels_as_int", str, "False"),
    ("seed", int, 104),
    ("gpu_to_use", int, None),
    ("num_dataprovider_workers", int, 4),
    ("max_models_to_save", int, 5),
    ("dataset_name", str, "omniglot_dataset"),
    ("dataset_path", str, "datasets/omniglot_dataset"),
    ("reset_stored_paths", str, "False"),
    ("experiment_name", str, None),
    ("architecture_name", str, None),
    ("continue_from_epoch", str, "latest"),
    ("dropout_rate_value", float, 0.3),
    ("num_target_samples", int, 15),
    ("second_order", str, "False"),
    ("total_epochs", int, 200),
    ("total_iter_per_epoch", int, 500),
    ("min_learning_rate", float, 0.00001),
    ("meta_learning_rate", float, 0.001),
    ("meta_opt_bn", str, "False"),
    ("task_learning_rate", float, 0.1),
    ("norm_layer", str, "batch_norm"),
    ("max_pooling", str, "False"),
    ("per_step_bn_statistics", str, "False"),
    ("num_classes_per_set", int, 20),
    ("cnn_num_blocks", int, 4),
    ("number_of_training_steps_per_iter", int, 1),
    ("number_of_evaluation_steps_per_iter", int, 1),
    ("cnn_num_filters", int, 64),
    ("cnn_blocks_per_stage", int, 1),
    ("num_samples_per_class", int, 1),
    ("name_of_args_json_file", str, "None"),
]

# Keys the hot path reads that only ever come from the JSON files; defaults used when a
# caller builds args programmatically (bench / tests) without a JSON file.
_JSON_ONLY_DEFAULTS = {
    "num_stages": 4,
    "conv_padding": True,
    "learnable_bn_gamma": True,
    "learnable_bn_beta": True,
    "enable_inner_loop_optimizable_bn_params": False,
    "learnable_per_layer_per_step_inner_loop_learning_rate": False,
    "use_multi_step_loss_optimization": False,
    "multi_step_loss_num_epochs": 10,
    "first_order_to_second_order_epoch": -1,
    "total_epochs_before_pause": 100,
    "train_seed": 0,
    "val_seed": 0,
}


class Bunch(object):
    """Attribute bag, same role as the reference's ``Bunch`` (utils/parser_utils.py:92-94)."""

    def __init__(self, adict):
        self.__dict__.update(adict)

    def __repr__(self):
        return "Bunch(%r)" % (self.__dict__,)


def _boolify(d):
    for key in list(d.keys()):
        s = str(d[key]).lower()
        if s == "true":
            d[key] = True
        elif s == "false":
            d[key] = False
    return d


def default_args_dict():
    d = {name: default for name, _, default in _DEFAULTS}
    d.update(_JSON_ONLY_DEFAULTS)
    return d


def extract_args_from_json(json_file_path, args_dict):
    """JSON keys override the dict, except continue_from*/gpu_to_use (reference :96-106)."""
    with open(json_file_path) as f:
        summary = json.load(f)
    for key, value in summary.items():
        if "continue_from" not in key and "gpu_to_use" not in key:
            args_dict[key] = value
    return args_dict


def args_from_json(json_file_path=None, require_dataset_dir=False, **overrides):
    """Build the args Bunch the way the reference does, without touching ``sys.argv``.

    ``overrides`` are applied last (used by bench/tests to change e.g. ``batch_size``).
    """
    d = default_args_dict()
    if json_file_path is not None:
        d["name_of_args_json_file"] = json_file_path
        d = extract_args_from_json(json_file_path, d)
    d.update(overrides)
    d = _boolify(d)
    if require_dataset_dir:
        d["dataset_path"] = os.path.join(os.environ["DATASET_DIR"], d["dataset_path"])
    elif "DATASET_DIR" in os.environ:
        d["dataset_path"] = os.path.join(os.environ["DATASET_DIR"], d["dataset_path"])
    args = Bunch(d)
    _finish(args)
    return args


def _finish(args):
    import torch
    args.use_cuda = torch.cuda.is_available()


def get_args(argv=None):
    """CLI entry: ``--name_of_args_json_file cfg.json --gpu_to_use N`` like the reference.

    Returns ``(args, device)``.
    """
    import torch

    parser = argparse.ArgumentParser(description="H100-native MAML++ training system")
    for name, typ, default in _DEFAULTS:
        if name in ("gpu_to_use", "experiment_name", "architecture_name"):
            parser.add_argument("--" + name, nargs="?", type=typ)
        else:
            parser.add_argument("--" + name, nargs="?", type=typ, default=default)
    ns = parser.parse_args(argv)
    d = dict(_JSON_ONLY_DEFAULTS)
    d.update(vars(ns))
    if ns.name_of_args_json_file != "None":
        d = extract_args_from_json(ns.name_of_args_json_file, d)
    d = _boolify(d)
    # the reference raises KeyError when DATASET_DIR is unset (parser_utils.py:67-69); the
    # hot path itself never reads dataset_path, so only prefix when it is available.
    if "DATASET_DIR" in os.environ:
        d["dataset_path"] = os.path.join(os.environ["DATASET_DIR"], d["dataset_path"])
    args = Bunch(d)
    _finish(args)
    if torch.cuda.is_available():
        device = torch.device("cuda", torch.cuda.current_device())
    else:
        device = torch.device("cpu")
    return args, device
