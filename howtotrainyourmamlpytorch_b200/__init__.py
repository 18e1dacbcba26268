"""H100-native MAML / MAML++ inner-loop engine behind the reference's Python surface.

Public surface (same names as the reference repo's modules):
  few_shot_learning_system.MAMLFewShotClassifier      -- B0: run_train_iter / run_validation_iter
  meta_neural_network_architectures.VGGReLUNormNetwork -- B1: parameter container (state_dict names)
  inner_loop_optimizers.LSLRGradientDescentLearningRule -- B2
  utils.parser_utils.get_args / args_from_json          -- JSON config schema
The arithmetic runs in ``lib/libmaml_b200.so`` (C ABI: ``include/maml_b200.h``), built in-tree by
``python -m howtotrainyourmamlpytorch_b200.build``.  Importing the package does not need a GPU.
"""
from .configs import CONFIGS, make_args  # noqa: F401
from .few_shot_learning_system import MAMLFewShotClassifier  # noqa: F401
from .inner_loop_optimizers import LSLRGradientDescentLearningRule  # noqa: F401
from .meta_neural_network_architectures import VGGReLUNormNetwork  # noqa: F401
from .synthetic import synthetic_batch  # noqa: F401

__version__ = "0.1.0"
