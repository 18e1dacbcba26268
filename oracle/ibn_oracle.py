"""ORACLE TOOLING -- TEST INFRASTRUCTURE ONLY.  The fp64 oracle of the network with
``enable_inner_loop_optimizable_bn_params`` is ``oracle/maml_oracle.py``, which branches on the flag; this module keeps the
entry points under the name that existing test code and scripts import.  It holds no arithmetic of its own."""
from oracle.maml_oracle import autograd_train_iter, inner_param_names, manual_train_iter, trainable_names  # noqa: F401
