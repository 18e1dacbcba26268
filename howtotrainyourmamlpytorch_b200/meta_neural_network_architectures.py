"""Functional-network surface (level B1 of the drop-in boundary, SURVEY.md section 8b).

The reference's ``VGGReLUNormNetwork`` (``meta_neural_network_architectures.py:545-688``) is a
4-block conv3x3 -> BatchNorm(batch statistics, per-step gamma/beta) -> leaky-ReLU -> maxpool2 net
followed by a linear layer, all taking externally supplied ("fast") weights.  Here the classes keep
the reference's module tree and parameter names -- so ``state_dict`` keys, shapes, registration
order (= Adam parameter order) and initialisation RNG consumption are identical -- but they are
parameter containers: the arithmetic of the path runs in the CUDA engine (``csrc/``), which sees
these parameters as one flat buffer.  ``VGGReLUNormNetwork.forward`` is the functional-network operator of the
boundary (level B1): forward, backward and the backward of that backward (second-order MAML) all run on the engine
through ``torch.autograd.Function``.

Initialisation restates reference ``:62-66`` (xavier_uniform_ conv weight, zero bias),
``:114-118`` (xavier_uniform_ linear weights), ``:177-192`` (running_mean zeros; running_var ones
per-step but ZEROS in shared mode; beta zeros; gamma ones).
"""
import itertools

import torch
import torch.autograd.forward_ad as fwAD
import torch.nn as nn


class MetaConv2dLayer(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, use_bias, groups=1, dilation_rate=1):
        super().__init__()
        if int(kernel_size) != 3 or int(stride) != 1 or int(padding) != 1 or int(groups) != 1 or int(dilation_rate) != 1:
            raise NotImplementedError("the engine implements the shipped configuration only: 3x3, stride 1, "
                                      "padding 1 (max_pooling=true, conv_padding=true)")
        self.stride, self.padding, self.dilation_rate, self.groups, self.use_bias = 1, 1, 1, 1, bool(use_bias)
        self.weight = nn.Parameter(torch.empty(out_channels, in_channels, 3, 3))
        nn.init.xavier_uniform_(self.weight)
        if self.use_bias:
            self.bias = nn.Parameter(torch.zeros(out_channels))


class MetaLinearLayer(nn.Module):
    def __init__(self, input_shape, num_filters, use_bias):
        super().__init__()
        _, c = input_shape
        self.use_bias = bool(use_bias)
        self.weights = nn.Parameter(torch.ones(num_filters, int(c)))
        nn.init.xavier_uniform_(self.weights)
        if self.use_bias:
            self.bias = nn.Parameter(torch.zeros(num_filters))


class MetaBatchNormLayer(nn.Module):
    def __init__(self, num_features, device, args, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True,
                 meta_batch_norm=True, no_learnable_params=False, use_per_step_bn_statistics=False):
        super().__init__()
        inner_bn = bool(getattr(args, "enable_inner_loop_optimizable_bn_params", False))
        if inner_bn and not (args.learnable_bn_gamma and args.learnable_bn_beta):
            raise NotImplementedError("enable_inner_loop_optimizable_bn_params with a frozen BatchNorm gamma or beta "
                                      "(learnable_bn_gamma / learnable_bn_beta false) is outside the accelerated path")
        self.num_features, self.eps, self.momentum = int(num_features), eps, momentum
        self.use_per_step_bn_statistics = bool(use_per_step_bn_statistics)
        S = int(args.number_of_training_steps_per_iter)
        shape = (S, self.num_features) if self.use_per_step_bn_statistics else (self.num_features,)
        self.running_mean = nn.Parameter(torch.zeros(shape), requires_grad=False)
        self.running_var = nn.Parameter(torch.ones(shape) if self.use_per_step_bn_statistics else torch.zeros(shape),
                                        requires_grad=False)
        self.bias = nn.Parameter(torch.zeros(shape), requires_grad=bool(args.learnable_bn_beta))
        self.weight = nn.Parameter(torch.ones(shape), requires_grad=bool(args.learnable_bn_gamma))
        if inner_bn:
            # reference :194-198: inner-loop gamma / beta are one [F] row each, even with per-step statistics; re-assigned
            # into their slots, so the registration order stays running_mean, running_var, bias, weight
            self.bias = nn.Parameter(torch.zeros(self.num_features), requires_grad=True)
            self.weight = nn.Parameter(torch.ones(self.num_features), requires_grad=True)
        if self.use_per_step_bn_statistics:
            # Reference quirk: while building itself the reference network pushes an all-zero dummy batch
            # through every block twice with num_step=0 (build_block :365 and build_network :603), and
            # F.batch_norm's EMA side effect leaves running_var[0] = 0.9 * 0.9 * 1 (fp32) in a fresh model.
            with torch.no_grad():
                for _ in range(2):
                    self.running_var[0].mul_(1.0 - momentum)


class MetaLayerNormLayer(nn.Module):
    """Reference ``MetaLayerNormLayer`` (:261-322): ``F.layer_norm`` over the conv output [F, h, w] of each image (the size
    BEFORE pooling), eps 1e-5.  ``weight`` is registered first, as ones with ``requires_grad=False``: the reference never
    trains it, but ``F.layer_norm`` multiplies by it, so the engine accepts only all-ones weights (it adds the bias to the
    normalised values).  ``bias`` [F, h, w] is an outer (Adam) parameter, not adapted in the inner loop.  No running
    statistics, no per-step index."""

    def __init__(self, input_feature_shape, eps=1e-5, elementwise_affine=True):
        super().__init__()
        if not elementwise_affine:
            raise NotImplementedError("MetaLayerNormLayer without elementwise_affine is not on the accelerated path "
                                      "(the reference network always builds it with the affine parameters)")
        self.normalized_shape = torch.Size(int(d) for d in input_feature_shape)
        self.eps = eps
        self.elementwise_affine = True
        self.weight = nn.Parameter(torch.ones(self.normalized_shape), requires_grad=False)
        self.bias = nn.Parameter(torch.zeros(self.normalized_shape))

    def restore_backup_stats(self):
        pass


class MetaConvNormLayerReLU(nn.Module):
    def __init__(self, input_shape, num_filters, kernel_size, stride, padding, use_bias, args, normalization=True,
                 meta_layer=True, no_bn_learnable_params=False, device=None):
        super().__init__()
        norm = getattr(args, "norm_layer", "batch_norm")
        if not normalization or norm not in ("batch_norm", "layer_norm"):
            raise NotImplementedError("only norm_layer='batch_norm' or 'layer_norm' is on the accelerated path")
        self.layer_dict = nn.ModuleDict()
        self.conv = MetaConv2dLayer(in_channels=int(input_shape[1]), out_channels=num_filters, kernel_size=kernel_size,
                                    stride=stride, padding=padding, use_bias=use_bias)
        if norm == "layer_norm":
            if getattr(args, "enable_inner_loop_optimizable_bn_params", False):
                raise NotImplementedError("enable_inner_loop_optimizable_bn_params with norm_layer='layer_norm' is "
                                          "outside the accelerated path")
            # normalized_shape = the conv output of one image: 3x3 / stride 1 / padding 1 keeps h x w
            self.norm_layer = MetaLayerNormLayer(input_feature_shape=(num_filters, int(input_shape[2]), int(input_shape[3])))
        else:
            self.norm_layer = MetaBatchNormLayer(num_filters, device=device, args=args,
                                                 use_per_step_bn_statistics=args.per_step_bn_statistics)


class VGGReLUNormNetwork(nn.Module):
    def __init__(self, im_shape, num_output_classes, args, device, meta_classifier=True):
        super().__init__()
        if not args.max_pooling:
            raise NotImplementedError("strided-conv / avg-pool variant (max_pooling=false) is outside the "
                                      "accelerated path (all shipped configs use max pooling)")
        _, c, h, w = im_shape
        self.args, self.device = args, device
        self.num_stages = int(args.num_stages)
        self.cnn_filters = int(args.cnn_num_filters)
        self.num_output_classes = int(num_output_classes)
        self.layer_dict = nn.ModuleDict()
        shape = [int(im_shape[0]), int(c), int(h), int(w)]
        for i in range(self.num_stages):
            self.layer_dict["conv%d" % i] = MetaConvNormLayerReLU(
                input_shape=shape, num_filters=self.cnn_filters, kernel_size=3, stride=1,
                padding=int(bool(args.conv_padding)), use_bias=True, args=args, device=device)
            shape = [shape[0], self.cnn_filters, shape[2] // 2, shape[3] // 2]
            if shape[2] < 1 or shape[3] < 1:
                raise ValueError("image too small for %d stages" % self.num_stages)
        self.encoder_features_shape = list(shape)
        feat = shape[1] * shape[2] * shape[3]
        self.layer_dict["linear"] = MetaLinearLayer(input_shape=(shape[0], feat), num_filters=self.num_output_classes,
                                                    use_bias=True)

    def _layer_norm(self):
        return getattr(self.args, "norm_layer", "batch_norm") == "layer_norm"

    def _inner_bn(self):
        """BatchNorm gamma / beta are inner-loop fast weights (enable_inner_loop_optimizable_bn_params)."""
        return bool(getattr(self.args, "enable_inner_loop_optimizable_bn_params", False))

    def _segment_names(self):
        """The operator's tensors in the engine's meta-vector order: per block conv.weight, conv.bias, then BatchNorm's
        norm_layer.bias / norm_layer.weight (beta / gamma) or the layer norm's norm_layer.bias [F, h, w] alone (its frozen
        all-ones weight is not a segment); then the linear layer."""
        norm = ("norm_layer.bias",) if self._layer_norm() else ("norm_layer.bias", "norm_layer.weight")
        names = []
        for i in range(self.num_stages):
            names += ["layer_dict.conv%d.%s" % (i, n) for n in ("conv.weight", "conv.bias") + norm]
        return names + ["layer_dict.linear.weights", "layer_dict.linear.bias"]

    def _norm_segments(self):
        """(indices of the norm parameters among ``_segment_names``, whether the engine's tangent passes take directions
        along them).  The layer-norm biases do (a bias tangent enters after the normalisation), and so do BatchNorm gamma
        / beta when they are inner-loop fast weights (enable_inner_loop_optimizable_bn_params: per task, like the conv
        weights); the shared per-step gamma / beta of a plain BatchNorm network do not."""
        idx = tuple(i for i, n in enumerate(self._segment_names()) if ".norm_layer." in n)
        return idx, self._layer_norm() or self._inner_bn()

    def _segment_tensors(self, params):
        """Tensors in the engine's meta-vector order (``_segment_names``): ``params``' entries, else the module's own."""
        own = dict(self.named_parameters())
        fast = self._fast(params)
        return [fast.get(n, own[n]) for n in self._segment_names()]

    def _fast(self, params):
        """``params`` keyed like the module's own parameters, without the reference's replica dim."""
        own = dict(self.named_parameters())
        fast = {}
        if params is not None:
            for k, v in params.items():
                k = k.replace("module.", "")
                fast[k] = v[0] if v.dim() == own[k].dim() + 1 else v   # strip the reference's replica dim
        return fast

    def _check_layer_norm_weights(self, params=None):
        """The engine applies the layer norm's frozen weight as ones (the reference creates it so and never trains it):
        any other value, in ``params`` or in the module, is refused before anything runs.  The module's own weights are
        checked again only when replaced or modified in place."""
        fast, own = self._fast(params), dict(self.named_parameters())
        ws = [(n, fast.get(n, own[n])) for n in ("layer_dict.conv%d.norm_layer.weight" % l for l in range(self.num_stages))]
        key = tuple((n in fast, w.data_ptr(), w._version) for n, w in ws)
        if not any(n in fast for n, _ in ws) and key == self.__dict__.get("_ln_weight_key"):
            return
        for n, w in ws:
            if not bool(torch.all(w.detach() == 1)):
                raise ValueError("%s is not all ones: the layer-norm network runs with the reference's frozen all-ones "
                                 "weight only" % n)
        self.__dict__["_ln_weight_key"] = key

    def _handles(self, x, spec=None):
        """The operator's engine handles for x's batch size, device and number of tasks (``spec``: None = one batch, else
        a ``_Tasks``; x then may carry a leading task dim), created on first use.  Each task count torch.func.vmap runs
        with keeps handles sized for it; ``vmap(..., chunk_size=)`` bounds that count, and with it the memory."""
        cache = self.__dict__.setdefault("_operator_handles", {})
        tasks = 1 if spec is None else spec.B
        key = (int(x.shape[-4]), x.device.index) + ((tasks,) if tasks > 1 else ())
        if key not in cache:
            cache[key] = _OperatorHandles(self, x, tasks)
        return cache[key]

    def forward(self, x, num_step, params=None, training=False, backup_running_statistics=False):
        """Logits of a batch under externally supplied ("fast") weights -- reference
        ``VGGReLUNormNetwork.forward`` (:620-660): ``params`` maps ``layer_dict.conv{i}.conv.{weight,bias}`` /
        ``layer_dict.linear.{weights,bias}`` to tensors carrying a leading replica dim (as the reference passes them)
        or not; missing entries fall back to the module's own parameters.  BatchNorm always uses batch statistics
        (the reference hard-codes ``training=True``, :246-247) with the gamma / beta of ``num_step``, and -- like
        ``F.batch_norm`` there -- leaves its EMA update in ``running_mean / running_var[num_step]`` (per-step BN only).
        With ``enable_inner_loop_optimizable_bn_params`` gamma / beta are [F] fast weights, taken from ``params`` (or the
        module) without a step index, as the reference does (:226-234); ``num_step`` then selects only the running-
        statistics row.
        The layer-norm network (``norm_layer: "layer_norm"``) normalises each image on its own, adds the bias
        [F, h, w] (an outer parameter: differentiable, and a valid tangent or cotangent direction wherever the weights
        are), has no running statistics and ignores ``num_step``; its frozen weight must be all ones (ValueError).

        Runs on the CUDA engine (C ABI ``maml_b200_net_forward`` / ``maml_b200_net_backward``) and is differentiable
        through ``torch.autograd`` with respect to every weight it uses (conv / linear fast weights, BatchNorm gamma /
        beta), which is what the reference's ``apply_inner_loop_update`` needs (``torch.autograd.grad`` of the support
        loss, few_shot_learning_system.py:138-139).  Twice differentiable: with ``create_graph=True`` the returned
        gradients are differentiable w.r.t. the weights (and the upstream d(logits)) through ``maml_b200_net_hvp``, so the
        reference's second-order loop runs on this operator (a layer-norm bias gradient too, and an inner-loop BatchNorm
        gamma / beta gradient); a plain BatchNorm network's gamma / beta gradient is not (see ``_FunctionalBackward``).  When ``x`` requires grad the operator is differentiable w.r.t. the images too
        (``maml_b200_net_input_grad``), and with ``create_graph=True`` the weight gradients are differentiable w.r.t. ``x``
        (``maml_b200_net_hvp_input_grad``: the mixed term an outer loss needs to reach support images through the inner
        loop); the image gradient itself is not differentiable again.  With ``x`` not requiring grad none of this runs.
        The batch size must be a multiple of the number of classes (episode shaped).

        ``torch.func`` transforms work too: ``grad`` / ``vjp`` / ``jacrev`` (up to second order) and ``vmap`` over tasks,
        which runs the B mapped calls as ONE engine call with n_tasks = B (``maml_b200_net_*_tasks``) -- images, fast
        weights and upstream cotangents may each be batched or shared.  A plain BatchNorm network's gamma / beta and the
        layer-norm biases stay shared by the tasks (a batched one raises NotImplementedError); inner-loop BatchNorm gamma /
        beta may be batched (per task after the first inner step, as the functorch loop makes them); ``torch.func.jvp`` / ``jacfwd`` /
        ``hessian`` (forward mode runs through ``torch.autograd.forward_ad``) and third order raise it too.  A vmapped
        forward leaves the EMA of its B batches in task order, so a vmapped inner loop updates the running statistics
        step-major (every task's support pass at step s, then every target pass), not task-major as the reference's loop
        over tasks does."""
        from . import _native
        if x.device.type != "cuda":
            if self._inner_bn():
                raise NotImplementedError("VGGReLUNormNetwork.forward on a network with "
                                          "enable_inner_loop_optimizable_bn_params runs on the CUDA engine only (sm_90a): "
                                          "no CPU fallback")
            if self._layer_norm():
                raise NotImplementedError("VGGReLUNormNetwork.forward on the layer-norm network runs on the CUDA engine "
                                          "only (sm_90a): no CPU fallback")
            raise _native.NativeLibraryError("VGGReLUNormNetwork.forward needs a CUDA (sm_90a) device: no CPU fallback")
        n = int(x.shape[0])
        if n % self.num_output_classes != 0:
            raise ValueError("batch size %d is not a multiple of num_output_classes %d" % (n, self.num_output_classes))
        if self._layer_norm():
            self._check_layer_norm_weights(params)
        tensors = self._segment_tensors(params)
        return _FunctionalForward.apply(self, None, x, int(num_step), *tensors)

    def zero_grad(self, params=None):
        """Reference :662-677: clears the gradients of ``params`` (or of the module's own parameters)."""
        if params is None:
            for p in self.parameters():
                p.grad = None
        else:
            for p in params.values():
                if getattr(p, "grad", None) is not None:
                    p.grad = None

    def restore_backup_stats(self):
        """The reference's evaluation backup of the running statistics is ``copy(tensor.data)`` -- an alias of the live
        storage (:240-242) -- so its restore (:250-255) puts the already-mutated values back: a no-op on the values,
        which is what this is."""
        return None


def _f32(t):
    """What the engine reads of a tensor: its values, float32, contiguous."""
    return t.detach().to(torch.float32).contiguous()


class _Tasks:
    """B independent problems run as ONE engine call (what ``torch.func.vmap`` over the operator becomes): which operands
    carry a leading task dim (the others are shared by every task).  Every output of a call with a ``_Tasks`` is per task
    ([B, ...]); a node's backward sums the per-task gradients of a shared operand."""

    def __init__(self, B, x, tensors, directions=()):
        self.B, self.x = int(B), bool(x)
        self.tensors, self.directions = tuple(bool(b) for b in tensors), tuple(bool(b) for b in directions)


class _Needs:
    """Which of d/dx, d/d(dlogits) and the per-tensor d/dtheta a ``_FunctionalHvp`` call computes."""

    def __init__(self, x, dl, tensors):
        self.x, self.dl, self.tensors = bool(x), bool(dl), tuple(bool(b) for b in tensors)


# every engine forward of the operator gets a number, so that a backward can tell whether its forward's activations are
# still the ones a handle holds (and replay the forward first if not)
_FORWARDS = itertools.count(1)


def _batched(spec, n):
    return spec.tensors if spec is not None else (False,) * n


def _images(x, spec, B):
    """x as the engine reads it: [B, n, C, H, W] float32 (a shared batch copied per task) or, without spec, [n, C, H, W]."""
    return _f32(x if spec is None or spec.x else x.expand(B, *x.shape))


def _fill(eng, buf, tensors, batched):
    """buf[t] <- task t's tensors (None: zeros) in the engine's meta layout.  With no tensor batched only row 0 is
    written and every task reads it (task stride 0); a shared tensor among batched ones is broadcast into every row.
    Returns the task stride in floats."""
    stride = eng.meta_size if any(batched) else 0
    rows = buf if stride else buf[:1]
    with torch.no_grad():
        for (off, size), t, b in zip(eng.segments, tensors, batched):
            if t is None:
                rows[:, off:off + size].zero_()
            else:
                rows[:, off:off + size].copy_(t.detach().reshape(rows.shape[0] if b else 1, size).to(torch.float32))
    return stride


def _unpack(eng, buf, tensors, needs, spec, cast=False):
    """Per-tensor copies of an engine result buffer [B, result_size] (None where not needed): [B, *shape] per task with a
    spec, the tensor's own shape without; in each tensor's dtype when `cast`."""
    out = []
    for (off, size), t, need, b in zip(eng.segments, tensors, needs, _batched(spec, len(tensors))):
        if not need:
            out.append(None)
            continue
        v = buf[0, off:off + size].view(t.shape) if spec is None else buf[:, off:off + size].view(-1, *t.shape[int(b):])
        out.append(v.to(t.dtype if cast else buf.dtype, copy=True))
    return out


def _image_buffer(buf, x, B):
    """`buf`, or on first use an engine output buffer for the image gradients of B batches shaped like x's."""
    return buf if buf is not None else torch.empty((B,) + tuple(x.shape[-4:]), dtype=torch.float32, device=x.device)


def _add(a, b):
    return a if b is None else b if a is None else a + b


def _per_task(t, batched, B):
    """t with a leading task dim: itself when batched, else a stride-0 view."""
    return t if batched else t.unsqueeze(0).expand(B, *t.shape)


def _to_front(t, dim):
    return t if t is None or dim is None else t.movedim(dim, 0)


def _shared_sum(g, batched):
    """The gradient of an operand from per-task gradients g [B, ...]: g itself if the operand is batched, else (shared by
    the tasks) their sum."""
    return g if g is None or batched else g.sum(0)


def _refuse_nested(spec):
    if spec is not None:
        raise NotImplementedError("nested torch.func.vmap over the functional network operator is not supported: the "
                                  "engine has one task dimension (flatten the task dims into one vmap)")


def _refuse_batched_norm(net, dims):
    """Inner-loop BatchNorm gamma / beta are per-task fast weights: batched ones are what the functorch loop passes after
    its first inner step.  The other norm parameters are shared by the tasks of a call."""
    if net._inner_bn():
        return
    if any(dims[i] is not None for i in net._norm_segments()[0]):
        if net._layer_norm():
            raise NotImplementedError(
                "a layer-norm bias batched under torch.func.vmap: the engine shares the layer-norm biases between the "
                "tasks of a call (they are outer parameters, the same for every task)")
        raise NotImplementedError(
            "a BatchNorm gamma / beta batched under torch.func.vmap: the engine shares gamma / beta between the tasks "
            "of a call (per-task gamma / beta are inner-loop BatchNorm parameters: set "
            "enable_inner_loop_optimizable_bn_params)")


def _refuse_functorch_jvp(ctx, *tensors):
    if getattr(ctx, "spec", None) is not None or any(
            isinstance(t, torch.Tensor) and torch._C._functorch.is_functorch_wrapped_tensor(t)
            for t in tuple(ctx.saved_tensors) + tensors):
        raise NotImplementedError(
            "torch.func.jvp / jacfwd / hessian through the functional network operator are not supported: its forward "
            "mode runs through torch.autograd.forward_ad (fwAD.dual_level / make_dual), and reverse mode through "
            "torch.func.grad / vjp / jacrev")


def _refuse_third_order():
    raise NotImplementedError("third-order derivatives of the functional network operator are not supported (the "
                              "engine differentiates its backward once: second-order MAML)")


class _OperatorHandles:
    """The engine handles behind ``VGGReLUNormNetwork.forward`` for one batch size, device and task count B (1, or the
    batch size of a ``torch.func.vmap`` over tasks), one method per use.

    The first-order handle holds the batch as its target pass (``maml_b200_net_forward_tasks`` / ``net_backward_tasks``
    / ``net_input_grad``, the running-statistics update).  It keeps the activations of its LAST forward only: ``token``
    names that forward, so that a backward of another one replays its own first (``gen`` counts the forwards it ran).  The second-order handle, created on first
    use, holds the batch as its SUPPORT pass, the buffers the tangent pass runs on (``net_hvp_image_tasks`` /
    ``net_hvp_input_grad`` / ``net_jvp_tasks``): a model that is only differentiated once pays nothing for it.  Every call
    runs the per-task entries with per-task results; for B = 1 and shared weights they compute what ``net_forward`` /
    ``net_backward`` / ``net_hvp_image`` / ``net_jvp`` do, bit for bit.  A network with inner-loop BatchNorm gamma / beta
    gets inner_bn handles, which run the per-task entries only: their gamma / beta follow each task's weights."""

    def __init__(self, net, x, tasks):
        a = net.args
        self.B = int(tasks)
        self.n, self.N, self.device = int(x.shape[-4]), net.num_output_classes, x.device
        self.layer_norm, self.inner_bn = net._layer_norm(), net._inner_bn()
        self.cfg = dict(n_way=self.N, channels=int(x.shape[-3]), height=int(x.shape[-2]), width=int(x.shape[-1]),
                        filters=net.cnn_filters, num_stages=net.num_stages, inner_steps=int(a.number_of_training_steps_per_iter),
                        per_step_bn=bool(a.per_step_bn_statistics), max_tasks=self.B)
        self.first_order = eng = self._engine(k_shot=1, t_target=self.n // self.N)
        self.token, self.gen = None, 0
        self.meta = torch.zeros(self.B, eng.meta_size, dtype=torch.float32, device=self.device)
        self.meta_stride = 0
        self.logits = torch.empty(self.B, self.n, self.N, dtype=torch.float32, device=self.device)
        self.grad = torch.zeros(self.B, eng.result_size, dtype=torch.float32, device=self.device)
        S = int(a.number_of_training_steps_per_iter) if a.per_step_bn_statistics else 1
        self.run = torch.zeros(2, net.num_stages, S, net.cnn_filters, dtype=torch.float32, device=self.device)
        self.dx = self.second_order = self.dxdot = None

    def _engine(self, **shape):
        from . import _native
        with torch.cuda.device(self.device):
            return _native.Engine(**shape, **self.cfg, layer_norm=self.layer_norm, inner_bn=self.inner_bn)

    def _second(self):
        if self.second_order is None:
            eng = self._engine(k_shot=self.n // self.N, t_target=1)
            self.meta2 = torch.zeros(self.B, eng.meta_size, dtype=torch.float32, device=self.device)
            self.v = torch.zeros(self.B, eng.meta_size, dtype=torch.float32, device=self.device)
            self.jv = torch.empty(self.B, self.n, self.N, dtype=torch.float32, device=self.device)
            self.hv = torch.zeros(self.B, eng.result_size, dtype=torch.float32, device=self.device)
            self.second_order = eng
        return self.second_order

    def _out(self, buf, spec, dtype=None):
        """An engine output [B, ...] as the caller's copy: per task with a spec, else batch 0's."""
        return (buf if spec is not None else buf[0]).to(dtype or buf.dtype, copy=True)

    def _run_forward(self, spec, x, num_step, tensors):
        eng = self.first_order
        self.meta_stride = _fill(eng, self.meta, tensors, _batched(spec, len(tensors)))
        eng.net_forward_tasks(self.B, num_step, self.meta, self.meta_stride, _images(x, spec, self.B), self.logits)
        self.gen += 1

    def forward(self, net, spec, x, num_step, tensors):
        """The logits (``net_forward_tasks``), and F.batch_norm's EMA of net's running statistics at num_step from the B
        batches in task order (per-step BatchNorm only; the layer norm has no running statistics)."""
        eng = self.first_order
        with torch.cuda.device(self.device):
            self._run_forward(spec, x, num_step, tensors)
            if net.args.per_step_bn_statistics and not self.layer_norm:
                bns = [net.layer_dict["conv%d" % l].norm_layer for l in range(net.num_stages)]
                with torch.no_grad():
                    for l, bn in enumerate(bns):
                        self.run[0, l].copy_(bn.running_mean.data)
                        self.run[1, l].copy_(bn.running_var.data)
                    eng.net_running_update(self.B, num_step, self.run[0], self.run[1])
                    for l, bn in enumerate(bns):
                        bn.running_mean.data.copy_(self.run[0, l])
                        bn.running_var.data.copy_(self.run[1, l])
        self.token = next(_FORWARDS)
        net.__dict__["_operator_forward"] = self.token
        return self._out(self.logits, spec)

    def backward(self, token, num_step, spec, x, tensors, dl, need_x, needs):
        """J^T dl (``net_backward_tasks``) at the forward named `token`, replayed first when this handle's last forward was
        another one (the replay has no EMA side effect), and J_x^T dl (``net_input_grad``) when need_x.  Returns (dx or
        None, the per-tensor gradients in float32, None where not needed), per task with a spec."""
        eng = self.first_order
        with torch.no_grad(), torch.cuda.device(self.device):
            if self.token != token:
                self._run_forward(spec, x, num_step, tensors)
                self.token = token
            eng.net_backward_tasks(self.B, num_step, self.meta, self.meta_stride, _f32(dl).view(self.B, self.n, self.N),
                                   self.grad)
            dx = None
            if need_x:
                self.dx = _image_buffer(self.dx, x, self.B)
                eng.net_input_grad(self.B, self.dx)
                dx = self._out(self.dx, spec, x.dtype)
            return dx, _unpack(eng, self.grad, tensors, needs, spec)

    def hvp(self, num_step, spec, x, xdot, dlogits, tensors, directions, need_x, needs, cast=False):
        """Along the weight directions and the image tangent xdot (None: none): J v and d/dtheta <dlogits, J v>
        (``net_hvp_image_tasks``), and d/dx <dlogits, J v> (``net_hvp_input_grad``) when need_x.  Returns (d/dx or None,
        J v as float32 [(B,) n, N], the per-tensor d/dtheta as by ``_unpack(..., needs, spec, cast)``)."""
        eng = self._second()
        dirs = spec.directions if spec is not None else (False,) * len(directions)
        ms = _fill(eng, self.meta2, tensors, _batched(spec, len(tensors)))
        ds = _fill(eng, self.v, directions, dirs)
        with torch.cuda.device(self.device):
            eng.net_hvp_image_tasks(self.B, num_step, self.meta2, ms, _images(x, spec, self.B),
                                    None if xdot is None else _f32(xdot), _f32(dlogits).view(self.B, self.n, self.N),
                                    self.v, ds, self.jv, self.hv)
            d_x = None
            if need_x:
                self.dxdot = _image_buffer(self.dxdot, x, self.B)
                eng.net_hvp_input_grad(self.B, self.dxdot)
                d_x = self._out(self.dxdot, spec, x.dtype)
        return d_x, (self.jv if spec is not None else self.jv[0]), _unpack(eng, self.hv, tensors, needs, spec, cast)

    def jvp(self, num_step, x, xdot, tensors, tangents):
        """The logits tangent J_theta t + J_x xdot (``net_jvp_tasks`` at strides 0; xdot may be None; one batch)."""
        eng = self._second()
        _fill(eng, self.meta2, tensors, (False,) * len(tensors))
        _fill(eng, self.v, tangents, (False,) * len(tangents))
        with torch.cuda.device(self.device):
            eng.net_jvp_tasks(1, num_step, self.meta2, 0, _f32(x), self.v, 0, None if xdot is None else _f32(xdot), self.jv)
        return self.jv[0].clone()


class _FunctionalForward(torch.autograd.Function):
    """``VGGReLUNormNetwork.forward`` as an autograd node: forward = ``maml_b200_net_forward_tasks``, backward =
    ``_FunctionalBackward`` (``maml_b200_net_backward_tasks``: head backward for an external d(logits), BatchNorm / pool /
    leaky-ReLU backward, dgrad and wgrad kernels of the engine), itself differentiable once more.  The engine keeps the
    activations of its LAST forward only, so a backward that arrives after another forward of the same shape first replays
    its own forward (cheap) -- correctness does not depend on the call order.

    ``spec`` is None for one batch, or a ``_Tasks`` when the ``vmap`` rule below runs B mapped calls as one: the rule moves
    the batch dims to the front and calls this node again with the spec at the level below, so that the levels above
    (an outer ``torch.autograd`` or ``torch.func.grad``) see a graph.  In ``setup_context`` form for ``torch.func``."""

    @staticmethod
    def forward(net, spec, x, num_step, *tensors):
        return net._handles(x, spec).forward(net, spec, x, num_step, tensors)

    @staticmethod
    def setup_context(ctx, inputs, output):
        net, spec, x, num_step, *tensors = inputs
        # the forward that produced `output` ran last: a torch.func level calls this right after it
        ctx.net, ctx.spec, ctx.num_step, ctx.token = net, spec, num_step, net.__dict__["_operator_forward"]
        # x and the weights themselves: a double backward differentiates w.r.t. them, forward mode at them
        ctx.save_for_backward(x, *tensors)
        ctx.save_for_forward(x, *tensors)

    @staticmethod
    def backward(ctx, dlogits):
        x, tensors = ctx.saved_tensors[0], ctx.saved_tensors[1:]
        norm, directions = ctx.net._norm_segments()
        for i in () if directions else norm:
            if fwAD.unpack_dual(tensors[i]).tangent is not None:
                raise NotImplementedError(
                    "differentiating the gradient in forward mode along a BatchNorm gamma / beta tangent needs gamma / beta "
                    "tangent directions in the backward tangent pass, which the engine implements for inner-loop BatchNorm "
                    "parameters only (enable_inner_loop_optimizable_bn_params), not for the shared per-step gamma / beta")
        out = _FunctionalBackward.apply(ctx, ctx.spec, x, dlogits, *tensors)
        if ctx.spec is not None:
            out = [_shared_sum(o, b) for o, b in zip(out, (ctx.spec.x,) + ctx.spec.tensors)]
        return (None, None, out[0], None) + tuple(out[1:])

    @staticmethod
    def jvp(ctx, _net_t, _spec_t, x_t, _step_t, *tangents):
        """Forward mode (``torch.autograd.forward_ad``): the logits tangent J_theta t + J_x x_t through
        ``maml_b200_net_jvp_tasks`` on the second-order handle -- one primal forward and one tangent forward.  Tangents may sit
        on the images, the conv / linear weights and the BatchNorm gamma / beta or layer-norm biases."""
        _refuse_functorch_jvp(ctx, x_t, *tangents)
        x = ctx.saved_tensors[0]
        return ctx.net._handles(x).jvp(ctx.num_step, x, x_t, ctx.saved_tensors[1:], tangents)

    @staticmethod
    def vmap(info, in_dims, net, spec, x, num_step, *tensors):
        _refuse_nested(spec)
        dims = in_dims[4:]
        _refuse_batched_norm(net, dims)
        spec = _Tasks(info.batch_size, in_dims[2] is not None, [d is not None for d in dims])
        logits = _FunctionalForward.apply(net, spec, _to_front(x, in_dims[2]), num_step,
                                          *[_to_front(t, d) for t, d in zip(tensors, dims)])
        return logits, 0


class _FunctionalBackward(torch.autograd.Function):
    """Backward of ``_FunctionalForward`` as an autograd node of its own, so that ``torch.autograd.grad(...,
    create_graph=True)`` of a loss on the operator's logits can be differentiated again (second-order MAML, reference
    few_shot_learning_system.py:138-139 and the outer ``loss.backward()``).

    forward  = ``maml_b200_net_backward_tasks``: B(dl, theta) = J^T dl for every tensor (conv / linear, BatchNorm gamma /
               beta of ``num_step`` or the layer-norm biases), and -- only when x requires grad -- ``maml_b200_net_input_grad``: J_x^T dl (else
               None).  With grad mode off this is the whole first-order backward.
    backward = ``_FunctionalHvp`` along the cotangents v of the conv / linear gradients (and of the layer-norm bias
               gradients: bias directions, which the engine's tangent forward adds after the normalisation; and of
               inner-loop BatchNorm gamma / beta gradients: gamma / beta directions).  Third order is not supported.
    A cotangent on an inner-loop BatchNorm gamma / beta gradient (enable_inner_loop_optimizable_bn_params) is a gamma /
    beta direction of the tangent pass, per task like the weights' (the engine reads it into the tangent forward's
    gamma-dot / beta-dot and the tangent backward's gamma-dot term).  A cotangent on a plain BatchNorm network's shared
    gamma / beta GRADIENT would need gamma / beta tangent directions shared by the tasks, and one on the image gradient dx
    would need image tangent directions (the first conv's tangent driven by x-dot); the engine's tangent pass has neither:
    both are refused (the second e.g. for a penalty on the image gradient's norm that is differentiated again).  ``spec`` and the ``vmap`` rule as in ``_FunctionalForward``; with a
    spec, dlogits is [B, n, N] and every gradient is per task."""

    @staticmethod
    def forward(fwd_ctx, spec, x, dlogits, *tensors):
        need = fwd_ctx.needs_input_grad
        dx, grads = fwd_ctx.net._handles(x, spec).backward(fwd_ctx.token, fwd_ctx.num_step, spec, x, tensors, dlogits,
                                                           need[2], need[4:])
        return (dx,) + tuple(grads)

    @staticmethod
    def setup_context(ctx, inputs, output):
        fwd_ctx, spec, x, dlogits, *tensors = inputs
        ctx.set_materialize_grads(False)
        ctx.fwd_ctx, ctx.spec = fwd_ctx, spec
        ctx.save_for_backward(x, dlogits, *tensors)
        ctx.save_for_forward(x, dlogits, *tensors)

    @staticmethod
    def jvp(ctx, _fwd_ctx_t, _spec_t, x_t, dl_t, *tangents):
        """Forward-over-reverse: the tangent of every gradient this node returned, along (x_t, dl_t, tangents).  For a
        weight gradient J_theta^T dl_t + d/dtheta <dl, J_theta t + J_x x_t>; for dx the same with d/dx.  The first term is
        ``maml_b200_net_backward_tasks`` (+ ``net_input_grad``) of dl_t on the first-order handle, the second
        ``maml_b200_net_hvp_image_tasks`` (+ ``net_hvp_input_grad``) on the second-order handle; a term whose tangents are
        all None is skipped.  A layer-norm bias tangent is a bias direction of that pass, an inner-loop BatchNorm gamma /
        beta tangent a gamma / beta direction.  A tangent on a plain BatchNorm network's gamma / beta never gets here:
        ``_FunctionalForward.backward`` refuses it before this node runs."""
        _refuse_functorch_jvp(ctx, x_t, dl_t, *tangents)
        fwd_ctx = ctx.fwd_ctx
        x, dlogits, tensors = ctx.saved_tensors[0], ctx.saved_tensors[1], ctx.saved_tensors[2:]
        ops, need = fwd_ctx.net._handles(x), fwd_ctx.needs_input_grad
        dx_t, grads_t = None, [None] * len(tensors)
        if dl_t is not None:                              # J^T dl_t on the first-order handle
            dx_t, grads_t = ops.backward(fwd_ctx.token, fwd_ctx.num_step, None, x, tensors, dl_t, need[2], need[4:])
        if x_t is not None or any(t is not None for t in tangents):    # d/d(theta, x) <dl, J_theta t + J_x x_t>
            d_x, _, hv = ops.hvp(fwd_ctx.num_step, None, x, x_t, dlogits, tensors, tangents, need[2], need[4:])
            dx_t = _add(dx_t, d_x)
            grads_t = [_add(g, h) for g, h in zip(grads_t, hv)]
        return (dx_t if need[2] else None,) + tuple(grads_t)

    @staticmethod
    def backward(ctx, dx_cotangent, *cotangents):
        fwd_ctx = ctx.fwd_ctx
        x, dlogits, tensors = ctx.saved_tensors[0], ctx.saved_tensors[1], ctx.saved_tensors[2:]
        if dx_cotangent is not None:
            raise NotImplementedError(
                "differentiating through the gradient with respect to the images needs image tangent directions, which "
                "the engine's tangent pass does not implement")
        norm, directions = fwd_ctx.net._norm_segments()
        for i in () if directions else norm:
            if cotangents[i] is not None:
                raise NotImplementedError(
                    "differentiating through the gradient of a BatchNorm gamma / beta needs gamma / beta tangent "
                    "directions, which the engine implements for inner-loop BatchNorm parameters only "
                    "(enable_inner_loop_optimizable_bn_params), not for the shared per-step gamma / beta")
        if all(c is None for c in cotangents):
            return (None,) * (4 + len(tensors))
        need = ctx.needs_input_grad
        spec = ctx.spec
        if spec is not None:       # the cotangents of per-task gradients are per task
            spec = _Tasks(spec.B, spec.x, spec.tensors, [True] * len(tensors))
        out = _FunctionalHvp.apply(fwd_ctx, spec, _Needs(need[2], need[3], need[4:]), x, dlogits, *tensors, *cotangents)
        if spec is not None:
            out = [_shared_sum(out[0], spec.x), out[1]] + [_shared_sum(o, b) for o, b in zip(out[2:], spec.tensors)]
        return (None, None) + tuple(out)

    @staticmethod
    def vmap(info, in_dims, fwd_ctx, spec, x, dlogits, *tensors):
        _refuse_nested(spec)
        dims = in_dims[4:]
        _refuse_batched_norm(fwd_ctx.net, dims)
        B = info.batch_size
        spec = _Tasks(B, in_dims[2] is not None, [d is not None for d in dims])
        out = _FunctionalBackward.apply(fwd_ctx, spec, _to_front(x, in_dims[2]),
                                        _per_task(_to_front(dlogits, in_dims[3]), in_dims[3] is not None, B),
                                        *[_to_front(t, d) for t, d in zip(tensors, dims)])
        return out, tuple(None if o is None else 0 for o in out)


class _FunctionalHvp(torch.autograd.Function):
    """Backward of ``_FunctionalBackward``: along the cotangents v of the conv / linear (and layer-norm bias, or inner-loop
    BatchNorm gamma / beta) gradients,
    ``maml_b200_net_hvp_image_tasks`` -- one forward-over-reverse pass with dl held constant -- gives J v (the cotangent of
    dl) and d/dtheta <dl, J v> (that of every tensor); ``maml_b200_net_hvp_input_grad`` on the same handle gives
    d/dx <dl, J v> (that of x) when ``needs.x``.  torch carries J v on through the loss's own double backward.  A node of its
    own so that ``torch.func.vmap`` can run it per task; its own backward (third order) is refused."""

    @staticmethod
    def forward(fwd_ctx, spec, needs, x, dlogits, *tensors_and_directions):
        k = len(tensors_and_directions) // 2
        tensors, directions = tensors_and_directions[:k], tensors_and_directions[k:]
        d_x, jv, hv = fwd_ctx.net._handles(x, spec).hvp(fwd_ctx.num_step, spec, x, None, dlogits, tensors, directions,
                                                        needs.x, needs.tensors, cast=True)
        return (d_x, jv.to(dlogits.dtype).clone() if needs.dl else None) + tuple(hv)

    @staticmethod
    def setup_context(ctx, inputs, output):
        pass

    @staticmethod
    def backward(ctx, *cotangents):
        _refuse_third_order()

    @staticmethod
    def vmap(info, in_dims, fwd_ctx, spec, needs, x, dlogits, *tensors_and_directions):
        _refuse_nested(spec)
        k = len(tensors_and_directions) // 2
        dims = in_dims[5:]
        _refuse_batched_norm(fwd_ctx.net, dims[:k])
        B = info.batch_size
        spec = _Tasks(B, in_dims[3] is not None, [d is not None for d in dims[:k]], [d is not None for d in dims[k:]])
        out = _FunctionalHvp.apply(fwd_ctx, spec, needs, _to_front(x, in_dims[3]),
                                   _per_task(_to_front(dlogits, in_dims[4]), in_dims[4] is not None, B),
                                   *[_to_front(t, d) for t, d in zip(tensors_and_directions, dims)])
        return out, tuple(None if o is None else 0 for o in out)
