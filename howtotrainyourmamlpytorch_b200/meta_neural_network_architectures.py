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
        if getattr(args, "enable_inner_loop_optimizable_bn_params", False):
            raise NotImplementedError("enable_inner_loop_optimizable_bn_params is outside the accelerated path "
                                      "(no shipped config sets it)")
        self.num_features, self.eps, self.momentum = int(num_features), eps, momentum
        self.use_per_step_bn_statistics = bool(use_per_step_bn_statistics)
        S = int(args.number_of_training_steps_per_iter)
        shape = (S, self.num_features) if self.use_per_step_bn_statistics else (self.num_features,)
        self.running_mean = nn.Parameter(torch.zeros(shape), requires_grad=False)
        self.running_var = nn.Parameter(torch.ones(shape) if self.use_per_step_bn_statistics else torch.zeros(shape),
                                        requires_grad=False)
        self.bias = nn.Parameter(torch.zeros(shape), requires_grad=bool(args.learnable_bn_beta))
        self.weight = nn.Parameter(torch.ones(shape), requires_grad=bool(args.learnable_bn_gamma))
        if self.use_per_step_bn_statistics:
            # Reference quirk: while building itself the reference network pushes an all-zero dummy batch
            # through every block twice with num_step=0 (build_block :365 and build_network :603), and
            # F.batch_norm's EMA side effect leaves running_var[0] = 0.9 * 0.9 * 1 (fp32) in a fresh model.
            with torch.no_grad():
                for _ in range(2):
                    self.running_var[0].mul_(1.0 - momentum)


class MetaConvNormLayerReLU(nn.Module):
    def __init__(self, input_shape, num_filters, kernel_size, stride, padding, use_bias, args, normalization=True,
                 meta_layer=True, no_bn_learnable_params=False, device=None):
        super().__init__()
        if not normalization or getattr(args, "norm_layer", "batch_norm") != "batch_norm":
            raise NotImplementedError("only norm_layer='batch_norm' is on the accelerated path")
        self.layer_dict = nn.ModuleDict()
        self.conv = MetaConv2dLayer(in_channels=int(input_shape[1]), out_channels=num_filters, kernel_size=kernel_size,
                                    stride=stride, padding=padding, use_bias=use_bias)
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

    def _segment_tensors(self, params):
        """Tensors in the engine's meta-vector order (conv.weight, conv.bias, norm.bias, norm.weight per block; linear)."""
        own = dict(self.named_parameters())
        fast = {}
        if params is not None:
            for k, v in params.items():
                k = k.replace("module.", "")
                fast[k] = v[0] if v.dim() == own[k].dim() + 1 else v   # strip the reference's replica dim
        out = []
        for i in range(self.num_stages):
            p = "layer_dict.conv%d." % i
            for n in (p + "conv.weight", p + "conv.bias", p + "norm_layer.bias", p + "norm_layer.weight"):
                out.append(fast.get(n, own[n]))
        for n in ("layer_dict.linear.weights", "layer_dict.linear.bias"):
            out.append(fast.get(n, own[n]))
        return out

    def _operator_engine(self, x):
        """(engine, meta-layout scratch, logits out, gradient out, running-stat scratch) for this batch shape."""
        from . import _native
        n, N = int(x.shape[0]), self.num_output_classes
        key = (n, x.device.index)
        cache = self.__dict__.setdefault("_engines", {})
        if key not in cache:
            a = self.args
            with torch.cuda.device(x.device):
                eng = _native.Engine(n_way=N, k_shot=1, t_target=n // N, channels=int(x.shape[1]), height=int(x.shape[2]),
                                     width=int(x.shape[3]), filters=self.cnn_filters, num_stages=self.num_stages,
                                     inner_steps=int(a.number_of_training_steps_per_iter),
                                     per_step_bn=bool(a.per_step_bn_statistics), max_tasks=1)
            S = int(a.number_of_training_steps_per_iter) if a.per_step_bn_statistics else 1
            cache[key] = {"eng": eng, "gen": 0,
                          "meta": torch.zeros(eng.meta_size, dtype=torch.float32, device=x.device),
                          "logits": torch.empty(1, n, N, dtype=torch.float32, device=x.device),
                          "grad": torch.zeros(eng.result_size, dtype=torch.float32, device=x.device),
                          "run": torch.zeros(2, self.num_stages, S, self.cnn_filters, dtype=torch.float32, device=x.device)}
        return cache[key]

    def _hvp_engine(self, x):
        """Engine of ``maml_b200_net_hvp`` for this batch shape, created on the first double backward: a second handle whose
        SUPPORT buffers (those the tangent pass runs on) hold the batch, so the operator's first-order handle and its
        users pay nothing for them."""
        from . import _native
        st = self._operator_engine(x)
        if "hvp" not in st:
            a, n, N = self.args, int(x.shape[0]), self.num_output_classes
            with torch.cuda.device(x.device):
                eng = _native.Engine(n_way=N, k_shot=n // N, t_target=1, channels=int(x.shape[1]), height=int(x.shape[2]),
                                     width=int(x.shape[3]), filters=self.cnn_filters, num_stages=self.num_stages,
                                     inner_steps=int(a.number_of_training_steps_per_iter),
                                     per_step_bn=bool(a.per_step_bn_statistics), max_tasks=1)
            st["hvp"] = {"eng": eng,
                         "meta": torch.zeros(eng.meta_size, dtype=torch.float32, device=x.device),
                         "v": torch.zeros(eng.meta_size, dtype=torch.float32, device=x.device),
                         "jv": torch.empty(1, n, N, dtype=torch.float32, device=x.device),
                         "hv": torch.zeros(eng.result_size, dtype=torch.float32, device=x.device)}
        return st["hvp"]

    def forward(self, x, num_step, params=None, training=False, backup_running_statistics=False):
        """Logits of a batch under externally supplied ("fast") weights -- reference
        ``VGGReLUNormNetwork.forward`` (:620-660): ``params`` maps ``layer_dict.conv{i}.conv.{weight,bias}`` /
        ``layer_dict.linear.{weights,bias}`` to tensors carrying a leading replica dim (as the reference passes them)
        or not; missing entries fall back to the module's own parameters.  BatchNorm always uses batch statistics
        (the reference hard-codes ``training=True``, :246-247) with the gamma / beta of ``num_step``, and -- like
        ``F.batch_norm`` there -- leaves its EMA update in ``running_mean / running_var[num_step]`` (per-step BN only).

        Runs on the CUDA engine (C ABI ``maml_b200_net_forward`` / ``maml_b200_net_backward``) and is differentiable
        through ``torch.autograd`` with respect to every weight it uses (conv / linear fast weights, BatchNorm gamma /
        beta), which is what the reference's ``apply_inner_loop_update`` needs (``torch.autograd.grad`` of the support
        loss, few_shot_learning_system.py:138-139).  Twice differentiable: with ``create_graph=True`` the returned
        gradients are differentiable w.r.t. the weights (and the upstream d(logits)) through ``maml_b200_net_hvp``, so the
        reference's second-order loop runs on this operator; a BatchNorm gamma / beta gradient is not (see
        ``_FunctionalBackward``).  When ``x`` requires grad the operator is differentiable w.r.t. the images too
        (``maml_b200_net_input_grad``), and with ``create_graph=True`` the weight gradients are differentiable w.r.t. ``x``
        (``maml_b200_net_hvp_input_grad``: the mixed term an outer loss needs to reach support images through the inner
        loop); the image gradient itself is not differentiable again.  With ``x`` not requiring grad none of this runs.
        The batch size must be a multiple of the number of classes (episode shaped)."""
        from . import _native
        if x.device.type != "cuda":
            raise _native.NativeLibraryError("VGGReLUNormNetwork.forward needs a CUDA (sm_90a) device: no CPU fallback")
        n = int(x.shape[0])
        if n % self.num_output_classes != 0:
            raise ValueError("batch size %d is not a multiple of num_output_classes %d" % (n, self.num_output_classes))
        tensors = self._segment_tensors(params)
        return _FunctionalForward.apply(self, x, int(num_step), *tensors)

    def _apply_running_ema(self, st, num_step):
        if not self.args.per_step_bn_statistics:
            return
        run = st["run"]
        with torch.no_grad():
            for l in range(self.num_stages):
                bn = self.layer_dict["conv%d" % l].norm_layer
                run[0, l].copy_(bn.running_mean.data)
                run[1, l].copy_(bn.running_var.data)
            st["eng"].net_running_update(1, num_step, run[0], run[1])
            for l in range(self.num_stages):
                bn = self.layer_dict["conv%d" % l].norm_layer
                bn.running_mean.data.copy_(run[0, l])
                bn.running_var.data.copy_(run[1, l])

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


class _FunctionalForward(torch.autograd.Function):
    """``VGGReLUNormNetwork.forward`` as an autograd node: forward = ``maml_b200_net_forward``, backward =
    ``_FunctionalBackward`` (``maml_b200_net_backward``: head backward for an external d(logits), BatchNorm / pool / leaky-ReLU
    backward, dgrad and wgrad kernels of the engine), itself differentiable once more.  The engine keeps the activations of
    its LAST forward only, so a backward that arrives after another forward of the same shape first replays its own forward
    (cheap) -- correctness does not depend on the call order."""

    @staticmethod
    def forward(ctx, net, x, num_step, *tensors):
        st = net._operator_engine(x)
        eng, meta_like, logits = st["eng"], st["meta"], st["logits"]
        xin = x.detach().to(torch.float32).contiguous()
        with torch.no_grad():
            for (off, size), t in zip(eng.segments, tensors):
                meta_like[off:off + size].copy_(t.detach().reshape(-1).to(torch.float32))
        with torch.cuda.device(x.device):
            eng.net_forward(1, num_step, meta_like, xin, logits)
            net._apply_running_ema(st, num_step)
        st["gen"] += 1
        ctx.net, ctx.num_step, ctx.gen = net, num_step, st["gen"]
        # x and the weights themselves: a double backward differentiates w.r.t. them, forward mode at them
        ctx.save_for_backward(x, *tensors)
        ctx.save_for_forward(x, *tensors)
        return logits[0].clone()

    @staticmethod
    def backward(ctx, dlogits):
        x, tensors = ctx.saved_tensors[0], ctx.saved_tensors[1:]
        for i, t in enumerate(tensors[:4 * ctx.net.num_stages]):
            if i % 4 >= 2 and fwAD.unpack_dual(t).tangent is not None:
                raise NotImplementedError(
                    "differentiating the gradient in forward mode along a BatchNorm gamma / beta tangent needs gamma / beta "
                    "tangent directions in the backward tangent pass, which the engine does not implement (BatchNorm "
                    "parameters as inner-loop fast weights, enable_inner_loop_optimizable_bn_params, are outside the "
                    "accelerated path)")
        out = _FunctionalBackward.apply(ctx, x, dlogits, *tensors)
        return (None, out[0], None) + tuple(out[1:])

    @staticmethod
    def jvp(ctx, _net_t, x_t, _step_t, *tangents):
        """Forward mode (``torch.autograd.forward_ad``): the logits tangent J_theta t + J_x x_t through
        ``maml_b200_net_jvp`` on the second (HVP) handle -- one primal forward and one tangent forward.  Tangents may sit
        on the images, the conv / linear weights and the BatchNorm gamma / beta."""
        x, tensors = ctx.saved_tensors[0], ctx.saved_tensors[1:]
        xin = x.detach().to(torch.float32).contiguous()
        hs = ctx.net._hvp_engine(xin)
        eng, meta_like, t_like, jv = hs["eng"], hs["meta"], hs["v"], hs["jv"]
        _fill_meta(eng, meta_like, tensors, t_like, tangents)
        xdot = None if x_t is None else x_t.detach().to(torch.float32).contiguous()
        with torch.cuda.device(xin.device):
            eng.net_jvp(1, ctx.num_step, meta_like, xin, t_like, xdot, jv)
        return jv[0].clone()


def _fill_meta(eng, meta_like, tensors, v_like, directions):
    """meta_like <- the tensors, v_like <- the directions (None: zero) in the engine's meta layout."""
    with torch.no_grad():
        v_like.zero_()
        for (off, size), t, d in zip(eng.segments, tensors, directions):
            meta_like[off:off + size].copy_(t.detach().reshape(-1).to(torch.float32))
            if d is not None:
                v_like[off:off + size].copy_(d.detach().reshape(-1).to(torch.float32))


def _net_backward(fwd_ctx, xin, tensors, dl, x_dtype):
    """J^T dl on the operator's handle (``maml_b200_net_backward``), after replaying ``fwd_ctx``'s forward when another
    forward of this shape ran since (the handle keeps the activations of its last forward only; the replay has no EMA side
    effect), and J_x^T dl (``maml_b200_net_input_grad``) when x requires grad.  Returns (the handle's state, whose "grad"
    holds the weight gradients in the meta layout; dx or None)."""
    net, num_step = fwd_ctx.net, fwd_ctx.num_step
    st = net._operator_engine(xin)
    eng, meta_like, logits, grad = st["eng"], st["meta"], st["logits"], st["grad"]
    with torch.no_grad(), torch.cuda.device(xin.device):
        if st["gen"] != fwd_ctx.gen:
            for (off, size), t in zip(eng.segments, tensors):
                meta_like[off:off + size].copy_(t.detach().reshape(-1).to(torch.float32))
            eng.net_forward(1, num_step, meta_like, xin, logits)
            st["gen"] += 1
            fwd_ctx.gen = st["gen"]
        eng.net_backward(1, num_step, meta_like, dl.detach().to(torch.float32).contiguous().view(1, *dl.shape), grad)
        dx = None
        if fwd_ctx.needs_input_grad[1]:
            dx = st.setdefault("dx", torch.empty((1,) + tuple(xin.shape), dtype=torch.float32, device=xin.device))
            eng.net_input_grad(1, dx)
            dx = dx[0].to(x_dtype, copy=True)
    return st, dx


class _FunctionalBackward(torch.autograd.Function):
    """Backward of ``_FunctionalForward`` as an autograd node of its own, so that ``torch.autograd.grad(...,
    create_graph=True)`` of a loss on the operator's logits can be differentiated again (second-order MAML, reference
    few_shot_learning_system.py:138-139 and the outer ``loss.backward()``).

    forward  = ``maml_b200_net_backward``: B(dl, theta) = J^T dl for every tensor (conv / linear, BatchNorm gamma / beta of
               ``num_step``), and -- only when x requires grad -- ``maml_b200_net_input_grad``: J_x^T dl (else None).  With
               grad mode off this is the whole first-order backward.
    backward = ``maml_b200_net_hvp`` along the cotangents v of the conv / linear gradients: one forward-over-reverse pass with
               dl held constant gives J v (the cotangent of dl) and d/dtheta <dl, J v> (that of every tensor); when x
               requires grad, ``maml_b200_net_hvp_input_grad`` on the same handle gives d/dx <dl, J v> (that of x).  torch
               carries J v on through the loss's own double backward.  Third order is not supported.
    A cotangent on a BatchNorm gamma / beta GRADIENT would need gamma / beta tangent directions, and one on the image
    gradient dx would need image tangent directions (the first conv's tangent driven by x-dot); the engine's tangent pass
    has neither: both are refused (the first only arises when BatchNorm parameters are inner-loop fast weights,
    enable_inner_loop_optimizable_bn_params, which the network refuses too; the second e.g. for a penalty on the image
    gradient's norm that is differentiated again)."""

    @staticmethod
    def forward(ctx, fwd_ctx, x, dlogits, *tensors):
        net, num_step = fwd_ctx.net, fwd_ctx.num_step
        xin = x.detach().to(torch.float32).contiguous()
        st, dx = _net_backward(fwd_ctx, xin, tensors, dlogits, x.dtype)
        eng, grad = st["eng"], st["grad"]
        ctx.set_materialize_grads(False)
        ctx.net, ctx.num_step, ctx.fwd_ctx = net, num_step, fwd_ctx
        ctx.save_for_backward(x, dlogits, *tensors)
        ctx.save_for_forward(x, dlogits, *tensors)
        grads = []
        for (off, size), t, need in zip(eng.segments, tensors, fwd_ctx.needs_input_grad[3:]):
            grads.append(grad[off:off + size].view(t.shape).clone() if need else None)
        return (dx,) + tuple(grads)

    @staticmethod
    def jvp(ctx, _fwd_ctx_t, x_t, dl_t, *tangents):
        """Forward-over-reverse: the tangent of every gradient this node returned, along (x_t, dl_t, tangents).  For a
        weight gradient J_theta^T dl_t + d/dtheta <dl, J_theta t + J_x x_t>; for dx the same with d/dx.  The first term is
        ``maml_b200_net_backward`` (+ ``net_input_grad``) of dl_t on the operator's handle, the second
        ``maml_b200_net_hvp_image`` (+ ``net_hvp_input_grad``) on the HVP handle; a term whose tangents are all None is
        skipped.  A tangent on a BatchNorm gamma / beta input never gets here: ``_FunctionalForward.backward`` refuses it
        before this node runs."""
        net, num_step, fwd_ctx = ctx.net, ctx.num_step, ctx.fwd_ctx
        x, dlogits, tensors = ctx.saved_tensors[0], ctx.saved_tensors[1], ctx.saved_tensors[2:]
        need_x = fwd_ctx.needs_input_grad[1]
        needs = fwd_ctx.needs_input_grad[3:]
        xin = x.detach().to(torch.float32).contiguous()
        dx_t, grads_t = None, [None] * len(tensors)

        def add(acc, v):
            return v if acc is None else acc + v
        with torch.cuda.device(xin.device):
            if dl_t is not None:                              # J^T dl_t on the operator's handle
                st, dx_t = _net_backward(fwd_ctx, xin, tensors, dl_t, x.dtype)
                eng, grad = st["eng"], st["grad"]
                for k, ((off, size), t) in enumerate(zip(eng.segments, tensors)):
                    if needs[k]:
                        grads_t[k] = add(grads_t[k], grad[off:off + size].view(t.shape).clone())
            if x_t is not None or any(t is not None for t in tangents):    # d/d(theta, x) <dl, J_theta t + J_x x_t>
                hs = net._hvp_engine(xin)
                eng, meta_like, v_like, jv, hv = hs["eng"], hs["meta"], hs["v"], hs["jv"], hs["hv"]
                _fill_meta(eng, meta_like, tensors, v_like, tangents)
                xdot = None if x_t is None else x_t.detach().to(torch.float32).contiguous()
                eng.net_hvp_image(1, num_step, meta_like, xin, xdot,
                                  dlogits.detach().to(torch.float32).contiguous().view(1, *dlogits.shape), v_like, jv, hv)
                if need_x:
                    dxdot = hs.setdefault("dxdot", torch.empty((1,) + tuple(xin.shape), dtype=torch.float32, device=xin.device))
                    eng.net_hvp_input_grad(1, dxdot)
                    dx_t = add(dx_t, dxdot[0].to(x.dtype, copy=True))
                for k, ((off, size), t) in enumerate(zip(eng.segments, tensors)):
                    if needs[k]:
                        grads_t[k] = add(grads_t[k], hv[off:off + size].view(t.shape).clone())
        return (dx_t if need_x else None,) + tuple(grads_t)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dx_cotangent, *cotangents):
        net, num_step = ctx.net, ctx.num_step
        x, dlogits, tensors = ctx.saved_tensors[0], ctx.saved_tensors[1], ctx.saved_tensors[2:]
        if dx_cotangent is not None:
            raise NotImplementedError(
                "differentiating through the gradient with respect to the images needs image tangent directions, which "
                "the engine's tangent pass does not implement")
        xin = x.detach().to(torch.float32).contiguous()
        n_conv = 4 * net.num_stages
        for i, c in enumerate(cotangents[:n_conv]):
            if c is not None and i % 4 >= 2:
                raise NotImplementedError(
                    "differentiating through the gradient of a BatchNorm gamma / beta needs gamma / beta tangent "
                    "directions, which the engine does not implement (BatchNorm parameters as inner-loop fast weights, "
                    "enable_inner_loop_optimizable_bn_params, are outside the accelerated path)")
        if all(c is None for c in cotangents):
            return (None,) * (3 + len(tensors))
        hs = net._hvp_engine(xin)
        eng, meta_like, v_like, jv, hv = hs["eng"], hs["meta"], hs["v"], hs["jv"], hs["hv"]
        with torch.no_grad():
            v_like.zero_()
            for (off, size), t, c in zip(eng.segments, tensors, cotangents):
                meta_like[off:off + size].copy_(t.reshape(-1).to(torch.float32))
                if c is not None:
                    v_like[off:off + size].copy_(c.reshape(-1).to(torch.float32))
        with torch.cuda.device(xin.device):
            eng.net_hvp(1, num_step, meta_like, xin, dlogits.to(torch.float32).contiguous().view(1, *dlogits.shape), v_like,
                        jv, hv)
            d_x = None
            if ctx.needs_input_grad[1]:
                dxdot = hs.setdefault("dxdot", torch.empty((1,) + tuple(xin.shape), dtype=torch.float32, device=xin.device))
                eng.net_hvp_input_grad(1, dxdot)
                d_x = dxdot[0].to(x.dtype, copy=True)
        d_dlogits = jv[0].to(dlogits.dtype).clone() if ctx.needs_input_grad[2] else None
        grads = []
        for (off, size), t, need in zip(eng.segments, tensors, ctx.needs_input_grad[3:]):
            grads.append(hv[off:off + size].view(t.shape).to(t.dtype).clone() if need else None)
        return (None, d_x, d_dlogits) + tuple(grads)
