"""MAML / MAML++ meta-learning system on the H100 engine (level B0 of the drop-in boundary).

``MAMLFewShotClassifier`` keeps the reference's public contract (reference
``few_shot_learning_system.py:26-424``; SURVEY.md section 8b): constructor
``(im_shape, device, args)``, ``run_train_iter(data_batch, epoch)``,
``run_validation_iter(data_batch)``, ``save_model`` / ``load_model``, the ``losses`` dict keys,
``per_task_target_preds`` and the ``state_dict`` names/shapes/order, so the reference's
``ExperimentBuilder`` can drive it unchanged.

What is different underneath: the reference runs ~3500 eager autograd ops per task; here one call of
the C ABI (``include/maml_b200.h``) runs the whole meta-batch -- inner-loop unroll, hand-rolled
gradients, LSLR updates, second-order reverse sweep -- as hand-written sm_90a kernels, one
all-reduce sums the flat meta-gradient over ranks (tasks are sharded over GPUs), and a fused kernel
applies clamp + Adam.  All parameters live in ONE flat fp32 device buffer; the ``nn.Parameter``s
are views into it.

There is no CPU fallback: without the built library or without a CUDA device the iteration
methods raise.
"""
import math
import os

import numpy as np
import torch
import torch.nn as nn

from . import _native
from . import sharding
from .inner_loop_optimizers import LSLRGradientDescentLearningRule
from .meta_neural_network_architectures import VGGReLUNormNetwork


def set_torch_seed(seed):
    """Same seeding recipe as the reference (few_shot_learning_system.py:13-23)."""
    rng = np.random.RandomState(seed=seed)
    torch_seed = rng.randint(0, 999999)
    torch.manual_seed(seed=torch_seed)
    return rng


class _FlatAdamState(object):
    """Adam state kept as flat device buffers, (de)serialised in ``torch.optim.Adam``'s format so
    checkpoints stay interchangeable with the reference (``state['optimizer']``, reference :406-407)."""

    def __init__(self, system):
        self.system = system
        self.step_count = 0

    def state_dict(self):
        sysm = self.system
        params = sysm._trainable_param_list()
        state = {}
        if self.step_count > 0:
            for i, (name, p) in enumerate(params):
                off, size = sysm._flat_slices[name]
                state[i] = {"step": torch.tensor(float(self.step_count)),
                            "exp_avg": sysm._exp_avg[off:off + size].view(p.shape).clone(),
                            "exp_avg_sq": sysm._exp_avg_sq[off:off + size].view(p.shape).clone()}
        group = {"lr": sysm._current_lr, "betas": (0.9, 0.999), "eps": 1e-08, "weight_decay": 0, "amsgrad": False,
                 "maximize": False, "foreach": None, "capturable": False, "differentiable": False, "fused": None,
                 "decoupled_weight_decay": False, "initial_lr": float(sysm.args.meta_learning_rate),
                 "params": list(range(len(params)))}
        return {"state": state, "param_groups": [group]}

    def load_state_dict(self, sd):
        sysm = self.system
        params = sysm._trainable_param_list()
        sysm._exp_avg.zero_()
        sysm._exp_avg_sq.zero_()
        steps = []
        for i, (name, p) in enumerate(params):
            st = sd["state"].get(i, sd["state"].get(str(i)))
            if st is None:
                continue
            off, size = sysm._flat_slices[name]
            sysm._exp_avg[off:off + size].copy_(st["exp_avg"].reshape(-1).to(sysm._exp_avg.device, torch.float32))
            sysm._exp_avg_sq[off:off + size].copy_(st["exp_avg_sq"].reshape(-1).to(sysm._exp_avg.device, torch.float32))
            steps.append(int(float(st["step"])))
        self.step_count = max(steps) if steps else 0

    def zero_grad(self):
        pass


class MAMLFewShotClassifier(nn.Module):
    def __init__(self, im_shape, device, args):
        super().__init__()
        self.args = args
        self.device = torch.device(device) if not isinstance(device, torch.device) else device
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.batch_size = args.batch_size
        self.use_cuda = getattr(args, "use_cuda", torch.cuda.is_available())
        self.im_shape = im_shape
        self.current_epoch = 0

        self.rng = set_torch_seed(seed=args.seed)
        self.classifier = VGGReLUNormNetwork(im_shape=self.im_shape, num_output_classes=args.num_classes_per_set,
                                             args=args, device=self.device, meta_classifier=True)
        self.task_learning_rate = args.task_learning_rate
        self.inner_loop_optimizer = LSLRGradientDescentLearningRule(
            device=self.device, init_learning_rate=self.task_learning_rate,
            total_num_inner_loop_steps=args.number_of_training_steps_per_iter,
            use_learnable_learning_rates=args.learnable_per_layer_per_step_inner_loop_learning_rate)
        self.inner_loop_optimizer.initialise(
            names_weights_dict=self.get_inner_loop_parameter_dict(params=self.classifier.named_parameters()))

        self._engine = None
        self._engine_tasks = 0
        self._flat = None
        self._build_flat_storage()
        self.optimizer = _FlatAdamState(self)
        self._current_lr = float(args.meta_learning_rate)
        self._staging = {}
        self.rank, self.world_size = 0, 1          # resolved at call time (_dist)

    # ------------------------------------------------------------------ parameters / flat storage
    def get_inner_loop_parameter_dict(self, params):
        """The tensors adapted in the inner loop (reference :105-120): everything that requires grad
        except the norm parameters, which join with enable_inner_loop_optimizable_bn_params."""
        inner_bn = self.classifier._inner_bn()
        return {name: p for name, p in params if p.requires_grad and (inner_bn or "norm_layer" not in name)}

    def trainable_parameters(self):
        for p in self.parameters():
            if p.requires_grad:
                yield p

    def _trainable_param_list(self):
        return [(n, p) for n, p in self.named_parameters() if p.requires_grad]

    def _meta_param_names(self):
        """Flat-buffer order = the network's engine segment order (``_segment_names``), then the LSLR vectors.  (Equals
        the reference's Adam parameter order.)"""
        names = ["classifier." + n for n in self.classifier._segment_names()]
        inner = [n for n in names if self.classifier._inner_bn() or "norm_layer" not in n]
        names += ["inner_loop_optimizer.names_learning_rates_dict." + n[len("classifier."):].replace(".", "-")
                  for n in inner]
        return names

    def _build_flat_storage(self):
        named = dict(self.named_parameters())
        order = self._meta_param_names()
        total = sum(named[n].numel() for n in order)
        L, F = int(self.args.num_stages), int(self.args.cnn_num_filters)
        S = int(self.args.number_of_training_steps_per_iter)
        run_rows = S if self.args.per_step_bn_statistics else 1
        dev = self.device
        flat = torch.empty(total, dtype=torch.float32, device=dev)
        run = torch.empty(2, L, run_rows, F, dtype=torch.float32, device=dev)
        self._flat_slices = {}
        off = 0
        for n in order:
            p = named[n]
            size = p.numel()
            flat[off:off + size].copy_(p.data.reshape(-1))
            p.data = flat[off:off + size].view(p.shape)
            self._flat_slices[n] = (off, size)
            off += size
        for l in range(L if not self.classifier._layer_norm() else 0):      # layer norm keeps no running statistics
            bn = self.classifier.layer_dict["conv%d" % l].norm_layer
            run[0, l].copy_(bn.running_mean.data.reshape(run_rows, F))
            run[1, l].copy_(bn.running_var.data.reshape(run_rows, F))
            bn.running_mean.data = run[0, l].view(bn.running_mean.shape)
            bn.running_var.data = run[1, l].view(bn.running_var.shape)
        self._flat, self._running = flat, run
        self._exp_avg = torch.zeros_like(flat)
        self._exp_avg_sq = torch.zeros_like(flat)
        self._order = order
        # per-segment masks in engine segment order
        self._trainable_mask, self._clamp_mask = 0, 0
        for i, n in enumerate(order):
            if named[n].requires_grad:
                self._trainable_mask |= (1 << i)
            if n.startswith("classifier.") and "imagenet" in self.args.dataset_name:
                self._clamp_mask |= (1 << i)

    def _views_intact(self):
        named = dict(self.named_parameters())
        base = self._flat.data_ptr()
        for n, (off, size) in self._flat_slices.items():
            if named[n].data_ptr() != base + 4 * off:
                return False
        return True

    def _apply(self, fn, *a, **kw):
        out = super()._apply(fn, *a, **kw)
        if getattr(self, "_flat", None) is not None and not self._views_intact():
            # .to()/.cuda() re-allocated the parameters: re-pack them into a fresh flat buffer
            first = next(self.parameters())
            self.device = first.device
            m, v = self._exp_avg, self._exp_avg_sq
            self._build_flat_storage()
            self._exp_avg.copy_(m.to(self.device))
            self._exp_avg_sq.copy_(v.to(self.device))
            self._engine = None
        return out

    # ------------------------------------------------------------------ schedules (host logic)
    def get_per_step_loss_importance_vector(self):
        """MSL weights from ``self.current_epoch`` (reference :83-103), fp32-rounded like the reference."""
        S = int(self.args.number_of_training_steps_per_iter)
        w = np.ones(shape=(S,)) * (1.0 / S)
        decay_rate = 1.0 / S / self.args.multi_step_loss_num_epochs
        min_nonfinal = 0.03 / S
        for i in range(S - 1):
            w[i] = np.maximum(w[i] - (self.current_epoch * decay_rate), min_nonfinal)
        w[-1] = np.minimum(w[-1] + (self.current_epoch * (S - 1) * decay_rate), 1.0 - ((S - 1) * min_nonfinal))
        return torch.tensor(w, dtype=torch.float32)

    def _cosine_lr(self, epoch):
        """Closed form of CosineAnnealingLR.step(epoch=epoch) (reference :70-71, :346)."""
        base, eta_min, T = float(self.args.meta_learning_rate), float(self.args.min_learning_rate), int(self.args.total_epochs)
        return eta_min + (base - eta_min) * (1.0 + math.cos(math.pi * epoch / T)) / 2.0

    def _logged_lr(self, epoch):
        """What the reference logs: ``scheduler.get_lr()[0]`` evaluated OUTSIDE ``step`` (reference :365) --
        the recursive form applied to the already-updated lr (a logging quirk, reproduced as is)."""
        base, eta_min, T = float(self.args.meta_learning_rate), float(self.args.min_learning_rate), int(self.args.total_epochs)
        lr = self._cosine_lr(epoch)
        # torch 2.11 CosineAnnealingLR.get_lr: the `_is_initial` shortcut only holds inside the constructor, so
        # even at epoch 0 the recursive (chainable) form is evaluated on the closed-form lr.
        if (epoch - 1 - T) % (2 * T) == 0:
            return lr + (base - eta_min) * (1 - math.cos(math.pi / T)) / 2
        return (1 + math.cos(math.pi * epoch / T)) / (1 + math.cos(math.pi * (epoch - 1) / T)) * (lr - eta_min) + eta_min

    def _schedule(self, epoch, training_phase):
        """Memoised ``_schedule_uncached`` (it only depends on the epochs and the phase; host time between two
        iterations is GPU idle time in the end-to-end loop)."""
        key = (int(epoch), int(self.current_epoch), bool(training_phase))
        cache = self.__dict__.setdefault("_sched_cache", {})
        hit = cache.get(key)
        if hit is None:
            if len(cache) > 64:
                cache.clear()
            hit = cache[key] = self._schedule_uncached(epoch, training_phase)
        return hit

    def _schedule_uncached(self, epoch, training_phase):
        """(num_steps, second_order, target_mask, target_weights) -- reference :232-244, :304-305, :318-321."""
        S = int(self.args.number_of_training_steps_per_iter)
        if training_phase:
            num_steps = S
            second = bool(self.args.second_order) and epoch > self.args.first_order_to_second_order_epoch
            use_msl = bool(self.args.use_multi_step_loss_optimization) and epoch < self.args.multi_step_loss_num_epochs
        else:
            num_steps = int(self.args.number_of_evaluation_steps_per_iter)
            second, use_msl = False, False
        if num_steps > S:
            raise ValueError("number_of_evaluation_steps_per_iter > number_of_training_steps_per_iter is ill-defined "
                             "in the reference (per-step BN arrays are sized by the training steps)")
        w_msl = self.get_per_step_loss_importance_vector()
        mask, weights = 0, [0.0] * _native.MAX_STEPS
        for s in range(num_steps):
            if use_msl:
                mask |= (1 << s)
                weights[s] = float(w_msl[s])
            elif s == S - 1:
                mask |= (1 << s)
                weights[s] = 1.0
        if mask == 0:
            raise ValueError("no target pass is scheduled (evaluation steps < training steps): the reference "
                             "crashes here too (target_preds undefined)")
        return num_steps, second, mask, weights, w_msl

    # ------------------------------------------------------------------ engine plumbing
    def _ensure_engine(self, n_tasks):
        if self.device.type != "cuda":
            raise _native.NativeLibraryError(
                "MAMLFewShotClassifier needs a CUDA (sm_90a) device: the hot path has no CPU fallback")
        if self._engine is None or n_tasks > self._engine_tasks:
            a = self.args
            with torch.cuda.device(self.device):
                self._engine = _native.Engine(
                    n_way=int(a.num_classes_per_set), k_shot=int(a.num_samples_per_class),
                    t_target=int(a.num_target_samples), channels=int(self.im_shape[1]), height=int(self.im_shape[2]),
                    width=int(self.im_shape[3]), filters=int(a.cnn_num_filters), num_stages=int(a.num_stages),
                    inner_steps=int(a.number_of_training_steps_per_iter), per_step_bn=bool(a.per_step_bn_statistics),
                    max_tasks=int(n_tasks), keep_target_passes=bool(getattr(self, "_debug_keep_target_passes", False)),
                    force_fp32_convs=bool(getattr(self, "_debug_force_fp32_convs", False)),
                    layer_norm=self.classifier._layer_norm(), inner_bn=self.classifier._inner_bn())
            self._engine_tasks = int(n_tasks)
            if self._engine.meta_size != self._flat.numel():
                raise RuntimeError("engine / module parameter layout mismatch (%d vs %d floats)" %
                                   (self._engine.meta_size, self._flat.numel()))
            for (off, size), n in zip(self._engine.segments, self._order):
                if (off, size) != self._flat_slices[n]:
                    raise RuntimeError("engine segment layout mismatch at %s" % n)
            self._result = torch.zeros(self._engine.result_size, dtype=torch.float32, device=self.device)
            self._comm_mode = None          # decided (collectively) by the first sharded call on this engine
        if not self._views_intact():
            self._build_flat_storage()
        return self._engine

    # number of staging slots: a batch is staged into slot i % 2, so the host may fill the next batch's pinned block
    # while the device still reads the previous one (replaces the reference's unpinned, synchronous
    # ``torch.Tensor(x).float().to(device)``, :355-358)
    _STAGE_SLOTS = 2

    def _expected_shapes(self, B):
        a = self.args
        N, K, T = int(a.num_classes_per_set), int(a.num_samples_per_class), int(a.num_target_samples)
        C, H, W = int(self.im_shape[1]), int(self.im_shape[2]), int(self.im_shape[3])
        return ((B, N, K, C, H, W), (B, N, T, C, H, W), (B, N, K), (B, N, T))

    def _check_batch(self, ts):
        """The engine reads raw pointers: reject anything whose shape is not the episode shape ``args`` describes
        (the reference would fail inside ``.view`` / the conv; here it would be an out-of-bounds read)."""
        if len(ts) != 4:
            raise ValueError("data_batch must be (x_support, x_target, y_support, y_target)")
        if ts[0].dim() != 6:
            raise ValueError("x_support must be [B, N, K, C, H, W], got %s" % (tuple(ts[0].shape),))
        B = int(ts[0].shape[0])
        for name, t, want in zip(("x_support", "x_target", "y_support", "y_target"), ts, self._expected_shapes(B)):
            if tuple(t.shape) != want:
                raise ValueError("%s has shape %s, the engine was configured for %s (args: N=%d K=%d T=%d, image %s)"
                                 % (name, tuple(t.shape), want, want[1], self._expected_shapes(B)[0][2],
                                    self._expected_shapes(B)[1][2], tuple(self.im_shape[1:])))
        return B

    def _stage_batch(self, data_batch):
        """Episode batch -> persistent device block.  Host batches: the four tensors are packed into ONE pinned staging
        block and moved with ONE asynchronous H2D copy; device batches: four D2D copies into the same block.  Either
        way the engine always sees the same (two) sets of addresses, which keeps its CUDA-graph cache hot -- a caller
        that allocates fresh device tensors every iteration would otherwise force a re-capture per step.  Labels follow
        the reference's float -> long conversion (:357-358); host labels are range-checked (torch's cross_entropy
        raises on a bad label, the kernel would index shared memory with it)."""
        want = (torch.float32, torch.float32, torch.int64, torch.int64)
        ts = [t if torch.is_tensor(t) else torch.as_tensor(np.asarray(t)) for t in data_batch]
        B = self._check_batch(ts)
        on_dev = [t.device.type == "cuda" for t in ts]
        conv = []
        for t, d, dev in zip(ts, want, on_dev):
            if d == torch.int64:
                t = t.to(torch.float32).long() if t.is_floating_point() else t.long()      # reference :357-358
                if not dev and t.numel():
                    lo, hi = torch.aminmax(t)
                    if int(lo) < 0 or int(hi) >= int(self.args.num_classes_per_set):
                        raise ValueError("labels must lie in [0, num_classes_per_set)")
            else:
                t = t.to(d)
            conv.append(t)
        key = tuple(tuple(t.shape) for t in conv)
        st = self._staging.get("batch")
        if st is None or st["key"] != key:
            offs, total = [], 0
            for t in conv:
                offs.append(total)
                total += (t.numel() * t.element_size() + 15) // 16 * 16

            def views(block):
                return [block[o:o + t.numel() * t.element_size()].view(t.dtype).view(t.shape) for o, t in zip(offs, conv)]
            st = {"key": key, "slots": [], "next": 0}
            for _ in range(self._STAGE_SLOTS):
                pin = torch.empty(total, dtype=torch.uint8).pin_memory()
                dev = torch.empty(total, dtype=torch.uint8, device=self.device)
                st["slots"].append({"pin": pin, "dev": dev, "pin_views": views(pin), "dev_views": views(dev),
                                    "copied": torch.cuda.Event()})
            self._staging["batch"] = st
        slot = st["slots"][st["next"]]
        st["next"] = (st["next"] + 1) % self._STAGE_SLOTS
        with torch.cuda.device(self.device):
            if all(on_dev):
                for v, t in zip(slot["dev_views"], conv):
                    v.copy_(t, non_blocking=True)
            else:
                slot["copied"].synchronize()          # the H2D copy that last read this pinned block has finished
                for v, t in zip(slot["pin_views"], conv):
                    v.copy_(t)                        # (device-resident members come through the host: rare, mixed batches)
                slot["dev"].copy_(slot["pin"], non_blocking=True)
                slot["copied"].record()
        return tuple(slot["dev_views"])

    def _dist(self):
        """(rank, world_size), resolved at call time: a process group initialised AFTER the model was built must not
        leave the ranks silently training independent replicas."""
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            return torch.distributed.get_rank(), torch.distributed.get_world_size()
        return 0, 1

    def _run(self, data_batch, epoch, training_phase, apply_update):
        if self.device.type != "cuda":
            raise _native.NativeLibraryError(
                "MAMLFewShotClassifier needs a CUDA (sm_90a) device: the hot path has no CPU fallback")
        # _shard_override = (rank, world): test hook -- act as one rank of a sharded job without a process group
        self.rank, self.world_size = getattr(self, "_shard_override", None) or self._dist()
        xs, xt, ys, yt = self._stage_batch(data_batch)
        if self.classifier._layer_norm():
            self.classifier._check_layer_norm_weights()
        B = xs.shape[0]
        n_t = xt.shape[1] * xt.shape[2]
        N = int(self.args.num_classes_per_set)
        eng = self._ensure_engine(B)
        num_steps, second, mask, weights, w_msl = self._schedule(epoch, training_phase)
        task_offset, B_global = sharding.shard_of(self.rank, self.world_size, B)
        out = self._staging.get(("out", B))
        if out is None:
            # [loss, n_correct | logits]: one device block, so that _finish needs ONE device-to-host read
            out = torch.empty(2 + B * n_t * N, dtype=torch.float32, device=self.device)
            self._staging[("out", B)] = out
        logits = out[2:].view(B, n_t, N)
        if self.world_size > 1 and getattr(self, "_shard_override", None) is None:
            self._ensure_comm(eng)
            eng = self._engine
        with torch.cuda.device(self.device):
            eng.fwd_bwd(n_tasks=B, task_offset=task_offset, tasks_global=B_global, num_steps=num_steps,
                        second_order=second, training=training_phase, target_mask=mask, target_weight=weights,
                        meta=self._flat, xs=xs, ys=ys, xt=xt, yt=yt, result=self._result, last_logits=logits)
            reduced = self._all_reduce_result(eng)
            if self.world_size > 1 and self._comm_mode == "peer":
                # a rank that waited 30 s for a peer gives up and flags it; surface that instead of training on garbage
                self._comm_checks = getattr(self, "_comm_checks", 0) + 1
                if self._comm_checks % 512 == 0 and eng.comm_status() != 0:
                    raise RuntimeError("peer-memory all-reduce timed out waiting for another rank (status %#x)" % eng.comm_status())
            ms = eng.meta_size
            head = (reduced[ms:ms + 2], out[2:])      # [loss, n_correct] of the (reduced) result vector, logits: read by _finish
            if training_phase and apply_update:
                self.optimizer.step_count += 1
                eng.adam_step(self._flat, reduced, self._exp_avg, self._exp_avg_sq, lr=self._current_lr,
                              step=self.optimizer.step_count, trainable_mask=self._trainable_mask,
                              clamp_mask=self._clamp_mask)
            if self.args.per_step_bn_statistics and not self.classifier._layer_norm() and (apply_update or not training_phase):
                # F.batch_norm's EMA side effect on running_*[step].  Evaluation passes leave it behind as well: the
                # reference's backup is copy(tensor.data), an alias, so restore_backup_stats restores the mutated values
                # (meta_neural_network_architectures.py:240-255; pinned by the val/ golden entries).
                S = int(self.args.number_of_training_steps_per_iter)
                dkey = (mask, num_steps, S, B_global)
                dcache = self.__dict__.setdefault("_decay_cache", {})
                decay = dcache.get(dkey)
                if decay is None:
                    if len(dcache) > 64:
                        dcache.clear()
                    decay = dcache[dkey] = tuple(sharding.decay_vector(mask, num_steps, S, B_global))
                eng.running_stats_update(reduced, self._running[0], self._running[1], decay)
        return head, logits, w_msl, B_global, n_t

    def _ensure_comm(self, eng):
        """Connect the engine's peer-memory communicator (once per engine; every rank must get here together, like any
        collective).  Each rank allocates a communication block inside the engine, the 64-byte CUDA IPC handles travel
        through ``torch.distributed`` (plumbing), every rank maps its peers' blocks.  If ANY rank cannot (IPC unavailable
        in this container, > 8 ranks, peers on another node) all ranks fall back to ``torch.distributed.all_reduce``
        -- reported by ``collective_desc`` -- so the ranks never disagree about who sums."""
        if self._comm_mode is not None:
            return self._comm_mode
        dist = torch.distributed
        ok, why = 1, ""
        if os.environ.get("MAML_B200_COLLECTIVE", "").lower() == "nccl":
            ok, why = 0, "disabled by MAML_B200_COLLECTIVE=nccl"
        handle = b"\0" * 64
        if ok:
            try:
                with torch.cuda.device(self.device):
                    handle = eng.comm_init(self.rank, self.world_size)
            except Exception as exc:
                ok, why = 0, repr(exc)[:200]
        gathered = [None] * self.world_size
        dist.all_gather_object(gathered, (ok, handle, why))
        if all(g[0] for g in gathered):
            try:
                with torch.cuda.device(self.device):
                    eng.comm_connect([g[1] for g in gathered])
            except Exception as exc:
                ok, why = 0, repr(exc)[:200]
        else:
            ok, why = 0, next(g[2] for g in gathered if not g[0])
        flags = [None] * self.world_size
        dist.all_gather_object(flags, (ok, why))
        if all(f[0] for f in flags):
            self._comm_mode = "peer"
            self._comm_why = ""
        else:
            self._comm_mode = "nccl"
            self._comm_why = next(f[1] for f in flags if not f[0])
            if eng.comm_world() > 1:           # this rank did connect, another one could not: rebuild without
                self._engine = None
                eng = self._ensure_engine(self._engine_tasks)
                self._comm_mode, self._comm_why = "nccl", self._comm_why
        return self._comm_mode

    def _all_reduce_result(self, eng):
        """Sum of the flat result vector over the ranks -- the ONE collective of an iteration (SURVEY.md section 8e).
        ``peer`` mode: nothing to do here, the engine call already ran its all-reduce kernel over peer memory inside the
        iteration's CUDA graph and ``_result`` holds the sum.  ``nccl`` mode (fallback): one library all-reduce."""
        if self.world_size > 1 and getattr(self, "_shard_override", None) is None and self._comm_mode == "nccl":
            torch.distributed.all_reduce(self._result, op=torch.distributed.ReduceOp.SUM)
        return self._result

    def collective_desc(self):
        mode = getattr(self, "_comm_mode", None)
        if self.world_size <= 1 or mode is None:
            return {"kind": "none (single GPU)"}
        if mode == "peer":
            return {"kind": "in-engine peer-memory all-reduce (export kernel publishes into an IPC-mapped slot, "
                            "allreduce_kernel pulls every rank's slot over NVLink and sums in rank order; inside the "
                            "iteration's CUDA graph)", "bytes": 4 * int(self._engine.result_size), "ranks": self.world_size}
        return {"kind": "torch.distributed.all_reduce (NCCL) -- FALLBACK", "why": getattr(self, "_comm_why", ""),
                "bytes": 4 * int(self._engine.result_size), "ranks": self.world_size}

    def collective_launches(self):
        """Kernels of THIS repo launched per iteration for the collective beyond what the engine call already counts
        (peer mode: the all-reduce kernel is a node of the iteration graph and is in ``last_launch_count``; the NCCL
        fallback's kernel is not ours)."""
        return 0

    def time_collective(self, iters=20):
        """Duration (us, minimum over ``iters``) of the stand-alone all-reduce of a result-sized vector, CUDA events on the
        launching stream (bench.py's per-rank ``collective_us``).  Every rank must call it."""
        if self.world_size <= 1 or self._engine is None:
            return 0.0
        vec = torch.zeros_like(self._result)
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
        with torch.cuda.device(self.device):
            for i in range(iters + 3):
                torch.distributed.barrier()
                if i >= 3:
                    ev[i - 3][0].record()
                if self._comm_mode == "peer":
                    self._engine.all_reduce(vec)
                else:
                    torch.distributed.all_reduce(vec)
                if i >= 3:
                    ev[i - 3][1].record()
            torch.cuda.synchronize()
        ts = sorted(a.elapsed_time(b) * 1e3 for a, b in ev)
        return ts[0]      # minimum: the other samples include the launch skew between the ranks (they wait for each other)

    def _finish(self, head, logits, w_msl, B_global, n_t):
        """One D2H read of (loss, n_correct, logits) -- the reference syncs per task (:246,:249,:261)."""
        # [loss, n_correct | logits]: two asynchronous copies into one pinned block, ONE wait (``.cpu()`` goes through
        # pageable memory: an extra staging copy and a full stream synchronisation)
        n = 2 + head[1].numel()
        hp = self._staging.get(("host_out", n))
        if hp is None:
            hp = self._staging[("host_out", n)] = (torch.empty(n, dtype=torch.float32).pin_memory(), torch.cuda.Event())
        with torch.cuda.device(self.device):
            hp[0][:2].copy_(head[0], non_blocking=True)
            hp[0][2:].copy_(head[1], non_blocking=True)
            hp[1].record()
        hp[1].synchronize()
        host = hp[0].clone()                   # the caller keeps the arrays; the pinned block is reused next iteration
        head_h = host[:2]
        preds = host[2:].view(logits.shape).numpy()
        losses = {"loss": head_h[0].clone(), "accuracy": float(head_h[1]) / float(B_global * n_t)}
        for i, item in enumerate(w_msl):
            losses["loss_importance_vector_{}".format(i)] = item.numpy()
        return losses, [preds[b] for b in range(preds.shape[0])]

    # ------------------------------------------------------------------ public API (reference names)
    def run_train_iter(self, data_batch, epoch):
        """One outer-loop update on a batch of tasks (reference :338-369)."""
        epoch = int(epoch)
        self._current_lr = self._cosine_lr(epoch)
        if self.current_epoch != epoch:
            self.current_epoch = epoch
        if not self.training:
            self.train()
        head, logits, w_msl, Bg, n_t = self._run(data_batch, epoch, training_phase=True, apply_update=True)
        losses, preds = self._finish(head, logits, w_msl, Bg, n_t)
        losses["learning_rate"] = self._logged_lr(epoch)
        return losses, preds

    def run_validation_iter(self, data_batch):
        """Evaluation on a batch of tasks: first-order adaptation, final-step target loss only (reference :371-397,
        :311-323).  Like the reference, the pass leaves its BatchNorm EMA updates in ``running_mean`` / ``running_var``
        (the reference's backup/restore, meta_neural_network_architectures.py:240-255, aliases the live tensor)."""
        if self.training:
            self.eval()
        head, logits, w_msl, Bg, n_t = self._run(data_batch, self.current_epoch, training_phase=False, apply_update=False)
        return self._finish(head, logits, w_msl, Bg, n_t)

    def meta_gradient(self, data_batch, epoch):
        """Test / inspection helper: the outer gradient of one batch WITHOUT applying the update.
        Returns (losses, preds, {name: grad tensor}) in reference parameter names."""
        epoch = int(epoch)
        self.current_epoch = epoch
        head, logits, w_msl, Bg, n_t = self._run(data_batch, epoch, training_phase=True, apply_update=False)
        losses, preds = self._finish(head, logits, w_msl, Bg, n_t)
        named = dict(self.named_parameters())
        grads = {n: self._result[off:off + size].view(named[n].shape).clone()
                 for n, (off, size) in self._flat_slices.items()}
        return losses, preds, grads

    def save_model(self, model_save_dir, state):
        state["network"] = self.state_dict()
        state["optimizer"] = self.optimizer.state_dict()
        torch.save(state, f=model_save_dir)

    def load_model(self, model_save_dir, model_name, model_idx):
        filepath = os.path.join(model_save_dir, "{}_{}".format(model_name, model_idx))
        state = torch.load(filepath, map_location="cpu", weights_only=False)
        network = {k.replace("classifier.module.", "classifier."): v for k, v in state["network"].items()}
        self.optimizer.load_state_dict(state["optimizer"])
        self.load_state_dict(state_dict=network)
        return state
