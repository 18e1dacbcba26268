"""ctypes binding of ``libmaml_b200.so`` (C ABI declared in ``include/maml_b200.h``).

The product path has NO CPU fallback: if the library is missing or a CUDA device is absent the
calls below raise.  PyTorch is used by the callers only for device memory, streams and
``torch.distributed``; every pointer crossing this boundary is a raw device pointer.
"""
import ctypes
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
# MAML_B200_LIB: diagnostic override (A/B of compile-time variants built by scripts/build_variant.sh)
LIB_PATH = os.environ.get("MAML_B200_LIB") or os.path.join(_PKG, "lib", "libmaml_b200.so")

MAX_STAGES = 4
MAX_STEPS = 8
ABI_VERSION = 5

EXPORTED_SYMBOLS = [
    "maml_b200_abi_version", "maml_b200_last_error", "maml_b200_create", "maml_b200_destroy",
    "maml_b200_workspace_bytes", "maml_b200_num_segments", "maml_b200_segment", "maml_b200_meta_size",
    "maml_b200_result_size", "maml_b200_meta_batch_fwd_bwd", "maml_b200_adam_step",
    "maml_b200_running_stats_update", "maml_b200_debug_read", "maml_b200_last_launch_count",
    "maml_b200_profile", "maml_b200_profile_read", "maml_b200_net_forward",
    "maml_b200_trace", "maml_b200_trace_read",
    "maml_b200_comm_init", "maml_b200_comm_connect", "maml_b200_comm_world", "maml_b200_all_reduce",
    "maml_b200_comm_status", "maml_b200_net_backward", "maml_b200_net_running_update", "maml_b200_episode_gather",
    "maml_b200_net_hvp", "maml_b200_net_input_grad", "maml_b200_net_hvp_input_grad",
    "maml_b200_net_hvp_image", "maml_b200_net_jvp", "maml_b200_net_forward_tasks", "maml_b200_net_backward_tasks",
    "maml_b200_net_hvp_image_tasks", "maml_b200_net_jvp_tasks",
]
PROF_CATS = ["conv_igemm", "conv_first_block", "wgrad", "wgrad_first_block", "bn_act_pool", "head", "param"]


class Config(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in (
        "n_way", "k_shot", "t_target", "channels", "height", "width", "filters", "num_stages",
        "inner_steps", "per_step_bn", "max_tasks", "reserved", "norm_layer", "inner_bn")]


class IterArgs(ctypes.Structure):
    _fields_ = [("n_tasks", ctypes.c_int32), ("task_offset", ctypes.c_int32), ("tasks_global", ctypes.c_int32),
                ("num_steps", ctypes.c_int32), ("second_order", ctypes.c_int32), ("training", ctypes.c_int32),
                ("target_mask", ctypes.c_uint32), ("target_weight", ctypes.c_float * MAX_STEPS)]


_lib = None


class NativeLibraryError(RuntimeError):
    pass


def load_library():
    """Load (once) and type the shared library.  Raises loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryError(
            "CUDA engine %s not found: build it with `python -m howtotrainyourmamlpytorch_b200.build` "
            "(or __graft_entry__.build()).  There is no CPU fallback for this path." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    vp, i32, i64, u32, f32 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_uint32, ctypes.c_float
    lib.maml_b200_abi_version.restype = ctypes.c_int
    lib.maml_b200_last_error.restype = ctypes.c_char_p
    lib.maml_b200_create.argtypes = [ctypes.POINTER(Config), ctypes.POINTER(vp)]
    lib.maml_b200_create.restype = ctypes.c_int
    lib.maml_b200_destroy.argtypes = [vp]
    lib.maml_b200_destroy.restype = None
    lib.maml_b200_workspace_bytes.argtypes = [vp]
    lib.maml_b200_workspace_bytes.restype = i64
    lib.maml_b200_num_segments.argtypes = [vp]
    lib.maml_b200_num_segments.restype = i32
    lib.maml_b200_segment.argtypes = [vp, i32, ctypes.POINTER(i64), ctypes.POINTER(i64)]
    lib.maml_b200_segment.restype = ctypes.c_int
    lib.maml_b200_meta_size.argtypes = [vp]
    lib.maml_b200_meta_size.restype = i64
    lib.maml_b200_result_size.argtypes = [vp]
    lib.maml_b200_result_size.restype = i64
    lib.maml_b200_meta_batch_fwd_bwd.argtypes = [vp, ctypes.POINTER(IterArgs), vp, vp, vp, vp, vp, vp, vp, vp]
    lib.maml_b200_meta_batch_fwd_bwd.restype = ctypes.c_int
    lib.maml_b200_net_forward.argtypes = [vp, i32, i32, vp, vp, vp, vp]
    lib.maml_b200_net_forward.restype = ctypes.c_int
    lib.maml_b200_net_backward.argtypes = [vp, i32, i32, vp, vp, vp, vp]
    lib.maml_b200_net_backward.restype = ctypes.c_int
    lib.maml_b200_net_hvp.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp, vp]
    lib.maml_b200_net_hvp.restype = ctypes.c_int
    lib.maml_b200_net_hvp_image.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.maml_b200_net_hvp_image.restype = ctypes.c_int
    lib.maml_b200_net_jvp.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp]
    lib.maml_b200_net_jvp.restype = ctypes.c_int
    lib.maml_b200_net_forward_tasks.argtypes = [vp, i32, i32, vp, i64, vp, vp, vp]
    lib.maml_b200_net_forward_tasks.restype = ctypes.c_int
    lib.maml_b200_net_backward_tasks.argtypes = [vp, i32, i32, vp, i64, vp, vp, i32, vp]
    lib.maml_b200_net_backward_tasks.restype = ctypes.c_int
    lib.maml_b200_net_hvp_image_tasks.argtypes = [vp, i32, i32, vp, i64, vp, vp, vp, vp, i64, vp, vp, i32, vp]
    lib.maml_b200_net_hvp_image_tasks.restype = ctypes.c_int
    lib.maml_b200_net_jvp_tasks.argtypes = [vp, i32, i32, vp, i64, vp, vp, i64, vp, vp, vp]
    lib.maml_b200_net_jvp_tasks.restype = ctypes.c_int
    lib.maml_b200_net_input_grad.argtypes = [vp, i32, vp, vp]
    lib.maml_b200_net_input_grad.restype = ctypes.c_int
    lib.maml_b200_net_hvp_input_grad.argtypes = [vp, i32, vp, vp]
    lib.maml_b200_net_hvp_input_grad.restype = ctypes.c_int
    lib.maml_b200_net_running_update.argtypes = [vp, i32, i32, vp, vp, vp]
    lib.maml_b200_net_running_update.restype = ctypes.c_int
    lib.maml_b200_episode_gather.argtypes = [vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, ctypes.POINTER(f32),
                                             ctypes.POINTER(f32), vp, vp, vp, vp, vp]
    lib.maml_b200_episode_gather.restype = ctypes.c_int
    lib.maml_b200_adam_step.argtypes = [vp, vp, vp, vp, vp, f32, i32, ctypes.c_uint64, ctypes.c_uint64, vp]
    lib.maml_b200_adam_step.restype = ctypes.c_int
    lib.maml_b200_running_stats_update.argtypes = [vp, vp, vp, vp, ctypes.POINTER(f32), vp]
    lib.maml_b200_running_stats_update.restype = ctypes.c_int
    lib.maml_b200_debug_read.argtypes = [vp, ctypes.c_char_p, i32, i32, i32, vp, i64]
    lib.maml_b200_debug_read.restype = i64
    lib.maml_b200_last_launch_count.argtypes = [vp]
    lib.maml_b200_last_launch_count.restype = i64
    lib.maml_b200_trace.argtypes = [vp, i32]
    lib.maml_b200_trace.restype = ctypes.c_int
    lib.maml_b200_trace_read.argtypes = [vp, ctypes.POINTER(ctypes.c_uint64), i64]
    lib.maml_b200_trace_read.restype = i64
    lib.maml_b200_profile.argtypes = [vp, i32]
    lib.maml_b200_profile.restype = ctypes.c_int
    lib.maml_b200_profile_read.argtypes = [vp, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double),
                                           ctypes.POINTER(i64), i32]
    lib.maml_b200_profile_read.restype = ctypes.c_int
    lib.maml_b200_comm_init.argtypes = [vp, i32, i32, vp]
    lib.maml_b200_comm_init.restype = ctypes.c_int
    lib.maml_b200_comm_connect.argtypes = [vp, vp]
    lib.maml_b200_comm_connect.restype = ctypes.c_int
    lib.maml_b200_comm_world.argtypes = [vp]
    lib.maml_b200_comm_world.restype = ctypes.c_int
    lib.maml_b200_all_reduce.argtypes = [vp, vp, vp]
    lib.maml_b200_all_reduce.restype = ctypes.c_int
    lib.maml_b200_comm_status.argtypes = [vp]
    lib.maml_b200_comm_status.restype = i64
    if lib.maml_b200_abi_version() != ABI_VERSION:
        raise NativeLibraryError("libmaml_b200.so ABI version mismatch: rebuild the library")
    _lib = lib
    return lib


def _check(lib, rc, what):
    if rc != 0:
        raise RuntimeError("%s failed: %s" % (what, lib.maml_b200_last_error().decode()))


def episode_gather(dataset, image_index, rot_k, n_tasks, n_way, k_shot, t_target, channels, height, width, mean, std,
                   xs, xt, ys, yt):
    """``maml_b200_episode_gather`` on the current stream (all tensors on the current CUDA device)."""
    import torch
    lib = load_library()
    mean_arr = (ctypes.c_float * channels)(*[float(v) for v in mean]) if mean is not None else None
    std_arr = (ctypes.c_float * channels)(*[float(v) for v in std]) if std is not None else None
    rc = lib.maml_b200_episode_gather(dataset.data_ptr(), image_index.data_ptr(), rot_k.data_ptr(), int(n_tasks), int(n_way),
                                      int(k_shot), int(t_target), int(channels), int(height), int(width), mean_arr, std_arr,
                                      xs.data_ptr(), xt.data_ptr(), ys.data_ptr(), yt.data_ptr(),
                                      ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    _check(lib, rc, "maml_b200_episode_gather")


class Engine(object):
    """Owns one ``maml_b200_handle`` (one static task shape on the current CUDA device)."""

    def __init__(self, n_way, k_shot, t_target, channels, height, width, filters, num_stages, inner_steps,
                 per_step_bn, max_tasks, keep_target_passes=False, force_fp32_convs=False, layer_norm=False,
                 inner_bn=False):
        import torch
        if not torch.cuda.is_available():
            raise NativeLibraryError("the MAML engine needs a CUDA (sm_90a) device; there is no CPU fallback")
        self.lib = load_library()
        self.cfg = Config(n_way=n_way, k_shot=k_shot, t_target=t_target, channels=channels, height=height, width=width,
                          filters=filters, num_stages=num_stages, inner_steps=inner_steps,
                          per_step_bn=int(bool(per_step_bn)), max_tasks=max_tasks,
                          reserved=(1 if keep_target_passes else 0) | (2 if force_fp32_convs else 0),
                          norm_layer=1 if layer_norm else 0, inner_bn=1 if inner_bn else 0)
        h = ctypes.c_void_p()
        _check(self.lib, self.lib.maml_b200_create(ctypes.byref(self.cfg), ctypes.byref(h)), "maml_b200_create")
        self.h = h
        self.meta_size = int(self.lib.maml_b200_meta_size(self.h))
        self.result_size = int(self.lib.maml_b200_result_size(self.h))
        self.workspace_bytes = int(self.lib.maml_b200_workspace_bytes(self.h))
        self.segments = []
        for i in range(self.lib.maml_b200_num_segments(self.h)):
            off, size = ctypes.c_int64(), ctypes.c_int64()
            _check(self.lib, self.lib.maml_b200_segment(self.h, i, ctypes.byref(off), ctypes.byref(size)), "segment")
            self.segments.append((off.value, size.value))

    def close(self):
        if getattr(self, "h", None):
            self.lib.maml_b200_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _stream():
        import torch
        return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def fwd_bwd(self, n_tasks, task_offset, tasks_global, num_steps, second_order, training, target_mask,
                target_weight, meta, xs, ys, xt, yt, result, last_logits):
        key = (n_tasks, task_offset, tasks_global, num_steps, bool(second_order), bool(training), target_mask,
               tuple(float(w) for w in target_weight))
        cache = self.__dict__.setdefault("_iter_args", {})
        it = cache.get(key)
        if it is None:
            it = IterArgs(n_tasks=n_tasks, task_offset=task_offset, tasks_global=tasks_global, num_steps=num_steps,
                          second_order=int(bool(second_order)), training=int(bool(training)), target_mask=target_mask)
            for i in range(MAX_STEPS):
                it.target_weight[i] = float(target_weight[i]) if i < len(target_weight) else 0.0
            if len(cache) > 64:
                cache.clear()
            cache[key] = it
        rc = self.lib.maml_b200_meta_batch_fwd_bwd(
            self.h, ctypes.byref(it), meta.data_ptr(), xs.data_ptr(), ys.data_ptr(), xt.data_ptr(), yt.data_ptr(),
            result.data_ptr(), last_logits.data_ptr() if last_logits is not None else None, self._stream())
        _check(self.lib, rc, "maml_b200_meta_batch_fwd_bwd")

    def net_forward(self, n_tasks, num_step, meta_like, x, logits):
        rc = self.lib.maml_b200_net_forward(self.h, int(n_tasks), int(num_step), meta_like.data_ptr(), x.data_ptr(),
                                            logits.data_ptr(), self._stream())
        _check(self.lib, rc, "maml_b200_net_forward")

    def net_backward(self, n_tasks, num_step, meta_like, dlogits, grad_out):
        rc = self.lib.maml_b200_net_backward(self.h, int(n_tasks), int(num_step), meta_like.data_ptr(), dlogits.data_ptr(),
                                             grad_out.data_ptr(), self._stream())
        _check(self.lib, rc, "maml_b200_net_backward")

    def net_hvp(self, n_tasks, num_step, meta_like, x, dlogits, v_like, jv_out, hv_out):
        rc = self.lib.maml_b200_net_hvp(self.h, int(n_tasks), int(num_step), meta_like.data_ptr(), x.data_ptr(),
                                        dlogits.data_ptr(), v_like.data_ptr(), jv_out.data_ptr(), hv_out.data_ptr(),
                                        self._stream())
        _check(self.lib, rc, "maml_b200_net_hvp")

    def net_hvp_image(self, n_tasks, num_step, meta_like, x, xdot, dlogits, v_like, jv_out, hv_out):
        """``net_hvp`` along (v_like, xdot); ``xdot`` None is ``net_hvp``."""
        rc = self.lib.maml_b200_net_hvp_image(self.h, int(n_tasks), int(num_step), meta_like.data_ptr(), x.data_ptr(),
                                              None if xdot is None else xdot.data_ptr(), dlogits.data_ptr(),
                                              v_like.data_ptr(), jv_out.data_ptr(), hv_out.data_ptr(), self._stream())
        _check(self.lib, rc, "maml_b200_net_hvp_image")

    def net_jvp(self, n_tasks, num_step, meta_like, x, t_like, xdot, jv_out):
        """Logits tangent J_theta t + J_x xdot (``xdot`` may be None)."""
        rc = self.lib.maml_b200_net_jvp(self.h, int(n_tasks), int(num_step), meta_like.data_ptr(), x.data_ptr(),
                                        t_like.data_ptr(), None if xdot is None else xdot.data_ptr(), jv_out.data_ptr(),
                                        self._stream())
        _check(self.lib, rc, "maml_b200_net_jvp")

    def net_forward_tasks(self, n_tasks, num_step, meta_like, meta_stride, x, logits):
        """``net_forward`` with task t's weights at ``meta_like`` + t * meta_stride floats (0: shared)."""
        rc = self.lib.maml_b200_net_forward_tasks(self.h, int(n_tasks), int(num_step), meta_like.data_ptr(), int(meta_stride),
                                                  x.data_ptr(), logits.data_ptr(), self._stream())
        _check(self.lib, rc, "maml_b200_net_forward_tasks")

    def net_backward_tasks(self, n_tasks, num_step, meta_like, meta_stride, dlogits, grad_out, sum_tasks=False):
        """``net_backward`` with per-task weights; grad_out [n_tasks, result_size] (one vector per task) unless sum_tasks."""
        rc = self.lib.maml_b200_net_backward_tasks(self.h, int(n_tasks), int(num_step), meta_like.data_ptr(), int(meta_stride),
                                                   dlogits.data_ptr(), grad_out.data_ptr(), int(bool(sum_tasks)),
                                                   self._stream())
        _check(self.lib, rc, "maml_b200_net_backward_tasks")

    def net_hvp_image_tasks(self, n_tasks, num_step, meta_like, meta_stride, x, xdot, dlogits, v_like, dir_stride, jv_out,
                            hv_out, sum_tasks=False):
        """``net_hvp_image`` with per-task weights and directions; hv_out [n_tasks, result_size] unless sum_tasks."""
        rc = self.lib.maml_b200_net_hvp_image_tasks(self.h, int(n_tasks), int(num_step), meta_like.data_ptr(),
                                                    int(meta_stride), x.data_ptr(), None if xdot is None else xdot.data_ptr(),
                                                    dlogits.data_ptr(), v_like.data_ptr(), int(dir_stride),
                                                    jv_out.data_ptr(), hv_out.data_ptr(), int(bool(sum_tasks)),
                                                    self._stream())
        _check(self.lib, rc, "maml_b200_net_hvp_image_tasks")

    def net_jvp_tasks(self, n_tasks, num_step, meta_like, meta_stride, x, t_like, dir_stride, xdot, jv_out):
        """``net_jvp`` with task t's weights at ``meta_like`` + t * meta_stride and its tangent at ``t_like`` + t *
        dir_stride floats (0: shared)."""
        rc = self.lib.maml_b200_net_jvp_tasks(self.h, int(n_tasks), int(num_step), meta_like.data_ptr(), int(meta_stride),
                                              x.data_ptr(), t_like.data_ptr(), int(dir_stride),
                                              None if xdot is None else xdot.data_ptr(), jv_out.data_ptr(), self._stream())
        _check(self.lib, rc, "maml_b200_net_jvp_tasks")

    def net_input_grad(self, n_tasks, dx_out):
        rc = self.lib.maml_b200_net_input_grad(self.h, int(n_tasks), dx_out.data_ptr(), self._stream())
        _check(self.lib, rc, "maml_b200_net_input_grad")

    def net_hvp_input_grad(self, n_tasks, dxdot_out):
        rc = self.lib.maml_b200_net_hvp_input_grad(self.h, int(n_tasks), dxdot_out.data_ptr(), self._stream())
        _check(self.lib, rc, "maml_b200_net_hvp_input_grad")

    def net_running_update(self, n_tasks, num_step, running_mean, running_var):
        rc = self.lib.maml_b200_net_running_update(self.h, int(n_tasks), int(num_step), running_mean.data_ptr(),
                                                   running_var.data_ptr(), self._stream())
        _check(self.lib, rc, "maml_b200_net_running_update")

    def adam_step(self, meta, grad, exp_avg, exp_avg_sq, lr, step, trainable_mask, clamp_mask):
        rc = self.lib.maml_b200_adam_step(self.h, meta.data_ptr(), grad.data_ptr(), exp_avg.data_ptr(),
                                          exp_avg_sq.data_ptr(), ctypes.c_float(lr), int(step), int(trainable_mask),
                                          int(clamp_mask), self._stream())
        _check(self.lib, rc, "maml_b200_adam_step")

    def running_stats_update(self, result, running_mean, running_var, decay):
        cache = self.__dict__.setdefault("_decay_arrays", {})
        key = tuple(decay)
        arr = cache.get(key)
        if arr is None:
            if len(cache) > 64:
                cache.clear()
            arr = cache[key] = (ctypes.c_float * MAX_STEPS)(*([float(d) for d in decay] + [1.0] * (MAX_STEPS - len(decay))))
        rc = self.lib.maml_b200_running_stats_update(self.h, result.data_ptr(), running_mean.data_ptr(),
                                                     running_var.data_ptr(), arr, self._stream())
        _check(self.lib, rc, "maml_b200_running_stats_update")

    # ---- multi-GPU: peer-memory all-reduce of the result vector (CUDA IPC handles are exchanged by the caller)
    def comm_init(self, rank, world):
        """Allocate this rank's communication block; returns its 64-byte IPC handle (bytes)."""
        buf = ctypes.create_string_buffer(64)
        _check(self.lib, self.lib.maml_b200_comm_init(self.h, int(rank), int(world), buf), "maml_b200_comm_init")
        return bytes(buf.raw)

    def comm_connect(self, handles):
        blob = b"".join(handles)
        buf = ctypes.create_string_buffer(blob, len(blob))
        _check(self.lib, self.lib.maml_b200_comm_connect(self.h, buf), "maml_b200_comm_connect")

    def comm_world(self):
        return int(self.lib.maml_b200_comm_world(self.h))

    def all_reduce(self, vec):
        _check(self.lib, self.lib.maml_b200_all_reduce(self.h, vec.data_ptr(), self._stream()), "maml_b200_all_reduce")

    def comm_status(self):
        return int(self.lib.maml_b200_comm_status(self.h))

    def trace(self, enable):
        _check(self.lib, self.lib.maml_b200_trace(self.h, int(bool(enable))), "maml_b200_trace")

    def trace_read(self, capacity=4096):
        """[(t_ns, kernel_id, launch_tag)] of every kernel started since trace(True) / the last read, in start order
        (launch_tag = launch sequence number inside the iteration = kernel-node order of the captured graph)."""
        buf = (ctypes.c_uint64 * capacity)()
        n = self.lib.maml_b200_trace_read(self.h, buf, capacity)
        if n < 0:
            raise RuntimeError("maml_b200_trace_read: " + self.lib.maml_b200_last_error().decode())
        return [(int(buf[i]) >> 20, int(buf[i]) & 0xff, (int(buf[i]) >> 8) & 0xfff) for i in range(n)]

    def profile(self, enable):
        _check(self.lib, self.lib.maml_b200_profile(self.h, int(bool(enable))), "maml_b200_profile")

    def profile_read(self):
        """{category: (ms, algorithmic_flops, launches)} since profile(True); synchronises."""
        n = len(PROF_CATS)
        ms, fl, ln = (ctypes.c_double * n)(), (ctypes.c_double * n)(), (ctypes.c_int64 * n)()
        _check(self.lib, self.lib.maml_b200_profile_read(self.h, ms, fl, ln, n), "maml_b200_profile_read")
        return {PROF_CATS[i]: (ms[i], fl[i], ln[i]) for i in range(n)}

    def last_launch_count(self):
        return int(self.lib.maml_b200_last_launch_count(self.h))

    def debug_read(self, name, task=0, step=0, layer=0):
        import numpy as np
        n = self.lib.maml_b200_debug_read(self.h, name.encode(), task, step, layer, None, 0)
        if n < 0:
            raise RuntimeError("debug_read(%s): %s" % (name, self.lib.maml_b200_last_error().decode()))
        out = np.empty(int(n), dtype=np.float32)
        n2 = self.lib.maml_b200_debug_read(self.h, name.encode(), task, step, layer,
                                           out.ctypes.data_as(ctypes.c_void_p), int(n))
        if n2 < 0:
            raise RuntimeError("debug_read(%s): %s" % (name, self.lib.maml_b200_last_error().decode()))
        return out
