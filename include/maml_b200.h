/*
 * maml_b200.h -- C ABI of the H100-native MAML / MAML++ inner-loop engine.
 *
 * Drop-in boundary for ONE hot path of AntreasAntoniou/HowToTrainYourMAMLPytorch:
 *   MAMLFewShotClassifier.run_train_iter / run_validation_iter
 *     (reference few_shot_learning_system.py:338-369, :371-397)
 *   -> forward over tasks and inner steps            (reference :170-263)
 *   -> VGGReLUNormNetwork.forward                    (reference meta_neural_network_architectures.py:620-660)
 *   -> LSLRGradientDescentLearningRule.update_params (reference inner_loop_optimizers.py:99-113)
 *   -> meta_update: backward + clamp + Adam          (reference few_shot_learning_system.py:325-336)
 *
 * The reference has no FFI of its own (it is pure Python on top of PyTorch); these entry
 * points are what a ctypes binding inside the reference's MAMLFewShotClassifier would call
 * (the stub is shown in INTEGRATION.md).  Plain pointers and sizes only -- no torch types.
 * All `const float*` / `float*` data pointers are DEVICE pointers owned by the caller;
 * kernels are enqueued on the caller's stream (`stream` is a cudaStream_t passed as void*)
 * and nothing synchronises with the host unless stated.  Every function returns 0 on
 * success and a non-zero code on failure; maml_b200_last_error() gives the message.
 */
#ifndef MAML_B200_H_
#define MAML_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MAML_B200_MAX_STAGES 4
#define MAML_B200_MAX_STEPS 8
#define MAML_B200_ABI_VERSION 5

/* Static shape of the path.  Mirrors the args the reference reads on this path:
 * num_classes_per_set, num_samples_per_class, num_target_samples, image_{channels,height,width},
 * cnn_num_filters, num_stages, number_of_training_steps_per_iter, per_step_bn_statistics, norm_layer,
 * enable_inner_loop_optimizable_bn_params. */
typedef struct maml_b200_config {
  int32_t n_way;        /* N  classes per task                         */
  int32_t k_shot;       /* K  support samples per class                */
  int32_t t_target;     /* T  target samples per class                 */
  int32_t channels;     /* C  image channels                           */
  int32_t height;       /* H                                           */
  int32_t width;        /* W                                           */
  int32_t filters;      /* F  cnn_num_filters, multiple of 16, <= 64   */
  int32_t num_stages;   /* conv blocks, 1..4                           */
  int32_t inner_steps;  /* S  number_of_training_steps_per_iter, <= 8  */
  int32_t per_step_bn;  /* per_step_bn_statistics (MAML++) 0/1         */
  int32_t max_tasks;    /* max tasks per call on this GPU (workspace)  */
  int32_t reserved;     /* test switches. bit 0: keep the activations of EVERY target pass for debug_read;
                           bit 1: run blocks l >= 1 on the fp32 FFMA kernels instead of wgmma 3xTF32 */
  int32_t norm_layer;   /* 0: batch norm; 1: layer norm (reference MetaLayerNormLayer: statistics per image over
                           [F, h, w], frozen all-ones weight, learnable bias [F, h, w]; per_step_bn is then ignored,
                           there are no running statistics).  Layer-norm handles run every entry; the layer norm has
                           no per-step rows, so the functional entries (maml_b200_net_*) compute the same at every
                           num_step, and maml_b200_net_running_update is a no-op. */
  int32_t inner_bn;     /* 1: enable_inner_loop_optimizable_bn_params (batch norm only: refused with norm_layer = 1).  Each
                           block's norm_layer.bias / .weight (beta, gamma) are [F] whatever per_step_bn is, and are
                           inner-loop fast weights: per task, updated by the LSLR rule with their own rate vectors, and
                           differentiated to second order like the conv weights.  The running statistics keep their
                           per-step rows when per_step_bn is set.  Of the functional entries (maml_b200_net_*) these
                           handles run the per-task ones (maml_b200_net_*_tasks), the image gradients and the running-
                           statistics update; the shared-weight entries (net_forward, net_backward, net_hvp,
                           net_hvp_image, net_jvp) refuse them. */
} maml_b200_config;

/* Per-call schedule: what reference forward(...) derives from epoch / phase (:232-244,:304-305). */
typedef struct maml_b200_iter_args {
  int32_t n_tasks;        /* tasks in this call (local shard), <= max_tasks                  */
  int32_t task_offset;    /* global index of the first local task (running-stat ordering)    */
  int32_t tasks_global;   /* B: global meta-batch size (gradient / loss mean denominator)     */
  int32_t num_steps;      /* inner steps to run (training: S; eval: evaluation steps)        */
  int32_t second_order;   /* 1: use Hessian-vector terms (reference use_second_order)        */
  int32_t training;       /* 1: produce meta-gradient; 0: evaluation (forward only)          */
  uint32_t target_mask;   /* bit s set: target pass after inner step s                       */
  float target_weight[MAML_B200_MAX_STEPS]; /* loss weight of that pass (MSL weight or 1)    */
} maml_b200_iter_args;

typedef struct maml_b200_handle maml_b200_handle;

int maml_b200_abi_version(void);
const char* maml_b200_last_error(void);

/* Create / destroy an engine for one static shape on the current CUDA device.  Allocates the
 * activation / fast-weight workspace (cudaMalloc) sized for cfg->max_tasks. */
int maml_b200_create(const maml_b200_config* cfg, maml_b200_handle** out);
void maml_b200_destroy(maml_b200_handle* h);
int64_t maml_b200_workspace_bytes(const maml_b200_handle* h);

/* Flat meta-parameter vector ("meta"), reference layout and reference Adam order
 * (reference few_shot_learning_system.py:288-294): per block conv.weight[F,Cin,3,3],
 * conv.bias[F], norm_layer.bias[S|1,F], norm_layer.weight[S|1,F] (layer norm: conv.weight, conv.bias,
 * norm_layer.bias[F,h_l,w_l]; inner_bn: norm_layer.bias[F], norm_layer.weight[F]); then linear.weights[N,D], linear.bias[N];
 * then the LSLR vectors [S+1] in inner-parameter order (the reference's get_inner_loop_parameter_dict): 2*stages+2 of them
 * (per block conv.weight, conv.bias; then linear.weights, linear.bias), or with inner_bn 4*stages+2 (per block conv.weight,
 * conv.bias, norm_layer.bias, norm_layer.weight; then the linear layer's).
 * Fast weights (per task, inside the engine): the inner tensors in that order, conv weights as [3*3][Cin][F]. */
int32_t maml_b200_num_segments(const maml_b200_handle* h);
int maml_b200_segment(const maml_b200_handle* h, int32_t idx, int64_t* offset, int64_t* size);
int64_t maml_b200_meta_size(const maml_b200_handle* h);

/* Result vector written by maml_b200_meta_batch_fwd_bwd (floats):
 *   [0, meta_size)                     meta-gradient, same layout as meta, already (1/B)-scaled
 *                                      and summed over the LOCAL tasks (all-reduce SUM completes it)
 *   [meta_size]                        sum over local tasks of task_loss / B
 *   [meta_size + 1]                    number of correct last-step target predictions (local)
 *   [meta_size + 2, +stages*S*F)       running-mean EMA partial sums   (per_step_bn batch norm only)
 *   [.. , +stages*S*F)                 running-var  EMA partial sums   (per_step_bn batch norm only)
 * The whole vector is linear in the tasks, so ONE all-reduce(sum) over ranks finishes it. */
int64_t maml_b200_result_size(const maml_b200_handle* h);

/* The hot path: for every local task, S inner steps of (support forward, hand-rolled
 * gradient, LSLR fast-weight update, target forward), then the reverse sweep producing the
 * (second-order) meta-gradient.  Replaces reference forward() + loss.backward().
 *   meta        [meta_size]                      flat meta-parameters (see above)
 *   x_support   [n_tasks, N*K, C, H, W] fp32     y_support [n_tasks, N*K] int64
 *   x_target    [n_tasks, N*T, C, H, W] fp32     y_target  [n_tasks, N*T] int64
 *   result      [result_size]                    (out)
 *   last_logits [n_tasks, N*T, N]                (out) logits of the last target pass
 */
int maml_b200_meta_batch_fwd_bwd(maml_b200_handle* h, const maml_b200_iter_args* it,
                                 const float* meta,
                                 const float* x_support, const int64_t* y_support,
                                 const float* x_target, const int64_t* y_target,
                                 float* result, float* last_logits, void* stream);

/* Stand-alone functional forward: replaces reference VGGReLUNormNetwork.forward(x, num_step, params)
 * (meta_neural_network_architectures.py:620-660) for batches of N*T images: conv / BatchNorm(batch statistics, gamma and
 * beta of `num_step`) or layer norm (per-image statistics, + bias) / leaky-ReLU / maxpool x stages, flatten, linear.  `meta_like`: same layout as the meta vector,
 * conv / linear entries = the (fast) weights to use.  x [n_tasks, N*T, C, H, W]; logits [n_tasks, N*T, N] (out). */
int maml_b200_net_forward(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like,
                          const float* x, float* logits, void* stream);

/* Backward of maml_b200_net_forward (so that torch.autograd can differentiate through the functional operator, as the
 * reference's apply_inner_loop_update does with torch.autograd.grad, few_shot_learning_system.py:138-139; first order).
 * Must directly follow maml_b200_net_forward (or another maml_b200_net_backward of it) on the same handle with the same
 * (n_tasks, num_step, meta_like).  Another order, n_tasks or num_step makes it fail with an error and launch nothing (the
 * handle records its last functional call; meta_like it cannot check).
 *   dlogits  [n_tasks, N*T, N]   d(loss) / d(logits)
 *   grad_out [result_size]       (out) first meta_size floats = d(loss) / d(meta_like) in the meta layout (conv / linear
 *                                weights and biases, BatchNorm beta / gamma rows of num_step or the layer-norm biases;
 *                                LSLR entries 0), summed over
 *                                the n_tasks batches.  The gradient with respect to the images is a separate call,
 *                                maml_b200_net_input_grad. */
int maml_b200_net_backward(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like,
                           const float* dlogits, float* grad_out, void* stream);

/* Second-order companion of maml_b200_net_backward: for the batch x, weights meta_like and upstream dlogits, one
 * forward-over-reverse pass along v_like (meta layout; its LSLR entries are not read, nor are its BatchNorm entries on a
 * plain BatchNorm handle, which has no gamma / beta tangent directions; on a layer-norm handle its bias entries are bias
 * directions, and an inner_bn handle's gamma / beta directions run through maml_b200_net_hvp_image_tasks).  Self-contained: it recomputes the forward and the backward of dlogits itself, so it
 * needs no earlier call.  The batch has the handle's SUPPORT shape: N*K images (create the handle with k_shot = batch / N).
 *   x          [n_tasks, N*K, C, H, W]
 *   dlogits    [n_tasks, N*K, N]  d(loss) / d(logits), held constant along v
 *   jv_out     [n_tasks, N*K, N]  = J(meta_like) v           (tangent of the logits)
 *   hv_out     result_size floats; first meta_size = d/d(meta_like) <dlogits, J v> in the meta layout
 *              (conv / linear weights and biases, BatchNorm gamma / beta of num_step or the layer-norm biases, +H v;
 *              LSLR entries 0), summed over the n_tasks batches
 * No running-statistics side effect; it overwrites the batch statistics maml_b200_net_running_update reads. */
int maml_b200_net_hvp(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like, const float* x,
                      const float* dlogits, const float* v_like, float* jv_out, float* hv_out, void* stream);

/* maml_b200_net_hvp with an image tangent as well: the tangent direction is (v_like, xdot), xdot [n_tasks, N*K, C, H, W]
 * or NULL (then exactly maml_b200_net_hvp).  jv_out = J_theta v + J_x xdot; hv_out = d/d(meta_like) <dlogits, jv_out>,
 * laid out as in maml_b200_net_hvp.  Like it, it may be followed by maml_b200_net_hvp_input_grad, which then gives
 * d/dx <dlogits, jv_out>.  The image-tangent buffer is allocated by the first call with xdot != NULL, outside the
 * workspace. */
int maml_b200_net_hvp_image(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like, const float* x,
                            const float* xdot, const float* dlogits, const float* v_like, float* jv_out, float* hv_out,
                            void* stream);

/* Forward mode of the functional operator: the logits tangent J_theta t + J_x xdot at the weights meta_like, for batches of
 * the handle's SUPPORT shape (N*K images).  Self-contained: one primal forward, then one tangent forward; no backward.
 *   x, xdot    [n_tasks, N*K, C, H, W]; xdot may be NULL (no image tangent)
 *   t_like     meta layout: conv / linear tangents and the BatchNorm beta / gamma tangents of num_step (layer norm: the
 *              bias tangents); LSLR entries are not read
 *   jv_out     [n_tasks, N*K, N]
 * No running-statistics side effect; it overwrites the batch statistics maml_b200_net_running_update reads.  Its small
 * buffers (zero d(logits), the image tangent) are allocated by the first call that needs them, outside the workspace. */
int maml_b200_net_jvp(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like, const float* x,
                      const float* t_like, const float* xdot, float* jv_out, void* stream);

/* Per-task forms of net_forward / net_backward / net_hvp_image / net_jvp: n_tasks independent problems in one call, each with its
 * own weights (what torch.func.vmap over tasks runs as one call).  Same shapes, ordering rules and side effects as the
 * entries above, plus:
 *   meta_stride  floats between consecutive tasks' meta_like vectors: task t's conv / linear weights are at
 *                meta_like + t * meta_stride; 0 = one vector shared by every task (the entries above)
 *   dir_stride   the same for v_like / t_like (0 = shared)
 *   sum_tasks    1: grad_out / hv_out = result_size floats summed over the tasks (the entries above);
 *                0: n_tasks x result_size floats, task t's vector (not summed) at + t * result_size
 * BatchNorm gamma / beta and the layer-norm biases are shared by the tasks of a call: they are read from task 0's vector
 * (meta_like's own rows), whatever meta_stride is; so are net_jvp_tasks' BatchNorm gamma / beta tangents, whatever
 * dir_stride is.  The layer-norm bias DIRECTIONS of net_hvp_image_tasks / net_jvp_tasks follow dir_stride (per task), and
 * each task's bias gradient goes to its own result vector.  On an inner_bn handle gamma / beta are per-task fast weights:
 * they follow meta_stride (each task's own beta / gamma rows), their directions and tangents follow dir_stride, and each
 * task's beta / gamma gradient (+H_beta v, +H_gamma v for net_hvp_image_tasks) goes to its own result vector (or into the
 * sum).  A stride that is neither 0 nor >= meta_size is an error.
 * maml_b200_net_input_grad, maml_b200_net_hvp_input_grad and maml_b200_net_running_update already work per task and follow
 * these entries as they follow the ones above. */
int maml_b200_net_forward_tasks(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like,
                                int64_t meta_stride, const float* x, float* logits, void* stream);
int maml_b200_net_backward_tasks(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like,
                                 int64_t meta_stride, const float* dlogits, float* grad_out, int32_t sum_tasks, void* stream);
int maml_b200_net_hvp_image_tasks(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like,
                                  int64_t meta_stride, const float* x, const float* xdot, const float* dlogits,
                                  const float* v_like, int64_t dir_stride, float* jv_out, float* hv_out, int32_t sum_tasks,
                                  void* stream);
int maml_b200_net_jvp_tasks(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like,
                            int64_t meta_stride, const float* x, const float* t_like, int64_t dir_stride, const float* xdot,
                            float* jv_out, void* stream);

/* Gradients with respect to the images.  Each reads the buffers of the functional call that ran last on this handle and
 * must follow it immediately, with the same n_tasks: another call on the handle in between (a functional call, an
 * iteration) makes it fail with an error and launch nothing.
 *   net_input_grad      after maml_b200_net_backward:  dx_out    [n_tasks, N*T, C, H, W] = J_x^T dlogits
 *   net_hvp_input_grad  after maml_b200_net_hvp:       dxdot_out [n_tasks, N*K, C, H, W] = d/dx <dlogits, J v>
 *                       (the mixed second-order term: the tangent of the image gradient along v) */
int maml_b200_net_input_grad(maml_b200_handle* h, int32_t n_tasks, float* dx_out, void* stream);
int maml_b200_net_hvp_input_grad(maml_b200_handle* h, int32_t n_tasks, float* dxdot_out, void* stream);

/* EMA side effect of the functional forward (F.batch_norm updating running_mean / running_var at num_step, reference
 * meta_neural_network_architectures.py:226-247) from the batch statistics of the last maml_b200_net_forward call.  Like
 * maml_b200_net_backward it must follow that forward (or a maml_b200_net_backward of it) with the same n_tasks and
 * num_step, and otherwise fails with an error and launches nothing: another functional call in between, e.g.
 * maml_b200_net_hvp, overwrites those statistics.  running_mean / running_var: [stages][S][F] device.  No-op without
 * per-step BatchNorm (shared BatchNorm, layer norm). */
int maml_b200_net_running_update(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, float* running_mean,
                                 float* running_var, void* stream);

/* Outer step on the flat vectors: optional clamp to [-10,10] (reference :332-335), Adam
 * (betas 0.9/0.999, eps 1e-8, no weight decay; reference :69,:336).  `grad` is the first
 * meta_size floats of (the all-reduced) result.  Bit i of trainable_mask / clamp_mask refers to
 * segment i (an inner_bn handle with 4 blocks has 36 segments).  `step` is the 1-based Adam step count of this update. */
int maml_b200_adam_step(maml_b200_handle* h, float* meta, const float* grad,
                        float* exp_avg, float* exp_avg_sq,
                        float lr, int32_t step, uint64_t trainable_mask, uint64_t clamp_mask,
                        void* stream);

/* Running-statistics EMA finalisation (side effect of F.batch_norm in the reference,
 * meta_neural_network_architectures.py:226-247): running[l][s][f] = decay[s]*running + part.
 * `result` is the (all-reduced) result vector; decay[s] = 0.9^(updates at step s), host array
 * of inner_steps floats.  running_mean / running_var: [stages][S][F] device. */
int maml_b200_running_stats_update(maml_b200_handle* h, const float* result,
                                   float* running_mean, float* running_var,
                                   const float* decay_host, void* stream);

/* Multi-GPU (one process per GPU, all on one node): the ONE collective of an iteration -- all-reduce(SUM) of the result
 * vector over the ranks -- runs as kernels over peer memory (NVLink / NVSwitch) inside the iteration's own CUDA graph.
 * It replaces the reference's nn.DataParallel scatter / gather (few_shot_learning_system.py:74-77).
 *   comm_init     allocates this rank's communication block and returns its 64-byte CUDA IPC handle;
 *   (the caller exchanges the handles between the ranks, e.g. torch.distributed.all_gather_object)
 *   comm_connect  maps every peer's block: all_handles = world x 64 bytes in rank order.
 * Afterwards every maml_b200_meta_batch_fwd_bwd call with tasks_global > n_tasks leaves the all-reduced vector in
 * `result` on every rank (bit-identical: the ranks are summed in rank order).  All ranks must issue the same sequence of
 * sharded calls.  A rank that waits more than 30 s for a peer gives up and reports it through comm_status. */
int maml_b200_comm_init(maml_b200_handle* h, int32_t rank, int32_t world, void* ipc_handle_out);
int maml_b200_comm_connect(maml_b200_handle* h, const void* all_handles);
int maml_b200_comm_world(const maml_b200_handle* h);
int maml_b200_all_reduce(maml_b200_handle* h, float* vec, void* stream);   /* stand-alone, in place, result_size floats */
int64_t maml_b200_comm_status(maml_b200_handle* h);

/* GPU-resident episode assembly -- replaces the reference's worker-process loader for in-memory datasets
 * (data.py:478-524 get_set: class / sample selection is seeded host arithmetic, the image work happens here):
 *   dataset      [n_images, H, W, C] fp32 device (what the reference keeps in RAM: Omniglot binary floats, ImageNet x/255)
 *   image_index  [n_tasks, N, K+T] int64 device: dataset row of every sampled image (support samples first)
 *   rot_k        [n_tasks, N] int32 device: np.rot90 count of the class (Omniglot train augmentation, data.py:17-34), 0 = none
 *   mean/std     host arrays of C floats (ImageNet normalisation, data.py:100-106) or NULL
 * Writes x_support [n_tasks,N,K,C,H,W], x_target [n_tasks,N,T,C,H,W] (fp32) and the class-major labels (int64). */
int maml_b200_episode_gather(const float* dataset, const int64_t* image_index, const int32_t* rot_k, int32_t n_tasks,
                             int32_t n_way, int32_t k_shot, int32_t t_target, int32_t channels, int32_t height, int32_t width,
                             const float* mean_host, const float* std_host, float* x_support, float* x_target,
                             int64_t* y_support, int64_t* y_target, void* stream);

/* Debug / test hook: copy one named internal buffer of the last call to host memory.
 * Returns the number of floats the buffer holds (or <0 on error); copies at most `capacity`.
 * Names: see DESIGN.md ("debug taps").  Synchronises the device. */
int64_t maml_b200_debug_read(maml_b200_handle* h, const char* name, int32_t task, int32_t step,
                             int32_t layer, float* host_out, int64_t capacity);

/* Per-launch profiling with CUDA events on the launching stream (bench.py's roofline leg; adds two event
 * records per launch, so never leave it on in a timed throughput run).  Categories (MAML_B200_PROF_*):
 * 0 implicit-GEMM conv (forward / tangent / dgrad), 1 first-block conv, 2 wgrad, 3 first-block wgrad,
 * 4 BatchNorm/leaky-ReLU/pool kernels, 5 classifier head, 6 parameter-space kernels.
 * profile_read synchronises the device, sums elapsed ms, ALGORITHMIC flops (conv MACs x 2 on valid pixels,
 * SURVEY.md section 8d) and launch counts per category since profile(h, 1), and clears the records. */
#define MAML_B200_PROF_CATS 7
int maml_b200_profile(maml_b200_handle* h, int32_t enable);
int maml_b200_profile_read(maml_b200_handle* h, double* ms_by_cat, double* flops_by_cat,
                           int64_t* launches_by_cat, int32_t ncat);

/* Device-side launch trace (debug): while enabled, CTA (0,0,0) of every kernel appends (globaltimer ns << 20 | launch
 * tag << 8 | kernel id; tag = launch sequence number inside the iteration = kernel-node order of the captured graph) to a device buffer -- the start-time sequence of the kernels of the following calls, also inside a replayed CUDA
 * graph.  trace_read synchronises, copies at most `capacity` entries (start order), clears, and returns the count.
 * Kernel ids: scripts/trace_kernel_ids.json. */
int maml_b200_trace(maml_b200_handle* h, int32_t enable);
int64_t maml_b200_trace_read(maml_b200_handle* h, uint64_t* out, int64_t capacity);

/* Number of kernel launches issued by the last maml_b200_meta_batch_fwd_bwd call. */
int64_t maml_b200_last_launch_count(const maml_b200_handle* h);

#ifdef __cplusplus
}
#endif
#endif /* MAML_B200_H_ */
