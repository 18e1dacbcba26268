"""Task sharding across ranks (SURVEY.md section 8e) -- host-side arithmetic.

Tasks are independent given the meta-parameters and every output of an iteration is LINEAR in the
tasks, so rank r of G takes tasks [r*B_local, (r+1)*B_local) and one all-reduce(SUM) of the flat result
vector finishes the iteration:
  * meta-gradient and loss: each rank contributes (1/B_global) * sum over its tasks;
  * accuracy: count of correct predictions;
  * BatchNorm running statistics: the reference applies r <- 0.9 r + 0.1 stat sequentially over the
    GLOBAL task order (support pass, then target pass if one runs at that step).  Unrolled,
        r_new = 0.9^U r_old + sum_k 0.1 * 0.9^(U-1-k) stat_k,      U = updates at that step,
    so each rank pre-weights its own statistics by their (static) position k and the same all-reduce
    reproduces the sequential result.  (csrc/kernels_param.cu: export_kernel computes the weighted sums.)
    The layer-norm network (norm_layer "layer_norm") has no running statistics: its result vector ends after the
    number of correct predictions, and nothing here applies to it.
"""

BN_MOMENTUM = 0.1


def shard_of(rank, world_size, local_tasks):
    """(task_offset, tasks_global) of a rank holding ``local_tasks`` tasks."""
    return rank * local_tasks, world_size * local_tasks


def updates_per_task(step_has_target):
    return 2 if step_has_target else 1


def ema_decay(step_has_target, tasks_global):
    """0.9^U: factor applied to the old running statistic of one inner step."""
    return (1.0 - BN_MOMENTUM) ** (updates_per_task(step_has_target) * tasks_global)


def ema_weight(global_task, which, step_has_target, tasks_global):
    """Weight of one statistic in the unrolled EMA.  ``which``: 0 = support pass, 1 = target pass."""
    c = updates_per_task(step_has_target)
    U = c * tasks_global
    k = c * global_task + which
    return BN_MOMENTUM * (1.0 - BN_MOMENTUM) ** (U - 1 - k)


def decay_vector(target_mask, num_steps, inner_steps, tasks_global):
    """Per-step decay factors handed to ``maml_b200_running_stats_update`` (1.0 for steps not run)."""
    return [ema_decay(bool((target_mask >> s) & 1), tasks_global) if s < num_steps else 1.0
            for s in range(inner_steps)]
