// Classifier head: flatten + linear + mean softmax cross-entropy, its gradient, and the forward-mode
// tangent of both.  One CTA per task (n <= ~100 rows, N <= 32 classes, D <= a few thousand).
// Restates reference meta_neural_network_architectures.py:657-658 / :141 (view + F.linear) and
// few_shot_learning_system.py:284 (F.cross_entropy, mean reduction); tangent: SURVEY.md appendix A3.
//
// Feature order: f[i][d] with d = pixel * F + channel (grid order).  The fast weights keep W_fc in
// the same internal order; import / export kernels permute from / to the reference's
// channel-major flatten (NCHW .view(n, -1)).
#include "common.cuh"

#include "head_body.cuh"

template <bool COMPACT, bool EXT_TAN>
__global__ void __launch_bounds__(256) head_kernel(HeadArgs a) {
  pdl_prologue(14, a.tag);
  extern __shared__ float smh[];
  __shared__ float s_rowloss[64];
  __shared__ float s_rowcorrect[64];
  head_body<COMPACT, EXT_TAN>(a, blockIdx.y, blockIdx.x, smh, s_rowloss, s_rowcorrect);
}

void launch_head(const HeadArgs& a, cudaStream_t st) {
  ProfScope prof_scope__(PROF_HEAD, 0.0, st);
  const size_t smem = (size_t)5 * a.rows_per_cta * a.N * sizeof(float);
  dim3 grid((a.n + a.rows_per_cta - 1) / a.rows_per_cta, a.tasks);
  // small feature vectors (Omniglot: D = 64): the rolled-loop body (less code to fetch for a kernel that runs once);
  // large ones (Mini-ImageNet: D = 1200): the compiler's unrolled D-loops
  // HEAD_EXTERNAL_TAN (functional operator only) has instantiations of its own: the iteration's heads keep their code
  if (a.mode == HEAD_EXTERNAL_TAN) {
    if (a.D <= 256) launch_pdl(head_kernel<true, true>, dim3(grid), dim3(256), (size_t)(smem), st, tagged(a));
    else launch_pdl(head_kernel<false, true>, dim3(grid), dim3(256), (size_t)(smem), st, tagged(a));
  } else {
    if (a.D <= 256) launch_pdl(head_kernel<true, false>, dim3(grid), dim3(256), (size_t)(smem), st, tagged(a));
    else launch_pdl(head_kernel<false, false>, dim3(grid), dim3(256), (size_t)(smem), st, tagged(a));
  }
  CUDA_CHECK_LAUNCH();
}

MAML_TRACE_SETTER(trace_set_head)
