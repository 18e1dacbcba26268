// Classifier-head device code shared by kernels_head.cu (stand-alone kernel) and kernels_bn.cu (fused last-block kernels).
#pragma once
#include "common.cuh"

// loop prefix used inside head_body: `#pragma unroll 1` cannot depend on a template parameter, so the body is compiled from
// this header twice through the macro below (see head_body_compact / head_body_unrolled at the end)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Body of the head for (row group `group`, task `task`): everything except the weight gradient is row-local, so each
// CTA owns `rows_per_cta` rows of the batch and writes its own chunk of (gW, gb); the parameter-space kernel sums the
// chunks in order.  `smh`: 5 * rows_per_cta * N floats of shared memory; 256 threads.  Also called by the fused
// last-block kernels (kernels_bn.cu).
// COMPACT = true: every loop stays rolled.  The fused last-block kernels and the small-D heads (Omniglot: D = 64) execute this
// code ONCE per launch and are instruction-fetch bound; rolled loops cut their SASS
// from ~6.2 k to ~3.8 k instructions.  Large-D heads (Mini-ImageNet: D = 1200) keep the
// compiler's unrolling: rolled, their D-loops ran 2x slower.
#define HEAD_LOOP _Pragma("unroll 1")
#define HEAD_BODY_NAME head_body_compact
#include "head_body_impl.inc"
#undef HEAD_LOOP
#undef HEAD_BODY_NAME
#define HEAD_LOOP
#define HEAD_BODY_NAME head_body_unrolled
#include "head_body_impl.inc"
#undef HEAD_LOOP
#undef HEAD_BODY_NAME

// EXT_TAN = false compiles the HEAD_EXTERNAL_TAN branch out, so the kernels that run the fused iteration's modes (the fused
// last-block kernels, the head kernel's default instantiations) keep their code; launch_head picks EXT_TAN by mode.
template <bool COMPACT, bool EXT_TAN = false>
__device__ __forceinline__ void head_body(const HeadArgs& a, int task, int group, float* smh, float* s_rowloss, float* s_rowcorrect) {
  if constexpr (COMPACT) head_body_compact<EXT_TAN>(a, task, group, smh, s_rowloss, s_rowcorrect);
  else head_body_unrolled<EXT_TAN>(a, task, group, smh, s_rowloss, s_rowcorrect);
}
