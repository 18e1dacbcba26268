// Parameter-space kernels: import of the meta-parameters into the per-task fast-weight layout, the
// LSLR fast-weight update fused with the deterministic reduction of the wgrad partials, the reverse
// sweep bookkeeping (alpha-bar, u = alpha * theta-bar), export of the meta-gradient in the
// reference's layout, fused clamp + Adam, running-statistic EMA.
//
// Restates reference inner_loop_optimizers.py:99-113 (theta' = theta - alpha[name][step] * g),
// few_shot_learning_system.py:105-120 (which tensors adapt), :325-336 (clamp + Adam),
// meta_neural_network_architectures.py:226-247 (running-stat EMA side effect) and SURVEY.md A4.
#include "common.cuh"

// internal index (per-task fast-weight vector) -> index in the reference-layout flat meta vector
__device__ __forceinline__ long long internal_to_meta(const ParamLayout& pl, long long i, int* seg_out) {
  const int spb = seg_per_block(pl);
  for (int l = 0; l < pl.L; ++l) {
    const long long wsz = 9LL * pl.cin[l] * pl.F;
    if (i >= pl.w_off[l] && i < pl.w_off[l] + wsz) {
      const long long rel = i - pl.w_off[l];
      const int f = (int)(rel % pl.F);
      const int c = (int)((rel / pl.F) % pl.cin[l]);
      const int tap = (int)(rel / ((long long)pl.F * pl.cin[l]));
      *seg_out = spb * l;
      return pl.m_w[l] + ((long long)f * pl.cin[l] + c) * 9 + tap;
    }
    if (i >= pl.b_off[l] && i < pl.b_off[l] + pl.F) {
      *seg_out = spb * l + 1;
      return pl.m_b[l] + (i - pl.b_off[l]);
    }
    if (pl.inner_bn && i >= pl.beta_off[l] && i < pl.beta_off[l] + 2 * pl.F) {     // beta_l, then gamma_l
      const bool is_gamma = i >= pl.gamma_off[l];
      *seg_out = spb * l + (is_gamma ? 3 : 2);
      return is_gamma ? pl.m_gamma[l] + (i - pl.gamma_off[l]) : pl.m_beta[l] + (i - pl.beta_off[l]);
    }
  }
  const long long D = (long long)pl.pix * pl.F;
  if (i >= pl.fcw_off && i < pl.fcw_off + (long long)pl.N * D) {
    const long long rel = i - pl.fcw_off;
    const int k = (int)(rel / D);
    const int r2 = (int)(rel % D);
    const int pix = r2 / pl.F, c = r2 % pl.F;
    *seg_out = spb * pl.L;
    return pl.m_fcw + (long long)k * D + (long long)c * pl.pix + pix;
  }
  *seg_out = spb * pl.L + 1;
  return pl.m_fcb + (i - pl.fcb_off);
}

// src_stride 0: one meta vector broadcast to every task; otherwise task t reads meta + t * src_stride
__global__ void import_theta_kernel(ParamLayout pl, const float* __restrict__ meta, float* __restrict__ theta0,
                                    long long stride, int tasks, long long src_stride, int tag) {
  pdl_prologue(15, tag);
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= pl.P) return;
  int seg;
  const long long mi = internal_to_meta(pl, i, &seg);
  for (int t = 0; t < tasks; ++t) theta0[(long long)t * stride + i] = meta[(long long)t * src_stride + mi];
}

void launch_import_theta(const ParamLayout& pl, const float* meta, float* theta0, long long stride, int tasks,
                         cudaStream_t st, long long meta_task_stride) {
  ProfScope prof_scope__(PROF_PARAM, 0.0, st);
  launch_pdl(import_theta_kernel, dim3((unsigned)((pl.P + 255) / 256)), dim3(256), (size_t)(0), st, pl, meta, theta0, stride, tasks,
             meta_task_stride, launch_tag());
  CUDA_CHECK_LAUNCH();
}

__device__ __forceinline__ int seg_of(const ParamLayout& pl, long long i) {
  int s = 0;
  for (int k = 1; k < pl.nseg_inner; ++k)
    if (i >= pl.seg_off[k]) s = k;
  return s;
}

// reduce the gradient chunks of every inner tensor (fixed order; inner-loop BatchNorm beta / gamma: read the fp64 sums, see
// PartialDesc) and
//   PR_UPDATE: g_out = sum; theta_out = theta_in - alpha[seg][step] * sum     (LSLR step)
//   PR_STORE : g_out = sum
//   PR_SUB   : tbar -= sum
__global__ void param_reduce_kernel(ParamLayout pl, PartialDesc pd, const float* __restrict__ partial, int mode,
                                    const float* __restrict__ theta_in, float* __restrict__ theta_out,
                                    float* __restrict__ g_out, float* __restrict__ tbar,
                                    const float* __restrict__ meta, int step, long long task_stride, long long i_lo,
                                    long long i_hi, int tag) {
  pdl_prologue(16, tag);
  const long long i = i_lo + (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= i_hi) return;
  const int task = blockIdx.y;
  const int seg = seg_of(pl, i);
  float s = 0.f;
  if (pd.nchunks[seg] == 0) {
    // beta_l (segment 2 of block l: S1 = sum dy) or gamma_l (segment 3: S2 = sum dy * zh); nothing without sums
    const int spb = seg_per_block(pl);
    if (pd.bn_sums)
      s = (float)pd.bn_sums[(long long)task * pd.bn_task_stride + (long long)(seg / spb) * pd.bn_layer_stride +
                            (i - pl.seg_off[seg]) * 2 + (seg % spb - 2)];
  } else {
    const float* p = partial + (long long)task * pd.task_stride + pd.off[seg] + (i - pl.seg_off[seg]);
    for (int c = 0; c < pd.nchunks[seg]; ++c) s += p[(long long)c * pd.cstride[seg]];   // fixed order: deterministic
  }
  const long long o = (long long)task * task_stride + i;
  if (mode == PR_UPDATE) {
    const float alpha = meta[pl.m_lslr + (long long)seg * (pl.S + 1) + step];
    g_out[o] = s;
    theta_out[o] = theta_in[o] - alpha * s;
  } else if (mode == PR_STORE) {
    g_out[o] = s;
  } else {
    tbar[o] -= s;
  }
}

void launch_param_reduce(const ParamLayout& pl, const PartialDesc& pd, const float* partial, int mode,
                         const float* theta_in, float* theta_out, float* g_out, float* tbar, const float* meta, int step,
                         long long task_stride, int tasks, cudaStream_t st, int seg_lo, int seg_hi) {
  // inner tensors [seg_lo, seg_hi) only (default: all) -- the engine reduces the first block's tensors separately
  // because their gradient chunks are the last thing a backward pass produces
  if (seg_hi < 0 || seg_hi > pl.nseg_inner) seg_hi = pl.nseg_inner;
  if (seg_lo >= seg_hi) return;
  const long long i_lo = pl.seg_off[seg_lo];
  const long long i_hi = seg_hi == pl.nseg_inner ? pl.P : pl.seg_off[seg_hi];
  ProfScope prof_scope__(PROF_PARAM, 0.0, st);
  dim3 grid((unsigned)((i_hi - i_lo + 255) / 256), tasks);
  launch_pdl(param_reduce_kernel, dim3(grid), dim3(256), (size_t)(0), st, pl, pd, partial, mode, theta_in, theta_out, g_out, tbar, meta, step, task_stride, i_lo, i_hi, launch_tag());
  CUDA_CHECK_LAUNCH();
}

// per task:  tbar += tgrad (optional);  abar[seg][step] = -<tbar_seg, g_seg> (fp64);  u = alpha[seg][step] * tbar
// grid (P / 2048, tasks): each CTA covers 2048 consecutive elements, which may straddle a few inner tensors.
__global__ void __launch_bounds__(256) dots_u_kernel(ParamLayout pl, float* __restrict__ tbar, const float* __restrict__ tgrad,
                                                     const float* __restrict__ g, float* __restrict__ u,
                                                     double* __restrict__ abar, const float* __restrict__ meta, int step,
                                                     long long task_stride, int tag) {
  pdl_prologue(17, tag);
  __shared__ double red[8];
  const int task = blockIdx.y;
  const long long lo = (long long)blockIdx.x * 2048, hi = min(pl.P, lo + 2048);
  const long long base = (long long)task * task_stride;
  for (int seg = 0; seg < pl.nseg_inner; ++seg) {
    const long long s0 = max(lo, pl.seg_off[seg]), s1 = min(hi, pl.seg_off[seg] + pl.seg_size[seg]);
    if (s0 >= s1) continue;                                  // CTA-uniform
    const float alpha = meta[pl.m_lslr + (long long)seg * (pl.S + 1) + step];
    double dot = 0.0;
    for (long long i = s0 + threadIdx.x; i < s1; i += 256) {
      float tb = tbar[base + i];
      if (tgrad) { tb += tgrad[base + i]; tbar[base + i] = tb; }
      dot += (double)tb * (double)g[base + i];
      u[base + i] = alpha * tb;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = dot;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int w = 0; w < 8; ++w) t += red[w];
      atomicAdd(&abar[((long long)task * pl.nseg_inner + seg) * MAML_MAX_STEPS + step], -t);
    }
  }
}

void launch_dots_u(const ParamLayout& pl, float* tbar, const float* tgrad, const float* g, float* u, double* abar,
                   const float* meta, int step, long long task_stride, int tasks, cudaStream_t st) {
  ProfScope prof_scope__(PROF_PARAM, 0.0, st);
  dim3 grid((unsigned)((pl.P + 2047) / 2048), tasks);
  launch_pdl(dots_u_kernel, dim3(grid), dim3(256), (size_t)(0), st, pl, tbar, tgrad, g, u, abar, meta, step, task_stride, launch_tag());
  CUDA_CHECK_LAUNCH();
}

// ---------------------------------------------------------------------------------------------
// export: result = [meta-gradient (reference layout) | loss | n_correct | running-mean parts | running-var parts]
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ const double* stat_ptr(const ExportArgs& a, int task, int kind, int step, int layer) {
  return a.stats + (long long)task * a.stats_task_stride + ((long long)kind * MAML_MAX_STEPS + step) * a.st_pass_stride +
         (long long)layer * a.st_layer_stride;
}

__device__ __forceinline__ void export_body(const ExportArgs& a, float* __restrict__ result);

// ---- peer-memory signalling (system scope: the flag lives in ANOTHER GPU's memory, reached over NVLink) ----
__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ float4 ld_relaxed_sys_v4(const float* p) {
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
// Called by every thread of a publishing kernel after its stores: the LAST block to arrive makes the whole slot visible
// system-wide and raises this rank's flag in every peer's memory.
__device__ __forceinline__ void comm_signal_when_last(const CommDev& c, unsigned seq) {
  __threadfence();                                        // this block's stores are in L2 (the point peers read from)
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned done = atomicAdd(&c.counters[0], 1u);
    if (done == gridDim.x * gridDim.y - 1) {
      __threadfence_system();
      c.counters[0] = 0;                                  // re-armed for the next launch
      for (int p = 0; p < c.world; ++p)
        if (p != c.rank) st_release_sys(c.peer_flags[p] + c.rank, seq);
    }
  }
}

// __grid_constant__: the argument block (~0.9 KB, indexed dynamically by layer / segment) is read in place from the
// constant bank.  By value -- and with the result pointer patched in the struct -- every thread first copied all of it to
// its local-memory stack: 808 B x 278 k threads = 159 MB of DRAM writes per launch.
__global__ void export_kernel(const __grid_constant__ ExportArgs a) {
  pdl_prologue(18, a.tag);
  unsigned seq = 0;
  float* result = a.result;
  if (a.comm.world > 1) {
    // multi-GPU: write straight into this round's communication slot (peers read it over NVLink) and signal
    seq = *(volatile unsigned*)a.comm.seq;
    result = a.comm.local_data + (long long)(seq & 1u) * a.comm.slot_stride;
  }
  export_body(a, result);
  if (a.comm.world > 1) comm_signal_when_last(a.comm, seq);
}

// Layout of the launch: blocks [0, ceil(P / 256)) = range 1, one THREAD per inner (fast-weight) element; the remaining
// blocks = range 2, one WARP per remaining entry of the result vector (BatchNorm beta / gamma, LSLR, loss, accuracy count,
// running-stat partial sums): the lanes share the (task, step) terms of the entry and a fixed shuffle tree adds them
// (fp64, deterministic).  Each of those entries is a sum of 8..80 scattered fp64 loads (+ a pow() per term for the
// running statistics); as a sequential per-thread loop they were the tail of the kernel.
__device__ __forceinline__ long long export_range1_blocks(const ParamLayout& pl) { return (pl.P + 255) / 256; }
__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void export_body(const ExportArgs& a, float* __restrict__ result) {
  const ParamLayout& pl = a.pl;
  const long long LSF = (long long)pl.L * pl.S * pl.F;
  const double invB = 1.0 / (double)a.tasks_global;
  const long long nb1 = export_range1_blocks(pl);
  // the tasks this block adds up: all of them, or (per-task mode) task blockIdx.y alone
  const int t0 = a.per_task ? (int)blockIdx.y : 0, nt = a.per_task ? 1 : a.tasks;
  if (a.per_task) result += (long long)t0 * a.result_stride;
  // ---- range 1: the inner (fast-weight) tensors, walked in the INTERNAL order so that the per-task reads are coalesced
  // (the reference layout is a transposition of it: [F][C][3][3] vs [tap][c][f]); one scattered 4-byte store per element
  if ((long long)blockIdx.x < nb1) {
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= pl.P) return;
    int seg;
    const long long mi = internal_to_meta(pl, gid, &seg);
    double val = 0.0;
    if (a.training)
      for (int t = t0; t < t0 + nt; ++t) val += (double)a.tbar[(long long)t * a.task_stride + gid];
    result[mi] = (float)(val * invB);
    return;
  }
  // ---- range 2: one warp per entry
  const int lane = threadIdx.x & 31;
  long long e = ((long long)blockIdx.x - nb1) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  // BatchNorm beta / gamma rows (per_step_gb: one per step).  Inner-loop beta / gamma are fast weights: range 1 exports them
  const long long bnsz = (long long)(pl.per_step_gb ? pl.S : 1) * pl.F;
  const long long E_bn = (pl.ln || pl.inner_bn) ? 0 : 2LL * pl.L * bnsz, E_lslr = (long long)pl.nseg_inner * (pl.S + 1), E_run = pl.per_step_bn ? 2 * LSF : 0;
  double val = 0.0, scale = invB;
  long long dst;
  if (e < E_bn) {
    // BatchNorm beta / gamma: target-pass gradient minus the Hessian-vector terms (second order)
    const int l = (int)(e / (2 * bnsz));
    const long long r = e - (long long)l * 2 * bnsz;
    const bool is_gamma = r >= bnsz;
    const long long rel = r - (is_gamma ? bnsz : 0);
    dst = (is_gamma ? pl.m_gamma[l] : pl.m_beta[l]) + rel;
    if (a.training) {
      const int f = (int)(rel % pl.F), s_sel = (int)(rel / pl.F), which = is_gamma ? 1 : 0;
      const int per = pl.per_step_gb ? 1 : a.num_steps;               // steps that feed this entry
      if (!pl.per_step_gb || s_sel < a.num_steps) {
        for (int k = lane; k < nt * per; k += 32) {
          const int tk = k / per, t = t0 + tk, s = pl.per_step_gb ? s_sel : k - tk * per;
          val += stat_ptr(a, t, PASS_TGT_BWD, s, l)[f * 2 + which];
          val -= stat_ptr(a, t, PASS_TAN_BWD, s, l)[f * 2 + which];
        }
      }
    }
  } else if ((e -= E_bn) < E_lslr) {
    const int seg = (int)(e / (pl.S + 1)), s = (int)(e % (pl.S + 1));
    dst = pl.m_lslr + e;
    if (a.training && s < a.num_steps)
      for (int t = t0 + lane; t < t0 + nt; t += 32) val += a.abar[((long long)t * pl.nseg_inner + seg) * MAML_MAX_STEPS + s];
  } else if ((e -= E_lslr) < 2) {
    dst = pl.meta_size + e;
    if (e == 0) {
      for (int k = lane; k < nt * a.num_steps; k += 32) {
        const int tk = k / a.num_steps, t = t0 + tk, s = k - tk * a.num_steps;
        if (a.target_mask & (1u << s)) val += (double)a.weights[s] * (double)a.losses[(long long)t * MAML_MAX_STEPS + s];
      }
    } else {
      for (int t = t0 + lane; t < t0 + nt; t += 32) val += (double)a.correct[t];
      scale = 1.0;
    }
  } else if ((e -= 2) < E_run) {
    // running-statistic partial sums (per-step BN only).  For block l, step s the reference applies, for
    // global task g = 0..B-1 in order: support update, then (if a target pass runs at s) target update;
    // r <- 0.9 r + 0.1 stat.  Unrolled: r_new = 0.9^U r_old + sum_k 0.1 * 0.9^(U-1-k) stat_k.
    dst = pl.meta_size + 2 + e;
    scale = 1.0;
    long long rel = e;
    const int which = (int)(rel / LSF);           // 0: mean, 1: var
    rel -= (long long)which * LSF;
    const int l = (int)(rel / ((long long)pl.S * pl.F));
    const int s = (int)((rel / pl.F) % pl.S);
    const int f = (int)(rel % pl.F);
    // evaluation passes leave the EMA side effect behind too (the reference's backup is an alias, see run_validation_iter)
    if (s < a.num_steps) {
      const bool has_t = (a.target_mask >> s) & 1u;
      const int c = has_t ? 2 : 1;
      const int U = c * a.tasks_global;
      for (int kk = lane; kk < nt * c; kk += 32) {
        const int tk = kk / c, t = t0 + tk, j = kk - tk * c;
        const int k = c * (a.task_offset + t) + j;
        const double wgt = 0.1 * pow(0.9, (double)(U - 1 - k));
        const double* sp = stat_ptr(a, t, j == 0 ? PASS_SUP_FWD : PASS_TGT_FWD, s, l);
        const double m = (double)(j == 0 ? a.n_s : a.n_t) * (double)a.hw[l];
        const double mean = sp[f * 2] / m;
        if (which == 0) val += wgt * mean;
        else {
          double var = sp[f * 2 + 1] / m - mean * mean;
          if (var < 0.0) var = 0.0;
          val += wgt * var * (m / (m > 1.0 ? m - 1.0 : 1.0));
        }
      }
    }
  } else if (pl.ln && (e -= E_run) < pl.lnb_off[pl.L]) {
    // layer-norm bias: target-pass gradients minus the Hessian-vector terms of every step (one step-independent tensor)
    int l = 0;
    while (e >= pl.lnb_off[l + 1]) ++l;
    dst = pl.m_lnb[l] + (e - pl.lnb_off[l]);
    if (a.training) {
      const long long row = pl.lnb_off[pl.L];
      for (int k = lane; k < nt * a.num_steps; k += 32) {
        const int tk = k / a.num_steps, t = t0 + tk, s = k - tk * a.num_steps;
        const float* r = a.lnb + ((long long)t * 2 * pl.S + s) * row + e;
        val += (double)r[0] - (double)r[(long long)pl.S * row];
      }
    }
  } else {
    return;                                        // warp-uniform
  }
  val = warp_sum_f64(val);
  if (lane == 0) result[dst] = (float)(val * scale);
}

void launch_export(const ExportArgs& a, cudaStream_t st) {
  ProfScope prof_scope__(PROF_PARAM, 0.0, st);
  const ParamLayout& pl = a.pl;
  const long long bnsz = (long long)(pl.per_step_gb ? pl.S : 1) * pl.F;
  const long long entries = (pl.ln ? pl.lnb_off[pl.L] : pl.inner_bn ? 0 : 2LL * pl.L * bnsz) + (long long)pl.nseg_inner * (pl.S + 1) + 2 +
                            (pl.per_step_bn ? 2LL * pl.L * pl.S * pl.F : 0);
  const long long blocks = (pl.P + 255) / 256 + (entries + 7) / 8;        // range 1: thread per element; range 2: warp per entry
  launch_pdl(export_kernel, dim3((unsigned)blocks, a.per_task ? (unsigned)a.tasks : 1u), dim3(256), (size_t)(0), st, tagged(a));
  CUDA_CHECK_LAUNCH();
}

// ---------------------------------------------------------------------------------------------
// The ONE collective of an iteration (replaces the reference's DataParallel gather, few_shot_learning_system.py:74-77):
// all-reduce(SUM) of the result vector as a kernel over peer memory.  Every block waits until all peers have raised
// their flag for this round (their slot is complete and visible), then each thread pulls one float4 from every rank's
// slot -- peer loads over NVLink / NVSwitch, all issued before the first add -- and sums them in rank order, so every
// rank computes bit-identical sums.  Two slots suffice: a rank rewrites slot k two rounds later, after its own reduce of
// the round in between, which needed every peer's flag for that round, which a peer raises only after ITS reduce of
// round k (stream order) -- i.e. after it finished reading the slot.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) allreduce_kernel(CommDev c, float* __restrict__ result, long long n, int tag) {
  const long long n4 = (n + 3) / 4;
  pdl_prologue(29, tag);
  const unsigned seq = *(volatile unsigned*)c.seq;
  if (threadIdx.x < c.world && threadIdx.x != c.rank) {
    const unsigned* f = c.local_flags + threadIdx.x;
    unsigned long long t0;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    unsigned spins = 0;
    while ((int)(ld_acquire_sys(f) - seq) < 0) {
      if ((++spins & 0x3ff) == 0) {
        unsigned long long t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (t1 - t0 > 30ull * 1000000000ull) {           // a peer never arrived: report instead of hanging the GPU
          atomicExch((unsigned long long*)c.status, (unsigned long long)seq | (1ull << 40) | ((unsigned long long)threadIdx.x << 32));
          break;
        }
      }
      __nanosleep(64);
    }
  }
  __syncthreads();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n4) {
    const long long off = (long long)(seq & 1u) * c.slot_stride + i * 4;
    float4 v[MAML_MAX_RANKS];
#pragma unroll
    for (int p = 0; p < MAML_MAX_RANKS; ++p)
      if (p < c.world) v[p] = ld_relaxed_sys_v4(c.peer_data[p] + off);
    float4 acc = v[0];
#pragma unroll
    for (int p = 1; p < MAML_MAX_RANKS; ++p)
      if (p < c.world) { acc.x += v[p].x; acc.y += v[p].y; acc.z += v[p].z; acc.w += v[p].w; }
    if (i * 4 + 4 <= n) *reinterpret_cast<float4*>(result + i * 4) = acc;
    else {                                                 // ragged tail (slots are padded to 4 floats, `result` is not)
      const float t[4] = {acc.x, acc.y, acc.z, acc.w};
      for (int k = 0; i * 4 + k < n; ++k) result[i * 4 + k] = t[k];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned done = atomicAdd(&c.counters[1], 1u);
    if (done == gridDim.x - 1) { c.counters[1] = 0; __threadfence(); *(volatile unsigned*)c.seq = seq + 1u; }
  }
}

void launch_allreduce(const CommDev& c, float* result, long long n, cudaStream_t st) {
  ProfScope prof_scope__(PROF_PARAM, 0.0, st);
  const long long n4 = (n + 3) / 4;
  launch_pdl(allreduce_kernel, dim3((unsigned)((n4 + 255) / 256)), dim3(256), (size_t)(0), st, c, result, n, launch_tag());
  CUDA_CHECK_LAUNCH();
}

__global__ void __launch_bounds__(256) publish_kernel(CommDev c, const float* __restrict__ src, long long n, int tag) {
  pdl_prologue(30, tag);
  const unsigned seq = *(volatile unsigned*)c.seq;
  float* dst = c.local_data + (long long)(seq & 1u) * c.slot_stride;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[i];
  comm_signal_when_last(c, seq);
}

void launch_publish(const CommDev& c, const float* src, long long n, cudaStream_t st) {
  ProfScope prof_scope__(PROF_PARAM, 0.0, st);
  launch_pdl(publish_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), (size_t)(0), st, c, src, n, launch_tag());
  CUDA_CHECK_LAUNCH();
}

// ---------------------------------------------------------------------------------------------
// fused clamp + Adam over the flat vectors
// ---------------------------------------------------------------------------------------------
struct SegEnds { long long e[32]; int n; };

__global__ void adam_kernel(float* __restrict__ meta, const float* __restrict__ grad, float* __restrict__ m,
                            float* __restrict__ v, long long n, float lr, float bc1, float bc2, SegEnds se,
                            unsigned trainable_mask, unsigned clamp_mask, int tag) {
  pdl_prologue(19, tag);
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int seg = 0;
  for (int k = 0; k < se.n; ++k)
    if (i >= se.e[k]) seg = k + 1;
  if (!((trainable_mask >> seg) & 1u)) return;
  float g = grad[i];
  if ((clamp_mask >> seg) & 1u) g = fminf(fmaxf(g, -10.f), 10.f);
  const float b1 = 0.9f, b2 = 0.999f, eps = 1e-8f;
  // torch.optim.Adam (single-tensor path): exp_avg.lerp_(grad, 1-beta1); exp_avg_sq.mul_(beta2).addcmul_(g, g, 1-beta2)
  const float mi = m[i] + (g - m[i]) * (1.f - b1);
  const float vi = v[i] * b2 + (1.f - b2) * g * g;
  m[i] = mi;
  v[i] = vi;
  const float denom = sqrtf(vi) / sqrtf(bc2) + eps;
  meta[i] = meta[i] - (lr / bc1) * (mi / denom);
}

void launch_adam(float* meta, const float* grad, float* m, float* v, long long n, float lr, float bc1, float bc2,
                 const long long* seg_end_host, int nseg, unsigned trainable_mask, unsigned clamp_mask, cudaStream_t st) {
  ProfScope prof_scope__(PROF_PARAM, 0.0, st);
  SegEnds se;
  se.n = nseg - 1;
  for (int k = 0; k < nseg - 1 && k < 32; ++k) se.e[k] = seg_end_host[k];
  launch_pdl(adam_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), (size_t)(0), st, meta, grad, m, v, n, lr, bc1, bc2, se, trainable_mask, clamp_mask, launch_tag());
  CUDA_CHECK_LAUNCH();
}

__global__ void running_update_kernel(const float* __restrict__ pm, const float* __restrict__ pv, float* __restrict__ rm,
                                      float* __restrict__ rv, const float* __restrict__ decay, int L, int S, int F, int tag) {
  pdl_prologue(20, tag);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L * S * F) return;
  const int s = (i / F) % S;
  const float d = decay[s];
  rm[i] = d * rm[i] + pm[i];
  rv[i] = d * rv[i] + pv[i];
}

void launch_running_update(const float* part_mean, const float* part_var, float* rm, float* rv, const float* decay_dev,
                           int L, int S, int F, cudaStream_t st) {
  ProfScope prof_scope__(PROF_PARAM, 0.0, st);
  const int n = L * S * F;
  launch_pdl(running_update_kernel, dim3((n + 255) / 256), dim3(256), (size_t)(0), st, part_mean, part_var, rm, rv, decay_dev, L, S, F, launch_tag());
  CUDA_CHECK_LAUNCH();
}

// Functional operator (VGGReLUNormNetwork.forward as a stand-alone call): the reference's F.batch_norm leaves
// running[step] <- 0.9 running[step] + 0.1 batch statistic behind for every block (meta_neural_network_architectures.py:
// 226-247), one update per forward call (= per task here, in task order).
struct HwArr { int v[MAML_MAX_LAYERS]; };
__global__ void running_ema_from_stats_kernel(const double* __restrict__ stats, long long task_stride, long long layer_stride, int tasks,
                                              float* __restrict__ rm, float* __restrict__ rv, int L, int S, int F, int step, HwArr hw, int n,
                                              int tag) {
  pdl_prologue(26, tag);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L * F) return;
  const int l = i / F, f = i - l * F;
  const double m = (double)n * (double)hw.v[l];
  float* pm = rm + ((long long)l * S + step) * F + f;
  float* pv = rv + ((long long)l * S + step) * F + f;
  float a = *pm, b = *pv;
  for (int t = 0; t < tasks; ++t) {
    const double* sp = stats + (long long)t * task_stride + (long long)l * layer_stride;
    const double mean = sp[f * 2] / m;
    double var = sp[f * 2 + 1] / m - mean * mean;
    if (var < 0.0) var = 0.0;
    const double unbiased = var * (m / (m > 1.0 ? m - 1.0 : 1.0));
    a = 0.9f * a + 0.1f * (float)mean;          // fp32 like the reference's running buffers
    b = 0.9f * b + 0.1f * (float)unbiased;
  }
  *pm = a; *pv = b;
}

void launch_running_ema_from_stats(const double* stats, long long stats_task_stride, long long layer_stride, int tasks, float* rm,
                                   float* rv, int L, int S, int F, int step, const int* hw_host, int n, cudaStream_t st) {
  ProfScope prof_scope__(PROF_PARAM, 0.0, st);
  HwArr hw{};
  for (int l = 0; l < L; ++l) hw.v[l] = hw_host[l];
  launch_pdl(running_ema_from_stats_kernel, dim3((L * F + 127) / 128), dim3(128), (size_t)(0), st, stats, stats_task_stride, layer_stride,
             tasks, rm, rv, L, S, F, step, hw, n, launch_tag());
  CUDA_CHECK_LAUNCH();
}

// ---------------------------------------------------------------------------------------------
// GPU-resident episode assembly (replaces the reference's 4-worker PIL / NumPy loader for in-memory datasets,
// data.py:478-524): gather the sampled images of every task from the device-resident dataset [image][H][W][C],
// apply the class's rot90 (Omniglot train augmentation, data.py:17-34 -- np.rot90, counter-clockwise) or the
// ImageNet normalisation (data.py:100-106: ToTensor then (x - mean) / std), write NCHW support / target tensors and
// the class-major labels.  One thread per output pixel.
// ---------------------------------------------------------------------------------------------
struct EpisodeArgs {
  const float* dataset; const long long* image_index; const int* rot_k;
  int B, N, K, T, C, H, W;
  float mean[4], stdv[4]; int normalise;
  float* xs; float* xt; long long* ys; long long* yt;
};
__global__ void episode_gather_kernel(EpisodeArgs a, int tag) {
  pdl_prologue(28, tag);
  const long long per_img = (long long)a.C * a.H * a.W;
  const long long total = (long long)a.B * a.N * (a.K + a.T) * per_img;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int x = (int)(i % a.W), y = (int)((i / a.W) % a.H), c = (int)((i / ((long long)a.W * a.H)) % a.C);
  const long long img = i / per_img;                                   // (b, n, j) flattened, j over K + T
  const int j = (int)(img % (a.K + a.T)), n = (int)((img / (a.K + a.T)) % a.N), b = (int)(img / ((long long)(a.K + a.T) * a.N));
  const int k = a.rot_k[b * a.N + n] & 3;
  int sy = y, sx = x;                                                  // np.rot90(m, k): out[y][x] = in[sy][sx]
  if (k == 1) { sy = x; sx = a.W - 1 - y; }
  else if (k == 2) { sy = a.H - 1 - y; sx = a.W - 1 - x; }
  else if (k == 3) { sy = a.H - 1 - x; sx = y; }
  const long long src = a.image_index[img];
  float v = a.dataset[((src * a.H + sy) * a.W + sx) * a.C + c];
  if (a.normalise) v = __fdiv_rn(__fsub_rn(v, a.mean[c]), a.stdv[c]);
  if (j < a.K) {
    a.xs[((((long long)b * a.N + n) * a.K + j) * a.C + c) * a.H * a.W + (long long)y * a.W + x] = v;
    if (c == 0 && y == 0 && x == 0) a.ys[((long long)b * a.N + n) * a.K + j] = n;
  } else {
    const int jt = j - a.K;
    a.xt[((((long long)b * a.N + n) * a.T + jt) * a.C + c) * a.H * a.W + (long long)y * a.W + x] = v;
    if (c == 0 && y == 0 && x == 0) a.yt[((long long)b * a.N + n) * a.T + jt] = n;
  }
}

void launch_episode_gather(const float* dataset, const long long* image_index, const int* rot_k, int B, int N, int K, int T, int C,
                           int H, int W, const float* mean, const float* stdv, float* xs, float* xt, long long* ys, long long* yt,
                           cudaStream_t st) {
  EpisodeArgs a{};
  a.dataset = dataset; a.image_index = image_index; a.rot_k = rot_k;
  a.B = B; a.N = N; a.K = K; a.T = T; a.C = C; a.H = H; a.W = W;
  a.normalise = (mean && stdv) ? 1 : 0;
  for (int c = 0; c < 4; ++c) { a.mean[c] = (a.normalise && c < C) ? mean[c] : 0.f; a.stdv[c] = (a.normalise && c < C) ? stdv[c] : 1.f; }
  a.xs = xs; a.xt = xt; a.ys = ys; a.yt = yt;
  const long long total = (long long)B * N * (K + T) * C * H * W;
  launch_pdl(episode_gather_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), (size_t)(0), st, a, launch_tag());
  CUDA_CHECK_LAUNCH();
}

MAML_TRACE_SETTER(trace_set_param)
