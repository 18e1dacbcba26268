// BatchNorm(batch statistics) + leaky-ReLU(0.01) + 2x2 max-pool: forward, backward and the
// forward-mode tangents of both (Hessian-vector pass), on the padded pixel-grid layout.
//
// Restates reference meta_neural_network_architectures.py:246-247 (F.batch_norm, training=True
// always), :426 (F.leaky_relu), :651-652 (F.max_pool2d k=2,s=2, floor, first max wins) and their
// derivatives; equations are SURVEY.md appendix A1-A3 (validated against the reference).
//
// Work item = (pooling window, channel quad).  A window is the 2x2 block (2wy+dy, 2wx+dx);
// windows on the odd last row/column are "partial": they produce no pooled value and receive no
// pooled gradient, but their positions still take part in BatchNorm.
#include "common.cuh"
#include "head_body.cuh"

struct Chan4 { float4 mu, r, g, b; };

__device__ __forceinline__ float leaky(float y) { return y > 0.f ? y : LEAKY_SLOPE_F * y; }
__device__ __forceinline__ float slope_of(float y) { return y > 0.f ? 1.f : LEAKY_SLOPE_F; }

// per-channel constants from the fp64 sums (sum z, sum z^2)
__device__ __forceinline__ void chan_setup(const double* __restrict__ st, const float* __restrict__ gamma,
                                           const float* __restrict__ beta, double m, int F, float* s_mu, float* s_r,
                                           float* s_g, float* s_b) {
  const int tid = threadIdx.x;
  if (tid < F) {
    const double mean = st[tid * 2 + 0] / m;
    double var = st[tid * 2 + 1] / m - mean * mean;
    if (var < 0.0) var = 0.0;
    s_mu[tid] = (float)mean;
    s_r[tid] = (float)(1.0 / sqrt(var + BN_EPS_D));
    s_g[tid] = gamma[tid];
    s_b[tid] = beta[tid];
  }
}

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
// TF32 operand split for the tensor-core kernels: x ~= hi + lo, hi = rna_tf32(x), lo = rna_tf32(x - hi)
__device__ __forceinline__ float tf32_rna_bn(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
__device__ __forceinline__ void st4_split(float* hi, float* lo, long long idx, float4 v) {
  float4 h, l;
  h.x = tf32_rna_bn(v.x); h.y = tf32_rna_bn(v.y); h.z = tf32_rna_bn(v.z); h.w = tf32_rna_bn(v.w);
  l.x = tf32_rna_bn(v.x - h.x); l.y = tf32_rna_bn(v.y - h.y); l.z = tf32_rna_bn(v.z - h.z); l.w = tf32_rna_bn(v.w - h.w);
  st4(hi + idx, h);
  st4(lo + idx, l);
}
__device__ __forceinline__ float4 ld4s(const float* s, int q) { return make_float4(s[q * 4], s[q * 4 + 1], s[q * 4 + 2], s[q * 4 + 3]); }

#define F4_OP(out, expr) { out.x = expr(x); out.y = expr(y); out.z = expr(z); out.w = expr(w); }

struct WinIter {
  int hc, wc, NW, F4, WPB, q, lane;
  __device__ WinIter(const BnGeom& g) {
    hc = (g.h + 1) >> 1; wc = (g.w + 1) >> 1; NW = g.n * hc * wc; F4 = g.F >> 2;
    WPB = blockDim.x / F4; q = threadIdx.x % F4; lane = threadIdx.x / F4;
  }
  // work item wi -> image, window row, window column
  __device__ __forceinline__ void window(int wi, int& img, int& wy, int& wx) const {
    img = wi / (hc * wc);
    const int rem = wi - img * hc * wc;
    wy = rem / wc; wx = rem - wy * wc;
  }
  // offset of this thread's channel quad at pixel (yy, xx) of image img on the block's padded grid
  __device__ __forceinline__ long long grid(const BnGeom& g, int img, int yy, int xx) const {
    return ((long long)img * g.G + (yy + 1) * g.gw + (xx + 1)) * g.F + q * 4;
  }
  // offset of this thread's channel quad at window (wy, wx) of image img on the grid of the pooled output
  __device__ __forceinline__ long long pooled(const BnGeom& g, int img, int wy, int wx) const {
    return ((long long)img * g.pG + (wy + g.pb) * g.pgw + (wx + g.pb)) * g.F + q * 4;
  }
};

// ------------------------------------------------------------------------------- forward
__device__ __forceinline__ void bnact_phase(const BnActArgs& a, const BnGeom& g, int task, int cta, int ncta, const WinIter& it,
                                            const float* s_mu, const float* s_r, const float* s_g, const float* s_b) {
  if (it.lane >= it.WPB) return;
  const float4 mu = ld4s(s_mu, it.q), r = ld4s(s_r, it.q), ga = ld4s(s_g, it.q), be = ld4s(s_b, it.q);
  float* z = a.z + (long long)task * a.z_stride;
  float* p = a.p + (long long)task * a.p_stride;
  for (int wi = cta * it.WPB + it.lane; wi < it.NW; wi += ncta * it.WPB) {
    int img, wy, wx; it.window(wi, img, wy, wx);
    float4 best = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
      if (yy < g.h && xx < g.w) {
        const long long idx = it.grid(g, img, yy, xx);
        const float4 zv = ld4(z + idx);
        float4 zh, act;
        zh.x = (zv.x - mu.x) * r.x; zh.y = (zv.y - mu.y) * r.y; zh.z = (zv.z - mu.z) * r.z; zh.w = (zv.w - mu.w) * r.w;
        st4(z + idx, zh);
        act.x = leaky(fmaf(ga.x, zh.x, be.x)); act.y = leaky(fmaf(ga.y, zh.y, be.y));
        act.z = leaky(fmaf(ga.z, zh.z, be.z)); act.w = leaky(fmaf(ga.w, zh.w, be.w));
        if (k == 0) best = act;
        else {
          if (act.x > best.x) best.x = act.x;
          if (act.y > best.y) best.y = act.y;
          if (act.z > best.z) best.z = act.z;
          if (act.w > best.w) best.w = act.w;
        }
      }
    }
    if (wy < g.ph && wx < g.pw) {
      const long long pidx = it.pooled(g, img, wy, wx);
      st4(p + pidx, best);
      if (a.p_hi) st4_split(a.p_hi + (long long)task * a.p_stride, a.p_lo + (long long)task * a.p_stride, pidx, best);
    }
  }
}

__global__ void __launch_bounds__(256) bnact_kernel(BnActArgs a) {
  pdl_prologue(6, a.tag);
  __shared__ float s_mu[64], s_r[64], s_g[64], s_b[64];
  const BnGeom g = a.g;
  const int task = blockIdx.y;
  chan_setup(a.stats + (long long)task * a.stats_stride, a.gamma, a.beta, (double)g.n * g.h * g.w, g.F, s_mu, s_r, s_g, s_b);
  __syncthreads();
  WinIter it(g);
  bnact_phase(a, g, task, blockIdx.x, gridDim.x, it, s_mu, s_r, s_g, s_b);
}

// Host side of WinIter: the pooling windows of one task (NW) and the windows a 256-thread CTA works on at once (wpb, one
// thread per channel quad)
struct WinGeom { int NW, wpb; };
static inline WinGeom win_geom(const BnGeom& g) {
  return WinGeom{g.n * ((g.h + 1) / 2) * ((g.w + 1) / 2), 256 / (g.F / 4)};
}

static inline dim3 bn_grid(const BnGeom& g, int tasks, int* block) {
  const WinGeom wg = win_geom(g);
  *block = wg.wpb * (g.F / 4);
  int bx = (wg.NW + wg.wpb - 1) / wg.wpb;
  if (bx > 4 * num_sms()) bx = 4 * num_sms();
  if (bx < 1) bx = 1;
  return dim3(bx, tasks);
}

void launch_bnact(const BnActArgs& a, cudaStream_t st) {
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  int block; dim3 grid = bn_grid(a.g, a.tasks, &block);
  launch_pdl(bnact_kernel, dim3(grid), dim3(block), (size_t)(0), st, tagged(a));
  CUDA_CHECK_LAUNCH();
}

// value of one window position: loads zh, recomputes y; used by all backward-type kernels
struct WinPos { float4 zh; float4 y; bool ok; long long idx; };

__device__ __forceinline__ void argmax_window(const float* __restrict__ zhp, const BnGeom& g, int img, int wy, int wx,
                                              const WinIter& it, const float4& ga, const float4& be, float4 (&zh)[4],
                                              long long (&idx)[4], int4& arg, float4& slope_at) {
  float4 best = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 ybest = best;
  arg = make_int4(0, 0, 0, 0);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
    idx[k] = it.grid(g, img, yy, xx);
    zh[k] = ld4(zhp + idx[k]);
    float4 y, act;
    y.x = fmaf(ga.x, zh[k].x, be.x); y.y = fmaf(ga.y, zh[k].y, be.y);
    y.z = fmaf(ga.z, zh[k].z, be.z); y.w = fmaf(ga.w, zh[k].w, be.w);
    act.x = leaky(y.x); act.y = leaky(y.y); act.z = leaky(y.z); act.w = leaky(y.w);
    if (k == 0) { best = act; ybest = y; }
    else {
      if (act.x > best.x) { best.x = act.x; ybest.x = y.x; arg.x = k; }
      if (act.y > best.y) { best.y = act.y; ybest.y = y.y; arg.y = k; }
      if (act.z > best.z) { best.z = act.z; ybest.z = y.z; arg.z = k; }
      if (act.w > best.w) { best.w = act.w; ybest.w = y.w; arg.w = k; }
    }
  }
  slope_at.x = slope_of(ybest.x); slope_at.y = slope_of(ybest.y); slope_at.z = slope_of(ybest.z); slope_at.w = slope_of(ybest.w);
}

// component `comp` (a literal at every call site) of v[k], k = the run-time arg-max position: a select chain -- indexing
// the register array with k would move it to local memory (STL / LDL in the middle of latency-bound kernels)
__device__ __forceinline__ float pick(const float4 (&v)[4], int k, int comp) {
  const float a0 = comp == 0 ? v[0].x : comp == 1 ? v[0].y : comp == 2 ? v[0].z : v[0].w;
  const float a1 = comp == 0 ? v[1].x : comp == 1 ? v[1].y : comp == 2 ? v[1].z : v[1].w;
  const float a2 = comp == 0 ? v[2].x : comp == 1 ? v[2].y : comp == 2 ? v[2].z : v[2].w;
  const float a3 = comp == 0 ? v[3].x : comp == 1 ? v[3].y : comp == 2 ? v[3].z : v[3].w;
  return k == 0 ? a0 : k == 1 ? a1 : k == 2 ? a2 : a3;
}

// block-level reduction of per-thread (4 channels x 2 sums) fp64 partials, then one atomic per channel
__device__ __forceinline__ void block_reduce_stats(double (&s1)[4], double (&s2)[4], const WinIter& it, double* stats, int F) {
  __shared__ double red[256 * 8];
  const int tid = threadIdx.x;
#pragma unroll
  for (int c = 0; c < 4; ++c) { red[tid * 8 + c * 2] = s1[c]; red[tid * 8 + c * 2 + 1] = s2[c]; }
  __syncthreads();
  for (int o = tid; o < F * 2; o += blockDim.x) {
    const int ch = o >> 1, which = o & 1;
    const int q = ch >> 2, comp = ch & 3;
    double t = 0.0;
    for (int l = 0; l < it.WPB; ++l) t += red[(l * it.F4 + q) * 8 + comp * 2 + which];
    atomicAdd(&stats[ch * 2 + which], t);
  }
}

// ---- thread-block-cluster helpers for the fused (reduce -> cluster all-reduce -> apply) backward kernels
__device__ __forceinline__ void bn_cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void bn_cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t bn_cluster_rank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t bn_cluster_size() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void bn_dsmem_st_f64(double* local, uint32_t rank, double v) {
  const uint32_t la = (uint32_t)__cvta_generic_to_shared(local);
  uint32_t ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(la), "r"(rank));
  asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(ra), "d"(v) : "memory");
}
// CTA totals of the per-thread partials (fixed summation order): thread o < 2F returns the total of (channel o/2,
// sum o%2); other threads return 0
__device__ __forceinline__ double block_reduce_totals(double (&s1)[4], double (&s2)[4], const WinIter& it, int F) {
  __shared__ double red2[256 * 8];
  const int tid = threadIdx.x;
#pragma unroll
  for (int c = 0; c < 4; ++c) { red2[tid * 8 + c * 2] = s1[c]; red2[tid * 8 + c * 2 + 1] = s2[c]; }
  __syncthreads();
  double t = 0.0;
  if (tid < F * 2) {
    const int ch = tid >> 1, which = tid & 1;
    const int q = ch >> 2, comp = ch & 3;
    for (int l = 0; l < it.WPB; ++l) t += red2[(l * it.F4 + q) * 8 + comp * 2 + which];
  }
  return t;
}
// All-reduce of the CTA totals over the cluster with ONE barrier: every CTA pushes its totals into slot [own rank] of
// every CTA's `gather` array (remote shared-memory stores), barrier.cluster (release / acquire), then each CTA sums its
// local copy in rank order (deterministic).  Nobody touches remote shared memory after the barrier, so CTAs may exit
// independently.  Publishes sums / m in shared memory and (rank 0) the raw sums in the global statistics arena.
__device__ __forceinline__ void cluster_allreduce_stats(double t, double (*gather)[128], int F, double m, float* s_a, float* s_b2,
                                                        double* gstats) {
  const uint32_t n = bn_cluster_size(), me = bn_cluster_rank();
  const int tid = threadIdx.x;
  // completes the barrier phase opened by bn_cluster_arrive() at kernel start: every CTA of the cluster is running,
  // so its shared memory may be written remotely
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
  if (tid < F * 2)
    for (uint32_t z = 0; z < n; ++z) bn_dsmem_st_f64(&gather[me][tid], z, t);
  __syncwarp();
  bn_cluster_sync();
  if (tid < F * 2) {
    double tt = 0.0;
    for (uint32_t z = 0; z < n; ++z) tt += gather[z][tid];
    ((tid & 1) ? s_b2 : s_a)[tid >> 1] = (float)(tt / m);
    if (me == 0) gstats[tid] = tt;
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------- backward: reduce
__device__ __forceinline__ void bnbwd_reduce_phase(const BnBwdArgs& a, const BnGeom& g, int task, int cta, int ncta, const WinIter& it,
                                                   const float* s_g, const float* s_b, double (&s1)[4], double (&s2)[4]) {
  if (it.lane >= it.WPB) return;
  const float4 ga = ld4s(s_g, it.q), be = ld4s(s_b, it.q);
  const float* zhp = a.zh + (long long)task * a.zh_stride;
  const float* dp = a.dp + (long long)task * a.dp_stride;
  for (int wi = cta * it.WPB + it.lane; wi < it.NW; wi += ncta * it.WPB) {
    int img, wy, wx; it.window(wi, img, wy, wx);
    if (wy >= g.ph || wx >= g.pw) continue;
    float4 zh[4]; long long idx[4]; int4 arg; float4 sl;
    argmax_window(zhp, g, img, wy, wx, it, ga, be, zh, idx, arg, sl);
    const float4 d = ld4(dp + it.pooled(g, img, wy, wx));
    const float dy0 = d.x * sl.x, dy1 = d.y * sl.y, dy2 = d.z * sl.z, dy3 = d.w * sl.w;
    s1[0] += dy0; s2[0] += (double)dy0 * (double)pick(zh, arg.x, 0);
    s1[1] += dy1; s2[1] += (double)dy1 * (double)pick(zh, arg.y, 1);
    s1[2] += dy2; s2[2] += (double)dy2 * (double)pick(zh, arg.z, 2);
    s1[3] += dy3; s2[3] += (double)dy3 * (double)pick(zh, arg.w, 3);
  }
}

__global__ void __launch_bounds__(256) bnbwd_reduce_kernel(BnBwdArgs a) {
  pdl_prologue(7, a.tag);
  __shared__ float s_g[64], s_b[64];
  const BnGeom g = a.g;
  const int task = blockIdx.y;
  if (threadIdx.x < g.F) { s_g[threadIdx.x] = a.gamma[threadIdx.x]; s_b[threadIdx.x] = a.beta[threadIdx.x]; }
  __syncthreads();
  WinIter it(g);
  double s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  bnbwd_reduce_phase(a, g, task, blockIdx.x, gridDim.x, it, s_g, s_b, s1, s2);
  block_reduce_stats(s1, s2, it, a.stats_bwd + (long long)task * a.stats_bwd_stride, g.F);
}

void launch_bnbwd_reduce(const BnBwdArgs& a, cudaStream_t st) {
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  int block; dim3 grid = bn_grid(a.g, a.tasks, &block);
  if ((int)grid.x > num_sms()) grid.x = num_sms();
  launch_pdl(bnbwd_reduce_kernel, dim3(grid), dim3(block), (size_t)(0), st, tagged(a));
  CUDA_CHECK_LAUNCH();
}

// ------------------------------------------------------------------------------- backward: apply
// dz = r * gamma * (dy - S1/m - zh * S2/m)   at every valid position (dy != 0 only at the arg-max)
__device__ __forceinline__ void bnbwd_apply_phase(const BnBwdArgs& a, const BnGeom& g, int task, int cta, int ncta, const WinIter& it,
                                                  const float* s_r, const float* s_g, const float* s_b, const float* s_c1,
                                                  const float* s_c2) {
  if (it.lane >= it.WPB) return;
  const float4 r = ld4s(s_r, it.q), ga = ld4s(s_g, it.q), be = ld4s(s_b, it.q), c1 = ld4s(s_c1, it.q), c2 = ld4s(s_c2, it.q);
  const float4 rg = make_float4(r.x * ga.x, r.y * ga.y, r.z * ga.z, r.w * ga.w);
  const float* zhp = a.zh + (long long)task * a.zh_stride;
  const float* dp = a.dp + (long long)task * a.dp_stride;
  float* dz = a.dz + (long long)task * a.dz_stride;
  for (int wi = cta * it.WPB + it.lane; wi < it.NW; wi += ncta * it.WPB) {
    int img, wy, wx; it.window(wi, img, wy, wx);
    const bool full = (wy < g.ph && wx < g.pw);
    if (full) {
      float4 zh[4]; long long idx[4]; int4 arg; float4 sl;
      argmax_window(zhp, g, img, wy, wx, it, ga, be, zh, idx, arg, sl);
      const float4 d = ld4(dp + it.pooled(g, img, wy, wx));
      const float4 dyv = make_float4(d.x * sl.x, d.y * sl.y, d.z * sl.z, d.w * sl.w);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float4 o;
        o.x = rg.x * ((arg.x == k ? dyv.x : 0.f) - c1.x - zh[k].x * c2.x);
        o.y = rg.y * ((arg.y == k ? dyv.y : 0.f) - c1.y - zh[k].y * c2.y);
        o.z = rg.z * ((arg.z == k ? dyv.z : 0.f) - c1.z - zh[k].z * c2.z);
        o.w = rg.w * ((arg.w == k ? dyv.w : 0.f) - c1.w - zh[k].w * c2.w);
        st4(dz + idx[k], o);
        if (a.dz_hi) st4_split(a.dz_hi + (long long)task * a.dz_stride, a.dz_lo + (long long)task * a.dz_stride, idx[k], o);
      }
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
        if (yy < g.h && xx < g.w) {
          const long long idx = it.grid(g, img, yy, xx);
          const float4 zh = ld4(zhp + idx);
          float4 o;
          o.x = rg.x * (-c1.x - zh.x * c2.x); o.y = rg.y * (-c1.y - zh.y * c2.y);
          o.z = rg.z * (-c1.z - zh.z * c2.z); o.w = rg.w * (-c1.w - zh.w * c2.w);
          st4(dz + idx, o);
          if (a.dz_hi) st4_split(a.dz_hi + (long long)task * a.dz_stride, a.dz_lo + (long long)task * a.dz_stride, idx, o);
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256) bnbwd_apply_kernel(BnBwdArgs a) {
  pdl_prologue(8, a.tag);
  __shared__ float s_mu[64], s_r[64], s_g[64], s_b[64], s_c1[64], s_c2[64];
  const BnGeom g = a.g;
  const int task = blockIdx.y;
  const double m = (double)g.n * g.h * g.w;
  chan_setup(a.stats_fwd + (long long)task * a.stats_fwd_stride, a.gamma, a.beta, m, g.F, s_mu, s_r, s_g, s_b);
  if (threadIdx.x < g.F) {
    const double* sb = a.stats_bwd + (long long)task * a.stats_bwd_stride;
    s_c1[threadIdx.x] = (float)(sb[threadIdx.x * 2] / m);
    s_c2[threadIdx.x] = (float)(sb[threadIdx.x * 2 + 1] / m);
  }
  __syncthreads();
  WinIter it(g);
  bnbwd_apply_phase(a, g, task, blockIdx.x, gridDim.x, it, s_r, s_g, s_b, s_c1, s_c2);
}

// fused: one cluster of CTAs per task does reduce -> all-reduce through distributed shared memory -> apply
__global__ void __launch_bounds__(256) bnbwd_fused_kernel(BnBwdArgs a) {
  pdl_prologue(9, a.tag);
  bn_cluster_arrive();
  __shared__ float s_mu[64], s_r[64], s_g[64], s_b[64], s_c1[64], s_c2[64];
  __shared__ double gather[8][128];
  const BnGeom g = a.g;
  const int task = blockIdx.y;
  const double m = (double)g.n * g.h * g.w;
  chan_setup(a.stats_fwd + (long long)task * a.stats_fwd_stride, a.gamma, a.beta, m, g.F, s_mu, s_r, s_g, s_b);
  __syncthreads();
  WinIter it(g);
  double s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  bnbwd_reduce_phase(a, g, task, blockIdx.x, gridDim.x, it, s_g, s_b, s1, s2);
  const double tot = block_reduce_totals(s1, s2, it, g.F);
  cluster_allreduce_stats(tot, gather, g.F, m, s_c1, s_c2, a.stats_bwd + (long long)task * a.stats_bwd_stride);
  bnbwd_apply_phase(a, g, task, blockIdx.x, gridDim.x, it, s_r, s_g, s_b, s_c1, s_c2);
}

// cluster size for the fused kernels: enough CTAs for <= 4 windows per thread, else 0 (two-kernel path: the block needs
// more than 32 CTAs at one window per thread, or the handle's BN_FUSE option is off)
static inline int bn_fused_cluster(const BnGeom& g) {
  if (!launch_ctx().opt->bn_fuse) return 0;
  const WinGeom wg = win_geom(g);
  const int need = (wg.NW + wg.wpb - 1) / wg.wpb;
  if (need > 32) return 0;
  int cl = 1;
  while (cl < need && cl < 8) cl <<= 1;
  return cl;
}
template <class A>
static inline void launch_cluster(void (*kernel)(A), const A& a, int cl, int tasks, int block, cudaStream_t st) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(cl, tasks); cfg.blockDim = dim3(block); cfg.dynamicSmemBytes = 0; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cl; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kernel, a);
}

// BatchNorm backward of one block (reduce + apply), fused into one cluster kernel when the block is small
void launch_bnbwd(const BnBwdArgs& a, cudaStream_t st) {
  const int cl = bn_fused_cluster(a.g);
  if (cl == 0) { launch_bnbwd_reduce(a, st); launch_bnbwd_apply(a, st); return; }
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  int block; bn_grid(a.g, a.tasks, &block);
  launch_cluster(bnbwd_fused_kernel, tagged(a), cl, a.tasks, block, st);
  CUDA_CHECK_LAUNCH();
}

void launch_bnbwd_apply(const BnBwdArgs& a, cudaStream_t st) {
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  int block; dim3 grid = bn_grid(a.g, a.tasks, &block);
  launch_pdl(bnbwd_apply_kernel, dim3(grid), dim3(block), (size_t)(0), st, tagged(a));
  CUDA_CHECK_LAUNCH();
}

// ------------------------------------------------------------------------------- tangent forward
// zhdot = r * (zdot - mean(zdot) - zh * mean(zh * zdot));  pdot = slope * gamma * zhdot at the arg-max
__device__ __forceinline__ void bnact_tan_setup(const BnActTanArgs& a, const BnGeom& g, int task, double m, float* s_mu, float* s_r,
                                                float* s_g, float* s_b, float* s_md, float* s_q) {
  chan_setup(a.stats_fwd + (long long)task * a.stats_fwd_stride, a.gamma, a.beta, m, g.F, s_mu, s_r, s_g, s_b);
  if (threadIdx.x < g.F) {
    const double* stt = a.stats_tan + (long long)task * a.stats_tan_stride;
    s_md[threadIdx.x] = (float)(stt[threadIdx.x * 2] / m);
    s_q[threadIdx.x] = (float)(stt[threadIdx.x * 2 + 1] / m);
  }
}

// GB: gamma / beta carry tangents (s_gd, s_bd): pdot = slope * (gamma zhdot + gdot zh + bdot) at the arg-max
template <bool GB = false>
__device__ __forceinline__ void bnact_tan_phase(const BnActTanArgs& a, const BnGeom& g, int task, int cta, int ncta, const WinIter& it,
                                                const float* s_r, const float* s_g, const float* s_b, const float* s_md,
                                                const float* s_q, const float* s_gd = nullptr, const float* s_bd = nullptr) {
  if (it.lane >= it.WPB) return;
  const float4 r = ld4s(s_r, it.q), ga = ld4s(s_g, it.q), be = ld4s(s_b, it.q), md = ld4s(s_md, it.q), qq = ld4s(s_q, it.q);
  float4 gd = make_float4(0.f, 0.f, 0.f, 0.f), bd = gd;
  if constexpr (GB) { gd = ld4s(s_gd, it.q); bd = ld4s(s_bd, it.q); }
  float* zd = a.zdot + (long long)task * a.zdot_stride;
  const float* zd2 = a.zdot2 ? a.zdot2 + (long long)task * a.zdot_stride : nullptr;
  const float* zhp = a.zh + (long long)task * a.zh_stride;
  float* pd = a.pdot + (long long)task * a.pdot_stride;
  for (int wi = cta * it.WPB + it.lane; wi < it.NW; wi += ncta * it.WPB) {
    int img, wy, wx; it.window(wi, img, wy, wx);
    float4 best = make_float4(0.f, 0.f, 0.f, 0.f), pbest = best;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
      if (yy < g.h && xx < g.w) {
        const long long idx = it.grid(g, img, yy, xx);
        const float4 zh = ld4(zhp + idx);
        float4 zv = ld4(zd + idx);
        if (zd2) { const float4 z2 = ld4(zd2 + idx); zv.x += z2.x; zv.y += z2.y; zv.z += z2.z; zv.w += z2.w; }
        float4 zhd;
        zhd.x = r.x * (zv.x - md.x - zh.x * qq.x); zhd.y = r.y * (zv.y - md.y - zh.y * qq.y);
        zhd.z = r.z * (zv.z - md.z - zh.z * qq.z); zhd.w = r.w * (zv.w - md.w - zh.w * qq.w);
        st4(zd + idx, zhd);
        float4 y, act, pdv;
        y.x = fmaf(ga.x, zh.x, be.x); y.y = fmaf(ga.y, zh.y, be.y); y.z = fmaf(ga.z, zh.z, be.z); y.w = fmaf(ga.w, zh.w, be.w);
        act.x = leaky(y.x); act.y = leaky(y.y); act.z = leaky(y.z); act.w = leaky(y.w);
        if constexpr (GB) {
          pdv.x = slope_of(y.x) * (ga.x * zhd.x + fmaf(gd.x, zh.x, bd.x)); pdv.y = slope_of(y.y) * (ga.y * zhd.y + fmaf(gd.y, zh.y, bd.y));
          pdv.z = slope_of(y.z) * (ga.z * zhd.z + fmaf(gd.z, zh.z, bd.z)); pdv.w = slope_of(y.w) * (ga.w * zhd.w + fmaf(gd.w, zh.w, bd.w));
        } else {
          pdv.x = slope_of(y.x) * ga.x * zhd.x; pdv.y = slope_of(y.y) * ga.y * zhd.y;
          pdv.z = slope_of(y.z) * ga.z * zhd.z; pdv.w = slope_of(y.w) * ga.w * zhd.w;
        }
        if (k == 0) { best = act; pbest = pdv; }
        else {
          if (act.x > best.x) { best.x = act.x; pbest.x = pdv.x; }
          if (act.y > best.y) { best.y = act.y; pbest.y = pdv.y; }
          if (act.z > best.z) { best.z = act.z; pbest.z = pdv.z; }
          if (act.w > best.w) { best.w = act.w; pbest.w = pdv.w; }
        }
      }
    }
    if (wy < g.ph && wx < g.pw) {
      const long long pidx = it.pooled(g, img, wy, wx);
      st4(pd + pidx, pbest);
      if (a.pdot_hi) st4_split(a.pdot_hi + (long long)task * a.pdot_stride, a.pdot_lo + (long long)task * a.pdot_stride, pidx, pbest);
    }
  }
}

__global__ void __launch_bounds__(256) bnact_tan_kernel(BnActTanArgs a) {
  pdl_prologue(10, a.tag);
  __shared__ float s_mu[64], s_r[64], s_g[64], s_b[64], s_md[64], s_q[64];
  const BnGeom g = a.g;
  const int task = blockIdx.y;
  bnact_tan_setup(a, g, task, (double)g.n * g.h * g.w, s_mu, s_r, s_g, s_b, s_md, s_q);
  __syncthreads();
  WinIter it(g);
  bnact_tan_phase(a, g, task, blockIdx.x, gridDim.x, it, s_r, s_g, s_b, s_md, s_q);
}

// forward tangent with gamma / beta tangents (functional operator's forward mode); a kernel of its own, so that the
// fused iteration's bnact_tan_kernel keeps its code
__global__ void __launch_bounds__(256) bnact_tan_gb_kernel(BnActTanArgs a, const float* gdot, const float* bdot) {
  pdl_prologue(32, a.tag);
  __shared__ float s_mu[64], s_r[64], s_g[64], s_b[64], s_md[64], s_q[64], s_gd[64], s_bd[64];
  const BnGeom g = a.g;
  const int task = blockIdx.y;
  bnact_tan_setup(a, g, task, (double)g.n * g.h * g.w, s_mu, s_r, s_g, s_b, s_md, s_q);
  if (threadIdx.x < g.F) { s_gd[threadIdx.x] = gdot[threadIdx.x]; s_bd[threadIdx.x] = bdot[threadIdx.x]; }
  __syncthreads();
  WinIter it(g);
  bnact_tan_phase<true>(a, g, task, blockIdx.x, gridDim.x, it, s_r, s_g, s_b, s_md, s_q, s_gd, s_bd);
}

void launch_bnact_tan(const BnActTanArgs& a, cudaStream_t st, const float* gdot, const float* bdot) {
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  int block; dim3 grid = bn_grid(a.g, a.tasks, &block);
  if (gdot) launch_pdl(bnact_tan_gb_kernel, dim3(grid), dim3(block), (size_t)(0), st, tagged(a), gdot, bdot);
  else launch_pdl(bnact_tan_kernel, dim3(grid), dim3(block), (size_t)(0), st, tagged(a));
  CUDA_CHECK_LAUNCH();
}

// ------------------------------------------------------------------------------- tangent backward: reduce
// T1 = sum dydot,  T2 = sum (dydot * zh + dy * zhdot)   (both only at the arg-max position)
__device__ __forceinline__ void bnbwd_tan_reduce_phase(const BnBwdTanArgs& a, const BnGeom& g, int task, int cta, int ncta,
                                                       const WinIter& it, const float* s_g, const float* s_b, double (&s1)[4],
                                                       double (&s2)[4]) {
  if (it.lane >= it.WPB) return;
  const float4 ga = ld4s(s_g, it.q), be = ld4s(s_b, it.q);
  const float* zhp = a.zh + (long long)task * a.zh_stride;
  const float* zhd = a.zhdot + (long long)task * a.zhdot_stride;
  const float* dp = a.dp + (long long)task * a.dp_stride;
  const float* dpd = a.dpdot + (long long)task * a.dpdot_stride;
  for (int wi = cta * it.WPB + it.lane; wi < it.NW; wi += ncta * it.WPB) {
    int img, wy, wx; it.window(wi, img, wy, wx);
    if (wy >= g.ph || wx >= g.pw) continue;
    float4 zh[4]; long long idx[4]; int4 arg; float4 sl;
    argmax_window(zhp, g, img, wy, wx, it, ga, be, zh, idx, arg, sl);
    const long long pidx = it.pooled(g, img, wy, wx);
    const float4 d = ld4(dp + pidx);
    float4 dd = ld4(dpd + pidx);
    if (a.dpdot2) {
      const float4 d2 = ld4(a.dpdot2 + (long long)task * a.dpdot_stride + pidx);
      dd.x += d2.x; dd.y += d2.y; dd.z += d2.z; dd.w += d2.w;
    }
    const int ar[4] = {arg.x, arg.y, arg.z, arg.w};
    const float slv[4] = {sl.x, sl.y, sl.z, sl.w};
    const float dv[4] = {d.x, d.y, d.z, d.w};
    const float ddv[4] = {dd.x, dd.y, dd.z, dd.w};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float zhk = pick(zh, ar[c], c);
      const float zhdk = zhd[idx[ar[c]] + c];
      const float dy = dv[c] * slv[c], dyd = ddv[c] * slv[c];
      s1[c] += dyd;
      s2[c] += (double)dyd * (double)zhk + (double)dy * (double)zhdk;
    }
  }
}

__global__ void __launch_bounds__(256) bnbwd_tan_reduce_kernel(BnBwdTanArgs a) {
  pdl_prologue(11, a.tag);
  __shared__ float s_g[64], s_b[64];
  const BnGeom g = a.g;
  const int task = blockIdx.y;
  if (threadIdx.x < g.F) { s_g[threadIdx.x] = a.gamma[threadIdx.x]; s_b[threadIdx.x] = a.beta[threadIdx.x]; }
  __syncthreads();
  WinIter it(g);
  double s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  bnbwd_tan_reduce_phase(a, g, task, blockIdx.x, gridDim.x, it, s_g, s_b, s1, s2);
  block_reduce_stats(s1, s2, it, a.stats_tbwd + (long long)task * a.stats_tbwd_stride, g.F);
}

void launch_bnbwd_tan_reduce(const BnBwdTanArgs& a, cudaStream_t st) {
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  int block; dim3 grid = bn_grid(a.g, a.tasks, &block);
  if ((int)grid.x > num_sms()) grid.x = num_sms();
  launch_pdl(bnbwd_tan_reduce_kernel, dim3(grid), dim3(block), (size_t)(0), st, tagged(a));
  CUDA_CHECK_LAUNCH();
}

// ------------------------------------------------------------------------------- tangent backward: apply
// dzdot = -r*q*dz + r*gamma*(dydot - T1/m - zhdot*S2/m - zh*T2/m)
__device__ __forceinline__ void bnbwd_tan_apply_phase(const BnBwdTanArgs& a, const BnGeom& g, int task, int cta, int ncta,
                                                      const WinIter& it, const float* s_r, const float* s_g, const float* s_b,
                                                      const float* s_q, const float* s_c2, const float* s_t1, const float* s_t2) {
  if (it.lane >= it.WPB) return;
  const float4 r = ld4s(s_r, it.q), ga = ld4s(s_g, it.q), be = ld4s(s_b, it.q);
  const float4 qq = ld4s(s_q, it.q), c2 = ld4s(s_c2, it.q), t1 = ld4s(s_t1, it.q), t2 = ld4s(s_t2, it.q);
  const float4 rg = make_float4(r.x * ga.x, r.y * ga.y, r.z * ga.z, r.w * ga.w);
  const float4 rq = make_float4(-r.x * qq.x, -r.y * qq.y, -r.z * qq.z, -r.w * qq.w);
  const float* zhp = a.zh + (long long)task * a.zh_stride;
  const float* zhd = a.zhdot + (long long)task * a.zhdot_stride;
  const float* dzp = a.dz + (long long)task * a.dz_stride;
  const float* dpd = a.dpdot + (long long)task * a.dpdot_stride;
  float* dzd = a.dzdot + (long long)task * a.dzdot_stride;
  for (int wi = cta * it.WPB + it.lane; wi < it.NW; wi += ncta * it.WPB) {
    int img, wy, wx; it.window(wi, img, wy, wx);
    const bool full = (wy < g.ph && wx < g.pw);
    int4 arg = make_int4(-1, -1, -1, -1);
    float4 dyd = make_float4(0.f, 0.f, 0.f, 0.f);
    if (full) {
      float4 zh[4]; long long idx[4]; float4 sl;
      argmax_window(zhp, g, img, wy, wx, it, ga, be, zh, idx, arg, sl);
      const long long pidx = it.pooled(g, img, wy, wx);
      float4 dd = ld4(dpd + pidx);
      if (a.dpdot2) {
        const float4 d2 = ld4(a.dpdot2 + (long long)task * a.dpdot_stride + pidx);
        dd.x += d2.x; dd.y += d2.y; dd.z += d2.z; dd.w += d2.w;
      }
      dyd = make_float4(dd.x * sl.x, dd.y * sl.y, dd.z * sl.z, dd.w * sl.w);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
      if (yy < g.h && xx < g.w) {
        const long long idx = it.grid(g, img, yy, xx);
        const float4 zh = ld4(zhp + idx), zd = ld4(zhd + idx), dzv = ld4(dzp + idx);
        float4 o;
        o.x = rq.x * dzv.x + rg.x * ((arg.x == k ? dyd.x : 0.f) - t1.x - zd.x * c2.x - zh.x * t2.x);
        o.y = rq.y * dzv.y + rg.y * ((arg.y == k ? dyd.y : 0.f) - t1.y - zd.y * c2.y - zh.y * t2.y);
        o.z = rq.z * dzv.z + rg.z * ((arg.z == k ? dyd.z : 0.f) - t1.z - zd.z * c2.z - zh.z * t2.z);
        o.w = rq.w * dzv.w + rg.w * ((arg.w == k ? dyd.w : 0.f) - t1.w - zd.w * c2.w - zh.w * t2.w);
        st4(dzd + idx, o);
        if (a.dzdot_hi) st4_split(a.dzdot_hi + (long long)task * a.dzdot_stride, a.dzdot_lo + (long long)task * a.dzdot_stride, idx, o);
      }
    }
  }
}

__device__ __forceinline__ void bnbwd_tan_setup(const BnBwdTanArgs& a, const BnGeom& g, int task, double m, float* s_mu, float* s_r,
                                                float* s_g, float* s_b, float* s_q, float* s_c2) {
  chan_setup(a.stats_fwd + (long long)task * a.stats_fwd_stride, a.gamma, a.beta, m, g.F, s_mu, s_r, s_g, s_b);
  if (threadIdx.x < g.F) {
    const int c = threadIdx.x;
    s_q[c] = (float)((a.stats_tan + (long long)task * a.stats_tan_stride)[c * 2 + 1] / m);
    s_c2[c] = (float)((a.stats_bwd + (long long)task * a.stats_bwd_stride)[c * 2 + 1] / m);
  }
}

__global__ void __launch_bounds__(256) bnbwd_tan_apply_kernel(BnBwdTanArgs a) {
  pdl_prologue(12, a.tag);
  __shared__ float s_mu[64], s_r[64], s_g[64], s_b[64], s_q[64], s_c2[64], s_t1[64], s_t2[64];
  const BnGeom g = a.g;
  const int task = blockIdx.y;
  const double m = (double)g.n * g.h * g.w;
  bnbwd_tan_setup(a, g, task, m, s_mu, s_r, s_g, s_b, s_q, s_c2);
  if (threadIdx.x < g.F) {
    const int c = threadIdx.x;
    const double* tb = a.stats_tbwd + (long long)task * a.stats_tbwd_stride;
    s_t1[c] = (float)(tb[c * 2] / m);
    s_t2[c] = (float)(tb[c * 2 + 1] / m);
  }
  __syncthreads();
  WinIter it(g);
  bnbwd_tan_apply_phase(a, g, task, blockIdx.x, gridDim.x, it, s_r, s_g, s_b, s_q, s_c2, s_t1, s_t2);
}

__global__ void __launch_bounds__(256) bnbwd_tan_fused_kernel(BnBwdTanArgs a) {
  pdl_prologue(13, a.tag);
  bn_cluster_arrive();
  __shared__ float s_mu[64], s_r[64], s_g[64], s_b[64], s_q[64], s_c2[64], s_t1[64], s_t2[64];
  __shared__ double gather[8][128];
  const BnGeom g = a.g;
  const int task = blockIdx.y;
  const double m = (double)g.n * g.h * g.w;
  bnbwd_tan_setup(a, g, task, m, s_mu, s_r, s_g, s_b, s_q, s_c2);
  __syncthreads();
  WinIter it(g);
  double s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  bnbwd_tan_reduce_phase(a, g, task, blockIdx.x, gridDim.x, it, s_g, s_b, s1, s2);
  const double tot = block_reduce_totals(s1, s2, it, g.F);
  cluster_allreduce_stats(tot, gather, g.F, m, s_t1, s_t2, a.stats_tbwd + (long long)task * a.stats_tbwd_stride);
  bnbwd_tan_apply_phase(a, g, task, blockIdx.x, gridDim.x, it, s_r, s_g, s_b, s_q, s_c2, s_t1, s_t2);
}

void launch_bnbwd_tan_apply(const BnBwdTanArgs& a, cudaStream_t st) {
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  int block; dim3 grid = bn_grid(a.g, a.tasks, &block);
  launch_pdl(bnbwd_tan_apply_kernel, dim3(grid), dim3(block), (size_t)(0), st, tagged(a));
  CUDA_CHECK_LAUNCH();
}

void launch_bnbwd_tan(const BnBwdTanArgs& a, cudaStream_t st) {
  const int cl = bn_fused_cluster(a.g);
  if (cl == 0) { launch_bnbwd_tan_reduce(a, st); launch_bnbwd_tan_apply(a, st); return; }
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  int block; bn_grid(a.g, a.tasks, &block);
  launch_cluster(bnbwd_tan_fused_kernel, tagged(a), cl, a.tasks, block, st);
  CUDA_CHECK_LAUNCH();
}

// ---------------------------------------------------------------------------------------------------------------
// Fused last block + head: when the last block of a task is tiny (<= 4 pooling windows per thread, <= 16 rows), its
// BatchNorm/activation/pool, the classifier head (logits, loss gradient, weight-gradient chunk, feature gradient) and
// the BatchNorm backward of the same block are ONE kernel with one CTA per task: the three stages exchange their data
// through global memory written and re-read by the same CTA (visible after __syncthreads), the backward sums need no
// cluster.  Replaces three dependent launches on the critical path of every support / tangent pass.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) tail_fused_kernel(BnActArgs fa, HeadArgs ha, BnBwdArgs ba) {
  pdl_prologue(23, fa.tag);
  extern __shared__ float smh[];
  __shared__ float s_mu[64], s_r[64], s_g[64], s_b[64], s_c1[64], s_c2[64];
  __shared__ float s_rowloss[64], s_rowcorrect[64];
  const BnGeom g = fa.g;
  const int task = blockIdx.y;
  const double m = (double)g.n * g.h * g.w;
  chan_setup(fa.stats + (long long)task * fa.stats_stride, fa.gamma, fa.beta, m, g.F, s_mu, s_r, s_g, s_b);
  __syncthreads();
  WinIter it(g);
  bnact_phase(fa, g, task, 0, 1, it, s_mu, s_r, s_g, s_b);
  __syncthreads();
  head_body<true>(ha, task, 0, smh, s_rowloss, s_rowcorrect);
  __syncthreads();
  double s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  bnbwd_reduce_phase(ba, g, task, 0, 1, it, s_g, s_b, s1, s2);
  const double t = block_reduce_totals(s1, s2, it, g.F);
  if (threadIdx.x < g.F * 2) {
    ((threadIdx.x & 1) ? s_c2 : s_c1)[threadIdx.x >> 1] = (float)(t / m);
    (ba.stats_bwd + (long long)task * ba.stats_bwd_stride)[threadIdx.x] = t;
  }
  __syncthreads();
  bnbwd_apply_phase(ba, g, task, 0, 1, it, s_r, s_g, s_b, s_c1, s_c2);
}

__global__ void __launch_bounds__(256) tail_tan_fused_kernel(BnActTanArgs fa, HeadArgs ha, BnBwdTanArgs ba) {
  pdl_prologue(24, fa.tag);
  extern __shared__ float smh[];
  __shared__ float s_mu[64], s_r[64], s_g[64], s_b[64], s_md[64], s_q[64], s_c2[64], s_t1[64], s_t2[64];
  __shared__ float s_rowloss[64], s_rowcorrect[64];
  const BnGeom g = fa.g;
  const int task = blockIdx.y;
  const double m = (double)g.n * g.h * g.w;
  bnact_tan_setup(fa, g, task, m, s_mu, s_r, s_g, s_b, s_md, s_q);
  if (threadIdx.x < g.F) s_c2[threadIdx.x] = (float)((ba.stats_bwd + (long long)task * ba.stats_bwd_stride)[threadIdx.x * 2 + 1] / m);
  __syncthreads();
  WinIter it(g);
  bnact_tan_phase(fa, g, task, 0, 1, it, s_r, s_g, s_b, s_md, s_q);
  __syncthreads();
  head_body<true>(ha, task, 0, smh, s_rowloss, s_rowcorrect);
  __syncthreads();
  double s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  bnbwd_tan_reduce_phase(ba, g, task, 0, 1, it, s_g, s_b, s1, s2);
  const double t = block_reduce_totals(s1, s2, it, g.F);
  if (threadIdx.x < g.F * 2) {
    ((threadIdx.x & 1) ? s_t2 : s_t1)[threadIdx.x >> 1] = (float)(t / m);
    (ba.stats_tbwd + (long long)task * ba.stats_tbwd_stride)[threadIdx.x] = t;
  }
  __syncthreads();
  bnbwd_tan_apply_phase(ba, g, task, 0, 1, it, s_r, s_g, s_b, s_q, s_c2, s_t1, s_t2);
}

// On-chip variant of tail_fused_kernel (primal): what the three stages exchange stays in shared memory / registers.
//   stage 1  every thread owns <= MAXI (pooling window, channel quad) items: loads z once, keeps zh[4], the arg-max and
//            the leaky slope in REGISTERS, writes zh / p to global for later passes and p into shared memory (features);
//   stage 2  head_body runs on shared-memory copies of the features, W_fc, b_fc and leaves df in shared memory;
//   stage 3  BatchNorm backward of the same items from registers + shared df: block reduction -> c1, c2 -> dz.
// One global round trip (z, statistics, W_fc in parallel) instead of ~8 dependent ones.
template <int MAXI>
__global__ void __launch_bounds__(256) tail_onchip_kernel(BnActArgs fa, HeadArgs ha, BnBwdArgs ba) {
  pdl_prologue(25, fa.tag);
  extern __shared__ float smh[];                  // [head scratch 5*R*N | f n*D | df n*D | W N*D | b N]
  __shared__ float s_mu[64], s_r[64], s_g[64], s_b[64], s_c1[64], s_c2[64];
  __shared__ float s_rowloss[64], s_rowcorrect[64];
  const BnGeom g = fa.g;
  const int task = blockIdx.y;
  const int tid = threadIdx.x;
  const int n = ha.n, N = ha.N, D = ha.D;
  float* s_f = smh + 5 * ha.rows_per_cta * N;
  float* s_df = s_f + n * D;
  float* s_W = s_df + n * D;
  float* s_bfc = s_W + N * D;
  const double m = (double)g.n * g.h * g.w;
  chan_setup(fa.stats + (long long)task * fa.stats_stride, fa.gamma, fa.beta, m, g.F, s_mu, s_r, s_g, s_b);
  {
    const float* W = ha.Wfc + (long long)task * ha.theta_stride;
    const float* bb = ha.bfc + (long long)task * ha.theta_stride;
    for (int o = tid; o < N * D; o += 256) s_W[o] = W[o];
    if (tid < N) s_bfc[tid] = bb[tid];
  }
  __syncthreads();
  WinIter it(g);
  const bool worker = it.lane < it.WPB;
  float4 zh[MAXI][4]; int4 arg[MAXI]; float4 sl[MAXI]; int wy_[MAXI], wx_[MAXI], img_[MAXI]; bool have[MAXI], full[MAXI];
  float4 mu, r, ga, be;
  if (worker) { mu = ld4s(s_mu, it.q); r = ld4s(s_r, it.q); ga = ld4s(s_g, it.q); be = ld4s(s_b, it.q); }
  float* z = fa.z + (long long)task * fa.z_stride;
  float* pg = fa.p + (long long)task * fa.p_stride;
  // ---------------- stage 1: BatchNorm + leaky-ReLU + max-pool (first max wins)
#pragma unroll
  for (int i = 0; i < MAXI; ++i) {
    const int wi = it.lane + i * it.WPB;
    have[i] = worker && wi < it.NW;
    full[i] = false;
    if (!have[i]) continue;
    int img, wy, wx; it.window(wi, img, wy, wx);
    img_[i] = img; wy_[i] = wy; wx_[i] = wx;
    float4 best = make_float4(0.f, 0.f, 0.f, 0.f), ybest = best;
    int4 am = make_int4(0, 0, 0, 0);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
      zh[i][k] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (yy < g.h && xx < g.w) {
        const long long idx = it.grid(g, img, yy, xx);
        const float4 zv = ld4(z + idx);
        float4 zz, y, act;
        zz.x = (zv.x - mu.x) * r.x; zz.y = (zv.y - mu.y) * r.y; zz.z = (zv.z - mu.z) * r.z; zz.w = (zv.w - mu.w) * r.w;
        st4(z + idx, zz);
        zh[i][k] = zz;
        y.x = fmaf(ga.x, zz.x, be.x); y.y = fmaf(ga.y, zz.y, be.y); y.z = fmaf(ga.z, zz.z, be.z); y.w = fmaf(ga.w, zz.w, be.w);
        act.x = leaky(y.x); act.y = leaky(y.y); act.z = leaky(y.z); act.w = leaky(y.w);
        if (k == 0) { best = act; ybest = y; }
        else {
          if (act.x > best.x) { best.x = act.x; ybest.x = y.x; am.x = k; }
          if (act.y > best.y) { best.y = act.y; ybest.y = y.y; am.y = k; }
          if (act.z > best.z) { best.z = act.z; ybest.z = y.z; am.z = k; }
          if (act.w > best.w) { best.w = act.w; ybest.w = y.w; am.w = k; }
        }
      }
    }
    arg[i] = am;
    sl[i] = make_float4(slope_of(ybest.x), slope_of(ybest.y), slope_of(ybest.z), slope_of(ybest.w));
    full[i] = (wy < g.ph && wx < g.pw);
    if (full[i]) {
      const long long pidx = it.pooled(g, img, wy, wx);
      st4(pg + pidx, best);
      st4(s_f + pidx, best);                       // pb = 0 on the last block: pidx is the feature index img * D + ...
    }
  }
  __syncthreads();
  // ---------------- stage 2: classifier head on the shared-memory copies
  {
    HeadArgs hs = ha;
    hs.f = s_f; hs.f_stride = 0;
    hs.Wfc = s_W; hs.bfc = s_bfc; hs.theta_stride = 0;
    hs.df = s_df; hs.df_stride = 0;
    head_body<true>(hs, task, 0, smh, s_rowloss, s_rowcorrect);
  }
  __syncthreads();
  {
    float* dfg = ha.df + (long long)task * ha.df_stride;     // phase B reads the primal df again
    for (int o = tid; o < n * D; o += 256) dfg[o] = s_df[o];
  }
  // ---------------- stage 3: BatchNorm backward of the same items
  double s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  float4 dyv[MAXI];
#pragma unroll
  for (int i = 0; i < MAXI; ++i) {
    dyv[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!have[i] || !full[i]) continue;
    const long long pidx = it.pooled(g, img_[i], wy_[i], wx_[i]);
    const float4 d = ld4(s_df + pidx);
    dyv[i] = make_float4(d.x * sl[i].x, d.y * sl[i].y, d.z * sl[i].z, d.w * sl[i].w);
    s1[0] += dyv[i].x; s2[0] += (double)dyv[i].x * (double)pick(zh[i], arg[i].x, 0);
    s1[1] += dyv[i].y; s2[1] += (double)dyv[i].y * (double)pick(zh[i], arg[i].y, 1);
    s1[2] += dyv[i].z; s2[2] += (double)dyv[i].z * (double)pick(zh[i], arg[i].z, 2);
    s1[3] += dyv[i].w; s2[3] += (double)dyv[i].w * (double)pick(zh[i], arg[i].w, 3);
  }
  const double t = block_reduce_totals(s1, s2, it, g.F);
  if (tid < g.F * 2) {
    ((tid & 1) ? s_c2 : s_c1)[tid >> 1] = (float)(t / m);
    (ba.stats_bwd + (long long)task * ba.stats_bwd_stride)[tid] = t;
  }
  __syncthreads();
  if (!worker) return;
  const float4 c1 = ld4s(s_c1, it.q), c2 = ld4s(s_c2, it.q);
  const float4 rg = make_float4(r.x * ga.x, r.y * ga.y, r.z * ga.z, r.w * ga.w);
  float* dz = ba.dz + (long long)task * ba.dz_stride;
#pragma unroll
  for (int i = 0; i < MAXI; ++i) {
    if (!have[i]) continue;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = 2 * wy_[i] + (k >> 1), xx = 2 * wx_[i] + (k & 1);
      if (yy < g.h && xx < g.w) {
        const long long idx = it.grid(g, img_[i], yy, xx);
        float4 o;
        o.x = rg.x * ((full[i] && arg[i].x == k ? dyv[i].x : 0.f) - c1.x - zh[i][k].x * c2.x);
        o.y = rg.y * ((full[i] && arg[i].y == k ? dyv[i].y : 0.f) - c1.y - zh[i][k].y * c2.y);
        o.z = rg.z * ((full[i] && arg[i].z == k ? dyv[i].z : 0.f) - c1.z - zh[i][k].z * c2.z);
        o.w = rg.w * ((full[i] && arg[i].w == k ? dyv[i].w : 0.f) - c1.w - zh[i][k].w * c2.w);
        st4(dz + idx, o);
        if (ba.dz_hi) st4_split(ba.dz_hi + (long long)task * ba.dz_stride, ba.dz_lo + (long long)task * ba.dz_stride, idx, o);
      }
    }
  }
}

// On-chip variant of tail_tan_fused_kernel (tangent pass), same plan as tail_onchip_kernel:
//   stage 1  every thread owns <= MAXI (pooling window, channel quad) items: loads the primal zh and the tangent zdot
//            (both addends) once, keeps zh[4], zhdot[4], the arg-max and the leaky slope in REGISTERS, writes zhdot / pdot to
//            global for the record and pdot into shared memory (tangent features);
//   stage 2  head_body (HEAD_TANGENT) on shared-memory copies of f, fdot, W_fc, u_W, b_fc, u_b; leaves d(f)dot in shared memory;
//   stage 3  tangent BatchNorm backward of the same items from registers + shared memory; the primal dp / dz it also needs
//            are loaded at the top of the kernel (they were written in phase A).
template <int MAXI>
__global__ void __launch_bounds__(256) tail_tan_onchip_kernel(BnActTanArgs fa, HeadArgs ha, BnBwdTanArgs ba) {
  pdl_prologue(24, fa.tag);
  extern __shared__ float smh[];                  // [head scratch 5*R*N | f n*D | fdot n*D | dfdot n*D | W N*D | uW N*D | b N | ub N]
  __shared__ float s_mu[64], s_r[64], s_g[64], s_b[64], s_md[64], s_q[64], s_c2[64], s_t1[64], s_t2[64];
  __shared__ float s_rowloss[64], s_rowcorrect[64];
  const BnGeom g = fa.g;
  const int task = blockIdx.y;
  const int tid = threadIdx.x;
  const int n = ha.n, N = ha.N, D = ha.D;
  float* s_f = smh + 5 * ha.rows_per_cta * N;
  float* s_fd = s_f + n * D;
  float* s_dfd = s_fd + n * D;
  float* s_W = s_dfd + n * D;
  float* s_uW = s_W + N * D;
  float* s_bfc = s_uW + N * D;
  float* s_ub = s_bfc + N;
  const double m = (double)g.n * g.h * g.w;
  bnact_tan_setup(fa, g, task, m, s_mu, s_r, s_g, s_b, s_md, s_q);
  if (tid < g.F) s_c2[tid] = (float)((ba.stats_bwd + (long long)task * ba.stats_bwd_stride)[tid * 2 + 1] / m);
  {
    const float* W = ha.Wfc + (long long)task * ha.theta_stride;
    const float* bb = ha.bfc + (long long)task * ha.theta_stride;
    const float* uW = ha.uW + (long long)task * ha.u_stride;
    const float* ub = ha.ub + (long long)task * ha.u_stride;
    const float* f = ha.f + (long long)task * ha.f_stride;
    for (int o = tid; o < N * D; o += 256) { s_W[o] = W[o]; s_uW[o] = uW[o]; }
    for (int o = tid; o < n * D; o += 256) s_f[o] = f[o];
    if (tid < N) { s_bfc[tid] = bb[tid]; s_ub[tid] = ub[tid]; }
  }
  __syncthreads();
  WinIter it(g);
  const bool worker = it.lane < it.WPB;
  float4 zh[MAXI][4], zhd[MAXI][4]; int4 arg[MAXI]; float4 sl[MAXI]; float4 dprim[MAXI];
  int wy_[MAXI], wx_[MAXI], img_[MAXI]; bool have[MAXI], full[MAXI];
  float4 r, ga, be, md, qq;
  if (worker) { r = ld4s(s_r, it.q); ga = ld4s(s_g, it.q); be = ld4s(s_b, it.q); md = ld4s(s_md, it.q); qq = ld4s(s_q, it.q); }
  float* zd = fa.zdot + (long long)task * fa.zdot_stride;
  const float* zd2 = fa.zdot2 ? fa.zdot2 + (long long)task * fa.zdot_stride : nullptr;
  const float* zhp = fa.zh + (long long)task * fa.zh_stride;
  float* pdg = fa.pdot + (long long)task * fa.pdot_stride;
  const float* dpp = ba.dp + (long long)task * ba.dp_stride;
  // ---------------- stage 1: tangent of BatchNorm + leaky-ReLU + max-pool at the primal arg-max (first max wins)
#pragma unroll
  for (int i = 0; i < MAXI; ++i) {
    const int wi = it.lane + i * it.WPB;
    have[i] = worker && wi < it.NW;
    full[i] = false;
    dprim[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!have[i]) continue;
    int img, wy, wx; it.window(wi, img, wy, wx);
    img_[i] = img; wy_[i] = wy; wx_[i] = wx;
    full[i] = (wy < g.ph && wx < g.pw);
    const long long pidx = it.pooled(g, img, wy, wx);
    if (full[i]) dprim[i] = ld4(dpp + pidx);                 // primal d(loss)/d(pooled), written in phase A
    float4 best = make_float4(0.f, 0.f, 0.f, 0.f), ybest = best, pbest = best;
    int4 am = make_int4(0, 0, 0, 0);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
      zh[i][k] = make_float4(0.f, 0.f, 0.f, 0.f);
      zhd[i][k] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (yy < g.h && xx < g.w) {
        const long long idx = it.grid(g, img, yy, xx);
        const float4 z = ld4(zhp + idx);
        float4 zv = ld4(zd + idx);
        if (zd2) { const float4 z2 = ld4(zd2 + idx); zv.x += z2.x; zv.y += z2.y; zv.z += z2.z; zv.w += z2.w; }
        float4 d;
        d.x = r.x * (zv.x - md.x - z.x * qq.x); d.y = r.y * (zv.y - md.y - z.y * qq.y);
        d.z = r.z * (zv.z - md.z - z.z * qq.z); d.w = r.w * (zv.w - md.w - z.w * qq.w);
        st4(zd + idx, d);
        zh[i][k] = z; zhd[i][k] = d;
        float4 y, act, pdv;
        y.x = fmaf(ga.x, z.x, be.x); y.y = fmaf(ga.y, z.y, be.y); y.z = fmaf(ga.z, z.z, be.z); y.w = fmaf(ga.w, z.w, be.w);
        act.x = leaky(y.x); act.y = leaky(y.y); act.z = leaky(y.z); act.w = leaky(y.w);
        pdv.x = slope_of(y.x) * ga.x * d.x; pdv.y = slope_of(y.y) * ga.y * d.y;
        pdv.z = slope_of(y.z) * ga.z * d.z; pdv.w = slope_of(y.w) * ga.w * d.w;
        if (k == 0) { best = act; ybest = y; pbest = pdv; }
        else {
          if (act.x > best.x) { best.x = act.x; ybest.x = y.x; pbest.x = pdv.x; am.x = k; }
          if (act.y > best.y) { best.y = act.y; ybest.y = y.y; pbest.y = pdv.y; am.y = k; }
          if (act.z > best.z) { best.z = act.z; ybest.z = y.z; pbest.z = pdv.z; am.z = k; }
          if (act.w > best.w) { best.w = act.w; ybest.w = y.w; pbest.w = pdv.w; am.w = k; }
        }
      }
    }
    arg[i] = am;
    sl[i] = make_float4(slope_of(ybest.x), slope_of(ybest.y), slope_of(ybest.z), slope_of(ybest.w));
    if (full[i]) {
      st4(pdg + pidx, pbest);
      st4(s_fd + pidx, pbest);                     // pb = 0 on the last block: pidx is the feature index img * D + ...
    }
  }
  __syncthreads();
  // ---------------- stage 2: tangent of the classifier head on the shared-memory copies
  {
    HeadArgs hs = ha;
    hs.f = s_f; hs.f_stride = 0;
    hs.fdot = s_fd; hs.fdot_stride = 0;
    hs.Wfc = s_W; hs.bfc = s_bfc; hs.theta_stride = 0;
    hs.uW = s_uW; hs.ub = s_ub; hs.u_stride = 0;
    hs.df = s_dfd; hs.df_stride = 0;
    head_body<true>(hs, task, 0, smh, s_rowloss, s_rowcorrect);
  }
  __syncthreads();
  {
    float* dfg = ha.df + (long long)task * ha.df_stride;
    for (int o = tid; o < n * D; o += 256) dfg[o] = s_dfd[o];
  }
  // ---------------- stage 3: tangent BatchNorm backward of the same items
  //   T1 = sum dydot, T2 = sum (dydot * zh + dy * zhdot) at the arg-max;  dzdot = -r q dz + r gamma (dydot - T1/m - zhdot S2/m - zh T2/m)
  const float* dzp = ba.dz + (long long)task * ba.dz_stride;
  double s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  float4 dydv[MAXI];
#pragma unroll
  for (int i = 0; i < MAXI; ++i) {
    dydv[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!have[i] || !full[i]) continue;
    const long long pidx = it.pooled(g, img_[i], wy_[i], wx_[i]);
    const float4 dd = ld4(s_dfd + pidx);
    const int ar[4] = {arg[i].x, arg[i].y, arg[i].z, arg[i].w};
    const float slv[4] = {sl[i].x, sl[i].y, sl[i].z, sl[i].w};
    const float dv[4] = {dprim[i].x, dprim[i].y, dprim[i].z, dprim[i].w};
    const float ddv[4] = {dd.x, dd.y, dd.z, dd.w};
    float dydc[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float zhk = pick(zh[i], ar[c], c);
      const float zhdk = pick(zhd[i], ar[c], c);
      const float dy = dv[c] * slv[c], dyd = ddv[c] * slv[c];
      dydc[c] = dyd;
      s1[c] += dyd;
      s2[c] += (double)dyd * (double)zhk + (double)dy * (double)zhdk;
    }
    dydv[i] = make_float4(dydc[0], dydc[1], dydc[2], dydc[3]);
  }
  const double t = block_reduce_totals(s1, s2, it, g.F);
  if (tid < g.F * 2) {
    ((tid & 1) ? s_t2 : s_t1)[tid >> 1] = (float)(t / m);
    (ba.stats_tbwd + (long long)task * ba.stats_tbwd_stride)[tid] = t;
  }
  __syncthreads();
  if (!worker) return;
  const float4 c2 = ld4s(s_c2, it.q), t1 = ld4s(s_t1, it.q), t2 = ld4s(s_t2, it.q);
  const float4 rg = make_float4(r.x * ga.x, r.y * ga.y, r.z * ga.z, r.w * ga.w);
  const float4 rq = make_float4(-r.x * qq.x, -r.y * qq.y, -r.z * qq.z, -r.w * qq.w);
  float* dzd = ba.dzdot + (long long)task * ba.dzdot_stride;
#pragma unroll
  for (int i = 0; i < MAXI; ++i) {
    if (!have[i]) continue;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = 2 * wy_[i] + (k >> 1), xx = 2 * wx_[i] + (k & 1);
      if (yy < g.h && xx < g.w) {
        const long long idx = it.grid(g, img_[i], yy, xx);
        const float4 dzv = ld4(dzp + idx);
        const float4 z = zh[i][k], zdk = zhd[i][k];
        float4 o;
        o.x = rq.x * dzv.x + rg.x * ((full[i] && arg[i].x == k ? dydv[i].x : 0.f) - t1.x - zdk.x * c2.x - z.x * t2.x);
        o.y = rq.y * dzv.y + rg.y * ((full[i] && arg[i].y == k ? dydv[i].y : 0.f) - t1.y - zdk.y * c2.y - z.y * t2.y);
        o.z = rq.z * dzv.z + rg.z * ((full[i] && arg[i].z == k ? dydv[i].z : 0.f) - t1.z - zdk.z * c2.z - z.z * t2.z);
        o.w = rq.w * dzv.w + rg.w * ((full[i] && arg[i].w == k ? dydv[i].w : 0.f) - t1.w - zdk.w * c2.w - z.w * t2.w);
        st4(dzd + idx, o);
        if (ba.dzdot_hi) st4_split(ba.dzdot_hi + (long long)task * ba.dzdot_stride, ba.dzdot_lo + (long long)task * ba.dzdot_stride, idx, o);
      }
    }
  }
}

// the last block of `n` images is small enough for the fused kernels
bool tail_fusable(const BnGeom& g, int n_rows, int rows_per_cta) {
  const WinGeom wg = win_geom(g);
  return launch_ctx().opt->bn_fuse && g.F <= 64 && n_rows <= rows_per_cta && wg.NW <= 4 * wg.wpb;
}

// Windows per thread (MAXI) of the on-chip tail kernel, 0: the global-memory one.  On chip needs option bit `onchip_bit`,
// no pooled border, none of the inputs / outputs it lacks (`other_io`: TF32 planes, a second tangent addend), <= 2 windows
// per thread and its `words` floats of dynamic shared memory within 40 KB.
static int tail_onchip_items(const BnGeom& g, int onchip_bit, bool other_io, size_t words) {
  const WinGeom wg = win_geom(g);
  if (!(launch_ctx().opt->tail_onchip & onchip_bit) || g.pb != 0 || other_io || wg.NW > 2 * wg.wpb ||
      words * sizeof(float) > 40 * 1024)
    return 0;
  return wg.NW <= wg.wpb ? 1 : 2;
}

void launch_tail_fused(const BnActArgs& fa, const HeadArgs& ha, const BnBwdArgs& ba, cudaStream_t st) {
  ProfScope prof_scope__(PROF_HEAD, 0.0, st);
  const size_t words = (size_t)5 * ha.rows_per_cta * ha.N + 2 * (size_t)ha.n * ha.D + (size_t)ha.N * ha.D + ha.N;
  const int items = tail_onchip_items(fa.g, 1, fa.p_hi != nullptr, words);
  auto kernel = items == 0 ? tail_fused_kernel : items == 1 ? tail_onchip_kernel<1> : tail_onchip_kernel<2>;
  const size_t smem = (items ? words : (size_t)5 * ha.rows_per_cta * ha.N) * sizeof(float);
  launch_pdl(kernel, dim3(1, fa.tasks), dim3(256), smem, st, tagged(fa), ha, ba);
  CUDA_CHECK_LAUNCH();
}

void launch_tail_tan_fused(const BnActTanArgs& fa, const HeadArgs& ha, const BnBwdTanArgs& ba, cudaStream_t st) {
  ProfScope prof_scope__(PROF_HEAD, 0.0, st);
  const size_t words = (size_t)5 * ha.rows_per_cta * ha.N + 3 * (size_t)ha.n * ha.D + 2 * (size_t)ha.N * ha.D + 2 * ha.N;
  const int items = tail_onchip_items(fa.g, 2, fa.pdot_hi != nullptr || ba.dpdot2 != nullptr, words);
  auto kernel = items == 0 ? tail_tan_fused_kernel : items == 1 ? tail_tan_onchip_kernel<1> : tail_tan_onchip_kernel<2>;
  const size_t smem = (items ? words : (size_t)5 * ha.rows_per_cta * ha.N) * sizeof(float);
  launch_pdl(kernel, dim3(1, fa.tasks), dim3(256), smem, st, tagged(fa), ha, ba);
  CUDA_CHECK_LAUNCH();
}

MAML_TRACE_SETTER(trace_set_bn)
