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

__device__ __forceinline__ float leaky(float y) { return y > 0.f ? y : LEAKY_SLOPE_F * y; }
__device__ __forceinline__ float slope_of(float y) { return y > 0.f ? 1.f : LEAKY_SLOPE_F; }

// mean and r = 1 / sqrt(var + eps) of m values from their fp64 sums st[0] = sum z, st[1] = sum z^2
__device__ __forceinline__ void norm_consts(const double* __restrict__ st, double m, float& mu, float& r) {
  const double mean = st[0] / m;
  double var = st[1] / m - mean * mean;
  if (var < 0.0) var = 0.0;
  mu = (float)mean;
  r = (float)(1.0 / sqrt(var + BN_EPS_D));
}

// per-channel constants from the fp64 sums (sum z, sum z^2)
__device__ __forceinline__ void chan_setup(const double* __restrict__ st, const float* __restrict__ gamma,
                                           const float* __restrict__ beta, double m, int F, float* s_mu, float* s_r,
                                           float* s_g, float* s_b) {
  const int tid = threadIdx.x;
  if (tid < F) {
    norm_consts(st + tid * 2, m, s_mu[tid], s_r[tid]);
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
// p[i] + p2[i]: a tangent that arrives as two addends; p2 may be null (one addend)
__device__ __forceinline__ float4 ld4_sum(const float* p, const float* p2, long long i) {
  float4 v = ld4(p + i);
  if (p2) { const float4 v2 = ld4(p2 + i); v.x += v2.x; v.y += v2.y; v.z += v2.z; v.w += v2.w; }
  return v;
}
// channel c of a quad; c is a constant at every use (the loops over channels are unrolled)
template <class V> __device__ __forceinline__ auto comp(const V& v, int c) { return c == 0 ? v.x : c == 1 ? v.y : c == 2 ? v.z : v.w; }
// f applied channel by channel to the quads v...: make_float4(f(v.x...), f(v.y...), f(v.z...), f(v.w...))
template <class F, class... V> __device__ __forceinline__ float4 map4(F f, const V&... v) {
  return make_float4(f(v.x...), f(v.y...), f(v.z...), f(v.w...));
}
__device__ __forceinline__ float4 mul4(const float4& a, const float4& b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
__device__ __forceinline__ float4 slope_of(const float4& y) { return make_float4(slope_of(y.x), slope_of(y.y), slope_of(y.z), slope_of(y.w)); }

// a_k for the run-time arg-max position k, as a select chain: indexing a register array with k would move it to local
// memory (STL / LDL in the middle of latency-bound kernels)
template <class T> __device__ __forceinline__ T select4(int k, T a0, T a1, T a2, T a3) { return k == 0 ? a0 : k == 1 ? a1 : k == 2 ? a2 : a3; }
template <class T> __device__ __forceinline__ T pick(const T (&v)[4], int k) { return select4(k, v[0], v[1], v[2], v[3]); }
// channel c of v[k]
__device__ __forceinline__ float pick(const float4 (&v)[4], int k, int c) {
  return select4(k, comp(v[0], c), comp(v[1], c), comp(v[2], c), comp(v[3], c));
}

// ------------------------------------------------------------------------------- per-element formulas
// Every kernel below computes these through the functions here, so the forward and the backward-type kernels agree by
// construction.

// zh = (z - mu) * r
__device__ __forceinline__ float4 bn_normalize(const float4& z, const float4& mu, const float4& r) {
  return map4([](float z, float mu, float r) { return (z - mu) * r; }, z, mu, r);
}

// y = gamma * zh + beta (one explicit fma) and act = leaky(y) at one window position
struct BnAct { float4 y, act; };
__device__ __forceinline__ BnAct bn_act(const float4& ga, const float4& zh, const float4& be) {
  BnAct v;
  v.y = map4([](float ga, float zh, float be) { return fmaf(ga, zh, be); }, ga, zh, be);
  v.act = map4([](float y) { return leaky(y); }, v.y);
  return v;
}

// The max-pool decision.  The positions k = 0..3 of a window are offered in order (k = 0 is always inside the image); per
// channel, a position replaces the maximum so far only if its act is strictly greater, so the first maximum wins, as in
// F.max_pool2d.  No mask is stored: every backward-type kernel recomputes the decision from zh through bn_act and this
// function, and so reaches the forward's decision.  The maximum carries the winner's y, position and p (a value of the
// caller's: the tangent of the pooled value).  A window starts from WinMax{} (arg = 0 for position 0).
struct WinMax { int4 arg; float4 p, y, act; };
__device__ __forceinline__ void keep_first_max(int k, const BnAct& v, WinMax& w, const float4& p = float4()) {
  if (k == 0) { w.act = v.act; w.y = v.y; w.p = p; }
  else {
    if (v.act.x > w.act.x) { w.act.x = v.act.x; w.y.x = v.y.x; w.p.x = p.x; w.arg.x = k; }
    if (v.act.y > w.act.y) { w.act.y = v.act.y; w.y.y = v.y.y; w.p.y = p.y; w.arg.y = k; }
    if (v.act.z > w.act.z) { w.act.z = v.act.z; w.y.z = v.y.z; w.p.z = p.z; w.arg.z = k; }
    if (v.act.w > w.act.w) { w.act.w = v.act.w; w.y.w = v.y.w; w.p.w = p.w; w.arg.w = k; }
  }
}

// tangent of act at one position: slope * gamma * zhdot; GB (gamma / beta carry tangents gd, bd):
// slope * (gamma zhdot + gd zh + bd).  Two formulas: the first is not the second with gd = bd = 0 (rounding).
template <bool GB>
__device__ __forceinline__ float4 act_tangent(const BnAct& v, const float4& ga, const float4& zhd, const float4& zh,
                                              const float4& gd = float4(), const float4& bd = float4()) {
  return map4([](float y, float ga, float zhd, float zh, float gd, float bd) {
    return GB ? slope_of(y) * (ga * zhd + fmaf(gd, zh, bd)) : slope_of(y) * ga * zhd;
  }, v.y, ga, zhd, zh, gd, bd);
}

// tangent of zh: zhdot = r * (zdot - mean(zdot) - zh * q), q = mean(zh * zdot)
__device__ __forceinline__ float4 bn_tan_normalize(const float4& zd, const float4& zh, const float4& r, const float4& md,
                                                   const float4& qq) {
  return map4([](float zd, float zh, float r, float md, float q) { return r * (zd - md - zh * q); }, zd, zh, r, md, qq);
}

// backward sums of a full window at its arg-max: S1 += dy, S2 += dy * zh (fp64), dy = dp * slope.  Returns dy.
__device__ __forceinline__ float4 bn_bwd_sums(const float4& dp, const float4& sl, const float4 (&zh)[4], const int4& arg,
                                              double (&s1)[4], double (&s2)[4]) {
  const float4 dy = mul4(dp, sl);
  s1[0] += dy.x; s2[0] += (double)dy.x * (double)pick(zh, arg.x, 0);
  s1[1] += dy.y; s2[1] += (double)dy.y * (double)pick(zh, arg.y, 1);
  s1[2] += dy.z; s2[2] += (double)dy.z * (double)pick(zh, arg.z, 2);
  s1[3] += dy.w; s2[3] += (double)dy.w * (double)pick(zh, arg.w, 3);
  return dy;
}

// tangent backward sums of a full window at its arg-max: T1 += dydot, T2 += dydot * zh + dy * zhdot (fp64), with
// dy = dp * slope, dydot = dpdot * slope and zhd_at(k, c) = zhdot of channel c at position k.  Returns dydot.
template <class ZhdAt>
__device__ __forceinline__ float4 bn_tan_bwd_sums(const float4& dp, const float4& dpd, const float4& sl, const float4 (&zh)[4],
                                                  const int4& arg, ZhdAt zhd_at, double (&s1)[4], double (&s2)[4]) {
  float dyd[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int k = comp(arg, c);
    const float zhk = pick(zh, k, c), zhdk = zhd_at(k, c);
    const float dy = comp(dp, c) * comp(sl, c);
    dyd[c] = comp(dpd, c) * comp(sl, c);
    s1[c] += dyd[c];
    s2[c] += (double)dyd[c] * (double)zhk + (double)dy * (double)zhdk;
  }
  return make_float4(dyd[0], dyd[1], dyd[2], dyd[3]);
}

// dz = r * gamma * (dy - S1/m - zh * S2/m) at window position k, rg = r * gamma, c1 / c2 = S1/m / S2/m; dy (the pooled
// gradient times the slope) reaches only the arg-max of a full window.  NO_DY: a position of a partial window,
// r * gamma * (-S1/m - zh * S2/m); its zero results can differ in sign from those of 0 - S1/m - ...
template <bool NO_DY = false>
__device__ __forceinline__ float4 bn_bwd_dz(const float4& rg, const float4& c1, const float4& zh, const float4& c2, int k = 0,
                                            const int4& arg = int4(), const float4& dy = float4(), bool full = true) {
  return map4([k, full](float rg, float c1, float zh, float c2, int arg, float dy) {
    return rg * ((NO_DY ? -c1 : (full && arg == k ? dy : 0.f) - c1) - zh * c2);
  }, rg, c1, zh, c2, arg, dy);
}

// dzdot = -r * q * dz + r * gamma * (dydot - T1/m - zhdot * S2/m - zh * T2/m) at window position k, rq = -r * q; dydot
// reaches only the arg-max of a full window
__device__ __forceinline__ float4 bn_tan_bwd_dz(const float4& rq, const float4& dz, const float4& rg, const float4& t1,
                                                const float4& zhd, const float4& c2, const float4& zh, const float4& t2, int k,
                                                const int4& arg, const float4& dyd, bool full = true) {
  return map4([k, full](float rq, float dz, float rg, float t1, float zhd, float c2, float zh, float t2, int arg, float dyd) {
    return rq * dz + rg * ((full && arg == k ? dyd : 0.f) - t1 - zhd * c2 - zh * t2);
  }, rq, dz, rg, t1, zhd, c2, zh, t2, arg, dyd);
}

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

// ------------------------------------------------------------------------------- per-window bodies
// One pooling window (wy, wx) of image img for this thread's channel quad, shared by the BatchNorm phases and the layer-norm
// kernels.  The constants (mu, r, gamma, the sums / m) are per channel for BatchNorm and per image for layer norm (gamma =
// 1); be_at(yy, xx) is beta at pixel (yy, xx): BatchNorm's per-channel quad at every position, layer norm's bias there.

// v at idx, and its TF32 split into the planes hi / lo (nullable) `toff` floats from their task's start
__device__ __forceinline__ void st4_out(float* p, float* hi, float* lo, long long toff, long long idx, float4 v) {
  st4(p + idx, v);
  if (hi) st4_split(hi + toff, lo + toff, idx, v);
}

// a full window of the backward-type kernels: loads zh at its four positions and recomputes the forward's pooling decision
template <class BeAt>
__device__ __forceinline__ void argmax_window(const float* __restrict__ zhp, const BnGeom& g, int img, int wy, int wx,
                                              const WinIter& it, const float4& ga, BeAt be_at, float4 (&zh)[4],
                                              long long (&idx)[4], int4& arg, float4& slope_at) {
  WinMax w{};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
    idx[k] = it.grid(g, img, yy, xx);
    zh[k] = ld4(zhp + idx[k]);
    keep_first_max(k, bn_act(ga, zh[k], be_at(yy, xx)), w);
  }
  arg = w.arg;
  slope_at = slope_of(w.y);
}

// forward: zh = (z - mu) * r in place, p = max-pool(leaky(gamma * zh + beta)) at a full window
template <class BeAt>
__device__ __forceinline__ void act_window(const WinIter& it, const BnGeom& g, int img, int wy, int wx, float* z, const float4& mu,
                                           const float4& r, const float4& ga, BeAt be_at, float* p, float* p_hi, float* p_lo,
                                           long long p_toff) {
  WinMax w{};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
    if (yy < g.h && xx < g.w) {
      const long long idx = it.grid(g, img, yy, xx);
      const float4 zh = bn_normalize(ld4(z + idx), mu, r);
      st4(z + idx, zh);
      keep_first_max(k, bn_act(ga, zh, be_at(yy, xx)), w);
    }
  }
  if (wy < g.ph && wx < g.pw) st4_out(p, p_hi, p_lo, p_toff, it.pooled(g, img, wy, wx), w.act);
}

// backward sums of a full window at its arg-max (partial windows add nothing): S1 += dy, S2 += dy * zh
template <class BeAt>
__device__ __forceinline__ void bwd_reduce_window(const WinIter& it, const BnGeom& g, int img, int wy, int wx, const float* zhp,
                                                  const float4& ga, BeAt be_at, const float* dp, double (&s1)[4], double (&s2)[4]) {
  if (wy >= g.ph || wx >= g.pw) return;
  float4 zh[4]; long long idx[4]; int4 arg; float4 sl;
  argmax_window(zhp, g, img, wy, wx, it, ga, be_at, zh, idx, arg, sl);
  bn_bwd_sums(ld4(dp + it.pooled(g, img, wy, wx)), sl, zh, arg, s1, s2);
}

// tangent backward sums of a full window at its arg-max: T1 += dydot, T2 += dydot * zh + dy * zhdot; dpdot = dpd (+ dpd2)
template <class BeAt>
__device__ __forceinline__ void bwd_tan_reduce_window(const WinIter& it, const BnGeom& g, int img, int wy, int wx, const float* zhp,
                                                      const float4& ga, BeAt be_at, const float* zhd, const float* dp,
                                                      const float* dpd, const float* dpd2, double (&s1)[4], double (&s2)[4]) {
  if (wy >= g.ph || wx >= g.pw) return;
  float4 zh[4]; long long idx[4]; int4 arg; float4 sl;
  argmax_window(zhp, g, img, wy, wx, it, ga, be_at, zh, idx, arg, sl);
  const long long pidx = it.pooled(g, img, wy, wx);
  const float4 d = ld4(dp + pidx);
  const float4 dd = ld4_sum(dpd, dpd2, pidx);
  bn_tan_bwd_sums(d, dd, sl, zh, arg, [&](int k, int c) { return zhd[pick(idx, k) + c]; }, s1, s2);
}

// dz = r * gamma * (dy - S1/m - zh * S2/m) at every position inside the image (dy != 0 only at the arg-max); rg = r * gamma,
// c1 = S1/m, c2 = S2/m
template <class BeAt>
__device__ __forceinline__ void bwd_apply_window(const WinIter& it, const BnGeom& g, int img, int wy, int wx, const float* zhp,
                                                 const float4& ga, BeAt be_at, const float* dp, const float4& rg, const float4& c1,
                                                 const float4& c2, float* dz, float* dz_hi, float* dz_lo, long long dz_toff) {
  const bool full = (wy < g.ph && wx < g.pw);
  if (full) {
    float4 zh[4]; long long idx[4]; int4 arg; float4 sl;
    argmax_window(zhp, g, img, wy, wx, it, ga, be_at, zh, idx, arg, sl);
    const float4 dyv = mul4(ld4(dp + it.pooled(g, img, wy, wx)), sl);
#pragma unroll
    for (int k = 0; k < 4; ++k) st4_out(dz, dz_hi, dz_lo, dz_toff, idx[k], bn_bwd_dz(rg, c1, zh[k], c2, k, arg, dyv));
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
      if (yy < g.h && xx < g.w) {
        const long long idx = it.grid(g, img, yy, xx);
        st4_out(dz, dz_hi, dz_lo, dz_toff, idx, bn_bwd_dz<true>(rg, c1, ld4(zhp + idx), c2));
      }
    }
  }
}

// ------------------------------------------------------------------------------- forward
__device__ __forceinline__ void bnact_phase(const BnActArgs& a, const BnGeom& g, int task, int cta, int ncta, const WinIter& it,
                                            const float* s_mu, const float* s_r, const float* s_g, const float* s_b) {
  if (it.lane >= it.WPB) return;
  const float4 mu = ld4s(s_mu, it.q), r = ld4s(s_r, it.q), ga = ld4s(s_g, it.q), be = ld4s(s_b, it.q);
  float* z = a.z + (long long)task * a.z_stride;
  float* p = a.p + (long long)task * a.p_stride;
  for (int wi = cta * it.WPB + it.lane; wi < it.NW; wi += ncta * it.WPB) {
    int img, wy, wx; it.window(wi, img, wy, wx);
    act_window(it, g, img, wy, wx, z, mu, r, ga, [&](int, int) { return be; }, p, a.p_hi, a.p_lo, (long long)task * a.p_stride);
  }
}

// PT (this kernel and the five streaming kernels below): gamma / beta per task (inner-loop gamma / beta: fast weights), task
// t's at gamma / beta + t * gbs.  gbs is a trailing kernel parameter, so the Bn*Args structs keep their layout.
template <bool PT>
__global__ void __launch_bounds__(256) bnact_kernel(BnActArgs a, long long gbs) {
  pdl_prologue(PT ? 43 : 6, a.tag);
  __shared__ float s_mu[64], s_r[64], s_g[64], s_b[64];
  const BnGeom g = a.g;
  const int task = blockIdx.y;
  const long long go = PT ? (long long)task * gbs : 0;
  chan_setup(a.stats + (long long)task * a.stats_stride, a.gamma + go, a.beta + go, (double)g.n * g.h * g.w, g.F, s_mu, s_r,
             s_g, s_b);
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

void launch_bnact(const BnActArgs& a, long long gb_stride, cudaStream_t st) {
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  int block; dim3 grid = bn_grid(a.g, a.tasks, &block);
  launch_pdl(gb_stride ? bnact_kernel<true> : bnact_kernel<false>, dim3(grid), dim3(block), (size_t)(0), st, tagged(a), gb_stride);
  CUDA_CHECK_LAUNCH();
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
  __shared__ double red[256 * 8];
  const int tid = threadIdx.x;
#pragma unroll
  for (int c = 0; c < 4; ++c) { red[tid * 8 + c * 2] = s1[c]; red[tid * 8 + c * 2 + 1] = s2[c]; }
  __syncthreads();
  double t = 0.0;
  if (tid < F * 2) {
    const int ch = tid >> 1, which = tid & 1;
    const int q = ch >> 2, comp = ch & 3;
    for (int l = 0; l < it.WPB; ++l) t += red[(l * it.F4 + q) * 8 + comp * 2 + which];
  }
  return t;
}
// CTA totals added to the statistics arena: one atomic per (channel, sum)
__device__ __forceinline__ void block_reduce_stats(double (&s1)[4], double (&s2)[4], const WinIter& it, double* stats, int F) {
  const double t = block_reduce_totals(s1, s2, it, F);
  if (threadIdx.x < F * 2) atomicAdd(&stats[threadIdx.x], t);
}
// CTA totals of a kernel that needs no cluster: publishes sums / m in shared memory and the raw sums in the statistics row
__device__ __forceinline__ void publish_totals(double t, int F, double m, float* s_a, float* s_b2, double* row) {
  const int tid = threadIdx.x;
  if (tid < F * 2) {
    ((tid & 1) ? s_b2 : s_a)[tid >> 1] = (float)(t / m);
    row[tid] = t;
  }
  __syncthreads();
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
    bwd_reduce_window(it, g, img, wy, wx, zhp, ga, [&](int, int) { return be; }, dp, s1, s2);
  }
}

template <bool PT>
__global__ void __launch_bounds__(256) bnbwd_reduce_kernel(BnBwdArgs a, long long gbs) {
  pdl_prologue(PT ? 44 : 7, a.tag);
  __shared__ float s_g[64], s_b[64];
  const BnGeom g = a.g;
  const int task = blockIdx.y;
  const long long go = PT ? (long long)task * gbs : 0;
  if (threadIdx.x < g.F) { s_g[threadIdx.x] = (a.gamma + go)[threadIdx.x]; s_b[threadIdx.x] = (a.beta + go)[threadIdx.x]; }
  __syncthreads();
  WinIter it(g);
  double s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  bnbwd_reduce_phase(a, g, task, blockIdx.x, gridDim.x, it, s_g, s_b, s1, s2);
  block_reduce_stats(s1, s2, it, a.stats_bwd + (long long)task * a.stats_bwd_stride, g.F);
}

static void launch_bnbwd_reduce(const BnBwdArgs& a, long long gb_stride, cudaStream_t st) {
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  int block; dim3 grid = bn_grid(a.g, a.tasks, &block);
  if ((int)grid.x > num_sms()) grid.x = num_sms();
  launch_pdl(gb_stride ? bnbwd_reduce_kernel<true> : bnbwd_reduce_kernel<false>, dim3(grid), dim3(block), (size_t)(0), st,
             tagged(a), gb_stride);
  CUDA_CHECK_LAUNCH();
}

// ------------------------------------------------------------------------------- backward: apply
// dz = r * gamma * (dy - S1/m - zh * S2/m)   at every valid position (dy != 0 only at the arg-max)
__device__ __forceinline__ void bnbwd_apply_phase(const BnBwdArgs& a, const BnGeom& g, int task, int cta, int ncta, const WinIter& it,
                                                  const float* s_r, const float* s_g, const float* s_b, const float* s_c1,
                                                  const float* s_c2) {
  if (it.lane >= it.WPB) return;
  const float4 r = ld4s(s_r, it.q), ga = ld4s(s_g, it.q), be = ld4s(s_b, it.q), c1 = ld4s(s_c1, it.q), c2 = ld4s(s_c2, it.q);
  const float4 rg = mul4(r, ga);
  const float* zhp = a.zh + (long long)task * a.zh_stride;
  const float* dp = a.dp + (long long)task * a.dp_stride;
  float* dz = a.dz + (long long)task * a.dz_stride;
  for (int wi = cta * it.WPB + it.lane; wi < it.NW; wi += ncta * it.WPB) {
    int img, wy, wx; it.window(wi, img, wy, wx);
    bwd_apply_window(it, g, img, wy, wx, zhp, ga, [&](int, int) { return be; }, dp, rg, c1, c2, dz, a.dz_hi, a.dz_lo,
                     (long long)task * a.dz_stride);
  }
}

template <bool PT>
__global__ void __launch_bounds__(256) bnbwd_apply_kernel(BnBwdArgs a, long long gbs) {
  pdl_prologue(PT ? 45 : 8, a.tag);
  __shared__ float s_mu[64], s_r[64], s_g[64], s_b[64], s_c1[64], s_c2[64];
  const BnGeom g = a.g;
  const int task = blockIdx.y;
  const double m = (double)g.n * g.h * g.w;
  const long long go = PT ? (long long)task * gbs : 0;
  chan_setup(a.stats_fwd + (long long)task * a.stats_fwd_stride, a.gamma + go, a.beta + go, m, g.F, s_mu, s_r, s_g, s_b);
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

static void launch_bnbwd_apply(const BnBwdArgs& a, long long gb_stride, cudaStream_t st) {
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  int block; dim3 grid = bn_grid(a.g, a.tasks, &block);
  launch_pdl(gb_stride ? bnbwd_apply_kernel<true> : bnbwd_apply_kernel<false>, dim3(grid), dim3(block), (size_t)(0), st,
             tagged(a), gb_stride);
  CUDA_CHECK_LAUNCH();
}

// BatchNorm backward of one block (reduce + apply), fused into one cluster kernel when the block is small and gamma / beta
// are shared: the cluster kernels (and the tail kernels) read shared gamma / beta only, so per-task ones (gb_stride != 0)
// always take the two streaming kernels
void launch_bnbwd(const BnBwdArgs& a, long long gb_stride, cudaStream_t st) {
  const int cl = gb_stride ? 0 : bn_fused_cluster(a.g);
  if (cl == 0) { launch_bnbwd_reduce(a, gb_stride, st); launch_bnbwd_apply(a, gb_stride, st); return; }
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  int block; bn_grid(a.g, a.tasks, &block);
  launch_cluster(bnbwd_fused_kernel, tagged(a), cl, a.tasks, block, st);
  CUDA_CHECK_LAUNCH();
}

// ------------------------------------------------------------------------------- tangent forward
// zhdot = r * (zdot - mean(zdot) - zh * mean(zh * zdot));  pdot = slope * gamma * zhdot at the arg-max.  go: the task's
// offset of gamma / beta
__device__ __forceinline__ void bnact_tan_setup(const BnActTanArgs& a, const BnGeom& g, int task, double m, float* s_mu, float* s_r,
                                                float* s_g, float* s_b, float* s_md, float* s_q, long long go = 0) {
  chan_setup(a.stats_fwd + (long long)task * a.stats_fwd_stride, a.gamma + go, a.beta + go, m, g.F, s_mu, s_r, s_g, s_b);
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
    WinMax w{};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
      if (yy < g.h && xx < g.w) {
        const long long idx = it.grid(g, img, yy, xx);
        const float4 zh = ld4(zhp + idx);
        const float4 zhd = bn_tan_normalize(ld4_sum(zd, zd2, idx), zh, r, md, qq);
        st4(zd + idx, zhd);
        const BnAct v = bn_act(ga, zh, be);
        keep_first_max(k, v, w, act_tangent<GB>(v, ga, zhd, zh, gd, bd));
      }
    }
    if (wy < g.ph && wx < g.pw) {
      const long long pidx = it.pooled(g, img, wy, wx);
      st4(pd + pidx, w.p);
      if (a.pdot_hi) st4_split(a.pdot_hi + (long long)task * a.pdot_stride, a.pdot_lo + (long long)task * a.pdot_stride, pidx, w.p);
    }
  }
}

// GB: gamma / beta carry tangents gdot / bdot, read like gamma / beta (the functional operator's forward mode; with PT, the
// inner loop's gamma / beta along u)
template <bool GB, bool PT>
__global__ void __launch_bounds__(256) bnact_tan_kernel(BnActTanArgs a, const float* gdot, const float* bdot, long long gbs) {
  pdl_prologue(PT ? 46 : GB ? 32 : 10, a.tag);
  __shared__ float s_mu[64], s_r[64], s_g[64], s_b[64], s_md[64], s_q[64], s_gd[64], s_bd[64];
  const BnGeom g = a.g;
  const int task = blockIdx.y;
  const long long go = PT ? (long long)task * gbs : 0;
  bnact_tan_setup(a, g, task, (double)g.n * g.h * g.w, s_mu, s_r, s_g, s_b, s_md, s_q, go);
  if (GB && threadIdx.x < g.F) { s_gd[threadIdx.x] = (gdot + go)[threadIdx.x]; s_bd[threadIdx.x] = (bdot + go)[threadIdx.x]; }
  __syncthreads();
  WinIter it(g);
  bnact_tan_phase<GB>(a, g, task, blockIdx.x, gridDim.x, it, s_r, s_g, s_b, s_md, s_q, s_gd, s_bd);
}

void launch_bnact_tan(const BnActTanArgs& a, const float* gdot, const float* bdot, long long gb_stride, cudaStream_t st) {
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  int block; dim3 grid = bn_grid(a.g, a.tasks, &block);
  const auto kernel = gb_stride ? bnact_tan_kernel<true, true> : gdot ? bnact_tan_kernel<true, false> : bnact_tan_kernel<false, false>;
  launch_pdl(kernel, dim3(grid), dim3(block), (size_t)(0), st, tagged(a), gdot, bdot, gb_stride);
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
  const float* dpd2 = a.dpdot2 ? a.dpdot2 + (long long)task * a.dpdot_stride : nullptr;
  for (int wi = cta * it.WPB + it.lane; wi < it.NW; wi += ncta * it.WPB) {
    int img, wy, wx; it.window(wi, img, wy, wx);
    bwd_tan_reduce_window(it, g, img, wy, wx, zhp, ga, [&](int, int) { return be; }, zhd, dp, dpd, dpd2, s1, s2);
  }
}

template <bool PT>
__global__ void __launch_bounds__(256) bnbwd_tan_reduce_kernel(BnBwdTanArgs a, long long gbs) {
  pdl_prologue(PT ? 47 : 11, a.tag);
  __shared__ float s_g[64], s_b[64];
  const BnGeom g = a.g;
  const int task = blockIdx.y;
  const long long go = PT ? (long long)task * gbs : 0;
  if (threadIdx.x < g.F) { s_g[threadIdx.x] = (a.gamma + go)[threadIdx.x]; s_b[threadIdx.x] = (a.beta + go)[threadIdx.x]; }
  __syncthreads();
  WinIter it(g);
  double s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  bnbwd_tan_reduce_phase(a, g, task, blockIdx.x, gridDim.x, it, s_g, s_b, s1, s2);
  block_reduce_stats(s1, s2, it, a.stats_tbwd + (long long)task * a.stats_tbwd_stride, g.F);
}

static void launch_bnbwd_tan_reduce(const BnBwdTanArgs& a, long long gb_stride, cudaStream_t st) {
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  int block; dim3 grid = bn_grid(a.g, a.tasks, &block);
  if ((int)grid.x > num_sms()) grid.x = num_sms();
  launch_pdl(gb_stride ? bnbwd_tan_reduce_kernel<true> : bnbwd_tan_reduce_kernel<false>, dim3(grid), dim3(block), (size_t)(0),
             st, tagged(a), gb_stride);
  CUDA_CHECK_LAUNCH();
}

// ------------------------------------------------------------------------------- tangent backward: apply
// bn_tan_bwd_dz plus the gamma-tangent term: dzdot = -r q dz + r gamma (dydot - T1/m - zhdot S2/m - zh T2/m)
//                                                 + r gdot (dy - S1/m - zh S2/m),   rgd = r * gdot, c1 = S1/m
// dy and dydot reach only the arg-max of a full window
__device__ __forceinline__ float4 bn_tan_bwd_dz_gd(const float4& rq, const float4& dz, const float4& rg, const float4& t1,
                                                   const float4& zhd, const float4& c2, const float4& zh, const float4& t2, int k,
                                                   const int4& arg, const float4& dyd, const float4& rgd, const float4& c1,
                                                   const float4& dy, bool full) {
  const float4 base = bn_tan_bwd_dz(rq, dz, rg, t1, zhd, c2, zh, t2, k, arg, dyd, full);
  return map4([k, full](float b, float rgd, float c1, float zh, float c2, int arg, float dy) {
    return b + rgd * (((full && arg == k) ? dy : 0.f) - c1 - zh * c2);
  }, base, rgd, c1, zh, c2, arg, dy);
}

// dzdot = -r*q*dz + r*gamma*(dydot - T1/m - zhdot*S2/m - zh*T2/m)
// GD (inner-loop gamma / beta, s_gd = gdot, s_c1 = S1/m): + r*gdot*(dy - S1/m - zh*S2/m), dy from the primal dp
template <bool GD = false>
__device__ __forceinline__ void bnbwd_tan_apply_phase(const BnBwdTanArgs& a, const BnGeom& g, int task, int cta, int ncta,
                                                      const WinIter& it, const float* s_r, const float* s_g, const float* s_b,
                                                      const float* s_q, const float* s_c2, const float* s_t1, const float* s_t2,
                                                      const float* s_gd = nullptr, const float* s_c1 = nullptr) {
  if (it.lane >= it.WPB) return;
  const float4 r = ld4s(s_r, it.q), ga = ld4s(s_g, it.q), be = ld4s(s_b, it.q);
  const float4 qq = ld4s(s_q, it.q), c2 = ld4s(s_c2, it.q), t1 = ld4s(s_t1, it.q), t2 = ld4s(s_t2, it.q);
  float4 c1 = make_float4(0.f, 0.f, 0.f, 0.f), rgd = c1;
  if constexpr (GD) { c1 = ld4s(s_c1, it.q); rgd = mul4(r, ld4s(s_gd, it.q)); }
  const float4 rg = mul4(r, ga);
  const float4 rq = make_float4(-r.x * qq.x, -r.y * qq.y, -r.z * qq.z, -r.w * qq.w);
  const float* zhp = a.zh + (long long)task * a.zh_stride;
  const float* zhd = a.zhdot + (long long)task * a.zhdot_stride;
  const float* dzp = a.dz + (long long)task * a.dz_stride;
  const float* dpp = a.dp + (long long)task * a.dp_stride;
  const float* dpd = a.dpdot + (long long)task * a.dpdot_stride;
  const float* dpd2 = a.dpdot2 ? a.dpdot2 + (long long)task * a.dpdot_stride : nullptr;
  float* dzd = a.dzdot + (long long)task * a.dzdot_stride;
  for (int wi = cta * it.WPB + it.lane; wi < it.NW; wi += ncta * it.WPB) {
    int img, wy, wx; it.window(wi, img, wy, wx);
    const bool full = (wy < g.ph && wx < g.pw);
    int4 arg = make_int4(-1, -1, -1, -1);
    float4 dyd = make_float4(0.f, 0.f, 0.f, 0.f), dy = dyd;
    if (full) {
      float4 zh[4]; long long idx[4]; float4 sl;
      argmax_window(zhp, g, img, wy, wx, it, ga, [&](int, int) { return be; }, zh, idx, arg, sl);
      const long long pidx = it.pooled(g, img, wy, wx);
      dyd = mul4(ld4_sum(dpd, dpd2, pidx), sl);
      if constexpr (GD) dy = mul4(ld4(dpp + pidx), sl);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
      if (yy < g.h && xx < g.w) {
        const long long idx = it.grid(g, img, yy, xx);
        const float4 zh = ld4(zhp + idx), zd = ld4(zhd + idx), dzv = ld4(dzp + idx);
        float4 o;
        if constexpr (GD) o = bn_tan_bwd_dz_gd(rq, dzv, rg, t1, zd, c2, zh, t2, k, arg, dyd, rgd, c1, dy, full);
        else o = bn_tan_bwd_dz(rq, dzv, rg, t1, zd, c2, zh, t2, k, arg, dyd);
        st4(dzd + idx, o);
        if (a.dzdot_hi) st4_split(a.dzdot_hi + (long long)task * a.dzdot_stride, a.dzdot_lo + (long long)task * a.dzdot_stride, idx, o);
      }
    }
  }
}

__device__ __forceinline__ void bnbwd_tan_setup(const BnBwdTanArgs& a, const BnGeom& g, int task, double m, float* s_mu, float* s_r,
                                                float* s_g, float* s_b, float* s_q, float* s_c2, long long go = 0) {
  chan_setup(a.stats_fwd + (long long)task * a.stats_fwd_stride, a.gamma + go, a.beta + go, m, g.F, s_mu, s_r, s_g, s_b);
  if (threadIdx.x < g.F) {
    const int c = threadIdx.x;
    s_q[c] = (float)((a.stats_tan + (long long)task * a.stats_tan_stride)[c * 2 + 1] / m);
    s_c2[c] = (float)((a.stats_bwd + (long long)task * a.stats_bwd_stride)[c * 2 + 1] / m);
  }
}

// PT: also the gamma-tangent term (bnbwd_tan_apply_phase<GD>), gdot read like gamma
template <bool PT>
__global__ void __launch_bounds__(256) bnbwd_tan_apply_kernel(BnBwdTanArgs a, const float* gdot, long long gbs) {
  pdl_prologue(PT ? 48 : 12, a.tag);
  __shared__ float s_mu[64], s_r[64], s_g[64], s_b[64], s_q[64], s_c2[64], s_t1[64], s_t2[64], s_gd[64], s_c1[64];
  const BnGeom g = a.g;
  const int task = blockIdx.y;
  const double m = (double)g.n * g.h * g.w;
  const long long go = PT ? (long long)task * gbs : 0;
  bnbwd_tan_setup(a, g, task, m, s_mu, s_r, s_g, s_b, s_q, s_c2, go);
  if (threadIdx.x < g.F) {
    const int c = threadIdx.x;
    const double* tb = a.stats_tbwd + (long long)task * a.stats_tbwd_stride;
    s_t1[c] = (float)(tb[c * 2] / m);
    s_t2[c] = (float)(tb[c * 2 + 1] / m);
    if (PT) {
      s_c1[c] = (float)((a.stats_bwd + (long long)task * a.stats_bwd_stride)[c * 2] / m);
      s_gd[c] = (gdot + go)[c];
    }
  }
  __syncthreads();
  WinIter it(g);
  bnbwd_tan_apply_phase<PT>(a, g, task, blockIdx.x, gridDim.x, it, s_r, s_g, s_b, s_q, s_c2, s_t1, s_t2, s_gd, s_c1);
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

static void launch_bnbwd_tan_apply(const BnBwdTanArgs& a, const float* gdot, long long gb_stride, cudaStream_t st) {
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  int block; dim3 grid = bn_grid(a.g, a.tasks, &block);
  launch_pdl(gb_stride ? bnbwd_tan_apply_kernel<true> : bnbwd_tan_apply_kernel<false>, dim3(grid), dim3(block), (size_t)(0), st,
             tagged(a), gdot, gb_stride);
  CUDA_CHECK_LAUNCH();
}

// per-task gamma / beta (gb_stride != 0) take the two streaming kernels, as in launch_bnbwd
void launch_bnbwd_tan(const BnBwdTanArgs& a, const float* gdot, long long gb_stride, cudaStream_t st) {
  const int cl = gb_stride ? 0 : bn_fused_cluster(a.g);
  if (cl == 0) { launch_bnbwd_tan_reduce(a, gb_stride, st); launch_bnbwd_tan_apply(a, gdot, gb_stride, st); return; }
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
  publish_totals(block_reduce_totals(s1, s2, it, g.F), g.F, m, s_c1, s_c2, ba.stats_bwd + (long long)task * ba.stats_bwd_stride);
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
  publish_totals(block_reduce_totals(s1, s2, it, g.F), g.F, m, s_t1, s_t2, ba.stats_tbwd + (long long)task * ba.stats_tbwd_stride);
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
    WinMax w{};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
      zh[i][k] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (yy < g.h && xx < g.w) {
        const long long idx = it.grid(g, img, yy, xx);
        const float4 zz = bn_normalize(ld4(z + idx), mu, r);
        st4(z + idx, zz);
        zh[i][k] = zz;
        keep_first_max(k, bn_act(ga, zz, be), w);
      }
    }
    arg[i] = w.arg;
    sl[i] = slope_of(w.y);
    full[i] = (wy < g.ph && wx < g.pw);
    if (full[i]) {
      const long long pidx = it.pooled(g, img, wy, wx);
      st4(pg + pidx, w.act);
      st4(s_f + pidx, w.act);                      // pb = 0 on the last block: pidx is the feature index img * D + ...
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
    dyv[i] = bn_bwd_sums(ld4(s_df + pidx), sl[i], zh[i], arg[i], s1, s2);
  }
  publish_totals(block_reduce_totals(s1, s2, it, g.F), g.F, m, s_c1, s_c2, ba.stats_bwd + (long long)task * ba.stats_bwd_stride);
  if (!worker) return;
  const float4 c1 = ld4s(s_c1, it.q), c2 = ld4s(s_c2, it.q);
  const float4 rg = mul4(r, ga);
  float* dz = ba.dz + (long long)task * ba.dz_stride;
#pragma unroll
  for (int i = 0; i < MAXI; ++i) {
    if (!have[i]) continue;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = 2 * wy_[i] + (k >> 1), xx = 2 * wx_[i] + (k & 1);
      if (yy < g.h && xx < g.w) {
        const long long idx = it.grid(g, img_[i], yy, xx);
        const float4 o = bn_bwd_dz(rg, c1, zh[i][k], c2, k, arg[i], dyv[i], full[i]);
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
    WinMax w{};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
      zh[i][k] = make_float4(0.f, 0.f, 0.f, 0.f);
      zhd[i][k] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (yy < g.h && xx < g.w) {
        const long long idx = it.grid(g, img, yy, xx);
        const float4 z = ld4(zhp + idx);
        const float4 d = bn_tan_normalize(ld4_sum(zd, zd2, idx), z, r, md, qq);
        st4(zd + idx, d);
        zh[i][k] = z; zhd[i][k] = d;
        const BnAct v = bn_act(ga, z, be);
        keep_first_max(k, v, w, act_tangent<false>(v, ga, d, z));
      }
    }
    arg[i] = w.arg;
    sl[i] = slope_of(w.y);
    if (full[i]) {
      st4(pdg + pidx, w.p);
      st4(s_fd + pidx, w.p);                       // pb = 0 on the last block: pidx is the feature index img * D + ...
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
    dydv[i] = bn_tan_bwd_sums(dprim[i], ld4(s_dfd + pidx), sl[i], zh[i], arg[i], [&](int k, int c) { return pick(zhd[i], k, c); },
                              s1, s2);
  }
  publish_totals(block_reduce_totals(s1, s2, it, g.F), g.F, m, s_t1, s_t2, ba.stats_tbwd + (long long)task * ba.stats_tbwd_stride);
  if (!worker) return;
  const float4 c2 = ld4s(s_c2, it.q), t1 = ld4s(s_t1, it.q), t2 = ld4s(s_t2, it.q);
  const float4 rg = mul4(r, ga);
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
        const float4 o = bn_tan_bwd_dz(rq, dzv, rg, t1, zhd[i][k], c2, zh[i][k], t2, k, arg[i], dydv[i], full[i]);
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

// ---------------------------------------------------------------------------------------------------------------
// Layer norm (reference MetaLayerNormLayer, meta_neural_network_architectures.py:261-322: F.layer_norm over the conv
// output [F, h, w] of each image, eps 1e-5, frozen all-ones weight, learnable bias [F, h, w]).  The statistics are per
// image, so a query image's output does not depend on the other images of the batch.  The per-element formulas are the
// BatchNorm ones above with gamma = 1 and per-image constants: bn_act(1, zh, b) = fmaf(1, zh, b) = zh + b exactly, and the
// pooling decision is keep_first_max's.  Every reduction is spread over several CTAs per image (grid (CTAs per image,
// images, tasks)); each CTA adds its two fp64 totals to the image's sums with one atomic each.  The bias gradient (sum over
// the images of dy at each position) runs one thread per (window, channel quad) over the images in order: deterministic.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 ones4() { return make_float4(1.f, 1.f, 1.f, 1.f); }
__device__ __forceinline__ float4 splat4(float v) { return make_float4(v, v, v, v); }

__device__ __forceinline__ const double* ln_st(const double* base, long long stride, int task, int img) {
  return base + (long long)task * stride + 2LL * img;
}
// the layer-norm bias of channel quad q at pixel (yy, xx): [F][h][w]
__device__ __forceinline__ float4 ln_bias4(const float* b, const BnGeom& g, int q, int yy, int xx) {
  const long long hw = (long long)g.h * g.w, o = (long long)(q * 4) * hw + (long long)yy * g.w + xx;
  return make_float4(b[o], b[o + hw], b[o + 2 * hw], b[o + 3 * hw]);
}
// CTA totals of (s1, s2) added to one image's sums (fixed order inside the CTA, one fp64 atomic per sum)
__device__ __forceinline__ void ln_block_add(double s1, double s2, double* dst) {
  __shared__ double red[2][32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
  const int w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  if ((threadIdx.x & 31) == 0) { red[0][w] = s1; red[1][w] = s2; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t1 = 0.0, t2 = 0.0;
    for (int k = 0; k < nw; ++k) { t1 += red[0][k]; t2 += red[1][k]; }
    atomicAdd(dst, t1);
    atomicAdd(dst + 1, t2);
  }
}
// Every per-image kernel below runs the windows of image blockIdx.y: wi = blockIdx.x * WPB + lane, stride gridDim.x * WPB.

// sums of one image: primal (sum z, sum z^2); tangent (sum zdot, sum zh * zdot) with zdot = z + z2
template <bool TAN>
__global__ void __launch_bounds__(256) ln_stats_kernel(LnArgs a) {
  pdl_prologue(TAN ? 34 : 33, a.tag);
  const BnGeom g = a.g;
  const int img = blockIdx.y, task = blockIdx.z;
  WinIter it(g);
  double s1 = 0.0, s2 = 0.0;
  if (it.lane < it.WPB) {
    const float* z = a.z + (long long)task * a.z_stride;
    const float* z2 = a.z2 ? a.z2 + (long long)task * a.z_stride : nullptr;
    const float* zhp = TAN ? a.zh + (long long)task * a.zh_stride : nullptr;
    for (int wi = blockIdx.x * it.WPB + it.lane; wi < it.hc * it.wc; wi += gridDim.x * it.WPB) {
      const int wy = wi / it.wc, wx = wi - wy * it.wc;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
        if (yy < g.h && xx < g.w) {
          const long long idx = it.grid(g, img, yy, xx);
          const float4 v = TAN ? ld4_sum(z, z2, idx) : ld4(z + idx);
          const float4 w = TAN ? ld4(zhp + idx) : v;
#pragma unroll
          for (int c = 0; c < 4; ++c) { s1 += (double)comp(v, c); s2 += (double)comp(v, c) * (double)comp(w, c); }
        }
      }
    }
  }
  ln_block_add(s1, s2, a.st_out + (long long)task * a.st_stride + 2LL * img);
}

// primal: zh = (z - mu) r in place, y = zh + b, p = max-pool(leaky(y)).  Tangent (z = zdot):
// zhdot = r (zdot - mean zdot - zh mean(zh zdot)) in place, pdot = slope * ydot at the arg-max, ydot = zhdot (+ bdot with
// BDOT: a bias tangent, read like the bias; b enters after the normalisation, so the statistics and zhdot do not see it).
template <bool TAN, bool BDOT = false>
__global__ void __launch_bounds__(256) ln_act_kernel(LnArgs a) {
  pdl_prologue(TAN ? 36 : 35, a.tag);
  const BnGeom g = a.g;
  const int img = blockIdx.y, task = blockIdx.z;
  const double m = (double)g.F * g.h * g.w;
  WinIter it(g);
  if (it.lane >= it.WPB) return;
  float mu, r;
  norm_consts(ln_st(a.st_fwd, a.st_stride, task, img), m, mu, r);
  float md = 0.f, qq = 0.f;
  if (TAN) {
    const double* stt = ln_st(a.st_tan, a.st_stride, task, img);
    md = (float)(stt[0] / m); qq = (float)(stt[1] / m);
  }
  float* z = a.z + (long long)task * a.z_stride;
  const float* z2 = a.z2 ? a.z2 + (long long)task * a.z_stride : nullptr;
  const float* zhp = TAN ? a.zh + (long long)task * a.zh_stride : nullptr;
  const float* bd = BDOT ? a.bdot + (long long)task * a.bdot_stride : nullptr;
  float* p = a.out + (long long)task * a.out_stride;
  const long long toff = (long long)task * a.out_stride;
  for (int wi = blockIdx.x * it.WPB + it.lane; wi < it.hc * it.wc; wi += gridDim.x * it.WPB) {
    const int wy = wi / it.wc, wx = wi - wy * it.wc;
    if (!TAN) {
      act_window(it, g, img, wy, wx, z, splat4(mu), splat4(r), ones4(), [&](int yy, int xx) { return ln_bias4(a.bias, g, it.q, yy, xx); },
                 p, a.out_hi, a.out_lo, toff);
      continue;
    }
    // the tangent, like bnact_tan_phase (whose code is kept apart: sharing it changes the BatchNorm kernels' SASS)
    WinMax w{};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
      if (yy < g.h && xx < g.w) {
        const long long idx = it.grid(g, img, yy, xx);
        const float4 zh = ld4(zhp + idx);
        const float4 zhd = bn_tan_normalize(ld4_sum(z, z2, idx), zh, splat4(r), splat4(md), splat4(qq));
        st4(z + idx, zhd);
        const BnAct v = bn_act(ones4(), zh, ln_bias4(a.bias, g, it.q, yy, xx));
        keep_first_max(k, v, w, act_tangent<BDOT>(v, ones4(), zhd, zh, float4(), BDOT ? ln_bias4(bd, g, it.q, yy, xx) : float4()));
      }
    }
    if (wy < g.ph && wx < g.pw) st4_out(p, a.out_hi, a.out_lo, toff, it.pooled(g, img, wy, wx), w.p);
  }
}

// per-image backward sums: primal (S1 = sum dy, S2 = sum dy zh); tangent (T1 = sum dydot, T2 = sum dydot zh + dy zhdot)
template <bool TAN>
__global__ void __launch_bounds__(256) ln_bwd_reduce_kernel(LnArgs a) {
  pdl_prologue(TAN ? 38 : 37, a.tag);
  const BnGeom g = a.g;
  const int img = blockIdx.y, task = blockIdx.z;
  WinIter it(g);
  double s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  if (it.lane < it.WPB) {
    const float* zhp = a.zh + (long long)task * a.zh_stride;
    const float* dp = a.dp + (long long)task * a.dp_stride;
    const auto be_at = [&](int yy, int xx) { return ln_bias4(a.bias, g, it.q, yy, xx); };
    for (int wi = blockIdx.x * it.WPB + it.lane; wi < it.hc * it.wc; wi += gridDim.x * it.WPB) {
      const int wy = wi / it.wc, wx = wi - wy * it.wc;
      if constexpr (TAN)
        bwd_tan_reduce_window(it, g, img, wy, wx, zhp, ones4(), be_at, a.zhd + (long long)task * a.zhd_stride, dp,
                              a.dpd + (long long)task * a.dpd_stride, a.dpd2 ? a.dpd2 + (long long)task * a.dpd_stride : nullptr,
                              s1, s2);
      else
        bwd_reduce_window(it, g, img, wy, wx, zhp, ones4(), be_at, dp, s1, s2);
    }
  }
  ln_block_add(s1[0] + s1[1] + s1[2] + s1[3], s2[0] + s2[1] + s2[2] + s2[3],
               a.st_out + (long long)task * a.st_stride + 2LL * img);
}

// primal: dz = r (dy - S1/m - zh S2/m); tangent: dzdot = -r q dz + r (dydot - T1/m - zhdot S2/m - zh T2/m)
template <bool TAN>
__global__ void __launch_bounds__(256) ln_bwd_apply_kernel(LnArgs a) {
  pdl_prologue(TAN ? 40 : 39, a.tag);
  const BnGeom g = a.g;
  const int img = blockIdx.y, task = blockIdx.z;
  const double m = (double)g.F * g.h * g.w;
  WinIter it(g);
  if (it.lane >= it.WPB) return;
  float mu, r;
  norm_consts(ln_st(a.st_fwd, a.st_stride, task, img), m, mu, r);
  // this pass's sums (primal S1, S2; tangent T1, T2) are in st_out; the tangent also reads the primal S2 and q
  const double* sc = ln_st(a.st_out, a.st_stride, task, img);
  const float4 rr = splat4(r);
  float4 c1 = splat4((float)(sc[0] / m)), c2 = splat4((float)(sc[1] / m)), rq = float4(), t1 = float4(), t2 = float4();
  if (TAN) {
    t1 = c1; t2 = c2;
    c2 = splat4((float)(ln_st(a.st_bwd, a.st_stride, task, img)[1] / m));
    rq = splat4(-r * (float)(ln_st(a.st_tan, a.st_stride, task, img)[1] / m));
  }
  const float* zhp = a.zh + (long long)task * a.zh_stride;
  float* dz = a.out + (long long)task * a.out_stride;
  const long long toff = (long long)task * a.out_stride;
  const auto be_at = [&](int yy, int xx) { return ln_bias4(a.bias, g, it.q, yy, xx); };
  for (int wi = blockIdx.x * it.WPB + it.lane; wi < it.hc * it.wc; wi += gridDim.x * it.WPB) {
    const int wy = wi / it.wc, wx = wi - wy * it.wc;
    if (!TAN) {
      bwd_apply_window(it, g, img, wy, wx, zhp, ones4(), be_at, a.dp + (long long)task * a.dp_stride, rr, c1, c2, dz, a.out_hi,
                       a.out_lo, toff);
      continue;
    }
    // the tangent, like bnbwd_tan_apply_phase (whose code is kept apart: sharing it changes the BatchNorm kernels' SASS)
    int4 arg = make_int4(-1, -1, -1, -1);
    float4 dy = float4();
    if (wy < g.ph && wx < g.pw) {
      float4 zh[4]; long long idx[4]; float4 sl;
      argmax_window(zhp, g, img, wy, wx, it, ones4(), be_at, zh, idx, arg, sl);
      dy = mul4(ld4_sum(a.dpd + (long long)task * a.dpd_stride, a.dpd2 ? a.dpd2 + (long long)task * a.dpd_stride : nullptr,
                        it.pooled(g, img, wy, wx)), sl);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
      if (yy < g.h && xx < g.w) {
        const long long idx = it.grid(g, img, yy, xx);
        st4_out(dz, a.out_hi, a.out_lo, toff, idx,
                bn_tan_bwd_dz(rq, ld4(a.dz + (long long)task * a.dz_stride + idx), rr, t1, ld4(a.zhd + (long long)task * a.zhd_stride + idx),
                              c2, ld4(zhp + idx), t2, k, arg, dy));
      }
    }
  }
}

// bias gradient of one pass: db[c][y][x] = sum over the images (in order) of dy (tangent: dydot) at (c, y, x); dy reaches
// only the arg-max of a full window.  One thread per (window, channel quad); grid (window groups, tasks).
template <bool TAN>
__global__ void __launch_bounds__(256) ln_bias_grad_kernel(LnArgs a) {
  pdl_prologue(TAN ? 42 : 41, a.tag);
  const BnGeom g = a.g;
  const int task = blockIdx.y;
  WinIter it(g);
  const int wi = blockIdx.x * it.WPB + it.lane;
  if (it.lane >= it.WPB || wi >= it.hc * it.wc) return;
  const int wy = wi / it.wc, wx = wi - wy * it.wc;
  float4 acc[4] = {float4(), float4(), float4(), float4()};
  if (wy < g.ph && wx < g.pw) {
    const float* zhp = a.zh + (long long)task * a.zh_stride;
    const float* src = TAN ? a.dpd + (long long)task * a.dpd_stride : a.dp + (long long)task * a.dp_stride;
    const float* src2 = TAN && a.dpd2 ? a.dpd2 + (long long)task * a.dpd_stride : nullptr;
    for (int img = 0; img < g.n; ++img) {
      float4 zh[4]; long long idx[4]; int4 arg; float4 sl;
      argmax_window(zhp, g, img, wy, wx, it, ones4(), [&](int yy, int xx) { return ln_bias4(a.bias, g, it.q, yy, xx); }, zh, idx,
                    arg, sl);
      const float4 dy = mul4(ld4_sum(src, src2, it.pooled(g, img, wy, wx)), sl);
#pragma unroll
      for (int k = 0; k < 4; ++k)
        acc[k] = map4([k](float s, int ar, float d) { return ar == k ? s + d : s; }, acc[k], arg, dy);
    }
  }
  float* db = a.db + (long long)task * a.db_stride;
  const long long hw = (long long)g.h * g.w;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int yy = 2 * wy + (k >> 1), xx = 2 * wx + (k & 1);
    if (yy < g.h && xx < g.w) {
      const long long o = (long long)(it.q * 4) * hw + (long long)yy * g.w + xx;
#pragma unroll
      for (int c = 0; c < 4; ++c) db[o + c * hw] = comp(acc[k], c);
    }
  }
}

// grid of the per-image kernels: (CTAs per image, images, tasks), at most about 4 CTAs per SM in all
static inline dim3 ln_grid(const BnGeom& g, int tasks, int* block) {
  const WinGeom wg = win_geom(g);
  *block = wg.wpb * (g.F / 4);
  const int per_img = ((g.h + 1) / 2) * ((g.w + 1) / 2);
  int bx = (per_img + wg.wpb - 1) / wg.wpb;
  const int cap = std::max(1, 4 * num_sms() / std::max(1, g.n * tasks));
  if (bx > cap) bx = cap;
  return dim3(bx, g.n, tasks);
}

template <class K>
static void ln_launch(K kernel, const LnArgs& a, cudaStream_t st) {
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  int block; const dim3 grid = ln_grid(a.g, a.tasks, &block);
  launch_pdl(kernel, grid, dim3(block), (size_t)(0), st, tagged(a));
  CUDA_CHECK_LAUNCH();
}

void launch_ln_stats(const LnArgs& a, bool tan, cudaStream_t st) { ln_launch(tan ? ln_stats_kernel<true> : ln_stats_kernel<false>, a, st); }
void launch_ln_act(const LnArgs& a, bool tan, cudaStream_t st) {
  ln_launch(!tan ? ln_act_kernel<false> : a.bdot ? ln_act_kernel<true, true> : ln_act_kernel<true>, a, st);
}
void launch_ln_bwd(const LnArgs& a, bool tan, cudaStream_t st) {
  ln_launch(tan ? ln_bwd_reduce_kernel<true> : ln_bwd_reduce_kernel<false>, a, st);
  ln_launch(tan ? ln_bwd_apply_kernel<true> : ln_bwd_apply_kernel<false>, a, st);
}
void launch_ln_bias_grad(const LnArgs& a, bool tan, cudaStream_t st) {
  ProfScope prof_scope__(PROF_BN, 0.0, st);
  const WinGeom wg = win_geom(a.g);
  const int per_img = ((a.g.h + 1) / 2) * ((a.g.w + 1) / 2);
  const dim3 grid((per_img + wg.wpb - 1) / wg.wpb, a.tasks);
  launch_pdl(tan ? ln_bias_grad_kernel<true> : ln_bias_grad_kernel<false>, grid, dim3(wg.wpb * (a.g.F / 4)), (size_t)(0), st, tagged(a));
  CUDA_CHECK_LAUNCH();
}
