// CUDA-core (fp32 FFMA) shifted-row GEMM kernels for the 3x3 / pad-1 convolutions of the
// MAML backbone: forward conv, tangent conv (two operand pairs), dgrad, wgrad, and the small-K
// first-block variants.  Restates (for the conv part) reference
// meta_neural_network_architectures.py:89-97 (F.conv2d) and its autograd derivatives
// (convolution_backward / double backward) -- see SURVEY.md appendix A1-A3.
//
// These kernels are the exact-fp32 path: used for the first block (K = 9*C_in is 9 or 27) and
// for shapes the wgmma 3xTF32 kernel (kernels_tc.cu) does not cover.
#include <algorithm>
#include "common.cuh"

long long g_launch_counter = 0;
long long g_launch_base = 0;
int g_trace_flag = 0;

__device__ __forceinline__ int tap_shift(int tap, int gw) { return (tap / 3 - 1) * gw + (tap % 3 - 1); }

__device__ __forceinline__ bool row_valid(int row, int rows, int G, int gw, int h, int w) {
  if (row >= rows) return false;
  int rr = row % G;
  int yy = rr / gw;
  int xx = rr - yy * gw;
  return yy >= 1 && yy <= h && xx >= 1 && xx <= w;
}

// ---------------------------------------------------------------------------------------------
// shared epilogue: + bias, store, and (optionally) per-channel batch statistics in fp64
//   CONV_FWD_STATS: (sum z, sum z^2)            -> BatchNorm batch mean / biased variance
//   CONV_TAN_STATS: (sum zdot, sum zh * zdot)   -> tangent of the BatchNorm statistics
// thread (ty, tx) owns rows j0 + ty*4 .. +3 and columns tx*FN .. +FN-1
// ---------------------------------------------------------------------------------------------
template <int FN, int R = 4>
__device__ __forceinline__ void conv_epilogue(float (&acc)[R][FN], int j0, int rows, int gw, int G, int h, int w,
                                              int mode, const float* __restrict__ bias, float* __restrict__ out,
                                              const float* __restrict__ zh, double* __restrict__ stats,
                                              double* sred) {
  constexpr int NC = 16 * FN;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  float bv[FN];
#pragma unroll
  for (int jn = 0; jn < FN; ++jn) bv[jn] = bias ? bias[tx * FN + jn] : 0.f;
  double s1[FN], s2[FN];
#pragma unroll
  for (int jn = 0; jn < FN; ++jn) { s1[jn] = 0.0; s2[jn] = 0.0; }
#pragma unroll
  for (int i = 0; i < R; ++i) {
    const int row = j0 + ty * R + i;
    if (row < rows) {
      const long long base = (long long)row * NC + tx * FN;
      const bool valid = (mode != CONV_PLAIN) && row_valid(row, rows, G, gw, h, w);
#pragma unroll
      for (int jn = 0; jn < FN; ++jn) {
        const float v = acc[i][jn] + bv[jn];
        out[base + jn] = v;
        if (valid) {
          if (mode == CONV_FWD_STATS) {
            s1[jn] += (double)v;
            s2[jn] += (double)v * (double)v;
          } else {
            const float zv = zh[base + jn];
            s1[jn] += (double)v;
            s2[jn] += (double)zv * (double)v;
          }
        }
      }
    }
  }
  if (mode != CONV_PLAIN) {
    const int warp = tid >> 5;
#pragma unroll
    for (int jn = 0; jn < FN; ++jn) {
      s1[jn] += __shfl_xor_sync(0xffffffffu, s1[jn], 16);
      s2[jn] += __shfl_xor_sync(0xffffffffu, s2[jn], 16);
    }
    if ((tid & 16) == 0) {
#pragma unroll
      for (int jn = 0; jn < FN; ++jn) {
        sred[(warp * NC + tx * FN + jn) * 2 + 0] = s1[jn];
        sred[(warp * NC + tx * FN + jn) * 2 + 1] = s2[jn];
      }
    }
    __syncthreads();
    for (int c = tid; c < NC * 2; c += 256) {
      double t = 0.0;
#pragma unroll
      for (int wq = 0; wq < 8; ++wq) t += sred[wq * NC * 2 + c];
      atomicAdd(&stats[c], t);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// generic shifted-row GEMM:  out[j, col] = sum_src sum_tap sum_k A_src[j +/- s_tap, k] * W_src[tap, k, col]
// CTA tile 64 rows x NC columns, 256 threads, 4 x FN micro-tile, K step 16, register prefetch.
// ---------------------------------------------------------------------------------------------
template <int FN>
__global__ void __launch_bounds__(256) conv_rows_kernel(ConvArgs a) {
  pdl_prologue(1, a.tag);
  constexpr int NC = 16 * FN;
  __shared__ __align__(16) float As[16][68];
  __shared__ __align__(16) float Ws[16][NC];
  __shared__ double sred[8 * NC * 2];
  const int task = blockIdx.y;
  const int j0 = blockIdx.x * 64;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;

  float acc[4][FN];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int jn = 0; jn < FN; ++jn) acc[i][jn] = 0.f;

  const int it0 = 9 * (a.src[0].kc >> 4);
  const int nit = it0 + (a.nsrc > 1 ? 9 * (a.src[1].kc >> 4) : 0);

  float4 ra = make_float4(0.f, 0.f, 0.f, 0.f), rw = make_float4(0.f, 0.f, 0.f, 0.f);
  int cur_wt = 0;

  auto fetch = [&](int it) {
    const int s = (it < it0) ? 0 : 1;
    const ConvSrc& src = a.src[s];
    const int local = (s == 0) ? it : it - it0;
    const int kch = src.kc >> 4;
    const int tap = local / kch;
    const int c0 = (local - tap * kch) << 4;
    const int sh = src.sign * tap_shift(tap, a.gw);
    {
      const int row = tid >> 2, cq = tid & 3;
      const int jr = j0 + row;
      if (jr < a.rows) {
        const float* p = src.A + (long long)task * src.a_stride + (long long)(jr + sh) * src.kc + c0 + cq * 4;
        ra = *reinterpret_cast<const float4*>(p);
      } else {
        ra = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    cur_wt = src.wt;
    if (tid < 4 * NC) {
      const float* wb = src.W + (long long)task * src.w_stride;
      if (src.wt == 0) {
        rw = *reinterpret_cast<const float4*>(wb + (long long)(tap * src.kc + c0) * NC + tid * 4);
      } else {
        const int col = tid >> 2, kq = tid & 3;
        rw = *reinterpret_cast<const float4*>(wb + (long long)(tap * NC + col) * src.kc + c0 + kq * 4);
      }
    }
  };

  fetch(0);
  for (int it = 0; it < nit; ++it) {
    {
      const int row = tid >> 2, cq = tid & 3;
      As[cq * 4 + 0][row] = ra.x; As[cq * 4 + 1][row] = ra.y; As[cq * 4 + 2][row] = ra.z; As[cq * 4 + 3][row] = ra.w;
      if (tid < 4 * NC) {
        if (cur_wt == 0) {
          const int k = (tid * 4) / NC, col = (tid * 4) - k * NC;
          *reinterpret_cast<float4*>(&Ws[k][col]) = rw;
        } else {
          const int col = tid >> 2, kq = tid & 3;
          Ws[kq * 4 + 0][col] = rw.x; Ws[kq * 4 + 1][col] = rw.y; Ws[kq * 4 + 2][col] = rw.z; Ws[kq * 4 + 3][col] = rw.w;
        }
      }
    }
    __syncthreads();
    if (it + 1 < nit) fetch(it + 1);
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 a4 = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      float b[FN];
#pragma unroll
      for (int jn = 0; jn < FN; ++jn) b[jn] = Ws[k][tx * FN + jn];
#pragma unroll
      for (int jn = 0; jn < FN; ++jn) {
        acc[0][jn] = fmaf(a4.x, b[jn], acc[0][jn]);
        acc[1][jn] = fmaf(a4.y, b[jn], acc[1][jn]);
        acc[2][jn] = fmaf(a4.z, b[jn], acc[2][jn]);
        acc[3][jn] = fmaf(a4.w, b[jn], acc[3][jn]);
      }
    }
    __syncthreads();
  }

  conv_epilogue<FN>(acc, j0, a.rows, a.gw, a.G, a.h, a.w, a.mode,
                    a.bias ? a.bias + (long long)task * a.bias_stride : nullptr,
                    a.out + (long long)task * a.out_stride,
                    a.zh ? a.zh + (long long)task * a.zh_stride : nullptr,
                    a.stats ? a.stats + (long long)task * a.stats_stride : nullptr, sred);
}

void launch_conv_rows(const ConvArgs& a, cudaStream_t st) {
  ProfScope prof_scope__(PROF_CONV, a.alg_flops, st);
  dim3 grid((a.rows + 63) / 64, a.tasks);
  switch (a.ncols / 16) {
    case 1: launch_pdl(conv_rows_kernel<1>, dim3(grid), dim3(256), (size_t)(0), st, tagged(a)); break;
    case 2: launch_pdl(conv_rows_kernel<2>, dim3(grid), dim3(256), (size_t)(0), st, tagged(a)); break;
    case 3: launch_pdl(conv_rows_kernel<3>, dim3(grid), dim3(256), (size_t)(0), st, tagged(a)); break;
    default: launch_pdl(conv_rows_kernel<4>, dim3(grid), dim3(256), (size_t)(0), st, tagged(a)); break;
  }
  CUDA_CHECK_LAUNCH();
}

// ---------------------------------------------------------------------------------------------
// first block: K = 9 * C0 (9 or 27) -- all weights and the image window live in shared memory
// ---------------------------------------------------------------------------------------------
template <int FN>
__global__ void __launch_bounds__(256) conv0_kernel(Conv0Args a) {
  pdl_prologue(2, a.tag);
  constexpr int NC = 16 * FN;
  extern __shared__ float sm0[];
  __shared__ double sred[8 * NC * 2];
  const int task = blockIdx.y;
  const int j0 = blockIdx.x * 64;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int c0 = a.c0;
  float* Ws = sm0;                       // [9*c0][NC]
  float* xs = sm0 + 9 * c0 * NC;         // [(64 + 2*(gw+1))][c0]
  const int halo = a.gw + 1;
  const int wrows = 64 + 2 * halo;
  const float* W = a.W + (long long)task * a.w_stride;
  for (int i = tid; i < 9 * c0 * NC; i += 256) Ws[i] = W[i];
  const float* X = a.X + (long long)task * a.x_stride;
  const int guard = a.gw + 2;
  for (int i = tid; i < wrows * c0; i += 256) {
    const int r = j0 - halo + i / c0;
    float v = 0.f;
    if (r >= -guard && r < a.rows + guard) v = X[(long long)(j0 - halo) * c0 + i];
    xs[i] = v;
  }
  __syncthreads();

  float acc[4][FN];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int jn = 0; jn < FN; ++jn) acc[i][jn] = 0.f;

  for (int tap = 0; tap < 9; ++tap) {
    const int sh = tap_shift(tap, a.gw) + halo;
    for (int c = 0; c < c0; ++c) {
      float b[FN];
#pragma unroll
      for (int jn = 0; jn < FN; ++jn) b[jn] = Ws[(tap * c0 + c) * NC + tx * FN + jn];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float av = xs[(ty * 4 + i + sh) * c0 + c];
#pragma unroll
        for (int jn = 0; jn < FN; ++jn) acc[i][jn] = fmaf(av, b[jn], acc[i][jn]);
      }
    }
  }
  conv_epilogue<FN>(acc, j0, a.rows, a.gw, a.G, a.h, a.w, a.mode,
                    a.bias ? a.bias + (long long)task * a.bias_stride : nullptr,
                    a.out + (long long)task * a.out_stride,
                    a.zh ? a.zh + (long long)task * a.zh_stride : nullptr,
                    a.stats ? a.stats + (long long)task * a.stats_stride : nullptr, sred);
}

// Register-blocked first-block conv (C0 = 1 or 3): a thread owns 8 CONSECUTIVE grid rows x FN columns.  For a filter row
// ky the inputs of those 8 rows and the three kx taps are 10 consecutive grid positions: they are read once into
// registers (10 * C0 broadcast loads) and feed 8 x 3 x C0 x FN FMAs, the weights of the row come as 3 * C0 vector loads
// -- ~4 FMAs per shared-memory load instead of 12 per 7 in conv0_kernel, 128 rows per CTA instead of 64.
// Measured on Mini-ImageNet target passes (75 images of 84x84x3 -> 48 channels per task): see DESIGN.md.
template <int FN, int C0>
__global__ void __launch_bounds__(256) conv0_rb_kernel(Conv0Args a, int tiles) {
  pdl_prologue(2, a.tag);
  constexpr int NC = 16 * FN, R = 8, ROWS = 16 * R;
  extern __shared__ float sm0[];
  __shared__ double sred[8 * NC * 2];
  const int task = blockIdx.y;
  const int j00 = blockIdx.x * ROWS * tiles;         // this CTA covers `tiles` consecutive 128-row tiles: weights, the input
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;   // window and the statistics reduction are paid once
  float* Ws = sm0;                       // [9*C0][NC]
  float* xs = sm0 + 9 * C0 * NC;         // [(ROWS*tiles + 2*(gw+1))][C0]
  const int halo = a.gw + 1;
  const int wrows = ROWS * tiles + 2 * halo;
  const float* W = a.W + (long long)task * a.w_stride;
  for (int i = tid; i < 9 * C0 * NC; i += 256) Ws[i] = W[i];
  const float* X = a.X + (long long)task * a.x_stride;
  const int guard = a.gw + 2;
  for (int i = tid; i < wrows * C0; i += 256) {
    const int r = j00 - halo + i / C0;
    float v = 0.f;
    if (r >= -guard && r < a.rows + guard) v = X[(long long)(j00 - halo) * C0 + i];
    xs[i] = v;
  }
  float bv[FN];
  {
    const float* bias = a.bias ? a.bias + (long long)task * a.bias_stride : nullptr;
#pragma unroll
    for (int jn = 0; jn < FN; ++jn) bv[jn] = bias ? bias[tx * FN + jn] : 0.f;
  }
  double s1[FN], s2[FN];
#pragma unroll
  for (int jn = 0; jn < FN; ++jn) { s1[jn] = 0.0; s2[jn] = 0.0; }
  float* out = a.out + (long long)task * a.out_stride;
  const float* zh = a.zh ? a.zh + (long long)task * a.zh_stride : nullptr;
  __syncthreads();

  for (int t = 0; t < tiles; ++t) {
    const int j0 = j00 + t * ROWS;
    if (j0 >= a.rows) break;
    float acc[R][FN];
#pragma unroll
    for (int i = 0; i < R; ++i)
#pragma unroll
      for (int jn = 0; jn < FN; ++jn) acc[i][jn] = 0.f;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      // positions t*ROWS + ty*R + (ky-1)*gw - 1 + halo .. + R + 1 of the window (always inside it)
      const float* xp = xs + (t * ROWS + ty * R + (ky - 1) * a.gw - 1 + halo) * C0;
      float xw[(R + 2) * C0];
#pragma unroll
      for (int i = 0; i < (R + 2) * C0; ++i) xw[i] = xp[i];
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
#pragma unroll
        for (int c = 0; c < C0; ++c) {
          float b[FN];
          const float* wp = Ws + ((ky * 3 + kx) * C0 + c) * NC + tx * FN;
#pragma unroll
          for (int jn = 0; jn < FN; ++jn) b[jn] = wp[jn];
#pragma unroll
          for (int i = 0; i < R; ++i) {
            const float av = xw[(i + kx) * C0 + c];
#pragma unroll
            for (int jn = 0; jn < FN; ++jn) acc[i][jn] = fmaf(av, b[jn], acc[i][jn]);
          }
        }
      }
    }
    // store + thread-local fp64 statistics; validity of the 8 consecutive rows is tracked incrementally (one division)
    int row = j0 + ty * R;
    int rr = row % a.G;
    int yy = rr / a.gw, xx = rr - yy * a.gw;
#pragma unroll
    for (int i = 0; i < R; ++i, ++row) {
      if (row < a.rows) {
        const long long base = (long long)row * NC + tx * FN;
        const bool valid = (a.mode != CONV_PLAIN) && yy >= 1 && yy <= a.h && xx >= 1 && xx <= a.w;
        float v[FN];
#pragma unroll
        for (int jn = 0; jn < FN; ++jn) v[jn] = acc[i][jn] + bv[jn];
        if constexpr (FN == 4) *reinterpret_cast<float4*>(out + base) = make_float4(v[0], v[1], v[2], v[3]);
        else if constexpr (FN == 2) *reinterpret_cast<float2*>(out + base) = make_float2(v[0], v[1]);
        else {
#pragma unroll
          for (int jn = 0; jn < FN; ++jn) out[base + jn] = v[jn];
        }
        if (valid) {
#pragma unroll
          for (int jn = 0; jn < FN; ++jn) {
            s1[jn] += (double)v[jn];
            s2[jn] += (a.mode == CONV_FWD_STATS) ? (double)v[jn] * (double)v[jn] : (double)zh[base + jn] * (double)v[jn];
          }
        }
      }
      if (++xx == a.gw) { xx = 0; if (++yy == a.G / a.gw) yy = 0; }
    }
  }
  if (a.mode != CONV_PLAIN) {
    const int warp = tid >> 5;
#pragma unroll
    for (int jn = 0; jn < FN; ++jn) {
      s1[jn] += __shfl_xor_sync(0xffffffffu, s1[jn], 16);
      s2[jn] += __shfl_xor_sync(0xffffffffu, s2[jn], 16);
    }
    if ((tid & 16) == 0) {
#pragma unroll
      for (int jn = 0; jn < FN; ++jn) {
        sred[(warp * NC + tx * FN + jn) * 2 + 0] = s1[jn];
        sred[(warp * NC + tx * FN + jn) * 2 + 1] = s2[jn];
      }
    }
    __syncthreads();
    double* stats = a.stats + (long long)task * a.stats_stride;
    for (int c = tid; c < NC * 2; c += 256) {
      double tt = 0.0;
#pragma unroll
      for (int wq = 0; wq < 8; ++wq) tt += sred[wq * NC * 2 + c];
      atomicAdd(&stats[c], tt);
    }
  }
}

template <int C0>
static bool launch_conv0_rb(const Conv0Args& a, cudaStream_t st) {
  // tiles per CTA: as many as keep >= ~3 CTAs per SM in flight (fixed per-CTA cost -- weights, window, fp64 statistics
  // reduction -- is then paid once per `tiles` x 128 rows); 1 for the small launches that sit on the latency-critical chain
  const long long t128 = (a.rows + 127) / 128;
  int tiles = (int)std::min<long long>(8, std::max<long long>(1, t128 * a.tasks / (3LL * num_sms())));
  dim3 grid((unsigned)((t128 + tiles - 1) / tiles), a.tasks);
  const size_t smem = (size_t)(9 * C0 * a.ncols + (128 * tiles + 2 * (a.gw + 1)) * C0) * sizeof(float);
  switch (a.ncols / 16) {
    case 1: launch_pdl(conv0_rb_kernel<1, C0>, dim3(grid), dim3(256), (size_t)(smem), st, tagged(a), tiles); break;
    case 2: launch_pdl(conv0_rb_kernel<2, C0>, dim3(grid), dim3(256), (size_t)(smem), st, tagged(a), tiles); break;
    case 3: launch_pdl(conv0_rb_kernel<3, C0>, dim3(grid), dim3(256), (size_t)(smem), st, tagged(a), tiles); break;
    default: launch_pdl(conv0_rb_kernel<4, C0>, dim3(grid), dim3(256), (size_t)(smem), st, tagged(a), tiles); break;
  }
  return true;
}

void launch_conv0(const Conv0Args& a, cudaStream_t st) {
  ProfScope prof_scope__(PROF_CONV0, a.alg_flops, st);
  if (a.c0 == 1 || a.c0 == 3) {
    if (a.c0 == 1) launch_conv0_rb<1>(a, st); else launch_conv0_rb<3>(a, st);
    CUDA_CHECK_LAUNCH();
    return;
  }
  dim3 grid((a.rows + 63) / 64, a.tasks);
  const size_t smem = (size_t)(9 * a.c0 * a.ncols + (64 + 2 * (a.gw + 1)) * a.c0) * sizeof(float);
  switch (a.ncols / 16) {
    case 1: launch_pdl(conv0_kernel<1>, dim3(grid), dim3(256), (size_t)(smem), st, tagged(a)); break;
    case 2: launch_pdl(conv0_kernel<2>, dim3(grid), dim3(256), (size_t)(smem), st, tagged(a)); break;
    case 3: launch_pdl(conv0_kernel<3>, dim3(grid), dim3(256), (size_t)(smem), st, tagged(a)); break;
    default: launch_pdl(conv0_kernel<4>, dim3(grid), dim3(256), (size_t)(smem), st, tagged(a)); break;
  }
  CUDA_CHECK_LAUNCH();
}

// ---------------------------------------------------------------------------------------------
// wgrad:  partial[chunk][tap][c][f] = sum_{j in chunk} sum_src A_src[j + s_tap, c] * D_src[j, f]
//         partial[chunk][bias][f]   = sum_{j in chunk} D_0[j, f]                 (centre filter row CTA)
// chunks are reduced (in fixed order => deterministic) by the parameter-space kernel that consumes the partial buffer.
// ---------------------------------------------------------------------------------------------
// One CTA handles the three taps (ky, kx = -1, 0, +1) of one filter row and chunk.  Their A rows are CONSECUTIVE
// (shifts s-1, s, s+1), so while a thread walks the rows of a K step it keeps a sliding window of three A rows in
// registers: per row 2 x LDS.128 feed 3 x CN x FN FMAs (one tap per CTA would need 2 x LDS.128 per CN x FN), the
// dz tile is staged once for three taps and the number of barriers per FMA drops 3x.  grid (nchunks * 3, tasks).
template <int CN, int FN>
__global__ void __launch_bounds__(256) wgrad_row_kernel(WgradArgs a) {
  pdl_prologue(3, a.tag);
  constexpr int KC = 16 * CN, NC = 16 * FN;
  constexpr int A4 = 18 * KC / 4;                  // float4 loads of the 18-row A window
  __shared__ __align__(16) float As[18][KC];
  __shared__ __align__(16) float Ds[16][NC];
  const int task = blockIdx.y;
  const int chunk = blockIdx.x / 3, ky = blockIdx.x - chunk * 3;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int sh = (ky - 1) * a.gw - 1;              // A window row 0 = output row + sh  (tap kx = -1)
  const int r_begin = chunk * a.rows_per_chunk;
  const int r_end = min(a.rows, r_begin + a.rows_per_chunk);
  const int guard = a.gw + 2;

  float acc[3][CN][FN];
#pragma unroll
  for (int t = 0; t < 3; ++t)
#pragma unroll
    for (int i = 0; i < CN; ++i)
#pragma unroll
      for (int jn = 0; jn < FN; ++jn) acc[t][i][jn] = 0.f;
  float bacc = 0.f;

  const int steps = (r_end > r_begin) ? (r_end - r_begin + 15) / 16 : 0;
  const int nit = steps * a.nsrc;
  float4 ra0 = make_float4(0.f, 0.f, 0.f, 0.f), ra1 = ra0, rd = ra0;

  auto fetch = [&](int it) {
    const int s = it / steps;
    const int r0 = r_begin + (it - s * steps) * 16;
    const float* A = a.A[s] + (long long)task * a.a_stride[s];
    {
      const int r = tid / (KC / 4), c4 = tid - r * (KC / 4);
      const int jr = r0 + sh + r;
      ra0 = (r < 18 && jr >= -guard && jr < a.rows + guard) ? *reinterpret_cast<const float4*>(A + (long long)jr * KC + c4 * 4)
                                                            : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (tid + 256 < A4) {
      const int e = tid + 256;
      const int r = e / (KC / 4), c4 = e - r * (KC / 4);
      const int jr = r0 + sh + r;
      ra1 = (jr >= -guard && jr < a.rows + guard) ? *reinterpret_cast<const float4*>(A + (long long)jr * KC + c4 * 4)
                                                  : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (tid < 4 * NC) {
      const int r = tid / (NC / 4), f4 = tid - r * (NC / 4);
      const int jr = r0 + r;
      rd = (jr < r_end) ? *reinterpret_cast<const float4*>(a.D[s] + (long long)task * a.d_stride[s] + (long long)jr * NC + f4 * 4)
                        : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };

  if (nit > 0) fetch(0);
  for (int it = 0; it < nit; ++it) {
    {
      const int r = tid / (KC / 4), c4 = tid - r * (KC / 4);
      if (r < 18) *reinterpret_cast<float4*>(&As[r][c4 * 4]) = ra0;
    }
    if (tid + 256 < A4) {
      const int e = tid + 256;
      const int r = e / (KC / 4), c4 = e - r * (KC / 4);
      *reinterpret_cast<float4*>(&As[r][c4 * 4]) = ra1;
    }
    if (tid < 4 * NC) {
      const int r = tid / (NC / 4), f4 = tid - r * (NC / 4);
      *reinterpret_cast<float4*>(&Ds[r][f4 * 4]) = rd;
    }
    __syncthreads();
    const bool bias_src = (it / steps) == 0;
    if (it + 1 < nit) fetch(it + 1);
    float w0[CN], w1[CN], w2[CN];
#pragma unroll
    for (int i = 0; i < CN; ++i) { w0[i] = As[0][ty * CN + i]; w1[i] = As[1][ty * CN + i]; }
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      float b[FN];
#pragma unroll
      for (int i = 0; i < CN; ++i) w2[i] = As[r + 2][ty * CN + i];
#pragma unroll
      for (int jn = 0; jn < FN; ++jn) b[jn] = Ds[r][tx * FN + jn];
#pragma unroll
      for (int i = 0; i < CN; ++i)
#pragma unroll
        for (int jn = 0; jn < FN; ++jn) {
          acc[0][i][jn] = fmaf(w0[i], b[jn], acc[0][i][jn]);
          acc[1][i][jn] = fmaf(w1[i], b[jn], acc[1][i][jn]);
          acc[2][i][jn] = fmaf(w2[i], b[jn], acc[2][i][jn]);
        }
#pragma unroll
      for (int i = 0; i < CN; ++i) { w0[i] = w1[i]; w1[i] = w2[i]; }
    }
    if (ky == 1 && bias_src && tid < NC) {
#pragma unroll
      for (int r = 0; r < 16; ++r) bacc += Ds[r][tid];
    }
    __syncthreads();
  }

  float* P = a.partial + (long long)task * a.partial_task_stride + (long long)chunk * a.chunk_stride;
#pragma unroll
  for (int t = 0; t < 3; ++t)
#pragma unroll
    for (int i = 0; i < CN; ++i)
#pragma unroll
      for (int jn = 0; jn < FN; ++jn) P[(long long)((ky * 3 + t) * KC + ty * CN + i) * NC + tx * FN + jn] = acc[t][i][jn];
  if (ky == 1 && tid < NC) P[(long long)9 * KC * NC + tid] = bacc;
}

void launch_wgrad(const WgradArgs& a, cudaStream_t st) {
  ProfScope prof_scope__(PROF_WGRAD, a.alg_flops, st);
  const int cn = a.kc / 16, fn = a.ncols / 16;
  dim3 grid(a.nchunks * 3, a.tasks);
#define WGR_CASE(C, F_) if (cn == C && fn == F_) { launch_pdl(wgrad_row_kernel<C, F_>, dim3(grid), dim3(256), (size_t)(0), st, tagged(a)); CUDA_CHECK_LAUNCH(); return; }
  WGR_CASE(1, 1) WGR_CASE(2, 2) WGR_CASE(3, 3) WGR_CASE(4, 4)
#undef WGR_CASE
}

// first block wgrad: A = image matrix [rows][c0] (c0 <= 4), D = dz [rows][F].
// Per 64-row sub-tile the dz rows and the image window (rows +/- halo) are staged in shared memory; thread
// (grp, f) accumulates the (tap, c) combinations q = grp, grp + NG, ... for output channel f.
template <int MAXQ>
__global__ void __launch_bounds__(256) wgrad0_kernel(WgradArgs a) {
  pdl_prologue(4, a.tag);
  extern __shared__ float smw[];
  const int task = blockIdx.y, chunk = blockIdx.x;
  const int tid = threadIdx.x;
  const int Fc = a.ncols, c0 = a.kc;
  const int NG = 256 / Fc;
  const int grp = tid / Fc, f = tid - grp * Fc;
  const bool active = grp < NG;
  const int ncombo = 9 * c0;            // host guarantees MAXQ * NG >= ncombo
  constexpr int RT = 64;
  const int halo = a.gw + 1;
  float* Ds = smw;                       // [RT][Fc]
  float* Xs = smw + RT * Fc;             // [(RT + 2*halo)][c0]
  float acc[MAXQ];
  int off[MAXQ];
#pragma unroll
  for (int i = 0; i < MAXQ; ++i) {
    acc[i] = 0.f;
    const int q = grp + i * NG;
    off[i] = (q < ncombo) ? (tap_shift(q / c0, a.gw) + halo) * c0 + (q % c0) : 0;
  }
  float bacc = 0.f;
  const int r_begin = chunk * a.rows_per_chunk;
  const int r_end = min(a.rows, r_begin + a.rows_per_chunk);
  const float* A = a.A[0] + (long long)task * a.a_stride[0];
  const float* D = a.D[0] + (long long)task * a.d_stride[0];
  const int guard = a.gw + 2;
  for (int r0 = r_begin; r0 < r_end; r0 += RT) {
    const int nr = min(RT, r_end - r0);
    for (int i = tid; i < RT * Fc / 4; i += 256) {
      const int r = (i * 4) / Fc;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < nr) v = *reinterpret_cast<const float4*>(D + (long long)r0 * Fc + (long long)i * 4);
      *reinterpret_cast<float4*>(Ds + i * 4) = v;
    }
    for (int i = tid; i < (RT + 2 * halo) * c0; i += 256) {
      const int r = r0 - halo + i / c0;
      float v = 0.f;
      if (r >= -guard && r < a.rows + guard) v = A[(long long)(r0 - halo) * c0 + i];
      Xs[i] = v;
    }
    __syncthreads();
    if (active) {
      for (int r = 0; r < nr; ++r) {
        const float d = Ds[r * Fc + f];
        const float* xr = Xs + r * c0;
#pragma unroll
        for (int i = 0; i < MAXQ; ++i) {
          const int q = grp + i * NG;
          if (q < ncombo) acc[i] = fmaf(xr[off[i]], d, acc[i]);
        }
        bacc += d;
      }
    }
    __syncthreads();
  }
  if (active) {
    float* P = a.partial + (long long)task * a.partial_task_stride + (long long)chunk * a.chunk_stride;
#pragma unroll
    for (int i = 0; i < MAXQ; ++i) {
      const int q = grp + i * NG;
      if (q < ncombo) P[(long long)q * Fc + f] = acc[i];
    }
    if (grp == 0) P[(long long)ncombo * Fc + f] = bacc;
  }
}

// Register-blocked first-block weight gradient (C0 = 1 or 3).  Per grid row the update is the outer product
// x[27 = tap x c] (x) dz[F]; a thread owns one filter row ky (3 kx x C0 taps) and 4 output channels: 12 * C0 accumulators.
// The CTA's threads form NS "row streams" of 3 * F/4 threads; a stream walks CONSECUTIVE rows of the staged tile, so the
// three x positions of a row slide by one per row: per row C0 broadcast loads + one LDS.128 of dz feed 12 * C0 FMAs
// (wgrad0_kernel: 7 loads per 6 FMAs).  Streams are summed through shared memory in stream order (deterministic).
// C0 = 1 is held to 48 registers (5 CTAs per SM); left to itself ptxas gives it 58 (4 CTAs).  0: no bound for C0 = 3.
template <int C0>
__global__ void __launch_bounds__(256, C0 == 1 ? 5 : 0) wgrad0_rb_kernel(WgradArgs a) {
  pdl_prologue(4, a.tag);
  extern __shared__ float smw[];
  const int task = blockIdx.y, chunk = blockIdx.x;
  const int tid = threadIdx.x;
  const int Fc = a.ncols, F4 = Fc >> 2;
  const int TPS = 3 * F4;                 // threads per row stream
  const int NS = 256 / TPS;               // row streams
  constexpr int L = 16;                   // consecutive rows per stream and tile
  const int RT = NS * L;                  // rows per staged tile
  const int stream = tid / TPS, rem = tid - stream * TPS;
  const int ky = rem / F4, f4 = rem - ky * F4;
  const bool active = stream < NS;
  const int halo = a.gw + 1;
  float* Ds = smw;                        // [RT][Fc]
  float* Xs = smw + RT * Fc;              // [(RT + 2*halo)][C0]
  float acc[3][C0][4];
#pragma unroll
  for (int kx = 0; kx < 3; ++kx)
#pragma unroll
    for (int c = 0; c < C0; ++c)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[kx][c][j] = 0.f;
  float bacc[4] = {0.f, 0.f, 0.f, 0.f};
  const int r_begin = chunk * a.rows_per_chunk;
  const int r_end = min(a.rows, r_begin + a.rows_per_chunk);
  const float* A = a.A[0] + (long long)task * a.a_stride[0];
  const float* D = a.D[0] + (long long)task * a.d_stride[0];
  const int guard = a.gw + 2;
  for (int r0 = r_begin; r0 < r_end; r0 += RT) {
    const int nr = min(RT, r_end - r0);
    for (int i = tid; i < RT * Fc / 4; i += 256) {
      const int r = (i * 4) / Fc;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < nr) v = *reinterpret_cast<const float4*>(D + (long long)r0 * Fc + (long long)i * 4);
      *reinterpret_cast<float4*>(Ds + i * 4) = v;                     // rows beyond nr are zero: they add nothing below
    }
    for (int i = tid; i < (RT + 2 * halo) * C0; i += 256) {
      const int r = r0 - halo + i / C0;
      float v = 0.f;
      if (r >= -guard && r < a.rows + guard) v = A[(long long)(r0 - halo) * C0 + i];
      Xs[i] = v;
    }
    __syncthreads();
    if (active) {
      const int rs = stream * L;                                        // first row of this stream in the tile
      // window row index of tap (ky, kx) for tile row r: r + halo + (ky-1)*gw + (kx-1)
      const float* xp = Xs + (rs + halo + (ky - 1) * a.gw - 1) * C0;
      float xw[3][C0];
#pragma unroll
      for (int c = 0; c < C0; ++c) { xw[1][c] = xp[c]; xw[2][c] = xp[C0 + c]; }
#pragma unroll 4
      for (int r = 0; r < L; ++r) {
#pragma unroll
        for (int c = 0; c < C0; ++c) { xw[0][c] = xw[1][c]; xw[1][c] = xw[2][c]; xw[2][c] = xp[(r + 2) * C0 + c]; }
        const float4 d = *reinterpret_cast<const float4*>(Ds + (rs + r) * Fc + f4 * 4);
#pragma unroll
        for (int kx = 0; kx < 3; ++kx)
#pragma unroll
          for (int c = 0; c < C0; ++c) {
            acc[kx][c][0] = fmaf(xw[kx][c], d.x, acc[kx][c][0]);
            acc[kx][c][1] = fmaf(xw[kx][c], d.y, acc[kx][c][1]);
            acc[kx][c][2] = fmaf(xw[kx][c], d.z, acc[kx][c][2]);
            acc[kx][c][3] = fmaf(xw[kx][c], d.w, acc[kx][c][3]);
          }
        bacc[0] += d.x; bacc[1] += d.y; bacc[2] += d.z; bacc[3] += d.w;
      }
    }
    __syncthreads();
  }
  // sum the row streams in order: red[stream][(tap * C0 + c)][f] (+ bias row)
  const int ncombo = 9 * C0;
  float* red = smw;                        // NS * (ncombo + 1) * Fc floats (fits: the launcher sizes shared memory for both uses)
  if (active) {
    float* mine = red + (long long)stream * (ncombo + 1) * Fc;
#pragma unroll
    for (int kx = 0; kx < 3; ++kx)
#pragma unroll
      for (int c = 0; c < C0; ++c)
#pragma unroll
        for (int j = 0; j < 4; ++j) mine[((ky * 3 + kx) * C0 + c) * Fc + f4 * 4 + j] = acc[kx][c][j];
    if (ky == 1) {
#pragma unroll
      for (int j = 0; j < 4; ++j) mine[ncombo * Fc + f4 * 4 + j] = bacc[j];
    }
  }
  __syncthreads();
  float* P = a.partial + (long long)task * a.partial_task_stride + (long long)chunk * a.chunk_stride;
  for (int i = tid; i < (ncombo + 1) * Fc; i += 256) {
    float t = 0.f;
    for (int st = 0; st < NS; ++st) t += red[(long long)st * (ncombo + 1) * Fc + i];
    P[i] = t;
  }
}

void launch_wgrad0(const WgradArgs& a, cudaStream_t st) {
  ProfScope prof_scope__(PROF_WGRAD0, a.alg_flops, st);
  dim3 grid(a.nchunks, a.tasks);
  if ((a.kc == 1 || a.kc == 3) && a.nsrc == 1 && (a.ncols % 4) == 0) {
    const int tps = 3 * (a.ncols / 4), ns = 256 / tps, rt = ns * 16;
    const size_t stage = (size_t)(rt * a.ncols + (rt + 2 * (a.gw + 1)) * a.kc) * sizeof(float);
    const size_t red = (size_t)ns * (9 * a.kc + 1) * a.ncols * sizeof(float);
    const size_t smem = stage > red ? stage : red;
    if (a.kc == 1) launch_pdl(wgrad0_rb_kernel<1>, dim3(grid), dim3(256), smem, st, tagged(a));
    else launch_pdl(wgrad0_rb_kernel<3>, dim3(grid), dim3(256), smem, st, tagged(a));
    CUDA_CHECK_LAUNCH();
    return;
  }
  const size_t smem = (size_t)(64 * a.ncols + (64 + 2 * (a.gw + 1)) * a.kc) * sizeof(float);
  const int need = (9 * a.kc + (256 / a.ncols) - 1) / (256 / a.ncols);      // (tap, c) combinations per thread
  if (need <= 3) launch_pdl(wgrad0_kernel<3>, dim3(grid), dim3(256), (size_t)(smem), st, tagged(a));
  else if (need <= 6) launch_pdl(wgrad0_kernel<6>, dim3(grid), dim3(256), (size_t)(smem), st, tagged(a));
  else if (need <= 9) launch_pdl(wgrad0_kernel<9>, dim3(grid), dim3(256), (size_t)(smem), st, tagged(a));
  else launch_pdl(wgrad0_kernel<36>, dim3(grid), dim3(256), (size_t)(smem), st, tagged(a));
  CUDA_CHECK_LAUNCH();
}

// ---------------------------------------------------------------------------------------------
// first-block data gradient (d loss / d images), written straight into NCHW [tasks][n][C0][h][w]:
//   dx[img][c][y][x] = sum_src sum_tap sum_f W_src[tap][c][f] * D_src[row(img, y, x) - s_tap][f]
// N = C0 <= 4 is below wgmma's smallest N (8) and K = 9 * F: register-blocked FFMA.  Thread (rg, fl) owns IG_R
// consecutive grid rows x all C0 outputs for the filter slice f = f0 + fl of each 16-wide chunk f0.  For a filter row ky
// the source rows of its IG_R rows and three kx taps are IG_R + 2 consecutive rows: read once from shared memory, they
// feed 3 x C0 x IG_R FMAs.  The 16 f lanes of a half-warp are summed by a fixed xor butterfly (no atomics: bit-identical
// run to run).  Source rows outside the valid h x w window (pad columns, pad rows, guard rows) are zero by index test:
// the kernel never reads what other passes left in the border rows of D.
// ---------------------------------------------------------------------------------------------
constexpr int IG_R = 8, IG_GROUPS = 32, IG_ROWS = IG_R * IG_GROUPS, IG_FC = 16;
constexpr int IG_P = IG_FC + 2;   // shared row pitch: the two half-warps of a warp (rows 8 apart) hit disjoint banks

template <int C0, int NSRC>
__global__ void __launch_bounds__(IG_GROUPS * 16) input_grad0_kernel(InputGradArgs a) {
  pdl_prologue(31, a.tag);
  extern __shared__ float smi[];
  const int task = blockIdx.y;
  const int j0 = blockIdx.x * IG_ROWS;
  const int tid = threadIdx.x, rg = tid >> 4, fl = tid & 15;
  const int F = a.ncols, halo = a.gw + 1, wrows = IG_ROWS + 2 * halo;
  float* Ws = smi;                                   // [NSRC][9][C0][F]
  float* Ds = Ws + NSRC * 9 * C0 * F;                // [wrows][IG_P]: one 16-wide filter chunk of the window
  int* vm = reinterpret_cast<int*>(Ds + wrows * IG_P);   // [wrows]: window row is a valid pixel
  for (int s = 0; s < NSRC; ++s) {
    const float* W = (s == 0 ? a.W[0] : a.W[1]) + (long long)task * a.w_stride;   // (no dynamic index into the parameters)
    for (int i = tid; i < 9 * C0 * F; i += IG_GROUPS * 16) Ws[s * 9 * C0 * F + i] = W[i];
  }
  for (int r = tid; r < wrows; r += IG_GROUPS * 16) {
    const int row = j0 - halo + r;
    int ok = 0;
    if (row >= 0 && row < a.rows) {
      const int rr = row % a.G, yy = rr / a.gw, xx = rr - yy * a.gw;
      ok = yy >= 1 && yy <= a.h && xx >= 1 && xx <= a.w;
    }
    vm[r] = ok;
  }
  float acc[IG_R][C0];
#pragma unroll
  for (int k = 0; k < IG_R; ++k)
#pragma unroll
    for (int c = 0; c < C0; ++c) acc[k][c] = 0.f;

  for (int s = 0; s < NSRC; ++s) {
    const float* D = s == 0 ? a.D[0] + (long long)task * a.d_stride[0] : a.D[1] + (long long)task * a.d_stride[1];
    for (int f0 = 0; f0 < F; f0 += IG_FC) {
      __syncthreads();                               // the previous chunk has been consumed
      for (int i = tid; i < wrows * (IG_FC / 4); i += IG_GROUPS * 16) {
        const int r = i >> 2, q = i & 3;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (vm[r]) v = *reinterpret_cast<const float4*>(D + (long long)(j0 - halo + r) * F + f0 + q * 4);
        float* d = Ds + r * IG_P + q * 4;
        d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
      }
      __syncthreads();
      const float* wp = Ws + s * 9 * C0 * F + f0 + fl;
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        // window rows rg*IG_R + halo - (ky-1)*gw - 1 .. + IG_R + 1: tap kx of local row k reads entry k + 2 - kx
        const float* dp = Ds + (rg * IG_R + halo - (ky - 1) * a.gw - 1) * IG_P + fl;
        float xw[IG_R + 2];
#pragma unroll
        for (int i = 0; i < IG_R + 2; ++i) xw[i] = dp[i * IG_P];
#pragma unroll
        for (int kx = 0; kx < 3; ++kx)
#pragma unroll
          for (int c = 0; c < C0; ++c) {
            const float wv = wp[((ky * 3 + kx) * C0 + c) * F];
#pragma unroll
            for (int k = 0; k < IG_R; ++k) acc[k][c] = fmaf(xw[k + 2 - kx], wv, acc[k][c]);
          }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < IG_R; ++k)
#pragma unroll
    for (int c = 0; c < C0; ++c)
#pragma unroll
      for (int o = 8; o >= 1; o >>= 1) acc[k][c] += __shfl_xor_sync(0xffffffffu, acc[k][c], o);

  // every lane of the half-warp now holds the same sums: lane fl stores row k = fl % 8, channels fl / 8, fl / 8 + 2
  const int k = fl & (IG_R - 1), ch = fl >> 3;
  const int row = j0 + rg * IG_R + k;
  if (row >= a.rows) return;
  const int img = row / a.G, rr = row - img * a.G, yy = rr / a.gw, xx = rr - yy * a.gw;
  if (yy < 1 || yy > a.h || xx < 1 || xx > a.w) return;
  const long long plane = (long long)a.h * a.w;
  float* out = a.dx + (long long)task * a.dx_stride + (long long)img * C0 * plane + (long long)(yy - 1) * a.w + (xx - 1);
#pragma unroll
  for (int cp = 0; cp < C0; cp += 2) {
    if (cp + ch < C0) {
      float v = 0.f;
#pragma unroll
      for (int kk = 0; kk < IG_R; ++kk)
        if (kk == k) v = ch ? acc[kk][cp + 1 < C0 ? cp + 1 : cp] : acc[kk][cp];
      out[(cp + ch) * plane] = v;
    }
  }
}

template <int C0, int NSRC>
static void launch_input_grad0_c(const InputGradArgs& a, cudaStream_t st) {
  const int wrows = IG_ROWS + 2 * (a.gw + 1);
  const size_t smem = (size_t)(NSRC * 9 * C0 * a.ncols + wrows * IG_P + wrows) * sizeof(float);
  if (smem > 48 * 1024) cudaFuncSetAttribute(input_grad0_kernel<C0, NSRC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  dim3 grid((a.rows + IG_ROWS - 1) / IG_ROWS, a.tasks);
  launch_pdl(input_grad0_kernel<C0, NSRC>, dim3(grid), dim3(IG_GROUPS * 16), smem, st, tagged(a));
}

void launch_input_grad0(const InputGradArgs& a, cudaStream_t st) {
  ProfScope prof_scope__(PROF_CONV0, a.alg_flops, st);
#define IG_CASE(C, S) if (a.c0 == C && a.nsrc == S) launch_input_grad0_c<C, S>(a, st); else
  IG_CASE(1, 1) IG_CASE(2, 1) IG_CASE(3, 1) IG_CASE(4, 1) IG_CASE(1, 2) IG_CASE(2, 2) IG_CASE(3, 2) IG_CASE(4, 2) {}
#undef IG_CASE
  CUDA_CHECK_LAUNCH();
}

// ---------------------------------------------------------------------------------------------
// image NCHW [tasks][n][C][H][W] -> padded-grid matrix [tasks][n*G][C] (valid positions only)
// ---------------------------------------------------------------------------------------------
__global__ void prep_x_kernel(const float* __restrict__ x, float* __restrict__ xg, long long xg_task_stride, int n,
                              int C, int H, int W, int tag) {
  pdl_prologue(5, tag);
  const int task = blockIdx.y;
  const long long total = (long long)n * H * W;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int xx = (int)(i % W);
  const int yy = (int)((i / W) % H);
  const int img = (int)(i / ((long long)W * H));
  const int gw = W + 1, G = (H + 1) * (W + 1);      // shared-padding grid (engine.cu build_geometry)
  const float* src = x + ((long long)task * n + img) * C * H * W + (long long)yy * W + xx;
  float* dst = xg + (long long)task * xg_task_stride + ((long long)img * G + (yy + 1) * gw + (xx + 1)) * C;
  for (int c = 0; c < C; ++c) dst[c] = src[(long long)c * H * W];
}

void launch_prep_x(const float* x, float* xg, long long xg_task_stride, int tasks, int n, int C, int H, int W,
                   cudaStream_t st) {
  ProfScope prof_scope__(PROF_PARAM, 0.0, st);
  const long long total = (long long)n * H * W;
  dim3 grid((unsigned)((total + 255) / 256), tasks);
  launch_pdl(prep_x_kernel, dim3(grid), dim3(256), (size_t)(0), st, x, xg, xg_task_stride, n, C, H, W, launch_tag());
  CUDA_CHECK_LAUNCH();
}

MAML_TRACE_SETTER(trace_set_conv)
