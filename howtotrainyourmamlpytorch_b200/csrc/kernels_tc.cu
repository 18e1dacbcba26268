// wgmma / TMA implicit-GEMM 3x3 convolution for sm_90a, fp32-faithful via the 3xTF32 operand split.
//
//   out[j, n] = sum_tap sum_k A[j +/- s_tap, k] * B[tap][n][k]        (fp32 result)
//
// Used for the forward conv, the tangent conv, dgrad and tangent dgrad of blocks l >= 1 (reference
// meta_neural_network_architectures.py:89-97 and its autograd derivatives).  One operand pair per launch: the two pairs
// of a tangent conv run as two launches whose outputs the BatchNorm kernels add.
//
// Why it maps to plain 2-D TMA tiles: activations live on the zero-padded pixel grid (common.cuh), so the A
// operand of filter tap (ky,kx) is the SAME [rows, C] matrix shifted by s_tap rows -- every (tap, k-chunk)
// stage is one 128 x 32 fp32 box (SWIZZLE_128B) per operand half, out-of-range rows are zero-filled by TMA.
//
// Precision: single-pass TF32 is not acceptable for this path (SURVEY.md appendix C: 40-130 % meta-gradient
// error).  Every operand x is pre-split by its producer kernel into hi = rna_tf32(x), lo = rna_tf32(x - hi);
// the kernel accumulates A_hi*B_hi and (A_lo*B_hi + A_hi*B_lo) in SEPARATE fp32 register accumulators.
// The tensor core's fp32 accumulation truncates when it aligns addends, so error grows with the number of
// sequential accumulations into one accumulator (one accumulator for all 216 MMAs of a 64-channel layer gave ~5x
// the fp32-FFMA error).  The big term is therefore spread round-robin over 4 accumulators (18 accumulations each
// instead of 216), the small terms get a fifth, and the epilogue adds the five with IEEE fp32 adds.
//
// CTA = one 128-row M tile x all N (<= 64) columns, 384 threads.  Warps 0..7 = two consumer warpgroups (rows 0..63 and
// 64..127 of the tile: wgmma m64nNk8, accumulators in registers, 5 x N / 2 per thread), warps 8..11 = producer
// warpgroup (one TMA thread; setmaxnreg moves its registers to the consumers).  Warps 0..3 then run the epilogue (+ bias, coalesced global store, fp64 BatchNorm statistics).  Shared-memory
// B ring with mbarrier full/empty pairs; a stage is released once wgmma.wait_group shows its MMAs complete.
#include <cuda.h>
#include <algorithm>
#include <map>
#include <utility>
#include "common.cuh"
#include "tc_common.cuh"

namespace {


__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// bounded spin: a mis-programmed pipeline traps (error) instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done = 0;
  for (long long spin = 0; spin < (1LL << 26); ++spin) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    if (done) return;
  }
  __trap();
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(dst), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// accumulator registers stay live across asynchronous wgmma groups: keep the compiler from moving their uses
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// K-major, SWIZZLE_128B shared-memory matrix descriptor (sm_90 wgmma):
//   [0,14) start address >> 4 | [16,30) LBO >> 4 (unused: one swizzle atom along K) | [32,46) SBO >> 4 = 1024 B
//   (8 rows x 128 B) | [49,52) base offset = 0 | [62,64) layout type = 1 (SWIZZLE_128B)
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)((1024u >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// wgmma.mma_async m64nNk8 tf32 x tf32 -> f32, D += A * B (accumulators are zero-initialised by the caller)
__device__ __forceinline__ void wgmma_tf32_n16(float (&d)[8], uint64_t adesc, uint64_t bdesc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
               : "l"(adesc), "l"(bdesc), "r"(1) : "memory");
}
__device__ __forceinline__ void wgmma_tf32_n32(float (&d)[16], uint64_t adesc, uint64_t bdesc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "l"(adesc), "l"(bdesc), "r"(1) : "memory");
}
__device__ __forceinline__ void wgmma_tf32_n48(float (&d)[24], uint64_t adesc, uint64_t bdesc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
               : "l"(adesc), "l"(bdesc), "r"(1) : "memory");
}
__device__ __forceinline__ void wgmma_tf32_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "l"(adesc), "l"(bdesc), "r"(1) : "memory");
}

// the same with the A fragment in registers (m64k8 tf32 layout per warp: see wgrad_tc_row_kernel)
__device__ __forceinline__ void wgmma_tf32_rs_n16(float (&d)[8], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7}, {%8, %9, %10, %11}, %12, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1) : "memory");
}
__device__ __forceinline__ void wgmma_tf32_rs_n32(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1) : "memory");
}
__device__ __forceinline__ void wgmma_tf32_rs_n48(float (&d)[24], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %29, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, {%24, %25, %26, %27}, %28, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1) : "memory");
}
__device__ __forceinline__ void wgmma_tf32_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(1) : "memory");
}

// thread-block-cluster helpers (split-K over the CTAs of one cluster, reduction through distributed shared memory)
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t dsmem_addr(uint32_t local, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local), "r"(rank));
  return r;
}
__device__ __forceinline__ void dsmem_st4(uint32_t addr, float4 v) {
  asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// Split-K reduction of one output tile across the S CTAs of a cluster.  CTA `zrank` finishes rows [zrank * 128/S, ...).
// Every CTA has already WRITTEN the rows it does not own into the owner's receive buffer
// recv[source rank][128 / S rows][NCOLS + 4] (st.shared::cluster, before the one cluster barrier), so the owner sums S
// LOCAL buffers in rank order (deterministic), adds the bias and writes global memory + a local copy for the statistics.
// Nobody reads a peer's shared memory after the barrier, so no second barrier keeps a CTA alive for its peers.
template <int NCOLS, int S>
__device__ __forceinline__ void splitk_reduce(const float* __restrict__ recv, int zrank, int et, const float* __restrict__ bias,
                                              float* __restrict__ tile2, float* __restrict__ out, int j0, int rows) {
  constexpr int P4 = NCOLS + 4;                         // receive / tile pitch (floats), keeps rows 16-byte aligned
  constexpr int ROWS = 128 / S;
  constexpr int TOTAL4 = ROWS * (NCOLS / 4);
  constexpr int ITEMS = (TOTAL4 + 127) / 128;
#pragma unroll
  for (int it = 0; it < ITEMS; ++it) {
    const int idx = et + it * 128;
    if (idx >= TOTAL4) continue;
    const int rr = idx / (NCOLS / 4), c4 = idx - rr * (NCOLS / 4);
    float4 v[S];
#pragma unroll
    for (int z = 0; z < S; ++z) v[z] = *reinterpret_cast<const float4*>(recv + ((z * ROWS + rr) * P4 + c4 * 4));
    float4 acc = v[0];
#pragma unroll
    for (int z = 1; z < S; ++z) { acc.x += v[z].x; acc.y += v[z].y; acc.z += v[z].z; acc.w += v[z].w; }
    if (bias) { acc.x += bias[c4 * 4]; acc.y += bias[c4 * 4 + 1]; acc.z += bias[c4 * 4 + 2]; acc.w += bias[c4 * 4 + 3]; }
    *reinterpret_cast<float4*>(tile2 + rr * P4 + c4 * 4) = acc;
    const int g = j0 + zrank * ROWS + rr;
    if (g < rows) *reinterpret_cast<float4*>(out + (long long)g * NCOLS + c4 * 4) = acc;
  }
}

// K-major SWIZZLE_128B descriptor whose start is `row_off` rows into a 1024B-aligned tile.  The 128B swizzle XOR is a
// function of the ABSOLUTE shared-memory address bits [7,10) (as for TMA writes), so a start address moved by
// row_off * 128 B addresses rows row_off .. row_off+63 of the tile correctly with the base-offset field left at 0.
// This is what lets ONE halo tile serve all nine filter taps.
// (the consumers add row_off * 128 B >> 4 to the descriptor's address field)

// debug timeline (clock64 at pipeline milestones of CTA (0,0)); written only when TcConvArgs::timeline != 0
__device__ long long g_tc_timeline[16];
#define TC_MARK(i) do { if (a.timeline && blockIdx.x == 0 && blockIdx.y == 0) g_tc_timeline[i] = clock64(); } while (0)

template <int NCOLS>
__device__ __forceinline__ void wgmma_tf32(float (&d)[NCOLS / 2], uint64_t adesc, uint64_t bdesc) {
  if constexpr (NCOLS == 16) wgmma_tf32_n16(d, adesc, bdesc);
  else if constexpr (NCOLS == 32) wgmma_tf32_n32(d, adesc, bdesc);
  else if constexpr (NCOLS == 48) wgmma_tf32_n48(d, adesc, bdesc);
  else wgmma_tf32_n64(d, adesc, bdesc);
}

constexpr int TC_THREADS = 384;      // 2 consumer warpgroups + 1 producer warpgroup

template <int NCOLS>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_kernel(const __grid_constant__ TcMaps maps, const TcConvArgs a) {
  pdl_trigger();
  trace_mark(22, a.tag);
  constexpr int B_BYTES = NCOLS * 128;
  constexpr int BSTAGE = 2 * B_BYTES;            // B_hi + B_lo of one (tap, k-chunk)
  constexpr int P4 = NCOLS + 4;                  // pitch (floats) of every tile / buffer row: 16-byte aligned rows
  constexpr int R = NCOLS / 2;                   // accumulator registers per thread of one m64nNk8 accumulator
  constexpr int MAXB = 8;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ uint64_t a_full[2], a_empty[2], b_full[MAXB], b_empty[MAXB];
  __shared__ int row_ok[128];
  __shared__ double sred[2][NCOLS][2];
  __shared__ float s_bias[NCOLS];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int task = blockIdx.y;
  const int j0 = blockIdx.x * 128;
  if (threadIdx.x == 0) TC_MARK(0);
  const int nph = (a.kc + 31) >> 5;              // A phases = k-chunks (a ragged last one, kc = 16 or 48, is zero-filled
                                                 // by TMA); 9 taps each
  const int nb = a.nb;                           // B ring depth
  // split-K: the gridDim.z CTAs of a cluster share one output tile; CTA z accumulates stages [st_lo, st_hi) of the
  // nph * 9 (phase, tap) stages and the partial tiles are summed through distributed shared memory in the epilogue
  const int nsplit = (int)gridDim.z, zrank = (int)blockIdx.z;
  const int st_lo = zrank * (nph * 9) / nsplit, st_hi = (zrank + 1) * (nph * 9) / nsplit;
  const int ph_lo = st_lo / 9;
  // a CTA writes into its peers' shared memory as soon as ITS accumulators are done, so every CTA of the cluster must be
  // known to have started by then: arrive here, wait right before the first remote store (free by then)
  if (nsplit > 1) cluster_arrive_relaxed();
  const int abuf = a.rpad * 128;                 // bytes of one A halo buffer (hi or lo)
  uint8_t* bring = smem + 4 * (size_t)abuf;
  float* recv = reinterpret_cast<float*>(bring + (size_t)nb * BSTAGE);   // split-K receive buffer [128][P4]
  float* zbuf = recv + (nsplit > 1 ? 128 * P4 : 0);                       // tangent mode: primal zh rows [128 / S][P4]

  if (threadIdx.x == 0) {
    for (int s = 0; s < 2; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 8); }
    for (int s = 0; s < nb; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], 8); }   // empty: one arrival per consumer warp
    fence_barrier_init();
  }
  if (threadIdx.x < 128) {
    // epilogue row flags (interior pixel of the padded grid) and the bias
    const int et = threadIdx.x;
    const int row = j0 + et;
    int ok = 0;
    if (row < a.rows) {
      const int rr = row % a.G;
      const int yy = rr / a.gw, xx = rr - yy * a.gw;
      ok = (yy >= 1 && yy <= a.h && xx >= 1 && xx <= a.w) ? 1 : 0;
    }
    row_ok[et] = ok;
    if (et < NCOLS) s_bias[et] = a.bias ? a.bias[(long long)task * a.bias_stride + et] : 0.f;
  }
  __syncthreads();
  pdl_wait();          // set-up above overlapped the previous kernel's tail; its results are needed from here on
  if (threadIdx.x == 0) TC_MARK(1);

  float* tile = reinterpret_cast<float*>(smem);  // the finished tile, once all MMAs have completed (operand buffers are free)
  if (warp >= 8) {
    // producer warpgroup: gives registers to the consumers (their five accumulators take 5 x NCOLS / 2 per thread)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 8 && lane == 0) {
      // ===== TMA producer: per phase (k-chunk) ONE halo tile of A (hi, lo) that all 9 taps read at row offsets,
      // double-buffered so that phase ph+1 streams in while the MMAs of phase ph run; per (phase, tap) one (B_hi, B_lo)
      // stage through the ring
      int stage = 0; uint32_t bphase = 0;
      for (int st = st_lo; st < st_hi; ++st) {
        const int ph = st / 9, tap = st - ph * 9;
        const int kc0 = ph << 5;
        if (tap == 0 || st == st_lo) {
          const int lp = ph - ph_lo;
          const int ab = lp & 1;
          mbar_wait(&a_empty[ab], (((uint32_t)lp >> 1) & 1u) ^ 1u);
          const int arow = a.a_row_base + task * a.a_task_rows + j0 - a.halo;
          const uint32_t ad = smem_u32(smem + (size_t)ab * 2 * abuf);
          mbar_arrive_expect_tx(&a_full[ab], 2u * (uint32_t)abuf);
          tma_load_2d(ad, &maps.m[0], &a_full[ab], kc0, arow);
          tma_load_2d(ad + abuf, &maps.m[1], &a_full[ab], kc0, arow);
        }
        mbar_wait(&b_empty[stage], bphase ^ 1u);
        const int brow = a.b_row_base + task * a.b_task_rows + tap * NCOLS;
        const uint32_t bd = smem_u32(bring + (size_t)stage * BSTAGE);
        mbar_arrive_expect_tx(&b_full[stage], BSTAGE);
        tma_load_2d(bd, &maps.m[2], &b_full[stage], kc0, brow);
        tma_load_2d(bd + B_BYTES, &maps.m[3], &b_full[stage], kc0, brow);
        if (++stage == nb) { stage = 0; bphase ^= 1u; }
      }
    }
    __syncwarp();
    if (nsplit > 1) {                            // the cluster barriers of the consumers' split-K epilogue, same sequence
      cluster_wait();
      cluster_sync_all();
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    // ===== consumers: warpgroup wg computes tile rows [64 wg, 64 wg + 64)
    const int wg = warp >> 2;
    if (a.mode == CONV_TAN_STATS && threadIdx.x < 128) {
      // tangent mode: the statistics below need the primal zh of the rows this CTA finishes.  Copy them into shared
      // memory first (coalesced float4 loads, a region of its own behind the ring / receive buffer) -- the statistics
      // loop then reads shared memory instead of one dependent global load per row
      constexpr int Q = NCOLS / 4;
      const float* zhg = a.zh + (long long)task * a.zh_stride;
      const int rows_own = 128 / nsplit, row0 = j0 + zrank * rows_own;
      for (int idx = threadIdx.x; idx < rows_own * Q; idx += 128) {
        const int rr = idx / Q, c4 = idx - rr * Q;
        const int gr = row0 + rr;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (gr < a.rows) v = *reinterpret_cast<const float4*>(zhg + (long long)gr * NCOLS + c4 * 4);
        *reinterpret_cast<float4*>(zbuf + rr * P4 + c4 * 4) = v;
      }
    }
    // accumulators 0..3: hi*hi, round-robin over the k-steps of a stage; 4: lo*hi + hi*lo
    float acc[5][R];
#pragma unroll
    for (int q = 0; q < 5; ++q)
#pragma unroll
      for (int i = 0; i < R; ++i) acc[q][i] = 0.f;
    const uint64_t desc_base = make_desc_sw128(0);
    int stage = 0; uint32_t bphase = 0;
    int prev_stage = -1, prev_ab = -1;           // operands of the previous stage, released once its MMAs have completed
    uint64_t ahd = 0, ald = 0;
    int ab = 0;
    for (int st = st_lo; st < st_hi; ++st) {
      const int ph = st / 9, tap = st - ph * 9;
      if (tap == 0 || st == st_lo) {
        const int lp = ph - ph_lo;
        ab = lp & 1;
        mbar_wait(&a_full[ab], ((uint32_t)lp >> 1) & 1u);
        if (st == st_lo && threadIdx.x == 0) TC_MARK(2);
        const uint32_t a_hi = smem_u32(smem + (size_t)ab * 2 * abuf) + (uint32_t)(wg * 64 * 128);
        ahd = desc_base + (uint64_t)(a_hi >> 4);
        ald = ahd + (uint64_t)(abuf >> 4);
      }
      mbar_wait(&b_full[stage], bphase);
      if (threadIdx.x == 0) { if (st == st_lo) TC_MARK(3); if (st == st_lo + 9) TC_MARK(4); }
      const int ty = tap / 3;
      const int row_off = a.halo + a.sign * ((ty - 1) * a.gw + (tap - 3 * ty - 1));    // in [0, 2 * halo]
      const uint64_t ah0 = ahd + (uint64_t)(row_off * 8);
      const uint64_t al0 = ald + (uint64_t)(row_off * 8);
      const uint64_t bh0 = desc_base + (uint64_t)(smem_u32(bring + (size_t)stage * BSTAGE) >> 4);
      const uint64_t bl0 = bh0 + (uint64_t)(B_BYTES >> 4);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {              // K step: +32 B = +2 in the 16-byte address field
        wgmma_tf32<NCOLS>(acc[4], al0 + 2 * k, bh0 + 2 * k);
        wgmma_tf32<NCOLS>(acc[4], ah0 + 2 * k, bl0 + 2 * k);
        wgmma_tf32<NCOLS>(acc[k], ah0 + 2 * k, bh0 + 2 * k);
      }
      wgmma_commit();
      wgmma_wait<1>();                           // the previous stage's MMAs have completed: hand its buffers back
      if (prev_stage >= 0 && lane == 0) {
        mbar_arrive(&b_empty[prev_stage]);
        if (prev_ab >= 0) mbar_arrive(&a_empty[prev_ab]);
      }
      prev_stage = stage;
      prev_ab = (tap == 8 || st == st_hi - 1) ? ab : -1;
      if (++stage == nb) { stage = 0; bphase ^= 1u; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int q = 0; q < 5; ++q) reg_fence<R>(acc[q]);
    if (threadIdx.x == 0) TC_MARK(5);
    // both warpgroups' MMAs have completed before the tile overwrites the operand buffers
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (threadIdx.x == 0) TC_MARK(6);
    {
      // accumulator fragment: register 4 i + 2 h + e holds row 16 (warp % 4) + lane / 4 + 8 h, column 8 i + 2 (lane % 4) + e
      const int rbase = wg * 64 + (warp & 3) * 16 + (lane >> 2);
      const int cq = (lane & 3) * 2;
#pragma unroll
      for (int i = 0; i < NCOLS / 8; ++i) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          float o[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int x = 4 * i + 2 * hh + e;
            const float big = (acc[0][x] + acc[1][x]) + (acc[2][x] + acc[3][x]);
            o[e] = big + acc[4][x];
          }
          *reinterpret_cast<float2*>(tile + (rbase + 8 * hh) * P4 + 8 * i + cq) = make_float2(o[0], o[1]);
        }
      }
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (warp < 4) {
      // ===== epilogue: thread r owns tile row r.  Without split-K: + bias, store its 4 * NCOLS contiguous bytes, keep the
      // biased row in the tile for the statistics.  Split-K: the row goes into the owner CTA's receive buffer.
      const int r = threadIdx.x;
      const int grow = j0 + r;
      float* trow = tile + r * P4;
      if (nsplit == 1) {
        float* orow = a.out + (long long)task * a.out_stride + (long long)grow * NCOLS;
        const bool want_stats = (a.mode != CONV_PLAIN);
#pragma unroll
        for (int c = 0; c < NCOLS; c += 4) {
          float4 v = *reinterpret_cast<const float4*>(trow + c);
          v.x += s_bias[c]; v.y += s_bias[c + 1]; v.z += s_bias[c + 2]; v.w += s_bias[c + 3];
          if (grow < a.rows) *reinterpret_cast<float4*>(orow + c) = v;
          if (want_stats) *reinterpret_cast<float4*>(trow + c) = v;
        }
      } else {
        cluster_wait();                          // phase 1 (arrived at kernel start): all peers are running
        const int rows_per = 128 / nsplit, owner = r / rows_per, rloc = r - owner * rows_per;
        const int recv_off = (zrank * rows_per + rloc) * P4;
        const uint32_t push_row = dsmem_addr(smem_u32(recv + recv_off), (uint32_t)owner);
        float* push_local = recv + recv_off;
#pragma unroll
        for (int c = 0; c < NCOLS; c += 4) {
          const float4 v = *reinterpret_cast<const float4*>(trow + c);
          if (owner == zrank) *reinterpret_cast<float4*>(push_local + c) = v;    // own rows: plain st.shared
          else dsmem_st4(push_row + (uint32_t)(c * 4), v);
        }
      }
      if (r == 0) TC_MARK(7);
    }

    // rows [row_lo, row_lo + row_n) of the tile are finished by this CTA (all 128 without split-K)
    int row_lo = 0, row_n = 128;
    const float* sbuf = tile;                      // where those rows live (row index relative to row_lo)
    if (nsplit > 1) {
      __syncwarp();
      if (warp >= 4) cluster_wait();                 // phase 1 for the consumer warps that did not push
      cluster_sync_all();                            // every receive buffer is complete
      if (threadIdx.x == 0) TC_MARK(10);
      row_n = 128 / nsplit; row_lo = zrank * row_n;
      float* tile2 = reinterpret_cast<float*>(smem + 40 * 1024);
      sbuf = tile2;
      if (warp < 4) {
        const int et = threadIdx.x;
        const float* bias = a.bias ? a.bias + (long long)task * a.bias_stride : nullptr;
        float* outp = a.out + (long long)task * a.out_stride;
        if (nsplit == 2) splitk_reduce<NCOLS, 2>(recv, zrank, et, bias, tile2, outp, j0, a.rows);
        else if (nsplit == 4) splitk_reduce<NCOLS, 4>(recv, zrank, et, bias, tile2, outp, j0, a.rows);
        else splitk_reduce<NCOLS, 8>(recv, zrank, et, bias, tile2, outp, j0, a.rows);
      }
    }

    if (threadIdx.x == 0) TC_MARK(11);
    if (warp < 4) {
      const int et = threadIdx.x;
      const bool want_stats = (a.mode != CONV_PLAIN);
      if (want_stats) {
        asm volatile("bar.sync 2, 128;" ::: "memory");
        constexpr int PARTS = 128 / NCOLS;           // 2 for 64 and 48, 4 for 32, 8 for 16
        const int col = et % NCOLS, part = et / NCOLS;
        double s1 = 0.0, s2 = 0.0;
        if (part < PARTS) {
          for (int rr = part; rr < row_n; rr += PARTS) {
            if (row_ok[row_lo + rr]) {
              const float v = sbuf[rr * P4 + col];
              if (a.mode == CONV_FWD_STATS) { s1 += (double)v; s2 += (double)v * (double)v; }
              else { s1 += (double)v; s2 += (double)zbuf[rr * P4 + col] * (double)v; }
            }
          }
          if (part < 2) { sred[part][col][0] = s1; sred[part][col][1] = s2; }
        }
        if (PARTS > 2) {
          asm volatile("bar.sync 2, 128;" ::: "memory");
          if (part >= 2 && part < PARTS) { atomicAdd(&sred[part & 1][col][0], s1); atomicAdd(&sred[part & 1][col][1], s2); }
        }
        asm volatile("bar.sync 2, 128;" ::: "memory");
        if (et < NCOLS * 2) {
          const int c = et >> 1, which = et & 1;
          double* stats = a.stats + (long long)task * a.stats_stride;
          atomicAdd(&stats[c * 2 + which], sred[0][c][which] + sred[1][c][which]);
        }
      }
    }
    if (threadIdx.x == 0) TC_MARK(12);
    if (threadIdx.x == 0) TC_MARK(8);
  }
  trace_mark(22 | 0x80, a.tag);     // end of CTA (0,0,0)
}

// ---------------------------------------------------------------------------------------------
// wgmma weight gradient of the 3x3 convolutions of blocks l >= 1, fp32-faithful via the 3xTF32 operand split:
//
//   partial[chunk][tap][c][f] = sum_src sum_{j in chunk} A_src[j + s_tap, c] * D_src[j, f]
//   partial[chunk][bias][f]   = sum_{j in chunk} D_0[j, f]                 (centre filter row CTA, fp32)
//
// GEMM M = c, N = f, K = j (pixels).  Both operands are stored pixel-major ([grid row][channel], common.cuh), i.e.
// MN-major for this GEMM, and TF32 wgmma reads shared-memory operands K-major only.  So A comes from REGISTERS (m64k8
// fragments loaded from shared memory with ld.shared) and every 32-row stage of D is transposed into K-major
// SWIZZLE_128B tiles ([f][32 j], the conv kernel's B layout).
//
// CTA = one (row chunk, filter row ky, task), the grid of wgrad_row_kernel, and three warpgroups: warpgroup kx computes
// tap (ky, kx).  The three taps of a filter row read A rows shifted by sh - 1, sh, sh + 1, so ONE staged window of
// 32 + 2 rows serves all three.  Every 32-row stage (A window and D rows, hi and lo; the fp32 D_0 rows too in the bias
// CTA) streams into a ring of WG_NS slots with cp.async, zero-filled outside the guarded A matrix and past the chunk
// end; each thread issues a share and its completions arrive on the slot's mbarrier.  There is no producer warp: a
// 13th warp would put 4 warps on one SM sub-partition and cap every thread at 128 registers (the accumulators need
// ~150); with 12 warps the cap is 168.
// Per stage the threads transpose D ONCE (each a share) into the slot's B tiles and one named barrier publishes them.
// The same barrier shows that every warpgroup has drained the previous stage, so its slot is refilled right after it.
// Each warpgroup then issues its 4 K steps -- A_hi*D_hi into one accumulator, A_hi*D_lo + A_lo*D_hi into a second --,
// transposes the NEXT stage while they run, and only then waits and drains both into fp32 register totals with IEEE
// adds (the tensor core's accumulation truncates, so no accumulator takes more than 8 MMAs).
// ---------------------------------------------------------------------------------------------
template <int NC>
__device__ __forceinline__ void wgmma_tf32_rs(float (&d)[NC / 2], const uint32_t (&a)[4], uint64_t bdesc) {
  if constexpr (NC == 16) wgmma_tf32_rs_n16(d, a, bdesc);
  else if constexpr (NC == 32) wgmma_tf32_rs_n32(d, a, bdesc);
  else if constexpr (NC == 48) wgmma_tf32_rs_n48(d, a, bdesc);
  else wgmma_tf32_rs_n64(d, a, bdesc);
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool ok) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16 : 0) : "memory");
}
// arrives on `bar` once every cp.async this thread has issued so far has landed (counts toward the init count)
__device__ __forceinline__ void cp_async_arrive(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

constexpr int WG_NS = 3;                   // ring slots
constexpr int WG_THREADS = 384;            // 3 warpgroups, one per tap kx

// one ring slot (bytes, 1024-aligned: the B tiles lead): B_hi, B_lo [NC][32] swizzled | A window hi, lo [34][NC + 8] |
// D hi, lo [32][NC] | fp32 D_0 [32][NC]
template <int NC> struct WgSlot {
  static constexpr int BT = NC * 128;
  static constexpr int AP = NC + 8;        // window pitch (floats): the fragment loads of a warp hit 32 distinct banks
  static constexpr int AW = 34 * AP * 4;
  static constexpr int DW = 32 * NC * 4;
  static constexpr int A_OFF = 2 * BT, D_OFF = A_OFF + 2 * AW, DF_OFF = D_OFF + 2 * DW;
  static constexpr int BYTES = (DF_OFF + DW + 1023) / 1024 * 1024;
};
template <int NC> constexpr size_t wgrad_tc_smem() { return (size_t)WG_NS * WgSlot<NC>::BYTES + 1024; }

template <int NC>
__global__ void __launch_bounds__(WG_THREADS, 1) wgrad_tc_row_kernel(const WgradArgs a) {
  pdl_prologue(27, a.tag);
  using S = WgSlot<NC>;
  constexpr int R = NC / 2;
  constexpr int Q = NC / 4;                // float4 per row
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ uint64_t full[WG_NS];
  const int task = blockIdx.y;
  const int chunk = blockIdx.x / 3, ky = blockIdx.x - chunk * 3;
  const int sh0 = (ky - 1) * a.gw - 1;     // window row 0 = output row + sh0 (tap kx = 0)
  const int r_begin = chunk * a.rows_per_chunk;
  const int r_end = min(a.rows, r_begin + a.rows_per_chunk);
  const int guard = a.gw + 2;
  const int steps = r_end > r_begin ? (r_end - r_begin + 31) / 32 : 0;
  const int nit = steps * a.nsrc;
  const bool bias_cta = (ky == 1);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    for (int s = 0; s < WG_NS; ++s) mbar_init(&full[s], WG_THREADS);
    fence_barrier_init();
  }
  __syncthreads();

  // this thread's share of stage `it` -> its slot
  auto load_stage = [&](int it) {
    const int slot = it % WG_NS;
    const int s = it / steps;
    const int r0 = r_begin + (it - s * steps) * 32;
    const float* Ah = a.A[s] + (long long)task * a.a_stride[s] + a.a_plane[s];
    const float* Al = Ah + a.a_plane[s];
    const float* Df = a.D[s] + (long long)task * a.d_stride[s];
    const float* Dh = Df + a.d_plane[s];
    const float* Dl = Dh + a.d_plane[s];
    const uint32_t base = smem_u32(smem + (size_t)slot * S::BYTES);
    for (int e = tid; e < 34 * Q; e += WG_THREADS) {
      const int r = e / Q, c4 = e - r * Q;
      const int jr = r0 + sh0 + r;
      const bool ok = jr >= -guard && jr < a.rows + guard;
      const long long go = ok ? (long long)jr * NC + c4 * 4 : 0;
      const uint32_t so = (uint32_t)((r * S::AP + c4 * 4) * 4);
      cp_async16(base + S::A_OFF + so, Ah + go, ok);
      cp_async16(base + S::A_OFF + S::AW + so, Al + go, ok);
    }
    const bool want_f = bias_cta && s == 0;
    for (int e = tid; e < 32 * Q; e += WG_THREADS) {
      const int r = e / Q;
      const int jr = r0 + r;
      const bool ok = jr < r_end;
      const long long go = ok ? (long long)jr * NC + (e - r * Q) * 4 : 0;
      cp_async16(base + S::D_OFF + e * 16, Dh + go, ok);
      cp_async16(base + S::D_OFF + S::DW + e * 16, Dl + go, ok);
      if (want_f) cp_async16(base + S::DF_OFF + e * 16, Df + go, ok);
    }
    cp_async_arrive(&full[slot]);
  };

  const int kx = warp >> 2;
  const int c0 = 16 * (warp & 3) + (lane >> 2), t4 = lane & 3;   // A fragment: channels c0 (+8), pixels t4 (+4) of a K step
  const bool c_ok = c0 < NC;                                      // NC < 64: the upper fragment rows are zero
  float big[R], small[R], tot[R];
#pragma unroll
  for (int i = 0; i < R; ++i) { big[i] = 0.f; small[i] = 0.f; tot[i] = 0.f; }
  float bacc = 0.f;

  // D stage of `slot` -> K-major tiles: element (f, j) at f * 128 + ((j / 4) ^ (f % 8)) * 16 + (j % 4) * 4.  Item =
  // (plane, j / 4, f), f fastest: four column reads of the row-major stage, one 16-byte store (8 consecutive f of a
  // quarter warp land in 8 distinct 16-byte bank groups)
  auto transpose = [&](int it) {
    const int slot = it % WG_NS;
    uint8_t* sb = smem + (size_t)slot * S::BYTES;
    mbar_wait(&full[slot], (uint32_t)(it / WG_NS) & 1u);
    for (int e = tid; e < 2 * 8 * NC; e += WG_THREADS) {
      const int pl = e / (8 * NC), rem = e - pl * 8 * NC;
      const int j4 = rem / NC, f = rem - j4 * NC;
      const float* src = reinterpret_cast<const float*>(sb + S::D_OFF + pl * S::DW) + (4 * j4) * NC + f;
      const float4 v = make_float4(src[0], src[NC], src[2 * NC], src[3 * NC]);
      *reinterpret_cast<float4*>(sb + pl * S::BT + f * 128 + ((j4 ^ (f & 7)) << 4)) = v;
    }
    if (bias_cta && tid < NC && it < steps) {        // bias: fp32 column sums of D_0, rows in order
      const float* df = reinterpret_cast<const float*>(sb + S::DF_OFF) + tid;
#pragma unroll 8
      for (int r = 0; r < 32; ++r) bacc += df[r * NC];
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma
  };

  for (int i = 0; i < WG_NS - 1 && i < nit; ++i) load_stage(i);
  if (nit > 0) transpose(0);
  for (int it = 0; it < nit; ++it) {
    const uint8_t* sb = smem + (size_t)(it % WG_NS) * S::BYTES;
    // stage it's B tiles are complete, and every warpgroup has drained stage it - 1: refill its slot
    __syncthreads();
    if (it + WG_NS - 1 < nit) load_stage(it + WG_NS - 1);
    // fragments of the stage's 4 K steps (m64k8 tf32: a0 (c0, t4), a1 (c0 + 8, t4), a2 (c0, t4 + 4), a3 (c0 + 8, t4 + 4));
    // tap kx reads window rows shifted by kx
    const float* wh = reinterpret_cast<const float*>(sb + S::A_OFF) + (kx + t4) * S::AP + c0;
    const float* wl = wh + S::AW / 4;
    uint32_t ah[4][4], al[4][4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int o = (8 * k + ((q & 2) ? 4 : 0)) * S::AP + ((q & 1) ? 8 : 0);
        ah[k][q] = c_ok ? __float_as_uint(wh[o]) : 0u;
        al[k][q] = c_ok ? __float_as_uint(wl[o]) : 0u;
      }
    const uint64_t desc_h = make_desc_sw128(smem_u32(sb)), desc_l = desc_h + (uint64_t)(S::BT >> 4);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {                      // rows past the chunk end are zero in D
      wgmma_tf32_rs<NC>(big, ah[k], desc_h + 2 * k);   // K step: +32 B = +2 in the 16-byte address field
      wgmma_tf32_rs<NC>(small, ah[k], desc_l + 2 * k);
      wgmma_tf32_rs<NC>(small, al[k], desc_h + 2 * k);
    }
    wgmma_commit();
    if (it + 1 < nit) transpose(it + 1);             // overlaps this stage's MMAs
    wgmma_wait<0>();
    reg_fence<R>(big);
    reg_fence<R>(small);
#pragma unroll
    for (int i = 0; i < R; ++i) { tot[i] += big[i] + small[i]; big[i] = 0.f; small[i] = 0.f; }
    // hide the zeros from the compiler: an accumulator it knows to be zero turns the first MMA into a non-accumulating
    // one and serialises the next on it
    reg_fence<R>(big);
    reg_fence<R>(small);
  }

  float* P = a.partial + (long long)task * a.partial_task_stride + (long long)a.chunk_stride * chunk;
  const int tap = ky * 3 + kx;
  // accumulator register 4 i + 2 h + e: channel c0 + 8 h, filter 8 i + 2 t4 + e
#pragma unroll
  for (int i = 0; i < NC / 8; ++i)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int c = c0 + 8 * hh;
      if (c < NC)
        *reinterpret_cast<float2*>(P + (long long)(tap * NC + c) * NC + 8 * i + 2 * t4) = make_float2(tot[4 * i + 2 * hh], tot[4 * i + 2 * hh + 1]);
    }
  if (bias_cta && tid < NC) P[(long long)9 * NC * NC + tid] = bacc;
}


}  // namespace

int tc_read_timeline(long long* out16) { return cudaMemcpyFromSymbol(out16, g_tc_timeline, 16 * sizeof(long long)) == cudaSuccess ? 0 : 1; }

// blocks l >= 1 only: kc == ncols (both are F)
void launch_wgrad_tc(const WgradArgs& a, cudaStream_t st) {
  ProfScope prof_scope__(PROF_WGRAD, a.alg_flops, st);
  dim3 grid(a.nchunks * 3, a.tasks);
  if (a.ncols == 64) launch_pdl(wgrad_tc_row_kernel<64>, grid, dim3(WG_THREADS), wgrad_tc_smem<64>(), st, tagged(a));
  else if (a.ncols == 48) launch_pdl(wgrad_tc_row_kernel<48>, grid, dim3(WG_THREADS), wgrad_tc_smem<48>(), st, tagged(a));
  else if (a.ncols == 32) launch_pdl(wgrad_tc_row_kernel<32>, grid, dim3(WG_THREADS), wgrad_tc_smem<32>(), st, tagged(a));
  else launch_pdl(wgrad_tc_row_kernel<16>, grid, dim3(WG_THREADS), wgrad_tc_smem<16>(), st, tagged(a));
  CUDA_CHECK_LAUNCH();
}

// halo tile rows (multiple of 8) for a grid of pitch gw, and the deepest B ring (at most 8 stages) that fits next to 4
// halo buffers and `extra` bytes behind the ring
int tc_conv_rpad(int gw) { return ((128 + 2 * (gw + 1)) + 7) / 8 * 8; }
int tc_conv_ring(int ncols, int gw, size_t extra) {
  const long long avail = 227LL * 1024 - 4096 /* static smem */ - 1024 /* alignment */ - 4LL * tc_conv_rpad(gw) * 128 - (long long)extra;
  long long nb = avail / (2LL * ncols * 128);
  if (nb > 8) nb = 8;
  return (int)nb;
}
// shared memory behind the B ring: with split-K (S > 1) the receive buffer [128 rows][ncols + 4] (peers write it while
// this CTA's MMAs may still read the operand buffers, so it cannot alias them); in tangent mode the primal zh rows the
// CTA finishes [128 / S][ncols + 4]
size_t tc_conv_extra_bytes(int ncols, int S, bool tangent) {
  const size_t row = (size_t)(ncols + 4) * 4;
  return (S > 1 ? 128 * row : 0) + (tangent ? (size_t)(128 / S) * row : 0);
}
static size_t tc_conv_smem_for(int ncols, int gw, int nb) { return (size_t)4 * tc_conv_rpad(gw) * 128 + (size_t)nb * 2 * ncols * 128 + 1024; }

int tc_conv_prepare() {
  const int maxs = 227 * 1024 - 4096;    // static shared memory (barriers, row flags, fp64 partials) takes the rest
  cudaError_t e1 = cudaFuncSetAttribute(conv_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxs);
  cudaError_t e2 = cudaFuncSetAttribute(conv_tc_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxs);
  cudaError_t e3 = cudaFuncSetAttribute(conv_tc_kernel<48>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxs);
  cudaError_t e4 = cudaFuncSetAttribute(conv_tc_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxs);
  cudaError_t w1 = cudaFuncSetAttribute(wgrad_tc_row_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wgrad_tc_smem<64>());
  cudaError_t w2 = cudaFuncSetAttribute(wgrad_tc_row_kernel<48>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wgrad_tc_smem<48>());
  cudaError_t w3 = cudaFuncSetAttribute(wgrad_tc_row_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wgrad_tc_smem<32>());
  cudaError_t w4 = cudaFuncSetAttribute(wgrad_tc_row_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wgrad_tc_smem<16>());
  return (e1 == cudaSuccess && e2 == cudaSuccess && e3 == cudaSuccess && e4 == cudaSuccess && w1 == cudaSuccess &&
          w2 == cudaSuccess && w3 == cudaSuccess && w4 == cudaSuccess) ? 0 : 1;
}

// Split-K factor: small layers have fewer tiles than SMs (Omniglot block 3: 8 tiles, block 2: 32), and one tile's
// serial pipeline (~18 stages x ~1000 cycles) is then the whole kernel.  Spreading the (phase, tap) stages of a tile
// over a cluster of S CTAs shortens that to 18 / S stages + one distributed-shared-memory reduction.  S is the largest
// of {8, 4, 2} (at most the handle's TC_SPLIT option) whose clusters are all co-resident (asked from the occupancy
// calculator once per shape).
template <int NCOLS>
static int max_clusters(size_t smem, int S) {
  static std::map<std::pair<size_t, int>, int> cache;
  auto it = cache.find({smem, S});
  if (it != cache.end()) return it->second;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(1, 1, S); cfg.blockDim = dim3(TC_THREADS); cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = S;
  cfg.attrs = attr; cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, conv_tc_kernel<NCOLS>, &cfg) != cudaSuccess) { cudaGetLastError(); n = 0; }
  cache[{smem, S}] = n;
  return n;
}

template <int NCOLS>
static void launch_conv_tc_n(const TcMaps& maps, const TcConvArgs& a_in, cudaStream_t st) {
  TcConvArgs a = a_in;
  const int tiles = ((a.rows + 127) / 128) * (a.plan_tasks > a.tasks ? a.plan_tasks : a.tasks);
  const int stages = ((a.kc + 31) / 32) * 9;
  // co-residency is asked for the split-K shape: the ring gives up the stages that the receive buffer takes
  const size_t recv_bytes = tc_conv_extra_bytes(NCOLS, 2, false);
  const size_t split_smem = tc_conv_smem_for(NCOLS, a.gw, std::min(a.nb, tc_conv_ring(NCOLS, a.gw, recv_bytes))) + recv_bytes;
  int S = 1;
  for (int cand = launch_ctx().opt->tc_split; cand >= 2; cand >>= 1) {
    if (cand > 8 || stages < 2 * cand) continue;
    if (tiles <= max_clusters<NCOLS>(split_smem, cand)) { S = cand; break; }
  }
  dim3 grid((a.rows + 127) / 128, a.tasks, S);
  // maml_b200_create admits a geometry only if a ring of 2 stages fits next to the largest extra (S = 2, tangent mode)
  const size_t extra = tc_conv_extra_bytes(NCOLS, S, a.mode == CONV_TAN_STATS);
  a.nb = std::min(a.nb, tc_conv_ring(NCOLS, a.gw, extra));
  const size_t smem = tc_conv_smem_for(NCOLS, a.gw, a.nb) + extra;
  if (S == 1) {
    launch_pdl(conv_tc_kernel<NCOLS>, grid, dim3(TC_THREADS), smem, st, maps, tagged(a));
    return;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = dim3(TC_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = S;
  cfg.attrs = attr; cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, conv_tc_kernel<NCOLS>, maps, tagged(a));
}

void launch_conv_tc(const TcMaps& maps, const TcConvArgs& a, cudaStream_t st) {
  ProfScope prof_scope__(PROF_CONV, a.alg_flops, st);
  if (a.ncols == 64) launch_conv_tc_n<64>(maps, a, st);
  else if (a.ncols == 48) launch_conv_tc_n<48>(maps, a, st);
  else if (a.ncols == 32) launch_conv_tc_n<32>(maps, a, st);
  else launch_conv_tc_n<16>(maps, a, st);
  CUDA_CHECK_LAUNCH();
}

// ---------------------------------------------------------------------------------------------
// weight packs: fast weights of blocks l >= 1 split into TF32 hi/lo, in both operand orientations
//   plane 0/1: W  [tap][c][f] hi/lo   (dgrad:  B[n = c][k = f])
//   plane 2/3: WT [tap][f][c] hi/lo   (conv:   B[n = f][k = c])
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// One CTA per (block, tap, task): the F x F tile [c][f] is read once (coalesced), written to the W planes as it is and
// to the WT planes through a shared-memory transpose, so every global access is a full line.  One thread per element
// with the transposed 4-byte stores going straight to global memory (a 256-byte stride between lanes) took 33 us per
// launch at F = 64, L = 4, 8 tasks and flooded every SM with 3456 CTAs while the main chain's next kernel waited for
// slots; the packs run at the head of every support and tangent pass.
__global__ void __launch_bounds__(256) pack_weights_kernel(ParamLayout pl, const float* __restrict__ theta,
                                                           long long theta_task_stride, float* __restrict__ pack,
                                                           long long pack_task_stride, long long plane_stride, int tag) {
  pdl_prologue(21, tag);
  __shared__ float s_hi[64 * 65], s_lo[64 * 65];              // F <= 64 (maml_b200_create); pitch F + 1: no bank conflicts
  const int F = pl.F, FF = F * F, task = blockIdx.y;
  const int l = 1 + blockIdx.x / 9, tap = blockIdx.x % 9;
  const long long tile = (long long)tap * FF;                  // (tap, c, f) -> tile + c * F + f inside W_l
  const float* src = theta + (long long)task * theta_task_stride + pl.w_off[l] + tile;
  float* p = pack + (long long)task * pack_task_stride + (long long)(l - 1) * 9 * FF + tile;
  for (int i = threadIdx.x; i < FF; i += blockDim.x) {
    const int c = i / F, f = i - c * F;
    const float x = src[i];
    const float hi = tf32_rna(x), lo = tf32_rna(x - hi);
    p[i] = hi;
    p[plane_stride + i] = lo;
    s_hi[f * (F + 1) + c] = hi;
    s_lo[f * (F + 1) + c] = lo;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < FF; i += blockDim.x) {        // WT: (tap, f, c) -> tile + f * F + c
    const int f = i / F, c = i - f * F;
    p[2 * plane_stride + i] = s_hi[f * (F + 1) + c];
    p[3 * plane_stride + i] = s_lo[f * (F + 1) + c];
  }
}

void launch_pack_weights(const ParamLayout& pl, const float* theta, long long theta_task_stride, float* pack,
                         long long pack_task_stride, long long plane_stride, int tasks, cudaStream_t st) {
  ProfScope prof_scope__(PROF_PARAM, 0.0, st);
  if (pl.L <= 1) return;
  dim3 grid(9 * (pl.L - 1), tasks);
  launch_pdl(pack_weights_kernel, dim3(grid), dim3(256), (size_t)(0), st, pl, theta, theta_task_stride, pack, pack_task_stride, plane_stride, launch_tag());
  CUDA_CHECK_LAUNCH();
}

MAML_TRACE_SETTER(trace_set_tc)
