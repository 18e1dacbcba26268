// Shared declarations for the MAML engine (sm_90a: H100).
//
// Activation layout ("padded pixel grid"): every activation-like tensor of block l lives as a
// row-major matrix [n * G_l, C] with G_l = (h_l + 1) * (w_l + 1) (zero padding shared between neighbours): one row per position of the
// zero-padded image, channels innermost (NHWC with an explicit border).  Row index of pixel
// (img, y, x) is img*G + (y+1)*gw + (x+1), gw = w+1.  With that layout a 3x3 / pad-1
// convolution is a GEMM whose A operand for tap (ky,kx) is the SAME matrix shifted by
// s_tap = (ky-1)*gw + (kx-1) rows -- plain 2-D tiles, which is what TMA wants.  Border rows of
// conv inputs are zero and are never written; border rows of conv outputs are garbage and are
// never read (they are masked out of every reduction).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>

#define MAML_MAX_LAYERS 4
#define MAML_MAX_STEPS 8
#define BN_EPS_D 1e-5
#define LEAKY_SLOPE_F 0.01f

struct LayerGeom {
  int h, w;        // conv output (= input) spatial size of this block
  int cin;         // input channels
  int gw, G;       // padded grid with shared padding: gw = w + 1, G = (h + 1) * (w + 1)
  int ph, pw;      // pooled size (floor)
  int pgw, pG, pb; // grid the pooled output is written to: pitch, rows per image, border (1 or 0)
  int guard;       // guard rows before/after a conv-input matrix on this grid (gw + 2)
};

// ---------------------------------------------------------------------------------------------
// launcher argument blocks (plain structs passed by value)
// ---------------------------------------------------------------------------------------------
struct ConvSrc {
  const float* A; long long a_stride;   // A: row 0 of the (guarded) input matrix; per-task stride in floats
  const float* W; long long w_stride;   // weights, per-task stride
  int kc;                               // channels of A (= K per tap), multiple of 16
  int wt;                               // 0: W[tap][kc][ncols]; 1: W[tap][ncols][kc] (dgrad: transposed use)
  int sign;                             // +1: row j + s_tap (conv); -1: row j - s_tap (dgrad)
};

enum { CONV_PLAIN = 0, CONV_FWD_STATS = 1, CONV_TAN_STATS = 2 };

struct ConvArgs {
  ConvSrc src[2]; int nsrc;
  const float* bias; long long bias_stride;    // nullable
  float* out; long long out_stride;
  int rows;                                    // n * G
  int gw, G, h, w;
  int ncols;                                   // output columns (16 * FN)
  int mode;
  const float* zh; long long zh_stride;        // CONV_TAN_STATS: normalised activations of the primal pass
  double* stats; long long stats_stride;       // [task][ncols][2]
  int tasks;
  double alg_flops;                            // algorithmic FLOPs of this launch (valid pixels only; profiling)
  int tag;          // launch sequence number inside the iteration (device trace)
};

struct Conv0Args {                             // first block: K = 9 * C0 is tiny, direct conv
  const float* X; long long x_stride;          // padded-grid image matrix [n*G][C0] (guarded)
  const float* W; long long w_stride;          // [9][C0][F]
  const float* bias; long long bias_stride;
  float* out; long long out_stride;
  int rows, gw, G, h, w, c0, ncols, mode;
  const float* zh; long long zh_stride;
  double* stats; long long stats_stride;
  int tasks;
  double alg_flops;
  int tag;          // launch sequence number inside the iteration (device trace)
};

struct WgradArgs {
  const float* A[2]; long long a_stride[2];    // conv inputs (guarded matrices) [rows][kc]
  const float* D[2]; long long d_stride[2];    // output gradients (zero-border matrices) [rows][ncols]
  long long a_plane[2], d_plane[2];            // tensor-core path: distance (floats) from the fp32 plane to its TF32 hi plane
                                               // (the lo plane follows at the same distance)
  int nsrc;
  int kc, ncols, rows, gw;
  int rows_per_chunk, nchunks;
  float* partial; long long partial_task_stride; long long chunk_stride;  // [task][chunk][9*kc*ncols + ncols]
  int tasks;
  double alg_flops;
  int tag;          // launch sequence number inside the iteration (device trace)
};

struct InputGradArgs {                         // first-block data gradient, written as NCHW images
  const float* D[2]; long long d_stride[2];    // output gradients of the first conv: row 0 of [rows][ncols], per task
  const float* W[2]; long long w_stride;       // first-block weights [9][C0][ncols], per task (D[s] pairs with W[s])
  float* dx; long long dx_stride;              // [n][C0][h][w], per task
  int nsrc;                                    // operand pairs summed into dx (1 or 2)
  int rows, gw, G, h, w, c0, ncols;
  int tasks;
  double alg_flops;
  int tag;          // launch sequence number inside the iteration (device trace)
};

struct BnGeom { int n, h, w, gw, G, ph, pw, pgw, pG, pb, F; };

struct BnActArgs {                // forward: z -> zh (in place), pooled activation p
  float* z; long long z_stride;
  const double* stats; long long stats_stride;     // (sum z, sum z^2)
  const float* gamma; const float* beta;
  float* p; long long p_stride;
  float* p_hi; float* p_lo;                         // nullable: TF32 hi/lo planes of p (same stride)
  BnGeom g; int tasks;
  int tag;          // launch sequence number inside the iteration (device trace)
};

struct BnActTanArgs {             // tangent forward: zdot -> zhdot (in place), pdot
  float* zdot; long long zdot_stride;
  const float* zdot2;              // optional second addend of zdot (same stride): the u-weight conv computed on a side stream
  const float* zh; long long zh_stride;
  const double* stats_fwd; long long stats_fwd_stride;   // primal (sum z, sum z^2) -> r
  const double* stats_tan; long long stats_tan_stride;   // (sum zdot, sum zh*zdot)
  const float* gamma; const float* beta;
  float* pdot; long long pdot_stride;
  float* pdot_hi; float* pdot_lo;
  BnGeom g; int tasks;
  int tag;          // launch sequence number inside the iteration (device trace)
};

struct BnBwdArgs {                // backward reduce / apply (primal)
  const float* dp; long long dp_stride;
  const float* zh; long long zh_stride;
  const double* stats_fwd; long long stats_fwd_stride;
  double* stats_bwd; long long stats_bwd_stride;          // (S1 = sum dy, S2 = sum dy*zh)
  const float* gamma; const float* beta;
  float* dz; long long dz_stride;
  float* dz_hi; float* dz_lo;
  BnGeom g; int tasks;
  int tag;          // launch sequence number inside the iteration (device trace)
};

struct BnBwdTanArgs {             // backward reduce / apply (tangent)
  const float* dp; long long dp_stride;
  const float* dpdot; long long dpdot_stride;
  const float* dpdot2;             // optional second addend of dpdot (same stride)
  const float* zh; long long zh_stride;
  const float* zhdot; long long zhdot_stride;
  const float* dz; long long dz_stride;
  const double* stats_fwd; long long stats_fwd_stride;
  const double* stats_bwd; long long stats_bwd_stride;    // primal (S1, S2)
  const double* stats_tan; long long stats_tan_stride;    // tangent forward (sum zdot, sum zh*zdot)
  double* stats_tbwd; long long stats_tbwd_stride;        // (T1, T2)
  const float* gamma; const float* beta;
  float* dzdot; long long dzdot_stride;
  float* dzdot_hi; float* dzdot_lo;
  BnGeom g; int tasks;
  int tag;          // launch sequence number inside the iteration (device trace)
};

enum { HEAD_SUPPORT = 0, HEAD_TARGET_FWD = 1, HEAD_TARGET_BWD = 2, HEAD_TANGENT = 3,
       HEAD_EXTERNAL_BWD = 4,       // backward of the linear layer for an externally supplied d(loss)/d(logits) (functional operator)
       HEAD_EXTERNAL_TAN = 5 };     // tangent of HEAD_EXTERNAL_BWD with d(loss)/d(logits) held constant; the logits tangent
                                    // goes to logits_out (second-order functional operator)

struct HeadArgs {
  int mode;
  int n, N, D;
  const float* f; long long f_stride;             // [n][D] features (grid order: pixel-major, channel-minor)
  const float* fdot; long long fdot_stride;       // tangent of f (HEAD_TANGENT, HEAD_EXTERNAL_TAN)
  const float* Wfc; const float* bfc; long long theta_stride;     // [N][D], [N] (internal order), per task
  const float* uW; const float* ub; long long u_stride;           // tangent direction (HEAD_TANGENT, HEAD_EXTERNAL_TAN)
  const long long* y; long long y_stride;         // labels [n]
  const float* dl_ext; long long dl_ext_stride;   // HEAD_EXTERNAL_*: upstream gradient w.r.t. the logits [n][N], per task
  float scale;                                    // loss weight folded into dlogits (1 for the support loss)
  float* gW; float* gb; long long g_stride;       // gradient (or H*u) output for the head tensors (chunk 0)
  long long g_chunk_stride;                       // stride between the row-group chunks of gW / gb
  int rows_per_cta;                               // rows of the batch handled by one CTA (grid.x = row groups)
  float* df; long long df_stride;                 // [n][D] gradient (or its tangent) w.r.t. features
  float* loss_out; long long loss_stride;         // per-task scalar (HEAD_TARGET_FWD)
  float* logits_out; long long logits_stride;     // nullable [n][N] (HEAD_EXTERNAL_TAN: the logits tangent, required)
  float* correct_out; long long correct_stride;   // nullable per-task count
  int tasks;
  int tag;          // launch sequence number inside the iteration (device trace)
};

// ---------------------------------------------------------------------------------------------
// parameter-space description (internal fast-weight layout)
// ---------------------------------------------------------------------------------------------
struct ParamLayout {
  int L, F, N, S, per_step_bn;
  int cin[MAML_MAX_LAYERS];
  int pix;                        // pooled pixels of the last block (D = pix * F)
  // internal (per task) fast-weight vector: W_l [9][cin][F], b_l [F], ..., Wfc [N][pix][F], bfc [N]
  long long w_off[MAML_MAX_LAYERS], b_off[MAML_MAX_LAYERS], fcw_off, fcb_off, P;
  // reference-layout flat meta vector offsets
  long long m_w[MAML_MAX_LAYERS], m_b[MAML_MAX_LAYERS], m_beta[MAML_MAX_LAYERS], m_gamma[MAML_MAX_LAYERS];
  long long m_fcw, m_fcb, m_lslr, meta_size;     // lslr: (2L+2) vectors of S+1
  int nseg_inner;                 // 2L + 2 inner tensors
  // per inner segment: internal offset / size and number of gradient chunks in a partial buffer
  long long seg_off[2 * MAML_MAX_LAYERS + 2];
  long long seg_size[2 * MAML_MAX_LAYERS + 2];
};

enum { PR_UPDATE = 0, PR_STORE = 1, PR_SUB = 2 };

struct PartialDesc {              // where each inner segment's gradient chunks live in a partial buffer
  long long off[2 * MAML_MAX_LAYERS + 2];   // offset (floats) of chunk 0 inside the per-task partial block
  long long cstride[2 * MAML_MAX_LAYERS + 2];
  int nchunks[2 * MAML_MAX_LAYERS + 2];
  long long task_stride;
};

// ---------------------------------------------------------------------------------------------
// launchers (kernels_*.cu)
// ---------------------------------------------------------------------------------------------
void launch_prep_x(const float* x, float* xg, long long xg_task_stride, int tasks, int n, int C, int H, int W,
                   cudaStream_t st);
void launch_conv_rows(const ConvArgs& a, cudaStream_t st);
void launch_conv0(const Conv0Args& a, cudaStream_t st);
void launch_wgrad(const WgradArgs& a, cudaStream_t st);
void launch_wgrad0(const WgradArgs& a, cudaStream_t st);
void launch_input_grad0(const InputGradArgs& a, cudaStream_t st);
void launch_bnact(const BnActArgs& a, cudaStream_t st);
void launch_bnact_tan(const BnActTanArgs& a, cudaStream_t st);
void launch_bnbwd_reduce(const BnBwdArgs& a, cudaStream_t st);
void launch_bnbwd_apply(const BnBwdArgs& a, cudaStream_t st);
void launch_bnbwd_tan_reduce(const BnBwdTanArgs& a, cudaStream_t st);
void launch_bnbwd_tan_apply(const BnBwdTanArgs& a, cudaStream_t st);
void launch_bnbwd(const BnBwdArgs& a, cudaStream_t st);          // reduce + apply (one cluster kernel for small blocks)
void launch_bnbwd_tan(const BnBwdTanArgs& a, cudaStream_t st);
bool tail_fusable(const BnGeom& g, int n_rows, int rows_per_cta);
void launch_tail_fused(const BnActArgs& fa, const HeadArgs& ha, const BnBwdArgs& ba, cudaStream_t st);
void launch_tail_tan_fused(const BnActTanArgs& fa, const HeadArgs& ha, const BnBwdTanArgs& ba, cudaStream_t st);
void launch_head(const HeadArgs& a, cudaStream_t st);

void launch_import_theta(const ParamLayout& pl, const float* meta, float* theta0, long long theta_task_stride,
                         int tasks, cudaStream_t st);
void launch_param_reduce(const ParamLayout& pl, const PartialDesc& pd, const float* partial, int mode,
                         const float* theta_in, float* theta_out, float* g_out, float* tbar,
                         const float* meta, int step, long long task_stride, int tasks, cudaStream_t st,
                         int seg_lo = 0, int seg_hi = -1);
void launch_dots_u(const ParamLayout& pl, float* tbar, const float* tgrad, const float* g, float* u, double* abar,
                   const float* meta, int step, long long task_stride, int tasks, cudaStream_t st);

// Peer-memory all-reduce of the result vector (kernels_param.cu: export_kernel publishes, allreduce_kernel sums).
// Every rank owns one cudaMalloc'ed communication block that its peers map through CUDA IPC:
//   [2 slots][slot_stride floats] data | flags[MAML_MAX_RANKS] | seq | counters[2]
// Round `seq` (device-side counter, so a replayed CUDA graph needs no new parameters) uses slot seq & 1.
#define MAML_MAX_RANKS 8
struct CommDev {
  int rank, world;                        // world <= 1: no collective, export writes the caller's result vector
  float* local_data; long long slot_stride;
  unsigned* local_flags;                  // [MAML_MAX_RANKS]: flags[p] = last round rank p has published (written BY p)
  unsigned* seq;                          // current round (starts at 1)
  unsigned* counters;                     // [0]: export blocks done, [1]: reduce blocks done
  const float* peer_data[MAML_MAX_RANKS]; // peer p's data block (peer_data[rank] = local_data)
  unsigned* peer_flags[MAML_MAX_RANKS];   // peer p's flag array
  long long* status;                      // [0] != 0: a wait timed out (peer missing); read by the host after a sync
};

struct ExportArgs {
  CommDev comm;
  ParamLayout pl;
  const float* tbar; long long task_stride;          // [tasks][P]
  const double* abar;                                // [tasks][nseg_inner][MAML_MAX_STEPS] (fp64 dot products)
  const double* stats; long long stats_task_stride;  // stats arena
  long long st_pass_stride, st_layer_stride;         // arena strides (doubles)
  const float* losses;                               // [tasks][MAML_MAX_STEPS] target losses
  const float* correct;                              // [tasks]
  float weights[MAML_MAX_STEPS];                     // target-pass loss weights
  unsigned target_mask; int num_steps; int training;
  int tasks, task_offset, tasks_global;
  int n_s, n_t;
  int hw[MAML_MAX_LAYERS];                           // h*w per block
  float* result;
  int tag;          // launch sequence number inside the iteration (device trace)
};
void launch_export(const ExportArgs& a, cudaStream_t st);
// all ranks' published slots of this round -> `result` (sum in rank order: bit-identical on every rank)
void launch_allreduce(const CommDev& c, float* result, long long n, cudaStream_t st);
// stand-alone publish of an existing vector (timing / tests): copy into this round's slot + signal the peers
void launch_publish(const CommDev& c, const float* src, long long n, cudaStream_t st);

void launch_adam(float* meta, const float* grad, float* m, float* v, long long n, float lr, float bc1, float bc2,
                 const long long* seg_end_host, int nseg, unsigned trainable_mask, unsigned clamp_mask,
                 cudaStream_t st);
void launch_running_update(const float* part_mean, const float* part_var, float* rm, float* rv,
                           const float* decay_dev, int L, int S, int F, cudaStream_t st);
// one sequential EMA update per task from the batch sums of a forward pass (functional operator's side effect)
void launch_running_ema_from_stats(const double* stats, long long stats_task_stride, long long layer_stride, int tasks, float* rm,
                                   float* rv, int L, int S, int F, int step, const int* hw_host, int n, cudaStream_t st);

void launch_episode_gather(const float* dataset, const long long* image_index, const int* rot_k, int B, int N, int K, int T, int C,
                           int H, int W, const float* mean, const float* stdv, float* xs, float* xt, long long* ys, long long* yt,
                           cudaStream_t st);

// stats arena pass ids
enum { PASS_SUP_FWD = 0, PASS_SUP_BWD = 1, PASS_TGT_FWD = 2, PASS_TGT_BWD = 3, PASS_TAN_FWD = 4, PASS_TAN_BWD = 5,
       PASS_KINDS = 6 };

// ---------------------------------------------------------------------------------------------
// Diagnostic switches of one engine handle (environment variables MAML_B200_<NAME>, read once when the handle is
// created: engine.cu read_options).  The value written here is the default.
// ---------------------------------------------------------------------------------------------
struct EngineOptions {
  bool no_graph = false;     // NO_GRAPH (set): eager launches instead of the captured CUDA graph
  bool one_stream = false;   // ONE_STREAM (set): every kernel on the caller's stream
  bool wgrad_tc = true;      // WGRAD_TC=0: FFMA weight gradient for blocks l >= 1
  int tc_split = 8;          // TC_SPLIT: largest split-K cluster size of the wgmma conv, in [1, 8] (1 = off)
  int tc_nb = 0;             // TC_NB: B ring depth of main-chain convs, in [2, 8] (0 = by regime)
  bool bn_fuse = true;       // BN_FUSE=0: BatchNorm backward always as two kernels (reduce, apply)
  bool tail_fuse = true;     // TAIL_FUSE=0: last block / head / its BatchNorm backward as separate kernels
  int tail_onchip = 3;       // TAIL_ONCHIP: fused last-block kernels on chip, bit 0 primal, bit 1 tangent
  int pdl = -1;              // PDL: programmatic dependent launch on the main chain, 0 off / 1 on (-1 = by regime)
  int tc_timeline = -1;      // TC_TIMELINE: clock64 milestones of one conv CTA of block l (0 = any block, -1 = off)
  std::string graph_dot;     // GRAPH_DOT: file the captured graph is written to (empty = none)
};

// ---------------------------------------------------------------------------------------------
// Launch context: what the launchers need to know about the handle whose call is enqueueing work.  The engine installs
// it for the duration of each handle call (engine.cu LaunchScope); with none installed PDL is off, the options are the
// defaults and nothing is profiled.
// ---------------------------------------------------------------------------------------------
struct Profiler;
struct LaunchContext {
  const EngineOptions* opt;
  bool pdl;                        // launches on main_stream take programmatic dependent launch
  cudaStream_t main_stream;        // stream of the call's main chain (null: the call has none)
  Profiler* prof;                  // non-null while the handle is profiling
};
const LaunchContext& launch_ctx();

// ---------------------------------------------------------------------------------------------
// Programmatic dependent launch: a kernel launched with the programmatic-stream-serialization attribute starts with
// `griddepcontrol.launch_dependents; griddepcontrol.wait;` -- the next kernel of the stream is scheduled while this one
// still runs (its launch latency and set-up overlap) and blocks until this grid has completed and flushed.  Only
// non-cluster launches on the main chain take the attribute, and only in the latency-bound regime (maml_b200_create)
// unless MAML_B200_PDL says otherwise.
// ---------------------------------------------------------------------------------------------
inline bool pdl_allowed(cudaStream_t st) {
  const LaunchContext& c = launch_ctx();
  return c.pdl && st == c.main_stream;
}
int num_sms();                     // streaming multiprocessors of the current device (queried once)

// Device-side launch trace (debug; maml_b200_trace): CTA (0,0,0) of every kernel appends (globaltimer ns << 8 | kernel
// id) to a buffer -> the start-time sequence of one captured iteration, the only timeline available without nsys.
// One pointer copy per translation unit (no relocatable device code), all set to the same buffer; null = off.
// The trace is armed through a bit of the launch tag, i.e. a kernel ARGUMENT: with tracing off no kernel touches memory for
// it.  Before, every thread of every kernel began with a load of the buffer pointer (a __device__ variable) and a branch on
// it -- a dependent global load in front of the first useful instruction.  Enabling the trace drops the handle's cached CUDA graphs so that they are re-captured with armed tags.
#define MAML_TRACE_ARMED 0x40000000
static __device__ unsigned long long* t_trace_buf = nullptr;
#define MAML_TRACE_SETTER(fn) void fn(unsigned long long* p) { cudaMemcpyToSymbol(t_trace_buf, &p, sizeof(p)); }
#define MAML_TRACE_CAP 4094
__device__ __forceinline__ void trace_mark(int kid, int tag = 0) {
  if (!(tag & MAML_TRACE_ARMED)) return;
  unsigned long long* t = t_trace_buf;
  if (t != nullptr && threadIdx.x == 0 && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) {
    unsigned long long now;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
    const unsigned long long slot = atomicAdd(t, 1ULL);
    // entry: [63:20] globaltimer ns (44 bits), [19:8] launch tag, [7:0] kernel id (bit 7 = end-of-CTA mark)
    if (slot < MAML_TRACE_CAP) t[1 + slot] = (now << 20) | ((unsigned long long)(tag & 0xfff) << 8) | (unsigned long long)(kid & 0xff);
  }
}
void trace_set_conv(unsigned long long* p);
void trace_set_bn(unsigned long long* p);
void trace_set_head(unsigned long long* p);
void trace_set_param(unsigned long long* p);
void trace_set_tc(unsigned long long* p);

__device__ __forceinline__ void pdl_prologue(int kid = 0, int tag = 0) {
  trace_mark(kid, tag);
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
template <typename... KArgs, typename... Args>
inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_allowed(st) ? 1 : 0;
  cfg.attrs = attr; cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

extern long long g_launch_counter;   // bumped by every launcher
extern long long g_launch_base;      // value of g_launch_counter when the current iteration started to be enqueued
extern int g_trace_flag;             // MAML_TRACE_ARMED while maml_b200_trace(h, 1) is in effect, else 0
inline int launch_tag() { return (int)(g_launch_counter - g_launch_base) | g_trace_flag; }
template <class A> inline A tagged(const A& a) { A t = a; t.tag = launch_tag(); return t; }

#define CUDA_CHECK_LAUNCH() do { g_launch_counter++; } while (0)

// ---------------------------------------------------------------------------------------------
// optional per-launch profiling with CUDA events on the launching stream (bench.py roofline leg)
// ---------------------------------------------------------------------------------------------
enum { PROF_CONV = 0, PROF_CONV0 = 1, PROF_WGRAD = 2, PROF_WGRAD0 = 3, PROF_BN = 4, PROF_HEAD = 5, PROF_PARAM = 6,
       PROF_CATS = 7 };
void prof_begin(Profiler* p, int cat, double flops, cudaStream_t st);
void prof_end(Profiler* p, cudaStream_t st);
struct ProfScope {
  cudaStream_t st; Profiler* prof;
  ProfScope(int cat, double flops, cudaStream_t s) : st(s), prof(launch_ctx().prof) { if (prof) prof_begin(prof, cat, flops, st); }
  ~ProfScope() { if (prof) prof_end(prof, st); }
};
