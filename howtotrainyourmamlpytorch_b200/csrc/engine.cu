// Host-side orchestration + C ABI (include/maml_b200.h) of the H100 MAML / MAML++ engine.
//
// One call of maml_b200_meta_batch_fwd_bwd replaces, for the local shard of tasks, the reference's
//   forward()   few_shot_learning_system.py:170-263  (task loop x inner-step loop, Python, autograd)
//   backward()  few_shot_learning_system.py:331      (second-order reverse sweep)
// with a fixed sequence of kernels batched over tasks (grid.y = task):
//   phase A (unroll):   for s: support forward -> hand-rolled support gradient -> LSLR update,
//                       target forward (+ its backward, stored as tgrad[s]) at theta^{s+1}
//   phase B (reverse):  for s = S-1..0: tbar += tgrad[s]; abar[s] = -<tbar, g_s>; u = alpha_s * tbar;
//                       Hessian-vector product by a forward-mode tangent pass; tbar -= H u
// No host synchronisation, no fast-weight round trip to the host; all intermediates stay in HBM / L2.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <string>
#include <vector>

#include "../../include/maml_b200.h"
#include "common.cuh"
#include "tc_common.cuh"

static thread_local std::string g_err;
static int fail(const std::string& m) { g_err = m; return 1; }

#define CK(call) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) { \
  return fail(std::string(#call) + ": " + cudaGetErrorString(e__)); } } while (0)

static inline long long rup(long long x, long long m) { return (x + m - 1) / m * m; }

// ---------------------------------------------------------------------------------------------
// per-launch profiler (CUDA events on the launching stream); off unless maml_b200_profile(h, 1)
// ---------------------------------------------------------------------------------------------
struct Profiler {
  struct Rec { int cat; double flops; cudaEvent_t a, b; };
  std::vector<Rec> recs;
  std::vector<cudaEvent_t> pool;
  size_t used = 0;
  cudaEvent_t get() {
    if (used == pool.size()) { cudaEvent_t e; cudaEventCreate(&e); pool.push_back(e); }
    return pool[used++];
  }
  void reset() { recs.clear(); used = 0; }
  ~Profiler() { for (auto e : pool) cudaEventDestroy(e); }
};
void prof_begin(Profiler* p, int cat, double flops, cudaStream_t st) {
  Profiler::Rec r; r.cat = cat; r.flops = flops; r.a = p->get(); r.b = p->get();
  cudaEventRecord(r.a, st);
  p->recs.push_back(r);
}
void prof_end(Profiler* p, cudaStream_t st) { cudaEventRecord(p->recs.back().b, st); }

// Every diagnostic switch of the engine, read from the environment once per handle (maml_b200_create).
static EngineOptions read_options() {
  auto flag = [](const char* name, bool def) { const char* v = getenv(name); return v ? atoi(v) != 0 : def; };
  auto num = [](const char* name, int def) { const char* v = getenv(name); return v ? atoi(v) : def; };
  auto clamp = [](int v, int lo, int hi) { return std::max(lo, std::min(hi, v)); };
  EngineOptions o;
  o.no_graph = getenv("MAML_B200_NO_GRAPH") != nullptr;
  o.one_stream = getenv("MAML_B200_ONE_STREAM") != nullptr;
  o.wgrad_tc = flag("MAML_B200_WGRAD_TC", o.wgrad_tc);
  o.tc_split = clamp(num("MAML_B200_TC_SPLIT", o.tc_split), 1, 8);
  if (getenv("MAML_B200_TC_NB")) o.tc_nb = clamp(num("MAML_B200_TC_NB", 0), 2, 8);
  o.bn_fuse = flag("MAML_B200_BN_FUSE", o.bn_fuse);
  o.tail_fuse = flag("MAML_B200_TAIL_FUSE", o.tail_fuse);
  o.tail_onchip = num("MAML_B200_TAIL_ONCHIP", o.tail_onchip);
  if (const char* v = getenv("MAML_B200_PDL")) o.pdl = atoi(v) != 0 ? 1 : 0;
  if (getenv("MAML_B200_TC_TIMELINE")) o.tc_timeline = std::max(0, num("MAML_B200_TC_TIMELINE", 0));
  if (const char* v = getenv("MAML_B200_GRAPH_DOT")) o.graph_dot = v;
  return o;
}

struct PassSet {            // activation buffers of one kind of pass (support: S slots, target / tangent: 1)
  int n = 0, slots = 0;
  float* xg = nullptr; long long xg_stride = 0;                       // block-0 input grid (row 0), per task
  float* ain[MAML_MAX_LAYERS + 1] = {}; long long ain_sz[MAML_MAX_LAYERS + 1] = {};   // per (task,slot) size; ptr at row 0
  float* zh[MAML_MAX_LAYERS] = {}; long long zh_sz[MAML_MAX_LAYERS] = {};
  float* dz[MAML_MAX_LAYERS] = {}; long long dz_sz[MAML_MAX_LAYERS] = {};
  float* dp[MAML_MAX_LAYERS] = {}; long long dp_sz[MAML_MAX_LAYERS] = {};
  // conv inputs of blocks l >= 1 (ain) and output gradients (dz) are stored as three planes: fp32, TF32-hi, TF32-lo
  // (the hi/lo planes feed the wgmma conv kernel through TMA; same geometry incl. guards)
  float* ain_base[MAML_MAX_LAYERS + 1] = {}; long long ain_plane[MAML_MAX_LAYERS + 1] = {};
  float* dz_base[MAML_MAX_LAYERS] = {}; long long dz_plane[MAML_MAX_LAYERS] = {};
  CUtensorMap ain_map[MAML_MAX_LAYERS][2];   // [layer][hi/lo]
  CUtensorMap dz_map[MAML_MAX_LAYERS][2];
};

struct ChunkPlan { int rows_per_chunk[MAML_MAX_LAYERS]; int nchunks[MAML_MAX_LAYERS]; PartialDesc pd; long long size; int head_groups; };
// rows of a batch one head CTA handles: small batches (<= 16 rows: the Omniglot 5-way passes) stay in ONE CTA so that the
// last block / head / BatchNorm-backward fusion applies; larger ones are cut into groups of 4 rows -- the head of a 75-row
// Mini-ImageNet target pass would otherwise run as 5 latency-bound CTAs per task
static inline int head_rows(int n) { return n <= 16 ? 16 : 4; }

struct maml_b200_handle {
  maml_b200_config cfg;
  EngineOptions opt;
  int L, F, N, S, C, H, W, n_s, n_t, maxT, D, pix;
  LayerGeom geo[MAML_MAX_LAYERS];
  ParamLayout pl;
  long long Ppad;
  // meta segments
  std::vector<long long> seg_off, seg_size;
  // workspace
  char* ws = nullptr; long long ws_bytes = 0;
  PassSet sup, tgt, tan, tan2;      // tan2: second addends of the tangent pass (u-weight convs, computed on a side stream)
  float *theta = nullptr, *g = nullptr, *tgrad = nullptr, *tbar = nullptr, *u = nullptr;
  float *sup_partial = nullptr, *tgt_partial = nullptr;
  ChunkPlan plan_sup, plan_tgt;
  double* stats = nullptr; long long stats_task_stride = 0, st_pass_stride = 0, st_layer_stride = 0, stats_count = 0;
  float *losses = nullptr, *correct = nullptr, *decay_dev = nullptr;
  double* abar = nullptr;
  // layer-norm handles (cfg.norm_layer = 1): per-image sums [task][pass kind][step][block][image][2] and the bias-gradient
  // rows [task][2][S][pl.lnb_off[L]] (see ExportArgs::lnb)
  bool ln = false;
  double* ln_stats = nullptr; long long ln_task_stride = 0, ln_pass_stride = 0;
  float* lnb = nullptr;
  long long* zero_labels = nullptr;   // [max(n_s, n_t)] zeros (label-free forward)
  float* pinned = nullptr;            // host staging ring for small per-call scalars (16 slots x 32 floats)
  int pin_slot = 0;
  long long last_launches = 0;
  int last_tasks = 0;
  // the functional call (net_forward / net_backward / net_hvp) whose buffers the handle holds; FN_NONE after any other
  // call that launched, or failed after launching.  The entries that read those buffers check it first (require_call).
  int fn_kind = 0, fn_tasks = 0, fn_step = 0;
  // forward-mode buffers outside the workspace, allocated by the first call that needs them (handles that never see
  // forward mode keep their footprint): the image tangent on the support grid, zero d(logits) for the logits-tangent head
  float* xdot_g = nullptr;
  float* zero_dl = nullptr;
  Profiler prof;
  bool profiling = false;             // maml_b200_profile(h, 1): this handle's launches are recorded into prof
  // side streams / events for fork-join inside one iteration, CUDA-graph cache
  cudaStream_t s_cap = nullptr, s_tgt = nullptr, s_tgt2 = nullptr, s_wg = nullptr;
  int tgt_slots = 1;       // target passes of consecutive steps are independent: double-buffered on two streams (min(S, 2))
  cudaEvent_t ev_fork = nullptr, ev_wg = nullptr, ev_pack = nullptr, ev_tgt[MAML_MAX_STEPS] = {};
  cudaEvent_t ev_pre[2 * MAML_MAX_LAYERS] = {};     // tangent pre-computed addends: [l] forward conv, [MAX_LAYERS + l] dgrad
  bool use_graphs = true;
  bool pdl = false;                                   // programmatic dependent launch on the main chain (see common.cuh)
  int nb_main = 8;                                    // shared-memory B ring depth of the tensor-core conv kernel (see maml_b200_create)
  // results produced on s_wg (upper-block parameter reduction, weight packs) that the main chain has not joined yet:
  // consumed right before the first kernel that reads them (block 1's convolution / the head)
  bool wg_pending = false;
  struct GraphEntry { maml_b200_iter_args it; const void* p[7]; cudaGraphExec_t exec; long long launches; unsigned long long stamp; };
  std::vector<GraphEntry> graphs;
  unsigned long long graph_clock = 0;
  // tensor-core path (blocks l >= 1 when F % 32 == 0)
  bool use_tc = false;
  float *pack_theta = nullptr, *pack_u = nullptr;       // [4 planes][steps][T][(L-1)*9*F*F]
  long long pack_theta_plane = 0, pack_u_plane = 0, pack_task = 0;
  CUtensorMap theta_map[4], u_map[4];                   // planes: W hi, W lo, WT hi, WT lo
  // multi-GPU: peer-memory all-reduce of the result vector (maml_b200_comm_*)
  CommDev comm{};                                       // world <= 1 until connected
  char* comm_block = nullptr; long long comm_bytes = 0;
  void* comm_opened[MAML_MAX_RANKS] = {};               // peer blocks mapped with cudaIpcOpenMemHandle
  bool comm_connected = false;
};

enum { FN_NONE = 0, FN_FORWARD = 1, FN_BACKWARD = 2, FN_HVP = 4 };     // bits: require_call takes a set of kinds
static void record_call(maml_b200_handle* h, int kind, int n_tasks, int num_step) {
  h->fn_kind = kind; h->fn_tasks = n_tasks; h->fn_step = num_step;
}
static std::string call_names(int kinds) {
  std::string s;
  for (int k : {FN_FORWARD, FN_BACKWARD, FN_HVP})
    if (kinds & k)
      s += std::string(s.empty() ? "" : " or ") + (k == FN_FORWARD ? "maml_b200_net_forward" : k == FN_BACKWARD ? "maml_b200_net_backward" : "maml_b200_net_hvp");
  return s;
}
// An entry that reads the buffers of an earlier functional call first checks the handle's record of that call: its kind
// must be one of `kinds`, with the same n_tasks and (num_step >= 0) the same num_step.  Fails without touching the record.
static int require_call(const maml_b200_handle* h, int kinds, int n_tasks, int num_step, const char* entry) {
  const std::string e(entry), last = call_names(h->fn_kind);
  if (!(h->fn_kind & kinds)) return fail(e + " must immediately follow " + call_names(kinds) + " on this handle");
  if (n_tasks != h->fn_tasks) return fail(e + ": n_tasks differs from the preceding " + last);
  if (num_step >= 0 && num_step != h->fn_step) return fail(e + ": num_step differs from the preceding " + last);
  return 0;
}

// launch context of the handle call in progress on this thread (common.cuh); the default one has PDL off
static const EngineOptions g_default_options;
static thread_local LaunchContext g_launch_ctx{&g_default_options, false, nullptr, nullptr};
const LaunchContext& launch_ctx() { return g_launch_ctx; }

// Installs a handle's launch context for the duration of one call and restores the previous one.  Calls that enqueue an
// iteration chain pass its main stream and launch with the handle's PDL mode; the other calls launch without PDL.
struct LaunchScope {
  LaunchContext saved;
  explicit LaunchScope(maml_b200_handle* h) : LaunchScope(h, false, nullptr) {}
  LaunchScope(maml_b200_handle* h, cudaStream_t main) : LaunchScope(h, h->pdl, main) {}
  ~LaunchScope() { g_launch_ctx = saved; }
 private:
  LaunchScope(maml_b200_handle* h, bool pdl, cudaStream_t main) : saved(g_launch_ctx) {
    g_launch_ctx = LaunchContext{&h->opt, pdl, main, h->profiling ? &h->prof : nullptr};
  }
};

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

extern "C" int maml_b200_abi_version(void) { return MAML_B200_ABI_VERSION; }
extern "C" const char* maml_b200_last_error(void) { return g_err.c_str(); }

static void build_geometry(maml_b200_handle* h) {
  int hh = h->H, ww = h->W, cin = h->C;
  for (int l = 0; l < h->L; ++l) {
    LayerGeom& g = h->geo[l];
    g.h = hh; g.w = ww; g.cin = cin;
    // shared zero padding: column 0 of a grid row is the left pad of that row AND the right pad of the row above,
    // row 0 of an image block is its top pad AND the bottom pad of the image before it (the guard rows close the last
    // image) -> (h+1)(w+1) rows per image instead of (h+2)(w+2); tap shifts are unchanged ((ky-1) gw + (kx-1))
    g.gw = ww + 1; g.G = (hh + 1) * (ww + 1);
    g.ph = hh / 2; g.pw = ww / 2;
    if (l < h->L - 1) { g.pgw = g.pw + 1; g.pG = (g.ph + 1) * (g.pw + 1); g.pb = 1; }
    else { g.pgw = g.pw; g.pG = g.ph * g.pw; g.pb = 0; }
    g.guard = g.gw + 2;
    hh = g.ph; ww = g.pw; cin = h->F;
  }
  h->pix = h->geo[h->L - 1].ph * h->geo[h->L - 1].pw;
  h->D = h->pix * h->F;
}

static void build_layout(maml_b200_handle* h) {
  ParamLayout& pl = h->pl;
  memset(&pl, 0, sizeof(pl));
  pl.L = h->L; pl.F = h->F; pl.N = h->N; pl.S = h->S; pl.pix = h->pix;
  pl.ln = h->ln ? 1 : 0;
  pl.per_step_bn = h->ln ? 0 : h->cfg.per_step_bn;       // layer norm: no per-step parameters, no running statistics
  // inner-loop gamma / beta are one [F] row each, whatever per_step_bn is (the running statistics stay per step)
  pl.inner_bn = h->cfg.inner_bn ? 1 : 0;
  pl.per_step_gb = pl.per_step_bn && !pl.inner_bn;
  const int spb = seg_per_block(pl);
  long long o = 0, m = 0;
  const long long bnsz = (long long)(pl.per_step_gb ? h->S : 1) * h->F;
  for (int l = 0; l < h->L; ++l) {
    pl.cin[l] = h->geo[l].cin;
    const long long wsz = 9LL * pl.cin[l] * h->F;
    pl.w_off[l] = o; o += wsz;
    pl.b_off[l] = o; o += h->F;
    if (pl.inner_bn) { pl.beta_off[l] = o; o += h->F; pl.gamma_off[l] = o; o += h->F; }
    pl.m_w[l] = m; h->seg_off.push_back(m); h->seg_size.push_back(wsz); m += wsz;
    pl.m_b[l] = m; h->seg_off.push_back(m); h->seg_size.push_back(h->F); m += h->F;
    if (h->ln) {
      // norm_layer.bias [F, h_l, w_l]; the frozen all-ones weight is not a meta-parameter (the reference's Adam skips it)
      const long long lsz = (long long)h->F * h->geo[l].h * h->geo[l].w;
      pl.m_lnb[l] = m; h->seg_off.push_back(m); h->seg_size.push_back(lsz); m += lsz;
      pl.lnb_off[l + 1] = pl.lnb_off[l] + lsz;
    } else {
      pl.m_beta[l] = m; h->seg_off.push_back(m); h->seg_size.push_back(bnsz); m += bnsz;
      pl.m_gamma[l] = m; h->seg_off.push_back(m); h->seg_size.push_back(bnsz); m += bnsz;
    }
    pl.seg_off[spb * l] = pl.w_off[l]; pl.seg_size[spb * l] = wsz;
    pl.seg_off[spb * l + 1] = pl.b_off[l]; pl.seg_size[spb * l + 1] = h->F;
    if (pl.inner_bn) {
      pl.seg_off[spb * l + 2] = pl.beta_off[l]; pl.seg_size[spb * l + 2] = h->F;
      pl.seg_off[spb * l + 3] = pl.gamma_off[l]; pl.seg_size[spb * l + 3] = h->F;
    }
  }
  pl.fcw_off = o; o += (long long)h->N * h->D;
  pl.fcb_off = o; o += h->N;
  pl.P = o;
  pl.m_fcw = m; h->seg_off.push_back(m); h->seg_size.push_back((long long)h->N * h->D); m += (long long)h->N * h->D;
  pl.m_fcb = m; h->seg_off.push_back(m); h->seg_size.push_back(h->N); m += h->N;
  pl.nseg_inner = spb * h->L + 2;
  pl.seg_off[spb * h->L] = pl.fcw_off; pl.seg_size[spb * h->L] = (long long)h->N * h->D;
  pl.seg_off[spb * h->L + 1] = pl.fcb_off; pl.seg_size[spb * h->L + 1] = h->N;
  pl.m_lslr = m;
  for (int k = 0; k < pl.nseg_inner; ++k) { h->seg_off.push_back(m); h->seg_size.push_back(h->S + 1); m += h->S + 1; }
  pl.meta_size = m;
  h->Ppad = rup(pl.P, 64);
}

static void plan_chunks(maml_b200_handle* h, int n, ChunkPlan* cp) {
  long long off = 0;
  memset(&cp->pd, 0, sizeof(cp->pd));     // inner-loop beta / gamma segments have no chunks (nchunks 0)
  const int spb = seg_per_block(h->pl);
  for (int l = 0; l < h->L; ++l) {
    const long long rows = (long long)n * h->geo[l].G;
    int nch, rpc;
    if (l == 0) {
      nch = (int)std::min<long long>(512, std::max<long long>(1, (rows + 63) / 64));
    } else {
      // ONE wgrad CTA per SM, and 3 filter rows x tasks x chunks should just fill one slot per SM -- 720 CTAs (128-row
      // chunks at 8 tasks) ran as 1.2 waves = 2x the time.  wgrad_tc_row_kernel: a CTA holds its SM's whole register file
      // (384 threads x 168 registers), so a second CTA could only run behind the first.  wgrad_row_kernel<4,4>: 105
      // registers x 256 threads, whose 48 independent accumulators per thread keep the FMA pipe fed with 8 warps; a
      // second CTA per SM would take the register file away from the main chain's kernels running beside it.
      // Chunks are multiples of 16 rows: a partial 32-row stage of the tensor-core kernel costs a full one, but the rows
      // of a chunk (and so the summation order of the gradient) do not depend on which kernel runs
      long long want = std::max<long long>(1, num_sms() / (3LL * h->maxT));
      nch = (int)std::min<long long>(std::min<long long>(64, want), std::max<long long>(1, (rows + 15) / 16));
    }
    rpc = (int)rup((rows + nch - 1) / nch, 16);
    nch = (int)((rows + rpc - 1) / rpc);
    cp->rows_per_chunk[l] = rpc; cp->nchunks[l] = nch;
    const long long cs = 9LL * h->geo[l].cin * h->F + h->F;
    cp->pd.off[spb * l] = off; cp->pd.cstride[spb * l] = cs; cp->pd.nchunks[spb * l] = nch;
    cp->pd.off[spb * l + 1] = off + 9LL * h->geo[l].cin * h->F; cp->pd.cstride[spb * l + 1] = cs; cp->pd.nchunks[spb * l + 1] = nch;
    off += cs * nch;
  }
  // head: one gradient chunk per row group of the batch (gW [N][D] followed by gb [N] inside each chunk)
  const int hg = (n + head_rows(n) - 1) / head_rows(n);
  const long long hcs = (long long)h->N * h->D + h->N;
  cp->head_groups = hg;
  cp->pd.off[spb * h->L] = off; cp->pd.cstride[spb * h->L] = hcs; cp->pd.nchunks[spb * h->L] = hg;
  cp->pd.off[spb * h->L + 1] = off + (long long)h->N * h->D; cp->pd.cstride[spb * h->L + 1] = hcs; cp->pd.nchunks[spb * h->L + 1] = hg;
  off += hcs * hg;
  cp->size = rup(off, 64);
  cp->pd.task_stride = cp->size;
}

// bump allocator over the workspace (two passes: size, then assign)
struct Bump {
  char* base; long long off;
  float* f(long long count) { float* p = base ? (float*)(base + off) : nullptr; off += rup(count * 4, 256); return p; }
  double* d(long long count) { double* p = base ? (double*)(base + off) : nullptr; off += rup(count * 8, 256); return p; }
};

// 2-D fp32 tensor map [rows][cols] with a [box_rows][32] box, SWIZZLE_128B, zero fill out of bounds
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}
static int make_map(CUtensorMap* m, const float* base, long long rows, int cols, int box_rows,
                    CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail("cuTensorMapEncodeTiled entry point not available");
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)cols * sizeof(float)};
  cuuint32_t box[2] = {32u, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled failed with code " + std::to_string((int)r));
  return 0;
}
static int make_pass_maps(maml_b200_handle* h, PassSet& ps, bool has_dz) {
  for (int l = 1; l < h->L; ++l) {
    for (int pl = 0; pl < 2; ++pl) {
      const int rp = tc_conv_rpad(h->geo[l].gw);       // one TMA box = the 128-row tile plus its halo
      if (make_map(&ps.ain_map[l][pl], ps.ain_base[l] + (pl + 1) * ps.ain_plane[l], ps.ain_plane[l] / h->F, h->F, rp)) return 1;
      if (has_dz && make_map(&ps.dz_map[l][pl], ps.dz_base[l] + (pl + 1) * ps.dz_plane[l], ps.dz_plane[l] / h->F, h->F, rp)) return 1;
    }
  }
  return 0;
}
static int make_all_maps(maml_b200_handle* h) {
  if (!h->use_tc) return 0;
  if (make_pass_maps(h, h->sup, true) || make_pass_maps(h, h->tgt, true) || make_pass_maps(h, h->tan, true)) return 1;
  for (int pl = 0; pl < 4; ++pl) {
    if (make_map(&h->theta_map[pl], h->pack_theta + pl * h->pack_theta_plane, h->pack_theta_plane / h->F, h->F, h->F)) return 1;
    if (make_map(&h->u_map[pl], h->pack_u + pl * h->pack_u_plane, h->pack_u_plane / h->F, h->F, h->F)) return 1;
  }
  if (tc_conv_prepare()) return fail("cudaFuncSetAttribute(max dynamic shared memory) failed for the wgmma conv / weight-gradient kernels");
  return 0;
}

static void carve_pass(maml_b200_handle* h, Bump& b, PassSet& ps, int n, int slots, bool need_x, bool need_bwd) {
  ps.n = n; ps.slots = slots;
  const long long T = h->maxT;
  if (need_x) {
    const long long gr = (long long)h->geo[0].guard * h->C;
    const long long body = (long long)n * h->geo[0].G * h->C;
    ps.xg_stride = rup(body + 2 * gr, 64);
    float* p = b.f(ps.xg_stride * T);
    ps.xg = p ? p + gr : nullptr;
  }
  for (int l = 1; l < h->L; ++l) {
    const long long gr = (long long)h->geo[l].guard * h->F;
    const long long body = (long long)n * h->geo[l].G * h->F;
    ps.ain_sz[l] = rup(body + 2 * gr, 192);
    ps.ain_plane[l] = ps.ain_sz[l] * T * slots;
    float* p = b.f(ps.ain_plane[l] * 3);
    ps.ain_base[l] = p;
    ps.ain[l] = p ? p + gr : nullptr;
  }
  ps.ain_sz[h->L] = rup((long long)n * h->D, 64);
  ps.ain[h->L] = b.f(ps.ain_sz[h->L] * T * slots);
  for (int l = 0; l < h->L; ++l) {
    ps.zh_sz[l] = rup((long long)n * h->geo[l].G * h->F, 64);
    ps.zh[l] = b.f(ps.zh_sz[l] * T * slots);
    if (need_bwd) {
      const long long gr = (long long)h->geo[l].guard * h->F;
      ps.dz_sz[l] = rup((long long)n * h->geo[l].G * h->F + 2 * gr, 192);
      ps.dz_plane[l] = ps.dz_sz[l] * T * slots;
      float* p = b.f(ps.dz_plane[l] * 3);
      ps.dz_base[l] = p;
      ps.dz[l] = p ? p + gr : nullptr;
      ps.dp_sz[l] = rup((long long)n * h->geo[l].pG * h->F, 64);
      ps.dp[l] = b.f(ps.dp_sz[l] * T * slots);
    }
  }
}

static void carve(maml_b200_handle* h, Bump& b) {
  const long long T = h->maxT;
  carve_pass(h, b, h->sup, h->n_s, h->S, true, true);
  h->tgt_slots = std::min(h->S, 2);
  carve_pass(h, b, h->tgt, h->n_t, (h->cfg.reserved & 1) ? h->S : h->tgt_slots, true, true);   // reserved bit 0: keep every target pass (tests)
  carve_pass(h, b, h->tan, h->n_s, 1, false, true);
  carve_pass(h, b, h->tan2, h->n_s, 1, false, true);
  h->theta = b.f((long long)(h->S + 1) * T * h->Ppad);
  h->g = b.f((long long)h->S * T * h->Ppad);
  h->tgrad = b.f((long long)h->S * T * h->Ppad);
  h->tbar = b.f(T * h->Ppad);
  h->u = b.f(T * h->Ppad);
  h->pack_task = (long long)(h->L - 1) * 9 * h->F * h->F;
  h->pack_theta_plane = (long long)(h->S + 1) * T * h->pack_task;
  h->pack_u_plane = T * h->pack_task;
  if (h->use_tc && h->L > 1) {
    h->pack_theta = b.f(4 * h->pack_theta_plane);
    h->pack_u = b.f(4 * h->pack_u_plane);
  }
  h->sup_partial = b.f(T * h->plan_sup.size);
  h->tgt_partial = b.f(T * h->plan_tgt.size * h->tgt_slots);
  h->st_layer_stride = (long long)h->F * 2;
  h->st_pass_stride = (long long)h->L * h->F * 2;
  h->stats_task_stride = (long long)PASS_KINDS * MAML_MAX_STEPS * h->st_pass_stride;
  h->stats_count = h->stats_task_stride * T;
  h->stats = b.d(h->stats_count);
  h->losses = b.f(T * MAML_MAX_STEPS);
  h->correct = b.f(T);
  h->abar = b.d(T * h->pl.nseg_inner * MAML_MAX_STEPS);
  h->decay_dev = b.f(MAML_MAX_STEPS);
  h->zero_labels = (long long*)b.d(std::max(h->n_s, h->n_t));
  if (h->ln) {
    h->ln_pass_stride = (long long)MAML_MAX_STEPS * h->L * std::max(h->n_s, h->n_t) * 2;
    h->ln_task_stride = PASS_KINDS * h->ln_pass_stride;
    h->ln_stats = b.d(h->ln_task_stride * T);
    h->lnb = b.f(T * 2 * h->S * h->pl.lnb_off[h->L]);
  }
}

extern "C" int maml_b200_create(const maml_b200_config* cfg, maml_b200_handle** out) {
  if (!cfg || !out) return fail("null argument");
  if (cfg->filters % 16 != 0 || cfg->filters < 16 || cfg->filters > 64) return fail("filters must be a multiple of 16 in [16, 64]");
  if (cfg->num_stages < 1 || cfg->num_stages > MAML_MAX_LAYERS) return fail("num_stages must be in [1, 4]");
  if (cfg->inner_steps < 1 || cfg->inner_steps > MAML_MAX_STEPS) return fail("inner_steps must be in [1, 8]");
  if (cfg->channels < 1 || cfg->channels > 4) return fail("channels must be in [1, 4]");
  if (cfg->max_tasks < 1) return fail("max_tasks must be >= 1");
  if (cfg->norm_layer != 0 && cfg->norm_layer != 1) return fail("norm_layer must be 0 (batch norm) or 1 (layer norm)");
  if (cfg->inner_bn != 0 && cfg->inner_bn != 1) return fail("inner_bn must be 0 or 1");
  if (cfg->inner_bn && cfg->norm_layer == 1) return fail("inner_bn (inner-loop BatchNorm gamma / beta) needs norm_layer 0 (batch norm)");
  if (cfg->n_way < 2 || cfg->n_way > 32) return fail("n_way must be in [2, 32]");
  const int n_s = cfg->n_way * cfg->k_shot, n_t = cfg->n_way * cfg->t_target;
  if (n_s < 1 || n_t < 1 || n_s > 128 || n_t > 128) return fail("N*K and N*T must be in [1, 128]");
  {
    int hh = cfg->height, ww = cfg->width;
    for (int l = 0; l < cfg->num_stages; ++l) { if (hh < 2 || ww < 2) return fail("image too small for num_stages"); hh /= 2; ww /= 2; }
  }
  maml_b200_handle* h = new maml_b200_handle();
  h->cfg = *cfg;
  h->opt = read_options();
  h->L = cfg->num_stages; h->F = cfg->filters; h->N = cfg->n_way; h->S = cfg->inner_steps;
  h->C = cfg->channels; h->H = cfg->height; h->W = cfg->width; h->n_s = n_s; h->n_t = n_t; h->maxT = cfg->max_tasks;
  h->ln = cfg->norm_layer == 1;
  build_geometry(h);
  build_layout(h);
  // tensor-core (wgmma / TMA, 3xTF32) convolutions for blocks l >= 1; reserved bit 1 forces the fp32 FFMA kernels (tests)
  h->use_tc = (h->L > 1) && !(cfg->reserved & 2);
  // (any F in {16, 32, 48, 64}: ragged K chunks are zero-filled by TMA).  The image must fit one halo box, and a ring of
  // 2 B stages must fit next to the halo buffers and the largest buffer behind the ring, which is that of split-K over 2
  // CTAs in tangent mode (receive buffer + 64 staged primal zh rows; S = 1 stages 128 rows, larger S fewer)
  for (int l = 1; l < h->L && h->use_tc; ++l) {
    const int gw = h->geo[l].gw;
    if (tc_conv_rpad(gw) > 256 || tc_conv_ring(h->F, gw, tc_conv_extra_bytes(h->F, 2, true)) < 2) h->use_tc = false;
  }
  plan_chunks(h, h->n_s, &h->plan_sup);
  plan_chunks(h, h->n_t, &h->plan_tgt);
  Bump sz{nullptr, 0};
  carve(h, sz);
  h->ws_bytes = sz.off;
  cudaError_t e = cudaMalloc((void**)&h->ws, (size_t)h->ws_bytes);
  if (e != cudaSuccess) { std::string m = std::string("cudaMalloc workspace (") + std::to_string(h->ws_bytes) + " B): " + cudaGetErrorString(e); delete h; return fail(m); }
  e = cudaMemset(h->ws, 0, (size_t)h->ws_bytes);
  if (e != cudaSuccess) { cudaFree(h->ws); delete h; return fail(std::string("cudaMemset: ") + cudaGetErrorString(e)); }
  Bump as{h->ws, 0};
  carve(h, as);
  if (make_all_maps(h)) { cudaFree(h->ws); delete h; return 1; }
  e = cudaMallocHost((void**)&h->pinned, 16 * 32 * sizeof(float));
  if (e != cudaSuccess) { cudaFree(h->ws); delete h; return fail(std::string("cudaMallocHost: ") + cudaGetErrorString(e)); }
  h->use_graphs = !(cfg->reserved & 4) && !h->opt.no_graph;
  // Two regimes, told apart by whether one iteration's block-1 tiles (support + target, all tasks) fit one wave of SMs.
  //  * latency-bound (at most one tile per SM; on an H100's 132 SMs Omniglot 5-way up to 7 tasks -- at 8 tasks its 144 tiles
  //    are more than 132, and it runs throughput-bound): programmatic dependent launch on the MAIN chain only (the next
  //    kernel of the support / tangent chain is scheduled while the current one drains; on every stream, early-launched
  //    CTAs hold the SM slots the other streams want), deep shared-memory rings (all B stages of a short pipeline
  //    prefetched at once).
  //  * throughput-bound (on an H100 every benchmarked workload: Omniglot at 8 tasks, Mini-ImageNet, 20-way): no PDL, conv
  //    ring 4 (the shared memory it gives up lets the BatchNorm / first-block kernels of the other streams share the SM).
  {
    const int l1 = h->L > 1 ? 1 : 0;
    const long long tiles = (((long long)h->n_s * h->geo[l1].G + 127) / 128 + ((long long)h->n_t * h->geo[l1].G + 127) / 128) * h->maxT;
    const bool small = tiles <= num_sms();
    h->pdl = h->opt.pdl >= 0 ? h->opt.pdl != 0 : small;
    h->nb_main = h->opt.tc_nb > 0 ? h->opt.tc_nb : (small ? 8 : 4);
  }
  // Priorities: the support chain (capture stream) is the critical path; the weight-gradient and target streams only
  // have to finish by the end of a step.  Their many small CTAs would otherwise occupy every SM and keep the
  // whole-SM tensor-core conv CTAs of the critical path waiting.
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);      // lo = numerically largest = least urgent
  const int p_main = prio_hi, p_tgt = std::min(prio_lo, prio_hi + 1), p_wg = prio_lo;
  bool ok = cudaStreamCreateWithPriority(&h->s_cap, cudaStreamNonBlocking, p_main) == cudaSuccess &&
            cudaStreamCreateWithPriority(&h->s_tgt, cudaStreamNonBlocking, p_tgt) == cudaSuccess &&
            cudaStreamCreateWithPriority(&h->s_tgt2, cudaStreamNonBlocking, p_tgt) == cudaSuccess &&
            cudaStreamCreateWithPriority(&h->s_wg, cudaStreamNonBlocking, p_wg) == cudaSuccess &&
            cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming) == cudaSuccess &&
            cudaEventCreateWithFlags(&h->ev_wg, cudaEventDisableTiming) == cudaSuccess &&
            cudaEventCreateWithFlags(&h->ev_pack, cudaEventDisableTiming) == cudaSuccess;
  for (int s = 0; ok && s < MAML_MAX_STEPS; ++s) ok = cudaEventCreateWithFlags(&h->ev_tgt[s], cudaEventDisableTiming) == cudaSuccess;
  for (int s = 0; ok && s < 2 * MAML_MAX_LAYERS; ++s) ok = cudaEventCreateWithFlags(&h->ev_pre[s], cudaEventDisableTiming) == cudaSuccess;
  if (!ok) { maml_b200_destroy(h); return fail("stream / event creation failed"); }
  *out = h;
  return 0;
}

static void comm_release(maml_b200_handle* h) {
  for (int p = 0; p < MAML_MAX_RANKS; ++p) if (h->comm_opened[p]) { cudaIpcCloseMemHandle(h->comm_opened[p]); h->comm_opened[p] = nullptr; }
  if (h->comm_block) { cudaFree(h->comm_block); h->comm_block = nullptr; }
  h->comm = CommDev{}; h->comm_connected = false;
}

extern "C" void maml_b200_destroy(maml_b200_handle* h) {
  if (!h) return;
  comm_release(h);
  for (auto& g : h->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
  if (h->s_cap) cudaStreamDestroy(h->s_cap);
  if (h->s_tgt) cudaStreamDestroy(h->s_tgt);
  if (h->s_tgt2) cudaStreamDestroy(h->s_tgt2);
  if (h->s_wg) cudaStreamDestroy(h->s_wg);
  if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  if (h->ev_wg) cudaEventDestroy(h->ev_wg);
  if (h->ev_pack) cudaEventDestroy(h->ev_pack);
  for (int s = 0; s < MAML_MAX_STEPS; ++s) if (h->ev_tgt[s]) cudaEventDestroy(h->ev_tgt[s]);
  for (int s = 0; s < 2 * MAML_MAX_LAYERS; ++s) if (h->ev_pre[s]) cudaEventDestroy(h->ev_pre[s]);
  if (h->ws) cudaFree(h->ws);
  if (h->xdot_g) cudaFree(h->xdot_g - (long long)h->geo[0].guard * h->C);
  if (h->zero_dl) cudaFree(h->zero_dl);
  if (h->pinned) cudaFreeHost(h->pinned);
  delete h;
}

extern "C" int64_t maml_b200_workspace_bytes(const maml_b200_handle* h) { return h ? h->ws_bytes : -1; }
extern "C" int32_t maml_b200_num_segments(const maml_b200_handle* h) { return h ? (int32_t)h->seg_off.size() : -1; }
extern "C" int maml_b200_segment(const maml_b200_handle* h, int32_t idx, int64_t* offset, int64_t* size) {
  if (!h || idx < 0 || idx >= (int)h->seg_off.size()) return fail("bad segment index");
  *offset = h->seg_off[idx]; *size = h->seg_size[idx];
  return 0;
}
extern "C" int64_t maml_b200_meta_size(const maml_b200_handle* h) { return h ? h->pl.meta_size : -1; }
extern "C" int64_t maml_b200_result_size(const maml_b200_handle* h) {
  if (!h) return -1;
  return h->pl.meta_size + 2 + (h->pl.per_step_bn ? 2LL * h->L * h->S * h->F : 0);
}
extern "C" int64_t maml_b200_last_launch_count(const maml_b200_handle* h) { return h ? h->last_launches : -1; }

// ---------------------------------------------------------------------------------------------
// pass helpers
// ---------------------------------------------------------------------------------------------
static BnGeom bn_geom(const maml_b200_handle* h, int l, int n) {
  const LayerGeom& g = h->geo[l];
  BnGeom b; b.n = n; b.h = g.h; b.w = g.w; b.gw = g.gw; b.G = g.G; b.ph = g.ph; b.pw = g.pw; b.pgw = g.pgw; b.pG = g.pG; b.pb = g.pb; b.F = h->F;
  return b;
}
static double conv_flops(const maml_b200_handle* h, int l, int n, int T, int nsrc) {
  // algorithmic FLOPs (SURVEY.md section 8d): 2 * valid pixels * C_in * 9 * F per operand pair, per task
  const LayerGeom& g = h->geo[l];
  return 2.0 * (double)n * g.h * g.w * (double)g.cin * 9.0 * (double)h->F * (double)nsrc * (double)T;
}
static double* stat_at(const maml_b200_handle* h, int kind, int step, int layer) {
  return h->stats + ((long long)kind * MAML_MAX_STEPS + step) * h->st_pass_stride + (long long)layer * h->st_layer_stride;
}
// layer norm: the per-image sums of (pass kind, step, block), task 0; and the arguments every LN launch of block l over n
// images per task shares
static double* ln_stat_at(const maml_b200_handle* h, int kind, int step, int layer) {
  return h->ln_stats + (long long)kind * h->ln_pass_stride + ((long long)step * h->L + layer) * std::max(h->n_s, h->n_t) * 2;
}
static LnArgs ln_args(const maml_b200_handle* h, int l, int n, const float* meta, int T) {
  LnArgs a{};
  a.st_stride = h->ln_task_stride;
  a.bias = meta + h->pl.m_lnb[l];
  a.g = bn_geom(h, l, n); a.tasks = T;
  return a;
}
// bias-gradient row of (task 0, kind 0: target pass / 1: tangent pass, step)
static float* lnb_at(const maml_b200_handle* h, int kind, int step) {
  return h->lnb + ((long long)kind * h->S + step) * h->pl.lnb_off[h->L];
}

static const float* gamma_at(const maml_b200_handle* h, const float* meta, int l, int step) {
  return meta + h->pl.m_gamma[l] + (h->pl.per_step_gb ? (long long)step * h->F : 0);
}
static const float* beta_at(const maml_b200_handle* h, const float* meta, int l, int step) {
  return meta + h->pl.m_beta[l] + (h->pl.per_step_gb ? (long long)step * h->F : 0);
}
// BatchNorm gamma / beta of block l for a pass at inner step `step`: the meta vector's row, shared by the tasks (stride 0),
// or with inner_bn the fast weights `theta` (per task, stride Ppad)
struct NormParams { const float* gamma; const float* beta; long long stride; };
static NormParams norm_params(const maml_b200_handle* h, const float* meta, const float* theta, int l, int step) {
  if (h->pl.inner_bn) return NormParams{theta + h->pl.gamma_off[l], theta + h->pl.beta_off[l], h->Ppad};
  return NormParams{gamma_at(h, meta, l, step), beta_at(h, meta, l, step), 0};
}

struct Slot { const PassSet* ps; int slot; };
static float* slot_ptr(float* base, long long sz, int slots, int slot) { return base + (long long)slot * sz; }
#define AIN(ps, l, slot) slot_ptr((ps).ain[l], (ps).ain_sz[l], (ps).slots, slot)
#define ZH(ps, l, slot) slot_ptr((ps).zh[l], (ps).zh_sz[l], (ps).slots, slot)
#define DZ(ps, l, slot) slot_ptr((ps).dz[l], (ps).dz_sz[l], (ps).slots, slot)
#define DP(ps, l, slot) slot_ptr((ps).dp[l], (ps).dp_sz[l], (ps).slots, slot)
#define STRIDE(ps, what, l) ((ps).what##_sz[l] * (ps).slots)

#define AIN_HI(ps, l, slot) (AIN(ps, l, slot) + (ps).ain_plane[l])
#define AIN_LO(ps, l, slot) (AIN(ps, l, slot) + 2 * (ps).ain_plane[l])
#define DZ_HI(ps, l, slot) (DZ(ps, l, slot) + (ps).dz_plane[l])
#define DZ_LO(ps, l, slot) (DZ(ps, l, slot) + 2 * (ps).dz_plane[l])

// one operand pair of a tensor-core conv launch
struct TcOp {
  const CUtensorMap* a_maps;   // [hi, lo]
  int a_row_base, a_task_rows, sign;
  const CUtensorMap* b_maps;   // 4 planes: W hi, W lo, WT hi, WT lo
  int b_pair;                  // 0: W planes (dgrad), 2: WT planes (conv)
  int b_row_base, b_task_rows;
};

static int a_row_base_of(const maml_b200_handle* h, long long sz, int l, int slot) {
  return (int)(slot * (sz / h->F) + h->geo[l].guard);
}
static TcOp tc_op_ain(const maml_b200_handle* h, const PassSet& ps, int l, int slot, const CUtensorMap* bmaps, int b_step, int sign, int b_pair) {
  TcOp o;
  o.a_maps = ps.ain_map[l]; o.a_row_base = a_row_base_of(h, ps.ain_sz[l], l, slot);
  o.a_task_rows = (int)(ps.ain_sz[l] * ps.slots / h->F); o.sign = sign;
  o.b_maps = bmaps; o.b_pair = b_pair;
  o.b_row_base = (int)(((long long)b_step * h->maxT * (h->L - 1) + (l - 1)) * 9 * h->F);
  o.b_task_rows = (h->L - 1) * 9 * h->F;
  return o;
}
static TcOp tc_op_dz(const maml_b200_handle* h, const PassSet& ps, int l, int slot, const CUtensorMap* bmaps, int b_step, int sign, int b_pair) {
  TcOp o = tc_op_ain(h, ps, l, slot, bmaps, b_step, sign, b_pair);
  o.a_maps = ps.dz_map[l]; o.a_row_base = a_row_base_of(h, ps.dz_sz[l], l, slot);
  o.a_task_rows = (int)(ps.dz_sz[l] * ps.slots / h->F);
  return o;
}

// what a backward pass does with its gradient chunks once they are complete
struct ReduceSpec {
  int mode;                       // PR_UPDATE / PR_SUB
  const float* theta_in; float* theta_out; float* g_out; float* tbar;
  int step;
  int pack_step;                  // >= 0: re-pack theta[pack_step] for the tensor-core convs afterwards
  const double* bn_sums = nullptr;  // inner_bn: the pass's backward sums (kind, step, block 0, task 0), the beta / gamma gradient
};

static void pack_theta_step(maml_b200_handle* h, int step, int T, cudaStream_t st);

// The first block's weight gradient is the LAST product of a backward pass, every other tensor's chunks are complete
// much earlier.  So the reduction (+ LSLR update + tensor-core weight packing) of blocks >= 1 and the linear layer runs
// on the wgrad side stream while the main chain finishes block 0; only the 9*C*F + F first-block values are reduced on
// the critical path.  The main chain joins the side stream lazily (join_pending) before block 1 needs those weights.
// The partial-buffer description of a reduction: inner-loop beta / gamma read the pass's backward sums.
static PartialDesc with_bn_sums(const maml_b200_handle* h, const PartialDesc& pd, const double* bn_sums) {
  PartialDesc d = pd;
  d.bn_sums = bn_sums; d.bn_task_stride = h->stats_task_stride; d.bn_layer_stride = h->st_layer_stride;
  return d;
}

static void reduce_upper_on_side(maml_b200_handle* h, const ReduceSpec& rs, const PartialDesc& pd, const float* partial,
                                 const float* meta, int T) {
  // the first block's tensors (seg_per_block segments: with inner_bn its beta / gamma too, whose sums the main chain
  // finishes last) are reduced on the main chain by reduce_lower
  launch_param_reduce(h->pl, with_bn_sums(h, pd, rs.bn_sums), partial, rs.mode, rs.theta_in, rs.theta_out, rs.g_out, rs.tbar,
                      meta, rs.step, h->Ppad, T, h->s_wg, seg_per_block(h->pl), -1);
  if (rs.pack_step >= 0) pack_theta_step(h, rs.pack_step, T, h->s_wg);
  cudaEventRecord(h->ev_wg, h->s_wg);
  h->wg_pending = true;
}

static void reduce_lower(maml_b200_handle* h, const ReduceSpec& rs, const PartialDesc& pd, const float* partial,
                         const float* meta, int T, cudaStream_t st) {
  launch_param_reduce(h->pl, with_bn_sums(h, pd, rs.bn_sums), partial, rs.mode, rs.theta_in, rs.theta_out, rs.g_out, rs.tbar,
                      meta, rs.step, h->Ppad, T, st, 0, seg_per_block(h->pl));
}
static void join_pending(maml_b200_handle* h, cudaStream_t st) {
  if (!h->wg_pending) return;
  cudaStreamWaitEvent(st, h->ev_wg, 0);
  h->wg_pending = false;
}

static void tc_conv(maml_b200_handle* h, int l, int n, const TcOp& op, const float* bias, long long bias_stride,
                    float* out, long long out_stride, int mode, const float* zh, long long zh_stride, double* stats, int T,
                    cudaStream_t st) {
  const LayerGeom& g = h->geo[l];
  TcMaps maps;
  TcConvArgs a{};
  a.kc = h->F; a.rows = n * g.G; a.gw = g.gw; a.G = g.G; a.h = g.h; a.w = g.w; a.ncols = h->F; a.mode = mode; a.tasks = T; a.plan_tasks = h->maxT;
  a.halo = g.gw + 1; a.rpad = tc_conv_rpad(g.gw); a.nb = std::min(tc_conv_ring(h->F, g.gw), h->nb_main);
  a.timeline = (h->opt.tc_timeline == 0 || h->opt.tc_timeline == l) ? 1 : 0;
  maps.m[0] = op.a_maps[0]; maps.m[1] = op.a_maps[1];
  maps.m[2] = op.b_maps[op.b_pair]; maps.m[3] = op.b_maps[op.b_pair + 1];
  a.a_row_base = op.a_row_base; a.a_task_rows = op.a_task_rows; a.sign = op.sign;
  a.b_row_base = op.b_row_base; a.b_task_rows = op.b_task_rows;
  a.bias = bias; a.bias_stride = bias_stride; a.out = out; a.out_stride = out_stride;
  a.zh = zh; a.zh_stride = zh_stride; a.stats = stats; a.stats_stride = h->stats_task_stride;
  a.alg_flops = conv_flops(h, l, n, T, 1);
  launch_conv_tc(maps, a, st);
}

// one operand pair of an FFMA conv of block l: A (row 0 of a guarded pass buffer) times the block-l weights of the
// fast-weight vector `wv`, as stored (wt 0, conv: sign +1) or transposed (wt 1, dgrad: sign -1)
struct FfmaOp { const float* A; long long a_stride; const float* wv; int wt, sign; };

// FFMA conv of block l over n images per task: the sum of the operand pairs plus the block-l bias of `bias_vec`
// (nullable).  The caller sets the output and, in the statistics modes, the sums' address (and zh).
static ConvArgs ffma_conv(const maml_b200_handle* h, int l, int n, int mode, std::initializer_list<FfmaOp> ops,
                          const float* bias_vec, int T) {
  const LayerGeom& g = h->geo[l];
  ConvArgs a{};
  for (const FfmaOp& o : ops) a.src[a.nsrc++] = ConvSrc{o.A, o.a_stride, o.wv + h->pl.w_off[l], h->Ppad, h->F, o.wt, o.sign};
  if (bias_vec) { a.bias = bias_vec + h->pl.b_off[l]; a.bias_stride = h->Ppad; }
  a.rows = n * g.G; a.gw = g.gw; a.G = g.G; a.h = g.h; a.w = g.w; a.ncols = h->F; a.mode = mode;
  if (mode != CONV_PLAIN) a.stats_stride = h->stats_task_stride;
  a.tasks = T;
  a.alg_flops = conv_flops(h, l, n, T, a.nsrc);
  return a;
}

// First-block conv of pass `ps`'s images with the block-0 weights and bias of the fast-weight vector `wv` (nsrc = 2: the
// caller's second operand pair, see launch_conv0).  The caller sets the output and the statistics' address (and zh).
static Conv0Args conv0_args(const maml_b200_handle* h, const PassSet& ps, const float* wv, int mode, int nsrc, int T) {
  const LayerGeom& g = h->geo[0];
  Conv0Args a{};
  a.X = ps.xg; a.x_stride = ps.xg_stride;
  a.W = wv + h->pl.w_off[0]; a.w_stride = h->Ppad;
  a.bias = wv + h->pl.b_off[0]; a.bias_stride = h->Ppad;
  a.rows = ps.n * g.G; a.gw = g.gw; a.G = g.G; a.h = g.h; a.w = g.w; a.c0 = h->C; a.ncols = h->F; a.mode = mode;
  a.stats_stride = h->stats_task_stride; a.tasks = T;
  a.alg_flops = conv_flops(h, 0, ps.n, T, nsrc);
  return a;
}

// Weight gradient of block l over n images per task into that block's chunks of the partial buffer `partial` (laid out by
// `cp`).  The caller sets the operand pairs and alg_flops (launch_wgrad_upper does for blocks l >= 1).
static WgradArgs wgrad_args(const maml_b200_handle* h, int l, int n, const ChunkPlan& cp, float* partial, int T) {
  const LayerGeom& g = h->geo[l];
  WgradArgs w{};
  w.kc = l == 0 ? h->C : h->F; w.ncols = h->F; w.rows = n * g.G; w.gw = g.gw;
  w.rows_per_chunk = cp.rows_per_chunk[l]; w.nchunks = cp.nchunks[l];
  const int k = seg_per_block(h->pl) * l;
  w.partial = partial + cp.pd.off[k]; w.partial_task_stride = cp.pd.task_stride; w.chunk_stride = cp.pd.cstride[k];
  w.tasks = T;
  return w;
}

// one operand pair of the weight gradient of a block l >= 1: the conv input of `a` times the output gradient of `d`
struct WgPair { Slot a, d; };

// Weight gradient of block l >= 1, summed over the operand pairs: the tensor-core kernel (reading both operands' TF32
// planes) when the handle runs the tensor-core path and the option allows it, else the FFMA kernel.
static void launch_wgrad_upper(const maml_b200_handle* h, int l, int n, const ChunkPlan& cp, float* partial, int T,
                               std::initializer_list<WgPair> pairs, cudaStream_t st) {
  const bool tc = h->use_tc && h->opt.wgrad_tc;
  WgradArgs w = wgrad_args(h, l, n, cp, partial, T);
  for (const WgPair& p : pairs) {
    const PassSet& pa = *p.a.ps; const PassSet& pd = *p.d.ps;
    const int k = w.nsrc++;
    w.A[k] = AIN(pa, l, p.a.slot); w.a_stride[k] = STRIDE(pa, ain, l);
    w.D[k] = DZ(pd, l, p.d.slot); w.d_stride[k] = STRIDE(pd, dz, l);
    if (tc) { w.a_plane[k] = pa.ain_plane[l]; w.d_plane[k] = pd.dz_plane[l]; }
  }
  w.alg_flops = conv_flops(h, l, n, T, w.nsrc);
  if (tc) launch_wgrad_tc(w, st);
  else launch_wgrad(w, st);
}

// Head launch on the features of pass `ps` at `slot` (linear layer of the fast weights `theta`, zero labels); every mode
// but the target forward writes d(features) into the pass's DP(L-1).  The caller sets labels, outputs and (head_grad)
// where the linear layer's gradient goes.
static HeadArgs head_args(const maml_b200_handle* h, int mode, const PassSet& ps, int slot, const float* theta, int T) {
  HeadArgs a{};
  a.mode = mode; a.n = ps.n; a.N = h->N; a.D = h->D; a.scale = 1.f;
  a.f = AIN(ps, h->L, slot); a.f_stride = STRIDE(ps, ain, h->L);
  a.Wfc = theta + h->pl.fcw_off; a.bfc = theta + h->pl.fcb_off; a.theta_stride = h->Ppad;
  a.y = h->zero_labels; a.y_stride = 0;
  a.rows_per_cta = head_rows(ps.n);
  if (mode != HEAD_TARGET_FWD) { a.df = DP(ps, h->L - 1, slot); a.df_stride = STRIDE(ps, dp, h->L - 1); }
  a.tasks = T;
  return a;
}

// the head's gradient goes to the linear layer's chunks (one per row group) of the partial buffer `partial`
static void head_grad(const maml_b200_handle* h, HeadArgs& a, float* partial, const ChunkPlan& cp) {
  const int k = seg_per_block(h->pl) * h->L;
  a.gW = partial + cp.pd.off[k]; a.gb = partial + cp.pd.off[k + 1];
  a.g_stride = cp.pd.task_stride; a.g_chunk_stride = cp.pd.cstride[k];
}

// the last block of the support batch, the head and that block's BatchNorm backward run as one kernel
static bool support_tail_fused(const maml_b200_handle* h) {
  return h->opt.tail_fuse && !h->ln && !h->pl.inner_bn && tail_fusable(bn_geom(h, h->L - 1, h->n_s), h->n_s, head_rows(h->n_s));
}

enum { CLR_STATS = 1, CLR_ABAR = 2, CLR_LOSSES = 4, CLR_CORRECT = 8, CLR_BWD_STATS = 16 };
// zeroes the accumulators in `what` (CLR_* bits) for all maxT tasks on `st`; CLR_BWD_STATS: only the backward sums (kinds
// PASS_TGT_BWD / PASS_TAN_BWD) of the first bwd_tasks tasks.  Layer norm: both sums clear the bias-gradient rows too.
static int clear_accumulators(maml_b200_handle* h, unsigned what, cudaStream_t st, int bwd_tasks = 0) {
  if (what & CLR_STATS) CK(cudaMemsetAsync(h->stats, 0, (size_t)h->stats_count * sizeof(double), st));
  if ((what & CLR_STATS) && h->ln) CK(cudaMemsetAsync(h->ln_stats, 0, (size_t)h->ln_task_stride * h->maxT * sizeof(double), st));
  if (what & CLR_BWD_STATS)
    for (int kind : {PASS_TGT_BWD, PASS_TAN_BWD}) {
      CK(cudaMemset2DAsync(h->stats + (long long)kind * MAML_MAX_STEPS * h->st_pass_stride, (size_t)h->stats_task_stride * sizeof(double),
                           0, (size_t)MAML_MAX_STEPS * h->st_pass_stride * sizeof(double), (size_t)bwd_tasks, st));
      if (h->ln)
        CK(cudaMemset2DAsync(h->ln_stats + (long long)kind * h->ln_pass_stride, (size_t)h->ln_task_stride * sizeof(double), 0,
                             (size_t)h->ln_pass_stride * sizeof(double), (size_t)bwd_tasks, st));
    }
  if ((what & (CLR_STATS | CLR_BWD_STATS)) && h->ln) {
    const int tasks = (what & CLR_STATS) ? h->maxT : bwd_tasks;
    CK(cudaMemsetAsync(h->lnb, 0, (size_t)tasks * 2 * h->S * h->pl.lnb_off[h->L] * sizeof(float), st));
  }
  if (what & CLR_ABAR) CK(cudaMemsetAsync(h->abar, 0, (size_t)h->maxT * h->pl.nseg_inner * MAML_MAX_STEPS * sizeof(double), st));
  if (what & CLR_LOSSES) CK(cudaMemsetAsync(h->losses, 0, (size_t)h->maxT * MAML_MAX_STEPS * sizeof(float), st));
  if (what & CLR_CORRECT) CK(cudaMemsetAsync(h->correct, 0, (size_t)h->maxT * sizeof(float), st));
  return 0;
}

// The normalisation (+ leaky-ReLU + max-pool) of block l in each kind of pass, BatchNorm or layer norm.  defer_last: the
// last block's BatchNorm is not launched but returned; fused_head: it runs in the fused last-block kernel.
static void norm_forward(maml_b200_handle* h, const PassSet& ps, int slot, const float* theta, const float* meta, int l, int step,
                         int stat_kind, int T, cudaStream_t st, BnActArgs* defer_last) {
  if (h->ln) {                   // per-image sums of z, then normalise / bias / leaky-ReLU / pool
    LnArgs a = ln_args(h, l, ps.n, meta, T);
    a.z = ZH(ps, l, slot); a.z_stride = STRIDE(ps, zh, l);
    a.st_fwd = a.st_out = ln_stat_at(h, stat_kind, step, l);
    launch_ln_stats(a, false, st);
    a.out = AIN(ps, l + 1, slot); a.out_stride = STRIDE(ps, ain, l + 1);
    if (h->use_tc && l + 1 < h->L) { a.out_hi = AIN_HI(ps, l + 1, slot); a.out_lo = AIN_LO(ps, l + 1, slot); }
    launch_ln_act(a, false, st);
    return;
  }
  BnActArgs b{};
  b.z = ZH(ps, l, slot); b.z_stride = STRIDE(ps, zh, l);
  b.stats = stat_at(h, stat_kind, step, l); b.stats_stride = h->stats_task_stride;
  const NormParams np = norm_params(h, meta, theta, l, step);
  b.gamma = np.gamma; b.beta = np.beta;
  b.p = AIN(ps, l + 1, slot); b.p_stride = STRIDE(ps, ain, l + 1);
  if (h->use_tc && l + 1 < h->L) { b.p_hi = AIN_HI(ps, l + 1, slot); b.p_lo = AIN_LO(ps, l + 1, slot); }
  b.g = bn_geom(h, l, ps.n); b.tasks = T;
  if (defer_last && l == h->L - 1) *defer_last = b;
  else launch_bnact(b, np.stride, st);
}

static void norm_backward(maml_b200_handle* h, const PassSet& ps, int slot, const float* theta, const float* meta, int l, int step,
                          int kind_fwd, int kind_bwd, int T, cudaStream_t st, const BnActArgs* fused_act, const HeadArgs* fused_head) {
  if (h->ln) {
    LnArgs a = ln_args(h, l, ps.n, meta, T);
    a.dp = DP(ps, l, slot); a.dp_stride = STRIDE(ps, dp, l);
    a.zh = ZH(ps, l, slot); a.zh_stride = STRIDE(ps, zh, l);
    a.st_fwd = ln_stat_at(h, kind_fwd, step, l); a.st_out = ln_stat_at(h, kind_bwd, step, l);
    a.out = DZ(ps, l, slot); a.out_stride = STRIDE(ps, dz, l);
    if (h->use_tc && l >= 1) { a.out_hi = DZ_HI(ps, l, slot); a.out_lo = DZ_LO(ps, l, slot); }
    launch_ln_bwd(a, false, st);
    if (kind_bwd == PASS_TGT_BWD) {    // the bias is an outer parameter only: its gradient comes from the target loss
      a.db = lnb_at(h, 0, step) + h->pl.lnb_off[l]; a.db_stride = 2LL * h->S * h->pl.lnb_off[h->L];
      launch_ln_bias_grad(a, false, st);
    }
    return;
  }
  BnBwdArgs b{};
  b.dp = DP(ps, l, slot); b.dp_stride = STRIDE(ps, dp, l);
  b.zh = ZH(ps, l, slot); b.zh_stride = STRIDE(ps, zh, l);
  b.stats_fwd = stat_at(h, kind_fwd, step, l); b.stats_fwd_stride = h->stats_task_stride;
  b.stats_bwd = stat_at(h, kind_bwd, step, l); b.stats_bwd_stride = h->stats_task_stride;
  const NormParams np = norm_params(h, meta, theta, l, step);
  b.gamma = np.gamma; b.beta = np.beta;
  b.dz = DZ(ps, l, slot); b.dz_stride = STRIDE(ps, dz, l);
  if (h->use_tc && l >= 1) { b.dz_hi = DZ_HI(ps, l, slot); b.dz_lo = DZ_LO(ps, l, slot); }
  b.g = bn_geom(h, l, ps.n); b.tasks = T;
  if (fused_head && l == h->L - 1) launch_tail_fused(*fused_act, *fused_head, b, st);
  else launch_bnbwd(b, np.stride, st);
}

// inner_bn: gamma / beta are theta's and their tangents u's (per task); t_norm is then not read
static void norm_tangent_forward(maml_b200_handle* h, int s, const float* theta, const float* u, const float* meta, int l,
                                 const float* t_norm, long long t_stride, int T, cudaStream_t st, BnActTanArgs* defer_last) {
  const PassSet& sp = h->sup; const PassSet& tn = h->tan; const PassSet& t2 = h->tan2;
  if (h->ln) {                   // zdot (+ the side stream's addend) -> per-image sums -> zhdot, pdot
    LnArgs a = ln_args(h, l, sp.n, meta, T);
    a.z = ZH(tn, l, 0); a.z_stride = STRIDE(tn, zh, l);
    if (h->use_tc && l >= 1) a.z2 = ZH(t2, l, 0);
    a.zh = ZH(sp, l, s); a.zh_stride = STRIDE(sp, zh, l);
    a.st_fwd = ln_stat_at(h, PASS_SUP_FWD, s, l); a.st_tan = a.st_out = ln_stat_at(h, PASS_TAN_FWD, s, l);
    launch_ln_stats(a, true, st);
    a.out = AIN(tn, l + 1, 0); a.out_stride = STRIDE(tn, ain, l + 1);
    if (h->use_tc && l + 1 < h->L) { a.out_hi = AIN_HI(tn, l + 1, 0); a.out_lo = AIN_LO(tn, l + 1, 0); }
    if (t_norm) { a.bdot = t_norm + h->pl.m_lnb[l]; a.bdot_stride = t_stride; }
    launch_ln_act(a, true, st);
    return;
  }
  BnActTanArgs b{};
  b.zdot = ZH(tn, l, 0); b.zdot_stride = STRIDE(tn, zh, l);
  if (h->use_tc && l >= 1) b.zdot2 = ZH(t2, l, 0);
  b.zh = ZH(sp, l, s); b.zh_stride = STRIDE(sp, zh, l);
  b.stats_fwd = stat_at(h, PASS_SUP_FWD, s, l); b.stats_fwd_stride = h->stats_task_stride;
  b.stats_tan = stat_at(h, PASS_TAN_FWD, s, l); b.stats_tan_stride = h->stats_task_stride;
  const NormParams np = norm_params(h, meta, theta, l, s);
  b.gamma = np.gamma; b.beta = np.beta;
  b.pdot = AIN(tn, l + 1, 0); b.pdot_stride = STRIDE(tn, ain, l + 1);
  if (h->use_tc && l + 1 < h->L) { b.pdot_hi = AIN_HI(tn, l + 1, 0); b.pdot_lo = AIN_LO(tn, l + 1, 0); }
  b.g = bn_geom(h, l, sp.n); b.tasks = T;
  const float* gdot = np.stride ? u + h->pl.gamma_off[l] : t_norm ? gamma_at(h, t_norm, l, s) : nullptr;
  const float* bdot = np.stride ? u + h->pl.beta_off[l] : t_norm ? beta_at(h, t_norm, l, s) : nullptr;
  if (defer_last && l == h->L - 1) *defer_last = b;
  else launch_bnact_tan(b, gdot, bdot, np.stride, st);
}

static void norm_tangent_backward(maml_b200_handle* h, int s, const float* theta, const float* u, const float* meta, int l,
                                  int kind_tbwd, int T, cudaStream_t st, const BnActTanArgs* fused_act, const HeadArgs* fused_head) {
  const PassSet& sp = h->sup; const PassSet& tn = h->tan; const PassSet& t2 = h->tan2;
  if (h->ln) {
    LnArgs a = ln_args(h, l, sp.n, meta, T);
    a.dp = DP(sp, l, s); a.dp_stride = STRIDE(sp, dp, l);
    a.dpd = DP(tn, l, 0); a.dpd_stride = STRIDE(tn, dp, l);
    if (h->use_tc && l + 1 < h->L) a.dpd2 = DP(t2, l, 0);
    a.zh = ZH(sp, l, s); a.zh_stride = STRIDE(sp, zh, l);
    a.zhd = ZH(tn, l, 0); a.zhd_stride = STRIDE(tn, zh, l);
    a.dz = DZ(sp, l, s); a.dz_stride = STRIDE(sp, dz, l);
    a.st_fwd = ln_stat_at(h, PASS_SUP_FWD, s, l); a.st_bwd = ln_stat_at(h, PASS_SUP_BWD, s, l);
    a.st_tan = ln_stat_at(h, PASS_TAN_FWD, s, l); a.st_out = ln_stat_at(h, kind_tbwd, s, l);
    a.out = DZ(tn, l, 0); a.out_stride = STRIDE(tn, dz, l);
    if (h->use_tc && l >= 1) { a.out_hi = DZ_HI(tn, l, 0); a.out_lo = DZ_LO(tn, l, 0); }
    launch_ln_bwd(a, true, st);
    // H_b u, the tangent of the support loss's bias gradient: export subtracts kind 1 (fused iteration, b-bar -= H_b u)
    // and adds kind 0 (functional operator, +H_b v), as it does with the BatchNorm gamma / beta sums of kind_tbwd
    a.db = lnb_at(h, kind_tbwd == PASS_TGT_BWD ? 0 : 1, s) + h->pl.lnb_off[l];
    a.db_stride = 2LL * h->S * h->pl.lnb_off[h->L];
    launch_ln_bias_grad(a, true, st);
    return;
  }
  BnBwdTanArgs b{};
  b.dp = DP(sp, l, s); b.dp_stride = STRIDE(sp, dp, l);
  b.dpdot = DP(tn, l, 0); b.dpdot_stride = STRIDE(tn, dp, l);
  if (h->use_tc && l + 1 < h->L) b.dpdot2 = DP(t2, l, 0);
  b.zh = ZH(sp, l, s); b.zh_stride = STRIDE(sp, zh, l);
  b.zhdot = ZH(tn, l, 0); b.zhdot_stride = STRIDE(tn, zh, l);
  b.dz = DZ(sp, l, s); b.dz_stride = STRIDE(sp, dz, l);
  b.stats_fwd = stat_at(h, PASS_SUP_FWD, s, l); b.stats_fwd_stride = h->stats_task_stride;
  b.stats_bwd = stat_at(h, PASS_SUP_BWD, s, l); b.stats_bwd_stride = h->stats_task_stride;
  b.stats_tan = stat_at(h, PASS_TAN_FWD, s, l); b.stats_tan_stride = h->stats_task_stride;
  b.stats_tbwd = stat_at(h, kind_tbwd, s, l); b.stats_tbwd_stride = h->stats_task_stride;
  const NormParams np = norm_params(h, meta, theta, l, s);
  b.gamma = np.gamma; b.beta = np.beta;
  b.dzdot = DZ(tn, l, 0); b.dzdot_stride = STRIDE(tn, dz, l);
  if (h->use_tc && l >= 1) { b.dzdot_hi = DZ_HI(tn, l, 0); b.dzdot_lo = DZ_LO(tn, l, 0); }
  b.g = bn_geom(h, l, sp.n); b.tasks = T;
  if (fused_head && l == h->L - 1) launch_tail_tan_fused(*fused_act, *fused_head, b, st);
  else launch_bnbwd_tan(b, np.stride ? u + h->pl.gamma_off[l] : nullptr, np.stride, st);
}

// primal forward of one pass: conv -> stats -> BN/leaky/pool for every block
static void forward_pass(maml_b200_handle* h, const PassSet& ps, int slot, const float* theta, int th_step, const float* meta,
                         int bn_step, int stat_kind, int T, cudaStream_t st, BnActArgs* defer_last = nullptr) {
  for (int l = 0; l < h->L; ++l) {
    if (l == 1 && st != h->s_tgt && st != h->s_tgt2) join_pending(h, st);
    if (l == 0) {
      Conv0Args a = conv0_args(h, ps, theta, CONV_FWD_STATS, 1, T);
      a.out = ZH(ps, 0, slot); a.out_stride = STRIDE(ps, zh, 0);
      a.stats = stat_at(h, stat_kind, bn_step, 0);
      launch_conv0(a, st);
    } else if (h->use_tc) {
      tc_conv(h, l, ps.n, tc_op_ain(h, ps, l, slot, h->theta_map, th_step, +1, 2), theta + h->pl.b_off[l], h->Ppad,
              ZH(ps, l, slot), STRIDE(ps, zh, l), CONV_FWD_STATS, nullptr, 0,
              stat_at(h, stat_kind, bn_step, l), T, st);
    } else {
      ConvArgs a = ffma_conv(h, l, ps.n, CONV_FWD_STATS, {{AIN(ps, l, slot), STRIDE(ps, ain, l), theta, 0, +1}}, theta, T);
      a.out = ZH(ps, l, slot); a.out_stride = STRIDE(ps, zh, l);
      a.stats = stat_at(h, stat_kind, bn_step, l);
      launch_conv_rows(a, st);
    }
    norm_forward(h, ps, slot, theta, meta, l, bn_step, stat_kind, T, st, defer_last);
  }
}

// primal backward of one pass (dp[L-1] already written by the head): BN backward, wgrad, dgrad
static void backward_pass(maml_b200_handle* h, const PassSet& ps, int slot, const float* theta, int th_step, const float* meta,
                          int bn_step, int kind_fwd, int kind_bwd, float* partial, const ChunkPlan& cp, int T, cudaStream_t st,
                          bool fork_wgrad, const ReduceSpec* rs = nullptr, const BnActArgs* fused_act = nullptr,
                          const HeadArgs* fused_head = nullptr) {
  // wgrad of block l >= 1 only feeds the parameter-space reduction: it runs on a side stream, concurrently with
  // dgrad(l) and the BatchNorm backward of block l-1.  With a ReduceSpec the reduction itself is split (see
  // reduce_upper_on_side); without one the caller reduces after this function returns.
  cudaStream_t wst = fork_wgrad ? h->s_wg : st;
  const bool split = fork_wgrad && rs != nullptr;
  for (int l = h->L - 1; l >= 0; --l) {
    norm_backward(h, ps, slot, theta, meta, l, bn_step, kind_fwd, kind_bwd, T, st, fused_act, fused_head);
    if (fork_wgrad) { cudaEventRecord(h->ev_fork, st); cudaStreamWaitEvent(h->s_wg, h->ev_fork, 0); }

    if (l == 0) {
      WgradArgs w = wgrad_args(h, 0, ps.n, cp, partial, T);
      w.nsrc = 1;
      w.A[0] = ps.xg; w.a_stride[0] = ps.xg_stride;
      w.D[0] = DZ(ps, 0, slot); w.d_stride[0] = STRIDE(ps, dz, 0);
      w.alg_flops = conv_flops(h, 0, ps.n, T, 1);
      if (split && h->L == 1) reduce_upper_on_side(h, *rs, cp.pd, partial, meta, T);
      launch_wgrad0(w, split ? st : wst);
    } else {
      // dgrad (critical path) is enqueued before the side-stream wgrad so that its CTAs get SMs first
      if (h->use_tc) {
        tc_conv(h, l, ps.n, tc_op_dz(h, ps, l, slot, h->theta_map, th_step, -1, 0), nullptr, 0, DP(ps, l - 1, slot),
                STRIDE(ps, dp, l - 1), CONV_PLAIN, nullptr, 0, nullptr, T, st);
      } else {
        ConvArgs a = ffma_conv(h, l, ps.n, CONV_PLAIN, {{DZ(ps, l, slot), STRIDE(ps, dz, l), theta, 1, -1}}, nullptr, T);
        a.out = DP(ps, l - 1, slot); a.out_stride = STRIDE(ps, dp, l - 1);
        launch_conv_rows(a, st);
      }
      launch_wgrad_upper(h, l, ps.n, cp, partial, T, {{{&ps, slot}, {&ps, slot}}}, wst);
      if (split && l == 1) reduce_upper_on_side(h, *rs, cp.pd, partial, meta, T);
    }
  }
  if (split) reduce_lower(h, *rs, cp.pd, partial, meta, T, st);
  else if (fork_wgrad) { cudaEventRecord(h->ev_wg, h->s_wg); cudaStreamWaitEvent(st, h->ev_wg, 0); }
}

// What a tangent pass differentiates at its head, and where its BatchNorm gamma / beta sums go (export adds the
// PASS_TGT_BWD sums and subtracts the PASS_TAN_BWD ones).
//   fused iteration:       HEAD_TANGENT, support labels y, PASS_TAN_BWD   (gamma-bar -= H_gamma u)
//   functional operator:   HEAD_EXTERNAL_TAN, dl_ext (floats between tasks: dl_ext_stride) held constant, the logits
//                          tangent into jv_out, PASS_TGT_BWD (+H_gamma v)
struct TangentHead {
  int mode;
  const long long* y;
  const float* dl_ext; long long dl_ext_stride; float* jv_out;
  int kind_tbwd;
};

// Head of the tangent pass at support slot s in direction u: the support features and their tangent in tan, d(features)-dot
// into tan's DP(L-1), the tangent of the linear layer's gradient into the support chunks.
static HeadArgs tangent_head_args(const maml_b200_handle* h, int s, const float* theta, const float* u, const TangentHead& th,
                                  int T) {
  const PassSet& tn = h->tan;
  HeadArgs a = head_args(h, th.mode, h->sup, s, theta, T);
  a.fdot = AIN(tn, h->L, 0); a.fdot_stride = STRIDE(tn, ain, h->L);
  a.uW = u + h->pl.fcw_off; a.ub = u + h->pl.fcb_off; a.u_stride = h->Ppad;
  if (th.mode == HEAD_TANGENT) {
    a.y = th.y; a.y_stride = h->n_s;
  } else {
    a.dl_ext = th.dl_ext; a.dl_ext_stride = th.dl_ext_stride;
    a.logits_out = th.jv_out; a.logits_stride = (long long)h->n_s * h->N;
  }
  head_grad(h, a, h->sup_partial, h->plan_sup);
  a.df = DP(tn, h->L - 1, 0); a.df_stride = STRIDE(tn, dp, h->L - 1);
  return a;
}

// Forward half of the tangent pass at support slot s: the tangent of the support forward in direction u (weights), plus
// the image tangent xdot_g (padded grid, nullable: W_0 applied to it joins block 0's tangent conv as a second operand
// pair) and the norm parameters' tangents read from the meta-layout vector t_norm (nullable): BatchNorm gamma / beta of step
// s (shared by the tasks), or the layer-norm biases (t_stride floats between tasks, 0: shared).  Leaves the normalised tangents in
// tan.zh and the pooled ones in tan.ain; the features' tangent is tan.ain[L].
// pre_dgrad: also enqueue the u-weight dgrad convs of the backward half on spre, right behind the forward ones.
// defer_last: the last block's BatchNorm tangent is not launched but returned (the fused last-block kernel runs it).
static void tangent_forward(maml_b200_handle* h, int s, const float* theta, const float* u, const float* meta,
                            const float* xdot_g, const float* t_norm, long long t_stride, int T, cudaStream_t st,
                            cudaStream_t spre, bool pre_dgrad, BnActTanArgs* defer_last) {
  const PassSet& sp = h->sup; const PassSet& tn = h->tan; const PassSet& t2 = h->tan2;
  // Tangent convs of blocks >= 1 have two operand pairs; the pair (primal activation, u weights) depends only on u and
  // on what phase A saved, not on the tangent chain.  It is computed up front on the side stream (right behind the
  // u packs) into the tan2 buffers -- BatchNorm statistics contributions included, they are linear -- and the
  // consumers (bnact_tan / bnbwd_tan) add the two addends.  The main chain keeps the single-pair half: 18 instead of
  // 36 stages per tile on the critical path.  The FFMA convs (no tensor-core path) take both pairs in one launch.
  if (h->use_tc) {
    for (int l = 1; l < h->L; ++l) {
      tc_conv(h, l, sp.n, tc_op_ain(h, sp, l, s, h->u_map, 0, +1, 2),          // conv(a_in, u_W) + u_b
              u + h->pl.b_off[l], h->Ppad, ZH(t2, l, 0), STRIDE(t2, zh, l), CONV_TAN_STATS, ZH(sp, l, s),
              STRIDE(sp, zh, l), stat_at(h, PASS_TAN_FWD, s, l), T, spre);
      cudaEventRecord(h->ev_pre[l], spre);
    }
    for (int l = h->L - 1; l >= 1 && pre_dgrad; --l) {
      tc_conv(h, l, sp.n, tc_op_dz(h, sp, l, s, h->u_map, 0, -1, 0),           // dgrad(u_W, dz)
              nullptr, 0, DP(t2, l - 1, 0), STRIDE(t2, dp, l - 1), CONV_PLAIN, nullptr, 0, nullptr, T, spre);
      cudaEventRecord(h->ev_pre[MAML_MAX_LAYERS + l], spre);
    }
  }
  for (int l = 0; l < h->L; ++l) {
    if (l == 1) join_pending(h, st);
    if (l == 0) {
      Conv0Args a = conv0_args(h, sp, u, CONV_TAN_STATS, xdot_g ? 2 : 1, T);
      a.out = ZH(tn, 0, 0); a.out_stride = STRIDE(tn, zh, 0);
      a.zh = ZH(sp, 0, s); a.zh_stride = STRIDE(sp, zh, 0);
      a.stats = stat_at(h, PASS_TAN_FWD, s, 0);
      launch_conv0(a, st, xdot_g, xdot_g ? theta + h->pl.w_off[0] : nullptr);     // + conv(x_dot, W_0)
    } else if (h->use_tc) {
      tc_conv(h, l, sp.n, tc_op_ain(h, tn, l, 0, h->theta_map, s, +1, 2),       // conv(a_in_dot, W); the other addend is in tan2
              nullptr, 0, ZH(tn, l, 0), STRIDE(tn, zh, l), CONV_TAN_STATS, ZH(sp, l, s),
              STRIDE(sp, zh, l), stat_at(h, PASS_TAN_FWD, s, l), T, st);
      cudaStreamWaitEvent(st, h->ev_pre[l], 0);
    } else {
      ConvArgs a = ffma_conv(h, l, sp.n, CONV_TAN_STATS,
                             {{AIN(sp, l, s), STRIDE(sp, ain, l), u, 0, +1}, {AIN(tn, l, 0), STRIDE(tn, ain, l), theta, 0, +1}}, u, T);
      a.out = ZH(tn, l, 0); a.out_stride = STRIDE(tn, zh, l);
      a.zh = ZH(sp, l, s); a.zh_stride = STRIDE(sp, zh, l);
      a.stats = stat_at(h, PASS_TAN_FWD, s, l);
      launch_conv_rows(a, st);
    }
    norm_tangent_forward(h, s, theta, u, meta, l, t_norm, t_stride, T, st, defer_last);
  }
}

// forward-mode tangent of (support forward + support backward) at step s in direction u (and, with xdot_g, in the
// images' direction x-dot: pass the padded grid of x-dot; with t_norm, along the norm parameters' tangents, as in
// tangent_forward)  =>  H u into `partial`
static void tangent_pass(maml_b200_handle* h, int s, const float* theta, const float* u, const float* meta,
                         const TangentHead& th, int T, cudaStream_t st, const ReduceSpec& rs, cudaStream_t spre,
                         const float* xdot_g = nullptr, const float* t_norm = nullptr, long long t_stride = 0) {
  const PassSet& sp = h->sup; const PassSet& tn = h->tan;
  // the fused last-block kernels implement the cross-entropy tangent head only
  const bool fuse_tail = th.mode == HEAD_TANGENT && support_tail_fused(h);
  BnActTanArgs last_act{};
  tangent_forward(h, s, theta, u, meta, xdot_g, t_norm, t_stride, T, st, spre, true,
                  fuse_tail ? &last_act : nullptr);
  const ChunkPlan& cp = h->plan_sup;
  join_pending(h, st);
  const HeadArgs hd = tangent_head_args(h, s, theta, u, th, T);
  if (!fuse_tail) launch_head(hd, st);
  for (int l = h->L - 1; l >= 0; --l) {
    if (h->use_tc && l + 1 < h->L) cudaStreamWaitEvent(st, h->ev_pre[MAML_MAX_LAYERS + l + 1], 0);
    norm_tangent_backward(h, s, theta, u, meta, l, th.kind_tbwd, T, st, &last_act, fuse_tail ? &hd : nullptr);
    cudaEventRecord(h->ev_fork, st); cudaStreamWaitEvent(h->s_wg, h->ev_fork, 0);

    if (l == 0) {
      WgradArgs w = wgrad_args(h, 0, sp.n, cp, h->sup_partial, T);
      w.nsrc = 1;
      w.A[0] = sp.xg; w.a_stride[0] = sp.xg_stride;
      w.D[0] = DZ(tn, 0, 0); w.d_stride[0] = STRIDE(tn, dz, 0);
      if (xdot_g) {                                                    // + x_dot (x) dz: the image tangent's part
        w.nsrc = 2;
        w.A[1] = xdot_g; w.a_stride[1] = sp.xg_stride;
        w.D[1] = DZ(sp, 0, s); w.d_stride[1] = STRIDE(sp, dz, 0);
      }
      w.alg_flops = conv_flops(h, 0, sp.n, T, w.nsrc);
      if (h->L == 1) reduce_upper_on_side(h, rs, cp.pd, h->sup_partial, meta, T);
      launch_wgrad0(w, st);
    } else {
      if (h->use_tc) {
        tc_conv(h, l, sp.n, tc_op_dz(h, tn, l, 0, h->theta_map, s, -1, 0),      // dgrad(W, dz_dot); the other addend is in tan2
                nullptr, 0, DP(tn, l - 1, 0), STRIDE(tn, dp, l - 1), CONV_PLAIN, nullptr, 0, nullptr, T, st);
      } else {
        ConvArgs a = ffma_conv(h, l, sp.n, CONV_PLAIN,
                               {{DZ(tn, l, 0), STRIDE(tn, dz, l), theta, 1, -1}, {DZ(sp, l, s), STRIDE(sp, dz, l), u, 1, -1}}, nullptr, T);
        a.out = DP(tn, l - 1, 0); a.out_stride = STRIDE(tn, dp, l - 1);
        launch_conv_rows(a, st);
      }
      launch_wgrad_upper(h, l, sp.n, cp, h->sup_partial, T, {{{&sp, s}, {&tn, 0}}, {{&tn, 0}, {&sp, s}}}, h->s_wg);
      if (l == 1) reduce_upper_on_side(h, rs, cp.pd, h->sup_partial, meta, T);
    }
  }
  reduce_lower(h, rs, cp.pd, h->sup_partial, meta, T, st);
}

static void pack_theta_step(maml_b200_handle* h, int step, int T, cudaStream_t st) {
  if (!h->use_tc) return;
  const long long TP = (long long)h->maxT * h->Ppad;
  launch_pack_weights(h->pl, h->theta + (long long)step * TP, h->Ppad, h->pack_theta + (long long)step * h->maxT * h->pack_task,
                      h->pack_task, h->pack_theta_plane, T, st);
}
static void pack_u(maml_b200_handle* h, int T, cudaStream_t st) {
  if (!h->use_tc) return;
  launch_pack_weights(h->pl, h->u, h->Ppad, h->pack_u, h->pack_task, h->pack_u_plane, T, st);
}

// Forks the pre-stream of a tangent pass off `st` and packs u there (first needed by block 1 of the tangent forward, while
// the main chain runs block 0).  With the tensor-core path that is a target stream (idle then), so that the u-weight convs
// pre-computed there too do not queue in front of the weight gradients on the wgrad stream.
static int fork_direction(maml_b200_handle* h, int T, cudaStream_t st, cudaStream_t* spre) {
  *spre = h->use_tc ? h->s_tgt : h->s_wg;
  CK(cudaEventRecord(h->ev_fork, st));
  CK(cudaStreamWaitEvent(*spre, h->ev_fork, 0));
  pack_u(h, T, *spre);
  CK(cudaEventRecord(h->ev_wg, *spre));
  h->wg_pending = true;
  return 0;
}

// Export of a functional call: a plain sum over the n_tasks batches (tasks_global 1, no 1/B) into `result`, no target
// losses; with per_task, one unsummed result vector per batch at result + t * result_size.  The fused iteration sets its
// schedule on top.
static ExportArgs export_args(const maml_b200_handle* h, int T, float* result, bool per_task = false) {
  ExportArgs e{};
  e.pl = h->pl;
  e.tbar = h->tbar; e.task_stride = h->Ppad;
  e.abar = h->abar;
  e.stats = h->stats; e.stats_task_stride = h->stats_task_stride; e.st_pass_stride = h->st_pass_stride; e.st_layer_stride = h->st_layer_stride;
  e.losses = h->losses; e.correct = h->correct;
  e.target_mask = 0; e.num_steps = h->S; e.training = 1;
  e.tasks = T; e.task_offset = 0; e.tasks_global = 1;
  e.n_s = h->n_s; e.n_t = h->n_t;
  for (int l = 0; l < h->L; ++l) e.hw[l] = h->geo[l].h * h->geo[l].w;
  e.result = result;
  e.per_task = per_task ? 1 : 0; e.result_stride = maml_b200_result_size(h);
  e.lnb = h->lnb;
  return e;
}

// enqueue one whole iteration; `st` is either the caller's stream (eager / profiling) or the capture stream
static int enqueue_iteration(maml_b200_handle* h, const maml_b200_iter_args* it, const float* meta, const float* x_support,
                             const long long* ys, const float* x_target, const long long* yt, float* result, float* last_logits,
                             cudaStream_t st) {
  g_launch_base = g_launch_counter;      // launch tags (device trace) count from the start of the iteration
  LaunchScope launch_scope(h, st);
  const int T = it->n_tasks;
  const unsigned mask = it->target_mask & ((1u << it->num_steps) - 1u);
  const long long TP = (long long)h->maxT * h->Ppad;
  // diagnostic (MAML_B200_ONE_STREAM=1): everything on one stream -> the device trace shows true kernel durations
  struct StreamSwap {
    maml_b200_handle* h; cudaStream_t tgt, tgt2, wg; bool on;
    StreamSwap(maml_b200_handle* h_, cudaStream_t st) : h(h_), tgt(h_->s_tgt), tgt2(h_->s_tgt2), wg(h_->s_wg), on(h_->opt.one_stream) {
      if (on) { h->s_tgt = st; h->s_tgt2 = st; h->s_wg = st; }
    }
    ~StreamSwap() { if (on) { h->s_tgt = tgt; h->s_tgt2 = tgt2; h->s_wg = wg; } }
  } stream_swap(h, st);
  int last_t = 0;
  for (int s = 0; s < it->num_steps; ++s) if (mask & (1u << s)) last_t = s;

  if (clear_accumulators(h, CLR_STATS | CLR_ABAR | CLR_LOSSES | CLR_CORRECT, st)) return 1;

  launch_prep_x(x_support, h->sup.xg, h->sup.xg_stride, T, h->n_s, h->C, h->H, h->W, st);
  launch_import_theta(h->pl, meta, h->theta, h->Ppad, T, st);
  // The target images and the tensor-core packs of theta^0 are first needed after block 0 of the first support pass: both
  // go to the side stream (off the head of the main chain).  Every consumer already waits for ev_wg: the main chain
  // through join_pending before block 1, the target streams before each pass.
  CK(cudaEventRecord(h->ev_fork, st));
  CK(cudaStreamWaitEvent(h->s_wg, h->ev_fork, 0));
  launch_prep_x(x_target, h->tgt.xg, h->tgt.xg_stride, T, h->n_t, h->C, h->H, h->W, h->s_wg);
  pack_theta_step(h, 0, T, h->s_wg);
  CK(cudaEventRecord(h->ev_wg, h->s_wg));
  h->wg_pending = true;

  // ---------------- phase A: unroll the inner loop.  Support chain on `st`; the target pass of step s (forward at
  // theta^{s+1}, and its backward) only feeds phase B, so it runs on a side stream concurrently with step s+1.
  for (int s = 0; s < it->num_steps; ++s) {
    const float* th = h->theta + (long long)s * TP;
    float* th_next = h->theta + (long long)(s + 1) * TP;
    const bool fuse_tail = support_tail_fused(h);
    BnActArgs last_act{};
    forward_pass(h, h->sup, s, th, s, meta, s, PASS_SUP_FWD, T, st, fuse_tail ? &last_act : nullptr);
    join_pending(h, st);
    HeadArgs hd = head_args(h, HEAD_SUPPORT, h->sup, s, th, T);
    hd.y = ys; hd.y_stride = h->n_s;
    head_grad(h, hd, h->sup_partial, h->plan_sup);
    if (!fuse_tail) launch_head(hd, st);
    // LSLR update theta^{s+1} = theta^s - alpha[.][s] * g and the tensor-core packs of theta^{s+1}: blocks >= 1 and the
    // linear layer on the side stream, block 0 at the end of the main chain
    ReduceSpec rs{PR_UPDATE, th, th_next, h->g + (long long)s * TP, nullptr, s, s + 1, stat_at(h, PASS_SUP_BWD, s, 0)};
    backward_pass(h, h->sup, s, th, s, meta, s, PASS_SUP_FWD, PASS_SUP_BWD, h->sup_partial, h->plan_sup, T, st, true, &rs,
                  fuse_tail ? &last_act : nullptr, fuse_tail ? &hd : nullptr);
    if (mask & (1u << s)) {
      // target passes of different steps are independent (each only needs theta^{s+1}): alternate two streams and two
      // buffer slots so that pass s+1 does not queue behind pass s (the target chain was the longest path of phase A)
      const int tpar = (h->tgt_slots > 1) ? (s & 1) : 0;
      cudaStream_t ts_ = tpar ? h->s_tgt2 : h->s_tgt;
      float* tpart = h->tgt_partial + (long long)tpar * h->maxT * h->plan_tgt.size;
      CK(cudaEventRecord(h->ev_pack, st));
      CK(cudaStreamWaitEvent(ts_, h->ev_pack, 0));       // block-0 weights of theta^{s+1}
      CK(cudaStreamWaitEvent(ts_, h->ev_wg, 0));         // everything else + packs (side stream)
      const int ts = (h->cfg.reserved & 1) ? s : tpar;
      forward_pass(h, h->tgt, ts, th_next, s + 1, meta, s, PASS_TGT_FWD, T, ts_);
      HeadArgs a = head_args(h, HEAD_TARGET_FWD, h->tgt, ts, th_next, T);
      a.y = yt; a.y_stride = h->n_t;
      a.loss_out = h->losses + s; a.loss_stride = MAML_MAX_STEPS;
      if (s == last_t) {
        a.logits_out = last_logits; a.logits_stride = (long long)h->n_t * h->N;
        a.correct_out = h->correct; a.correct_stride = 1;
      }
      launch_head(a, ts_);
      if (it->training) {
        HeadArgs bqa = head_args(h, HEAD_TARGET_BWD, h->tgt, ts, th_next, T);
        bqa.y = yt; bqa.y_stride = h->n_t; bqa.scale = it->target_weight[s];
        head_grad(h, bqa, tpart, h->plan_tgt);
        launch_head(bqa, ts_);
        backward_pass(h, h->tgt, ts, th_next, s + 1, meta, s, PASS_TGT_FWD, PASS_TGT_BWD, tpart, h->plan_tgt, T, ts_, false);
        launch_param_reduce(h->pl, with_bn_sums(h, h->plan_tgt.pd, stat_at(h, PASS_TGT_BWD, s, 0)), tpart, PR_STORE, nullptr,
                            nullptr, h->tgrad + (long long)s * TP, nullptr, meta, s, h->Ppad, T, ts_);
      }
      CK(cudaEventRecord(h->ev_tgt[s], ts_));
    }
  }

  // ---------------- phase B: reverse sweep (joins the target chain step by step)
  if (it->training) {
    CK(cudaMemsetAsync(h->tbar, 0, (size_t)TP * sizeof(float), st));
    for (int s = it->num_steps - 1; s >= 0; --s) {
      const float* th = h->theta + (long long)s * TP;
      const float* tg = nullptr;
      if (mask & (1u << s)) { tg = h->tgrad + (long long)s * TP; CK(cudaStreamWaitEvent(st, h->ev_tgt[s], 0)); }
      join_pending(h, st);                               // g^s / tbar parts reduced on the side stream
      launch_dots_u(h->pl, h->tbar, tg, h->g + (long long)s * TP, h->u, h->abar, meta, s, h->Ppad, T, st);
      if (it->second_order) {
        cudaStream_t spre;
        if (fork_direction(h, T, st, &spre)) return 1;
        ReduceSpec rs{PR_SUB, nullptr, nullptr, nullptr, h->tbar, s, -1, stat_at(h, PASS_TAN_BWD, s, 0)};
        tangent_pass(h, s, th, h->u, meta, TangentHead{HEAD_TANGENT, ys, nullptr, 0, nullptr, PASS_TAN_BWD}, T, st, rs, spre);
      }
    }
    join_pending(h, st);
  } else {
    join_pending(h, st);
    for (int s = 0; s < it->num_steps; ++s) if (mask & (1u << s)) CK(cudaStreamWaitEvent(st, h->ev_tgt[s], 0));
  }

  ExportArgs e = export_args(h, T, result);
  for (int s = 0; s < MAML_MAX_STEPS; ++s) e.weights[s] = it->target_weight[s];
  e.target_mask = mask; e.num_steps = it->num_steps; e.training = it->training;
  e.task_offset = it->task_offset; e.tasks_global = it->tasks_global;
  // sharded call with a connected communicator: export publishes into the peer-visible slot and the all-reduce kernel
  // (same stream, same captured graph) leaves the SUM over ranks in `result` -- no host round trip, no library call
  const bool reduce = h->comm_connected && it->tasks_global > it->n_tasks;
  if (reduce) e.comm = h->comm;
  launch_export(e, st);
  if (reduce) launch_allreduce(h->comm, result, maml_b200_result_size(h), st);
  return 0;
}

extern "C" int maml_b200_meta_batch_fwd_bwd(maml_b200_handle* h, const maml_b200_iter_args* it, const float* meta,
                                            const float* x_support, const int64_t* y_support, const float* x_target,
                                            const int64_t* y_target, float* result, float* last_logits, void* stream) {
  if (!h || !it || !meta || !x_support || !y_support || !x_target || !y_target || !result) return fail("null argument");
  const int T = it->n_tasks;
  if (T < 1 || T > h->maxT) return fail("n_tasks out of range");
  if (it->num_steps < 1 || it->num_steps > h->S) return fail("num_steps out of range (must be <= inner_steps)");
  if (it->tasks_global < T) return fail("tasks_global < n_tasks");
  if ((it->target_mask & ((1u << it->num_steps) - 1u)) == 0) return fail("target_mask selects no target pass");
  if (h->comm_connected && (reinterpret_cast<uintptr_t>(result) & 15u) != 0) return fail("result must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const long long* ys = (const long long*)y_support;
  const long long* yt = (const long long*)y_target;
  h->last_tasks = T;
  record_call(h, FN_NONE, 0, 0);           // the iteration reuses the functional calls' buffers

  if (!h->use_graphs || h->profiling) {
    // eager: launches go straight to the caller's stream (side streams fork / join through events)
    const long long launches0 = g_launch_counter;
    if (enqueue_iteration(h, it, meta, x_support, ys, x_target, yt, result, last_logits, st)) return 1;
    h->last_launches = g_launch_counter - launches0;
    CK(cudaGetLastError());
    return 0;
  }

  // CUDA graph: the launch sequence depends only on the schedule and the buffer addresses -> capture once, replay.
  const void* ptrs[7] = {meta, x_support, y_support, x_target, y_target, result, last_logits};
  maml_b200_handle::GraphEntry* hit = nullptr;
  for (auto& g : h->graphs)
    if (memcmp(&g.it, it, sizeof(*it)) == 0 && memcmp(g.p, ptrs, sizeof(ptrs)) == 0) { hit = &g; break; }
  if (!hit) {
    if (h->graphs.size() >= 32) {           // evict the least recently used entry
      size_t victim = 0;
      for (size_t i = 1; i < h->graphs.size(); ++i) if (h->graphs[i].stamp < h->graphs[victim].stamp) victim = i;
      cudaGraphExecDestroy(h->graphs[victim].exec);
      h->graphs.erase(h->graphs.begin() + victim);
    }
    const long long launches0 = g_launch_counter;
    CK(cudaStreamBeginCapture(h->s_cap, cudaStreamCaptureModeThreadLocal));
    const int rc = enqueue_iteration(h, it, meta, x_support, ys, x_target, yt, result, last_logits, h->s_cap);
    cudaGraph_t graph = nullptr;
    cudaError_t e = cudaStreamEndCapture(h->s_cap, &graph);
    if (rc) { if (graph) cudaGraphDestroy(graph); return 1; }
    if (e != cudaSuccess) return fail(std::string("cudaStreamEndCapture: ") + cudaGetErrorString(e));
    if (!h->opt.graph_dot.empty()) cudaGraphDebugDotPrint(graph, h->opt.graph_dot.c_str(), cudaGraphDebugDotFlagsKernelNodeParams);
    maml_b200_handle::GraphEntry ge;
    ge.it = *it; memcpy(ge.p, ptrs, sizeof(ptrs)); ge.exec = nullptr; ge.launches = g_launch_counter - launches0; ge.stamp = 0;
    e = cudaGraphInstantiate(&ge.exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) return fail(std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e));
    h->graphs.push_back(ge);
    hit = &h->graphs.back();
  }
  hit->stamp = ++h->graph_clock;
  h->last_launches = hit->launches;
  CK(cudaGraphLaunch(hit->exec, st));
  return 0;
}

// Argument checks of the functional entries; `ptrs`: the entry's required pointers are all non-null.
static int check_call(const maml_b200_handle* h, bool ptrs, int n_tasks, int num_step) {
  if (!h || !ptrs) return fail("null argument");
  if (n_tasks < 1 || n_tasks > h->maxT) return fail("n_tasks out of range");
  if (num_step < 0 || num_step >= h->S) return fail("num_step out of range");
  return 0;
}

// The shared-weight entries (net_forward, net_backward, net_hvp, net_hvp_image, net_jvp) read the BatchNorm gamma / beta of
// num_step, shared by the tasks; an inner_bn handle has no such rows, its gamma / beta are per-task fast weights.
static int refuse_inner_bn(const maml_b200_handle* h, const char* entry, const char* per_task) {
  if (h && h->pl.inner_bn)
    return fail(std::string("maml_b200_") + entry + " shares BatchNorm gamma / beta between the tasks; an inner_bn handle "
                "(per-task gamma / beta) runs maml_b200_" + per_task);
  return 0;
}

// Stages a functional call's batch and runs its primal forward on pass set `ps` at `slot`: x (and the image tangent xdot,
// support grid only) onto the block-0 grid, meta_like into theta slot `slot` (and dir_like into u), the tensor-core packs
// of that slot, then the forward with the BatchNorm gamma / beta of num_step (read from task 0's meta_like; inner_bn: each
// task's own, imported into theta with its weights, and their directions into u).  meta_stride /
// dir_stride: floats between consecutive tasks' vectors (0: one vector for all tasks).  Returns the theta slot.
static const float* stage_forward(maml_b200_handle* h, const PassSet& ps, int slot, int stat_kind, int num_step, const float* meta_like,
                                  long long meta_stride, const float* x, const float* xdot, const float* dir_like, long long dir_stride,
                                  int T, cudaStream_t st) {
  float* th = h->theta + (long long)slot * h->maxT * h->Ppad;
  launch_prep_x(x, ps.xg, ps.xg_stride, T, ps.n, h->C, h->H, h->W, st);
  if (xdot) launch_prep_x(xdot, h->xdot_g, ps.xg_stride, T, ps.n, h->C, h->H, h->W, st);
  launch_import_theta(h->pl, meta_like, th, h->Ppad, T, st, meta_stride);
  if (dir_like) launch_import_theta(h->pl, dir_like, h->u, h->Ppad, T, st, dir_stride);
  pack_theta_step(h, slot, T, st);
  forward_pass(h, ps, slot, th, slot, meta_like, num_step, stat_kind, T, st);
  return th;
}

// Backward of an external d(logits) [T][ps.n][N] through pass set `ps` at `slot` (theta slot `slot`, BatchNorm gamma / beta
// of num_step): the HEAD_EXTERNAL_BWD head, then backward_pass into the weight-gradient chunks `partial`.
static void external_backward(maml_b200_handle* h, const PassSet& ps, int slot, int num_step, int kind_fwd, int kind_bwd,
                              const float* meta_like, const float* dlogits, float* partial, const ChunkPlan& cp, int T, cudaStream_t st) {
  const float* th = h->theta + (long long)slot * h->maxT * h->Ppad;
  HeadArgs a = head_args(h, HEAD_EXTERNAL_BWD, ps, slot, th, T);
  a.dl_ext = dlogits; a.dl_ext_stride = (long long)ps.n * h->N;
  head_grad(h, a, partial, cp);
  launch_head(a, st);
  backward_pass(h, ps, slot, th, slot, meta_like, num_step, kind_fwd, kind_bwd, partial, cp, T, st, false);
}

// Stand-alone functional forward (level B1 of the boundary): logits of `n_tasks` independent batches of N*T images
// under externally supplied weights.  `meta_like` has the layout of the meta vector (conv / linear entries = the
// weights to use, BatchNorm entries = gamma / beta; LSLR entries ignored).  BatchNorm uses batch statistics and the
// gamma / beta of `num_step`, exactly like reference VGGReLUNormNetwork.forward (training flag is ignored there too).
static int check_strides(long long meta_stride, long long dir_stride, int64_t meta_size) {
  if (meta_stride < 0 || dir_stride < 0) return fail("negative task stride");
  if ((meta_stride > 0 && meta_stride < meta_size) || (dir_stride > 0 && dir_stride < meta_size))
    return fail("task stride smaller than meta_size (consecutive tasks' vectors would overlap)");
  return 0;
}

extern "C" int maml_b200_net_forward_tasks(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like,
                                          int64_t meta_stride, const float* x, float* logits, void* stream) {
  if (check_call(h, meta_like && x && logits, n_tasks, num_step)) return 1;
  if (check_strides(meta_stride, 0, h->pl.meta_size)) return 1;
  cudaStream_t st = (cudaStream_t)stream;
  LaunchScope launch_scope(h, st);
  const int T = n_tasks;
  record_call(h, FN_NONE, 0, 0);
  if (clear_accumulators(h, CLR_STATS | CLR_LOSSES | CLR_CORRECT, st)) return 1;
  const float* th = stage_forward(h, h->tgt, 0, PASS_TGT_FWD, num_step, meta_like, meta_stride, x, nullptr, nullptr, 0, T, st);
  HeadArgs a = head_args(h, HEAD_TARGET_FWD, h->tgt, 0, th, T);
  a.loss_out = h->losses; a.loss_stride = MAML_MAX_STEPS;
  a.logits_out = logits; a.logits_stride = (long long)h->n_t * h->N;
  launch_head(a, st);
  CK(cudaGetLastError());
  record_call(h, FN_FORWARD, T, num_step);
  return 0;
}

extern "C" int maml_b200_net_forward(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like,
                                    const float* x, float* logits, void* stream) {
  if (refuse_inner_bn(h, "net_forward", "net_forward_tasks")) return 1;
  return maml_b200_net_forward_tasks(h, n_tasks, num_step, meta_like, 0, x, logits, stream);
}

// Backward of the functional forward above (level B1: lets torch.autograd differentiate through the operator, the way the
// reference's apply_inner_loop_update does with torch.autograd.grad, few_shot_learning_system.py:138-139, first order).
// Must follow maml_b200_net_forward (or another net_backward of it) on the same handle with the same (n_tasks, num_step,
// meta_like): the activations of that call are what this one differentiates.  The handle's call record refuses another
// order, n_tasks or num_step (meta_like it cannot check).  dlogits [n_tasks, N*T, N] = d(loss)/d(logits).  grad_out:
// result_size floats; the first meta_size hold d(loss)/d(meta_like) in the meta layout (conv / linear weights and biases,
// BatchNorm beta / gamma of `num_step`; LSLR entries 0), summed over the n_tasks batches (sum_tasks) or one vector per batch
// at grad_out + t * result_size.  No gradient w.r.t. the images.
extern "C" int maml_b200_net_backward_tasks(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like,
                                           int64_t meta_stride, const float* dlogits, float* grad_out, int32_t sum_tasks,
                                           void* stream) {
  if (check_call(h, meta_like && dlogits && grad_out, n_tasks, num_step)) return 1;
  if (check_strides(meta_stride, 0, h->pl.meta_size)) return 1;
  if (require_call(h, FN_FORWARD | FN_BACKWARD, n_tasks, num_step, "maml_b200_net_backward")) return 1;
  cudaStream_t st = (cudaStream_t)stream;
  LaunchScope launch_scope(h, st);
  const int T = n_tasks;
  record_call(h, FN_NONE, 0, 0);
  // backward sums (and the tangent ones export subtracts) start from zero; the forward sums of net_forward are kept.  Layer
  // norm: export sums both kinds of bias-gradient rows over every step
  if (clear_accumulators(h, CLR_BWD_STATS | CLR_ABAR | CLR_LOSSES | CLR_CORRECT, st, T)) return 1;
  external_backward(h, h->tgt, 0, num_step, PASS_TGT_FWD, PASS_TGT_BWD, meta_like, dlogits, h->tgt_partial, h->plan_tgt, T, st);
  // inner_bn: the beta / gamma rows are each task's backward sums S1 / S2 (export has no gamma / beta rows of its own)
  const PartialDesc pd = h->pl.inner_bn ? with_bn_sums(h, h->plan_tgt.pd, stat_at(h, PASS_TGT_BWD, num_step, 0)) : h->plan_tgt.pd;
  launch_param_reduce(h->pl, pd, h->tgt_partial, PR_STORE, nullptr, nullptr, h->tbar, nullptr, meta_like, num_step, h->Ppad, T, st);
  launch_export(export_args(h, T, grad_out, !sum_tasks), st);
  CK(cudaGetLastError());
  record_call(h, FN_BACKWARD, T, num_step);
  return 0;
}

extern "C" int maml_b200_net_backward(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like,
                                     const float* dlogits, float* grad_out, void* stream) {
  if (refuse_inner_bn(h, "net_backward", "net_backward_tasks")) return 1;
  return maml_b200_net_backward_tasks(h, n_tasks, num_step, meta_like, 0, dlogits, grad_out, 1, stream);
}

// A forward-mode buffer allocated on first use and zeroed on the call's stream (the kernels that read it run there; a
// plain cudaMemset would not be ordered before them on a non-blocking stream).  Nothing is kept if a step fails.
static int alloc_zeroed(float** out, size_t bytes, cudaStream_t st) {
  float* p = nullptr;
  CK(cudaMalloc((void**)&p, bytes));
  const cudaError_t e = cudaMemsetAsync(p, 0, bytes, st);
  if (e != cudaSuccess) { cudaFree(p); return fail(std::string("cudaMemsetAsync: ") + cudaGetErrorString(e)); }
  *out = p;
  return 0;
}

// The support-grid buffer of the image tangent x-dot (guard rows included, as sup.xg; zero outside the images).
static int ensure_xdot(maml_b200_handle* h, cudaStream_t st) {
  if (h->xdot_g) return 0;
  float* p = nullptr;
  if (alloc_zeroed(&p, (size_t)h->sup.xg_stride * h->maxT * sizeof(float), st)) return 1;
  h->xdot_g = p + (long long)h->geo[0].guard * h->C;
  return 0;
}

// Second-order companion of maml_b200_net_backward: what torch.autograd needs to differentiate the backward of the
// functional operator once more (the reference's loss.backward() through torch.autograd.grad(..., create_graph=True),
// few_shot_learning_system.py:138-139).  Self-contained: meta_like is imported into theta[num_step] and the whole chain
// runs at support slot s = num_step, exactly as the fused iteration's support chain does at step s -- forward, backward of
// the external dlogits, then the tangent pass along v_like with dlogits held constant (HEAD_EXTERNAL_TAN).  Batches of
// N*K images (the handle's support shape).  jv_out [n_tasks, N*K, N] = J v.  hv_out: result_size floats; the first meta_size
// hold d/d(meta_like) <dlogits, J v> in the meta layout, summed over the batches: conv / linear entries are stored into
// tbar by the parameter reduction, the BatchNorm gamma / beta sums go to the PASS_TGT_BWD statistics, which export adds
// (+H_gamma v, +H_beta v), and a layer-norm handle's bias sums to the bias-gradient rows export adds (+H_b v); LSLR
// entries 0.  v_like's BatchNorm and LSLR entries are not read; on a layer-norm handle its bias entries are the bias
// directions (the tangent forward's b-dot).  Overwrites the batch statistics maml_b200_net_running_update reads; no
// running-statistics side effect of its own.
// meta_stride / dir_stride / sum_tasks: as in maml_b200_net_hvp_image_tasks.
static int net_hvp_impl(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like, long long meta_stride,
                        const float* x, const float* xdot, const float* dlogits, const float* v_like, long long dir_stride,
                        float* jv_out, float* hv_out, bool sum_tasks, void* stream) {
  if (check_call(h, meta_like && x && dlogits && v_like && jv_out && hv_out, n_tasks, num_step)) return 1;
  if (check_strides(meta_stride, dir_stride, h->pl.meta_size)) return 1;
  cudaStream_t st = (cudaStream_t)stream;
  LaunchScope launch_scope(h, st);
  const int T = n_tasks, s = num_step;
  record_call(h, FN_NONE, 0, 0);                 // at num_step 0 this overwrites the weights net_forward imported
  if (xdot && ensure_xdot(h, st)) return 1;
  if (clear_accumulators(h, CLR_STATS | CLR_ABAR | CLR_LOSSES | CLR_CORRECT, st)) return 1;
  const float* th = stage_forward(h, h->sup, s, PASS_SUP_FWD, s, meta_like, meta_stride, x, xdot, v_like, dir_stride, T, st);
  // the tangent pass reads this backward's dz / dp and statistics; its weight-gradient chunks are overwritten unread
  external_backward(h, h->sup, s, s, PASS_SUP_FWD, PASS_SUP_BWD, meta_like, dlogits, h->sup_partial, h->plan_sup, T, st);
  cudaStream_t spre;
  if (fork_direction(h, T, st, &spre)) return 1;
  // inner_bn: the beta / gamma rows are the tangent backward's sums (kind_tbwd), stored as they are: +H_beta v, +H_gamma v
  const TangentHead th_ext{HEAD_EXTERNAL_TAN, nullptr, dlogits, (long long)h->n_s * h->N, jv_out, PASS_TGT_BWD};
  ReduceSpec rs{PR_STORE, nullptr, nullptr, h->tbar, nullptr, s, -1, h->pl.inner_bn ? stat_at(h, th_ext.kind_tbwd, s, 0) : nullptr};
  // Norm-parameter directions: an inner_bn handle's gamma / beta directions are u's (imported from v_like per task), a
  // layer-norm handle's bias directions are read from v_like's norm entries (t_norm); a plain BatchNorm handle has none
  tangent_pass(h, s, th, h->u, meta_like, th_ext, T, st, rs, spre, xdot ? h->xdot_g : nullptr, h->ln ? v_like : nullptr,
               dir_stride);
  join_pending(h, st);
  launch_export(export_args(h, T, hv_out, !sum_tasks), st);
  CK(cudaGetLastError());
  record_call(h, FN_HVP, T, num_step);
  return 0;
}

extern "C" int maml_b200_net_hvp(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like, const float* x,
                                 const float* dlogits, const float* v_like, float* jv_out, float* hv_out, void* stream) {
  if (refuse_inner_bn(h, "net_hvp", "net_hvp_image_tasks")) return 1;
  return net_hvp_impl(h, n_tasks, num_step, meta_like, 0, x, nullptr, dlogits, v_like, 0, jv_out, hv_out, true, stream);
}

// maml_b200_net_hvp along the images too: the tangent direction is (v_like's weights, xdot).  jv_out = J_theta v +
// J_x xdot; hv_out = d/d(meta_like) <dlogits, jv_out>.  The first block's tangent conv takes W_0 applied to xdot as a
// second operand pair and its weight-gradient tangent adds xdot (x) dz_0.  xdot NULL is maml_b200_net_hvp.
extern "C" int maml_b200_net_hvp_image(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like,
                                       const float* x, const float* xdot, const float* dlogits, const float* v_like, float* jv_out,
                                       float* hv_out, void* stream) {
  if (refuse_inner_bn(h, "net_hvp_image", "net_hvp_image_tasks")) return 1;
  return net_hvp_impl(h, n_tasks, num_step, meta_like, 0, x, xdot, dlogits, v_like, 0, jv_out, hv_out, true, stream);
}

// Per-task form of maml_b200_net_hvp_image: task t's weights at meta_like + t * meta_stride and its direction at
// v_like + t * dir_stride (0: shared); hv_out summed over the tasks (sum_tasks) or one vector per task.
extern "C" int maml_b200_net_hvp_image_tasks(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like,
                                             int64_t meta_stride, const float* x, const float* xdot, const float* dlogits,
                                             const float* v_like, int64_t dir_stride, float* jv_out, float* hv_out,
                                             int32_t sum_tasks, void* stream) {
  return net_hvp_impl(h, n_tasks, num_step, meta_like, meta_stride, x, xdot, dlogits, v_like, dir_stride, jv_out, hv_out,
                      sum_tasks != 0, stream);
}

// Forward mode of the functional operator: jv_out [n_tasks, N*K, N] = J_theta t + J_x xdot at the weights meta_like, for
// batches of N*K images (the handle's support shape).  Self-contained: the primal forward at support slot num_step, then
// the forward half of the tangent pass (no backward).  t_like in the meta layout: conv / linear entries are the weight
// tangents, the BatchNorm beta / gamma rows their tangents (inner_bn: per task, as the weights; otherwise those of
// num_step, shared) or the layer-norm bias tangents; LSLR entries are not read.  xdot may be NULL.  Task t's weights at
// meta_like + t * meta_stride, its tangent at t_like + t * dir_stride (0: shared).
// The logits tangent comes from the HEAD_EXTERNAL_TAN head with d(logits) = 0, whose gradient outputs are discarded.
// Overwrites the batch statistics maml_b200_net_running_update reads; no running-statistics side effect of its own.
extern "C" int maml_b200_net_jvp_tasks(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like,
                                       int64_t meta_stride, const float* x, const float* t_like, int64_t dir_stride,
                                       const float* xdot, float* jv_out, void* stream) {
  if (check_call(h, meta_like && x && t_like && jv_out, n_tasks, num_step)) return 1;
  if (check_strides(meta_stride, dir_stride, h->pl.meta_size)) return 1;
  cudaStream_t st = (cudaStream_t)stream;
  LaunchScope launch_scope(h, st);
  const int T = n_tasks, s = num_step;
  record_call(h, FN_NONE, 0, 0);
  if (xdot && ensure_xdot(h, st)) return 1;
  // zero d(logits) of one batch, read with a task stride of 0
  if (!h->zero_dl && alloc_zeroed(&h->zero_dl, (size_t)h->n_s * h->N * sizeof(float), st)) return 1;
  if (clear_accumulators(h, CLR_STATS, st)) return 1;
  const float* th = stage_forward(h, h->sup, s, PASS_SUP_FWD, s, meta_like, meta_stride, x, xdot, t_like, dir_stride, T, st);
  cudaStream_t spre;
  if (fork_direction(h, T, st, &spre)) return 1;
  tangent_forward(h, s, th, h->u, meta_like, xdot ? h->xdot_g : nullptr, t_like, dir_stride, T, st, spre, false, nullptr);
  join_pending(h, st);
  launch_head(tangent_head_args(h, s, th, h->u, TangentHead{HEAD_EXTERNAL_TAN, nullptr, h->zero_dl, 0, jv_out, PASS_TGT_BWD}, T), st);
  CK(cudaGetLastError());
  return 0;
}

extern "C" int maml_b200_net_jvp(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, const float* meta_like, const float* x,
                                 const float* t_like, const float* xdot, float* jv_out, void* stream) {
  if (refuse_inner_bn(h, "net_jvp", "net_jvp_tasks")) return 1;
  return maml_b200_net_jvp_tasks(h, n_tasks, num_step, meta_like, 0, x, t_like, 0, xdot, jv_out, stream);
}

// First-block data gradient of a functional call, straight into NCHW images: dx = sum over the pairs (W_k, D_k) of
// W_k^T applied to D_k, where D_k is a gradient at the first conv's output.
static int input_grad(maml_b200_handle* h, int n_tasks, const Slot* D, const float* const* W, int nsrc, float* dx_out,
                      cudaStream_t st) {
  LaunchScope launch_scope(h, st);
  const LayerGeom& g = h->geo[0];
  const PassSet& ps = *D[0].ps;
  InputGradArgs a{};
  for (int k = 0; k < nsrc; ++k) {
    a.D[k] = DZ(*D[k].ps, 0, D[k].slot); a.d_stride[k] = STRIDE(*D[k].ps, dz, 0); a.W[k] = W[k];
  }
  a.w_stride = h->Ppad;
  a.dx = dx_out; a.dx_stride = (long long)ps.n * h->C * h->H * h->W;
  a.nsrc = nsrc; a.rows = ps.n * g.G; a.gw = g.gw; a.G = g.G; a.h = g.h; a.w = g.w; a.c0 = h->C; a.ncols = h->F;
  a.tasks = n_tasks;
  a.alg_flops = conv_flops(h, 0, ps.n, n_tasks, nsrc);
  launch_input_grad0(a, st);
  CK(cudaGetLastError());
  return 0;
}

// d(loss)/d(x) of the immediately preceding maml_b200_net_backward on this handle: W_0^T applied to the first block's
// output gradient of that backward (target pass, theta slot 0 as imported by net_forward).
extern "C" int maml_b200_net_input_grad(maml_b200_handle* h, int32_t n_tasks, float* dx_out, void* stream) {
  if (!h || !dx_out) return fail("null argument");
  if (require_call(h, FN_BACKWARD, n_tasks, -1, "maml_b200_net_input_grad")) return 1;
  const Slot D[1] = {{&h->tgt, 0}};
  const float* W[1] = {h->theta + h->pl.w_off[0]};
  return input_grad(h, n_tasks, D, W, 1, dx_out, (cudaStream_t)stream);
}

// d/dx <dlogits, J v> of the immediately preceding maml_b200_net_hvp on this handle: the tangent of the image gradient
// along v, W_0^T applied to the tangent of the first block's output gradient plus U_0^T applied to that gradient itself
// (support pass and theta slot num_step of the hvp call, u = v's weights).
extern "C" int maml_b200_net_hvp_input_grad(maml_b200_handle* h, int32_t n_tasks, float* dxdot_out, void* stream) {
  if (!h || !dxdot_out) return fail("null argument");
  if (require_call(h, FN_HVP, n_tasks, -1, "maml_b200_net_hvp_input_grad")) return 1;
  const int s = h->fn_step;
  const Slot D[2] = {{&h->tan, 0}, {&h->sup, s}};
  const float* W[2] = {h->theta + (long long)s * h->maxT * h->Ppad + h->pl.w_off[0], h->u + h->pl.w_off[0]};
  return input_grad(h, n_tasks, D, W, 2, dxdot_out, (cudaStream_t)stream);
}

// Side effect of the functional forward in the reference: F.batch_norm's EMA update of running_mean / running_var at
// `num_step` (meta_neural_network_architectures.py:226-247), from the batch statistics of the last maml_b200_net_forward
// call (one update per batch, in order).  running_mean / running_var: [stages][S][F] device.  No-op for shared BatchNorm
// (the reference passes running stats = None there).  Another functional call on the same handle in between overwrites
// those statistics (net_backward keeps them): the handle's call record refuses any other order, n_tasks or num_step.
extern "C" int maml_b200_net_running_update(maml_b200_handle* h, int32_t n_tasks, int32_t num_step, float* running_mean,
                                           float* running_var, void* stream) {
  if (check_call(h, running_mean && running_var, n_tasks, num_step)) return 1;
  if (require_call(h, FN_FORWARD | FN_BACKWARD, n_tasks, num_step, "maml_b200_net_running_update")) return 1;
  if (!h->pl.per_step_bn) return 0;      // shared BatchNorm, and layer norm (no running statistics)
  LaunchScope launch_scope(h);
  int hw[MAML_MAX_LAYERS];
  for (int l = 0; l < h->L; ++l) hw[l] = h->geo[l].h * h->geo[l].w;
  launch_running_ema_from_stats(stat_at(h, PASS_TGT_FWD, num_step, 0), h->stats_task_stride, h->st_layer_stride, n_tasks, running_mean,
                                running_var, h->L, h->S, h->F, num_step, hw, h->n_t, (cudaStream_t)stream);
  CK(cudaGetLastError());
  return 0;
}

extern "C" int maml_b200_adam_step(maml_b200_handle* h, float* meta, const float* grad, float* exp_avg, float* exp_avg_sq,
                                   float lr, int32_t step, uint64_t trainable_mask, uint64_t clamp_mask, void* stream) {
  if (!h || !meta || !grad || !exp_avg || !exp_avg_sq) return fail("null argument");
  if (step < 1) return fail("step must be >= 1");
  LaunchScope launch_scope(h);
  std::vector<long long> ends;
  for (size_t k = 0; k < h->seg_off.size(); ++k) ends.push_back(h->seg_off[k] + h->seg_size[k]);
  const float bc1 = (float)(1.0 - pow(0.9, (double)step));
  const float bc2 = (float)(1.0 - pow(0.999, (double)step));
  // one launch per 32 segments (the kernel's segment table and masks): an inner_bn handle with 4 blocks has 36
  for (size_t k0 = 0; k0 < ends.size(); k0 += 32) {
    const size_t nk = std::min<size_t>(32, ends.size() - k0);
    const long long base = k0 ? ends[k0 - 1] : 0;
    std::vector<long long> rel(nk);
    for (size_t k = 0; k < nk; ++k) rel[k] = ends[k0 + k] - base;
    launch_adam(meta + base, grad + base, exp_avg + base, exp_avg_sq + base, rel[nk - 1], lr, bc1, bc2, rel.data(), (int)nk,
                (uint32_t)(trainable_mask >> k0), (uint32_t)(clamp_mask >> k0), (cudaStream_t)stream);
  }
  CK(cudaGetLastError());
  return 0;
}

extern "C" int maml_b200_running_stats_update(maml_b200_handle* h, const float* result, float* running_mean, float* running_var,
                                              const float* decay_host, void* stream) {
  if (!h || !result || !running_mean || !running_var || !decay_host) return fail("null argument");
  // shared-BN mode passes running stats = None in the reference, and layer norm has none: no update
  if (!h->pl.per_step_bn) return 0;
  LaunchScope launch_scope(h);
  cudaStream_t st = (cudaStream_t)stream;
  float* pin = h->pinned + 32 * (h->pin_slot++ & 15);
  for (int s = 0; s < h->S; ++s) pin[s] = decay_host[s];
  CK(cudaMemcpyAsync(h->decay_dev, pin, h->S * sizeof(float), cudaMemcpyHostToDevice, st));
  const long long LSF = (long long)h->L * h->S * h->F;
  launch_running_update(result + h->pl.meta_size + 2, result + h->pl.meta_size + 2 + LSF, running_mean, running_var, h->decay_dev,
                        h->L, h->S, h->F, st);
  CK(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------
// communicator: one cudaMalloc'ed block per rank, mapped by the peers through CUDA IPC
// ---------------------------------------------------------------------------------------------
static long long comm_slot_stride(const maml_b200_handle* h) { return rup(maml_b200_result_size(h), 64); }

extern "C" int maml_b200_comm_init(maml_b200_handle* h, int32_t rank, int32_t world, void* ipc_handle_out) {
  if (!h || !ipc_handle_out) return fail("null argument");
  if (world < 2 || world > MAML_MAX_RANKS || rank < 0 || rank >= world) return fail("comm_init: need 2 <= world <= 8 and 0 <= rank < world");
  comm_release(h);
  const long long stride = comm_slot_stride(h);
  const long long data_bytes = 2 * stride * (long long)sizeof(float);
  h->comm_bytes = data_bytes + 256;                      // + flags[8] | seq | counters[2] | status (one 256 B line group)
  CK(cudaMalloc((void**)&h->comm_block, (size_t)h->comm_bytes));
  CK(cudaMemset(h->comm_block, 0, (size_t)h->comm_bytes));
  unsigned* ctl = (unsigned*)(h->comm_block + data_bytes);
  const unsigned one = 1u;
  CK(cudaMemcpy(ctl + MAML_MAX_RANKS, &one, sizeof(one), cudaMemcpyHostToDevice));       // seq starts at 1 (flags start at 0)
  CommDev& c = h->comm;
  c.rank = rank; c.world = world;
  c.local_data = (float*)h->comm_block; c.slot_stride = stride;
  c.local_flags = ctl; c.seq = ctl + MAML_MAX_RANKS; c.counters = ctl + MAML_MAX_RANKS + 1;
  c.status = (long long*)(ctl + MAML_MAX_RANKS + 4);
  cudaIpcMemHandle_t hd;
  CK(cudaIpcGetMemHandle(&hd, h->comm_block));
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "ipc handle size");
  memcpy(ipc_handle_out, &hd, sizeof(hd));
  CK(cudaDeviceSynchronize());
  return 0;
}

extern "C" int maml_b200_comm_connect(maml_b200_handle* h, const void* all_handles) {
  if (!h || !all_handles) return fail("null argument");
  if (!h->comm_block) return fail("comm_connect before comm_init");
  CommDev& c = h->comm;
  const long long data_bytes = 2 * c.slot_stride * (long long)sizeof(float);
  for (int p = 0; p < c.world; ++p) {
    char* base = nullptr;
    if (p == c.rank) base = h->comm_block;
    else {
      cudaIpcMemHandle_t hd;
      memcpy(&hd, (const char*)all_handles + (size_t)p * sizeof(hd), sizeof(hd));
      void* ptr = nullptr;
      cudaError_t e = cudaIpcOpenMemHandle(&ptr, hd, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess) { cudaGetLastError(); return fail(std::string("cudaIpcOpenMemHandle(rank ") + std::to_string(p) + "): " + cudaGetErrorString(e)); }
      h->comm_opened[p] = ptr;
      base = (char*)ptr;
    }
    c.peer_data[p] = (const float*)base;
    c.peer_flags[p] = (unsigned*)(base + data_bytes);
  }
  h->comm_connected = true;
  for (auto& g : h->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);    // graphs captured without the collective are stale
  h->graphs.clear();
  return 0;
}

extern "C" int maml_b200_comm_world(const maml_b200_handle* h) { return (h && h->comm_connected) ? h->comm.world : 1; }

// Stand-alone all-reduce(SUM) of a result-sized vector, in place (publish + reduce kernels on `stream`).  The iteration
// call does the same inside its own graph; this entry exists for timing the collective and for tests.
extern "C" int maml_b200_all_reduce(maml_b200_handle* h, float* vec, void* stream) {
  if (!h || !vec) return fail("null argument");
  if (!h->comm_connected) return fail("all_reduce: communicator not connected");
  if ((reinterpret_cast<uintptr_t>(vec) & 15u) != 0) return fail("all_reduce: vector must be 16-byte aligned");
  LaunchScope launch_scope(h);
  cudaStream_t st = (cudaStream_t)stream;
  launch_publish(h->comm, vec, maml_b200_result_size(h), st);
  launch_allreduce(h->comm, vec, maml_b200_result_size(h), st);
  CK(cudaGetLastError());
  return 0;
}

// 0 = healthy; otherwise the round in which a wait for a peer timed out (| 1 << 40 | peer << 32).  Synchronises.
extern "C" int64_t maml_b200_comm_status(maml_b200_handle* h) {
  if (!h || !h->comm_block) return 0;
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  long long v = 0;
  cudaMemcpy(&v, h->comm.status, sizeof(v), cudaMemcpyDeviceToHost);
  return (int64_t)v;
}

// GPU-resident episode assembly (no handle: it only needs the current device).  mean / stdv: host arrays of `channels`
// floats or null (no normalisation).  rot_k[b][n] in {0,1,2,3}: np.rot90 count of class n of task b (needs H == W when odd).
extern "C" int maml_b200_episode_gather(const float* dataset, const int64_t* image_index, const int32_t* rot_k, int32_t n_tasks,
                                       int32_t n_way, int32_t k_shot, int32_t t_target, int32_t channels, int32_t height,
                                       int32_t width, const float* mean_host, const float* std_host, float* x_support,
                                       float* x_target, int64_t* y_support, int64_t* y_target, void* stream) {
  if (!dataset || !image_index || !rot_k || !x_support || !x_target || !y_support || !y_target) return fail("null argument");
  if (n_tasks < 1 || n_way < 1 || k_shot < 1 || t_target < 1 || channels < 1 || channels > 4 || height < 1 || width < 1)
    return fail("episode_gather: bad shape");
  launch_episode_gather(dataset, (const long long*)image_index, rot_k, n_tasks, n_way, k_shot, t_target, channels, height, width,
                        mean_host, std_host, x_support, x_target, (long long*)y_support, (long long*)y_target, (cudaStream_t)stream);
  CK(cudaGetLastError());
  return 0;
}

extern "C" int maml_b200_profile(maml_b200_handle* h, int32_t enable) {
  if (!h) return fail("null argument");
  if (enable) h->prof.reset();
  h->profiling = enable != 0;
  return 0;
}

extern "C" int maml_b200_profile_read(maml_b200_handle* h, double* ms_by_cat, double* flops_by_cat, int64_t* launches_by_cat,
                                      int32_t ncat) {
  if (!h || !ms_by_cat || !flops_by_cat || !launches_by_cat) return fail("null argument");
  CK(cudaDeviceSynchronize());
  for (int c = 0; c < ncat; ++c) { ms_by_cat[c] = 0; flops_by_cat[c] = 0; launches_by_cat[c] = 0; }
  for (auto& r : h->prof.recs) {
    if (r.cat < 0 || r.cat >= ncat) continue;
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, r.a, r.b));
    ms_by_cat[r.cat] += ms; flops_by_cat[r.cat] += r.flops; launches_by_cat[r.cat] += 1;
  }
  h->prof.reset();
  return 0;
}

// device-side launch trace (common.cuh: trace_mark): start timestamps of every kernel of the following calls
static unsigned long long* g_trace_dev = nullptr;
static void trace_set_all(unsigned long long* p) {
  trace_set_conv(p); trace_set_bn(p); trace_set_head(p); trace_set_param(p); trace_set_tc(p);
}
extern "C" int maml_b200_trace(maml_b200_handle* h, int32_t enable) {
  if (!h) return fail("null argument");
  CK(cudaDeviceSynchronize());
  // kernels trace only when their launch tag carries MAML_TRACE_ARMED: cached graphs hold the old tags -> re-capture
  g_trace_flag = enable ? MAML_TRACE_ARMED : 0;
  for (auto& g : h->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
  h->graphs.clear();
  if (enable) {
    if (!g_trace_dev) CK(cudaMalloc(&g_trace_dev, (size_t)(MAML_TRACE_CAP + 2) * sizeof(unsigned long long)));
    CK(cudaMemset(g_trace_dev, 0, (size_t)(MAML_TRACE_CAP + 2) * sizeof(unsigned long long)));
    trace_set_all(g_trace_dev);
  } else {
    trace_set_all(nullptr);
  }
  CK(cudaDeviceSynchronize());
  return 0;
}
// out[i] = (globaltimer_ns << 20) | (launch tag << 8) | kernel id, in start order; returns the number of entries (<0: error); clears the trace
extern "C" int64_t maml_b200_trace_read(maml_b200_handle* h, uint64_t* out, int64_t capacity) {
  if (!h || !out || !g_trace_dev) { fail("trace is not enabled"); return -1; }
  if (cudaDeviceSynchronize() != cudaSuccess) { fail("device error"); return -1; }
  unsigned long long n = 0;
  cudaMemcpy(&n, g_trace_dev, sizeof(n), cudaMemcpyDeviceToHost);
  if (n > MAML_TRACE_CAP) n = MAML_TRACE_CAP;
  const long long k = std::min<long long>((long long)n, capacity);
  cudaMemcpy(out, g_trace_dev + 1, (size_t)k * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
  cudaMemset(g_trace_dev, 0, sizeof(unsigned long long));
  return (int64_t)k;
}

// ---------------------------------------------------------------------------------------------
// debug taps (tests): raw copy of one internal buffer
// ---------------------------------------------------------------------------------------------
extern "C" int64_t maml_b200_debug_read(maml_b200_handle* h, const char* name, int32_t task, int32_t step, int32_t layer,
                                        float* host_out, int64_t capacity) {
  if (!h || !name) { fail("null argument"); return -1; }
  if (task < 0 || task >= h->maxT) { fail("bad task"); return -1; }
  cudaDeviceSynchronize();
  const std::string nm(name);
  const float* src = nullptr; long long count = 0;
  const long long TP = (long long)h->maxT * h->Ppad;
  auto pass_buf = [&](const PassSet& ps, const std::string& what, int slot) -> bool {
    if (slot < 0 || slot >= ps.slots) return false;
    if (what == "ain") {
      if (layer < 1 || layer > h->L) return false;
      count = (layer == h->L) ? (long long)ps.n * h->D : (long long)ps.n * h->geo[layer].G * h->F;
      src = ps.ain[layer] + ((long long)task * ps.slots + slot) * ps.ain_sz[layer];
    } else if (what == "zh") {
      if (layer < 0 || layer >= h->L) return false;
      count = (long long)ps.n * h->geo[layer].G * h->F;
      src = ps.zh[layer] + ((long long)task * ps.slots + slot) * ps.zh_sz[layer];
    } else if (what == "dz") {
      if (layer < 0 || layer >= h->L) return false;
      count = (long long)ps.n * h->geo[layer].G * h->F;
      src = ps.dz[layer] + ((long long)task * ps.slots + slot) * ps.dz_sz[layer];
    } else if (what == "dp") {
      if (layer < 0 || layer >= h->L) return false;
      count = (long long)ps.n * h->geo[layer].pG * h->F;
      src = ps.dp[layer] + ((long long)task * ps.slots + slot) * ps.dp_sz[layer];
    } else return false;
    return true;
  };
  bool ok = false;
  if (nm.rfind("sup_", 0) == 0) ok = pass_buf(h->sup, nm.substr(4), step);
  else if (nm.rfind("tgt_", 0) == 0) ok = pass_buf(h->tgt, nm.substr(4), (h->cfg.reserved & 1) ? step : 0);
  else if (nm.rfind("tan_", 0) == 0) ok = pass_buf(h->tan, nm.substr(4), 0);
  else if (nm == "theta") { if (step >= 0 && step <= h->S) { src = h->theta + (long long)step * TP + (long long)task * h->Ppad; count = h->pl.P; ok = true; } }
  else if (nm == "g") { if (step >= 0 && step < h->S) { src = h->g + (long long)step * TP + (long long)task * h->Ppad; count = h->pl.P; ok = true; } }
  else if (nm == "tgrad") { if (step >= 0 && step < h->S) { src = h->tgrad + (long long)step * TP + (long long)task * h->Ppad; count = h->pl.P; ok = true; } }
  else if (nm == "tbar") { src = h->tbar + (long long)task * h->Ppad; count = h->pl.P; ok = true; }
  else if (nm == "u") { src = h->u + (long long)task * h->Ppad; count = h->pl.P; ok = true; }
  else if (nm == "tc_timeline") {
    static long long tl[16]; static float tf[16];
    cudaDeviceSynchronize();
    if (tc_read_timeline(tl)) { fail("timeline read failed"); return -1; }
    for (int i = 0; i < 16; ++i) tf[i] = (float)(tl[i] - tl[0]);
    const long long ncopy = std::min<long long>(16, capacity);
    if (host_out && ncopy > 0) memcpy(host_out, tf, ncopy * sizeof(float));
    return 16;
  }
  else if (nm == "losses") { src = h->losses + (long long)task * MAML_MAX_STEPS; count = MAML_MAX_STEPS; ok = true; }
  if (!ok) { fail("unknown debug tap / bad index: " + nm); return -1; }
  const long long ncopy = std::min<long long>(count, capacity);
  if (host_out && ncopy > 0) {
    cudaError_t e = cudaMemcpy(host_out, src, (size_t)ncopy * sizeof(float), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { fail(std::string("debug memcpy: ") + cudaGetErrorString(e)); return -1; }
  }
  return count;
}
