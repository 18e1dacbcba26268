// Declarations shared by the wgmma conv and weight-gradient kernels (kernels_tc.cu) and the engine.
#pragma once
#include <cuda.h>
#include "common.cuh"

struct alignas(64) TcMaps { CUtensorMap m[4]; };   // A_hi, A_lo, B_hi, B_lo

struct TcConvArgs {
  int kc, rows, gw, G, h, w, ncols, mode, tasks;
  int plan_tasks;        // split-K is planned for this many tasks (the handle's max_tasks) so that a task's arithmetic
                         // does not depend on how many tasks share the call
  int halo, rpad, nb, timeline;   // halo = gw + 1 rows; rpad = halo-tile rows (multiple of 8); nb = B ring depth
  int a_row_base;        // row (in the A tensor map) of grid row 0 of task 0 for this pass slot (includes the guard)
  int a_task_rows;       // rows per task in the A tensor map
  int sign;              // +1 conv, -1 dgrad
  int b_row_base;        // row (in the B tensor map) of (task 0, tap 0, n 0)
  int b_task_rows;       // rows per task in the B tensor map
  const float* bias; long long bias_stride;
  float* out; long long out_stride;
  const float* zh; long long zh_stride;
  double* stats; long long stats_stride;
  double alg_flops;
  int tag;          // launch sequence number inside the iteration (device trace)
};

int tc_conv_rpad(int gw);
int tc_conv_ring(int ncols, int gw, size_t extra = 0);
size_t tc_conv_extra_bytes(int ncols, int S, bool tangent);
int tc_conv_prepare();     // shared-memory opt-in of the wgmma conv and weight-gradient kernels
int tc_read_timeline(long long* out16);
void launch_conv_tc(const TcMaps& maps, const TcConvArgs& a, cudaStream_t st);
void launch_pack_weights(const ParamLayout& pl, const float* theta, long long theta_task_stride, float* pack,
                         long long pack_task_stride, long long plane_stride, int tasks, cudaStream_t st);
void launch_wgrad_tc(const WgradArgs& a, cudaStream_t st);   // wgmma weight gradient of blocks l >= 1 (needs a_plane / d_plane)
