// Common device definitions for libhunter_b200: model constants in __constant__ memory and warp-level helpers.
// One warp owns one problem instance; all cooperation is through shared memory + __syncwarp / shuffles.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/hunter_model_constants.h"

#define HB_FULL_MASK 0xffffffffu

namespace hb {

constexpr int NX = HB_NX, NU = HB_NU, NQ = HB_NQ, NJ = HB_NJ, NC = HB_NC, NBODY = HB_NBODY, NWBC = HB_NWBC;

// Model data (copied from include/hunter_model_constants.h at context creation).
struct Model {
  double joint_xyz[NBODY * 3];
  int joint_axis[NBODY];      // 0 none, +-1 x, +-2 y, +-3 z
  double mass[NBODY];
  double com[NBODY * 3];
  double inertia[NBODY * 9];
  double total_mass;
  double contact_offset[NC * 3];
  double joint_lower[NJ], joint_upper[NJ], joint_vel_limit[NJ];
  double Q[NX];
  double R[NU * NU];          // input cost (initializeInputCostWeight, LeggedInterface.cpp:263-288)
  double torque_limit[NJ];
};

__constant__ Model c_model;  // single translation unit (hb_api.cu)
// Per-lane constants of lq_kernel in GLOBAL memory (16 doubles per lane): a constant-memory operand indexed by the lane serialises into one
// fetch per distinct address (22 for Q[lane], 10 x 10 for the velocity block of R), a global load of the same table is one L1 hit.
// [0] Q[l]; [1] R[l][l] (l < 12); [2..11] R[l][12..21] (12 <= l < 22); [12], [13] bounds of the lane's limit penalty (l < 20).
constexpr int LQ_LANE_TAB = 16;
__device__ double g_lq_lane[32 * LQ_LANE_TAB];

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(HB_FULL_MASK, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(HB_FULL_MASK, v, o));
  return v;
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(HB_FULL_MASK, v, o));
  return v;
}

// MotionPhaseDefinition.h:55-87: contact order {l_toe, r_toe, l_heel, r_heel}
__device__ __forceinline__ bool contact_flag(int mode, int c) {
  return (c & 1) ? (mode == 1 || mode == 3) : (mode == 2 || mode == 3);
}

// A per-robot setting as the kernels read it, passed by value: instances 0 .. n - 1 have a record. Default-constructed, it is unset.
template <class T> struct InstanceView {
  const T* recs;
  int n;
  // the record of instance i; null when the view is unset or i is beyond it
  __host__ __device__ __forceinline__ const T* of(int i) const { return (recs && i < n) ? recs + i : nullptr; }
};

}  // namespace hb
