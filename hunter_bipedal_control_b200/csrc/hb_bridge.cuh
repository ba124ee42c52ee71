// The motor bridge's codec (hb_motor_bridge, hunter_b200.h): the joint path of legged_bridge_hw in both directions, one body for the
// kernels and the host entry points. Every float32 operation is rounded on its own: the build contracts a * b + c to an FMA by default,
// and the device, the host and a float32 restatement only agree bit for bit without it.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/hunter_b200.h"

namespace hb {

__host__ __device__ __forceinline__ float bridge_sub(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
__host__ __device__ __forceinline__ float bridge_mul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ float bridge_div(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
__host__ __device__ __forceinline__ float bridge_add(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}

// One value through the protocol on [lo, hi] with `bits` bits (motor_control.c's clamp, then math_ops.c's float_to_uint and uint_to_float):
// with quantise, x is rounded to float32, clamped, encoded with truncation and decoded; without, clamped in double. The clamp lets NaN
// through, as the driver's does; a NaN then encodes as code 0.
__host__ __device__ __forceinline__ double bridge_value(double x, double lo, double hi, int bits, bool quantise) {
  if (!quantise) return x > hi ? hi : (x < lo ? lo : x);
  const float flo = (float)lo, fhi = (float)hi, span = bridge_sub(fhi, flo), n = (float)((1 << bits) - 1);
  float f = (float)x;
  f = f > fhi ? fhi : (f < flo ? flo : f);
  const int code = f != f ? 0 : (int)bridge_div(bridge_mul(bridge_sub(f, flo), n), span);
  return (double)bridge_add(bridge_div(bridge_mul((float)code, span), n), flo);
}

// Joint j's hybrid command c = (posDes, velDes, kp, kd, ff) in the joint frame -> the decoded motor command m = (pos_m, vel_m, kp_m, kd_m,
// ff_m) in the motor frame (BridgeHW::write, then the protocol's 16 / 12 / 12 / 9 / 12 bits)
__host__ __device__ __forceinline__ void bridge_command(const hb_motor_bridge& b, int j, const double* c, double* m) {
  const double s = b.command_scale[j], d = (double)b.direction[j];
  const bool qz = b.quantise != 0;
  m[0] = bridge_value(d * c[0] + b.zero[j], -b.pos_max[j], b.pos_max[j], 16, qz);
  m[1] = bridge_value(d * c[1], -b.vel_max[j], b.vel_max[j], 12, qz);
  m[2] = bridge_value(s * c[2], 0.0, b.kp_max[j], 12, qz);
  m[3] = bridge_value(s * c[3], 0.0, b.kd_max[j], 9, qz);
  m[4] = bridge_value(s * c[4] * d, -b.ff_max[j], b.ff_max[j], 12, qz);
}

// Joint j's readings q, qd (joint frame) through its encoder: to the motor frame, the protocol's 16 / 12 bits, and back (BridgeHW::read:
// float32 with quantise, as the driver's values are)
__host__ __device__ __forceinline__ void bridge_feedback(const hb_motor_bridge& b, int j, double* q, double* qd) {
  const double d = (double)b.direction[j], z = b.zero[j];
  const bool qz = b.quantise != 0;
  const double p = bridge_value(d * *q + z, -b.pos_max[j], b.pos_max[j], 16, qz), v = bridge_value(d * *qd, -b.vel_max[j], b.vel_max[j], 12, qz);
  if (qz) {
    *q = (double)bridge_mul(bridge_sub((float)p, (float)z), (float)d);
    *qd = (double)bridge_mul((float)v, (float)d);
  } else {
    *q = (p - z) * d;
    *qd = v * d;
  }
}

}  // namespace hb
