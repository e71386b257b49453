// Shared helpers for the deeptables_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include "../../include/deeptables_b200.h"

namespace dtb {

// ---- error plumbing (no exceptions across the C ABI) -------------------------------------
void set_error(const char* fmt, ...);
int sm_count();
void count_launch();

#define DTB_CHECK_ARG(cond, msg)                                   \
  do {                                                             \
    if (!(cond)) {                                                 \
      dtb::set_error("%s: invalid argument: %s", __func__, msg);   \
      return DTB_ERR_INVALID_ARG;                                  \
    }                                                              \
  } while (0)

#define DTB_CUDA_OK(expr)                                                               \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      dtb::set_error("%s: CUDA error %d (%s) at %s:%d", __func__, (int)_e,              \
                     cudaGetErrorString(_e), __FILE__, __LINE__);                       \
      return DTB_ERR_CUDA;                                                              \
    }                                                                                   \
  } while (0)

// every hand-written kernel launch is followed by this: error check + launch counter
#define DTB_LAUNCH_OK()                  \
  do {                                   \
    dtb::count_launch();                 \
    DTB_CUDA_OK(cudaGetLastError());     \
  } while (0)

static inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// ---- device helpers ----------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The class DeepTable.predict gives a row of the model output: numpy's argmax of what predict_proba returns.  On one
// column that is [1-p, p] (1 - p in float32), so class 1 when p > 1 - p; on several, the first maximum.
__device__ __forceinline__ int predicted_class(const float* __restrict__ prob, int64_t r, int cols) {
  if (cols == 1) {
    const float p = prob[r];
    return p > __fsub_rn(1.f, p) ? 1 : 0;
  }
  const float* pr = prob + r * cols;
  int arg = 0;
  float best = pr[0];
  for (int c = 1; c < cols; ++c)
    if (pr[c] > best) { best = pr[c]; arg = c; }
  return arg;
}

// Streaming 16-byte load that does not pollute L1 (embedding rows are touched once per kernel).
__device__ __forceinline__ float4 ldg_stream_f4(const float* p) {
  float4 r;
  // L2::64B: an embedding row is 64 bytes at a random address -- do not let L2 pull the neighbouring
  // 64 bytes of the 128-byte line from HBM (measured: 1.83x read amplification without the hint)
  asm volatile("ld.global.nc.L1::no_allocate.L2::64B.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}

// Vector reduction into global memory: one 16-byte RED instead of four 4-byte atomics (sm_90+).
__device__ __forceinline__ void red_add_f4(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}

// Counter-based dropout masks (dense_bn_loss.cu, pnn_attention.cu): element i of a call with seed s is kept when
// mix32(dropout_key(s) + i) >= threshold, threshold = rate * 2^32; forward and backward regenerate the same bits and
// nothing is stored.  The seed is a kernel argument, or is read from device memory when seed_dev is set (a train step
// captured in a CUDA graph must not bake the host's seed into its kernel arguments).
__device__ __forceinline__ uint32_t mix32(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdULL;
  x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL;
  x ^= x >> 33;
  return (uint32_t)x;
}
__device__ __forceinline__ uint64_t dropout_key(uint64_t seed, const unsigned long long* __restrict__ seed_dev) {
  return (seed_dev ? (uint64_t)*seed_dev : seed) * 0x9E3779B97F4A7C15ULL;
}
static inline uint32_t dropout_threshold(float rate) { return (uint32_t)((double)rate * 4294967296.0); }

// Row base (in floats) of categorical id `id` of field f, or -1 when out of range.
__device__ __forceinline__ int64_t table_row(const int64_t* __restrict__ row_offsets, int f, int id,
                                             int D, int* status) {
  const int64_t lo = row_offsets[f], hi = row_offsets[f + 1];
  if (id < 0 || (int64_t)id >= hi - lo) {
    if (status) atomicOr(status, 1 << (f & 31));
    return -1;
  }
  return (lo + id) * (int64_t)D;
}

// keras.optimizers.Adam.update_step on one element, with every rounding pinned by intrinsics so
// that the dense kernel and the exact-lazy row kernels (adam_rows.cu) produce identical bits:
//   m += (g-m)(1-b1) ; v += (g*g-v)(1-b2) ; p -= m*alpha/(sqrt(v)+eps)
__device__ __forceinline__ void adam_update(float& p, float& m, float& v, float g, float alpha, float omb1,
                                            float omb2, float eps) {
  m = __fmaf_rn(__fsub_rn(g, m), omb1, m);
  v = __fmaf_rn(__fsub_rn(__fmul_rn(g, g), v), omb2, v);
  p = __fsub_rn(p, __fdiv_rn(__fmul_rn(m, alpha), __fadd_rn(__fsqrt_rn(v), eps)));
}

// keras.optimizers.SGD.update_step, Keras's operation order, every rounding pinned (optim.cu):
//   momentum = 0 : p -= g*lr
//   otherwise    : m = m*mu - g*lr ; p += m   (nesterov: p += m*mu - g*lr)
__device__ __forceinline__ void sgd_update(float& p, float& m, float g, float lr, float mu, bool nesterov) {
  const float glr = __fmul_rn(g, lr);
  if (mu == 0.f) {
    p = __fsub_rn(p, glr);
    return;
  }
  m = __fsub_rn(__fmul_rn(m, mu), glr);
  p = __fadd_rn(p, nesterov ? __fsub_rn(__fmul_rn(m, mu), glr) : m);
}

// keras.optimizers.RMSprop.update_step: v = rho*v + (1-rho)*g^2 ; centered: a = rho*a + (1-rho)*g, den = v - a^2 + eps,
// else den = v + eps ; inc = lr*g / sqrt(den) ; momentum > 0: mom = mu*mom + inc, p -= mom ; else p -= inc
__device__ __forceinline__ void rmsprop_update(float& p, float& v, float& a, float& mom, float g, float lr, float rho,
                                               float omr, float mu, float eps, bool centered) {
  v = __fadd_rn(__fmul_rn(rho, v), __fmul_rn(omr, __fmul_rn(g, g)));
  float den;
  if (centered) {
    a = __fadd_rn(__fmul_rn(rho, a), __fmul_rn(omr, g));
    den = __fadd_rn(__fsub_rn(v, __fmul_rn(a, a)), eps);
  } else {
    den = __fadd_rn(v, eps);
  }
  const float inc = __fdiv_rn(__fmul_rn(lr, g), __fsqrt_rn(den));
  if (mu > 0.f) {
    mom = __fadd_rn(__fmul_rn(mu, mom), inc);
    p = __fsub_rn(p, mom);
  } else {
    p = __fsub_rn(p, inc);
  }
}

// keras.optimizers.Adagrad.update_step: acc += g^2 ; p -= lr*g / sqrt(acc + eps)
__device__ __forceinline__ void adagrad_update(float& p, float& acc, float g, float lr, float eps) {
  acc = __fadd_rn(acc, __fmul_rn(g, g));
  p = __fsub_rn(p, __fdiv_rn(__fmul_rn(lr, g), __fsqrt_rn(__fadd_rn(acc, eps))));
}

}  // namespace dtb
