// Exact-lazy row-wise Adam for the embedding tables.
//
// Keras Adam is dense (deepmodel.py:321-322): every step decays m and v of EVERY table row and
// moves every row whose m is non-zero -- 7 x 1.66 GB of HBM traffic per step at the Criteo shape.
// The arithmetic of a zero-gradient step depends only on the row's own (p, m, v) and the step
// number, so it can be deferred: last_step[row] records the last optimiser step applied to the row
// and the skipped zero-gradient steps are replayed, in order and with the same fp32 operations
// (dtb::adam_update with g = 0), the next time the row is read.  The result is bit-identical to the
// dense kernel (tests/test_native_gpu.py::test_lazy_adam_matches_dense) at ~1/15 of the traffic.
//
// Ownership of a row within one launch is claimed with atomicMax on last_step, so duplicate ids in
// a batch (and the union of several ranks' ids) update the row exactly once.
#include "dtb_common.cuh"

namespace dtb {

__device__ __forceinline__ void replay_zero_grad(float4& p, float4& m, float4& v,
                                                 const float* __restrict__ alpha_table, int from, int upto,
                                                 float omb1, float omb2, float eps) {
  if (m.x == 0.f && m.y == 0.f && m.z == 0.f && m.w == 0.f && v.x == 0.f && v.y == 0.f && v.z == 0.f &&
      v.w == 0.f)
    return;   // never-touched row: zero-gradient steps are the identity
  int s = from;
  for (; s <= upto; ++s) {
    const float4 m0 = m;
    const float a = __ldg(alpha_table + s);
    adam_update(p.x, m.x, v.x, 0.f, a, omb1, omb2, eps);
    adam_update(p.y, m.y, v.y, 0.f, a, omb1, omb2, eps);
    adam_update(p.z, m.z, v.z, 0.f, a, omb1, omb2, eps);
    adam_update(p.w, m.w, v.w, 0.f, a, omb1, omb2, eps);
    // Long gaps (rare ids of a long-tailed column).  After ~1000 zero-gradient steps m reaches the fixed point of its
    // decay (zero or the smallest denormals, |m| < 1e-44, so |m| <= 7 * 2^-149), and m stays there: its update with
    // g = 0 reads m and omb1 alone.  Every later step then moves p by u = fl(fl(m * a) / d) with d = fl(sqrt(v)) + eps
    // >= eps, and correctly rounded products and quotients are monotone, so |u| <= U = fl(fl(7 * 2^-149 * A) / eps)
    // for every step whose alpha a is at most A.  |p| > 1e-25 puts p at or above the binade [2^-84, 2^-83), whose
    // spacing is 2^-107: U < 2^-108 makes p - u round back to p.  p and m no longer change and only the decay of v is
    // left.  The exit is valid as long as that holds for A = the largest alpha of the steps still to replay; the caller
    // keeps the rows of a table whose alpha table breaks it on the dense sweep instead (DeepModel._select_table_optimizer).
    // With a constant rate and Keras's defaults, 7 * 2^-149 * alpha rounds to 0, far inside the bound; a schedule that
    // warms up, or a rate raised between epochs, can raise A, hence the check on the whole table.
    if (m.x == m0.x && m.y == m0.y && m.z == m0.z && m.w == m0.w && fabsf(m.x) < 1e-44f && fabsf(m.y) < 1e-44f &&
        fabsf(m.z) < 1e-44f && fabsf(m.w) < 1e-44f && fabsf(p.x) > 1e-25f && fabsf(p.y) > 1e-25f &&
        fabsf(p.z) > 1e-25f && fabsf(p.w) > 1e-25f) {
      ++s;
      break;
    }
  }
  // v-only tail: one fma per element per step (adam_update's v line with g = 0), until v reaches its own fixed point
  // (~90 000 steps): same bits as the dense kernel, bounded work per row.
  for (; s <= upto; ++s) {
    const float4 v0 = v;
    v.x = __fmaf_rn(__fsub_rn(0.f, v.x), omb2, v.x);
    v.y = __fmaf_rn(__fsub_rn(0.f, v.y), omb2, v.y);
    v.z = __fmaf_rn(__fsub_rn(0.f, v.z), omb2, v.z);
    v.w = __fmaf_rn(__fsub_rn(0.f, v.w), omb2, v.w);
    if (v.x == v0.x && v.y == v0.y && v.z == v0.z && v.w == v0.w) break;
  }
}

// MODE 0: catch-up to `step` (zero-gradient replay only)
// MODE 1: apply step `step` with the accumulated gradient row, zero the gradient row
template <int MODE>
__global__ void adam_rows_kernel(const int32_t* __restrict__ idx, const int64_t* __restrict__ row_offsets,
                                 float* __restrict__ table, float* __restrict__ m, float* __restrict__ v,
                                 float* __restrict__ grad, int32_t* __restrict__ last_step,
                                 const float* __restrict__ alpha_table, int step, float omb1, float omb2,
                                 float eps, int B, int F, int D, const int32_t* __restrict__ step_dev) {
  // CUDA-graph form: the step comes from device memory (`step` is then the offset: 0 = catch up to the steps done so
  // far, 1 = apply the next one)
  if (step_dev) step += *step_dev;
  if (step <= 0) return;
  const int Q = D >> 2;                      // lanes per row (power of two <= 32, checked by the host)
  const int64_t total = (int64_t)B * F * Q;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int lane = threadIdx.x & 31;
  // loop bound rounded up so that whole warps stay converged for the shuffles
  const int64_t total_pad = (total + 31) / 32 * 32;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total_pad; i += stride) {
    const bool live = i < total;
    const int64_t ref = live ? i / Q : 0;
    const int q = (int)(i - ref * Q);
    const int b = (int)(ref / F), f = (int)(ref - (int64_t)b * F);
    int64_t row = -1;
    if (live) {
      const int id = __ldg(idx + (int64_t)b * F + f);
      const int64_t lo = row_offsets[f];
      if (id >= 0 && id < row_offsets[f + 1] - lo) row = lo + id;
    }
    int old = 0x7fffffff;
    if (row >= 0 && q == 0) old = atomicMax(last_step + row, step);
    old = __shfl_sync(0xffffffffu, old, lane - q);   // leader of this row's lane group
    if (row < 0 || old >= step) continue;
    const int64_t off = row * D + (q << 2);
    float4 p4 = *reinterpret_cast<float4*>(table + off);
    float4 m4 = *reinterpret_cast<float4*>(m + off);
    float4 v4 = *reinterpret_cast<float4*>(v + off);
    if (MODE == 0) {
      replay_zero_grad(p4, m4, v4, alpha_table, old + 1, step, omb1, omb2, eps);
    } else {
      // rows_apply presumes the catch-up to step-1 already ran; replay defensively if it did not
      replay_zero_grad(p4, m4, v4, alpha_table, old + 1, step - 1, omb1, omb2, eps);
      const float4 g4 = *reinterpret_cast<float4*>(grad + off);
      const float a = __ldg(alpha_table + step);
      adam_update(p4.x, m4.x, v4.x, g4.x, a, omb1, omb2, eps);
      adam_update(p4.y, m4.y, v4.y, g4.y, a, omb1, omb2, eps);
      adam_update(p4.z, m4.z, v4.z, g4.z, a, omb1, omb2, eps);
      adam_update(p4.w, m4.w, v4.w, g4.w, a, omb1, omb2, eps);
      *reinterpret_cast<float4*>(grad + off) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    *reinterpret_cast<float4*>(table + off) = p4;
    *reinterpret_cast<float4*>(m + off) = m4;
    *reinterpret_cast<float4*>(v + off) = v4;
  }
}

__global__ void adam_rows_flush_kernel(float* __restrict__ table, float* __restrict__ m,
                                       float* __restrict__ v, int32_t* __restrict__ last_step,
                                       const float* __restrict__ alpha_table, int upto, float omb1,
                                       float omb2, float eps, int64_t n_rows, int D) {
  const int Q = D >> 2;
  const int64_t total = n_rows * Q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / Q;
    const int q = (int)(i - row * Q);
    const int old = last_step[row];
    if (old >= upto) continue;
    const int64_t off = row * D + (q << 2);
    float4 p4 = *reinterpret_cast<float4*>(table + off);
    float4 m4 = *reinterpret_cast<float4*>(m + off);
    float4 v4 = *reinterpret_cast<float4*>(v + off);
    replay_zero_grad(p4, m4, v4, alpha_table, old + 1, upto, omb1, omb2, eps);
    *reinterpret_cast<float4*>(table + off) = p4;
    *reinterpret_cast<float4*>(m + off) = m4;
    *reinterpret_cast<float4*>(v + off) = v4;
  }
}

__global__ void set_last_step_kernel(int32_t* __restrict__ last_step, int64_t n_rows, int upto) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_rows;
       i += (int64_t)gridDim.x * blockDim.x)
    if (last_step[i] < upto) last_step[i] = upto;
}

static bool rows_shape_ok(int D) {
  const int Q = D / 4;
  return D % 4 == 0 && Q >= 1 && Q <= 32 && (Q & (Q - 1)) == 0;
}

static int rows_grid(int64_t total) {
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = (int64_t)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  return (int)(blocks < 1 ? 1 : blocks);
}

}  // namespace dtb

using namespace dtb;

extern "C" {

int dtb_adam_rows_catchup(const int32_t* idx, const int64_t* row_offsets, float* table, float* m, float* v,
                          int32_t* last_step, const float* alpha_table, int upto, double beta1, double beta2,
                          float eps, int B, int F, int D, void* stream) {
  DTB_CHECK_ARG(idx && row_offsets && table && m && v && last_step && alpha_table, "NULL argument");
  DTB_CHECK_ARG(rows_shape_ok(D), "embedding dim must be 4*2^k (<=128) for the row-wise Adam");
  if (B <= 0 || F <= 0 || upto <= 0) return DTB_OK;
  const int64_t total = (int64_t)B * F * (D / 4);
  adam_rows_kernel<0><<<rows_grid(total), 256, 0, (cudaStream_t)stream>>>(
      idx, row_offsets, table, m, v, nullptr, last_step, alpha_table, upto, (float)(1.0 - beta1), (float)(1.0 - beta2), eps, B,
      F, D, nullptr);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

// The same two kernels with the step counter in DEVICE memory (*step_dev = optimiser steps completed so far): catch-up
// to *step_dev, apply step *step_dev + 1.  For train steps captured in a CUDA graph.
int dtb_adam_rows_catchup_dev(const int32_t* idx, const int64_t* row_offsets, float* table, float* m, float* v,
                              int32_t* last_step, const float* alpha_table, const int32_t* step_dev, double beta1,
                              double beta2, float eps, int B, int F, int D, void* stream) {
  DTB_CHECK_ARG(idx && row_offsets && table && m && v && last_step && alpha_table && step_dev, "NULL argument");
  DTB_CHECK_ARG(rows_shape_ok(D), "embedding dim must be 4*2^k (<=128) for the row-wise Adam");
  if (B <= 0 || F <= 0) return DTB_OK;
  const int64_t total = (int64_t)B * F * (D / 4);
  adam_rows_kernel<0><<<rows_grid(total), 256, 0, (cudaStream_t)stream>>>(
      idx, row_offsets, table, m, v, nullptr, last_step, alpha_table, 0, (float)(1.0 - beta1), (float)(1.0 - beta2), eps, B, F,
      D, step_dev);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_adam_rows_apply_dev(const int32_t* idx, const int64_t* row_offsets, float* table, float* m, float* v,
                            float* grad_table, int32_t* last_step, const float* alpha_table, const int32_t* step_dev,
                            double beta1, double beta2, float eps, int B, int F, int D, void* stream) {
  DTB_CHECK_ARG(idx && row_offsets && table && m && v && grad_table && last_step && alpha_table && step_dev,
                "NULL argument");
  DTB_CHECK_ARG(rows_shape_ok(D), "embedding dim must be 4*2^k (<=128) for the row-wise Adam");
  if (B <= 0 || F <= 0) return DTB_OK;
  const int64_t total = (int64_t)B * F * (D / 4);
  adam_rows_kernel<1><<<rows_grid(total), 256, 0, (cudaStream_t)stream>>>(
      idx, row_offsets, table, m, v, grad_table, last_step, alpha_table, 1, (float)(1.0 - beta1), (float)(1.0 - beta2), eps, B,
      F, D, step_dev);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

__global__ void step_increment_kernel(int32_t* step_dev) { *step_dev += 1; }

int dtb_step_increment(int32_t* step_dev, void* stream) {
  DTB_CHECK_ARG(step_dev, "NULL argument");
  step_increment_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(step_dev);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_adam_rows_apply(const int32_t* idx, const int64_t* row_offsets, float* table, float* m, float* v,
                        float* grad_table, int32_t* last_step, const float* alpha_table, int step,
                        double beta1, double beta2, float eps, int B, int F, int D, void* stream) {
  DTB_CHECK_ARG(idx && row_offsets && table && m && v && grad_table && last_step && alpha_table,
                "NULL argument");
  DTB_CHECK_ARG(rows_shape_ok(D), "embedding dim must be 4*2^k (<=128) for the row-wise Adam");
  DTB_CHECK_ARG(step >= 1, "step is 1-based");
  if (B <= 0 || F <= 0) return DTB_OK;
  const int64_t total = (int64_t)B * F * (D / 4);
  adam_rows_kernel<1><<<rows_grid(total), 256, 0, (cudaStream_t)stream>>>(
      idx, row_offsets, table, m, v, grad_table, last_step, alpha_table, step, (float)(1.0 - beta1), (float)(1.0 - beta2), eps,
      B, F, D, nullptr);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_adam_rows_flush(float* table, float* m, float* v, int32_t* last_step, const float* alpha_table,
                        int upto, double beta1, double beta2, float eps, int64_t n_rows, int D, void* stream) {
  DTB_CHECK_ARG(table && m && v && last_step && alpha_table, "NULL argument");
  DTB_CHECK_ARG(rows_shape_ok(D), "embedding dim must be 4*2^k (<=128) for the row-wise Adam");
  if (n_rows <= 0 || upto <= 0) return DTB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  adam_rows_flush_kernel<<<rows_grid(n_rows * (D / 4)), 256, 0, st>>>(
      table, m, v, last_step, alpha_table, upto, (float)(1.0 - beta1), (float)(1.0 - beta2), eps, n_rows, D);
  DTB_LAUNCH_OK();
  set_last_step_kernel<<<rows_grid(n_rows), 256, 0, st>>>(last_step, n_rows, upto);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------
// Data-parallel exchange of the embedding gradient without moving the dense [sum V, D] buffer:
//   pack   : every (b,f) reference claims its row once per step (atomicMax on claim[row]); the owner
//            MOVES the accumulated gradient row into packed[b,f,:] (and zeroes the table row), every
//            other reference of the same row writes zeros.  packed is what the ranks all-gather.
//   unpack : add one rank's packed rows into the local gradient table.  Within one launch at most one
//            reference per row carries data, so plain read-modify-write is race-free, and calling it
//            for rank 0,1,..,W-1 in order gives the same bits on every replica.
// ------------------------------------------------------------------------------------------
namespace dtb {

__global__ void grad_rows_pack_kernel(const int32_t* __restrict__ idx, const int64_t* __restrict__ row_offsets,
                                      float* __restrict__ grad, int32_t* __restrict__ claim, float* __restrict__ packed,
                                      int step, int B, int F, int D) {
  const int Q = D >> 2;
  const int64_t total = (int64_t)B * F * Q;
  const int64_t total_pad = (total + 31) / 32 * 32;
  const int lane = threadIdx.x & 31;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total_pad;
       i += (int64_t)gridDim.x * blockDim.x) {
    const bool live = i < total;
    const int64_t ref = live ? i / Q : 0;
    const int q = (int)(i - ref * Q);
    const int b = (int)(ref / F), f = (int)(ref - (int64_t)b * F);
    int64_t row = -1;
    if (live) {
      const int id = __ldg(idx + (int64_t)b * F + f);
      const int64_t lo = row_offsets[f];
      if (id >= 0 && id < row_offsets[f + 1] - lo) row = lo + id;
    }
    int old = 0x7fffffff;
    if (row >= 0 && q == 0) old = atomicMax(claim + row, step);
    old = __shfl_sync(0xffffffffu, old, lane - q);
    if (!live) continue;
    const bool mine = row >= 0 && old < step;
    float4* src = reinterpret_cast<float4*>(grad + (mine ? row : 0) * D + (q << 2));
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (mine) v = *src;
    *reinterpret_cast<float4*>(packed + ref * D + (q << 2)) = v;
    // Zero the row only AFTER the store above, which cannot issue before the load has returned.  A zero
    // store issued right behind the load hits the line while its miss is still pending and the LSU
    // replays it: measured 1.1 ms instead of 0.2 ms for this kernel (tools/pack_probe.cu, V2 vs V6).
    asm volatile("" ::: "memory");
    if (mine) *src = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

__global__ void grad_rows_unpack_kernel(const int32_t* __restrict__ idx, const int64_t* __restrict__ row_offsets,
                                        const float* __restrict__ packed, float* __restrict__ grad, int B, int F,
                                        int D) {
  const int Q = D >> 2;
  const int64_t total = (int64_t)B * F * Q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t ref = i / Q;
    const int q = (int)(i - ref * Q);
    const int b = (int)(ref / F), f = (int)(ref - (int64_t)b * F);
    const float4 v = *reinterpret_cast<const float4*>(packed + ref * D + (q << 2));
    if (v.x == 0.f && v.y == 0.f && v.z == 0.f && v.w == 0.f) continue;   // non-owner reference (or a zero gradient)
    const int id = __ldg(idx + (int64_t)b * F + f);
    const int64_t lo = row_offsets[f];
    if (id < 0 || id >= row_offsets[f + 1] - lo) continue;
    float4* dst = reinterpret_cast<float4*>(grad + (lo + id) * D + (q << 2));
    float4 g = *dst;
    g.x += v.x; g.y += v.y; g.z += v.z; g.w += v.w;
    *dst = g;
  }
}

}  // namespace dtb

extern "C" {

int dtb_grad_rows_pack(const int32_t* idx, const int64_t* row_offsets, float* grad_table, int32_t* claim,
                       float* packed, int step, int B, int F, int D, void* stream) {
  DTB_CHECK_ARG(idx && row_offsets && grad_table && claim && packed, "NULL argument");
  DTB_CHECK_ARG(rows_shape_ok(D), "embedding dim must be 4*2^k (<=128)");
  DTB_CHECK_ARG(step >= 1, "step is 1-based");
  if (B <= 0 || F <= 0) return DTB_OK;
  const int64_t total = (int64_t)B * F * (D / 4);
  grad_rows_pack_kernel<<<rows_grid(total), 256, 0, (cudaStream_t)stream>>>(idx, row_offsets, grad_table, claim, packed,
                                                                             step, B, F, D);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_grad_rows_unpack(const int32_t* idx, const int64_t* row_offsets, const float* packed, float* grad_table, int B,
                         int F, int D, void* stream) {
  DTB_CHECK_ARG(idx && row_offsets && grad_table && packed, "NULL argument");
  DTB_CHECK_ARG(rows_shape_ok(D), "embedding dim must be 4*2^k (<=128)");
  if (B <= 0 || F <= 0) return DTB_OK;
  const int64_t total = (int64_t)B * F * (D / 4);
  grad_rows_unpack_kernel<<<rows_grid(total), 256, 0, (cudaStream_t)stream>>>(idx, row_offsets, packed, grad_table, B, F,
                                                                               D);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

}  // extern "C"
