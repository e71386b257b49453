// keras.optimizers.SGD, RMSprop and Adagrad with Keras's dense semantics, on the dense parameters and on the
// embedding tables.
//
// Dense sweep: one pass over p, g and the optimiser's state slots (float4 accesses when every pointer is 16-byte
// aligned, scalar tail), zeroing g behind it -- the counterpart of adam_dense_impl (dense_bn_loss.cu).
//
// Row form: the exact-lazy scheme of adam_rows.cu.  A table row whose gradient is zero still takes Keras's step with
// g = 0.  Those steps are deferred: last_step[row] is the last step applied to the row, and the skipped steps are
// replayed, in order and with the same device function (dtb_common.cuh), the next time the row is read or before the
// table is exported.  The result is therefore bit-identical to the dense sweep by construction.
//   * SGD without momentum and Adagrad: a zero-gradient step is the identity (p - 0*lr, acc + 0), nothing to replay.
//   * SGD with momentum and RMSprop: a zero-gradient step decays the state and moves p by it.  The learning rate and
//     every other hyperparameter are constants, so the step function does not depend on the step number: once one
//     replayed step leaves p and every state word unchanged, all later ones do too and the replay stops there.  It
//     does NOT stop when the state reaches zero: the smallest denormals are fixed points of x*0.9 and a parameter at
//     or near 0 keeps moving by them; then the whole gap is replayed.
// Ownership of a row within one launch is claimed with atomicMax on last_step, so duplicate ids in a batch (and the
// union of several ranks' ids) update the row exactly once.
#include "dtb_common.cuh"

namespace dtb {

// The hyperparameters as the kernels use them, passed by value (a captured graph keeps them).
struct OptimHP {
  int kind;
  bool flag;        // SGD: nesterov; RMSprop: centered
  bool replay;      // zero-gradient steps change the state (SGD with momentum, RMSprop)
  float lr, mu, rho, omr, eps;
};

static bool zero_step_is_identity(const dtb_optim_params& h) {
  return h.kind == DTB_OPTIM_ADAGRAD || (h.kind == DTB_OPTIM_SGD && h.momentum == 0.f);
}

static OptimHP to_hp(const dtb_optim_params& h) {
  OptimHP o;
  o.kind = h.kind;
  o.flag = h.flag != 0;
  o.replay = !zero_step_is_identity(h);
  o.lr = h.lr;
  o.mu = h.momentum;
  o.rho = (float)h.rho;
  o.omr = (float)(1.0 - h.rho);     // keras multiplies by the python double (1 - rho) rounded to fp32
  o.eps = h.eps;
  return o;
}

// NULL when the slots match what the optimiser needs, else the complaint
static const char* check_hp(const dtb_optim_params* h, const float* s0, const float* s1, const float* s2) {
  if (!h) return "NULL hyperparameters";
  switch (h->kind) {
    case DTB_OPTIM_SGD:
      if (h->momentum < 0.f || h->momentum > 1.f) return "SGD momentum must be in [0, 1]";
      if (h->momentum > 0.f && !s0) return "SGD with momentum needs slot s0";
      return nullptr;
    case DTB_OPTIM_RMSPROP:
      if (!s0) return "RMSprop needs slot s0 (velocity)";
      if (h->flag && !s1) return "centered RMSprop needs slot s1 (average gradient)";
      if (h->momentum > 0.f && !s2) return "RMSprop with momentum needs slot s2";
      return nullptr;
    case DTB_OPTIM_ADAGRAD:
      return s0 ? nullptr : "Adagrad needs slot s0 (accumulator)";
    default:
      return "unknown optimiser kind";
  }
}

#define DTB_CHECK_HP(h, s0, s1, s2)               \
  do {                                            \
    const char* _msg = check_hp(h, s0, s1, s2);   \
    DTB_CHECK_ARG(_msg == nullptr, _msg);         \
  } while (0)

__device__ __forceinline__ void optim_update(const OptimHP& h, float& p, float& s0, float& s1, float& s2, float g) {
  if (h.kind == DTB_OPTIM_SGD)
    sgd_update(p, s0, g, h.lr, h.mu, h.flag);
  else if (h.kind == DTB_OPTIM_RMSPROP)
    rmsprop_update(p, s0, s1, s2, g, h.lr, h.rho, h.omr, h.mu, h.eps, h.flag);
  else
    adagrad_update(p, s0, g, h.lr, h.eps);
}

__device__ __forceinline__ void optim_update4(const OptimHP& h, float4& p, float4& s0, float4& s1, float4& s2,
                                              float4 g) {
  optim_update(h, p.x, s0.x, s1.x, s2.x, g.x);
  optim_update(h, p.y, s0.y, s1.y, s2.y, g.y);
  optim_update(h, p.z, s0.z, s1.z, s2.z, g.z);
  optim_update(h, p.w, s0.w, s1.w, s2.w, g.w);
}

__device__ __forceinline__ float4 load4_or_zero(const float* s, int64_t off) {
  return s ? *reinterpret_cast<const float4*>(s + off) : make_float4(0.f, 0.f, 0.f, 0.f);
}

__device__ __forceinline__ void store4_if(float* s, int64_t off, float4 v) {
  if (s) *reinterpret_cast<float4*>(s + off) = v;
}

__device__ __forceinline__ bool same_bits(float4 a, float4 b) {
  return __float_as_uint(a.x) == __float_as_uint(b.x) && __float_as_uint(a.y) == __float_as_uint(b.y) &&
         __float_as_uint(a.z) == __float_as_uint(b.z) && __float_as_uint(a.w) == __float_as_uint(b.w);
}

// zero-gradient steps from .. upto, stopping at the first one that changes nothing (see the file comment)
__device__ __forceinline__ void optim_replay(const OptimHP& h, float4& p, float4& s0, float4& s1, float4& s2,
                                             int from, int upto) {
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int s = from; s <= upto; ++s) {
    const float4 p0 = p, a0 = s0, b0 = s1, c0 = s2;
    optim_update4(h, p, s0, s1, s2, zero);
    if (same_bits(p, p0) && same_bits(s0, a0) && same_bits(s1, b0) && same_bits(s2, c0)) break;
  }
}

// ---- dense sweep ---------------------------------------------------------------------------------------------------
__global__ void optim_dense_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ s0,
                                   float* __restrict__ s1, float* __restrict__ s2, int64_t n, OptimHP h,
                                   int zero_grad) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float pi = p[i];
    float a = s0 ? s0[i] : 0.f, b = s1 ? s1[i] : 0.f, c = s2 ? s2[i] : 0.f;
    optim_update(h, pi, a, b, c, g[i]);
    p[i] = pi;
    if (s0) s0[i] = a;
    if (s1) s1[i] = b;
    if (s2) s2[i] = c;
    if (zero_grad) g[i] = 0.f;
  }
}

__global__ void optim_dense_vec4_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ s0,
                                        float* __restrict__ s1, float* __restrict__ s2, int64_t n4, OptimHP h,
                                        int zero_grad) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t off = i * 4;
    float4 p4 = *reinterpret_cast<float4*>(p + off);
    float4 a4 = load4_or_zero(s0, off), b4 = load4_or_zero(s1, off), c4 = load4_or_zero(s2, off);
    const float4 g4 = *reinterpret_cast<const float4*>(g + off);
    optim_update4(h, p4, a4, b4, c4, g4);
    *reinterpret_cast<float4*>(p + off) = p4;
    store4_if(s0, off, a4);
    store4_if(s1, off, b4);
    store4_if(s2, off, c4);
    if (zero_grad) *reinterpret_cast<float4*>(g + off) = make_float4(0.f, 0.f, 0.f, 0.f);   // after the stores above
  }
}

static int optim_grid(int64_t n) {
  int64_t blocks = (n + 255) / 256;
  const int64_t cap = (int64_t)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  return (int)(blocks < 1 ? 1 : blocks);
}

// ---- row form ------------------------------------------------------------------------------------------------------
// MODE 0: catch up to `step` (zero-gradient replay only)
// MODE 1: apply step `step` with the accumulated gradient row, zero the gradient row
// step_dev (CUDA-graph form): `step` is then an offset to *step_dev (0 = catch up, 1 = the next step)
template <int MODE>
__global__ void optim_rows_kernel(const int32_t* __restrict__ idx, const int64_t* __restrict__ row_offsets,
                                  float* __restrict__ table, float* __restrict__ s0, float* __restrict__ s1,
                                  float* __restrict__ s2, float* __restrict__ grad, int32_t* __restrict__ last_step,
                                  int step, OptimHP h, int B, int F, int D, const int32_t* __restrict__ step_dev) {
  if (step_dev) step += *step_dev;
  if (step <= 0) return;
  const int Q = D >> 2;                      // lanes per row (power of two <= 32, checked by the host)
  const int64_t total = (int64_t)B * F * Q;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int lane = threadIdx.x & 31;
  const int64_t total_pad = (total + 31) / 32 * 32;   // whole warps stay converged for the shuffle
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
    float4 a4 = load4_or_zero(s0, off), b4 = load4_or_zero(s1, off), c4 = load4_or_zero(s2, off);
    if (MODE == 0) {
      optim_replay(h, p4, a4, b4, c4, old + 1, step);
    } else {
      // rows_apply presumes the catch-up to step-1 already ran; replay defensively if it did not
      if (h.replay) optim_replay(h, p4, a4, b4, c4, old + 1, step - 1);
      const float4 g4 = *reinterpret_cast<const float4*>(grad + off);
      optim_update4(h, p4, a4, b4, c4, g4);
      *reinterpret_cast<float4*>(grad + off) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    *reinterpret_cast<float4*>(table + off) = p4;
    store4_if(s0, off, a4);
    store4_if(s1, off, b4);
    store4_if(s2, off, c4);
  }
}

__global__ void optim_rows_flush_kernel(float* __restrict__ table, float* __restrict__ s0, float* __restrict__ s1,
                                        float* __restrict__ s2, const int32_t* __restrict__ last_step, int upto,
                                        OptimHP h, int64_t n_rows, int D, const int32_t* __restrict__ step_dev) {
  if (step_dev) upto = *step_dev;
  const int Q = D >> 2;
  const int64_t total = n_rows * Q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / Q;
    const int q = (int)(i - row * Q);
    const int old = last_step[row];
    if (old >= upto) continue;
    const int64_t off = row * D + (q << 2);
    float4 p4 = *reinterpret_cast<float4*>(table + off);
    float4 a4 = load4_or_zero(s0, off), b4 = load4_or_zero(s1, off), c4 = load4_or_zero(s2, off);
    optim_replay(h, p4, a4, b4, c4, old + 1, upto);
    *reinterpret_cast<float4*>(table + off) = p4;
    store4_if(s0, off, a4);
    store4_if(s1, off, b4);
    store4_if(s2, off, c4);
  }
}

// runs after the flush kernel on the same stream: every row is current as of `upto`
__global__ void optim_set_last_step_kernel(int32_t* __restrict__ last_step, int64_t n_rows, int upto,
                                           const int32_t* __restrict__ step_dev) {
  if (step_dev) upto = *step_dev;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_rows; i += (int64_t)gridDim.x * blockDim.x)
    if (last_step[i] < upto) last_step[i] = upto;
}

static bool optim_rows_shape_ok(int D) {
  const int Q = D / 4;
  return D % 4 == 0 && Q >= 1 && Q <= 32 && (Q & (Q - 1)) == 0;
}

static int rows_impl(int mode, const int32_t* idx, const int64_t* row_offsets, float* table, float* s0, float* s1,
                     float* s2, float* grad, int32_t* last_step, int step, const int32_t* step_dev,
                     const dtb_optim_params* hp, int B, int F, int D, void* stream) {
  if (B <= 0 || F <= 0) return DTB_OK;
  if (mode == 0 && zero_step_is_identity(*hp)) return DTB_OK;
  const int64_t total = (int64_t)B * F * (D / 4);
  const OptimHP h = to_hp(*hp);
  if (mode == 0)
    optim_rows_kernel<0><<<optim_grid(total), 256, 0, (cudaStream_t)stream>>>(
        idx, row_offsets, table, s0, s1, s2, nullptr, last_step, step, h, B, F, D, step_dev);
  else
    optim_rows_kernel<1><<<optim_grid(total), 256, 0, (cudaStream_t)stream>>>(
        idx, row_offsets, table, s0, s1, s2, grad, last_step, step, h, B, F, D, step_dev);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

static int flush_impl(float* table, float* s0, float* s1, float* s2, int32_t* last_step, int upto,
                      const int32_t* step_dev, const dtb_optim_params* hp, int64_t n_rows, int D, void* stream) {
  if (n_rows <= 0 || zero_step_is_identity(*hp)) return DTB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  optim_rows_flush_kernel<<<optim_grid(n_rows * (D / 4)), 256, 0, st>>>(table, s0, s1, s2, last_step, upto,
                                                                         to_hp(*hp), n_rows, D, step_dev);
  DTB_LAUNCH_OK();
  optim_set_last_step_kernel<<<optim_grid(n_rows), 256, 0, st>>>(last_step, n_rows, upto, step_dev);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

}  // namespace dtb

using namespace dtb;

#define DTB_ROWS_SHAPE_OK(D) DTB_CHECK_ARG(optim_rows_shape_ok(D), "embedding dim must be 4*2^k (<=128) for the row-wise optimiser")

extern "C" {

int dtb_optim_dense(float* p, float* g, float* s0, float* s1, float* s2, int64_t n, const dtb_optim_params* hp,
                    int zero_grad, void* stream) {
  DTB_CHECK_ARG(p && g, "NULL argument");
  DTB_CHECK_HP(hp, s0, s1, s2);
  if (n <= 0) return DTB_OK;
  const OptimHP h = to_hp(*hp);
  const bool aligned = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) |
                         reinterpret_cast<uintptr_t>(s0) | reinterpret_cast<uintptr_t>(s1) |
                         reinterpret_cast<uintptr_t>(s2)) & 15) == 0;
  const int64_t n4 = aligned ? n / 4 : 0;
  if (n4 > 0) {
    optim_dense_vec4_kernel<<<optim_grid(n4), 256, 0, (cudaStream_t)stream>>>(p, g, s0, s1, s2, n4, h, zero_grad);
    DTB_LAUNCH_OK();
  }
  const int64_t done = n4 * 4;
  if (done < n) {
    optim_dense_kernel<<<optim_grid(n - done), 256, 0, (cudaStream_t)stream>>>(
        p + done, g + done, s0 ? s0 + done : nullptr, s1 ? s1 + done : nullptr, s2 ? s2 + done : nullptr, n - done, h,
        zero_grad);
    DTB_LAUNCH_OK();
  }
  return DTB_OK;
}

int dtb_optim_rows_catchup(const int32_t* idx, const int64_t* row_offsets, float* table, float* s0, float* s1,
                           float* s2, int32_t* last_step, int upto, const dtb_optim_params* hp, int B, int F, int D,
                           void* stream) {
  DTB_CHECK_ARG(idx && row_offsets && table && last_step, "NULL argument");
  DTB_CHECK_HP(hp, s0, s1, s2);
  DTB_ROWS_SHAPE_OK(D);
  if (upto <= 0) return DTB_OK;
  return rows_impl(0, idx, row_offsets, table, s0, s1, s2, nullptr, last_step, upto, nullptr, hp, B, F, D, stream);
}

int dtb_optim_rows_apply(const int32_t* idx, const int64_t* row_offsets, float* table, float* s0, float* s1, float* s2,
                         float* grad_table, int32_t* last_step, int step, const dtb_optim_params* hp, int B, int F,
                         int D, void* stream) {
  DTB_CHECK_ARG(idx && row_offsets && table && grad_table && last_step, "NULL argument");
  DTB_CHECK_HP(hp, s0, s1, s2);
  DTB_ROWS_SHAPE_OK(D);
  DTB_CHECK_ARG(step >= 1, "step is 1-based");
  return rows_impl(1, idx, row_offsets, table, s0, s1, s2, grad_table, last_step, step, nullptr, hp, B, F, D, stream);
}

int dtb_optim_rows_flush(float* table, float* s0, float* s1, float* s2, int32_t* last_step, int upto,
                         const dtb_optim_params* hp, int64_t n_rows, int D, void* stream) {
  DTB_CHECK_ARG(table && last_step, "NULL argument");
  DTB_CHECK_HP(hp, s0, s1, s2);
  DTB_ROWS_SHAPE_OK(D);
  if (upto <= 0) return DTB_OK;
  return flush_impl(table, s0, s1, s2, last_step, upto, nullptr, hp, n_rows, D, stream);
}

// CUDA-graph forms: *step_dev = optimiser steps completed so far; catch-up and flush to *step_dev, apply step
// *step_dev + 1
int dtb_optim_rows_catchup_dev(const int32_t* idx, const int64_t* row_offsets, float* table, float* s0, float* s1,
                               float* s2, int32_t* last_step, const int32_t* step_dev, const dtb_optim_params* hp,
                               int B, int F, int D, void* stream) {
  DTB_CHECK_ARG(idx && row_offsets && table && last_step && step_dev, "NULL argument");
  DTB_CHECK_HP(hp, s0, s1, s2);
  DTB_ROWS_SHAPE_OK(D);
  return rows_impl(0, idx, row_offsets, table, s0, s1, s2, nullptr, last_step, 0, step_dev, hp, B, F, D, stream);
}

int dtb_optim_rows_apply_dev(const int32_t* idx, const int64_t* row_offsets, float* table, float* s0, float* s1,
                             float* s2, float* grad_table, int32_t* last_step, const int32_t* step_dev,
                             const dtb_optim_params* hp, int B, int F, int D, void* stream) {
  DTB_CHECK_ARG(idx && row_offsets && table && grad_table && last_step && step_dev, "NULL argument");
  DTB_CHECK_HP(hp, s0, s1, s2);
  DTB_ROWS_SHAPE_OK(D);
  return rows_impl(1, idx, row_offsets, table, s0, s1, s2, grad_table, last_step, 1, step_dev, hp, B, F, D, stream);
}

int dtb_optim_rows_flush_dev(float* table, float* s0, float* s1, float* s2, int32_t* last_step,
                             const int32_t* step_dev, const dtb_optim_params* hp, int64_t n_rows, int D, void* stream) {
  DTB_CHECK_ARG(table && last_step && step_dev, "NULL argument");
  DTB_CHECK_HP(hp, s0, s1, s2);
  DTB_ROWS_SHAPE_OK(D);
  return flush_impl(table, s0, s1, s2, last_step, 0, step_dev, hp, n_rows, D, stream);
}

}  // extern "C"
