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
#include <initializer_list>

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

// ---- Keras weight regularizers (L1, L2, L1L2) ------------------------------------------------------------------------
// Loss l1*sum|w| + l2*sum w^2 and gradient l1*sign(w) + 2*l2*w (sign(0) = 0, TensorFlow's gradient of abs).  The total
// gradient is formed as g + (l1*sign(w) + (2*l2)*w) with every rounding pinned, in reg_grad_kernel* and in the fused
// sweeps alike, so dtb_reg_grad followed by the plain sweep gives the fused sweep's bits.  The loss term is summed in
// float64 from the weights before the step.
struct RegArgs {
  float l1, tl2;        // l1 and 2*l2 (exact in fp32)
  double l2;
  double* loss_acc;     // NULL: no loss term
  double scale;
};

__device__ __forceinline__ float reg_total_grad(float g, float w, const RegArgs& r) {
  const float s = w > 0.f ? 1.f : (w < 0.f ? -1.f : 0.f);
  return __fadd_rn(g, __fadd_rn(__fmul_rn(r.l1, s), __fmul_rn(r.tl2, w)));
}

__device__ __forceinline__ void reg_sums(float w, double& a1, double& a2) {
  const double d = (double)w;
  a1 += fabs(d);
  a2 = fma(d, d, a2);
}

// every thread of the block calls this once, after its loop
__device__ __forceinline__ void reg_loss_flush(const RegArgs& r, double a1, double a2) {
  __shared__ double part[32];
  double v = warp_sum(r.scale * ((double)r.l1 * a1 + r.l2 * a2));
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) part[wid] = v;
  __syncthreads();
  if (wid == 0) {
    v = warp_sum(lane < (int)(blockDim.x >> 5) ? part[lane] : 0.0);
    if (lane == 0) atomicAdd(r.loss_acc, v);
  }
}

// What a sweep does with (p, total g) at element i (scalar) or float4 index i; p and g are the values before the step.
struct RegGradOnly {          // dtb_reg_grad: write the total gradient back (g may be NULL: loss only)
  float* g;
  __device__ void prepare() {}
  __device__ void apply1(int64_t i, float, float gt) const { if (g) g[i] = gt; }
  __device__ void apply4(int64_t i, float4, float4 gt) const { if (g) reinterpret_cast<float4*>(g)[i] = gt; }
};

struct AdamStep {
  float *p, *m, *v, *g;
  float alpha, omb1, omb2, eps;
  const float* alpha_table;
  const int32_t* step_dev;
  int zero_grad;
  __device__ void prepare() { if (step_dev) alpha = alpha_table[*step_dev + 1]; }
  __device__ void apply1(int64_t i, float pi, float gt) const {
    float mi = m[i], vi = v[i];
    adam_update(pi, mi, vi, gt, alpha, omb1, omb2, eps);
    p[i] = pi;
    m[i] = mi;
    v[i] = vi;
    if (zero_grad) g[i] = 0.f;
  }
  __device__ void apply4(int64_t i, float4 p4, float4 g4) const {
    float4 m4 = reinterpret_cast<float4*>(m)[i], v4 = reinterpret_cast<float4*>(v)[i];
    adam_update(p4.x, m4.x, v4.x, g4.x, alpha, omb1, omb2, eps);
    adam_update(p4.y, m4.y, v4.y, g4.y, alpha, omb1, omb2, eps);
    adam_update(p4.z, m4.z, v4.z, g4.z, alpha, omb1, omb2, eps);
    adam_update(p4.w, m4.w, v4.w, g4.w, alpha, omb1, omb2, eps);
    reinterpret_cast<float4*>(p)[i] = p4;
    reinterpret_cast<float4*>(m)[i] = m4;
    reinterpret_cast<float4*>(v)[i] = v4;
    if (zero_grad) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
};

struct OptimStep {
  float *p, *g, *s0, *s1, *s2;
  OptimHP h;
  int zero_grad;
  __device__ void prepare() {}
  __device__ void apply1(int64_t i, float pi, float gt) const {
    float a = s0 ? s0[i] : 0.f, b = s1 ? s1[i] : 0.f, c = s2 ? s2[i] : 0.f;
    optim_update(h, pi, a, b, c, gt);
    p[i] = pi;
    if (s0) s0[i] = a;
    if (s1) s1[i] = b;
    if (s2) s2[i] = c;
    if (zero_grad) g[i] = 0.f;
  }
  __device__ void apply4(int64_t i, float4 p4, float4 g4) const {
    const int64_t off = i * 4;
    float4 a4 = load4_or_zero(s0, off), b4 = load4_or_zero(s1, off), c4 = load4_or_zero(s2, off);
    optim_update4(h, p4, a4, b4, c4, g4);
    *reinterpret_cast<float4*>(p + off) = p4;
    store4_if(s0, off, a4);
    store4_if(s1, off, b4);
    store4_if(s2, off, c4);
    if (zero_grad) *reinterpret_cast<float4*>(g + off) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
};

template <class Op>
__global__ void reg_sweep_kernel(const float* p, const float* g, int64_t n, RegArgs r, Op op) {
  op.prepare();
  double a1 = 0.0, a2 = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float w = p[i];
    if (r.loss_acc) reg_sums(w, a1, a2);
    op.apply1(i, w, reg_total_grad(g ? g[i] : 0.f, w, r));
  }
  if (r.loss_acc) reg_loss_flush(r, a1, a2);
}

template <class Op>
__global__ void reg_sweep_vec4_kernel(const float* p, const float* g, int64_t n4, RegArgs r, Op op) {
  op.prepare();
  double a1 = 0.0, a2 = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 w = reinterpret_cast<const float4*>(p)[i];
    if (r.loss_acc) {
      reg_sums(w.x, a1, a2);
      reg_sums(w.y, a1, a2);
      reg_sums(w.z, a1, a2);
      reg_sums(w.w, a1, a2);
    }
    const float4 g4 = g ? reinterpret_cast<const float4*>(g)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 gt = make_float4(reg_total_grad(g4.x, w.x, r), reg_total_grad(g4.y, w.y, r),
                                  reg_total_grad(g4.z, w.z, r), reg_total_grad(g4.w, w.w, r));
    op.apply4(i, w, gt);
  }
  if (r.loss_acc) reg_loss_flush(r, a1, a2);
}

static bool reg_factors_ok(float l1, float l2) {
  return l1 >= 0.f && l2 >= 0.f && l1 <= 3.0e38f && l2 <= 1.0e38f;   // finite, non-negative, 2*l2 finite
}

static RegArgs to_reg(float l1, float l2, double* loss_acc, double loss_scale) {
  return RegArgs{l1, 2.f * l2, (double)l2, loss_acc, loss_scale};
}

static bool all_aligned16(std::initializer_list<const void*> ptrs) {
  uintptr_t bits = 0;
  for (const void* q : ptrs) bits |= reinterpret_cast<uintptr_t>(q);
  return (bits & 15) == 0;
}

// float4 sweep over the first n/4*4 elements when `aligned`, scalar kernel over the rest; `shift(op, k)` is op moved
// k elements on
template <class Op, class Shift>
static int reg_sweep(const float* p, const float* g, int64_t n, bool aligned, const RegArgs& r, Op op, Shift shift,
                     void* stream) {
  if (n <= 0) return DTB_OK;
  const int64_t n4 = aligned ? n / 4 : 0;
  if (n4 > 0) {
    reg_sweep_vec4_kernel<<<optim_grid(n4), 256, 0, (cudaStream_t)stream>>>(p, g, n4, r, op);
    DTB_LAUNCH_OK();
  }
  const int64_t done = n4 * 4;
  if (done < n) {
    reg_sweep_kernel<<<optim_grid(n - done), 256, 0, (cudaStream_t)stream>>>(p + done, g ? g + done : nullptr, n - done,
                                                                             r, shift(op, done));
    DTB_LAUNCH_OK();
  }
  return DTB_OK;
}

static inline float* off_or_null(float* q, int64_t k) { return q ? q + k : nullptr; }

static int adam_dense_reg_impl(float* p, float* m, float* v, float* g, int64_t n, float alpha, const float* alpha_table,
                               const int32_t* step_dev, double beta1, double beta2, float eps, int zero_grad,
                               const RegArgs& r, void* stream) {
  // keras multiplies by the python double (1 - beta) rounded to fp32, as adam_dense_impl does
  const AdamStep op{p, m, v, g, alpha, (float)(1.0 - beta1), (float)(1.0 - beta2), eps, alpha_table, step_dev, zero_grad};
  return reg_sweep(p, g, n, all_aligned16({p, m, v, g}), r, op,
                   [](AdamStep o, int64_t k) { o.p += k; o.m += k; o.v += k; o.g += k; return o; }, stream);
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

#define DTB_REG_FACTORS_OK(l1, l2) \
  DTB_CHECK_ARG(reg_factors_ok(l1, l2), "regularization factors must be finite and non-negative")

int dtb_reg_grad(const float* p, float* g, int64_t n, float l1, float l2, double* loss_acc, double loss_scale,
                 void* stream) {
  DTB_CHECK_ARG(p, "NULL argument");
  DTB_REG_FACTORS_OK(l1, l2);
  return reg_sweep(p, g, n, all_aligned16({p, g}), to_reg(l1, l2, loss_acc, loss_scale), RegGradOnly{g},
                   [](RegGradOnly o, int64_t k) { o.g = off_or_null(o.g, k); return o; }, stream);
}

int dtb_adam_dense_reg(float* p, float* m, float* v, float* g, int64_t n, float alpha, double beta1, double beta2,
                       float eps, int zero_grad, float l1, float l2, double* loss_acc, double loss_scale, void* stream) {
  DTB_CHECK_ARG(p && m && v && g, "NULL argument");
  DTB_REG_FACTORS_OK(l1, l2);
  return adam_dense_reg_impl(p, m, v, g, n, alpha, nullptr, nullptr, beta1, beta2, eps, zero_grad,
                             to_reg(l1, l2, loss_acc, loss_scale), stream);
}

int dtb_adam_dense_reg_dev(float* p, float* m, float* v, float* g, int64_t n, const float* alpha_table,
                           const int32_t* step_dev, double beta1, double beta2, float eps, int zero_grad, float l1,
                           float l2, double* loss_acc, double loss_scale, void* stream) {
  DTB_CHECK_ARG(p && m && v && g && alpha_table && step_dev, "NULL argument");
  DTB_REG_FACTORS_OK(l1, l2);
  return adam_dense_reg_impl(p, m, v, g, n, 0.f, alpha_table, step_dev, beta1, beta2, eps, zero_grad,
                             to_reg(l1, l2, loss_acc, loss_scale), stream);
}

int dtb_optim_dense_reg(float* p, float* g, float* s0, float* s1, float* s2, int64_t n, const dtb_optim_params* hp,
                        int zero_grad, float l1, float l2, double* loss_acc, double loss_scale, void* stream) {
  DTB_CHECK_ARG(p && g, "NULL argument");
  DTB_CHECK_HP(hp, s0, s1, s2);
  DTB_REG_FACTORS_OK(l1, l2);
  const OptimStep op{p, g, s0, s1, s2, to_hp(*hp), zero_grad};
  return reg_sweep(p, g, n, all_aligned16({p, g, s0, s1, s2}), to_reg(l1, l2, loss_acc, loss_scale), op,
                   [](OptimStep o, int64_t k) {
                     o.p += k;
                     o.g += k;
                     o.s0 = off_or_null(o.s0, k);
                     o.s1 = off_or_null(o.s1, k);
                     o.s2 = off_or_null(o.s2, k);
                     return o;
                   },
                   stream);
}

}  // extern "C"
