// BatchNormalization, Dense, task losses and the dense Adam step.
//   BN     : keras BatchNormalization(axis=-1)  (deepmodel.py:359, layers.py:152, deepnets.py:422)
//   Dense  : keras Dense                        (deepnets.py:415-424, deepmodel.py:292,455)
//   losses : sigmoid+BCE / MSE / softmax+CCE    (deepmodel.py:319-346,436-457), the focal losses and
//            Keras 3's MAE, MAPE, MSLE, Huber, LogCosh, Poisson, the hinge losses, KL divergence and
//            label-smoothed BCE / CCE (ModelConfig.loss, losses.py)
//   Adam   : keras.optimizers.Adam.update_step  (deepmodel.py:321-322)
// The Dense GEMMs are plain fp32 library GEMMs (cuBLAS Sgemm); everything around them (bias,
// activation, narrow logit layers, reductions) is hand-written.  All of it is HBM-bound streaming.
#include <cfloat>
#include "dtb_common.cuh"
#include "dense_tc.h"

namespace dtb {

// ------------------------------------------------------------------------------------------
// column statistics over X[rows, cols]: block = 32 columns x 8 row-lanes, fp64 accumulation
// ------------------------------------------------------------------------------------------
constexpr int kColTile = 32;
constexpr int kRowLanes = 8;

// MODE 0: ws[c] += sum x ; ws[cols+c] += sum x^2
// MODE 1: ws[c] += sum dy ; ws[cols+c] += sum dy * xhat      (BN backward)
// MODE 2: ws[c] += sum a[r,c]*b[r]  (b is a per-row vector, used by narrow Dense backward), cols only
template <int MODE>
__global__ void col_reduce_kernel(const float* __restrict__ A, const float* __restrict__ Bm,
                                  const float* __restrict__ mean, const float* __restrict__ var, float eps,
                                  double* __restrict__ ws, int rows, int cols, int rows_per_block) {
  __shared__ double s0[kRowLanes][kColTile];
  __shared__ double s1[kRowLanes][kColTile];
  const int c = blockIdx.x * kColTile + threadIdx.x;
  const int r_begin = blockIdx.y * rows_per_block;
  const int r_end = min(rows, r_begin + rows_per_block);
  double a0 = 0.0, a1 = 0.0;
  if (c < cols) {
    float mu = 0.f, inv = 0.f;
    if (MODE == 1) {
      mu = mean[c];
      inv = rsqrtf(var[c] + eps);
    }
    for (int r = r_begin + threadIdx.y; r < r_end; r += kRowLanes) {
      const float x = A[(int64_t)r * cols + c];
      if (MODE == 0) {
        a0 += (double)x;
        a1 += (double)x * (double)x;
      } else if (MODE == 1) {
        const float dy = Bm[(int64_t)r * cols + c];
        a0 += (double)dy;
        a1 += (double)(dy * ((x - mu) * inv));
      } else {
        a0 += (double)(x * Bm[r]);
      }
    }
  }
  s0[threadIdx.y][threadIdx.x] = a0;
  s1[threadIdx.y][threadIdx.x] = a1;
  __syncthreads();
  if (threadIdx.y == 0 && c < cols) {
    for (int k = 1; k < kRowLanes; ++k) {
      a0 += s0[k][threadIdx.x];
      a1 += s1[k][threadIdx.x];
    }
    atomicAdd(ws + c, a0);
    if (MODE != 2) atomicAdd(ws + cols + c, a1);
  }
}

static void col_reduce_grid(int rows, int cols, dim3& grid, dim3& block, int& rows_per_block) {
  block = dim3(kColTile, kRowLanes);
  const int col_blocks = ceil_div(cols, kColTile);
  int row_blocks = ceil_div((int64_t)sm_count() * 8, col_blocks);
  const int max_row_blocks = ceil_div(rows, kRowLanes * 4);
  if (row_blocks > max_row_blocks) row_blocks = max_row_blocks;
  if (row_blocks < 1) row_blocks = 1;
  rows_per_block = ceil_div(rows, row_blocks);
  row_blocks = ceil_div(rows, rows_per_block);
  grid = dim3(col_blocks, row_blocks);
}

__global__ void bn_finalize_stats(const double* __restrict__ ws, float* __restrict__ moving_mean,
                                  float* __restrict__ moving_var, float* __restrict__ save_mean,
                                  float* __restrict__ save_var, int rows, int cols, float momentum) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  const double mean = ws[c] / rows;
  double var = ws[cols + c] / rows - mean * mean;   // biased variance (tf.nn.moments)
  if (var < 0.0) var = 0.0;
  save_mean[c] = (float)mean;
  save_var[c] = (float)var;
  moving_mean[c] = moving_mean[c] * momentum + (float)mean * (1.f - momentum);
  moving_var[c] = moving_var[c] * momentum + (float)var * (1.f - momentum);
}

__global__ void bn_apply_kernel(const float* __restrict__ X, float* __restrict__ Y,
                                const float* __restrict__ gamma, const float* __restrict__ beta,
                                const float* __restrict__ mean, const float* __restrict__ var, float eps,
                                int64_t total, int cols) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % cols);
    Y[i] = (X[i] - mean[c]) * rsqrtf(var[c] + eps) * gamma[c] + beta[c];
  }
}

// dX = dY * (rsqrt(var + eps) * gamma): the factors of bn_apply_kernel's scale in its order
__global__ void bn_infer_bwd_kernel(const float* __restrict__ dY, float* __restrict__ dX,
                                    const float* __restrict__ gamma, const float* __restrict__ var, float eps,
                                    int64_t total, int cols) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % cols);
    dX[i] = dY[i] * (rsqrtf(var[c] + eps) * gamma[c]);
  }
}

__global__ void bn_bwd_apply_kernel(const float* __restrict__ X, const float* __restrict__ dY,
                                    float* __restrict__ dX, const float* __restrict__ gamma,
                                    const float* __restrict__ mean, const float* __restrict__ var,
                                    const double* __restrict__ ws, float eps, int64_t total, int rows,
                                    int cols) {
  const float inv_n = 1.f / (float)rows;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % cols);
    const float inv = rsqrtf(var[c] + eps);
    const float xhat = (X[i] - mean[c]) * inv;
    const float dbeta = (float)ws[c], dgamma = (float)ws[cols + c];
    dX[i] = gamma[c] * inv * (dY[i] - dbeta * inv_n - xhat * dgamma * inv_n);
  }
}

__global__ void bn_bwd_commit_params(const double* __restrict__ ws, float* __restrict__ dgamma,
                                     float* __restrict__ dbeta, int cols) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  dbeta[c] += (float)ws[c];
  dgamma[c] += (float)ws[cols + c];
}

static int ew_grid(int64_t total) {
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = (int64_t)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  return (int)(blocks < 1 ? 1 : blocks);
}

// ------------------------------------------------------------------------------------------
// Dense epilogues and narrow (out_dim <= 8) logit layers
// ------------------------------------------------------------------------------------------
__global__ void act_bwd_kernel(const float* __restrict__ Y, float* __restrict__ dY, int64_t total, int act) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    if (act == DTB_ACT_TANH) {
      const float y = Y[i];
      dY[i] *= 1.f - y * y;
    } else if (!(Y[i] > 0.f)) {
      dY[i] = 0.f;
    }
  }
}

constexpr int kNarrow = 8;

// warp per row: y[r,o] = act(sum_k x[r,k] w[k,o] + b[o]),  out_dim <= kNarrow
__global__ void dense_narrow_fwd(const float* __restrict__ X, const float* __restrict__ W,
                                 const float* __restrict__ bias, float* __restrict__ Y, int rows, int in_dim,
                                 int out_dim, int act) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  for (int r = warp; r < rows; r += n_warps) {
    float acc[kNarrow];
#pragma unroll
    for (int o = 0; o < kNarrow; ++o) acc[o] = 0.f;
    for (int k = lane; k < in_dim; k += 32) {
      const float x = X[(int64_t)r * in_dim + k];
#pragma unroll
      for (int o = 0; o < kNarrow; ++o)
        if (o < out_dim) acc[o] += x * __ldg(W + (int64_t)k * out_dim + o);
    }
#pragma unroll
    for (int o = 0; o < kNarrow; ++o) {
      if (o >= out_dim) break;
      float v = warp_sum(acc[o]);
      if (lane == 0) {
        if (bias) v += bias[o];
        if (act == DTB_ACT_RELU) v = fmaxf(v, 0.f);
        else if (act == DTB_ACT_TANH) v = tanhf(v);
        Y[(int64_t)r * out_dim + o] = v;
      }
    }
  }
}

// dX[r,k] = sum_o dZ[r,o] W[k,o]
__global__ void dense_narrow_bwd_dx(const float* __restrict__ dZ, const float* __restrict__ W,
                                    float* __restrict__ dX, int64_t total, int in_dim, int out_dim) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / in_dim;
    const int k = (int)(i - r * in_dim);
    float s = 0.f;
    for (int o = 0; o < out_dim; ++o) s += dZ[r * out_dim + o] * __ldg(W + (int64_t)k * out_dim + o);
    dX[i] = s;
  }
}

// dW[k,o] += sum_r X[r,k] dZ[r,o]  for one o (blockIdx.z); same tiling as col_reduce (MODE 2 shape)
__global__ void dense_narrow_bwd_dw(const float* __restrict__ X, const float* __restrict__ dZ,
                                    float* __restrict__ dW, int rows, int in_dim, int out_dim,
                                    int rows_per_block) {
  __shared__ float s0[kRowLanes][kColTile];
  const int o = blockIdx.z;
  const int k = blockIdx.x * kColTile + threadIdx.x;
  const int r_begin = blockIdx.y * rows_per_block;
  const int r_end = min(rows, r_begin + rows_per_block);
  float a = 0.f;
  if (k < in_dim)
    for (int r = r_begin + threadIdx.y; r < r_end; r += kRowLanes)
      a += X[(int64_t)r * in_dim + k] * dZ[(int64_t)r * out_dim + o];
  s0[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.y == 0 && k < in_dim) {
    for (int j = 1; j < kRowLanes; ++j) a += s0[j][threadIdx.x];
    atomicAdd(dW + (int64_t)k * out_dim + o, a);
  }
}

// dbias[o] += sum_r dZ[r,o]   (any out_dim)
__global__ void col_sum_float_kernel(const float* __restrict__ A, float* __restrict__ out, int rows,
                                     int cols, int rows_per_block) {
  __shared__ float s0[kRowLanes][kColTile];
  const int c = blockIdx.x * kColTile + threadIdx.x;
  const int r_begin = blockIdx.y * rows_per_block;
  const int r_end = min(rows, r_begin + rows_per_block);
  float a = 0.f;
  if (c < cols)
    for (int r = r_begin + threadIdx.y; r < r_end; r += kRowLanes) a += A[(int64_t)r * cols + c];
  s0[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.y == 0 && c < cols) {
    for (int j = 1; j < kRowLanes; ++j) a += s0[j][threadIdx.x];
    atomicAdd(out + c, a);
  }
}

// ------------------------------------------------------------------------------------------
// losses
// ------------------------------------------------------------------------------------------
__global__ void loss_kernel(const float* __restrict__ z, const float* __restrict__ y,
                            const float* __restrict__ sw, float* __restrict__ prob, float* __restrict__ dz,
                            double* __restrict__ loss_sum, int rows, int cols, int task) {
  const float eps = 1e-7f;
  double local = 0.0;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
    const float w = sw ? sw[r] : 1.f;
    const float* zr = z + (int64_t)r * cols;
    const float* yr = y + (int64_t)r * cols;
    float* pr = prob + (int64_t)r * cols;
    float* dr = dz ? dz + (int64_t)r * cols : nullptr;
    float row_loss = 0.f;
    if (task == 0) {
      const float scale = w / ((float)rows * (float)cols);
      for (int c = 0; c < cols; ++c) {
        const float p = 1.f / (1.f + expf(-zr[c]));
        pr[c] = p;
        const float pc = fminf(fmaxf(p, eps), 1.f - eps);
        row_loss -= yr[c] * logf(pc) + (1.f - yr[c]) * logf(1.f - pc);
        if (dr) dr[c] = (p >= eps && p <= 1.f - eps) ? (p - yr[c]) * scale : 0.f;
      }
      row_loss /= (float)cols;
    } else if (task == 1) {
      const float scale = 2.f * w / ((float)rows * (float)cols);
      for (int c = 0; c < cols; ++c) {
        pr[c] = zr[c];
        const float d = zr[c] - yr[c];
        row_loss += d * d;
        if (dr) dr[c] = d * scale;
      }
      row_loss /= (float)cols;
    } else {
      float mx = -INFINITY;
      for (int c = 0; c < cols; ++c) mx = fmaxf(mx, zr[c]);
      float den = 0.f;
      for (int c = 0; c < cols; ++c) den += expf(zr[c] - mx);
      const float scale = w / (float)rows;
      // keras categorical_crossentropy on probabilities: renormalise (no-op after softmax), clip, -sum y log p
      float gdot = 0.f;   // sum_c y_c * [p_c unclipped]  -- softmax Jacobian contraction
      for (int c = 0; c < cols; ++c) {
        const float p = expf(zr[c] - mx) / den;
        pr[c] = p;
        const float pc = fminf(fmaxf(p, eps), 1.f - eps);
        row_loss -= yr[c] * logf(pc);
        if (p >= eps && p <= 1.f - eps) gdot += yr[c];
      }
      if (dr)
        for (int c = 0; c < cols; ++c) {
          const float p = pr[c];
          const float direct = (p >= eps && p <= 1.f - eps) ? yr[c] : 0.f;
          dr[c] = (p * gdot - direct) * scale;
        }
    }
    local += (double)(row_loss * w);
  }
  local = warp_sum(local);
  if (loss_sum && (threadIdx.x & 31) == 0 && local != 0.0) atomicAdd(loss_sum, local);
}

// Focal losses (reference layers.py:983-1083) on the task_output pre-activation.
// task 0: BinaryFocalLoss on p = sigmoid(z): pt_1 = (y == 1 ? p : 1), pt_0 = (y == 0 ? p : 0), both clipped to [eps, 1-eps];
//         loss = mean over ALL elements of  -alpha (1-pt_1)^gamma log pt_1 - (1-alpha) pt_0^gamma log(1-pt_0)  (a scalar).
// task 2: CategoricalFocalLoss on p = softmax(z): renormalise (identity, but its Jacobian is kept), clip,
//         per-sample sum_c alpha (1-p_c)^gamma (-y_c log p_c); Keras averages the samples.
//         dL/dz_k = p_k (g_k - sum_c g_c p_c) / rows,  g_c = dL/dq_c on the clipped renormalised probability.
__global__ void focal_loss_kernel(const float* __restrict__ z, const float* __restrict__ y, float* __restrict__ prob,
                                  float* __restrict__ dz, double* __restrict__ loss_sum, int rows, int cols, int task,
                                  float gamma, float alpha) {
  const float eps = 1e-7f;
  double local = 0.0;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
    const float* zr = z + (int64_t)r * cols;
    const float* yr = y + (int64_t)r * cols;
    float* pr = prob + (int64_t)r * cols;
    float* dr = dz ? dz + (int64_t)r * cols : nullptr;
    float row_loss = 0.f;
    if (task == 0) {
      const float scale = 1.f / ((float)rows * (float)cols);
      for (int c = 0; c < cols; ++c) {
        const float p = 1.f / (1.f + expf(-zr[c]));
        pr[c] = p;
        const bool is1 = yr[c] == 1.f, is0 = yr[c] == 0.f;
        const float pt1 = fminf(fmaxf(is1 ? p : 1.f, eps), 1.f - eps);
        const float pt0 = fminf(fmaxf(is0 ? p : 0.f, eps), 1.f - eps);
        row_loss += -alpha * powf(1.f - pt1, gamma) * logf(pt1) - (1.f - alpha) * powf(pt0, gamma) * logf(1.f - pt0);
        if (dr) {
          float g = 0.f;                                   // dLoss/dp: only the branch that depends on p, inside the clip range
          if (p >= eps && p <= 1.f - eps) {
            if (is1) g = alpha * (gamma * powf(1.f - p, gamma - 1.f) * logf(p) - powf(1.f - p, gamma) / p);
            else if (is0) g = (1.f - alpha) * (-gamma * powf(p, gamma - 1.f) * logf(1.f - p) + powf(p, gamma) / (1.f - p));
          }
          dr[c] = g * p * (1.f - p) * scale;
        }
      }
      row_loss /= (float)cols;
    } else {
      float mx = -INFINITY;
      for (int c = 0; c < cols; ++c) mx = fmaxf(mx, zr[c]);
      float den = 0.f;
      for (int c = 0; c < cols; ++c) den += expf(zr[c] - mx);
      float gp = 0.f;                                      // sum_c g_c p_c
      for (int c = 0; c < cols; ++c) {
        const float p = expf(zr[c] - mx) / den;
        pr[c] = p;
        const float q = fminf(fmaxf(p, eps), 1.f - eps);
        row_loss += alpha * powf(1.f - q, gamma) * (-yr[c] * logf(q));
        if (p >= eps && p <= 1.f - eps)
          gp += alpha * yr[c] * (gamma * powf(1.f - p, gamma - 1.f) * logf(p) - powf(1.f - p, gamma) / p) * p;
      }
      if (dr)
        for (int c = 0; c < cols; ++c) {
          const float p = pr[c];
          float g = 0.f;
          if (p >= eps && p <= 1.f - eps) g = alpha * yr[c] * (gamma * powf(1.f - p, gamma - 1.f) * logf(p) - powf(1.f - p, gamma) / p);
          dr[c] = p * (g - gp) / (float)rows;
        }
    }
    local += (double)row_loss;
  }
  local = warp_sum(local);
  if (loss_sum && (threadIdx.x & 31) == 0 && local != 0.0) atomicAdd(loss_sum, local);
}

// ------------------------------------------------------------------------------------------
// Keras 3 losses passed as ModelConfig.loss (losses.py), on the task output p of the pre-activation z:
// sigmoid (task 0), identity (task 1), softmax (task 2).  Per row: the loss l and, with dz, dz = w / rows * dl/dz,
// the derivative of the float32 expressions below under TensorFlow's conventions (clip passes the gradient on
// [lo, hi], maximum(a, b) to a where a >= b, abs'(0) = 0, a max over columns splits it among ties, where() to the
// branch taken).  Three passes over a row, all by the thread that owns it: the output (and CategoricalHinge's row
// statistics), the loss terms with g = d(term)/dp, then -- softmax or CategoricalCrossentropy only -- the chain
// through the renormalisation q = p / sum p and the softmax Jacobian, dz_k = p_k (h_k - sum_c h_c p_c).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float sign_f(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); }

// *not_binary = 1 when some label is neither 0 nor 1 (keras convert_binary_labels_to_hinge, batch-wide);
// the caller zeroes it first
__global__ void hinge_labels_kernel(const float* __restrict__ y, int64_t n, int* __restrict__ not_binary) {
  bool other = false;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = y[i];
    other |= !(v == 0.f || v == 1.f);
  }
  if (__syncthreads_or(other) && threadIdx.x == 0) *not_binary = 1;
}

__global__ void keras_loss_kernel(const float* __restrict__ z, const float* __restrict__ y,
                                  const float* __restrict__ sw, float* __restrict__ prob, float* __restrict__ dz,
                                  double* __restrict__ loss_sum, int rows, int cols, int task, int loss, float delta,
                                  float smoothing, const int* __restrict__ not_binary) {
  const float eps = 1e-7f;
  const bool to_pm1 = not_binary != nullptr && *not_binary == 0;     // hinge labels 0 / 1 -> -1 / 1
  const bool cce = loss == DTB_LOSS_CATEGORICAL_CROSSENTROPY;
  const bool summed = cce || loss == DTB_LOSS_KL_DIVERGENCE || loss == DTB_LOSS_CATEGORICAL_HINGE;   // else mean_c
  const bool late = task == 2 || cce;                                // dz needs a third pass over the row
  const float inv_c = 1.f / (float)cols;
  const float y_off = loss == DTB_LOSS_BINARY_CROSSENTROPY ? 0.5f * smoothing : smoothing * inv_c;
  double local = 0.0;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
    const float w = sw ? sw[r] : 1.f;
    const float* zr = z + (int64_t)r * cols;
    const float* yr = y + (int64_t)r * cols;
    float* pr = prob + (int64_t)r * cols;
    float* dr = dz ? dz + (int64_t)r * cols : nullptr;
    // pass 1: the task output; the row sum (renormalisation) and CategoricalHinge's pos / neg / ties
    float mx = -INFINITY, den = 0.f;
    if (task == 2) {
      for (int c = 0; c < cols; ++c) mx = fmaxf(mx, zr[c]);
      for (int c = 0; c < cols; ++c) den += expf(zr[c] - mx);
    }
    float s = 0.f, pos = 0.f, neg = -INFINITY;
    int ties = 0;
    for (int c = 0; c < cols; ++c) {
      const float p = task == 0 ? 1.f / (1.f + expf(-zr[c])) : (task == 1 ? zr[c] : expf(zr[c] - mx) / den);
      pr[c] = p;
      s += p;
      if (loss == DTB_LOSS_CATEGORICAL_HINGE) {
        const float t = (1.f - yr[c]) * p;
        pos += yr[c] * p;
        if (t > neg) {
          neg = t;
          ties = 1;
        } else if (t == neg) {
          ++ties;
        }
      }
    }
    const float margin = neg - pos + 1.f;                         // CategoricalHinge
    const bool ch_active = margin >= 0.f;
    // pass 2: loss terms and g = d(term)/dp (CategoricalCrossentropy: d/dq); g*p and g*q summed for pass 3
    float row = 0.f, gp = 0.f, gq = 0.f;
    const float scale = w / (float)rows;
    for (int c = 0; c < cols; ++c) {
      const float p = pr[c];
      const float yc = yr[c];
      float v = 0.f, g = 0.f;
      switch (loss) {
        case DTB_LOSS_MEAN_SQUARED_ERROR: {
          const float e = p - yc;
          v = e * e;
          g = 2.f * e;
          break;
        }
        case DTB_LOSS_MEAN_ABSOLUTE_ERROR:
          v = fabsf(yc - p);
          g = -sign_f(yc - p);
          break;
        case DTB_LOSS_MEAN_ABSOLUTE_PERCENTAGE_ERROR: {
          const float d = fmaxf(fabsf(yc), eps);
          const float q = (yc - p) / d;
          v = 100.f * fabsf(q);
          g = -100.f * sign_f(q) / d;
          break;
        }
        case DTB_LOSS_MEAN_SQUARED_LOGARITHMIC_ERROR: {
          const float pm = fmaxf(p, eps);
          const float e = logf(pm + 1.f) - logf(fmaxf(yc, eps) + 1.f);
          v = e * e;
          g = p >= eps ? 2.f * e / (pm + 1.f) : 0.f;
          break;
        }
        case DTB_LOSS_HUBER: {
          const float e = p - yc, ae = fabsf(e);
          if (ae <= delta) {
            v = 0.5f * (e * e);
            g = e;
          } else {
            v = delta * ae - 0.5f * (delta * delta);
            g = delta * sign_f(e);
          }
          break;
        }
        case DTB_LOSS_LOG_COSH: {
          const float e = p - yc, a = -2.f * e;
          const float softplus = a > 0.f ? a + log1pf(expf(-a)) : log1pf(expf(a));
          v = e + softplus - 0.69314718f;
          g = 1.f - 2.f / (1.f + expf(-a));                       // 1 - 2 sigmoid(-2e)
          break;
        }
        case DTB_LOSS_POISSON:
          v = p - yc * logf(p + eps);
          g = 1.f - yc / (p + eps);
          break;
        case DTB_LOSS_HINGE:
        case DTB_LOSS_SQUARED_HINGE: {
          const float yy = to_pm1 ? 2.f * yc - 1.f : yc;
          const float m = 1.f - yy * p;
          const float h = fmaxf(m, 0.f);
          const bool sq = loss == DTB_LOSS_SQUARED_HINGE;
          v = sq ? h * h : h;
          g = m >= 0.f ? (sq ? -2.f * h * yy : -yy) : 0.f;
          break;
        }
        case DTB_LOSS_CATEGORICAL_HINGE:
          g = ch_active ? (((1.f - yc) * p == neg ? (1.f - yc) / (float)ties : 0.f) - yc) : 0.f;
          break;
        case DTB_LOSS_KL_DIVERGENCE: {
          const float yh = fminf(fmaxf(yc, eps), 1.f), ph = fminf(fmaxf(p, eps), 1.f);
          v = yh * logf(yh / ph);
          g = (p >= eps && p <= 1.f) ? -yh / ph : 0.f;
          break;
        }
        case DTB_LOSS_BINARY_CROSSENTROPY: {
          const float ys = yc * (1.f - smoothing) + y_off;
          const float pc = fminf(fmaxf(p, eps), 1.f - eps);
          v = -(ys * logf(pc) + (1.f - ys) * logf(1.f - pc));
          g = (p >= eps && p <= 1.f - eps) ? (1.f - ys) / (1.f - pc) - ys / pc : 0.f;
          break;
        }
        default: {                                                // DTB_LOSS_CATEGORICAL_CROSSENTROPY
          const float ys = yc * (1.f - smoothing) + y_off;
          const float q = p / s;
          const float qc = fminf(fmaxf(q, eps), 1.f - eps);
          v = -ys * logf(qc);
          g = (q >= eps && q <= 1.f - eps) ? -ys / qc : 0.f;
          gq += g * q;
          break;
        }
      }
      row += v;
      if (!summed) g *= inv_c;
      if (dr) {
        if (late) {
          dr[c] = g;
          gp += g * p;
        } else {
          dr[c] = (task == 0 ? g * (p * (1.f - p)) : g) * scale;
        }
      }
    }
    if (loss == DTB_LOSS_CATEGORICAL_HINGE) row = fmaxf(margin, 0.f);
    else if (!summed) row /= (float)cols;
    // pass 3: h = dl/dp through the renormalisation (h_k = (g_k - sum g q) / s), then the activation
    if (dr && late) {
      const float inv_s = cce ? 1.f / s : 1.f;
      const float hp = cce ? (gp - gq * s) * inv_s : gp;           // sum_c h_c p_c
      for (int c = 0; c < cols; ++c) {
        const float p = pr[c];
        float h = cce ? (dr[c] - gq) * inv_s : dr[c];
        if (task == 0) h *= p * (1.f - p);
        else if (task == 2) h = p * (h - hp);
        dr[c] = h * scale;
      }
    }
    local += (double)(row * w);
  }
  local = warp_sum(local);
  if (loss_sum && (threadIdx.x & 31) == 0 && local != 0.0) atomicAdd(loss_sum, local);
}

// ------------------------------------------------------------------------------------------
// Dropout (keras Dropout / SpatialDropout1D on (B,1,D) field embeddings == element-wise): counter-based
// mask, so forward and backward regenerate the same bits from (seed, element index); nothing is stored.
// ------------------------------------------------------------------------------------------
__global__ void dropout_kernel(const float* __restrict__ X, float* __restrict__ Y, int64_t n, uint32_t threshold,
                               float scale, uint64_t seed, const unsigned long long* __restrict__ seed_dev) {
  const uint64_t key = dropout_key(seed, seed_dev);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    Y[i] = mix32(key + (uint64_t)i) >= threshold ? X[i] * scale : 0.f;
}

// end of a captured train step: every dropout call site's seed moves on by the number of sites, as the host's
// counter does between two passes (48-bit wrap of deepmodel._Scope.next_seed)
__global__ void seed_advance_kernel(unsigned long long* seeds, int n) {
  for (int k = 0; k < n; ++k) seeds[k] = (seeds[k] + (unsigned long long)n) & 0xFFFFFFFFFFFFULL;
}

// ------------------------------------------------------------------------------------------
// Adam (dense)
// ------------------------------------------------------------------------------------------
// alpha_table / step_dev (both or neither): the step size is read from alpha_table[*step_dev + 1] -- a step captured
// in a CUDA graph must not bake the host's step counter into its kernel arguments
__global__ void adam_dense_kernel(float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
                                  float* __restrict__ g, int64_t n, float alpha, float omb1, float omb2,
                                  float eps, int zero_grad, const float* __restrict__ alpha_table,
                                  const int32_t* __restrict__ step_dev) {
  if (step_dev) alpha = alpha_table[*step_dev + 1];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    float pi = p[i], mi = m[i], vi = v[i];
    adam_update(pi, mi, vi, g[i], alpha, omb1, omb2, eps);
    p[i] = pi;
    m[i] = mi;
    v[i] = vi;
    if (zero_grad) g[i] = 0.f;
  }
}

// Same arithmetic, 16 bytes per access: the 7 x 1.66 GB sweep over the embedding tables (dense table
// optimiser at world >= 4) is HBM-bound and scalar accesses leave bandwidth on the table.
__global__ void adam_dense_vec4_kernel(float4* __restrict__ p, float4* __restrict__ m, float4* __restrict__ v,
                                       float4* __restrict__ g, int64_t n4, float alpha, float omb1, float omb2,
                                       float eps, int zero_grad, const float* __restrict__ alpha_table,
                                       const int32_t* __restrict__ step_dev) {
  if (step_dev) alpha = alpha_table[*step_dev + 1];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (int64_t)gridDim.x * blockDim.x) {
    float4 p4 = p[i], m4 = m[i], v4 = v[i];
    const float4 g4 = g[i];
    adam_update(p4.x, m4.x, v4.x, g4.x, alpha, omb1, omb2, eps);
    adam_update(p4.y, m4.y, v4.y, g4.y, alpha, omb1, omb2, eps);
    adam_update(p4.z, m4.z, v4.z, g4.z, alpha, omb1, omb2, eps);
    adam_update(p4.w, m4.w, v4.w, g4.w, alpha, omb1, omb2, eps);
    p[i] = p4;
    m[i] = m4;
    v[i] = v4;
    if (zero_grad) g[i] = make_float4(0.f, 0.f, 0.f, 0.f);   // after the stores above: they depend on the loads
  }
}

}  // namespace dtb

using namespace dtb;

extern "C" {

int dtb_batchnorm_train_fwd(const float* X, float* Y, const float* gamma, const float* beta,
                            float* moving_mean, float* moving_var, float* save_mean, float* save_var,
                            double* workspace, int rows, int cols, float eps, float momentum, void* stream) {
  DTB_CHECK_ARG(X && Y && gamma && beta && moving_mean && moving_var && save_mean && save_var && workspace,
                "NULL argument");
  DTB_CHECK_ARG(rows > 0 && cols > 0, "rows/cols must be positive");
  cudaStream_t st = (cudaStream_t)stream;
  DTB_CUDA_OK(cudaMemsetAsync(workspace, 0, sizeof(double) * 2 * cols, st));
  dim3 grid, block;
  int rpb;
  col_reduce_grid(rows, cols, grid, block, rpb);
  col_reduce_kernel<0><<<grid, block, 0, st>>>(X, nullptr, nullptr, nullptr, 0.f, workspace, rows, cols, rpb);
  DTB_LAUNCH_OK();
  bn_finalize_stats<<<ceil_div(cols, 128), 128, 0, st>>>(workspace, moving_mean, moving_var, save_mean,
                                                        save_var, rows, cols, momentum);
  DTB_LAUNCH_OK();
  const int64_t total = (int64_t)rows * cols;
  bn_apply_kernel<<<ew_grid(total), 256, 0, st>>>(X, Y, gamma, beta, save_mean, save_var, eps, total, cols);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_batchnorm_infer_fwd(const float* X, float* Y, const float* gamma, const float* beta,
                            const float* moving_mean, const float* moving_var, int rows, int cols, float eps,
                            void* stream) {
  DTB_CHECK_ARG(X && Y && gamma && beta && moving_mean && moving_var, "NULL argument");
  DTB_CHECK_ARG(rows >= 0 && cols > 0, "bad shape");
  const int64_t total = (int64_t)rows * cols;
  if (total == 0) return DTB_OK;
  bn_apply_kernel<<<ew_grid(total), 256, 0, (cudaStream_t)stream>>>(X, Y, gamma, beta, moving_mean,
                                                                    moving_var, eps, total, cols);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_batchnorm_infer_bwd(const float* dY, float* dX, const float* gamma, const float* moving_var, int rows,
                            int cols, float eps, void* stream) {
  DTB_CHECK_ARG(dY && dX && gamma && moving_var, "NULL argument");
  DTB_CHECK_ARG(rows >= 0 && cols > 0, "bad shape");
  const int64_t total = (int64_t)rows * cols;
  if (total == 0) return DTB_OK;
  bn_infer_bwd_kernel<<<ew_grid(total), 256, 0, (cudaStream_t)stream>>>(dY, dX, gamma, moving_var, eps, total, cols);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_batchnorm_bwd(const float* X, const float* dY, float* dX, const float* gamma, const float* save_mean,
                      const float* save_var, float* dgamma, float* dbeta, double* workspace, int rows,
                      int cols, float eps, void* stream) {
  DTB_CHECK_ARG(X && dY && dX && gamma && save_mean && save_var && dgamma && dbeta && workspace,
                "NULL argument");
  DTB_CHECK_ARG(rows > 0 && cols > 0, "rows/cols must be positive");
  cudaStream_t st = (cudaStream_t)stream;
  DTB_CUDA_OK(cudaMemsetAsync(workspace, 0, sizeof(double) * 2 * cols, st));
  dim3 grid, block;
  int rpb;
  col_reduce_grid(rows, cols, grid, block, rpb);
  col_reduce_kernel<1><<<grid, block, 0, st>>>(X, dY, save_mean, save_var, eps, workspace, rows, cols, rpb);
  DTB_LAUNCH_OK();
  const int64_t total = (int64_t)rows * cols;
  bn_bwd_apply_kernel<<<ew_grid(total), 256, 0, st>>>(X, dY, dX, gamma, save_mean, save_var, workspace, eps,
                                                      total, rows, cols);
  DTB_LAUNCH_OK();
  bn_bwd_commit_params<<<ceil_div(cols, 128), 128, 0, st>>>(workspace, dgamma, dbeta, cols);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

size_t dtb_dense_workspace_bytes(int in_dim, int out_dim) {
  if (in_dim <= 0 || out_dim <= 0 || out_dim <= kNarrow) return 0;     // the narrow (logit) kernels need none
  const size_t a = dense_tc_pack_bytes(in_dim, out_dim), b = dense_tc_pack_bytes(out_dim, in_dim);
  return a > b ? a : b;
}

int dtb_dense_fwd(const float* X, const float* W, const float* bias, float* Y, void* workspace,
                  size_t workspace_bytes, int rows, int in_dim, int out_dim, int act, void* stream) {
  DTB_CHECK_ARG(X && W && Y, "NULL argument");
  DTB_CHECK_ARG(rows >= 0 && in_dim > 0 && out_dim > 0, "bad shape");
  DTB_CHECK_ARG(act == DTB_ACT_NONE || act == DTB_ACT_RELU || act == DTB_ACT_TANH, "unsupported activation");
  if (rows == 0) return DTB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (out_dim <= kNarrow) {
    int blocks = ceil_div(rows, 8);
    const int cap = sm_count() * 8;
    if (blocks > cap) blocks = cap;
    dense_narrow_fwd<<<blocks, 256, 0, st>>>(X, W, bias, Y, rows, in_dim, out_dim, act);
    DTB_LAUNCH_OK();
    return DTB_OK;
  }
  // wgmma GEMM with the bias / activation epilogue fused (dense_tc.cu)
  return dense_tc_rows(X, in_dim, W, out_dim, 0, bias, Y, out_dim, rows, in_dim, out_dim, act, workspace,
                       workspace_bytes, st);
}

int dtb_dense_bwd(const float* X, const float* W, const float* Y, float* dY, float* dX, float* dW,
                  float* dbias, void* workspace, size_t workspace_bytes, int rows, int in_dim, int out_dim, int act,
                  void* stream) {
  DTB_CHECK_ARG(X && W && dY && (dW || dX), "NULL argument");
  DTB_CHECK_ARG(dW || !dbias, "dbias without dW");
  DTB_CHECK_ARG(act == DTB_ACT_NONE || ((act == DTB_ACT_RELU || act == DTB_ACT_TANH) && Y), "relu / tanh backward needs Y");
  DTB_CHECK_ARG(rows >= 0 && in_dim > 0 && out_dim > 0, "bad shape");
  if (rows == 0) return DTB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t total_out = (int64_t)rows * out_dim;
  if (act != DTB_ACT_NONE) {
    act_bwd_kernel<<<ew_grid(total_out), 256, 0, st>>>(Y, dY, total_out, act);
    DTB_LAUNCH_OK();
  }
  dim3 grid, block;
  int rpb;
  if (out_dim <= kNarrow) {
    if (dbias) {
      col_reduce_grid(rows, out_dim, grid, block, rpb);
      col_sum_float_kernel<<<grid, block, 0, st>>>(dY, dbias, rows, out_dim, rpb);
      DTB_LAUNCH_OK();
    }
    if (dW) {
      col_reduce_grid(rows, in_dim, grid, block, rpb);
      grid.z = out_dim;
      dense_narrow_bwd_dw<<<grid, block, 0, st>>>(X, dY, dW, rows, in_dim, out_dim, rpb);
      DTB_LAUNCH_OK();
    }
    if (dX) {
      const int64_t total_in = (int64_t)rows * in_dim;
      dense_narrow_bwd_dx<<<ew_grid(total_in), 256, 0, st>>>(dY, W, dX, total_in, in_dim, out_dim);
      DTB_LAUNCH_OK();
    }
    return DTB_OK;
  }
  // dW[in,out] += X^T dZ and dbias += colsum(dZ) in one wgmma kernel; dX[rows,in] = dZ W^T in another
  int rc = DTB_OK;
  if (dW) rc = dense_tc_wgrad(X, in_dim, dY, out_dim, dW, out_dim, dbias, rows, in_dim, out_dim, st);
  if (rc != DTB_OK) return rc;
  if (dX)
    rc = dense_tc_rows(dY, out_dim, W, out_dim, 1, nullptr, dX, in_dim, rows, out_dim, in_dim, DTB_ACT_NONE, workspace,
                       workspace_bytes, st);
  return rc;
}

int dtb_loss_fwd_bwd(const float* z, const float* y_true, const float* sample_weight, float* prob, float* dz,
                     double* loss_sum, int rows, int cols, int task, void* stream) {
  DTB_CHECK_ARG(z && y_true && prob, "NULL argument");
  DTB_CHECK_ARG(rows >= 0 && cols > 0 && task >= 0 && task <= 2, "bad shape/task");
  if (rows == 0) return DTB_OK;
  int blocks = ceil_div(rows, 256);
  const int cap = sm_count() * 8;
  if (blocks > cap) blocks = cap;
  loss_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(z, y_true, sample_weight, prob, dz, loss_sum, rows,
                                                        cols, task);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_focal_loss_fwd_bwd(const float* z, const float* y_true, float* prob, float* dz, double* loss_sum, int rows, int cols,
                           int task, float gamma, float alpha, void* stream) {
  DTB_CHECK_ARG(z && y_true && prob, "NULL argument");
  DTB_CHECK_ARG(rows >= 0 && cols >= 1, "bad shape");
  DTB_CHECK_ARG(task == 0 || task == 2, "focal loss: task 0 (binary / multilabel) or 2 (multiclass)");
  DTB_CHECK_ARG(gamma >= 0.f && alpha >= 0.f && alpha <= 1.f, "focal loss: gamma >= 0, 0 <= alpha <= 1");
  if (rows == 0) return DTB_OK;
  int blocks = ceil_div(rows, 256);
  const int cap = sm_count() * 8;
  if (blocks > cap) blocks = cap;
  focal_loss_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(z, y_true, prob, dz, loss_sum, rows, cols, task, gamma, alpha);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_keras_loss_fwd_bwd(const float* z, const float* y_true, const float* sample_weight, float* prob, float* dz,
                           double* loss_sum, int rows, int cols, int task, const dtb_loss_params* lp, void* stream) {
  DTB_CHECK_ARG(z && y_true && prob && lp, "NULL argument");
  DTB_CHECK_ARG(rows >= 0 && cols > 0 && task >= 0 && task <= 2, "bad shape/task");
  const int loss = lp->loss;
  DTB_CHECK_ARG(loss >= DTB_LOSS_MEAN_SQUARED_ERROR && loss <= DTB_LOSS_CATEGORICAL_CROSSENTROPY, "unknown loss code");
  DTB_CHECK_ARG(loss != DTB_LOSS_HUBER || (lp->delta > 0.f && lp->delta <= FLT_MAX), "Huber delta must be positive and finite");
  DTB_CHECK_ARG(lp->label_smoothing >= 0.f && lp->label_smoothing <= 1.f, "label_smoothing must be in [0, 1]");
  const bool hinge = loss == DTB_LOSS_HINGE || loss == DTB_LOSS_SQUARED_HINGE;
  DTB_CHECK_ARG(!hinge || lp->scratch, "the hinge losses need lp->scratch (one device int)");
  if (rows == 0) return DTB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (hinge) {
    const int64_t n = (int64_t)rows * cols;
    DTB_CUDA_OK(cudaMemsetAsync(lp->scratch, 0, sizeof(int), st));
    hinge_labels_kernel<<<ew_grid(n), 256, 0, st>>>(y_true, n, lp->scratch);
    DTB_LAUNCH_OK();
  }
  int blocks = ceil_div(rows, 256);
  const int cap = sm_count() * 8;
  if (blocks > cap) blocks = cap;
  keras_loss_kernel<<<blocks, 256, 0, st>>>(z, y_true, sample_weight, prob, dz, loss_sum, rows, cols, task, loss,
                                            lp->delta, lp->label_smoothing, hinge ? lp->scratch : nullptr);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

static int dropout_impl(const float* X, float* Y, int64_t n, float rate, unsigned long long seed,
                        const unsigned long long* seed_dev, void* stream) {
  if (n <= 0) return DTB_OK;
  dropout_kernel<<<ew_grid(n), 256, 0, (cudaStream_t)stream>>>(X, Y, n, dropout_threshold(rate), 1.f / (1.f - rate), seed,
                                                               seed_dev);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_dropout(const float* X, float* Y, int64_t n, float rate, unsigned long long seed, void* stream) {
  DTB_CHECK_ARG(X && Y, "NULL argument");
  DTB_CHECK_ARG(rate >= 0.f && rate < 1.f, "rate must be in [0, 1)");
  return dropout_impl(X, Y, n, rate, seed, nullptr, stream);
}

int dtb_dropout_dev(const float* X, float* Y, int64_t n, float rate, const unsigned long long* seed, void* stream) {
  DTB_CHECK_ARG(X && Y && seed, "NULL argument");
  DTB_CHECK_ARG(rate >= 0.f && rate < 1.f, "rate must be in [0, 1)");
  return dropout_impl(X, Y, n, rate, 0, seed, stream);
}

int dtb_seed_advance(unsigned long long* seeds, int n, void* stream) {
  DTB_CHECK_ARG(seeds && n >= 1, "need a seed buffer of n >= 1 slots");
  seed_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(seeds, n);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

static int adam_dense_impl(float* p, float* m, float* v, float* g, int64_t n, float alpha, const float* alpha_table,
                           const int32_t* step_dev, double beta1, double beta2, float eps, int zero_grad, void* stream) {
  if (n <= 0) return DTB_OK;
  // keras multiplies by the python double (1 - beta) rounded to fp32, not by 1.f - float(beta)
  const float omb1 = (float)(1.0 - beta1), omb2 = (float)(1.0 - beta2);
  const bool aligned = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(m) |
                         reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(g)) & 15) == 0;
  const int64_t n4 = aligned ? n / 4 : 0;
  if (n4 > 0) {
    adam_dense_vec4_kernel<<<ew_grid(n4), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<float4*>(p), reinterpret_cast<float4*>(m), reinterpret_cast<float4*>(v),
        reinterpret_cast<float4*>(g), n4, alpha, omb1, omb2, eps, zero_grad, alpha_table, step_dev);
    DTB_LAUNCH_OK();
  }
  const int64_t done = n4 * 4;
  if (done < n) {
    adam_dense_kernel<<<ew_grid(n - done), 256, 0, (cudaStream_t)stream>>>(p + done, m + done, v + done, g + done,
                                                                           n - done, alpha, omb1, omb2, eps, zero_grad,
                                                                           alpha_table, step_dev);
    DTB_LAUNCH_OK();
  }
  return DTB_OK;
}

int dtb_adam_dense(float* p, float* m, float* v, float* g, int64_t n, float alpha, double beta1, double beta2,
                   float eps, int zero_grad, void* stream) {
  DTB_CHECK_ARG(p && m && v && g, "NULL argument");
  return adam_dense_impl(p, m, v, g, n, alpha, nullptr, nullptr, beta1, beta2, eps, zero_grad, stream);
}

int dtb_adam_dense_dev(float* p, float* m, float* v, float* g, int64_t n, const float* alpha_table,
                       const int32_t* step_dev, double beta1, double beta2, float eps, int zero_grad, void* stream) {
  DTB_CHECK_ARG(p && m && v && g && alpha_table && step_dev, "NULL argument");
  return adam_dense_impl(p, m, v, g, n, 0.f, alpha_table, step_dev, beta1, beta2, eps, zero_grad, stream);
}

}  // extern "C"
