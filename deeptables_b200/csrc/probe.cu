// Linear probes (deeptables_b200/probe.py): the objective and gradient of scikit-learn's lbfgs LogisticRegression
// over float32 layer features, evaluated in float64, and the predictions of the fitted probe.
//
// dtb_probe_loss_grad reads X once.  A CTA owns one fixed block of DTB_PROBE_BLOCK_ROWS rows and walks it in tiles of
// whole rows staged in shared memory by cp.async (two stages: the next tile loads while this one is used).  For each
// group of four staged rows a warp computes their K logits in float64, each W element loaded once for the four rows
// (lane l adds columns l, l+32, ... in order, then a fixed butterfly); then one thread per row computes its loss and
// residuals.  Each thread then adds r_k * x_j of every staged row, in row order, into the float64 accumulators of the
// columns it owns, kept in shared memory.  Every sum therefore runs over the block's rows in order whatever the tile
// height, so the block's partial is the same bits for any tile_rows.
// When K * (d + 1) accumulators do not fit, the gradient columns are cut into groups (gridDim.x): each group's CTA
// recomputes the logits of its block, which is the same arithmetic, and writes only its own columns.  The groups of a
// block are neighbours in the grid, so the later ones mostly find the block's rows in L2.
#include "dtb_common.cuh"

#include <cmath>

namespace dtb {

constexpr int kProbeThreads = 256;
constexpr int kProbeWarps = kProbeThreads / 32;
constexpr int kProbeAccPerThread = 56;          // float64 gradient accumulators per thread (in shared memory)
constexpr int kProbeMaxTileRows = 32;
constexpr int kProbeSmemBytes = 227 * 1024;      // the sm_90 opt-in limit per CTA

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)),
               "l"(gsrc)
               : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)),
               "l"(gsrc)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// z[r][k] = sum_j x_r[j] W[k, j] (+ W[k, d]) for the nrows (<= kLogitRows) rows x_r = x + r * ldx and k < K, written
// by lane 0 of the calling warp to z + r * K + k.  Lane l adds columns l, l+32, ... in order; the 32 lane sums meet in
// warp_sum's fixed butterfly, so a row's logits are the same bits whichever rows share the call.  Each W element
// loaded serves every row of the call.  x may be in shared or global memory.
constexpr int kLogitRows = 4;
__device__ __forceinline__ void rows_logits(const float* x, int64_t ldx, int nrows, int d, const double* __restrict__ W,
                                            int K, int fit_intercept, double* z, int lane) {
  const int ld = d + 1;
  for (int k0 = 0; k0 < K; k0 += 4) {
    const int kn = min(4, K - k0);
    double a[kLogitRows][4];
#pragma unroll
    for (int r = 0; r < kLogitRows; ++r)
#pragma unroll
      for (int q = 0; q < 4; ++q) a[r][q] = 0.0;
    const double* w0 = W + (int64_t)k0 * ld;
    for (int j = lane; j < d; j += 32) {
      double w[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) w[q] = q < kn ? __ldg(w0 + q * ld + j) : 0.0;
#pragma unroll
      for (int r = 0; r < kLogitRows; ++r) {
        if (r < nrows) {
          const double xv = (double)x[r * ldx + j];
#pragma unroll
          for (int q = 0; q < 4; ++q)
            if (q < kn) a[r][q] = fma(xv, w[q], a[r][q]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < kLogitRows; ++r) {
      if (r >= nrows) continue;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (q >= kn) continue;
        const double v = warp_sum(a[r][q]);
        if (lane == 0) z[r * K + k0 + q] = fit_intercept ? v + __ldg(w0 + q * ld + d) : v;
      }
    }
  }
}

// Loss of one row and its residuals, in place of the logits: binary (K = 1) log(1 + e^z) - y z and sigma(z) - y;
// multinomial logsumexp(z) - z_y and softmax(z) - onehot(y).
__device__ __forceinline__ double row_loss_residual(double* z, int K, int y) {
  if (K == 1) {
    const double v = z[0];
    const double yv = (double)y;
    const double loss = fmax(v, 0.0) + log1p(exp(-fabs(v))) - yv * v;
    const double p = v >= 0.0 ? 1.0 / (1.0 + exp(-v)) : exp(v) / (1.0 + exp(v));
    z[0] = p - yv;
    return loss;
  }
  double m = z[0];
  for (int k = 1; k < K; ++k) m = fmax(m, z[k]);
  double s = 0.0;
  for (int k = 0; k < K; ++k) s += exp(z[k] - m);
  const double lse = m + log(s);
  const double loss = lse - z[y];
  for (int k = 0; k < K; ++k) z[k] = exp(z[k] - lse) - (k == y ? 1.0 : 0.0);
  return loss;
}

__global__ void __launch_bounds__(kProbeThreads) probe_loss_grad_kernel(
    const float* __restrict__ X, int64_t ldx, const int32_t* __restrict__ y, const double* __restrict__ W, int64_t n,
    int d, int K, int fit_intercept, int tile_rows, int dp, int group_cols, int groups, int vec,
    double* __restrict__ partials) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int acc_cols = group_cols;                                     // columns of this CTA's group, padded
  double* acc = reinterpret_cast<double*>(smem);                       // [K][acc_cols]
  double* res = acc + (size_t)K * acc_cols;                            // [tile_rows][K] logits, then residuals
  double* rloss = res + (size_t)tile_rows * K;                         // [tile_rows]
  float* xs = reinterpret_cast<float*>(res + ((tile_rows * (K + 1) + 1) & ~1));  // [2][tile_rows][dp]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t block = blockIdx.x / groups;                           // the groups of a block run side by side
  const int g0 = (blockIdx.x - (int)(block * groups)) * group_cols;    // first gradient column of this CTA
  const int64_t r_lo = block * DTB_PROBE_BLOCK_ROWS;
  const int rows = (int)min((int64_t)DTB_PROBE_BLOCK_ROWS, n - r_lo);
  const int tiles = (rows + tile_rows - 1) / tile_rows;
  const int nvec = vec ? d / 4 : 0;                                    // 16-byte pieces of a row; the rest in 4 bytes
  const int ntail = d - 4 * nvec;

  for (int i = tid; i < K * acc_cols; i += kProbeThreads) acc[i] = 0.0;

  auto stage = [&](int t) {
    float* dst = xs + (size_t)(t & 1) * tile_rows * dp;
    const int64_t row0 = r_lo + (int64_t)t * tile_rows;
    const int nr = min(tile_rows, rows - t * tile_rows);
    for (int e = tid; e < nr * nvec; e += kProbeThreads) {
      const int i = e / nvec, c = e - i * nvec;
      cp_async16(dst + (size_t)i * dp + 4 * c, X + (row0 + i) * ldx + 4 * c);
    }
    for (int e = tid; e < nr * ntail; e += kProbeThreads) {
      const int i = e / ntail, c = 4 * nvec + (e - i * ntail);
      cp_async4(dst + (size_t)i * dp + c, X + (row0 + i) * ldx + c);
    }
    cp_async_commit();
  };

  double loss_sum = 0.0;                                               // thread 0's, rows in order
  stage(0);
  for (int t = 0; t < tiles; ++t) {
    const int nr = min(tile_rows, rows - t * tile_rows);
    if (t + 1 < tiles) {
      stage(t + 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const float* xt = xs + (size_t)(t & 1) * tile_rows * dp;
    for (int i = warp * kLogitRows; i < nr; i += kProbeWarps * kLogitRows)
      rows_logits(xt + (size_t)i * dp, dp, min(kLogitRows, nr - i), d, W, K, fit_intercept, res + (size_t)i * K, lane);
    __syncthreads();
    if (tid < nr) rloss[tid] = row_loss_residual(res + (size_t)tid * K, K, y[r_lo + (int64_t)t * tile_rows + tid]);
    __syncthreads();
    if (tid == 0 && g0 == 0)
      for (int i = 0; i < nr; ++i) loss_sum += rloss[i];
    // gradient: thread tid owns group columns c = tid, tid + 256, ...; column d is the intercept's (x = 1)
    for (int c = tid; c < acc_cols; c += kProbeThreads) {
      const int j = g0 + c;
      if (j > d || (j == d && !fit_intercept)) continue;
      for (int k0 = 0; k0 < K; k0 += 4) {
        const int kn = min(4, K - k0);
        double s0 = acc[(size_t)k0 * acc_cols + c];
        double s1 = kn > 1 ? acc[(size_t)(k0 + 1) * acc_cols + c] : 0.0;
        double s2 = kn > 2 ? acc[(size_t)(k0 + 2) * acc_cols + c] : 0.0;
        double s3 = kn > 3 ? acc[(size_t)(k0 + 3) * acc_cols + c] : 0.0;
        for (int i = 0; i < nr; ++i) {
          const double xv = j < d ? (double)xt[(size_t)i * dp + j] : 1.0;
          const double* r = res + (size_t)i * K + k0;
          s0 = fma(r[0], xv, s0);
          if (kn > 1) s1 = fma(r[1], xv, s1);
          if (kn > 2) s2 = fma(r[2], xv, s2);
          if (kn > 3) s3 = fma(r[3], xv, s3);
        }
        acc[(size_t)k0 * acc_cols + c] = s0;
        if (kn > 1) acc[(size_t)(k0 + 1) * acc_cols + c] = s1;
        if (kn > 2) acc[(size_t)(k0 + 2) * acc_cols + c] = s2;
        if (kn > 3) acc[(size_t)(k0 + 3) * acc_cols + c] = s3;
      }
    }
    __syncthreads();                                                   // the stage and res are rewritten next tile
  }
  double* out = partials + block * (1 + (int64_t)K * (d + 1));
  if (tid == 0 && g0 == 0) out[0] = loss_sum;
  for (int c = tid; c < acc_cols; c += kProbeThreads) {
    const int j = g0 + c;
    if (j > d) continue;
    for (int k = 0; k < K; ++k) out[1 + (int64_t)k * (d + 1) + j] = acc[(size_t)k * acc_cols + c];
  }
}

// out[c] = sum over blocks b = 0, 1, ... of partials[b, c], in that order.
__global__ void __launch_bounds__(kProbeThreads) probe_join_kernel(const double* __restrict__ partials,
                                                                   int64_t blocks, int width,
                                                                   double* __restrict__ out) {
  const int c = blockIdx.x * kProbeThreads + threadIdx.x;
  if (c >= width) return;
  double s = 0.0;
  int64_t b = 0;
  for (; b + 8 <= blocks; b += 8) {
    double v[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) v[q] = partials[(b + q) * width + c];
#pragma unroll
    for (int q = 0; q < 8; ++q) s += v[q];
  }
  for (; b < blocks; ++b) s += partials[b * width + c];
  out[c] = s;
}

// One warp per row: the logits, then the probabilities and the class code.
__global__ void __launch_bounds__(kProbeThreads) probe_predict_kernel(const float* __restrict__ X, int64_t ldx,
                                                                      const double* __restrict__ W, int64_t n, int d,
                                                                      int K, int fit_intercept,
                                                                      double* __restrict__ proba,
                                                                      int32_t* __restrict__ codes) {
  extern __shared__ double zbuf[];                                     // [warps][K]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* z = zbuf + (size_t)warp * K;
  const int64_t step = (int64_t)gridDim.x * kProbeWarps;
  for (int64_t r = (int64_t)blockIdx.x * kProbeWarps + warp; r < n; r += step) {
    rows_logits(X + r * ldx, ldx, 1, d, W, K, fit_intercept, z, lane);
    if (lane == 0) {
      if (K == 1) {
        const double v = z[0];
        const double p = v >= 0.0 ? 1.0 / (1.0 + exp(-v)) : exp(v) / (1.0 + exp(v));
        proba[2 * r] = 1.0 - p;
        proba[2 * r + 1] = p;
        codes[r] = v > 0.0 ? 1 : 0;
      } else {
        int arg = 0;
        double m = z[0];
        for (int k = 1; k < K; ++k)
          if (z[k] > m) { m = z[k]; arg = k; }
        double s = 0.0;
        for (int k = 0; k < K; ++k) s += exp(z[k] - m);
        for (int k = 0; k < K; ++k) proba[r * K + k] = exp(z[k] - m) / s;
        codes[r] = arg;
      }
    }
    __syncwarp();
  }
}

__global__ void __launch_bounds__(kProbeThreads) probe_correct_kernel(const int32_t* __restrict__ pred,
                                                                      const int32_t* __restrict__ truth, int64_t n,
                                                                      unsigned long long* __restrict__ count) {
  __shared__ unsigned int warp_counts[kProbeWarps];
  unsigned int c = 0;
  for (int64_t i = (int64_t)blockIdx.x * kProbeThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kProbeThreads)
    c += pred[i] == truth[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) warp_counts[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int w = 0; w < kProbeWarps; ++w) t += warp_counts[w];
    atomicAdd(count, t);
  }
}

// Shared memory of one loss_grad CTA at a given tile height.
static inline size_t probe_smem_bytes(int K, int group_cols, int tile_rows, int dp) {
  return sizeof(double) * ((size_t)K * group_cols + (((size_t)tile_rows * (K + 1) + 1) & ~(size_t)1)) +
         sizeof(float) * 2 * (size_t)tile_rows * dp;
}

static inline int probe_group_cols(int d, int K) {
  const int per_thread = K >= kProbeAccPerThread ? 1 : kProbeAccPerThread / K;  // columns per thread
  const int padded = (d + 1 + kProbeThreads - 1) / kProbeThreads;
  return kProbeThreads * min(per_thread, padded);
}

}  // namespace dtb

using namespace dtb;

extern "C" {

int dtb_probe_tile_rows(int d, int K) {
  if (d < 1 || K < 1 || K > DTB_PROBE_MAX_CLASSES) return 0;
  const int dp = (d + 3) & ~3;
  const int gc = probe_group_cols(d, K);
  for (int tr = kProbeMaxTileRows; tr >= 1; --tr)
    if (probe_smem_bytes(K, gc, tr, dp) <= (size_t)kProbeSmemBytes) return tr;
  return 0;
}

int dtb_probe_loss_grad(const float* X, int64_t ldx, const int32_t* y, const double* W, int64_t n, int d, int K,
                        int fit_intercept, int tile_rows, double* partials, void* stream) {
  DTB_CHECK_ARG(X && y && W && partials, "NULL pointer");
  DTB_CHECK_ARG(n > 0 && d > 0 && ldx >= d, "bad shape");
  DTB_CHECK_ARG(K >= 1 && K <= DTB_PROBE_MAX_CLASSES, "K out of range");
  const int most = dtb_probe_tile_rows(d, K);
  DTB_CHECK_ARG(most > 0, "a row of X does not fit in shared memory");
  DTB_CHECK_ARG(tile_rows >= 0 && tile_rows <= most, "tile_rows out of range");
  const int tr = tile_rows ? tile_rows : most;
  const int dp = (d + 3) & ~3;
  const int gc = probe_group_cols(d, K);
  const int groups = (d + 1 + gc - 1) / gc;
  const int64_t blocks = (n + DTB_PROBE_BLOCK_ROWS - 1) / DTB_PROBE_BLOCK_ROWS;
  DTB_CHECK_ARG(blocks * groups <= INT32_MAX, "too many rows");
  const int vec = ((uintptr_t)X % 16 == 0) && (ldx % 4 == 0);
  const size_t smem = probe_smem_bytes(K, gc, tr, dp);
  DTB_CUDA_OK(cudaFuncSetAttribute(probe_loss_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   kProbeSmemBytes));
  probe_loss_grad_kernel<<<(unsigned)(blocks * groups), kProbeThreads, smem, (cudaStream_t)stream>>>(
      X, ldx, y, W, n, d, K, fit_intercept, tr, dp, gc, groups, vec, partials);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_probe_join(const double* partials, int64_t blocks, int width, double* out, void* stream) {
  DTB_CHECK_ARG(partials && out, "NULL pointer");
  DTB_CHECK_ARG(blocks > 0 && width > 0, "bad shape");
  probe_join_kernel<<<ceil_div(width, kProbeThreads), kProbeThreads, 0, (cudaStream_t)stream>>>(partials, blocks,
                                                                                                 width, out);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_probe_predict(const float* X, int64_t ldx, const double* W, int64_t n, int d, int K, int fit_intercept,
                      double* proba, int32_t* codes, void* stream) {
  DTB_CHECK_ARG(X && W && proba && codes, "NULL pointer");
  DTB_CHECK_ARG(n > 0 && d > 0 && ldx >= d, "bad shape");
  DTB_CHECK_ARG(K >= 1 && K <= DTB_PROBE_MAX_CLASSES, "K out of range");
  const int64_t want = (n + kProbeWarps - 1) / kProbeWarps, cap = (int64_t)sm_count() * 16;
  probe_predict_kernel<<<(int)(want < cap ? want : cap), kProbeThreads, sizeof(double) * kProbeWarps * K,
                         (cudaStream_t)stream>>>(X, ldx, W, n, d, K, fit_intercept, proba, codes);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_probe_correct(const int32_t* pred, const int32_t* truth, int64_t n, unsigned long long* count,
                      void* stream) {
  DTB_CHECK_ARG(pred && truth && count, "NULL pointer");
  DTB_CHECK_ARG(n > 0, "bad shape");
  const int64_t want = (n + kProbeThreads - 1) / kProbeThreads, cap = (int64_t)sm_count() * 8;
  probe_correct_kernel<<<(int)(want < cap ? want : cap), kProbeThreads, 0, (cudaStream_t)stream>>>(pred, truth, n,
                                                                                                    count);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

}  // extern "C"
