// Permutation feature importance (deeptables_b200/importance.py): the per-pass permutation of one input column and
// the scores of a pass, reduced on the device into one float64 slot.
//
// A pass permutes the rows of one column.  dtb_perm_keys writes one 64-bit key per row, the row's 32-bit hash in the
// high half (sign bit flipped, so that a signed sort orders the hashes as unsigned numbers) and the row in the low
// half; sorting the keys (torch.sort, CUB) and keeping the low halves gives a uniformly random permutation that depends
// on (seed, iteration, column, rows) alone.  dtb_shuffle_column applies it to one column of a [rows, width] array.
//
// Every score is the same bits on every run: counts are integers (order-free atomics), and the float64 sums use a
// fixed grid and fixed-order trees, independent of the device's SM count.
#include <cmath>

#include "dtb_common.cuh"

namespace dtb {

constexpr int kImpThreads = 256;
constexpr int kSumBlocks = 256;           // fixed: the float64 reduction order must not depend on the device
constexpr int kMaxLabelClasses = 4096;    // per-class counters of the label metrics, in shared memory

__device__ __forceinline__ uint32_t perm_hash(uint32_t seed, uint32_t iter, uint32_t column, uint32_t row) {
  const uint64_t a = mix32(((uint64_t)seed << 32) | iter);
  const uint64_t b = mix32((a << 32) | column);
  return mix32((b << 32) | row);
}

__global__ void perm_keys_kernel(long long* __restrict__ keys, int64_t n, uint32_t seed, uint32_t iter,
                                 uint32_t column) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t h = perm_hash(seed, iter, column, (uint32_t)r) ^ 0x80000000u;
    keys[r] = (long long)((h << 32) | (uint64_t)r);
  }
}

__global__ void shuffle_column_kernel(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst,
                                      const long long* __restrict__ keys, int64_t n, int width, int column) {
  for (int64_t b = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; b < n; b += (int64_t)gridDim.x * blockDim.x) {
    const int64_t s = keys ? (int64_t)((unsigned long long)keys[b] & 0xffffffffull) : b;
    dst[b * width + column] = src[s * width + column];
  }
}

// ---- ROC AUC: Mann-Whitney rank sum with averaged tied ranks over ascending predictions --------------------------
// A tie group at sorted positions [lo, hi) has the 1-based average rank (lo + 1 + hi) / 2; twice the rank sum of the
// positives is an integer, so it is counted exactly.  sklearn's roc_auc_score computes the same quantity.
__device__ __forceinline__ int64_t lower_bound_f(const float* a, int64_t n, float v) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}
__device__ __forceinline__ int64_t upper_bound_f(const float* a, int64_t n, float v) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] <= v) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

__global__ void auc_count_kernel(const float* __restrict__ sorted, const long long* __restrict__ order,
                                 const int* __restrict__ positive, int64_t n, unsigned long long* __restrict__ acc) {
  unsigned long long rank2 = 0, npos = 0;
  int64_t cached = -1, lo = 0, hi = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (!positive[order[i]]) continue;
    const float v = sorted[i];
    if (cached < 0 || sorted[cached] != v) {
      lo = lower_bound_f(sorted, n, v);
      hi = upper_bound_f(sorted, n, v);
      cached = i;
    }
    rank2 += (unsigned long long)(lo + 1 + hi);
    ++npos;
  }
  for (int o = 16; o > 0; o >>= 1) {
    rank2 += __shfl_xor_sync(0xffffffffu, rank2, o);
    npos += __shfl_xor_sync(0xffffffffu, npos, o);
  }
  if ((threadIdx.x & 31) == 0 && npos) {
    atomicAdd(acc, rank2);
    atomicAdd(acc + 1, npos);
  }
}

__global__ void auc_finish_kernel(const unsigned long long* __restrict__ acc, int64_t n, double* __restrict__ out) {
  const double rank2 = (double)acc[0], npos = (double)acc[1], nneg = (double)n - npos;
  *out = (npos == 0.0 || nneg == 0.0) ? NAN : (rank2 - npos * (npos + 1.0)) / (2.0 * npos * nneg);
}

// ---- accuracy and F1 on predicted labels (predicted_class: dtb_common.cuh) ----------------------------------------
// counters: [0] correct rows; then per class k: [1+k] TP, [1+K+k] predicted, [1+2K+k] true
__global__ void label_count_kernel(const float* __restrict__ prob, const int* __restrict__ label, int64_t n, int cols,
                                   int classes, unsigned long long* __restrict__ acc) {
  extern __shared__ unsigned int sc[];
  const int words = 1 + 3 * classes;
  for (int i = threadIdx.x; i < words; i += blockDim.x) sc[i] = 0u;
  __syncthreads();
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const int pred = predicted_class(prob, r, cols), t = label[r];
    if (pred == t) {
      atomicAdd(sc, 1u);
      atomicAdd(sc + 1 + t, 1u);
    }
    atomicAdd(sc + 1 + classes + pred, 1u);
    atomicAdd(sc + 1 + 2 * classes + t, 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < words; i += blockDim.x)
    if (sc[i]) atomicAdd(acc + i, (unsigned long long)sc[i]);
}

// numpy's pairwise summation (np.sum / np.mean of a contiguous float64 array), so that a macro average has its bits
__device__ double numpy_pairwise_sum(const double* a, int n) {
  if (n < 8) {
    double res = 0.;
    for (int i = 0; i < n; ++i) res += a[i];
    return res;
  }
  if (n <= 128) {
    double r[8];
    for (int j = 0; j < 8; ++j) r[j] = a[j];
    int i = 8;
    for (; i < n - (n % 8); i += 8)
      for (int j = 0; j < 8; ++j) r[j] += a[i + j];
    double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) res += a[i];
    return res;
  }
  int n2 = n / 2;
  n2 -= n2 % 8;
  return numpy_pairwise_sum(a, n2) + numpy_pairwise_sum(a + n2, n - n2);
}

// sklearn's F-score of one class: 2 TP / (true + predicted), 0 when both are 0
__device__ __forceinline__ double f1_of(const unsigned long long* acc, int classes, int k) {
  const double denom = (double)acc[1 + 2 * classes + k] + (double)acc[1 + classes + k];
  return denom == 0.0 ? 0.0 : 2.0 * (double)acc[1 + k] / denom;
}

__global__ void label_finish_kernel(int metric, const unsigned long long* __restrict__ acc, int64_t n, int classes,
                                    int pos, double* __restrict__ f1s, double* __restrict__ out) {
  if (metric == DTB_IMPORTANCE_ACCURACY) {
    *out = (double)acc[0] / (double)n;
  } else if (metric == DTB_IMPORTANCE_F1) {
    *out = f1_of(acc, classes, pos);
  } else {          // macro F1 over the classes present in the labels or the predictions (sklearn's unique_labels)
    int m = 0;
    for (int k = 0; k < classes; ++k)
      if (acc[1 + 2 * classes + k] + acc[1 + classes + k]) f1s[m++] = f1_of(acc, classes, k);
    *out = numpy_pairwise_sum(f1s, m) / (double)m;
  }
}

// ---- float64 sums: log loss and the regression errors --------------------------------------------------------------
// log loss as sklearn.metrics.log_loss evaluates it on float32 probabilities: the probability of the true column
// (1 - p in float32 for column 0 of a one-column model), clipped to [eps, 1 - eps] with float32's eps, then -log,
// here in float64.
__device__ __forceinline__ double sum_term(int metric, const float* __restrict__ prob, const int* __restrict__ label,
                                           const double* __restrict__ target, int64_t r, int cols) {
  if (metric == DTB_IMPORTANCE_LOG_LOSS) {
    const float eps = 1.1920928955078125e-7f;
    float q;
    if (cols == 1) {
      const float p = prob[r];
      q = label[r] ? p : __fsub_rn(1.f, p);
    } else {
      q = prob[r * cols + label[r]];
    }
    q = fminf(fmaxf(q, eps), __fsub_rn(1.f, eps));
    return -log((double)q);
  }
  const double d = target[r] - (double)prob[r];
  return metric == DTB_IMPORTANCE_MAE ? fabs(d) : d * d;
}

__device__ __forceinline__ double block_tree_sum(double v, double* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = kImpThreads / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  return sh[0];
}

__global__ void __launch_bounds__(kImpThreads) sum_partials_kernel(int metric, const float* __restrict__ prob,
                                                                   const int* __restrict__ label,
                                                                   const double* __restrict__ target, int64_t n,
                                                                   int cols, double* __restrict__ partial) {
  __shared__ double sh[kImpThreads];
  double acc = 0.0;
  for (int64_t r = blockIdx.x * (int64_t)kImpThreads + threadIdx.x; r < n; r += (int64_t)kSumBlocks * kImpThreads)
    acc += sum_term(metric, prob, label, target, r, cols);
  const double s = block_tree_sum(acc, sh);
  if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

__global__ void __launch_bounds__(kImpThreads) sum_finish_kernel(int metric, const double* __restrict__ partial,
                                                                 int64_t n, double aux, double* __restrict__ out) {
  __shared__ double sh[kImpThreads];
  double acc = 0.0;
  for (int i = threadIdx.x; i < kSumBlocks; i += kImpThreads) acc += partial[i];
  const double s = block_tree_sum(acc, sh);
  if (threadIdx.x != 0) return;
  if (metric == DTB_IMPORTANCE_R2)   // sklearn r2_score: aux = sum (y - mean y)^2; a constant target scores 1 or 0
    *out = aux != 0.0 ? 1.0 - s / aux : (s == 0.0 ? 1.0 : 0.0);
  else if (metric == DTB_IMPORTANCE_RMSE)
    *out = sqrt(s / (double)n);
  else
    *out = s / (double)n;
}

static inline int grid_for(int64_t n) {
  const int64_t cap = (int64_t)sm_count() * 8;
  const int64_t blocks = (n + kImpThreads - 1) / kImpThreads;
  return (int)(blocks < 1 ? 1 : blocks > cap ? cap : blocks);
}

}  // namespace dtb

using namespace dtb;

extern "C" {

int dtb_perm_keys(long long* keys, int64_t rows, unsigned long long seed, int iter, int column, void* stream) {
  DTB_CHECK_ARG(keys, "NULL keys");
  DTB_CHECK_ARG(seed <= 0xffffffffull && iter >= 0 && column >= 0, "seed must fit 32 bits, iter and column >= 0");
  DTB_CHECK_ARG(rows > 0 && rows <= 0xffffffffll, "rows must be in [1, 2^32)");
  perm_keys_kernel<<<grid_for(rows), kImpThreads, 0, (cudaStream_t)stream>>>(keys, rows, (uint32_t)seed, (uint32_t)iter,
                                                                           (uint32_t)column);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_shuffle_column(const void* src, void* dst, const long long* sorted_keys, int64_t rows, int width, int column,
                       void* stream) {
  DTB_CHECK_ARG(src && dst && src != dst, "NULL or aliased src / dst");
  DTB_CHECK_ARG(rows > 0 && rows <= 0xffffffffll && width > 0 && column >= 0 && column < width, "bad shape");
  shuffle_column_kernel<<<grid_for(rows), kImpThreads, 0, (cudaStream_t)stream>>>(
      static_cast<const uint32_t*>(src), static_cast<uint32_t*>(dst), sorted_keys, rows, width, column);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_importance_auc(const float* sorted_prob, const long long* order, const int* positive, int64_t rows,
                       void* scratch, double* out, void* stream) {
  DTB_CHECK_ARG(sorted_prob && order && positive && scratch && out, "NULL argument");
  DTB_CHECK_ARG(rows > 0, "no rows");
  cudaStream_t s = (cudaStream_t)stream;
  unsigned long long* acc = static_cast<unsigned long long*>(scratch);
  DTB_CUDA_OK(cudaMemsetAsync(acc, 0, 2 * sizeof(unsigned long long), s));
  auc_count_kernel<<<grid_for(rows), kImpThreads, 0, s>>>(sorted_prob, order, positive, rows, acc);
  DTB_LAUNCH_OK();
  auc_finish_kernel<<<1, 1, 0, s>>>(acc, rows, out);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_importance_labels(int metric, const float* prob, const int* label, int64_t rows, int cols, int pos,
                          void* scratch, double* out, void* stream) {
  DTB_CHECK_ARG(prob && label && scratch && out, "NULL argument");
  DTB_CHECK_ARG(metric == DTB_IMPORTANCE_ACCURACY || metric == DTB_IMPORTANCE_F1 ||
                    metric == DTB_IMPORTANCE_F1_MACRO, "not a label metric");
  DTB_CHECK_ARG(rows > 0 && cols > 0, "bad shape");
  const int classes = cols == 1 ? 2 : cols;
  DTB_CHECK_ARG(classes <= kMaxLabelClasses, "too many classes");
  DTB_CHECK_ARG(pos >= 0 && pos < classes, "bad positive class");
  cudaStream_t s = (cudaStream_t)stream;
  const int words = 1 + 3 * classes;
  unsigned long long* acc = static_cast<unsigned long long*>(scratch);
  double* f1s = reinterpret_cast<double*>(acc + words);
  DTB_CUDA_OK(cudaMemsetAsync(acc, 0, words * sizeof(unsigned long long), s));
  label_count_kernel<<<grid_for(rows), kImpThreads, words * sizeof(unsigned int), s>>>(prob, label, rows, cols, classes,
                                                                                       acc);
  DTB_LAUNCH_OK();
  label_finish_kernel<<<1, 1, 0, s>>>(metric, acc, rows, classes, pos, f1s, out);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

size_t dtb_importance_scratch_bytes(int cols) {
  const int classes = cols == 1 ? 2 : cols;
  const size_t label_words = 1 + 4 * (size_t)classes;     // counters, then one float64 F-score per class
  return 8 * (label_words > (size_t)kSumBlocks ? label_words : (size_t)kSumBlocks);
}

int dtb_importance_sums(int metric, const float* prob, const int* label, const double* target, int64_t rows, int cols,
                        double aux, void* scratch, double* out, void* stream) {
  DTB_CHECK_ARG(prob && scratch && out, "NULL argument");
  DTB_CHECK_ARG(rows > 0 && cols > 0, "bad shape");
  if (metric == DTB_IMPORTANCE_LOG_LOSS) {
    DTB_CHECK_ARG(label, "log loss needs labels");
  } else {
    DTB_CHECK_ARG(metric == DTB_IMPORTANCE_MSE || metric == DTB_IMPORTANCE_RMSE || metric == DTB_IMPORTANCE_MAE ||
                      metric == DTB_IMPORTANCE_R2, "not a sum metric");
    DTB_CHECK_ARG(target && cols == 1, "regression metrics need a target and one column");
  }
  cudaStream_t s = (cudaStream_t)stream;
  double* partial = static_cast<double*>(scratch);
  sum_partials_kernel<<<kSumBlocks, kImpThreads, 0, s>>>(metric, prob, label, target, rows, cols, partial);
  DTB_LAUNCH_OK();
  sum_finish_kernel<<<1, kImpThreads, 0, s>>>(metric, partial, rows, aux, out);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

}  // extern "C"
