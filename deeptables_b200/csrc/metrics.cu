// Streaming metrics: keras.metrics accumulators (update_state per batch) as one device buffer of counters and sums,
// updated by ONE launch per batch for every configured metric (include/deeptables_b200.h gives the layout).
//
// One thread takes one row, the access pattern of loss_kernel (dense_bn_loss.cu): coalesced for one column, and the
// class rows of a multiclass model are a few floats.  Counts go to a per-block shared-memory copy of the counters
// with shared-memory atomics and are flushed with one 64-bit global atomic per non-zero counter.  Lanes of a warp that
// hit the same counter are combined first (__match_any_sync): an untrained model predicts ~0.5 for every row, so a
// whole warp lands in one bucket.  Integer counters make the result independent of block scheduling.  The float64 row
// sums are warp-reduced and added with atomicAdd(double), like loss_kernel's loss_sum (the per-column R2 sums through a
// per-block shared-memory copy, so a block adds each of them to global memory once): their last bits are free.
#include <cmath>

#include "dtb_common.cuh"

namespace dtb {

constexpr int kThreads = 256;
constexpr int kSmemCounters = 8192;   // counters kept per block in shared memory (32 KB); more go straight to global
constexpr int kNumSums = 7;

struct MetricArgs {
  dtb_metric_plan plan;
  int hist_off[DTB_METRIC_MAX_LISTS];   // first counter of each list's histogram
  int n_thr;                            // thresholds of all lists
  int n_counters;
  int smem_counters;                    // 1: counters live in shared memory until the block ends
  int n_r2;                             // per-block float64 R2 sums in shared memory: 3 * cols, or 0 without R2
};

static inline int counters_offset(int cols) { return 8 + 3 * cols; }   // in 8-byte words

// Fills hist_off / n_thr / n_counters; false when the plan is malformed.
static bool layout(const dtb_metric_plan* p, MetricArgs* a) {
  if (!p || p->cols < 1 || p->n_lists < 0 || p->n_lists > DTB_METRIC_MAX_LISTS) return false;
  if (p->argmax && p->top_k < 1) return false;
  a->plan = *p;
  int64_t counters = 3 + 3 * (int64_t)p->cols, thr = 0;
  for (int l = 0; l < p->n_lists; ++l) {
    if (p->list_len[l] < 1 || p->list_off[l] < 0) return false;
    a->hist_off[l] = (int)counters;
    counters += (int64_t)p->cols * 2 * (p->list_len[l] + 1);
    if (p->list_off[l] + p->list_len[l] > thr) thr = p->list_off[l] + p->list_len[l];
    if (counters > (1 << 28)) return false;
  }
  if (thr > DTB_METRIC_MAX_THRESHOLDS) return false;
  a->n_thr = (int)thr;
  a->n_counters = (int)counters;
  a->smem_counters = counters <= kSmemCounters;
  a->n_r2 = (p->sums & DTB_METRIC_SUM_R2) ? 3 * p->cols : 0;
  return true;
}

// counter[idx] += number of lanes of the warp that name it; idx < 0: the lane has nothing to count.
// Every lane of the warp calls this together.
__device__ __forceinline__ void count_add(unsigned int* sh, unsigned long long* gl, int idx) {
  const unsigned peers = __match_any_sync(0xffffffffu, idx);
  if (idx >= 0 && (int)(threadIdx.x & 31) == __ffs(peers) - 1) {
    const unsigned n = __popc(peers);
    if (sh) atomicAdd(sh + idx, n);
    else atomicAdd(gl + idx, (unsigned long long)n);
  }
}

__device__ __forceinline__ double softplus(double z) { return fmax(z, 0.0) + log1p(exp(-fabs(z))); }

__global__ void metrics_update_kernel(const float* __restrict__ prob, const float* __restrict__ y,
                                      unsigned long long* __restrict__ state, const float* __restrict__ thr, int rows,
                                      MetricArgs a) {
  extern __shared__ double smem_f64[];
  double* sr2 = smem_f64;                                    // [cols][3]: sum y, sum y^2, sum (y-p)^2 of this block
  unsigned int* smem = reinterpret_cast<unsigned int*>(smem_f64 + a.n_r2);
  float* sthr = reinterpret_cast<float*>(smem);
  unsigned int* sh = a.smem_counters ? smem + a.n_thr : nullptr;
  const int cols = a.plan.cols, sums = a.plan.sums;
  double* dsum = reinterpret_cast<double*>(state);
  unsigned long long* gl = state + 8 + 3 * cols;
  for (int i = threadIdx.x; i < a.n_thr; i += kThreads) sthr[i] = thr[i];
  for (int i = threadIdx.x; i < a.n_r2; i += kThreads) sr2[i] = 0.0;
  if (sh)
    for (int i = threadIdx.x; i < a.n_counters; i += kThreads) sh[i] = 0u;
  __syncthreads();

  const double eps = (double)1e-7f, one_m_eps = (double)(1.f - 1e-7f);
  const int lane = threadIdx.x & 31;
  double acc[kNumSums];
#pragma unroll
  for (int k = 0; k < kNumSums; ++k) acc[k] = 0.0;

  // whole warps walk the rows together: the counter updates and the R2 reductions are warp collectives
  for (int base = blockIdx.x * kThreads + threadIdx.x - lane; base < rows; base += gridDim.x * kThreads) {
    const int r = base + lane;
    const bool live = r < rows;
    const float* pr = prob + (int64_t)r * cols;
    const float* yr = y + (int64_t)r * cols;
    count_add(sh, gl, live ? 0 : -1);
    double row[kNumSums];
#pragma unroll
    for (int k = 0; k < kNumSums; ++k) row[k] = 0.0;
    float pmax = -INFINITY, ymax = -INFINITY, p_at_y = 0.f;
    double psum = 0.0;
    int p_arg = 0, y_arg = 0;
    for (int c = 0; c < cols; ++c) {
      const float p = live ? pr[c] : 0.f;
      const float t = live ? yr[c] : 0.f;
      const int label = t != 0.f;
      for (int l = 0; l < a.plan.n_lists; ++l) {
        const float* tl = sthr + a.plan.list_off[l];
        const int len = a.plan.list_len[l];
        int lo = 0, hi = len;               // thresholds strictly below p: a prefix of the ascending list
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (tl[mid] < p) lo = mid + 1;
          else hi = mid;
        }
        count_add(sh, gl, live ? a.hist_off[l] + (c * 2 + label) * (len + 1) + lo : -1);
      }
      if (sums) {
        const double pd = p, td = t, d = pd - td;
        if (sums & DTB_METRIC_SUM_SE) row[0] += d * d;
        if (sums & DTB_METRIC_SUM_AE) row[1] += fabs(d);
        if (sums & DTB_METRIC_SUM_APE) row[2] += 100.0 * fabs(d / fmax(fabs(td), eps));
        if (sums & DTB_METRIC_SUM_SLE) {
          const double e = log(fmax(pd, eps) + 1.0) - log(fmax(td, eps) + 1.0);
          row[3] += e * e;
        }
        if (sums & DTB_METRIC_SUM_LOGCOSH) row[4] += d + softplus(-2.0 * d) - 0.6931471805599453;
        if (sums & DTB_METRIC_SUM_BCE) {
          const double pc = fmin(fmax(pd, eps), one_m_eps);
          row[5] -= td * log(pc) + (1.0 - td) * log(1.0 - pc);
        }
        if (sums & DTB_METRIC_SUM_R2) {
          const double sy = warp_sum(td), syy = warp_sum(td * td), sdd = warp_sum(d * d);
          if (lane == 0) {
            atomicAdd(sr2 + 3 * c, sy);
            atomicAdd(sr2 + 3 * c + 1, syy);
            atomicAdd(sr2 + 3 * c + 2, sdd);
          }
        }
      }
      psum += (double)p;
      if (p > pmax) { pmax = p; p_arg = c; }
      if (c == 0 || t > ymax) { ymax = t; y_arg = c; p_at_y = p; }
    }
    if (sums & DTB_METRIC_SUM_CCE) {
      // keras categorical_crossentropy on probabilities: renormalise by the row sum, clip, -sum y log p
      for (int c = 0; c < cols; ++c) {
        const double q = fmin(fmax((double)(live ? pr[c] : 1.f) / psum, eps), one_m_eps);
        row[6] -= (double)(live ? yr[c] : 0.f) * log(q);
      }
    }
    if (a.plan.argmax) {
      int above = 0;
      for (int c = 0; c < cols; ++c) {
        const float p = live ? pr[c] : 0.f;
        const bool label = live && yr[c] != 0.f;
        const bool pred = p >= pmax && fabsf(p) > 1e-9f;
        above += p > p_at_y;
        count_add(sh, gl, live && pred && label ? 3 + c : -1);
        count_add(sh, gl, live && pred && !label ? 3 + cols + c : -1);
        count_add(sh, gl, live && !pred && label ? 3 + 2 * cols + c : -1);
      }
      count_add(sh, gl, live && p_arg == y_arg ? 1 : -1);
      count_add(sh, gl, live && isfinite(p_at_y) && above < a.plan.top_k ? 2 : -1);
    }
    if (live) {
#pragma unroll
      for (int k = 0; k < kNumSums - 1; ++k) acc[k] += row[k] / (double)cols;
      acc[6] += row[6];
    }
  }
#pragma unroll
  for (int k = 0; k < kNumSums; ++k) {
    if (sums & (1 << k)) {                      // uniform across the grid
      const double s = warp_sum(acc[k]);
      if (lane == 0 && s != 0.0) atomicAdd(dsum + k, s);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < a.n_r2; i += kThreads)
    if (sr2[i] != 0.0) atomicAdd(dsum + 8 + i, sr2[i]);
  if (sh) {
    for (int i = threadIdx.x; i < a.n_counters; i += kThreads) {
      const unsigned int n = sh[i];
      if (n) atomicAdd(gl + i, (unsigned long long)n);
    }
  }
}

}  // namespace dtb

using namespace dtb;

extern "C" {

size_t dtb_metrics_state_bytes(const dtb_metric_plan* plan) {
  MetricArgs a;
  if (!layout(plan, &a)) return 0;
  return 8 * ((size_t)counters_offset(plan->cols) + (size_t)a.n_counters);
}

int dtb_metrics_reset(void* state, const dtb_metric_plan* plan, void* stream) {
  MetricArgs a;
  DTB_CHECK_ARG(state, "NULL state");
  DTB_CHECK_ARG(layout(plan, &a), "bad plan");
  DTB_CUDA_OK(cudaMemsetAsync(state, 0, dtb_metrics_state_bytes(plan), (cudaStream_t)stream));
  return DTB_OK;
}

int dtb_metrics_update(const float* prob, const float* y_true, void* state, const float* thresholds_dev, int rows,
                       const dtb_metric_plan* plan, void* stream) {
  MetricArgs a;
  DTB_CHECK_ARG(prob && y_true && state, "NULL argument");
  DTB_CHECK_ARG(layout(plan, &a), "bad plan");
  DTB_CHECK_ARG(rows >= 0 && (a.n_thr == 0 || thresholds_dev), "bad rows / NULL thresholds");
  if (rows == 0) return DTB_OK;
  int blocks = ceil_div(rows, kThreads);
  const int cap = sm_count() * 8;
  if (blocks > cap) blocks = cap;
  const size_t smem = 8 * (size_t)a.n_r2 + 4 * ((size_t)a.n_thr + (a.smem_counters ? (size_t)a.n_counters : 0));
  DTB_CHECK_ARG(smem <= 48 * 1024, "too many columns for the R2 sums");
  metrics_update_kernel<<<blocks, kThreads, smem, (cudaStream_t)stream>>>(
      prob, y_true, static_cast<unsigned long long*>(state), thresholds_dev, rows, a);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

}  // extern "C"
