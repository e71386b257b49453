// Gradient-boosted trees for the leaf features of DefaultPreprocessor (deeptables_b200/gbm.py): LightGBM's gbdt at its
// sklearn defaults, restated.  The host grows each tree leaf-wise and reads one small record per split; the device bins
// the frame, computes gradients, builds histograms, searches splits, partitions rows and walks trees.
//
// Everything that decides a split is an integer or a float64 computed in a fixed order: gradients and hessians become
// int64 fixed point, histograms are integer sums (any summation order gives the same bits, so the larger child is the
// parent minus the smaller one, exactly), and the gain is evaluated with __dadd_rn / __dmul_rn / __ddiv_rn in the order
// the header writes, so no FMA contraction makes it differ from a float64 restatement.
#include "dtb_common.cuh"

namespace dtb {

constexpr int kGbdtThreads = 256;
constexpr int kHistThreads = 512;
constexpr int kHistSmemBytes = 96 * 1024;      // two histogram blocks per SM
constexpr int kSplitThreads = 256;

__device__ __forceinline__ float gbdt_value(const int32_t* __restrict__ cat, int cat_stride,
                                            const float* __restrict__ cont, int cont_stride, int col, int64_t r) {
  return col >= 0 ? __int2float_rn(cat[r * cat_stride + col]) : cont[r * cont_stride + (-1 - col)];
}

static inline int gbdt_grid(int64_t threads, int per_sm) {
  const int64_t cap = (int64_t)sm_count() * per_sm;
  const int64_t blocks = (threads + kGbdtThreads - 1) / kGbdtThreads;
  return (int)(blocks < 1 ? 1 : blocks > cap ? cap : blocks);
}

// bins[r, i] = number of edges of feature i below x (numpy's searchsorted side='left'); NaN -> the number of edges.
__global__ void __launch_bounds__(kGbdtThreads) gbdt_bin_kernel(
    const int32_t* __restrict__ cat, int cat_stride, const float* __restrict__ cont, int cont_stride,
    const int32_t* __restrict__ feat_col, const float* __restrict__ edges, const int32_t* __restrict__ edge_off,
    int64_t rows, int nf, uint8_t* __restrict__ bins) {
  const int64_t total = rows * nf;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = e / nf;
    const int i = (int)(e - r * nf);
    const float x = gbdt_value(cat, cat_stride, cont, cont_stride, feat_col[i], r);
    const float* ed = edges + edge_off[i];
    int lo = 0, hi = edge_off[i + 1] - edge_off[i];
    if (isnan(x)) {
      lo = hi;
    } else {
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (ed[mid] < x) lo = mid + 1; else hi = mid;
      }
    }
    bins[e] = (uint8_t)lo;
  }
}

__device__ __forceinline__ void atomic_max_nonneg(float* p, float v) {
  // non-negative floats order as their bit patterns
  atomicMax(reinterpret_cast<unsigned int*>(p), __float_as_uint(v));
}

__global__ void __launch_bounds__(kGbdtThreads) gbdt_grad_kernel(const double* __restrict__ scores,
                                                                 const float* __restrict__ label, int64_t rows, int K,
                                                                 int k, int objective, float* __restrict__ g,
                                                                 float* __restrict__ h, float* __restrict__ max_gh) {
  float mg = 0.f, mh = 0.f;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x) {
    const double* s = scores + r * K;
    double gd, hd;
    if (objective == DTB_GBDT_BINARY) {
      const double p = __ddiv_rn(1.0, __dadd_rn(1.0, exp(-s[0])));
      gd = __dsub_rn(p, (double)label[r]);
      hd = __dmul_rn(p, __dsub_rn(1.0, p));
    } else if (objective == DTB_GBDT_L2) {
      gd = __dsub_rn(s[0], (double)label[r]);
      hd = 1.0;
    } else {
      double m = s[0];
      for (int j = 1; j < K; ++j) m = fmax(m, s[j]);
      double sum = 0.0;
      for (int j = 0; j < K; ++j) sum = __dadd_rn(sum, exp(__dsub_rn(s[j], m)));
      const double p = __ddiv_rn(exp(__dsub_rn(s[k], m)), sum);
      gd = __dsub_rn(p, (int)label[r] == k ? 1.0 : 0.0);
      hd = __dmul_rn(__ddiv_rn((double)K, (double)(K - 1)), __dmul_rn(p, __dsub_rn(1.0, p)));
    }
    const float gf = __double2float_rn(gd), hf = __double2float_rn(hd);
    g[r] = gf;
    h[r] = hf;
    mg = fmaxf(mg, fabsf(gf));
    mh = fmaxf(mh, hf);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, o));
    mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, o));
  }
  if ((threadIdx.x & 31) == 0) {
    atomic_max_nonneg(max_gh, mg);
    atomic_max_nonneg(max_gh + 1, mh);
  }
}

__global__ void __launch_bounds__(kGbdtThreads) gbdt_fixed_kernel(const float* __restrict__ g,
                                                                  const float* __restrict__ h, int64_t rows,
                                                                  int shift_g, int shift_h, int64_t* __restrict__ gq,
                                                                  int64_t* __restrict__ hq) {
  const double sg = ldexp(1.0, shift_g), sh = ldexp(1.0, shift_h);
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x) {
    gq[r] = __double2ll_rn(__dmul_rn((double)g[r], sg));
    hq[r] = __double2ll_rn(__dmul_rn((double)h[r], sh));
  }
}

// Adds a 64-bit value held as two 32-bit cells (lo unsigned, hi two's complement) with native 32-bit shared atomics: a
// carry out of lo goes to hi.  Exact as long as the true hi sum fits in 32 bits, which the caller's fixed-point scale
// guarantees (sum of |value| over all rows below 2^62, so the hi halves sum below 2^30 plus one per row).
__device__ __forceinline__ void add_split64(unsigned* lo, unsigned* hi, unsigned long long v) {
  const unsigned l = (unsigned)v;
  const unsigned old = atomicAdd(lo, l);
  atomicAdd(hi, (unsigned)(v >> 32) + (old + l < old ? 1u : 0u));
}

// grid.y: feature group [f0, f0 + G); grid.x: slices of the segment.  Each block accumulates its rows into a shared
// histogram of the group, then adds it into the leaf's histogram with global integer atomics.
__global__ void __launch_bounds__(kHistThreads) gbdt_hist_kernel(
    const uint8_t* __restrict__ bins, const int32_t* __restrict__ index, int64_t count,
    const int64_t* __restrict__ gq, const int64_t* __restrict__ hq, int nf, int nb, int G,
    int64_t* __restrict__ hist_g, int64_t* __restrict__ hist_h, int32_t* __restrict__ hist_n) {
  extern __shared__ __align__(16) unsigned char gbdt_smem[];
  const int f0 = blockIdx.y * G;
  const int gs = min(G, nf - f0);
  const int cells = gs * nb, stride = G * nb;
  unsigned* s = reinterpret_cast<unsigned*>(gbdt_smem);     // [g lo | g hi | h lo | h hi | count], stride cells each
  for (int i = threadIdx.x; i < 5 * stride; i += blockDim.x) s[i] = 0u;
  __syncthreads();
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < count; p += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = index[p];
    const unsigned long long gv = (unsigned long long)gq[r], hv = (unsigned long long)hq[r];
    const uint8_t* br = bins + r * nf + f0;
    for (int f = 0; f < gs; ++f) {
      const int c = f * nb + br[f];
      add_split64(s + c, s + stride + c, gv);
      add_split64(s + 2 * stride + c, s + 3 * stride + c, hv);
      atomicAdd(s + 4 * stride + c, 1u);
    }
  }
  __syncthreads();
  const int64_t base = (int64_t)f0 * nb;
  for (int i = threadIdx.x; i < cells; i += blockDim.x) {
    const unsigned n = s[4 * stride + i];
    if (n == 0u) continue;
    const unsigned long long g = ((unsigned long long)s[stride + i] << 32) | s[i];
    const unsigned long long h = ((unsigned long long)s[3 * stride + i] << 32) | s[2 * stride + i];
    atomicAdd(reinterpret_cast<unsigned long long*>(hist_g + base + i), g);
    atomicAdd(reinterpret_cast<unsigned long long*>(hist_h + base + i), h);
    atomicAdd(reinterpret_cast<unsigned int*>(hist_n + base + i), n);
  }
}

__global__ void __launch_bounds__(kGbdtThreads) gbdt_hist_sub_kernel(int64_t* __restrict__ pg, int64_t* __restrict__ ph,
                                                                     int32_t* __restrict__ pn, int64_t* __restrict__ s_g,
                                                                     int64_t* __restrict__ s_h,
                                                                     int32_t* __restrict__ s_n, int64_t elements,
                                                                     int small_is_left) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < elements;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t g = pg[i] - s_g[i], h = ph[i] - s_h[i];
    const int32_t n = pn[i] - s_n[i];
    if (small_is_left) {
      pg[i] = s_g[i]; ph[i] = s_h[i]; pn[i] = s_n[i];
      s_g[i] = g; s_h[i] = h; s_n[i] = n;
    } else {
      pg[i] = g; ph[i] = h; pn[i] = n;
    }
  }
}

// T(G)^2 / (H + lambda), T the L1 soft threshold.
__device__ __forceinline__ double leaf_term(double G, double H, double l2, double l1) {
  const double t = G > l1 ? __dsub_rn(G, l1) : (G < -l1 ? __dadd_rn(G, l1) : 0.0);
  return __ddiv_rn(__dmul_rn(t, t), __dadd_rn(H, l2));
}

struct SplitBest {
  double gain;
  int feature, bin;
};

__device__ __forceinline__ bool better(const SplitBest& a, const SplitBest& b) {
  if (a.gain != b.gain) return a.gain > b.gain;
  if (a.feature != b.feature) return (unsigned)a.feature < (unsigned)b.feature;     // -1 (none) loses every tie
  return a.bin < b.bin;
}

// One block per leaf.  Thread j scans features j, j + 256, ... in order, keeping the first best candidate it meets.
__global__ void __launch_bounds__(kSplitThreads) gbdt_split_kernel(
    const int64_t* __restrict__ hist_g, const int64_t* __restrict__ hist_h, const int32_t* __restrict__ hist_n,
    const int32_t* __restrict__ leaves, const int32_t* __restrict__ n_bins, int nf, int nb,
    dtb_gbdt_split_params prm, dtb_gbdt_split_rec* __restrict__ out) {
  __shared__ unsigned long long tot[3];
  __shared__ SplitBest best[kSplitThreads];
  const int64_t base = (int64_t)leaves[blockIdx.x] * nf * nb;
  const int64_t* hg = hist_g + base;
  const int64_t* hh = hist_h + base;
  const int32_t* hn = hist_n + base;
  if (threadIdx.x < 3) tot[threadIdx.x] = 0ull;
  __syncthreads();
  for (int b = threadIdx.x; b < n_bins[0]; b += blockDim.x) {     // every row is in one bin of feature 0
    atomicAdd(&tot[0], (unsigned long long)hg[b]);
    atomicAdd(&tot[1], (unsigned long long)hh[b]);
    atomicAdd(&tot[2], (unsigned long long)hn[b]);
  }
  __syncthreads();
  const int64_t Gi = (int64_t)tot[0], Hi = (int64_t)tot[1];
  const int64_t Ni = (int64_t)tot[2];
  const double G = __dmul_rn(__ll2double_rn(Gi), prm.scale_g), H = __dmul_rn(__ll2double_rn(Hi), prm.scale_h);
  const double parent = leaf_term(G, H, prm.lambda_l2, prm.lambda_l1);
  SplitBest mine{0.0, -1, 0};
  for (int f = threadIdx.x; f < nf; f += blockDim.x) {
    int64_t gl = 0, hl = 0, nl = 0;
    const int64_t o = (int64_t)f * nb;
    for (int t = 0; t + 1 < n_bins[f]; ++t) {
      gl += hg[o + t];
      hl += hh[o + t];
      nl += hn[o + t];
      const int64_t nr = Ni - nl;
      if (nl < prm.min_child_samples || nr < prm.min_child_samples) continue;
      const double GL = __dmul_rn(__ll2double_rn(gl), prm.scale_g), HL = __dmul_rn(__ll2double_rn(hl), prm.scale_h);
      const double GR = __dmul_rn(__ll2double_rn(Gi - gl), prm.scale_g);
      const double HR = __dmul_rn(__ll2double_rn(Hi - hl), prm.scale_h);
      if (HL < prm.min_child_weight || HR < prm.min_child_weight) continue;
      const double gain = __dsub_rn(__dsub_rn(__dadd_rn(leaf_term(GL, HL, prm.lambda_l2, prm.lambda_l1),
                                                        leaf_term(GR, HR, prm.lambda_l2, prm.lambda_l1)),
                                              parent),
                                    prm.min_split_gain);
      if (gain > mine.gain) mine = SplitBest{gain, f, t};
    }
  }
  best[threadIdx.x] = mine;
  __syncthreads();
  if (threadIdx.x == 0) {
    SplitBest b = best[0];
    for (int j = 1; j < blockDim.x; ++j)
      if (better(best[j], b)) b = best[j];
    dtb_gbdt_split_rec rec;
    rec.gain = b.feature >= 0 ? b.gain : 0.0;
    rec.g = Gi;
    rec.h = Hi;
    rec.count = (int32_t)Ni;
    rec.feature = b.feature;
    rec.bin = b.feature >= 0 ? b.bin : 0;
    rec.left_g = rec.left_h = 0;
    rec.left_count = 0;
    if (b.feature >= 0) {
      const int64_t o = (int64_t)b.feature * nb;
      int64_t gl = 0, hl = 0, nl = 0;
      for (int t = 0; t <= b.bin; ++t) {
        gl += hg[o + t];
        hl += hh[o + t];
        nl += hn[o + t];
      }
      rec.left_g = gl;
      rec.left_h = hl;
      rec.left_count = (int32_t)nl;
    }
    out[blockIdx.x] = rec;
  }
}

// Left rows to scratch[0, left_count), right rows to scratch[left_count, count); counters at scratch[count .. +1].
__global__ void __launch_bounds__(kGbdtThreads) gbdt_partition_kernel(const uint8_t* __restrict__ bins, int nf,
                                                                      const int32_t* __restrict__ index,
                                                                      int64_t count, int feature, int bin,
                                                                      int64_t left_count,
                                                                      int32_t* __restrict__ scratch) {
  int32_t* counters = scratch + count;
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t base = blockIdx.x * (int64_t)blockDim.x; base < count; base += stride) {
    const int64_t p = base + threadIdx.x;
    const bool active = p < count;
    const int32_t r = active ? index[p] : 0;
    const bool left = active && bins[(int64_t)r * nf + feature] <= bin;
    const unsigned lm = __ballot_sync(0xffffffffu, left);
    const unsigned rm = __ballot_sync(0xffffffffu, active && !left);
    int lb = 0, rb = 0;
    if (lane == 0) {
      if (lm) lb = atomicAdd(counters, __popc(lm));
      if (rm) rb = atomicAdd(counters + 1, __popc(rm));
    }
    lb = __shfl_sync(0xffffffffu, lb, 0);
    rb = __shfl_sync(0xffffffffu, rb, 0);
    const unsigned below = (1u << lane) - 1u;
    if (left) scratch[lb + __popc(lm & below)] = r;
    else if (active) scratch[left_count + rb + __popc(rm & below)] = r;
  }
}

__global__ void __launch_bounds__(kGbdtThreads) gbdt_update_kernel(const int32_t* __restrict__ index,
                                                                   const int64_t* __restrict__ seg_begin,
                                                                   const int64_t* __restrict__ seg_count,
                                                                   const float* __restrict__ leaf_value,
                                                                   double* __restrict__ scores, int K, int k,
                                                                   int32_t* __restrict__ leaf_out,
                                                                   int64_t leaf_stride) {
  const int leaf = blockIdx.y;
  const int64_t b = seg_begin[leaf], c = seg_count[leaf];
  const double v = (double)leaf_value[leaf];
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < c; p += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = index[b + p];
    scores[r * K + k] += v;
    if (leaf_out) leaf_out[r * leaf_stride] = leaf;
  }
}

// Thread per row; the block stages a chunk of whole trees in shared memory, walks its rows through them, moves on.
__global__ void __launch_bounds__(kGbdtThreads) gbdt_leaves_kernel(
    const int32_t* __restrict__ cat, int cat_stride, const float* __restrict__ cont, int cont_stride,
    const int32_t* __restrict__ feat_col, const int32_t* __restrict__ node_feature,
    const float* __restrict__ node_threshold, const int32_t* __restrict__ node_left,
    const int32_t* __restrict__ node_right, const int32_t* __restrict__ node_off, int n_trees, int64_t rows,
    int32_t* __restrict__ out_cat, float* __restrict__ out_cont, int out_stride, int out_col) {
  extern __shared__ __align__(16) unsigned char gbdt_smem[];
  int32_t* s_col = reinterpret_cast<int32_t*>(gbdt_smem);      // the feature's input column, resolved once
  float* s_thr = reinterpret_cast<float*>(s_col + DTB_GBDT_STAGE_NODES);
  int32_t* s_left = reinterpret_cast<int32_t*>(s_thr + DTB_GBDT_STAGE_NODES);
  int32_t* s_right = s_left + DTB_GBDT_STAGE_NODES;
  for (int t0 = 0; t0 < n_trees;) {
    int t1 = t0;
    while (t1 < n_trees && node_off[t1 + 1] - node_off[t0] <= DTB_GBDT_STAGE_NODES) ++t1;
    if (t1 == t0) return;      // a tree larger than the stage: refused by the entry point
    const int n0 = node_off[t0], nodes = node_off[t1] - n0;
    __syncthreads();
    for (int i = threadIdx.x; i < nodes; i += blockDim.x) {
      s_col[i] = feat_col[node_feature[n0 + i]];
      s_thr[i] = node_threshold[n0 + i];
      s_left[i] = node_left[n0 + i];
      s_right[i] = node_right[n0 + i];
    }
    __syncthreads();
    for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x) {
      for (int t = t0; t < t1; ++t) {
        const int first = node_off[t] - n0, end = node_off[t + 1] - n0;
        int leaf = 0;
        if (end > first) {
          int node = 0;
          while (node >= 0) {
            const int i = first + node;
            const float x = gbdt_value(cat, cat_stride, cont, cont_stride, s_col[i], r);
            node = x <= s_thr[i] ? s_left[i] : s_right[i];
          }
          leaf = ~node;
        }
        const int64_t o = r * out_stride + out_col + t;
        if (out_cat) out_cat[o] = leaf; else out_cont[o] = (float)leaf;
      }
    }
    t0 = t1;
  }
}

static int set_smem(const void* fn, int bytes) {
  DTB_CUDA_OK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  return DTB_OK;
}

}  // namespace dtb

using namespace dtb;

extern "C" {

int dtb_gbdt_bin(const int32_t* cat, int cat_stride, const float* cont, int cont_stride, const int32_t* feat_col,
                 const float* edges, const int32_t* edge_off, int64_t rows, int nf, uint8_t* bins, void* stream) {
  DTB_CHECK_ARG(feat_col && edge_off && bins, "NULL argument");
  DTB_CHECK_ARG(rows > 0 && nf > 0, "bad shape");
  gbdt_bin_kernel<<<gbdt_grid(rows * nf, 16), kGbdtThreads, 0, (cudaStream_t)stream>>>(
      cat, cat_stride, cont, cont_stride, feat_col, edges, edge_off, rows, nf, bins);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_gbdt_grad(const double* scores, const float* label, int64_t rows, int K, int k, int objective, float* g,
                  float* h, float* max_gh, void* stream) {
  DTB_CHECK_ARG(scores && label && g && h && max_gh, "NULL argument");
  DTB_CHECK_ARG(rows > 0 && K > 0 && k >= 0 && k < K, "bad shape");
  DTB_CHECK_ARG((objective == DTB_GBDT_SOFTMAX && K > 1) ||
                    ((objective == DTB_GBDT_BINARY || objective == DTB_GBDT_L2) && K == 1),
                "objective must be BINARY or L2 on one score column, SOFTMAX on several");
  gbdt_grad_kernel<<<gbdt_grid(rows, 8), kGbdtThreads, 0, (cudaStream_t)stream>>>(scores, label, rows, K, k,
                                                                                   objective, g, h, max_gh);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_gbdt_fixed(const float* g, const float* h, int64_t rows, int shift_g, int shift_h, int64_t* gq, int64_t* hq,
                   void* stream) {
  DTB_CHECK_ARG(g && h && gq && hq, "NULL argument");
  DTB_CHECK_ARG(rows > 0 && shift_g > -1000 && shift_g < 1000 && shift_h > -1000 && shift_h < 1000, "bad shape");
  gbdt_fixed_kernel<<<gbdt_grid(rows, 8), kGbdtThreads, 0, (cudaStream_t)stream>>>(g, h, rows, shift_g, shift_h, gq,
                                                                                    hq);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_gbdt_hist(const uint8_t* bins, const int32_t* index, int64_t begin, int64_t count, const int64_t* gq,
                  const int64_t* hq, int nf, int nb, int64_t* hist_g, int64_t* hist_h, int32_t* hist_n,
                  void* stream) {
  DTB_CHECK_ARG(bins && index && gq && hq && hist_g && hist_h && hist_n, "NULL argument");
  DTB_CHECK_ARG(begin >= 0 && count >= 0 && nf > 0 && nb > 0 && nb <= 256, "bad shape");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t cells = (size_t)nf * nb;
  DTB_CUDA_OK(cudaMemsetAsync(hist_g, 0, cells * sizeof(int64_t), s));
  DTB_CUDA_OK(cudaMemsetAsync(hist_h, 0, cells * sizeof(int64_t), s));
  DTB_CUDA_OK(cudaMemsetAsync(hist_n, 0, cells * sizeof(int32_t), s));
  if (count == 0) return DTB_OK;
  const int per_feature = nb * 5 * (int)sizeof(unsigned);
  const int gmax = kHistSmemBytes / per_feature;
  const int groups = (nf + gmax - 1) / gmax;
  const int G = (nf + groups - 1) / groups;
  const int smem = G * per_feature;
  static bool configured = false;
  if (!configured) {
    if (set_smem((const void*)gbdt_hist_kernel, kHistSmemBytes) != DTB_OK) return DTB_ERR_CUDA;
    configured = true;
  }
  const int64_t want = (count + 4 * kHistThreads - 1) / (4 * kHistThreads);
  const int64_t cap = ((int64_t)sm_count() * 4 + groups - 1) / groups;
  const dim3 grid((unsigned)(want < cap ? want : cap), (unsigned)groups);
  gbdt_hist_kernel<<<grid, kHistThreads, smem, s>>>(bins, index + begin, count, gq, hq, nf, nb, G, hist_g, hist_h,
                                                    hist_n);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_gbdt_hist_sub(int64_t* parent_g, int64_t* parent_h, int32_t* parent_n, int64_t* small_g, int64_t* small_h,
                      int32_t* small_n, int64_t elements, int small_is_left, void* stream) {
  DTB_CHECK_ARG(parent_g && parent_h && parent_n && small_g && small_h && small_n, "NULL argument");
  DTB_CHECK_ARG(elements > 0, "bad shape");
  gbdt_hist_sub_kernel<<<gbdt_grid(elements, 8), kGbdtThreads, 0, (cudaStream_t)stream>>>(
      parent_g, parent_h, parent_n, small_g, small_h, small_n, elements, small_is_left);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_gbdt_split(const int64_t* hist_g, const int64_t* hist_h, const int32_t* hist_n, const int32_t* leaves,
                   int n_leaves, const int32_t* n_bins, int nf, int nb, const dtb_gbdt_split_params* params_host,
                   dtb_gbdt_split_rec* out, void* stream) {
  DTB_CHECK_ARG(hist_g && hist_h && hist_n && leaves && n_bins && params_host && out, "NULL argument");
  DTB_CHECK_ARG(n_leaves > 0 && nf > 0 && nb > 0 && nb <= 256, "bad shape");
  gbdt_split_kernel<<<n_leaves, kSplitThreads, 0, (cudaStream_t)stream>>>(hist_g, hist_h, hist_n, leaves, n_bins, nf,
                                                                          nb, *params_host, out);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_gbdt_partition(const uint8_t* bins, int nf, int32_t* index, int64_t begin, int64_t count, int feature,
                       int bin, int64_t left_count, int32_t* scratch, void* stream) {
  DTB_CHECK_ARG(bins && index && scratch, "NULL argument");
  DTB_CHECK_ARG(nf > 0 && feature >= 0 && feature < nf && begin >= 0 && count > 0 && left_count >= 0 &&
                    left_count <= count && count < (1ll << 31),
                "bad shape");
  cudaStream_t s = (cudaStream_t)stream;
  DTB_CUDA_OK(cudaMemsetAsync(scratch + count, 0, 2 * sizeof(int32_t), s));
  gbdt_partition_kernel<<<gbdt_grid(count, 8), kGbdtThreads, 0, s>>>(bins, nf, index + begin, count, feature, bin,
                                                                      left_count, scratch);
  DTB_LAUNCH_OK();
  DTB_CUDA_OK(cudaMemcpyAsync(index + begin, scratch, count * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
  return DTB_OK;
}

int dtb_gbdt_update(const int32_t* index, const int64_t* seg_begin, const int64_t* seg_count, int n_leaves,
                    int64_t max_count, const float* leaf_value, double* scores, int K, int k, int32_t* leaf_out,
                    int64_t leaf_stride, void* stream) {
  DTB_CHECK_ARG(index && seg_begin && seg_count && leaf_value && scores, "NULL argument");
  DTB_CHECK_ARG(n_leaves > 0 && n_leaves <= 65535 && max_count > 0 && K > 0 && k >= 0 && k < K, "bad shape");
  const int64_t want = (max_count + kGbdtThreads - 1) / kGbdtThreads;
  const int64_t cap = ((int64_t)sm_count() * 16 + n_leaves - 1) / n_leaves;
  const dim3 grid((unsigned)(want < cap ? want : cap), (unsigned)n_leaves);
  gbdt_update_kernel<<<grid, kGbdtThreads, 0, (cudaStream_t)stream>>>(index, seg_begin, seg_count, leaf_value, scores,
                                                                       K, k, leaf_out, leaf_stride);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_gbdt_leaves(const int32_t* cat, int cat_stride, const float* cont, int cont_stride, const int32_t* feat_col,
                    const int32_t* node_feature, const float* node_threshold, const int32_t* node_left,
                    const int32_t* node_right, const int32_t* node_off, int n_trees, int max_tree_nodes,
                    int64_t rows, int32_t* out_cat, float* out_cont, int out_stride, int out_col, void* stream) {
  DTB_CHECK_ARG(feat_col && node_off && (out_cat || out_cont), "NULL argument");
  DTB_CHECK_ARG(rows > 0 && n_trees > 0 && out_col >= 0 && out_col + n_trees <= out_stride, "bad shape");
  DTB_CHECK_ARG(max_tree_nodes >= 0 && max_tree_nodes <= DTB_GBDT_STAGE_NODES,
                "a tree has more than DTB_GBDT_STAGE_NODES nodes");
  const int smem = DTB_GBDT_STAGE_NODES * 16;
  static bool configured = false;
  if (!configured) {
    if (set_smem((const void*)gbdt_leaves_kernel, smem) != DTB_OK) return DTB_ERR_CUDA;
    configured = true;
  }
  gbdt_leaves_kernel<<<gbdt_grid(rows, 6), kGbdtThreads, smem, (cudaStream_t)stream>>>(
      cat, cat_stride, cont, cont_stride, feat_col, node_feature, node_threshold, node_left, node_right, node_off,
      n_trees, rows, out_cat, out_cont, out_stride, out_col);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

}  // extern "C"
