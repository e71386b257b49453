// Target encoding (deeptables_b200/target_encoding.py): per-category target statistics of each cross-fitting fold and
// the encodings built from them.
//
// Each column's rows are sorted (stably) by the key (code * folds + fold) * classes + class, so every (category, fold)
// -- and for class targets every (category, fold, class) -- is one contiguous segment of the sorted order.  Counts are
// segment lengths (dtb_te_segment_starts).  Float sums of a continuous target are reduced per segment in chunks of
// kTeChunk rows counted from the segment's start: one warp per chunk, lane l adding rows l, l+32, ... in order, then a
// fixed butterfly (dtb_te_segment_stats); the chunks are then added in order (dtb_te_segment_join).  A category holding
// half of the rows is reduced by many warps at once, no value is added by an atomic, and the bits depend only on the
// data, not on the tile size or on which other columns share a launch.
#include <math.h>
#include "dtb_common.cuh"

namespace dtb {

constexpr int kTeThreads = 256;
constexpr int kTeChunk = DTB_TE_CHUNK;
static_assert((kTeChunk & (kTeChunk - 1)) == 0, "the chunk is a power of two");
constexpr int kTeMinSamplesLeaf = 20;

static inline int te_grid(int64_t threads) {
  const int64_t cap = (int64_t)sm_count() * 32;
  const int64_t blocks = (threads + kTeThreads - 1) / kTeThreads;
  return (int)(blocks < 1 ? 1 : blocks > cap ? cap : blocks);
}

__global__ void __launch_bounds__(kTeThreads) te_remap_kernel(const int64_t* __restrict__ in,
                                                              const int32_t* __restrict__ map, int64_t n, int map_len,
                                                              int32_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)kTeThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kTeThreads) {
    const int64_t c = in[i];
    out[i] = (c >= 0 && c < map_len) ? map[c] : -1;
  }
}

__global__ void __launch_bounds__(kTeThreads) te_keys_kernel(const int32_t* __restrict__ codes,
                                                             const uint8_t* __restrict__ fold,
                                                             const int32_t* __restrict__ cls, int64_t n, int folds,
                                                             int classes, int unknown_code,
                                                             int64_t* __restrict__ keys) {
  const int c_mul = classes > 0 ? classes : 1;
  for (int64_t i = blockIdx.x * (int64_t)kTeThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kTeThreads) {
    int64_t c = codes ? (int64_t)codes[i] : 0;
    if (c < 0) c = unknown_code;
    const int k = fold ? (int)fold[i] : 0;
    const int j = classes > 0 ? cls[i] : 0;
    keys[i] = c < 0 ? -1 : (c * folds + k) * c_mul + j;
  }
}

// Position i (0 <= i <= n) starts every slot in (keys[i-1], keys[i]]: each slot is written by exactly one thread.
__global__ void __launch_bounds__(kTeThreads) te_starts_kernel(const int64_t* __restrict__ keys, int64_t n,
                                                               int64_t slots, int64_t* __restrict__ starts) {
  for (int64_t i = blockIdx.x * (int64_t)kTeThreads + threadIdx.x; i <= n; i += (int64_t)gridDim.x * kTeThreads) {
    const int64_t prev = i > 0 ? max(keys[i - 1], (int64_t)-1) : (int64_t)-1;
    const int64_t cur = i < n ? keys[i] : slots;
    for (int64_t s = prev + 1; s <= cur; ++s) starts[s] = i;
  }
}

// One CTA per tile of tile_rows sorted positions; its warps take the tile's 32-position blocks in turn and reduce every
// chunk that starts in them.  A chunk may run past the tile: the tile only decides who does the work.
__global__ void __launch_bounds__(kTeThreads) te_stats_kernel(const int64_t* __restrict__ keys,
                                                              const int64_t* __restrict__ perm,
                                                              const double* __restrict__ y,
                                                              const int64_t* __restrict__ starts,
                                                              const double* __restrict__ seg_sum, int64_t n,
                                                              int tile_rows, double* __restrict__ partial) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t lo = (int64_t)blockIdx.x * tile_rows;
  const int64_t hi = min(lo + tile_rows, n);
  for (int64_t base = lo + 32 * warp; base < hi; base += kTeThreads) {
    const int64_t p = base + lane;
    bool head = false;
    if (p < hi) {
      const int64_t s = keys[p];
      head = s >= 0 && ((uint64_t)(p - starts[s]) & (kTeChunk - 1)) == 0;
    }
    unsigned heads = __ballot_sync(0xffffffffu, head);
    while (heads) {
      const int b = __ffs(heads) - 1;
      heads &= heads - 1;
      const int64_t q = base + b;
      const int64_t s = keys[q];
      const int64_t seg_end = starts[s + 1];
      const int64_t end = min(q + kTeChunk, seg_end);
      double center = 0.0;
      if (seg_sum) center = seg_sum[s] / (double)(seg_end - starts[s]);
      double acc = 0.0;
      for (int64_t r = q + lane; r < end; r += 32) {
        const double v = y[perm[r]];
        if (seg_sum) {
          const double d = v - center;
          acc = __dadd_rn(acc, __dmul_rn(d, d));
        } else {
          acc += v;
        }
      }
      acc = warp_sum(acc);
      if (lane == 0) partial[q] = acc;
    }
  }
}

__global__ void __launch_bounds__(kTeThreads) te_join_kernel(const int64_t* __restrict__ starts,
                                                             const double* __restrict__ partial, int64_t slots,
                                                             double* __restrict__ out) {
  for (int64_t s = blockIdx.x * (int64_t)kTeThreads + threadIdx.x; s < slots; s += (int64_t)gridDim.x * kTeThreads) {
    const int64_t b = starts[s], e = starts[s + 1];
    double acc = 0.0;
    for (int64_t q = b; q < e; q += kTeChunk) acc += partial[q];
    out[s] = acc;
  }
}

// Rows and target sum of (category v, fold k): a class target's sum is the number of rows of class j; a continuous
// target's is the joined chunk sums.
struct TeStats {
  const int64_t* starts;
  const double* sums;
  const double* m2;
  int folds, classes;

  __device__ __forceinline__ double count(int64_t v, int k) const {
    const int c = classes > 0 ? classes : 1;
    const int64_t s = (v * folds + k) * c;
    return (double)(starts[s + c] - starts[s]);
  }
  __device__ __forceinline__ double sum(int64_t v, int k, int j) const {
    if (classes == 0) return sums[v * folds + k];
    const int64_t s = (v * folds + k) * classes + j;
    return (double)(starts[s + 1] - starts[s]);
  }
};

// Group g: g = 0 is every fold, g = 1 + f every fold but f (only when folds > 1).
__device__ __forceinline__ bool te_in_group(int g, int k) { return g == 0 || k != g - 1; }

// n, S and the sum of squared differences from the group mean S / n of category v over the folds of group g, each
// added in increasing fold order.  Class targets: the squares of an indicator's differences have the closed form
// S (1 - m)^2 + (n - S) m^2.  Continuous targets: the per-fold sums of squares around the fold's own mean, plus
// n_k (mean_k - m)^2 for each fold.
__device__ void te_group_stats(const TeStats& st, int64_t v, int g, int j, bool want_ssd, double& n, double& S,
                               double& ssd) {
  n = 0.0;
  S = 0.0;
  for (int k = 0; k < st.folds; ++k)
    if (te_in_group(g, k)) {
      n += st.count(v, k);
      S += st.sum(v, k, j);
    }
  ssd = 0.0;
  if (!want_ssd) return;
  const double m = S / n;
  if (st.classes > 0) {
    const double a = 1.0 - m;
    ssd = __dadd_rn(__dmul_rn(S, __dmul_rn(a, a)), __dmul_rn(n - S, __dmul_rn(m, m)));
    return;
  }
  for (int k = 0; k < st.folds; ++k) {
    if (!te_in_group(g, k)) continue;
    const double nk = st.count(v, k);
    if (nk == 0.0) continue;
    const double d = st.sums[v * st.folds + k] / nk - m;
    ssd += __dadd_rn(st.m2[v * st.folds + k], __dmul_rn(nk, __dmul_rn(d, d)));
  }
}

__global__ void __launch_bounds__(kTeThreads) te_encodings_kernel(TeStats st, TeStats pst, int64_t cats, int groups,
                                                                  int n_out, int formula, double smooth,
                                                                  double* __restrict__ table,
                                                                  double* __restrict__ prior) {
  const int64_t items = (int64_t)groups * (cats + 1) * n_out;
  for (int64_t it = blockIdx.x * (int64_t)kTeThreads + threadIdx.x; it < items;
       it += (int64_t)gridDim.x * kTeThreads) {
    const int j = (int)(it % n_out);
    const int64_t gv = it / n_out;
    const int64_t v = gv % (cats + 1);
    const int g = (int)(gv / (cats + 1));
    // the class whose indicator output j encodes: class 1 of a binary target, class j of a multiclass one
    const int cj = st.classes > 2 ? j : 1;
    const bool is_auto = formula == DTB_TE_AUTO;
    double pn, pS, pssd;
    te_group_stats(pst, 0, g, cj, is_auto, pn, pS, pssd);
    const double mu = pS / pn;
    if (v == cats) {
      if (prior) prior[(int64_t)g * n_out + j] = mu;
      continue;
    }
    double n, S, ssd;
    te_group_stats(st, v, g, cj, is_auto, n, S, ssd);
    double enc;
    if (formula == DTB_TE_SMOOTH) {
      const double den = smooth + n;
      enc = den == 0.0 ? mu : (smooth * mu + S) / den;
    } else if (formula == DTB_TE_AUTO) {
      const double var = pssd / pn;
      const double lam = var * n / (var * n + ssd / n);
      enc = isnan(lam) ? mu : lam * (S / n) + (1.0 - lam) * mu;
    } else {
      const double s = 1.0 / (1.0 + exp(-(n - kTeMinSamplesLeaf) / smooth));
      enc = n == 0.0 ? mu : mu * (1.0 - s) + (S / n) * s;
    }
    table[((int64_t)g * cats + v) * n_out + j] = enc;
  }
}

__global__ void __launch_bounds__(kTeThreads) te_gather_kernel(const int32_t* __restrict__ codes,
                                                               const uint8_t* __restrict__ fold,
                                                               const double* __restrict__ table,
                                                               const int64_t* __restrict__ table_off,
                                                               const int32_t* __restrict__ cats,
                                                               const double* __restrict__ prior, int64_t n, int cols,
                                                               int n_out, int unknown_group, int out_stride,
                                                               double* __restrict__ out) {
  const int64_t per_row = (int64_t)cols * n_out;
  for (int64_t it = blockIdx.x * (int64_t)kTeThreads + threadIdx.x; it < n * per_row;
       it += (int64_t)gridDim.x * kTeThreads) {
    const int64_t r = it / per_row;
    const int cj = (int)(it - r * per_row);
    const int c = cj / n_out, j = cj - c * n_out;
    const int g = fold ? 1 + fold[r] : 0;
    const int32_t code = codes[(int64_t)c * n + r];
    const int32_t V = cats[c];
    double v;
    if (code < 0) v = prior[(int64_t)(unknown_group >= 0 ? unknown_group : g) * n_out + j];
    else if (code < V) v = table[table_off[c] + ((int64_t)g * V + code) * n_out + j];
    else v = nan("");
    out[r * out_stride + cj] = v;
  }
}

}  // namespace dtb

using namespace dtb;

extern "C" {

int dtb_te_remap(const int64_t* in, const int32_t* map, int64_t n, int map_len, int32_t* out, void* stream) {
  DTB_CHECK_ARG(in && out && (map || map_len == 0), "NULL pointer");
  DTB_CHECK_ARG(n >= 0 && map_len >= 0, "bad shape");
  if (n == 0) return DTB_OK;
  te_remap_kernel<<<te_grid(n), kTeThreads, 0, (cudaStream_t)stream>>>(in, map, n, map_len, out);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_te_keys(const int32_t* codes, const uint8_t* fold, const int32_t* cls, int64_t n, int folds, int classes,
                int unknown_code, int64_t* keys, void* stream) {
  DTB_CHECK_ARG(keys && (classes == 0 || cls), "NULL keys or cls");
  DTB_CHECK_ARG(n >= 0 && folds >= 1 && folds <= 255 && classes >= 0 && unknown_code >= -1, "bad shape");
  if (n == 0) return DTB_OK;
  te_keys_kernel<<<te_grid(n), kTeThreads, 0, (cudaStream_t)stream>>>(codes, fold, cls, n, folds, classes,
                                                                      unknown_code, keys);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_te_segment_starts(const int64_t* keys, int64_t n, int64_t slots, int64_t* starts, void* stream) {
  DTB_CHECK_ARG(starts && (keys || n == 0), "NULL pointer");
  DTB_CHECK_ARG(n >= 0 && slots >= 0, "bad shape");
  te_starts_kernel<<<te_grid(n + 1), kTeThreads, 0, (cudaStream_t)stream>>>(keys, n, slots, starts);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_te_segment_stats(const int64_t* keys, const int64_t* perm, const double* y, const int64_t* starts,
                         const double* seg_sum, int64_t n, int tile_rows, double* partial, void* stream) {
  DTB_CHECK_ARG(keys && perm && y && starts && partial, "NULL pointer");
  DTB_CHECK_ARG(n >= 0 && tile_rows >= 32 && tile_rows % 32 == 0, "bad shape");
  if (n == 0) return DTB_OK;
  const int64_t tiles = (n + tile_rows - 1) / tile_rows;
  DTB_CHECK_ARG(tiles <= INT32_MAX, "too many tiles");
  te_stats_kernel<<<(int)tiles, kTeThreads, 0, (cudaStream_t)stream>>>(keys, perm, y, starts, seg_sum, n, tile_rows,
                                                                       partial);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_te_segment_join(const int64_t* starts, const double* partial, int64_t slots, double* out, void* stream) {
  DTB_CHECK_ARG(starts && partial && out, "NULL pointer");
  DTB_CHECK_ARG(slots >= 0, "bad shape");
  if (slots == 0) return DTB_OK;
  te_join_kernel<<<te_grid(slots), kTeThreads, 0, (cudaStream_t)stream>>>(starts, partial, slots, out);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_te_encodings(const int64_t* starts, const double* sums, const double* m2, const int64_t* p_starts,
                     const double* p_sums, const double* p_m2, int64_t cats, int folds, int classes, int formula,
                     double smooth, double* table, double* prior, void* stream) {
  DTB_CHECK_ARG(starts && p_starts && table, "NULL pointer");
  DTB_CHECK_ARG(classes > 0 || (sums && p_sums), "continuous target without sums");
  DTB_CHECK_ARG(classes > 0 || formula != DTB_TE_AUTO || (m2 && p_m2), "auto smoothing without sums of squares");
  DTB_CHECK_ARG(cats >= 0 && folds >= 1 && folds <= 255 && classes >= 0 && classes != 1, "bad shape");
  DTB_CHECK_ARG(formula == DTB_TE_SMOOTH || formula == DTB_TE_AUTO || formula == DTB_TE_RECALLED, "bad formula");
  DTB_CHECK_ARG(formula == DTB_TE_AUTO || smooth >= 0.0, "negative smooth");
  const int groups = folds > 1 ? folds + 1 : 1;
  const int n_out = classes > 2 ? classes : 1;
  const TeStats st{starts, sums, m2, folds, classes};
  const TeStats pst{p_starts, p_sums, p_m2, folds, classes};
  te_encodings_kernel<<<te_grid((int64_t)groups * (cats + 1) * n_out), kTeThreads, 0, (cudaStream_t)stream>>>(
      st, pst, cats, groups, n_out, formula, smooth, table, prior);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_te_gather(const int32_t* codes, const uint8_t* fold, const double* table, const int64_t* table_off,
                  const int32_t* cats, const double* prior, int64_t n, int cols, int n_out, int unknown_group,
                  int out_stride, double* out, void* stream) {
  DTB_CHECK_ARG(codes && table && table_off && cats && prior && out, "NULL pointer");
  DTB_CHECK_ARG(n >= 0 && cols >= 1 && n_out >= 1 && out_stride >= cols * n_out && unknown_group >= -1, "bad shape");
  if (n == 0) return DTB_OK;
  te_gather_kernel<<<te_grid(n * cols * n_out), kTeThreads, 0, (cudaStream_t)stream>>>(
      codes, fold, table, table_off, cats, prior, n, cols, n_out, unknown_group, out_stride, out);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

}  // extern "C"
