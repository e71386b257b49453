// Quantile-bin codes of the continuous columns for DefaultPreprocessor's auto_discrete (deeptables_b200/discrete.py):
// scikit-learn's KBinsDiscretizer(encode='ordinal').transform, np.searchsorted(bin_edges[1:-1], x, side='right'), on
// the model's own float32 inputs, with the edges and the comparison in float64.
#include "dtb_common.cuh"

namespace dtb {

constexpr int kDiscreteThreads = 256;

// One thread per (row, column), columns fastest: a warp reads neighbouring floats of a few rows and writes neighbouring
// codes.  The search reads the edges from global memory through the read-only path.  Its first levels are the same few
// addresses for every row of a column and stay in L1; the deeper levels come from L2 (13 columns of 10^5 float64 edges
// are 10 MB).  Ties go to the upper bin (e <= x), and -0.0 == 0.0 as float64 comparisons give.
__global__ void __launch_bounds__(kDiscreteThreads) discretize_kernel(
    const float* __restrict__ cont, int cont_stride, int64_t rows, const int32_t* __restrict__ src_col,
    const double* __restrict__ edges, const int64_t* __restrict__ edge_off, int n_cols, int32_t* __restrict__ out_cat,
    int out_stride, int out_col) {
  const int64_t total = rows * n_cols;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = e / n_cols;
    const int j = (int)(e - r * n_cols);
    const double x = (double)cont[r * cont_stride + src_col[j]];
    const int64_t begin = edge_off[j];
    const double* ed = edges + begin;
    int64_t lo = 0, len = edge_off[j + 1] - begin;
    while (len > 0) {                 // upper bound: lo = the number of edges <= x
      const int64_t half = len >> 1;
      if (__ldg(ed + lo + half) <= x) {
        lo += half + 1;
        len -= half + 1;
      } else {
        len = half;
      }
    }
    out_cat[r * out_stride + out_col + j] = (int32_t)lo;
  }
}

}  // namespace dtb

using namespace dtb;

extern "C" {

int dtb_discretize(const float* cont, int cont_stride, int64_t rows, const int32_t* src_col, const double* edges,
                   const int64_t* edge_off, int n_cols, int32_t* out_cat, int out_stride, int out_col, void* stream) {
  DTB_CHECK_ARG(cont && src_col && edges && edge_off && out_cat, "NULL argument");
  DTB_CHECK_ARG(rows > 0 && n_cols > 0 && cont_stride > 0 && out_stride > 0 && out_col >= 0 &&
                    (int64_t)out_col + n_cols <= out_stride,
                "bad shape");
  const int64_t blocks = (rows * n_cols + kDiscreteThreads - 1) / kDiscreteThreads;
  const int64_t cap = (int64_t)sm_count() * 8;
  discretize_kernel<<<(unsigned)(blocks < cap ? blocks : cap), kDiscreteThreads, 0, (cudaStream_t)stream>>>(
      cont, cont_stride, rows, src_col, edges, edge_off, n_cols, out_cat, out_stride, out_col);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

}  // extern "C"
