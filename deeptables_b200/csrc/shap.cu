// Kernel SHAP (deeptables_b200/explain.py, utils/shap.py): the synthetic rows of a range of coalitions, and the mean
// of the model function over each coalition's rows.
//
// A coalition k is a bit mask over the varying columns of one explained row x (x_index[k]).  Its N synthetic rows are
// the N background rows with every encoded column whose bit is set in mask k replaced by x's value; row k*N + j is
// background row j.  An encoded column that does not vary for the row has bit -1 and always keeps the background's
// value.  DefaultPreprocessor encodes each cell on its own, so composing encoded columns is composing raw ones.
//
// The means are float64 sums over a coalition's rows in a fixed order (one warp per coalition, a fixed lane stride and
// a fixed butterfly), so they are the same bits on every run and every device.
#include "dtb_common.cuh"

namespace dtb {

constexpr int kShapThreads = 256;

__device__ __forceinline__ bool takes_x(const uint32_t* __restrict__ mask, int bit) {
  return bit >= 0 && ((mask[bit >> 5] >> (bit & 31)) & 1u);
}

// One thread per output element: elements [0, rows*F) are ids, [rows*F, rows*(F+C)) continuous values.
__global__ void __launch_bounds__(kShapThreads) shap_compose_kernel(
    const int32_t* __restrict__ x_cat, const float* __restrict__ x_cont, const int32_t* __restrict__ bg_cat,
    const float* __restrict__ bg_cont, const uint32_t* __restrict__ masks, int words,
    const int32_t* __restrict__ x_index, const int32_t* __restrict__ cat_bit, const int32_t* __restrict__ cont_bit,
    int64_t rows, int bg_rows, int fields, int conts, int32_t* __restrict__ out_cat, float* __restrict__ out_cont) {
  const int64_t n_cat = rows * fields, total = n_cat + rows * conts;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    if (e < n_cat) {
      const int64_t r = e / fields;
      const int f = (int)(e - r * fields);
      const int64_t k = r / bg_rows;
      const int j = (int)(r - k * bg_rows);
      out_cat[e] = takes_x(masks + k * words, cat_bit[f]) ? x_cat[(int64_t)x_index[k] * fields + f]
                                                          : bg_cat[(int64_t)j * fields + f];
    } else {
      const int64_t i = e - n_cat, r = i / conts;
      const int c = (int)(i - r * conts);
      const int64_t k = r / bg_rows;
      const int j = (int)(r - k * bg_rows);
      out_cont[i] = takes_x(masks + k * words, cont_bit[c]) ? x_cont[(int64_t)x_index[k] * conts + c]
                                                            : bg_cont[(int64_t)j * conts + c];
    }
  }
}

// The model function of one output row: the prediction itself, or DeepTable.predict's class code.
__device__ __forceinline__ double model_value(const float* __restrict__ prob, int64_t r, int cols, int kind) {
  return kind == DTB_SHAP_VALUE ? (double)prob[r] : (double)predicted_class(prob, r, cols);
}

// One warp per group: lane l sums rows l, l+32, ... in order, then a fixed butterfly.
__global__ void __launch_bounds__(kShapThreads) shap_means_kernel(const float* __restrict__ prob, int64_t groups,
                                                                  int n, int cols, int kind, double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (kShapThreads / 32);
  for (int64_t g = blockIdx.x * (int64_t)(kShapThreads / 32) + (threadIdx.x >> 5); g < groups; g += warps) {
    double acc = 0.0;
    for (int j = lane; j < n; j += 32) acc += model_value(prob, g * n + j, cols, kind);
    acc = warp_sum(acc);
    if (lane == 0) out[g] = acc / (double)n;
  }
}

static inline int grid_for(int64_t threads) {
  const int64_t cap = (int64_t)sm_count() * 16;
  const int64_t blocks = (threads + kShapThreads - 1) / kShapThreads;
  return (int)(blocks < 1 ? 1 : blocks > cap ? cap : blocks);
}

}  // namespace dtb

using namespace dtb;

extern "C" {

int dtb_shap_compose(const int32_t* x_cat, const float* x_cont, const int32_t* bg_cat, const float* bg_cont,
                     const uint32_t* masks, int mask_words, const int32_t* x_index, const int32_t* cat_bit,
                     const int32_t* cont_bit, int64_t coalitions, int bg_rows, int fields, int conts,
                     int32_t* out_cat, float* out_cont, void* stream) {
  DTB_CHECK_ARG(masks && x_index, "NULL masks or x_index");
  DTB_CHECK_ARG(coalitions > 0 && bg_rows > 0 && mask_words > 0 && fields >= 0 && conts >= 0 && fields + conts > 0,
                "bad shape");
  DTB_CHECK_ARG(fields == 0 || (x_cat && bg_cat && cat_bit && out_cat), "NULL categorical argument");
  DTB_CHECK_ARG(conts == 0 || (x_cont && bg_cont && cont_bit && out_cont), "NULL continuous argument");
  const int64_t rows = coalitions * bg_rows;
  shap_compose_kernel<<<grid_for(rows * (fields + conts)), kShapThreads, 0, (cudaStream_t)stream>>>(
      x_cat, x_cont, bg_cat, bg_cont, masks, mask_words, x_index, cat_bit, cont_bit, rows, bg_rows, fields, conts,
      out_cat, out_cont);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_shap_means(const float* prob, int64_t groups, int rows_per_group, int cols, int kind, double* out,
                   void* stream) {
  DTB_CHECK_ARG(prob && out, "NULL argument");
  DTB_CHECK_ARG(groups > 0 && rows_per_group > 0 && cols > 0, "bad shape");
  DTB_CHECK_ARG(kind == DTB_SHAP_CLASS || (kind == DTB_SHAP_VALUE && cols == 1),
                "kind must be DTB_SHAP_CLASS, or DTB_SHAP_VALUE on one column");
  shap_means_kernel<<<grid_for(groups * 32), kShapThreads, 0, (cudaStream_t)stream>>>(prob, groups, rows_per_group,
                                                                                      cols, kind, out);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

}  // extern "C"
