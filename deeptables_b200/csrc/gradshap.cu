// Expected gradients (deeptables_b200/explain.py gradient_values, utils/shap.py DeepTablesGradientExplainer): the
// interpolated inputs of a range of (explained row, sample) pairs, each pair's per-column value from the gradient of
// one output at that input, and the mean over each row's samples.
//
// Pair p interpolates between explained row x_index[p] and background row bg_index[p] at alpha[p]: for categorical
// field f, e = E[j,f] + alpha * (E[i,f] - E[j,f]) on the embedding rows of the two ids; for continuous column c,
// z = b_c + alpha * (x_c - b_c).  Each step is rounded on its own (no fused multiply-add) so the host can restate the
// bits.  The value of pair p in field f is sum_d g[p,f,d] * (E[i,f,d] - E[j,f,d]) in float64, d in order, and in
// continuous column c it is g[p,c] * (x_c - b_c); a zero difference contributes exactly 0.  Every value depends only
// on its own pair, and the means add a row's samples in sample order, so the results are the same bits however the
// pairs are cut into launches.
#include "dtb_common.cuh"

namespace dtb {

constexpr int kGradShapThreads = 256;

// The embedding value of id `id` of field f at column d, zero for an id out of range (as the gather kernels read it).
__device__ __forceinline__ float emb_at(const float* __restrict__ table, const int64_t* __restrict__ row_offsets,
                                        int f, int id, int table_dim, int d) {
  const int64_t base = table_row(row_offsets, f, id, table_dim, nullptr);
  return base < 0 ? 0.f : table[base + d];
}

// Elements [0, pairs*fields*table_dim) are embedding coordinates (field-major (f, p, d) order when field_major, else
// (p, f, d); coordinates d >= the field's width are skipped), the rest continuous values (p, c).
__global__ void __launch_bounds__(kGradShapThreads) gradshap_compose_kernel(
    const int32_t* __restrict__ x_cat, const float* __restrict__ x_cont, const int32_t* __restrict__ bg_cat,
    const float* __restrict__ bg_cont, const float* __restrict__ table, const int64_t* __restrict__ row_offsets,
    const int32_t* __restrict__ col_offsets, int table_dim, const int32_t* __restrict__ x_index,
    const int32_t* __restrict__ bg_index, const float* __restrict__ alpha, int64_t pairs, int fields, int conts,
    int field_major, float* __restrict__ out_emb, float* __restrict__ out_cont) {
  const int64_t n_emb = pairs * fields * table_dim, total = n_emb + pairs * conts;
  const int width = fields ? col_offsets[fields] : 0;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    if (e < n_emb) {
      const int d = (int)(e % table_dim);
      const int64_t q = e / table_dim;
      int64_t p;
      int f;
      if (field_major) {
        p = q % pairs;
        f = (int)(q / pairs);
      } else {
        f = (int)(q % fields);
        p = q / fields;
      }
      const int lo = col_offsets[f];
      if (d >= col_offsets[f + 1] - lo) continue;
      const float a = alpha[p];
      const float ei = emb_at(table, row_offsets, f, x_cat[(int64_t)x_index[p] * fields + f], table_dim, d);
      const float ej = emb_at(table, row_offsets, f, bg_cat[(int64_t)bg_index[p] * fields + f], table_dim, d);
      const float v = __fadd_rn(ej, __fmul_rn(a, __fsub_rn(ei, ej)));
      if (field_major)
        out_emb[q * table_dim + d] = v;                              // [F, P, D]: q = f * pairs + p
      else
        out_emb[p * width + lo + d] = v;                             // [P, sum D_f]
    } else {
      const int64_t i = e - n_emb, p = i / conts;
      const int c = (int)(i - p * conts);
      const float xv = x_cont[(int64_t)x_index[p] * conts + c], bv = bg_cont[(int64_t)bg_index[p] * conts + c];
      out_cont[i] = __fadd_rn(bv, __fmul_rn(alpha[p], __fsub_rn(xv, bv)));
    }
  }
}

// One thread per (pair, encoded column): out [pairs, fields + conts].
__global__ void __launch_bounds__(kGradShapThreads) gradshap_reduce_kernel(
    const int32_t* __restrict__ x_cat, const float* __restrict__ x_cont, const int32_t* __restrict__ bg_cat,
    const float* __restrict__ bg_cont, const float* __restrict__ table, const int64_t* __restrict__ row_offsets,
    const int32_t* __restrict__ col_offsets, int table_dim, const int32_t* __restrict__ x_index,
    const int32_t* __restrict__ bg_index, int64_t pairs, int fields, int conts, const float* __restrict__ g_emb,
    const float* __restrict__ g_cont, double* __restrict__ out) {
  const int cols = fields + conts;
  const int width = fields ? col_offsets[fields] : 0;
  const int64_t total = pairs * cols;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = e / cols;
    const int k = (int)(e - p * cols);
    double acc = 0.0;
    if (k < fields) {
      const int lo = col_offsets[k], w = col_offsets[k + 1] - lo;
      const int64_t bi = table_row(row_offsets, k, x_cat[(int64_t)x_index[p] * fields + k], table_dim, nullptr);
      const int64_t bj = table_row(row_offsets, k, bg_cat[(int64_t)bg_index[p] * fields + k], table_dim, nullptr);
      const float* gp = g_emb + p * width + lo;
      for (int d = 0; d < w; ++d) {
        const float delta = __fsub_rn(bi < 0 ? 0.f : table[bi + d], bj < 0 ? 0.f : table[bj + d]);
        if (delta != 0.f) acc = __dadd_rn(acc, __dmul_rn((double)gp[d], (double)delta));
      }
    } else {
      const int c = k - fields;
      const float delta = __fsub_rn(x_cont[(int64_t)x_index[p] * conts + c], bg_cont[(int64_t)bg_index[p] * conts + c]);
      if (delta != 0.f) acc = __dmul_rn((double)g_cont[p * conts + c], (double)delta);
    }
    out[e] = acc;
  }
}

// One thread per (row, column): the row's n samples added in sample order, then divided by n.
__global__ void __launch_bounds__(kGradShapThreads) gradshap_means_kernel(const double* __restrict__ values,
                                                                        int64_t rows, int n, int cols,
                                                                        double* __restrict__ out) {
  const int64_t total = rows * cols;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = e / cols;
    const int c = (int)(e - r * cols);
    const double* v = values + r * n * cols + c;
    double acc = 0.0;
    for (int s = 0; s < n; ++s) acc = __dadd_rn(acc, v[(int64_t)s * cols]);
    out[e] = __ddiv_rn(acc, (double)n);
  }
}

// One thread per row: dz [rows, cols] = d out_k / d z of the task's output activation.
__global__ void __launch_bounds__(kGradShapThreads) gradshap_output_grad_kernel(const float* __restrict__ z,
                                                                              int64_t rows, int cols, int k, int kind,
                                                                              float* __restrict__ dz) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x) {
    const float* zr = z + r * cols;
    float* dr = dz + r * cols;
    if (kind == DTB_GRADSHAP_SOFTMAX) {
      float m = zr[0];
      for (int j = 1; j < cols; ++j) m = fmaxf(m, zr[j]);
      float s = 0.f;
      for (int j = 0; j < cols; ++j) s += expf(zr[j] - m);
      const float pk = expf(zr[k] - m) / s;
      for (int j = 0; j < cols; ++j) {
        const float pj = expf(zr[j] - m) / s;
        dr[j] = pk * ((j == k ? 1.f : 0.f) - pj);
      }
    } else {
      for (int j = 0; j < cols; ++j) dr[j] = 0.f;
      if (kind == DTB_GRADSHAP_SIGMOID) {
        const float p = 1.f / (1.f + expf(-zr[k]));
        dr[k] = p * (1.f - p);
      } else {
        dr[k] = 1.f;
      }
    }
  }
}

static inline int gradshap_grid(int64_t threads) {
  const int64_t cap = (int64_t)sm_count() * 16;
  const int64_t blocks = (threads + kGradShapThreads - 1) / kGradShapThreads;
  return (int)(blocks < 1 ? 1 : blocks > cap ? cap : blocks);
}

}  // namespace dtb

using namespace dtb;

extern "C" {

int dtb_gradshap_compose(const int32_t* x_cat, const float* x_cont, const int32_t* bg_cat, const float* bg_cont,
                         const float* table, const int64_t* row_offsets, const int32_t* col_offsets, int table_dim,
                         const int32_t* x_index, const int32_t* bg_index, const float* alpha, int64_t pairs,
                         int fields, int conts, int field_major, float* out_emb, float* out_cont, void* stream) {
  DTB_CHECK_ARG(x_index && bg_index && alpha, "NULL x_index, bg_index or alpha");
  DTB_CHECK_ARG(pairs > 0 && fields >= 0 && conts >= 0 && fields + conts > 0, "bad shape");
  DTB_CHECK_ARG(fields == 0 || (x_cat && bg_cat && table && row_offsets && col_offsets && out_emb && table_dim > 0),
                "NULL categorical argument");
  DTB_CHECK_ARG(conts == 0 || (x_cont && bg_cont && out_cont), "NULL continuous argument");
  DTB_CHECK_ARG(field_major == 0 || field_major == 1, "field_major must be 0 or 1");
  const int64_t total = pairs * ((int64_t)fields * table_dim + conts);
  gradshap_compose_kernel<<<gradshap_grid(total), kGradShapThreads, 0, (cudaStream_t)stream>>>(
      x_cat, x_cont, bg_cat, bg_cont, table, row_offsets, col_offsets, table_dim, x_index, bg_index, alpha, pairs,
      fields, conts, field_major, out_emb, out_cont);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_gradshap_reduce(const int32_t* x_cat, const float* x_cont, const int32_t* bg_cat, const float* bg_cont,
                        const float* table, const int64_t* row_offsets, const int32_t* col_offsets, int table_dim,
                        const int32_t* x_index, const int32_t* bg_index, int64_t pairs, int fields, int conts,
                        const float* g_emb, const float* g_cont, double* out, void* stream) {
  DTB_CHECK_ARG(x_index && bg_index && out, "NULL x_index, bg_index or out");
  DTB_CHECK_ARG(pairs > 0 && fields >= 0 && conts >= 0 && fields + conts > 0, "bad shape");
  DTB_CHECK_ARG(fields == 0 || (x_cat && bg_cat && table && row_offsets && col_offsets && g_emb && table_dim > 0),
                "NULL categorical argument");
  DTB_CHECK_ARG(conts == 0 || (x_cont && bg_cont && g_cont), "NULL continuous argument");
  gradshap_reduce_kernel<<<gradshap_grid(pairs * (fields + conts)), kGradShapThreads, 0, (cudaStream_t)stream>>>(
      x_cat, x_cont, bg_cat, bg_cont, table, row_offsets, col_offsets, table_dim, x_index, bg_index, pairs, fields,
      conts, g_emb, g_cont, out);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_gradshap_means(const double* values, int64_t rows, int samples, int cols, double* out, void* stream) {
  DTB_CHECK_ARG(values && out, "NULL values or out");
  DTB_CHECK_ARG(rows > 0 && samples > 0 && cols > 0, "bad shape");
  gradshap_means_kernel<<<gradshap_grid(rows * cols), kGradShapThreads, 0, (cudaStream_t)stream>>>(values, rows,
                                                                                                   samples, cols, out);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_gradshap_output_grad(const float* z, int64_t rows, int cols, int k, int kind, float* dz, void* stream) {
  DTB_CHECK_ARG(z && dz, "NULL z or dz");
  DTB_CHECK_ARG(rows > 0 && cols > 0 && k >= 0 && k < cols, "bad shape or output column");
  DTB_CHECK_ARG(kind == DTB_GRADSHAP_IDENTITY || kind == DTB_GRADSHAP_SIGMOID || kind == DTB_GRADSHAP_SOFTMAX,
                "kind must be DTB_GRADSHAP_IDENTITY, _SIGMOID or _SOFTMAX");
  gradshap_output_grad_kernel<<<gradshap_grid(rows), kGradShapThreads, 0, (cudaStream_t)stream>>>(z, rows, cols, k,
                                                                                                  kind, dz);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

}  // extern "C"
