// flatten_embeddings + concat_embedding_dense for columns of different embedding widths
// (ModelConfig.fixed_embedding_dim=False; reference layers.py:862-877, deepmodel.py:269-278, 348-357).
//
// Storage: the F tables live in the usual [sum V, Dmax] buffer; field f uses columns [0, D_f) of its rows and the
// columns [D_f, Dmax) are padding that no kernel here reads or writes.  Output row b of X is
//   [e(b,0)[0:D_0], e(b,1)[0:D_1], ..., e(b,F-1)[0:D_{F-1}], dense[b, 0:C]],   width W = sum D_f + C.
//
// Every block first builds a chunk map in shared memory: one int per VEC-wide chunk of the embedding part of a row,
// (field << 16) | first column inside the field.  Chunk k covers output columns [k*VEC, (k+1)*VEC), so the main loop
// needs no divide or search to find a column's field.  VEC = 4 when every D_f and Dmax are multiples of 4 (16-byte
// table loads and 16-byte REDs into the gradient), otherwise 1.  One warp handles one batch row at a time.
#include "dtb_common.cuh"

namespace dtb {

constexpr int kRaggedThreads = 256;
constexpr int kRaggedMaxFields = 960;           // keeps the kernel parameter block under 4 KiB
constexpr int kRaggedMaxChunks = 12 * 1024;     // 48 KiB of chunk map

// column prefix sums of the field widths, passed by value (no device allocation, graph-capturable)
struct RaggedCols {
  int col0[kRaggedMaxFields + 1];
};

template <int VEC>
__device__ __forceinline__ void build_chunk_map(const RaggedCols& cols, int F, int* map) {
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    const int lo = cols.col0[f], hi = cols.col0[f + 1];
    for (int c = lo; c < hi; c += VEC) map[c / VEC] = (f << 16) | (c - lo);
  }
  __syncthreads();
}

template <int VEC>
__global__ void __launch_bounds__(kRaggedThreads)
ragged_concat_fwd_kernel(const int32_t* __restrict__ idx, const float* __restrict__ table,
                         const int64_t* __restrict__ row_offsets, const float* __restrict__ dense,
                         float* __restrict__ X, int B, int F, int Dmax, int C, int n_chunks, bool vec_store,
                         const __grid_constant__ RaggedCols cols, int* status) {
  extern __shared__ int map[];
  build_chunk_map<VEC>(cols, F, map);
  const int SD = n_chunks * VEC;
  const int W = SD + C;
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < B; row += warps) {
    const int32_t* ids = idx + (int64_t)row * F;
    float* xr = X + (int64_t)row * W;
    for (int k = lane; k < n_chunks; k += 32) {
      const int e = map[k];
      const int f = e >> 16, d = e & 0xffff;
      const int64_t rb = table_row(row_offsets, f, __ldg(ids + f), Dmax, status);
      if (VEC == 4) {
        const float4 v = rb >= 0 ? __ldg(reinterpret_cast<const float4*>(table + rb + d)) : make_float4(0.f, 0.f, 0.f, 0.f);
        float* dst = xr + k * 4;
        if (vec_store) {
          *reinterpret_cast<float4*>(dst) = v;
        } else {
          dst[0] = v.x;
          dst[1] = v.y;
          dst[2] = v.z;
          dst[3] = v.w;
        }
      } else {
        xr[k] = rb >= 0 ? __ldg(table + rb + d) : 0.f;
      }
    }
    for (int c = lane; c < C; c += 32) xr[SD + c] = __ldg(dense + (int64_t)row * C + c);
  }
}

// grad_table[row(f, id), d] += dX[b, col]  over the embedding part of dX (row stride W); padding is never touched
template <int VEC>
__global__ void __launch_bounds__(kRaggedThreads)
ragged_concat_bwd_kernel(const int32_t* __restrict__ idx, const int64_t* __restrict__ row_offsets,
                         const float* __restrict__ dX, float* __restrict__ grad_table, int B, int F, int Dmax, int W,
                         int n_chunks, const __grid_constant__ RaggedCols cols) {
  extern __shared__ int map[];
  build_chunk_map<VEC>(cols, F, map);
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < B; row += warps) {
    const int32_t* ids = idx + (int64_t)row * F;
    const float* gr = dX + (int64_t)row * W;
    for (int k = lane; k < n_chunks; k += 32) {
      const int e = map[k];
      const int f = e >> 16, d = e & 0xffff;
      const int64_t rb = table_row(row_offsets, f, __ldg(ids + f), Dmax, nullptr);
      if (rb < 0) continue;
      if (VEC == 4) {
        const float* src = gr + k * 4;
        red_add_f4(grad_table + rb + d, make_float4(__ldg(src), __ldg(src + 1), __ldg(src + 2), __ldg(src + 3)));
      } else {
        atomicAdd(grad_table + rb + d, __ldg(gr + k));
      }
    }
  }
}

// validates the widths and fills the column prefix sums; returns the embedding width sum D_f or -1
static int ragged_cols(const int* dims_host, int F, int Dmax, RaggedCols* cols, bool* all4) {
  int s = 0;
  bool a4 = Dmax % 4 == 0;
  for (int f = 0; f < F; ++f) {
    const int d = dims_host[f];
    if (d < 1 || d > Dmax) return -1;
    cols->col0[f] = s;
    s += d;
    a4 = a4 && d % 4 == 0;
  }
  cols->col0[F] = s;
  *all4 = a4;
  return s;
}

static int ragged_grid(int B) {
  const int warps = kRaggedThreads / 32;
  int64_t blocks = ((int64_t)B + warps - 1) / warps;
  const int64_t cap = (int64_t)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  return (int)(blocks < 1 ? 1 : blocks);
}

}  // namespace dtb

using namespace dtb;

extern "C" {

int dtb_ragged_concat_emb_dense_fwd(const int32_t* idx, const float* table, const int64_t* row_offsets,
                                    const int* dims_host, const float* dense, float* X, int B, int F, int Dmax, int C,
                                    int* status, void* stream) {
  DTB_CHECK_ARG(B >= 0 && C >= 0 && X, "bad shape / X NULL");
  DTB_CHECK_ARG(F >= 1 && F <= kRaggedMaxFields, "F must be in [1, 960]");
  DTB_CHECK_ARG(Dmax >= 1 && Dmax <= 0xffff, "Dmax must be in [1, 65535]");
  DTB_CHECK_ARG(idx && table && row_offsets && dims_host, "NULL table argument");
  DTB_CHECK_ARG(C == 0 || dense, "dense NULL with C > 0");
  RaggedCols cols;
  bool all4 = false;
  const int SD = ragged_cols(dims_host, F, Dmax, &cols, &all4);
  DTB_CHECK_ARG(SD > 0, "every width must be in [1, Dmax]");
  const bool vec = all4 && (reinterpret_cast<uintptr_t>(table) % 16) == 0;
  const int n_chunks = vec ? SD / 4 : SD;
  DTB_CHECK_ARG(n_chunks <= kRaggedMaxChunks, "more than 12288 chunks per row (sum of widths too large)");
  if (B == 0) return DTB_OK;
  const int W = SD + C;
  const bool vec_store = W % 4 == 0 && (reinterpret_cast<uintptr_t>(X) % 16) == 0;
  const size_t smem = (size_t)n_chunks * sizeof(int);
  cudaStream_t st = (cudaStream_t)stream;
  if (vec)
    ragged_concat_fwd_kernel<4><<<ragged_grid(B), kRaggedThreads, smem, st>>>(idx, table, row_offsets, dense, X, B, F,
                                                                             Dmax, C, n_chunks, vec_store, cols,
                                                                             status);
  else
    ragged_concat_fwd_kernel<1><<<ragged_grid(B), kRaggedThreads, smem, st>>>(idx, table, row_offsets, dense, X, B, F,
                                                                             Dmax, C, n_chunks, false, cols, status);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_ragged_concat_emb_dense_bwd(const int32_t* idx, const int64_t* row_offsets, const int* dims_host,
                                    const float* dX, float* grad_table, int B, int F, int Dmax, int C, void* stream) {
  DTB_CHECK_ARG(B >= 0 && C >= 0, "negative shape");
  DTB_CHECK_ARG(F >= 1 && F <= kRaggedMaxFields, "F must be in [1, 960]");
  DTB_CHECK_ARG(Dmax >= 1 && Dmax <= 0xffff, "Dmax must be in [1, 65535]");
  DTB_CHECK_ARG(idx && row_offsets && dims_host && dX && grad_table, "NULL argument");
  RaggedCols cols;
  bool all4 = false;
  const int SD = ragged_cols(dims_host, F, Dmax, &cols, &all4);
  DTB_CHECK_ARG(SD > 0, "every width must be in [1, Dmax]");
  const bool vec = all4 && (reinterpret_cast<uintptr_t>(grad_table) % 16) == 0;
  const int n_chunks = vec ? SD / 4 : SD;
  DTB_CHECK_ARG(n_chunks <= kRaggedMaxChunks, "more than 12288 chunks per row (sum of widths too large)");
  if (B == 0) return DTB_OK;
  const int W = SD + C;
  const size_t smem = (size_t)n_chunks * sizeof(int);
  cudaStream_t st = (cudaStream_t)stream;
  if (vec)
    ragged_concat_bwd_kernel<4><<<ragged_grid(B), kRaggedThreads, smem, st>>>(idx, row_offsets, dX, grad_table, B, F,
                                                                             Dmax, W, n_chunks, cols);
  else
    ragged_concat_bwd_kernel<1><<<ragged_grid(B), kRaggedThreads, smem, st>>>(idx, row_offsets, dX, grad_table, B, F,
                                                                             Dmax, W, n_chunks, cols);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

}  // extern "C"
