// PNN products (InnerProduct / OuterProduct, layers.py:473-487, 541-581; gather fused) and the
// AutoInt attention core (MultiheadAttention.call, layers.py:129-150: per-head softmax(QK^T/sqrt(dh))V
// + residual + relu; the four relu(Dense) projections and the BatchNormalization around it are Dense /
// BatchNorm calls of this library).  Both are small-F pairwise ops on CUDA cores: per batch row the
// (F x D) block lives in shared memory; there is no large dense contraction to put on tensor cores.
#include "dtb_common.cuh"

namespace dtb {

constexpr int kPnnRows = 8;      // batch rows per CTA (the outer-product kernel is reused across them)
constexpr int kMaxD = 64;

__device__ __forceinline__ void pair_of(int p, int F, int& i, int& j) {
  // pairs (i<j) in row-major order (layers.py:478-483)
  int ii = 0, rem = p;
  while (rem >= F - 1 - ii) {
    rem -= F - 1 - ii;
    ++ii;
  }
  i = ii;
  j = ii + 1 + rem;
}

__device__ __forceinline__ void stage_rows(const int32_t* __restrict__ idx, const float* __restrict__ table,
                                           const int64_t* __restrict__ row_offsets, float* __restrict__ es, int row0,
                                           int n_rows, int B, int F, int D, int* status) {
  for (int e = threadIdx.x; e < n_rows * F * D; e += blockDim.x) {
    const int r = e / (F * D);
    const int rem = e - r * F * D;
    const int f = rem / D, d = rem - f * D;
    float v = 0.f;
    if (row0 + r < B) {
      const int64_t rb = table_row(row_offsets, f, __ldg(idx + (int64_t)(row0 + r) * F + f), D, status);
      if (rb >= 0) v = __ldg(table + rb + d);
    }
    es[e] = v;
  }
}

// thread = pair; loops over the CTA's kPnnRows rows with the kernel slice of the pair held per k-step
__global__ void pnn_fwd_kernel(const int32_t* __restrict__ idx, const float* __restrict__ table,
                               const int64_t* __restrict__ row_offsets, const float* __restrict__ kern,
                               float* __restrict__ ip, float* __restrict__ op, int B, int F, int D, int P, int ktype,
                               int* status) {
  extern __shared__ float es[];    // [rows][F][D]
  const int row0 = blockIdx.x * kPnnRows;
  stage_rows(idx, table, row_offsets, es, row0, kPnnRows, B, F, D, status);
  __syncthreads();
  const int p = threadIdx.x;
  if (p >= P) return;
  int i, j;
  pair_of(p, F, i, j);
  float acc_ip[kPnnRows], acc_op[kPnnRows];
#pragma unroll
  for (int r = 0; r < kPnnRows; ++r) {
    acc_ip[r] = 0.f;
    acc_op[r] = 0.f;
    const float* ei = es + ((size_t)r * F + i) * D;
    const float* ej = es + ((size_t)r * F + j) * D;
    float s = 0.f;
    for (int d = 0; d < D; ++d) s += ei[d] * ej[d];
    acc_ip[r] = s;
  }
  if (op) {
    if (ktype == 0) {
      for (int k = 0; k < D; ++k) {
        const float* kr = kern + ((size_t)k * P + p) * D;
        float t[kPnnRows];
#pragma unroll
        for (int r = 0; r < kPnnRows; ++r) t[r] = 0.f;
        for (int d = 0; d < D; ++d) {
          const float kv = __ldg(kr + d);
#pragma unroll
          for (int r = 0; r < kPnnRows; ++r) t[r] += es[((size_t)r * F + i) * D + d] * kv;
        }
#pragma unroll
        for (int r = 0; r < kPnnRows; ++r) acc_op[r] += t[r] * es[((size_t)r * F + j) * D + k];
      }
    } else if (ktype == 1) {
      for (int d = 0; d < D; ++d) {
        const float kv = __ldg(kern + (size_t)p * D + d);
#pragma unroll
        for (int r = 0; r < kPnnRows; ++r)
          acc_op[r] += es[((size_t)r * F + i) * D + d] * es[((size_t)r * F + j) * D + d] * kv;
      }
    } else {
      const float kv = __ldg(kern + p);
#pragma unroll
      for (int r = 0; r < kPnnRows; ++r) acc_op[r] = acc_ip[r] * kv;
    }
  }
#pragma unroll
  for (int r = 0; r < kPnnRows; ++r) {
    if (row0 + r < B) {
      if (ip) ip[(size_t)(row0 + r) * P + p] = acc_ip[r];
      if (op) op[(size_t)(row0 + r) * P + p] = acc_op[r];
    }
  }
}

// dE: thread = pair, per-row contributions accumulated in shared memory, then one RED per element
__global__ void pnn_bwd_de_kernel(const int32_t* __restrict__ idx, const float* __restrict__ table,
                                  const int64_t* __restrict__ row_offsets, const float* __restrict__ kern,
                                  const float* __restrict__ d_ip, const float* __restrict__ d_op,
                                  float* __restrict__ grad_table, int B, int F, int D, int P, int ktype) {
  extern __shared__ float sm[];
  float* es = sm;                                   // [rows][F][D]
  float* des = sm + (size_t)kPnnRows * F * D;       // [rows][F][D]
  const int row0 = blockIdx.x * kPnnRows;
  stage_rows(idx, table, row_offsets, es, row0, kPnnRows, B, F, D, nullptr);
  for (int e = threadIdx.x; e < kPnnRows * F * D; e += blockDim.x) des[e] = 0.f;
  __syncthreads();
  const int p = threadIdx.x;
  if (p < P) {
    int i, j;
    pair_of(p, F, i, j);
    for (int r = 0; r < kPnnRows; ++r) {
      if (row0 + r >= B) break;
      const float gi = d_ip ? d_ip[(size_t)(row0 + r) * P + p] : 0.f;
      const float go = d_op ? d_op[(size_t)(row0 + r) * P + p] : 0.f;
      const float* ei = es + ((size_t)r * F + i) * D;
      const float* ej = es + ((size_t)r * F + j) * D;
      float* di = des + ((size_t)r * F + i) * D;
      float* dj = des + ((size_t)r * F + j) * D;
      if (d_ip)
        for (int d = 0; d < D; ++d) {
          atomicAdd(di + d, gi * ej[d]);
          atomicAdd(dj + d, gi * ei[d]);
        }
      if (d_op) {
        if (ktype == 0) {
          // op = sum_k (sum_d ei[d] K[k,p,d]) ej[k]
          float gi_acc[kMaxD];
          for (int d = 0; d < D; ++d) gi_acc[d] = 0.f;
          for (int k = 0; k < D; ++k) {
            const float* kr = kern + ((size_t)k * P + p) * D;
            float t = 0.f;
            const float ejk = ej[k];
            for (int d = 0; d < D; ++d) {
              const float kv = __ldg(kr + d);
              t += ei[d] * kv;
              gi_acc[d] += kv * ejk;
            }
            atomicAdd(dj + k, go * t);
          }
          for (int d = 0; d < D; ++d) atomicAdd(di + d, go * gi_acc[d]);
        } else if (ktype == 1) {
          for (int d = 0; d < D; ++d) {
            const float kv = __ldg(kern + (size_t)p * D + d);
            atomicAdd(di + d, go * ej[d] * kv);
            atomicAdd(dj + d, go * ei[d] * kv);
          }
        } else {
          const float kv = __ldg(kern + p);
          for (int d = 0; d < D; ++d) {
            atomicAdd(di + d, go * kv * ej[d]);
            atomicAdd(dj + d, go * kv * ei[d]);
          }
        }
      }
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < kPnnRows * F * D; e += blockDim.x) {
    const int r = e / (F * D);
    if (row0 + r >= B) continue;
    const int rem = e - r * F * D;
    const int f = rem / D, d = rem - f * D;
    const int64_t rb = table_row(row_offsets, f, __ldg(idx + (int64_t)(row0 + r) * F + f), D, nullptr);
    if (rb >= 0 && des[e] != 0.f) atomicAdd(grad_table + rb + d, des[e]);
  }
}

// dK: persistent CTAs, thread = pair, k outermost so the accumulator is D registers; one atomic per
// kernel element per CTA
__global__ void pnn_bwd_dk_kernel(const int32_t* __restrict__ idx, const float* __restrict__ table,
                                  const int64_t* __restrict__ row_offsets, const float* __restrict__ d_op,
                                  float* __restrict__ d_kern, int B, int F, int D, int P, int ktype,
                                  int rows_per_cta) {
  const int p = threadIdx.x;
  if (p >= P) return;
  int i, j;
  pair_of(p, F, i, j);
  const int r_begin = blockIdx.x * rows_per_cta;
  const int r_end = min(B, r_begin + rows_per_cta);
  if (ktype == 0) {
    for (int k = 0; k < D; ++k) {
      float acc[kMaxD];
      for (int d = 0; d < D; ++d) acc[d] = 0.f;
      for (int r = r_begin; r < r_end; ++r) {
        const int64_t bi = table_row(row_offsets, i, __ldg(idx + (int64_t)r * F + i), D, nullptr);
        const int64_t bj = table_row(row_offsets, j, __ldg(idx + (int64_t)r * F + j), D, nullptr);
        if (bi < 0 || bj < 0) continue;
        const float w = d_op[(size_t)r * P + p] * __ldg(table + bj + k);
        for (int d = 0; d < D; ++d) acc[d] += w * __ldg(table + bi + d);
      }
      for (int d = 0; d < D; ++d)
        if (acc[d] != 0.f) atomicAdd(d_kern + ((size_t)k * P + p) * D + d, acc[d]);
    }
  } else {
    float acc[kMaxD];
    const int n = ktype == 1 ? D : 1;
    for (int d = 0; d < n; ++d) acc[d] = 0.f;
    for (int r = r_begin; r < r_end; ++r) {
      const int64_t bi = table_row(row_offsets, i, __ldg(idx + (int64_t)r * F + i), D, nullptr);
      const int64_t bj = table_row(row_offsets, j, __ldg(idx + (int64_t)r * F + j), D, nullptr);
      if (bi < 0 || bj < 0) continue;
      const float go = d_op[(size_t)r * P + p];
      if (ktype == 1) {
        for (int d = 0; d < D; ++d) acc[d] += go * __ldg(table + bi + d) * __ldg(table + bj + d);
      } else {
        float s = 0.f;
        for (int d = 0; d < D; ++d) s += __ldg(table + bi + d) * __ldg(table + bj + d);
        acc[0] += go * s;
      }
    }
    for (int d = 0; d < n; ++d)
      if (acc[d] != 0.f) atomicAdd(d_kern + (size_t)p * n + d, acc[d]);
  }
}

// ------------------------------------------------------------------------------------------
// PNN kernels with the embedding width as a template parameter (DT = 4, 8, 16, 32).  The generic kernels above keep one
// pair per thread, re-read the (D x D) kernel slice of the pair from global memory for every batch row, index
// `gi_acc[kMaxD]` with a run-time bound (local memory) and merge the per-pair contributions with shared-memory float
// atomics: 6.2 ms for the embedding gradient at 16 384 rows x 26 fields x D = 16.  Here a thread is one (batch row, field):
// its embedding row and accumulators are registers, the kernel slices of the field's pairs sit in shared memory and are
// read as 128-bit warp broadcasts (all lanes of a CTA work on the same field), and nothing is merged across threads --
// the row's gradient leaves as one vector RED per 4 floats.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int pair_index(int a, int b, int F) {      // a < b, row-major order of pair_of()
  return a * (F - 1) - a * (a - 1) / 2 + (b - a - 1);
}

template <int DT>
__device__ __forceinline__ void load_row(const float* __restrict__ p, float (&o)[DT]) {
#pragma unroll
  for (int c = 0; c < DT / 4; ++c) {
    const float4 t = *reinterpret_cast<const float4*>(p + 4 * c);
    o[4 * c] = t.x;
    o[4 * c + 1] = t.y;
    o[4 * c + 2] = t.z;
    o[4 * c + 3] = t.w;
  }
}

template <int DT>
__device__ __forceinline__ void gather_row(const int32_t* __restrict__ idx, const float* __restrict__ table,
                                           const int64_t* __restrict__ row_offsets, int row, int F, int f,
                                           float (&o)[DT], int64_t* rb_out, int* status) {
  const int64_t rb = table_row(row_offsets, f, __ldg(idx + (int64_t)row * F + f), DT, status);
  if (rb_out) *rb_out = rb;
  if (rb >= 0) {
#pragma unroll
    for (int c = 0; c < DT / 4; ++c) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(table + rb) + c);
      o[4 * c] = t.x;
      o[4 * c + 1] = t.y;
      o[4 * c + 2] = t.z;
      o[4 * c + 3] = t.w;
    }
  } else {
#pragma unroll
    for (int c = 0; c < DT; ++c) o[c] = 0.f;
  }
}

// kernel slices of `n` pairs into shared memory: ktype 0 -> ks[q][k][d], ktype 1 -> ks[q][d], ktype 2 -> ks[q]
template <int DT>
__device__ __forceinline__ void stage_kernel_slices(const float* __restrict__ kern, float* __restrict__ ks, int n, int P,
                                                    int ktype, int f, int F, bool only_upper) {
  // pair of slot q: only_upper -> (f, f+1+q); else the other field is o = q < f ? q : q + 1
  const int per = ktype == 0 ? DT * DT : (ktype == 1 ? DT : 1);
  for (int e = threadIdx.x; e < n * per; e += blockDim.x) {
    const int q = e / per, rem = e - q * per;
    int p;
    if (only_upper) {
      p = pair_index(f, f + 1 + q, F);
    } else {
      const int o = q < f ? q : q + 1;
      p = o < f ? pair_index(o, f, F) : pair_index(f, o, F);
    }
    float v;
    if (ktype == 0) {
      const int k = rem / DT, d = rem - k * DT;
      v = __ldg(kern + ((size_t)k * P + p) * DT + d);
    } else if (ktype == 1) {
      v = __ldg(kern + (size_t)p * DT + rem);
    } else {
      v = __ldg(kern + p);
    }
    ks[e] = v;
  }
}

constexpr int kPnnTRows = 128;       // batch rows (= threads) per CTA of the (row, field) kernels

// grid (F-1, row-chunk groups): CTA x = field i computes the pairs (i, j > i) of its row chunks.  The CTAs of one chunk
// group are adjacent in launch order, so the 26 field rows of a batch row are fetched from HBM once and re-read from L2.
// The embedding row of the NEXT pair is requested before the current pair's FMAs.
template <int DT>
__global__ void __launch_bounds__(kPnnTRows) pnn_fwd_t_kernel(const int32_t* __restrict__ idx, const float* __restrict__ table,
                                                              const int64_t* __restrict__ row_offsets,
                                                              const float* __restrict__ kern, float* __restrict__ ip,
                                                              float* __restrict__ op, int B, int F, int P, int ktype,
                                                              int* status) {
  extern __shared__ __align__(16) float ks[];
  const int i = blockIdx.x, n = F - 1 - i;
  if (op) stage_kernel_slices<DT>(kern, ks, n, P, ktype, i, F, true);
  __syncthreads();
  const int p0 = pair_index(i, i + 1, F);
  const int n_chunks = (B + kPnnTRows - 1) / kPnnTRows;
  for (int chunk = blockIdx.y; chunk < n_chunks; chunk += gridDim.y) {
    const int row = chunk * kPnnTRows + threadIdx.x;
    if (row >= B) continue;
    float ei[DT], ej[DT], en[DT];
    gather_row<DT>(idx, table, row_offsets, row, F, i, ei, nullptr, status);
    gather_row<DT>(idx, table, row_offsets, row, F, i + 1, en, nullptr, i == 0 ? status : nullptr);
    for (int q = 0; q < n; ++q) {
#pragma unroll
      for (int d = 0; d < DT; ++d) ej[d] = en[d];
      if (q + 1 < n) gather_row<DT>(idx, table, row_offsets, row, F, i + 2 + q, en, nullptr, i == 0 ? status : nullptr);
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < DT; ++d) s = fmaf(ei[d], ej[d], s);
      if (ip) ip[(size_t)row * P + p0 + q] = s;
      if (op) {
        float acc = 0.f;
        if (ktype == 0) {
          const float* kq = ks + (size_t)q * DT * DT;
#pragma unroll
          for (int k = 0; k < DT; ++k) {
            float kv[DT];
            load_row<DT>(kq + k * DT, kv);
            float t = 0.f;
#pragma unroll
            for (int d = 0; d < DT; ++d) t = fmaf(ei[d], kv[d], t);
            acc = fmaf(t, ej[k], acc);
          }
        } else if (ktype == 1) {
          float kv[DT];
          load_row<DT>(ks + (size_t)q * DT, kv);
#pragma unroll
          for (int d = 0; d < DT; ++d) acc = fmaf(ei[d] * ej[d], kv[d], acc);
        } else {
          acc = s * ks[q];
        }
        op[(size_t)row * P + p0 + q] = acc;
      }
    }
  }
}

// grid (F, row-chunk groups): thread = (row, field f) accumulates dLoss/d e_f over the F-1 pairs that contain f
template <int DT>
__global__ void __launch_bounds__(kPnnTRows) pnn_bwd_de_t_kernel(const int32_t* __restrict__ idx, const float* __restrict__ table,
                                                                 const int64_t* __restrict__ row_offsets,
                                                                 const float* __restrict__ kern,
                                                                 const float* __restrict__ d_ip,
                                                                 const float* __restrict__ d_op,
                                                                 float* __restrict__ grad_table, int B, int F, int P,
                                                                 int ktype) {
  extern __shared__ __align__(16) float ks[];
  const int f = blockIdx.x;
  if (d_op) stage_kernel_slices<DT>(kern, ks, F - 1, P, ktype, f, F, false);
  __syncthreads();
  const int n_chunks = (B + kPnnTRows - 1) / kPnnTRows;
  for (int chunk = blockIdx.y; chunk < n_chunks; chunk += gridDim.y) {
    const int row = chunk * kPnnTRows + threadIdx.x;
    if (row >= B) continue;
    const int64_t rb = table_row(row_offsets, f, __ldg(idx + (int64_t)row * F + f), DT, nullptr);
    if (rb < 0) continue;
    float acc[DT], eo[DT], en[DT];
#pragma unroll
    for (int d = 0; d < DT; ++d) acc[d] = 0.f;
    gather_row<DT>(idx, table, row_offsets, row, F, f == 0 ? 1 : 0, en, nullptr, nullptr);
    float gi_n = 0.f, go_n = 0.f;
    {
      const int p = f == 0 ? pair_index(0, 1, F) : pair_index(0, f, F);
      if (d_ip) gi_n = __ldg(d_ip + (size_t)row * P + p);
      if (d_op) go_n = __ldg(d_op + (size_t)row * P + p);
    }
    for (int q = 0; q < F - 1; ++q) {
      const int o = q < f ? q : q + 1;
#pragma unroll
      for (int d = 0; d < DT; ++d) eo[d] = en[d];
      const float gi = gi_n, go = go_n;
      if (q + 1 < F - 1) {                       // next pair's operands are requested before this pair's FMAs
        const int on = q + 1 < f ? q + 1 : q + 2;
        const int pn = on < f ? pair_index(on, f, F) : pair_index(f, on, F);
        gather_row<DT>(idx, table, row_offsets, row, F, on, en, nullptr, nullptr);
        if (d_ip) gi_n = __ldg(d_ip + (size_t)row * P + pn);
        if (d_op) go_n = __ldg(d_op + (size_t)row * P + pn);
      }
      if (d_ip) {
#pragma unroll
        for (int d = 0; d < DT; ++d) acc[d] = fmaf(gi, eo[d], acc[d]);
      }
      if (d_op) {
        if (ktype == 0) {
          const float* kq = ks + (size_t)q * DT * DT;
          if (f < o) {
            // f is the first field of the pair: d e_f[d] = go * sum_k K[k,p,d] e_o[k]
#pragma unroll
            for (int k = 0; k < DT; ++k) {
              float kv[DT];
              load_row<DT>(kq + k * DT, kv);
              const float w = go * eo[k];
#pragma unroll
              for (int d = 0; d < DT; ++d) acc[d] = fmaf(w, kv[d], acc[d]);
            }
          } else {
            // f is the second field: d e_f[k] = go * sum_d e_o[d] K[k,p,d]
#pragma unroll
            for (int k = 0; k < DT; ++k) {
              float kv[DT];
              load_row<DT>(kq + k * DT, kv);
              float t = 0.f;
#pragma unroll
              for (int d = 0; d < DT; ++d) t = fmaf(eo[d], kv[d], t);
              acc[k] = fmaf(go, t, acc[k]);
            }
          }
        } else if (ktype == 1) {
          float kv[DT];
          load_row<DT>(ks + (size_t)q * DT, kv);
#pragma unroll
          for (int d = 0; d < DT; ++d) acc[d] = fmaf(go * kv[d], eo[d], acc[d]);
        } else {
          const float w = go * ks[q];
#pragma unroll
          for (int d = 0; d < DT; ++d) acc[d] = fmaf(w, eo[d], acc[d]);
        }
      }
    }
    float4* dst = reinterpret_cast<float4*>(grad_table + rb);
#pragma unroll
    for (int c = 0; c < DT / 4; ++c) {
      const float4 v = make_float4(acc[4 * c], acc[4 * c + 1], acc[4 * c + 2], acc[4 * c + 3]);
      if (v.x != 0.f || v.y != 0.f || v.z != 0.f || v.w != 0.f) atomicAdd(dst + c, v);
    }
  }
}

// 'mat' kernel gradient dK[k,p,d] = sum_r d_op[r,p] e_j[r,k] e_i[r,d].  grid (pair groups, row groups), 256 threads:
// thread = (pair of the group, k) with the D accumulators over d in registers; the rows arrive in chunks of `R` gathered
// embedding blocks in shared memory.  One vector RED per 4 kernel elements per CTA.
template <int DT>
__global__ void __launch_bounds__(256) pnn_bwd_dk_t_kernel(const int32_t* __restrict__ idx, const float* __restrict__ table,
                                                           const int64_t* __restrict__ row_offsets,
                                                           const float* __restrict__ d_op, float* __restrict__ d_kern, int B,
                                                           int F, int P, int rows_per_cta, int R) {
  constexpr int kPg = 256 / DT;                  // pairs per group
  extern __shared__ __align__(16) float sm[];
  float* es = sm;                                // [R][F][DT]
  float* gos = sm + (size_t)R * F * DT;          // [R][kPg]
  const int pl = threadIdx.x / DT, k = threadIdx.x - pl * DT;
  const int p = blockIdx.x * kPg + pl;
  const bool live = p < P;
  int i = 0, j = 1;
  if (live) pair_of(p, F, i, j);
  float acc[DT];
#pragma unroll
  for (int d = 0; d < DT; ++d) acc[d] = 0.f;
  const int r_begin = blockIdx.y * rows_per_cta;
  const int r_end = min(B, r_begin + rows_per_cta);
  for (int r0 = r_begin; r0 < r_end; r0 += R) {
    const int nr = min(R, r_end - r0);
    __syncthreads();
    // gather in batches of 8 per thread: 8 index loads in flight, then 8 row loads, then the stores (one load per
    // iteration left 64 % of the kernel's stall samples on the two dependent latencies)
    const int n_vec = nr * F * (DT / 4);
    for (int e0 = threadIdx.x; e0 < n_vec; e0 += 8 * blockDim.x) {
      int id[8];
      float4 v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int e = e0 + u * blockDim.x;
        if (e < n_vec) id[u] = __ldg(idx + (int64_t)r0 * F + e / (DT / 4));     // (r, f) row-major == e / (DT/4)
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int e = e0 + u * blockDim.x;
        v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (e < n_vec) {
          const int rf = e / (DT / 4), c = e - rf * (DT / 4);
          const int64_t rb = table_row(row_offsets, rf % F, id[u], DT, nullptr);
          if (rb >= 0) v[u] = __ldg(reinterpret_cast<const float4*>(table + rb) + c);
        }
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int e = e0 + u * blockDim.x;
        if (e < n_vec) reinterpret_cast<float4*>(es)[e] = v[u];
      }
    }
    for (int e = threadIdx.x; e < nr * kPg; e += blockDim.x) {
      const int r = e / kPg, q = e - r * kPg;
      const int pp = blockIdx.x * kPg + q;
      gos[e] = pp < P ? __ldg(d_op + (size_t)(r0 + r) * P + pp) : 0.f;
    }
    __syncthreads();
    if (live) {
      for (int r = 0; r < nr; ++r) {
        const float* er = es + (size_t)r * F * DT;
        const float w = gos[r * kPg + pl] * er[j * DT + k];
        float ei[DT];
        load_row<DT>(er + i * DT, ei);
#pragma unroll
        for (int d = 0; d < DT; ++d) acc[d] = fmaf(w, ei[d], acc[d]);
      }
    }
  }
  if (live) {
    float4* dst = reinterpret_cast<float4*>(d_kern + ((size_t)k * P + p) * DT);
#pragma unroll
    for (int c = 0; c < DT / 4; ++c) {
      const float4 v = make_float4(acc[4 * c], acc[4 * c + 1], acc[4 * c + 2], acc[4 * c + 3]);
      if (v.x != 0.f || v.y != 0.f || v.z != 0.f || v.w != 0.f) atomicAdd(dst + c, v);
    }
  }
}

// ------------------------------------------------------------------------------------------
// attention core.  qkvr: [B, F, 4*D] = relu projections [Q | K | V | R] of each field row.
// One CTA per batch row; thread = (head, field).
//
// Attention dropout (reference layers.py:135-143, DROP = true): in training each softmax weight is kept with
// probability 1 - rate and scaled by 1 / (1 - rate).  The weight of (batch row b, head h, query field q, key field k)
// has the element index
//     i = ((b * heads + h) * F + q) * F + k          (b counted from AttDrop::row0)
// and is kept when mix32(dropout_key(seed) + i) >= rate * 2^32, the mask of dropout_kernel.  The index depends neither
// on the batch size nor on how a launch groups batch rows per CTA, so a batch and its slices draw the same bits.  The
// backward regenerates the mask: with w = softmax, m = 0 or 1 / (1 - rate) and w' = w m,
//     dV = w'^T dout,   dw = (dout V^T) m,   ds = w (dw - sum_k dw w);
// no mask and no extra activation is stored.
// ------------------------------------------------------------------------------------------
constexpr int kMaxDh = 64;

struct AttDrop {
  uint32_t threshold;                    // rate * 2^32
  float scale;                           // 1 / (1 - rate)
  uint64_t seed;
  const unsigned long long* seed_dev;    // non-null: the seed is read from device memory
  int64_t row0;                          // index of the call's first batch row in the mask
};

// counter of weight (b, h, q, 0); the key fields follow at + k
__device__ __forceinline__ uint64_t att_counter(const AttDrop& dr, uint64_t key, int b, int heads, int h, int F, int q) {
  return key + (((uint64_t)(dr.row0 + b) * heads + h) * F + q) * F;
}
// factor of the weight at counter c: 0 or 1 / (1 - rate)
__device__ __forceinline__ float att_keep(const AttDrop& dr, uint64_t c) {
  return mix32(c) >= dr.threshold ? dr.scale : 0.f;
}

template <bool DROP>
__device__ __forceinline__ void attention_core_fwd_body(const float* __restrict__ qkvr, float* __restrict__ Y, int B, int F,
                                                        int D, int heads, int use_res, const AttDrop& dr) {
  extern __shared__ float sm[];     // [F][4D]
  const int dh = D / heads;
  const float scale = rsqrtf((float)dh);
  const uint64_t key = DROP ? dropout_key(dr.seed, dr.seed_dev) : 0;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    __syncthreads();
    const float* src = qkvr + (size_t)b * F * 4 * D;
    for (int e = threadIdx.x; e < F * 4 * D; e += blockDim.x) sm[e] = src[e];
    __syncthreads();
    const int t = threadIdx.x;
    if (t < heads * F) {
      const int h = t / F, i = t - h * F;
      const float* q = sm + (size_t)i * 4 * D + h * dh;
      float m = -INFINITY;
      for (int j = 0; j < F; ++j) {
        const float* k = sm + (size_t)j * 4 * D + D + h * dh;
        float s = 0.f;
        for (int c = 0; c < dh; ++c) s += q[c] * k[c];
        m = fmaxf(m, s * scale);
      }
      float sum = 0.f;
      float acc[kMaxDh];
      for (int c = 0; c < dh; ++c) acc[c] = 0.f;
      const uint64_t ctr = DROP ? att_counter(dr, key, b, heads, h, F, i) : 0;
      for (int j = 0; j < F; ++j) {
        const float* k = sm + (size_t)j * 4 * D + D + h * dh;
        const float* v = sm + (size_t)j * 4 * D + 2 * D + h * dh;
        float s = 0.f;
        for (int c = 0; c < dh; ++c) s += q[c] * k[c];
        const float pj = __expf(s * scale - m);
        sum += pj;
        if (DROP && att_keep(dr, ctr + j) == 0.f) continue;      // the 1 / (1 - rate) of the kept weights: below
        for (int c = 0; c < dh; ++c) acc[c] += pj * v[c];
      }
      const float inv = 1.f / sum;
      float* y = Y + ((size_t)b * F + i) * D + h * dh;
      const float* res = sm + (size_t)i * 4 * D + 3 * D + h * dh;
      for (int c = 0; c < dh; ++c) {
        float o = acc[c] * inv;
        if (DROP) o *= dr.scale;
        if (use_res) o += res[c];
        y[c] = fmaxf(o, 0.f);
      }
    }
  }
}

// the kernels: the bodies above without dropout, under the names they have always had, and with it
__global__ void attention_core_fwd_kernel(const float* __restrict__ qkvr, float* __restrict__ Y, int B, int F, int D,
                                          int heads, int use_res) {
  attention_core_fwd_body<false>(qkvr, Y, B, F, D, heads, use_res, AttDrop{});
}
__global__ void attention_core_dropout_fwd_kernel(const float* __restrict__ qkvr, float* __restrict__ Y, int B, int F,
                                                  int D, int heads, int use_res, AttDrop dr) {
  attention_core_fwd_body<true>(qkvr, Y, B, F, D, heads, use_res, dr);
}

template <bool DROP>
__device__ __forceinline__ void attention_core_bwd_body(const float* __restrict__ qkvr, const float* __restrict__ Y,
                                                        const float* __restrict__ dY, float* __restrict__ d_qkvr, int B,
                                                        int F, int D, int heads, int use_res, int mask_in,
                                                        const AttDrop& dr) {
  extern __shared__ float sm[];
  const uint64_t key = DROP ? dropout_key(dr.seed, dr.seed_dev) : 0;
  float* blk = sm;                          // [F][4D] inputs
  float* dz = sm + (size_t)F * 4 * D;       // [F][D]   dLoss / d(pre-relu output)
  float* st = dz + (size_t)F * D;           // [heads*F][3]: max, 1/sum, delta
  const int dh = D / heads;
  const float scale = rsqrtf((float)dh);
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    __syncthreads();
    const float* src = qkvr + (size_t)b * F * 4 * D;
    for (int e = threadIdx.x; e < F * 4 * D; e += blockDim.x) blk[e] = src[e];
    for (int e = threadIdx.x; e < F * D; e += blockDim.x) {
      const size_t o = (size_t)b * F * D + e;
      dz[e] = Y[o] > 0.f ? dY[o] : 0.f;
    }
    __syncthreads();
    const int t = threadIdx.x;
    float* dst = d_qkvr + (size_t)b * F * 4 * D;
    // phase 1: thread (h, i): softmax statistics, delta = dout . out, dQ row, dRes row
    if (t < heads * F) {
      const int h = t / F, i = t - h * F;
      const float* q = blk + (size_t)i * 4 * D + h * dh;
      const float* dout = dz + (size_t)i * D + h * dh;
      float m = -INFINITY;
      for (int j = 0; j < F; ++j) {
        const float* k = blk + (size_t)j * 4 * D + D + h * dh;
        float s = 0.f;
        for (int c = 0; c < dh; ++c) s += q[c] * k[c];
        m = fmaxf(m, s * scale);
      }
      const uint64_t ctr = DROP ? att_counter(dr, key, b, heads, h, F, i) : 0;
      float sum = 0.f, dsum = 0.f;       // dsum = sum_j p_j (dout . v_j)  (un-normalised)
      for (int j = 0; j < F; ++j) {
        const float* k = blk + (size_t)j * 4 * D + D + h * dh;
        const float* v = blk + (size_t)j * 4 * D + 2 * D + h * dh;
        float s = 0.f, dv = 0.f;
        for (int c = 0; c < dh; ++c) {
          s += q[c] * k[c];
          dv += dout[c] * v[c];
        }
        if (DROP) dv *= att_keep(dr, ctr + j);
        const float pj = __expf(s * scale - m);
        sum += pj;
        dsum += pj * dv;
      }
      const float inv = 1.f / sum;
      const float delta = dsum * inv;
      st[t * 3 + 0] = m;
      st[t * 3 + 1] = inv;
      st[t * 3 + 2] = delta;
      float dq[kMaxDh];
      for (int c = 0; c < dh; ++c) dq[c] = 0.f;
      for (int j = 0; j < F; ++j) {
        const float* k = blk + (size_t)j * 4 * D + D + h * dh;
        const float* v = blk + (size_t)j * 4 * D + 2 * D + h * dh;
        float s = 0.f, dv = 0.f;
        for (int c = 0; c < dh; ++c) {
          s += q[c] * k[c];
          dv += dout[c] * v[c];
        }
        if (DROP) dv *= att_keep(dr, ctr + j);
        const float ds = __expf(s * scale - m) * inv * (dv - delta);
        for (int c = 0; c < dh; ++c) dq[c] += ds * k[c];
      }
      float* o = dst + (size_t)i * 4 * D + h * dh;
      const float* res = blk + (size_t)i * 4 * D + 3 * D + h * dh;
      for (int c = 0; c < dh; ++c) {
        o[c] = (mask_in && !(q[c] > 0.f)) ? 0.f : dq[c] * scale;
        o[3 * D + c] = (use_res && !(mask_in && !(res[c] > 0.f))) ? dout[c] : 0.f;
      }
    }
    __syncthreads();
    // phase 2: thread (h, j): dK row, dV row
    if (t < heads * F) {
      const int h = t / F, j = t - h * F;
      const float* k = blk + (size_t)j * 4 * D + D + h * dh;
      const float* v = blk + (size_t)j * 4 * D + 2 * D + h * dh;
      float dk[kMaxDh], dvv[kMaxDh];
      for (int c = 0; c < dh; ++c) {
        dk[c] = 0.f;
        dvv[c] = 0.f;
      }
      for (int i = 0; i < F; ++i) {
        const float* q = blk + (size_t)i * 4 * D + h * dh;
        const float* dout = dz + (size_t)i * D + h * dh;
        const float* s3 = st + (h * F + i) * 3;
        float s = 0.f, dv = 0.f;
        for (int c = 0; c < dh; ++c) {
          s += q[c] * k[c];
          dv += dout[c] * v[c];
        }
        const float pij = __expf(s * scale - s3[0]) * s3[1];
        float pm = pij;                 // the dropped weight w' = w m
        if (DROP) {
          const float mk = att_keep(dr, att_counter(dr, key, b, heads, h, F, i) + j);
          dv *= mk;
          pm *= mk;
        }
        const float ds = pij * (dv - s3[2]);
        for (int c = 0; c < dh; ++c) {
          dk[c] += ds * q[c];
          dvv[c] += pm * dout[c];
        }
      }
      float* o = dst + (size_t)j * 4 * D + h * dh;
      for (int c = 0; c < dh; ++c) {
        o[D + c] = (mask_in && !(k[c] > 0.f)) ? 0.f : dk[c] * scale;
        o[2 * D + c] = (mask_in && !(v[c] > 0.f)) ? 0.f : dvv[c];
      }
    }
  }
}

__global__ void attention_core_bwd_kernel(const float* __restrict__ qkvr, const float* __restrict__ Y,
                                          const float* __restrict__ dY, float* __restrict__ d_qkvr, int B, int F,
                                          int D, int heads, int use_res, int mask_in) {
  attention_core_bwd_body<false>(qkvr, Y, dY, d_qkvr, B, F, D, heads, use_res, mask_in, AttDrop{});
}
__global__ void attention_core_dropout_bwd_kernel(const float* __restrict__ qkvr, const float* __restrict__ Y,
                                                  const float* __restrict__ dY, float* __restrict__ d_qkvr, int B, int F,
                                                  int D, int heads, int use_res, int mask_in, AttDrop dr) {
  attention_core_bwd_body<true>(qkvr, Y, dY, d_qkvr, B, F, D, heads, use_res, mask_in, dr);
}

// ------------------------------------------------------------------------------------------
// The same two kernels with the head width as a template parameter (DH = 1, 2, 4, ... 64): q / dout / k / v rows and
// the per-thread accumulators live in REGISTERS (the generic kernels above index `acc[kMaxDh]` with a run-time bound, i.e.
// from local memory, and every lane re-read its q row from shared memory at a stride of 4D floats = one bank: a 32-way
// conflict on the innermost loop -- 8.6 ms per launch at 65 536 rows x 26 fields x D = 32, 2 % of the HBM rate).  Shared
// rows are padded by 4 floats; key / value reads are warp broadcasts.
// ------------------------------------------------------------------------------------------
// q/k/v/dout slices of DH floats out of shared memory: 128-bit loads when DH is a multiple of 4 (the scalar form costs one
// shared-memory wavefront per float, and with one per FMA the kernels ran at the LDS issue rate: 0.93 / 2.7 ms forward /
// backward per launch at 65 536 rows x 26 fields x 4 heads of 8)
template <int DH>
__device__ __forceinline__ void lds_row(const float* __restrict__ p, float (&o)[DH]) {
  if constexpr (DH % 4 == 0) {
#pragma unroll
    for (int c = 0; c < DH / 4; ++c) {
      const float4 t = *reinterpret_cast<const float4*>(p + 4 * c);
      o[4 * c] = t.x;
      o[4 * c + 1] = t.y;
      o[4 * c + 2] = t.z;
      o[4 * c + 3] = t.w;
    }
  } else if constexpr (DH == 2) {
    const float2 t = *reinterpret_cast<const float2*>(p);
    o[0] = t.x;
    o[1] = t.y;
  } else {
#pragma unroll
    for (int c = 0; c < DH; ++c) o[c] = p[c];
  }
}

template <int DH>
__device__ __forceinline__ void store_row(float* __restrict__ p, const float (&v)[DH]) {
  if constexpr (DH % 4 == 0) {
#pragma unroll
    for (int c = 0; c < DH / 4; ++c)
      *reinterpret_cast<float4*>(p + 4 * c) = make_float4(v[4 * c], v[4 * c + 1], v[4 * c + 2], v[4 * c + 3]);
  } else if constexpr (DH == 2) {
    *reinterpret_cast<float2*>(p) = make_float2(v[0], v[1]);
  } else {
#pragma unroll
    for (int c = 0; c < DH; ++c) p[c] = v[c];
  }
}

// 16-byte asynchronous global -> shared copies: the next batch-row group is requested before the current one is computed
// (with the plain load -> store staging a third of the backward kernel's stall samples sat on the load latency in front of
// the CTA barrier)
__device__ __forceinline__ void cp_async16(float* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

template <int DH, bool DROP>
__device__ __forceinline__ void attention_core_fwd_t_body(const float* __restrict__ qkvr, float* __restrict__ Y, int B, int F,
                                                          int D, int heads, int use_res, int R, int nbuf, const AttDrop& dr) {
  extern __shared__ __align__(16) float sm_all[];     // [nbuf][R][F][4D + 4]
  const int RS = 4 * D + 4;
  const float scale = rsqrtf((float)DH);
  const uint64_t key = DROP ? dropout_key(dr.seed, dr.seed_dev) : 0;
  const int hf = heads * F;
  const int rr = threadIdx.x / hf, t = threadIdx.x - rr * hf;       // batch row of the CTA's group, (head, field)
  const size_t buf_floats = (size_t)R * F * RS;
  auto issue = [&](int b0n, int bufn) {
    const int nrn = min(R, B - b0n);
    float* dst = sm_all + bufn * buf_floats;
    const float4* src = reinterpret_cast<const float4*>(qkvr + (size_t)b0n * F * 4 * D);
    for (int e = threadIdx.x; e < nrn * F * D; e += blockDim.x) {     // D float4 per field row
      const int f = e / D, c4 = e - f * D;                            // f counts field rows across the group
      cp_async16(dst + (size_t)f * RS + 4 * c4, src + e);
    }
    cp_async_commit();
  };
  int buf = 0;
  if ((int)blockIdx.x * R < B) issue(blockIdx.x * R, 0);
  for (int b0 = blockIdx.x * R; b0 < B; b0 += gridDim.x * R) {
    const int nr = min(R, B - b0);
    const int b0n = b0 + gridDim.x * R;
    cp_async_wait_all();
    __syncthreads();                     // this group's block is complete; every thread is done with the other buffer
    if (nbuf == 2 && b0n < B) issue(b0n, buf ^ 1);
    const float* sm = sm_all + buf * buf_floats + (size_t)rr * F * RS;
    const int b = b0 + rr;
    if (rr < nr) {
      const int h = t / F, i = t - h * F;
      float q[DH], acc[DH], kk[DH], vv[DH];
      lds_row<DH>(sm + (size_t)i * RS + h * DH, q);
#pragma unroll
      for (int c = 0; c < DH; ++c) {
        q[c] *= scale;
        acc[c] = 0.f;
      }
      float m = -INFINITY;
      for (int j = 0; j < F; ++j) {
        lds_row<DH>(sm + (size_t)j * RS + D + h * DH, kk);
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < DH; ++c) s = fmaf(q[c], kk[c], s);
        m = fmaxf(m, s);
      }
      float sum = 0.f;
      const uint64_t ctr = DROP ? att_counter(dr, key, b, heads, h, F, i) : 0;
      for (int j = 0; j < F; ++j) {
        const float* k = sm + (size_t)j * RS + D + h * DH;
        lds_row<DH>(k, kk);
        lds_row<DH>(k + D, vv);
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < DH; ++c) s = fmaf(q[c], kk[c], s);
        float pj = __expf(s - m);
        sum += pj;
        if (DROP && att_keep(dr, ctr + j) == 0.f) pj = 0.f;      // the 1 / (1 - rate) of the kept weights: below
#pragma unroll
        for (int c = 0; c < DH; ++c) acc[c] = fmaf(pj, vv[c], acc[c]);
      }
      const float inv = 1.f / sum;
      lds_row<DH>(sm + (size_t)i * RS + 3 * D + h * DH, vv);       // residual
#pragma unroll
      for (int c = 0; c < DH; ++c) {
        float o = acc[c] * inv;
        if (DROP) o *= dr.scale;
        if (use_res) o += vv[c];
        acc[c] = fmaxf(o, 0.f);
      }
      store_row<DH>(Y + ((size_t)b * F + i) * D + h * DH, acc);
    }
    if (nbuf == 2) {
      buf ^= 1;
    } else if (b0n < B) {
      __syncthreads();
      issue(b0n, 0);
    }
  }
}

template <int DH>
__global__ void __launch_bounds__(256) attention_core_fwd_t_kernel(const float* __restrict__ qkvr, float* __restrict__ Y, int B, int F, int D,
                                                                    int heads, int use_res, int R, int nbuf) {
  attention_core_fwd_t_body<DH, false>(qkvr, Y, B, F, D, heads, use_res, R, nbuf, AttDrop{});
}
template <int DH>
__global__ void __launch_bounds__(256) attention_core_dropout_fwd_t_kernel(const float* __restrict__ qkvr, float* __restrict__ Y,
                                                                            int B, int F, int D, int heads, int use_res, int R,
                                                                            int nbuf, AttDrop dr) {
  attention_core_fwd_t_body<DH, true>(qkvr, Y, B, F, D, heads, use_res, R, nbuf, dr);
}

template <int DH, bool DROP>
__device__ __forceinline__ void attention_core_bwd_t_body(const float* __restrict__ qkvr, const float* __restrict__ Y,
                                                          const float* __restrict__ dY, float* __restrict__ d_qkvr, int B,
                                                          int F, int D, int heads, int use_res, int mask_in, int R, int nbuf,
                                                          const AttDrop& dr) {
  extern __shared__ __align__(16) float sm_all[];
  const uint64_t key = DROP ? dropout_key(dr.seed, dr.seed_dev) : 0;
  const int RS = 4 * D + 4, RZ = D + 4;
  const int hf = heads * F;
  const int rr = threadIdx.x / hf, t = threadIdx.x - rr * hf;       // batch row of the CTA's group, (head, field)
  // per buffer: [R][F][4D + 4] inputs | [R][F][D + 4] dY, masked in place to dLoss/d(pre-relu output) | [R][F][D + 4] Y
  const size_t blk_floats = (size_t)R * F * RS, z_floats = (size_t)R * F * RZ;
  const size_t buf_floats = blk_floats + 2 * z_floats;
  float* st = sm_all + nbuf * buf_floats + (size_t)rr * hf * 4;     // [R][heads*F][4]: max, 1/sum, delta, -
  const float scale = rsqrtf((float)DH);
  const int d4 = D / 4;
  auto issue = [&](int b0n, int bufn) {
    const int nrn = min(R, B - b0n);
    float* dst = sm_all + bufn * buf_floats;
    const float4* src = reinterpret_cast<const float4*>(qkvr + (size_t)b0n * F * 4 * D);
    for (int e = threadIdx.x; e < nrn * F * D; e += blockDim.x) {
      const int f = e / D, c4 = e - f * D;                            // f counts field rows across the group
      cp_async16(dst + (size_t)f * RS + 4 * c4, src + e);
    }
    const float4* y4 = reinterpret_cast<const float4*>(Y + (size_t)b0n * F * D);
    const float4* dy4 = reinterpret_cast<const float4*>(dY + (size_t)b0n * F * D);
    for (int e = threadIdx.x; e < nrn * F * d4; e += blockDim.x) {
      const int f = e / d4, c4 = e - f * d4;
      cp_async16(dst + blk_floats + (size_t)f * RZ + 4 * c4, dy4 + e);
      cp_async16(dst + blk_floats + z_floats + (size_t)f * RZ + 4 * c4, y4 + e);
    }
    cp_async_commit();
  };
  int buf = 0;
  if ((int)blockIdx.x * R < B) issue(blockIdx.x * R, 0);
  for (int b0 = blockIdx.x * R; b0 < B; b0 += gridDim.x * R) {
    const int nr = min(R, B - b0);
    const int b0n = b0 + gridDim.x * R;
    cp_async_wait_all();
    __syncthreads();                     // this group's blocks are complete; every thread is done with the other buffer
    if (nbuf == 2 && b0n < B) issue(b0n, buf ^ 1);
    float* bufp = sm_all + buf * buf_floats;
    for (int e = threadIdx.x; e < nr * F * d4; e += blockDim.x) {     // relu mask of the attention output
      const int f = e / d4, c4 = e - f * d4;
      float4* gp = reinterpret_cast<float4*>(bufp + blk_floats + (size_t)f * RZ + 4 * c4);
      const float4 y = *reinterpret_cast<const float4*>(bufp + blk_floats + z_floats + (size_t)f * RZ + 4 * c4);
      float4 g = *gp;
      g.x = y.x > 0.f ? g.x : 0.f;
      g.y = y.y > 0.f ? g.y : 0.f;
      g.z = y.z > 0.f ? g.z : 0.f;
      g.w = y.w > 0.f ? g.w : 0.f;
      *gp = g;
    }
    __syncthreads();
    const float* blk = bufp + (size_t)rr * F * RS;
    const float* dz = bufp + blk_floats + (size_t)rr * F * RZ;
    const int b = b0 + rr;
    const bool live = rr < nr;
    float* dst = d_qkvr + (size_t)b * F * 4 * D;
    // phase 1: thread (h, i): softmax statistics, delta = dout . out, dQ row, dRes row
    if (live) {
      const int h = t / F, i = t - h * F;
      float q[DH], dout[DH], dq[DH], kk[DH], vv[DH];
      lds_row<DH>(blk + (size_t)i * RS + h * DH, q);
      lds_row<DH>(dz + (size_t)i * RZ + h * DH, dout);
#pragma unroll
      for (int c = 0; c < DH; ++c) {
        q[c] *= scale;
        dq[c] = 0.f;
      }
      float m = -INFINITY;
      for (int j = 0; j < F; ++j) {
        lds_row<DH>(blk + (size_t)j * RS + D + h * DH, kk);
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < DH; ++c) s = fmaf(q[c], kk[c], s);
        m = fmaxf(m, s);
      }
      // one sweep: with p_j = exp(s_j - m) un-normalised, dQ = (sum_j p_j dv_j k_j - delta sum_j p_j k_j) / sum_j p_j
      float sum = 0.f, dsum = 0.f;       // dsum = sum_j p_j (dout . v_j)
      float pk[DH];
#pragma unroll
      for (int c = 0; c < DH; ++c) pk[c] = 0.f;
      const uint64_t ctr = DROP ? att_counter(dr, key, b, heads, h, F, i) : 0;
      for (int j = 0; j < F; ++j) {
        const float* k = blk + (size_t)j * RS + D + h * DH;
        lds_row<DH>(k, kk);
        lds_row<DH>(k + D, vv);
        float s = 0.f, dv = 0.f;
#pragma unroll
        for (int c = 0; c < DH; ++c) {
          s = fmaf(q[c], kk[c], s);
          dv = fmaf(dout[c], vv[c], dv);
        }
        if (DROP) dv *= att_keep(dr, ctr + j);
        const float pj = __expf(s - m);
        const float w = pj * dv;
        sum += pj;
        dsum += w;
#pragma unroll
        for (int c = 0; c < DH; ++c) {
          dq[c] = fmaf(w, kk[c], dq[c]);
          pk[c] = fmaf(pj, kk[c], pk[c]);
        }
      }
      const float inv = 1.f / sum;
      const float delta = dsum * inv;
      *reinterpret_cast<float4*>(st + t * 4) = make_float4(m, inv, delta, 0.f);
      float* o = dst + (size_t)i * 4 * D + h * DH;
      if (mask_in) lds_row<DH>(blk + (size_t)i * RS + 3 * D + h * DH, vv);      // residual projection (relu output)
#pragma unroll
      for (int c = 0; c < DH; ++c) {
        dq[c] = (dq[c] - delta * pk[c]) * inv * scale;
        if (!use_res) dout[c] = 0.f;
        if (mask_in) {                    // gradient w.r.t. the PRE-relu projections: zero where the relu output is zero
          if (!(q[c] > 0.f)) dq[c] = 0.f;
          if (!(vv[c] > 0.f)) dout[c] = 0.f;
        }
      }
      store_row<DH>(o, dq);
      store_row<DH>(o + 3 * D, dout);
    }
    __syncthreads();
    // phase 2: thread (h, j): dK row, dV row
    if (live) {
      const int h = t / F, j = t - h * F;
      float k[DH], v[DH], dk[DH], dvv[DH], q[DH], dout[DH];
      lds_row<DH>(blk + (size_t)j * RS + D + h * DH, k);
      lds_row<DH>(blk + (size_t)j * RS + 2 * D + h * DH, v);
#pragma unroll
      for (int c = 0; c < DH; ++c) {
        dk[c] = 0.f;
        dvv[c] = 0.f;
      }
      const uint64_t ctr = DROP ? att_counter(dr, key, b, heads, h, F, 0) + j : 0;     // weight (b, h, i, j) at + i * F
      for (int i = 0; i < F; ++i) {
        lds_row<DH>(blk + (size_t)i * RS + h * DH, q);
        lds_row<DH>(dz + (size_t)i * RZ + h * DH, dout);
        const float4 s3 = *reinterpret_cast<const float4*>(st + (h * F + i) * 4);
        float s = 0.f, dv = 0.f;
#pragma unroll
        for (int c = 0; c < DH; ++c) {
          s = fmaf(q[c], k[c], s);
          dv = fmaf(dout[c], v[c], dv);
        }
        const float pij = __expf(s * scale - s3.x) * s3.y;
        float pm = pij;                 // the dropped weight w' = w m
        if (DROP) {
          const float mk = att_keep(dr, ctr + (uint64_t)i * F);
          dv *= mk;
          pm *= mk;
        }
        const float ds = pij * (dv - s3.z);
#pragma unroll
        for (int c = 0; c < DH; ++c) {
          dk[c] = fmaf(ds, q[c], dk[c]);
          dvv[c] = fmaf(pm, dout[c], dvv[c]);
        }
      }
      float* o = dst + (size_t)j * 4 * D + h * DH;
#pragma unroll
      for (int c = 0; c < DH; ++c) {
        dk[c] *= scale;
        if (mask_in) {
          if (!(k[c] > 0.f)) dk[c] = 0.f;
          if (!(v[c] > 0.f)) dvv[c] = 0.f;
        }
      }
      store_row<DH>(o + D, dk);
      store_row<DH>(o + 2 * D, dvv);
    }
    if (nbuf == 2) {
      buf ^= 1;
    } else if (b0n < B) {
      __syncthreads();
      issue(b0n, 0);
    }
  }
}

template <int DH>
__global__ void __launch_bounds__(256) attention_core_bwd_t_kernel(const float* __restrict__ qkvr, const float* __restrict__ Y,
                                                                    const float* __restrict__ dY, float* __restrict__ d_qkvr, int B,
                                                                    int F, int D, int heads, int use_res, int mask_in,
                                                                    int R, int nbuf) {
  attention_core_bwd_t_body<DH, false>(qkvr, Y, dY, d_qkvr, B, F, D, heads, use_res, mask_in, R, nbuf, AttDrop{});
}
template <int DH>
__global__ void __launch_bounds__(256) attention_core_dropout_bwd_t_kernel(const float* __restrict__ qkvr,
                                                                            const float* __restrict__ Y,
                                                                            const float* __restrict__ dY,
                                                                            float* __restrict__ d_qkvr, int B, int F, int D,
                                                                            int heads, int use_res, int mask_in, int R, int nbuf,
                                                                            AttDrop dr) {
  attention_core_bwd_t_body<DH, true>(qkvr, Y, dY, d_qkvr, B, F, D, heads, use_res, mask_in, R, nbuf, dr);
}

}  // namespace dtb

using namespace dtb;

namespace {
constexpr size_t kPnnTSmemMax = 200 * 1024;
constexpr size_t kAttSmemMax = 220 * 1024;
// the (row, field) kernels need a power-of-two width in 4..32 and 16-byte aligned rows
// attention kernels: batch rows per CTA so that a CTA has about 128 (head, field) threads, two shared-memory buffers
// (the next group's loads run under this group's arithmetic) unless one row's blocks are too large for that
void att_plan(int hf, size_t row_bytes, size_t stat_bytes, int& R, int& nbuf) {
  const size_t budget = 96 * 1024, limit = 200 * 1024;
  nbuf = 2 * row_bytes + stat_bytes <= limit ? 2 : 1;
  R = hf >= 128 ? 1 : 128 / hf;
  while (R > 1 && (size_t)R * (nbuf * row_bytes + stat_bytes) > budget) --R;
}
int att_threads(int R, int hf) {
  const int t = (R * hf + 31) / 32 * 32;
  return t < 64 ? 64 : t;
}
bool pnn_t_shape(int D, const void* table, const void* grad_table) {
  if (D != 4 && D != 8 && D != 16 && D != 32) return false;
  if (reinterpret_cast<uintptr_t>(table) & 15) return false;
  if (grad_table && (reinterpret_cast<uintptr_t>(grad_table) & 15)) return false;
  return true;
}

// the attention launches; DROP = false launches the kernels that hold no dropout code
template <bool DROP>
int attention_fwd(const float* qkvr, float* Y, int B, int F, int D, int heads, int use_residual, const AttDrop& dr,
                  void* stream) {
  if (B == 0) return DTB_OK;
  const int threads = (heads * F + 31) / 32 * 32;
  int grid = sm_count() * 8;
  if (grid > B) grid = B;
  const int dh = D / heads;
  const int nthr = threads < 64 ? 64 : threads;
  if (D % 4 == 0 && nthr <= 256 && ((reinterpret_cast<uintptr_t>(qkvr) | reinterpret_cast<uintptr_t>(Y)) & 15) == 0) {
    const size_t row_bytes = (size_t)F * (4 * D + 4) * sizeof(float);
    int R, nbuf;
    att_plan(heads * F, row_bytes, 0, R, nbuf);
    const int nthr_t = att_threads(R, heads * F);
    const size_t smem_t = (size_t)nbuf * R * row_bytes;
    if (grid > ceil_div(B, R)) grid = ceil_div(B, R);
    if (smem_t <= kAttSmemMax) {
#define DTB_ATT_FWD(DHV)                                                                                                 \
  case DHV:                                                                                                              \
    if constexpr (DROP) {                                                                                                \
      DTB_CUDA_OK(cudaFuncSetAttribute(attention_core_dropout_fwd_t_kernel<DHV>,                                         \
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_t));                       \
      attention_core_dropout_fwd_t_kernel<DHV><<<grid, nthr_t, smem_t, (cudaStream_t)stream>>>(                          \
          qkvr, Y, B, F, D, heads, use_residual, R, nbuf, dr);                                                           \
    } else {                                                                                                             \
      DTB_CUDA_OK(cudaFuncSetAttribute(attention_core_fwd_t_kernel<DHV>, cudaFuncAttributeMaxDynamicSharedMemorySize,    \
                                       (int)smem_t));                                                                    \
      attention_core_fwd_t_kernel<DHV><<<grid, nthr_t, smem_t, (cudaStream_t)stream>>>(qkvr, Y, B, F, D, heads,          \
                                                                                       use_residual, R, nbuf);           \
    }                                                                                                                    \
    DTB_LAUNCH_OK();                                                                                                     \
    return DTB_OK;
    switch (dh) {
      DTB_ATT_FWD(1) DTB_ATT_FWD(2) DTB_ATT_FWD(4) DTB_ATT_FWD(8) DTB_ATT_FWD(16) DTB_ATT_FWD(32) DTB_ATT_FWD(64)
      default: break;
    }
    }
#undef DTB_ATT_FWD
  }
  const size_t smem = (size_t)F * 4 * D * sizeof(float);
  if constexpr (DROP) {
    DTB_CUDA_OK(cudaFuncSetAttribute(attention_core_dropout_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)smem));
    attention_core_dropout_fwd_kernel<<<grid, nthr, smem, (cudaStream_t)stream>>>(qkvr, Y, B, F, D, heads, use_residual,
                                                                                  dr);
  } else {
    DTB_CUDA_OK(cudaFuncSetAttribute(attention_core_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attention_core_fwd_kernel<<<grid, nthr, smem, (cudaStream_t)stream>>>(qkvr, Y, B, F, D, heads, use_residual);
  }
  DTB_LAUNCH_OK();
  return DTB_OK;
}

template <bool DROP>
int attention_bwd(const float* qkvr, const float* Y, const float* dY, float* d_qkvr, int B, int F, int D, int heads,
                  int use_residual, int mask_relu_inputs, const AttDrop& dr, void* stream) {
  if (B == 0) return DTB_OK;
  const int threads = (heads * F + 31) / 32 * 32;
  int grid = sm_count() * 8;
  if (grid > B) grid = B;
  const int dh = D / heads;
  const int nthr = threads < 64 ? 64 : threads;
  if (D % 4 == 0 && nthr <= 256 &&
      ((reinterpret_cast<uintptr_t>(qkvr) | reinterpret_cast<uintptr_t>(Y) | reinterpret_cast<uintptr_t>(dY) |
        reinterpret_cast<uintptr_t>(d_qkvr)) & 15) == 0) {
    const size_t row_bytes = ((size_t)F * (4 * D + 4) + 2 * (size_t)F * (D + 4)) * sizeof(float);
    const size_t stat_bytes = (size_t)heads * F * 4 * sizeof(float);
    int R, nbuf;
    att_plan(heads * F, row_bytes, stat_bytes, R, nbuf);
    const int nthr_t = att_threads(R, heads * F);
    const size_t smem_t = (size_t)R * (nbuf * row_bytes + stat_bytes);
    if (grid > ceil_div(B, R)) grid = ceil_div(B, R);
    if (smem_t <= kAttSmemMax) {
#define DTB_ATT_BWD(DHV)                                                                                                 \
  case DHV:                                                                                                              \
    if constexpr (DROP) {                                                                                                \
      DTB_CUDA_OK(cudaFuncSetAttribute(attention_core_dropout_bwd_t_kernel<DHV>,                                         \
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_t));                       \
      attention_core_dropout_bwd_t_kernel<DHV><<<grid, nthr_t, smem_t, (cudaStream_t)stream>>>(                          \
          qkvr, Y, dY, d_qkvr, B, F, D, heads, use_residual, mask_relu_inputs, R, nbuf, dr);                             \
    } else {                                                                                                             \
      DTB_CUDA_OK(cudaFuncSetAttribute(attention_core_bwd_t_kernel<DHV>, cudaFuncAttributeMaxDynamicSharedMemorySize,    \
                                       (int)smem_t));                                                                    \
      attention_core_bwd_t_kernel<DHV><<<grid, nthr_t, smem_t, (cudaStream_t)stream>>>(                                  \
          qkvr, Y, dY, d_qkvr, B, F, D, heads, use_residual, mask_relu_inputs, R, nbuf);                                 \
    }                                                                                                                    \
    DTB_LAUNCH_OK();                                                                                                     \
    return DTB_OK;
    switch (dh) {
      DTB_ATT_BWD(1) DTB_ATT_BWD(2) DTB_ATT_BWD(4) DTB_ATT_BWD(8) DTB_ATT_BWD(16) DTB_ATT_BWD(32)
      default: break;
    }
    // heads of 64 already spill at 255 registers without dropout; with the mask's 64-bit counters on top ptxas gives up
    // (32 registers, 10 KB of spill traffic per thread), so dropout at that width runs the any-shape kernel below
    if constexpr (!DROP) switch (dh) {
      DTB_ATT_BWD(64)
      default: break;
    }
    }
#undef DTB_ATT_BWD
  }
  const size_t smem = ((size_t)F * 5 * D + (size_t)heads * F * 3) * sizeof(float);
  if constexpr (DROP) {
    DTB_CUDA_OK(cudaFuncSetAttribute(attention_core_dropout_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)smem));
    attention_core_dropout_bwd_kernel<<<grid, nthr, smem, (cudaStream_t)stream>>>(qkvr, Y, dY, d_qkvr, B, F, D, heads,
                                                                                  use_residual, mask_relu_inputs, dr);
  } else {
    DTB_CUDA_OK(cudaFuncSetAttribute(attention_core_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attention_core_bwd_kernel<<<grid, nthr, smem, (cudaStream_t)stream>>>(qkvr, Y, dY, d_qkvr, B, F, D, heads,
                                                                          use_residual, mask_relu_inputs);
  }
  DTB_LAUNCH_OK();
  return DTB_OK;
}
}  // namespace

extern "C" {

int dtb_pnn_fwd(const int32_t* idx, const float* table, const int64_t* row_offsets, const float* op_kernel,
                float* ip, float* op, int B, int F, int D, int kernel_type, int* status, void* stream) {
  DTB_CHECK_ARG(idx && table && row_offsets, "NULL argument");
  DTB_CHECK_ARG(F >= 2 && D >= 1 && D <= kMaxD && B >= 0, "need F >= 2, 1 <= D <= 64");
  DTB_CHECK_ARG(kernel_type >= 0 && kernel_type <= 2, "kernel_type must be 0 (mat), 1 (vec) or 2 (num)");
  DTB_CHECK_ARG(!op || op_kernel, "outer product requested without a kernel");
  if (B == 0 || (!ip && !op)) return DTB_OK;
  const int P = F * (F - 1) / 2;
  if (P > 1024) {
    set_error("dtb_pnn_fwd: %d pairs exceed one CTA", P);
    return DTB_ERR_UNSUPPORTED;
  }
  {
    const size_t per = kernel_type == 0 ? (size_t)D * D : (kernel_type == 1 ? (size_t)D : 1);
    const size_t smem_t = op ? (size_t)(F - 1) * per * sizeof(float) : 0;
    if (pnn_t_shape(D, table, nullptr) && smem_t <= kPnnTSmemMax) {
      // chunk groups: about 8 resident CTAs per SM in total, each CTA amortising its kernel-slice staging over its chunks
      int groups = ceil_div(sm_count() * 8, F - 1);
      if (groups > ceil_div(B, kPnnTRows)) groups = ceil_div(B, kPnnTRows);
      const dim3 grid(F - 1, groups);
#define DTB_PNN_FWD(DV)                                                                                                  \
  case DV:                                                                                                               \
    DTB_CUDA_OK(cudaFuncSetAttribute(pnn_fwd_t_kernel<DV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_t));  \
    pnn_fwd_t_kernel<DV><<<grid, kPnnTRows, smem_t, (cudaStream_t)stream>>>(idx, table, row_offsets, op_kernel, ip, op,  \
                                                                            B, F, P, kernel_type, status);              \
    break;
      switch (D) { DTB_PNN_FWD(4) DTB_PNN_FWD(8) DTB_PNN_FWD(16) DTB_PNN_FWD(32) }
#undef DTB_PNN_FWD
      DTB_LAUNCH_OK();
      return DTB_OK;
    }
  }
  const int threads = (P + 31) / 32 * 32;
  const size_t smem = (size_t)kPnnRows * F * D * sizeof(float);
  DTB_CUDA_OK(cudaFuncSetAttribute(pnn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  pnn_fwd_kernel<<<ceil_div(B, kPnnRows), threads, smem, (cudaStream_t)stream>>>(idx, table, row_offsets, op_kernel,
                                                                                 ip, op, B, F, D, P, kernel_type, status);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_pnn_bwd(const int32_t* idx, const float* table, const int64_t* row_offsets, const float* op_kernel,
                const float* d_ip, const float* d_op, float* grad_table, float* d_op_kernel, int B, int F, int D,
                int kernel_type, void* stream) {
  DTB_CHECK_ARG(idx && table && row_offsets && grad_table, "NULL argument");
  DTB_CHECK_ARG(F >= 2 && D >= 1 && D <= kMaxD && B >= 0, "need F >= 2, 1 <= D <= 64");
  DTB_CHECK_ARG(!d_op || (op_kernel && d_op_kernel), "outer product gradient without kernel buffers");
  if (B == 0 || (!d_ip && !d_op)) return DTB_OK;
  const int P = F * (F - 1) / 2;
  if (P > 1024) {        // the forward's limit: the generic kernels below run one thread per pair
    set_error("dtb_pnn_bwd: %d pairs exceed one CTA", P);
    return DTB_ERR_UNSUPPORTED;
  }
  const int threads = (P + 31) / 32 * 32;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t per = kernel_type == 0 ? (size_t)D * D : (kernel_type == 1 ? (size_t)D : 1);
  const size_t smem_t = d_op ? (size_t)(F - 1) * per * sizeof(float) : 0;
  const bool t_shape = pnn_t_shape(D, table, grad_table) && smem_t <= kPnnTSmemMax;
  if (t_shape) {
    int groups = ceil_div(sm_count() * 8, F);
    if (groups > ceil_div(B, kPnnTRows)) groups = ceil_div(B, kPnnTRows);
    const dim3 grid(F, groups);
#define DTB_PNN_DE(DV)                                                                                                   \
  case DV:                                                                                                               \
    DTB_CUDA_OK(cudaFuncSetAttribute(pnn_bwd_de_t_kernel<DV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_t)); \
    pnn_bwd_de_t_kernel<DV><<<grid, kPnnTRows, smem_t, st>>>(idx, table, row_offsets, op_kernel, d_ip, d_op, grad_table, \
                                                             B, F, P, kernel_type);                                     \
    break;
    switch (D) { DTB_PNN_DE(4) DTB_PNN_DE(8) DTB_PNN_DE(16) DTB_PNN_DE(32) }
#undef DTB_PNN_DE
  } else {
    const size_t smem = (size_t)2 * kPnnRows * F * D * sizeof(float);
    DTB_CUDA_OK(cudaFuncSetAttribute(pnn_bwd_de_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    pnn_bwd_de_kernel<<<ceil_div(B, kPnnRows), threads, smem, st>>>(idx, table, row_offsets, op_kernel, d_ip, d_op,
                                                                    grad_table, B, F, D, P, kernel_type);
  }
  DTB_LAUNCH_OK();
  if (d_op && kernel_type == 0 && t_shape && (reinterpret_cast<uintptr_t>(d_op_kernel) & 15) == 0) {
    const int pg = 256 / D, groups = ceil_div(P, pg);
    int R = 32;
    while (R > 4 && (size_t)R * (F * D + pg) * sizeof(float) > kPnnTSmemMax / 2) R /= 2;
    const size_t smem_k = (size_t)R * (F * D + pg) * sizeof(float);
    if (smem_k <= kPnnTSmemMax) {
      int row_groups = ceil_div(sm_count() * 2, groups);
      if (row_groups > ceil_div(B, R)) row_groups = ceil_div(B, R);
      const int rows_per_cta = ceil_div(ceil_div(B, row_groups), R) * R;
      const dim3 grid(groups, ceil_div(B, rows_per_cta));
#define DTB_PNN_DK(DV)                                                                                                   \
  case DV:                                                                                                               \
    DTB_CUDA_OK(cudaFuncSetAttribute(pnn_bwd_dk_t_kernel<DV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_k)); \
    pnn_bwd_dk_t_kernel<DV><<<grid, 256, smem_k, st>>>(idx, table, row_offsets, d_op, d_op_kernel, B, F, P, rows_per_cta, \
                                                       R);                                                              \
    break;
      switch (D) { DTB_PNN_DK(4) DTB_PNN_DK(8) DTB_PNN_DK(16) DTB_PNN_DK(32) }
#undef DTB_PNN_DK
      DTB_LAUNCH_OK();
      return DTB_OK;
    }
  }
  if (d_op) {
    int ctas = sm_count() * 2;
    if (ctas > B) ctas = B;
    const int rows_per_cta = ceil_div(B, ctas);
    ctas = ceil_div(B, rows_per_cta);
    pnn_bwd_dk_kernel<<<ctas, threads, 0, st>>>(idx, table, row_offsets, d_op, d_op_kernel, B, F, D, P, kernel_type,
                                                rows_per_cta);
    DTB_LAUNCH_OK();
  }
  return DTB_OK;
}

#define DTB_ATT_CHECK_SHAPE()                                                                                          \
  DTB_CHECK_ARG(B >= 0 && F >= 1 && D >= 1 && heads >= 1 && D % heads == 0, "bad shape (num_heads must divide D)");     \
  DTB_CHECK_ARG(D / heads <= kMaxDh && heads * F <= 1024, "head width <= 64 and heads*fields <= 1024")

int dtb_attention_core_fwd(const float* qkvr, float* Y, int B, int F, int D, int heads, int use_residual,
                           void* stream) {
  DTB_CHECK_ARG(qkvr && Y, "NULL argument");
  DTB_ATT_CHECK_SHAPE();
  return attention_fwd<false>(qkvr, Y, B, F, D, heads, use_residual, AttDrop{}, stream);
}

int dtb_attention_core_bwd(const float* qkvr, const float* Y, const float* dY, float* d_qkvr, int B, int F, int D,
                           int heads, int use_residual, int mask_relu_inputs, void* stream) {
  DTB_CHECK_ARG(qkvr && Y && dY && d_qkvr, "NULL argument");
  DTB_ATT_CHECK_SHAPE();
  return attention_bwd<false>(qkvr, Y, dY, d_qkvr, B, F, D, heads, use_residual, mask_relu_inputs, AttDrop{}, stream);
}

int dtb_attention_core_dropout_fwd(const float* qkvr, float* Y, int B, int F, int D, int heads, int use_residual,
                                   float rate, unsigned long long seed, const unsigned long long* seed_dev,
                                   long long row_offset, void* stream) {
  DTB_CHECK_ARG(qkvr && Y, "NULL argument");
  DTB_ATT_CHECK_SHAPE();
  DTB_CHECK_ARG(rate >= 0.f && rate < 1.f && row_offset >= 0, "rate must be in [0, 1), row_offset >= 0");
  if (rate == 0.f) return attention_fwd<false>(qkvr, Y, B, F, D, heads, use_residual, AttDrop{}, stream);
  const AttDrop dr{dropout_threshold(rate), 1.f / (1.f - rate), seed, seed_dev, row_offset};
  return attention_fwd<true>(qkvr, Y, B, F, D, heads, use_residual, dr, stream);
}

int dtb_attention_core_dropout_bwd(const float* qkvr, const float* Y, const float* dY, float* d_qkvr, int B, int F,
                                   int D, int heads, int use_residual, int mask_relu_inputs, float rate,
                                   unsigned long long seed, const unsigned long long* seed_dev, long long row_offset,
                                   void* stream) {
  DTB_CHECK_ARG(qkvr && Y && dY && d_qkvr, "NULL argument");
  DTB_ATT_CHECK_SHAPE();
  DTB_CHECK_ARG(rate >= 0.f && rate < 1.f && row_offset >= 0, "rate must be in [0, 1), row_offset >= 0");
  if (rate == 0.f)
    return attention_bwd<false>(qkvr, Y, dY, d_qkvr, B, F, D, heads, use_residual, mask_relu_inputs, AttDrop{}, stream);
  const AttDrop dr{dropout_threshold(rate), 1.f / (1.f - rate), seed, seed_dev, row_offset};
  return attention_bwd<true>(qkvr, Y, dY, d_qkvr, B, F, D, heads, use_residual, mask_relu_inputs, dr, stream);
}
#undef DTB_ATT_CHECK_SHAPE

}  // extern "C"
