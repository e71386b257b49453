// Categorical-embedding gather fused into the HBM-bound consumers:
//   linear (deepnets.py:43-66) + FM (layers.py:53-62), flatten/concat (deepmodel.py:269-278),
//   plus the plain gather / scatter-add forms of MultiColumnEmbedding (layers.py:889-904).
//
// HBM roofline per batch row (F=26, D=16, C=13): 104 B ids + 1664 B table rows + 52 B dense + 8 B
// out = 1828 B, ~2.2 kFLOP -> bandwidth bound.  The fast path keeps the whole (F x D) block of a
// row in the registers of one warp: lane L owns float4 slot L, L+32, ... of the row-major block, so
// its slot%Q (Q = D/4) is fixed and the sum over fields is a lane-strided register sum followed by
// log2(32/Q) shuffles.  ROWS rows are processed per warp pass to keep >= 8 independent 16-byte
// loads in flight per lane (random 64-byte rows: latency-, not coalescing-, limited).
#include "dtb_common.cuh"

namespace dtb {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kRowsPerPass = 2;   // batch rows a warp handles per pass
constexpr int kChunk = 4;         // float4 slots per lane per row per chunk

__device__ __forceinline__ bool pow2(int x) { return x > 0 && (x & (x - 1)) == 0; }

// ------------------------------------------------------------------------------------------
// fast path: D % 4 == 0, Q = D/4 in {1,2,4,8,16,32}
// ------------------------------------------------------------------------------------------
template <int NCH>
__global__ void __launch_bounds__(kThreads)
fm_linear_fwd_vec(const int32_t* __restrict__ idx, const float* __restrict__ table,
                  const int64_t* __restrict__ row_offsets, const float* __restrict__ dense,
                  const float* __restrict__ w_lin, float* __restrict__ out_lin,
                  float* __restrict__ out_fm, int B, int F, int D, int C, int* status) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * kWarps) + (threadIdx.x >> 5);
  const int n_warps = gridDim.x * kWarps;
  const int Q = D >> 2;
  const int S = F * Q;
  const float qscale = (float)Q * (1.0f / 32.0f);
  // A lane's float4 slots (lane, lane+32, ...) are the same (field, quarter) pairs for EVERY batch row:
  // resolve field, table base pointer, vocabulary size and linear weight once, outside the row loop.
  // NCH chunks of 4 slots per lane cover F*D/4 <= NCH*128 float4 per row (wider rows: fm_linear_fwd_vec_loop).
  constexpr int kMaxSlots = NCH * kChunk;
  const float* sbase[kMaxSlots];
  int sfield[kMaxSlots];
  int svocab[kMaxSlots];
  float swl[kMaxSlots];
#pragma unroll
  for (int c = 0; c < kMaxSlots; ++c) {
    const int slot = c * 32 + lane;
    sfield[c] = -1;
    svocab[c] = 0;
    swl[c] = 0.f;
    sbase[c] = table;
    if (slot < S) {
      const int f = slot / Q;
      const int64_t lo = row_offsets[f];
      sfield[c] = f;
      svocab[c] = (int)(row_offsets[f + 1] - lo);
      sbase[c] = table + lo * D + ((slot - f * Q) << 2);
      swl[c] = out_lin ? __ldg(w_lin + f) : 0.f;
    }
  }

  for (int row0 = warp * kRowsPerPass; row0 < B; row0 += n_warps * kRowsPerPass) {
    float4 acc[kRowsPerPass];
    float sq[kRowsPerPass], lin[kRowsPerPass];
#pragma unroll
    for (int r = 0; r < kRowsPerPass; ++r) {
      acc[r] = make_float4(0.f, 0.f, 0.f, 0.f);
      sq[r] = 0.f;
      lin[r] = 0.f;
    }
#pragma unroll
    for (int cc = 0; cc < NCH; ++cc) {
      {
        int id[kRowsPerPass][kChunk];
#pragma unroll
        for (int r = 0; r < kRowsPerPass; ++r)
#pragma unroll
          for (int c = 0; c < kChunk; ++c) {
            const int k = cc * kChunk + c;
            id[r][c] = -1;
            if (sfield[k] >= 0 && row0 + r < B) id[r][c] = __ldg(idx + (int64_t)(row0 + r) * F + sfield[k]);
          }
        float4 e[kRowsPerPass][kChunk];
#pragma unroll
        for (int r = 0; r < kRowsPerPass; ++r)
#pragma unroll
          for (int c = 0; c < kChunk; ++c) {
            const int k = cc * kChunk + c;
            e[r][c] = make_float4(0.f, 0.f, 0.f, 0.f);
            if ((unsigned)id[r][c] < (unsigned)svocab[k]) {
              e[r][c] = ldg_stream_f4(sbase[k] + (int64_t)id[r][c] * D);
            } else if (status && sfield[k] >= 0 && row0 + r < B) {
              atomicOr(status, 1 << (sfield[k] & 31));
            }
          }
#pragma unroll
        for (int r = 0; r < kRowsPerPass; ++r)
#pragma unroll
          for (int c = 0; c < kChunk; ++c) {
            const float4 v = e[r][c];
            acc[r].x += v.x; acc[r].y += v.y; acc[r].z += v.z; acc[r].w += v.w;
            sq[r] += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
            lin[r] += swl[cc * kChunk + c] * ((v.x + v.y) + (v.z + v.w));
          }
      }
    }
#pragma unroll
    for (int r = 0; r < kRowsPerPass; ++r) {
      const int row = row0 + r;
      if (row >= B) break;   // warp-uniform
      if (out_fm) {
        float4 a = acc[r];
        for (int o = 16; o >= Q; o >>= 1) {
          a.x += __shfl_xor_sync(0xffffffffu, a.x, o);
          a.y += __shfl_xor_sync(0xffffffffu, a.y, o);
          a.z += __shfl_xor_sync(0xffffffffu, a.z, o);
          a.w += __shfl_xor_sync(0xffffffffu, a.w, o);
        }
        // every lane of a q-class now holds the class total: scale by Q/32 so the warp sum counts it once
        const float s2 = (a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w) * qscale;
        const float v = warp_sum(s2 - sq[r]);
        if (lane == 0) out_fm[row] = 0.5f * v;
      }
      if (out_lin) {
        float l = lin[r];
        for (int c = lane; c < C; c += 32) l += __ldg(w_lin + F + c) * __ldg(dense + (int64_t)row * C + c);
        l = warp_sum(l);
        if (lane == 0) out_lin[row] = l;
      }
    }
  }
}

// any-width variant (slots resolved inside the row loop)
__global__ void __launch_bounds__(kThreads)
fm_linear_fwd_vec_loop(const int32_t* __restrict__ idx, const float* __restrict__ table,
                  const int64_t* __restrict__ row_offsets, const float* __restrict__ dense,
                  const float* __restrict__ w_lin, float* __restrict__ out_lin,
                  float* __restrict__ out_fm, int B, int F, int D, int C, int* status) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * kWarps) + (threadIdx.x >> 5);
  const int n_warps = gridDim.x * kWarps;
  const int Q = D >> 2;
  const int S = F * Q;
  const float qscale = (float)Q * (1.0f / 32.0f);

  for (int row0 = warp * kRowsPerPass; row0 < B; row0 += n_warps * kRowsPerPass) {
    float4 acc[kRowsPerPass];
    float sq[kRowsPerPass], lin[kRowsPerPass];
#pragma unroll
    for (int r = 0; r < kRowsPerPass; ++r) {
      acc[r] = make_float4(0.f, 0.f, 0.f, 0.f);
      sq[r] = 0.f;
      lin[r] = 0.f;
    }
    for (int s0 = 0; s0 < S; s0 += 32 * kChunk) {
      int64_t base[kRowsPerPass][kChunk];
      float wl[kChunk];
#pragma unroll
      for (int c = 0; c < kChunk; ++c) {
        const int slot = s0 + c * 32 + lane;
        const int f = slot / Q;
        wl[c] = (slot < S && out_lin) ? __ldg(w_lin + f) : 0.f;
#pragma unroll
        for (int r = 0; r < kRowsPerPass; ++r) {
          const int row = row0 + r;
          base[r][c] = -1;
          if (slot < S && row < B) {
            const int id = __ldg(idx + (int64_t)row * F + f);
            const int64_t rb = table_row(row_offsets, f, id, D, status);
            base[r][c] = rb < 0 ? -1 : rb + ((slot - f * Q) << 2);
          }
        }
      }
      float4 e[kRowsPerPass][kChunk];
#pragma unroll
      for (int r = 0; r < kRowsPerPass; ++r)
#pragma unroll
        for (int c = 0; c < kChunk; ++c)
          e[r][c] = base[r][c] >= 0 ? ldg_stream_f4(table + base[r][c]) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int r = 0; r < kRowsPerPass; ++r)
#pragma unroll
        for (int c = 0; c < kChunk; ++c) {
          const float4 v = e[r][c];
          acc[r].x += v.x; acc[r].y += v.y; acc[r].z += v.z; acc[r].w += v.w;
          sq[r] += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
          lin[r] += wl[c] * ((v.x + v.y) + (v.z + v.w));
        }
    }
#pragma unroll
    for (int r = 0; r < kRowsPerPass; ++r) {
      const int row = row0 + r;
      if (row >= B) break;   // warp-uniform
      if (out_fm) {
        float4 a = acc[r];
        for (int o = 16; o >= Q; o >>= 1) {
          a.x += __shfl_xor_sync(0xffffffffu, a.x, o);
          a.y += __shfl_xor_sync(0xffffffffu, a.y, o);
          a.z += __shfl_xor_sync(0xffffffffu, a.z, o);
          a.w += __shfl_xor_sync(0xffffffffu, a.w, o);
        }
        // every lane of a q-class now holds the class total: scale by Q/32 so the warp sum counts it once
        const float s2 = (a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w) * qscale;
        const float v = warp_sum(s2 - sq[r]);
        if (lane == 0) out_fm[row] = 0.5f * v;
      }
      if (out_lin) {
        float l = lin[r];
        for (int c = lane; c < C; c += 32) l += __ldg(w_lin + F + c) * __ldg(dense + (int64_t)row * C + c);
        l = warp_sum(l);
        if (lane == 0) out_lin[row] = l;
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads)
fm_linear_bwd_vec(const int32_t* __restrict__ idx, const float* __restrict__ table,
                  const int64_t* __restrict__ row_offsets, const float* __restrict__ dense,
                  const float* __restrict__ w_lin, const float* __restrict__ g_lin,
                  const float* __restrict__ g_fm, float* __restrict__ grad_table,
                  float* __restrict__ grad_wlin, int B, int F, int D, int C) {
  extern __shared__ float s_gw[];   // [F + C] per-CTA partial of grad_wlin
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * kWarps) + (threadIdx.x >> 5);
  const int n_warps = gridDim.x * kWarps;
  const int Q = D >> 2;
  const int S = F * Q;
  if (g_lin) {
    for (int i = threadIdx.x; i < F + C; i += blockDim.x) s_gw[i] = 0.f;
    __syncthreads();
  }
  for (int row = warp; row < B; row += n_warps) {
    const float gf = g_fm ? __ldg(g_fm + row) : 0.f;
    const float gl = g_lin ? __ldg(g_lin + row) : 0.f;
    // pass 1: s[d] = sum_f e[f][d] (only the FM branch needs it)
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    if (g_fm) {
      for (int s0 = 0; s0 < S; s0 += 32 * kChunk) {
        float4 e[kChunk];
#pragma unroll
        for (int c = 0; c < kChunk; ++c) {
          const int slot = s0 + c * 32 + lane;
          e[c] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (slot < S) {
            const int f = slot / Q;
            const int64_t rb = table_row(row_offsets, f, __ldg(idx + (int64_t)row * F + f), D, nullptr);
            if (rb >= 0) e[c] = ldg_stream_f4(table + rb + ((slot - f * Q) << 2));
          }
        }
#pragma unroll
        for (int c = 0; c < kChunk; ++c) { a.x += e[c].x; a.y += e[c].y; a.z += e[c].z; a.w += e[c].w; }
      }
      for (int o = 16; o >= Q; o >>= 1) {
        a.x += __shfl_xor_sync(0xffffffffu, a.x, o);
        a.y += __shfl_xor_sync(0xffffffffu, a.y, o);
        a.z += __shfl_xor_sync(0xffffffffu, a.z, o);
        a.w += __shfl_xor_sync(0xffffffffu, a.w, o);
      }
    }
    // pass 2: dE = g_fm*(s - e) + g_lin*w_f ; scatter-add ; grad_wlin partials
    for (int s0 = 0; s0 < S; s0 += 32 * kChunk) {
#pragma unroll
      for (int c = 0; c < kChunk; ++c) {
        const int slot = s0 + c * 32 + lane;
        float rowsum = 0.f;
        int f = 0;
        if (slot < S) {
          f = slot / Q;
          const int64_t rb = table_row(row_offsets, f, __ldg(idx + (int64_t)row * F + f), D, nullptr);
          if (rb >= 0) {
            const int64_t off = rb + ((slot - f * Q) << 2);
            float4 e = make_float4(0.f, 0.f, 0.f, 0.f);
            if (g_fm || g_lin) e = ldg_stream_f4(table + off);
            const float lw = g_lin ? gl * __ldg(w_lin + f) : 0.f;
            float4 d;
            d.x = gf * (a.x - e.x) + lw;
            d.y = gf * (a.y - e.y) + lw;
            d.z = gf * (a.z - e.z) + lw;
            d.w = gf * (a.w - e.w) + lw;
            red_add_f4(grad_table + off, d);
            rowsum = (e.x + e.y) + (e.z + e.w);
          }
        }
        if (g_lin) {
          // the Q lanes of one field are consecutive: reduce them, lane with slot%Q==0 commits
          for (int o = 1; o < Q; o <<= 1) rowsum += __shfl_xor_sync(0xffffffffu, rowsum, o);
          if (slot < S && (slot % Q) == 0) atomicAdd(&s_gw[f], gl * rowsum);
        }
      }
    }
    if (g_lin)
      for (int c = lane; c < C; c += 32) atomicAdd(&s_gw[F + c], gl * __ldg(dense + (int64_t)row * C + c));
  }
  if (g_lin) {
    __syncthreads();
    for (int i = threadIdx.x; i < F + C; i += blockDim.x)
      if (s_gw[i] != 0.f) atomicAdd(grad_wlin + i, s_gw[i]);
  }
}

// ------------------------------------------------------------------------------------------
// generic path (any D): one thread per batch row, scalar loops.  Correctness path for odd dims.
// ------------------------------------------------------------------------------------------
__global__ void fm_linear_fwd_generic(const int32_t* __restrict__ idx, const float* __restrict__ table,
                                      const int64_t* __restrict__ row_offsets,
                                      const float* __restrict__ dense, const float* __restrict__ w_lin,
                                      float* __restrict__ out_lin, float* __restrict__ out_fm, int B, int F,
                                      int D, int C, int* status) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= B) return;
  float fm = 0.f;
  if (out_fm) {
    for (int d = 0; d < D; ++d) {
      float s = 0.f, q = 0.f;
      for (int f = 0; f < F; ++f) {
        const int64_t rb = table_row(row_offsets, f, idx[(int64_t)row * F + f], D, status);
        const float e = rb >= 0 ? table[rb + d] : 0.f;
        s += e;
        q += e * e;
      }
      fm += s * s - q;
    }
    out_fm[row] = 0.5f * fm;
  }
  if (out_lin) {
    float l = 0.f;
    for (int f = 0; f < F; ++f) {
      const int64_t rb = table_row(row_offsets, f, idx[(int64_t)row * F + f], D, status);
      float s = 0.f;
      if (rb >= 0)
        for (int d = 0; d < D; ++d) s += table[rb + d];
      l += w_lin[f] * s;
    }
    for (int c = 0; c < C; ++c) l += w_lin[F + c] * dense[(int64_t)row * C + c];
    out_lin[row] = l;
  }
}

__global__ void fm_linear_bwd_generic(const int32_t* __restrict__ idx, const float* __restrict__ table,
                                      const int64_t* __restrict__ row_offsets,
                                      const float* __restrict__ dense, const float* __restrict__ w_lin,
                                      const float* __restrict__ g_lin, const float* __restrict__ g_fm,
                                      float* __restrict__ grad_table, float* __restrict__ grad_wlin, int B,
                                      int F, int D, int C) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= B) return;
  const float gf = g_fm ? g_fm[row] : 0.f;
  const float gl = g_lin ? g_lin[row] : 0.f;
  for (int d = 0; d < D; ++d) {
    float s = 0.f;
    if (g_fm)
      for (int f = 0; f < F; ++f) {
        const int64_t rb = table_row(row_offsets, f, idx[(int64_t)row * F + f], D, nullptr);
        if (rb >= 0) s += table[rb + d];
      }
    for (int f = 0; f < F; ++f) {
      const int64_t rb = table_row(row_offsets, f, idx[(int64_t)row * F + f], D, nullptr);
      if (rb < 0) continue;
      const float e = table[rb + d];
      const float g = gf * (s - e) + (g_lin ? gl * w_lin[f] : 0.f);
      atomicAdd(grad_table + rb + d, g);
      if (g_lin) atomicAdd(grad_wlin + f, gl * e);
    }
  }
  if (g_lin)
    for (int c = 0; c < C; ++c) atomicAdd(grad_wlin + F + c, gl * dense[(int64_t)row * C + c]);
}

// ------------------------------------------------------------------------------------------
// gather -> [B, F*D (+C)] row-major (flatten_embeddings / concat_embedding_dense / plain gather)
// one thread per output element: 16 consecutive lanes read one 64-byte table row, stores coalesce.
// ------------------------------------------------------------------------------------------
__global__ void concat_fwd_kernel(const int32_t* __restrict__ idx, const float* __restrict__ table,
                                  const int64_t* __restrict__ row_offsets, const float* __restrict__ dense,
                                  float* __restrict__ X, int B, int F, int D, int C, int* status) {
  const int W = F * D + C;
  const int64_t total = (int64_t)B * W;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int row = (int)(i / W);
    const int col = (int)(i - (int64_t)row * W);
    float v;
    if (col < F * D) {
      const int f = col / D;
      const int64_t rb = table_row(row_offsets, f, __ldg(idx + (int64_t)row * F + f), D, status);
      v = rb >= 0 ? __ldg(table + rb + (col - f * D)) : 0.f;
    } else {
      v = __ldg(dense + (int64_t)row * C + (col - F * D));
    }
    X[i] = v;
  }
}

// scatter-add of dX[:, :F*D] (row stride W) into grad_table.  VEC=4: one 16-byte RED per slot.
template <int VEC>
__global__ void concat_bwd_kernel(const int32_t* __restrict__ idx, const int64_t* __restrict__ row_offsets,
                                  const float* __restrict__ dX, float* __restrict__ grad_table, int B, int F,
                                  int D, int W) {
  const int SD = D / VEC;
  const int64_t total = (int64_t)B * F * SD;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int row = (int)(i / (F * SD));
    const int rem = (int)(i - (int64_t)row * F * SD);
    const int f = rem / SD;
    const int d0 = (rem - f * SD) * VEC;
    const int64_t rb = table_row(row_offsets, f, __ldg(idx + (int64_t)row * F + f), D, nullptr);
    if (rb < 0) continue;
    const float* src = dX + (int64_t)row * W + f * D + d0;
    if (VEC == 4) {
      float4 v = make_float4(__ldg(src), __ldg(src + 1), __ldg(src + 2), __ldg(src + 3));
      red_add_f4(grad_table + rb + d0, v);
    } else {
      atomicAdd(grad_table + rb + d0, __ldg(src));
    }
  }
}

static int grid_for(int64_t work_items, int threads) {
  int64_t blocks = (work_items + threads - 1) / threads;
  const int64_t cap = (int64_t)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

static bool vec_ok(int D, const void* table) {
  const int Q = D / 4;
  return D % 4 == 0 && Q <= 32 && (Q & (Q - 1)) == 0 && (reinterpret_cast<uintptr_t>(table) % 16) == 0;
}


__global__ void linear_dense_grad_kernel(const float* __restrict__ g_lin, const float* __restrict__ w_dense,
                                         float* __restrict__ d_dense, int64_t total, int C) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    d_dense[i] = g_lin[i / C] * w_dense[i % C];
}

}  // namespace dtb

using namespace dtb;

extern "C" {

int dtb_linear_dense_grad(const float* g_lin, const float* w_dense, float* d_dense, int B, int C, void* stream) {
  DTB_CHECK_ARG(g_lin && w_dense && d_dense, "NULL argument");
  DTB_CHECK_ARG(B >= 0 && C > 0, "bad shape");
  const int64_t total = (int64_t)B * C;
  if (total == 0) return DTB_OK;
  int blocks = ceil_div(total, 256);
  const int cap = sm_count() * 8;
  if (blocks > cap) blocks = cap;
  linear_dense_grad_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(g_lin, w_dense, d_dense, total, C);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_fm_linear_fwd(const int32_t* idx, const float* table, const int64_t* row_offsets,
                      const float* dense, const float* w_lin, float* out_lin, float* out_fm, int B, int F,
                      int D, int C, int* status, void* stream) {
  DTB_CHECK_ARG(B >= 0 && F >= 0 && D >= 0 && C >= 0, "negative shape");
  DTB_CHECK_ARG(F == 0 || (idx && table && row_offsets && D > 0), "idx/table/row_offsets NULL with F > 0");
  DTB_CHECK_ARG(C == 0 || dense, "dense NULL with C > 0");
  DTB_CHECK_ARG(!out_lin || w_lin, "w_lin NULL");
  if (B == 0 || (!out_lin && !out_fm)) return DTB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (F > 0 && vec_ok(D, table)) {
    const int warps = ceil_div(B, kRowsPerPass);
    int blocks = ceil_div(warps, kWarps);
    const int cap = sm_count() * 8;
    if (blocks > cap) blocks = cap;
    const int S = F * (D / 4);
    if (S <= 128)
      fm_linear_fwd_vec<1><<<blocks, kThreads, 0, st>>>(idx, table, row_offsets, dense, w_lin, out_lin, out_fm, B, F,
                                                        D, C, status);
    else if (S <= 256)
      fm_linear_fwd_vec<2><<<blocks, kThreads, 0, st>>>(idx, table, row_offsets, dense, w_lin, out_lin, out_fm, B, F,
                                                        D, C, status);
    else
      fm_linear_fwd_vec_loop<<<blocks, kThreads, 0, st>>>(idx, table, row_offsets, dense, w_lin, out_lin, out_fm, B,
                                                          F, D, C, status);
  } else {
    fm_linear_fwd_generic<<<ceil_div(B, 128), 128, 0, st>>>(idx, table, row_offsets, dense, w_lin, out_lin,
                                                            out_fm, B, F, D, C, status);
  }
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_fm_linear_bwd(const int32_t* idx, const float* table, const int64_t* row_offsets,
                      const float* dense, const float* w_lin, const float* g_lin, const float* g_fm,
                      float* grad_table, float* grad_wlin, int B, int F, int D, int C, void* stream) {
  DTB_CHECK_ARG(B >= 0 && F >= 0 && D >= 0 && C >= 0, "negative shape");
  DTB_CHECK_ARG(F == 0 || (idx && table && row_offsets && grad_table && D > 0), "NULL table args with F > 0");
  DTB_CHECK_ARG(C == 0 || dense, "dense NULL with C > 0");
  DTB_CHECK_ARG(!g_lin || (w_lin && grad_wlin), "w_lin/grad_wlin NULL");
  if (B == 0 || (!g_lin && !g_fm)) return DTB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (F > 0 && vec_ok(D, table) && (reinterpret_cast<uintptr_t>(grad_table) % 16) == 0) {
    int blocks = ceil_div(B, kWarps);
    const int cap = sm_count() * 8;
    if (blocks > cap) blocks = cap;
    fm_linear_bwd_vec<<<blocks, kThreads, (F + C) * sizeof(float), st>>>(
        idx, table, row_offsets, dense, w_lin, g_lin, g_fm, grad_table, grad_wlin, B, F, D, C);
  } else {
    fm_linear_bwd_generic<<<ceil_div(B, 128), 128, 0, st>>>(idx, table, row_offsets, dense, w_lin, g_lin,
                                                            g_fm, grad_table, grad_wlin, B, F, D, C);
  }
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_concat_emb_dense_fwd(const int32_t* idx, const float* table, const int64_t* row_offsets,
                             const float* dense, float* X, int B, int F, int D, int C, int* status,
                             void* stream) {
  DTB_CHECK_ARG(B >= 0 && F >= 0 && D >= 0 && C >= 0 && X, "bad shape / X NULL");
  DTB_CHECK_ARG(F == 0 || (idx && table && row_offsets && D > 0), "NULL table args with F > 0");
  DTB_CHECK_ARG(C == 0 || dense, "dense NULL with C > 0");
  const int64_t total = (int64_t)B * (F * D + C);
  if (total == 0) return DTB_OK;
  concat_fwd_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(idx, table, row_offsets, dense,
                                                                             X, B, F, D, C, status);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_concat_emb_dense_bwd(const int32_t* idx, const int64_t* row_offsets, const float* dX,
                             float* grad_table, int B, int F, int D, int C, void* stream) {
  DTB_CHECK_ARG(B >= 0 && F >= 0 && D >= 0 && C >= 0, "negative shape");
  if (B == 0 || F == 0) return DTB_OK;
  DTB_CHECK_ARG(idx && row_offsets && dX && grad_table, "NULL argument");
  const int W = F * D + C;
  if (D % 4 == 0 && (reinterpret_cast<uintptr_t>(grad_table) % 16) == 0) {
    const int64_t total = (int64_t)B * F * (D / 4);
    concat_bwd_kernel<4><<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(idx, row_offsets, dX,
                                                                                 grad_table, B, F, D, W);
  } else {
    const int64_t total = (int64_t)B * F * D;
    concat_bwd_kernel<1><<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(idx, row_offsets, dX,
                                                                                 grad_table, B, F, D, W);
  }
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dtb_embedding_gather(const int32_t* idx, const float* table, const int64_t* row_offsets, float* out,
                         int B, int F, int D, int* status, void* stream) {
  return dtb_concat_emb_dense_fwd(idx, table, row_offsets, nullptr, out, B, F, D, 0, status, stream);
}

int dtb_embedding_scatter_add(const int32_t* idx, const int64_t* row_offsets, const float* d_out,
                              float* grad_table, int B, int F, int D, void* stream) {
  return dtb_concat_emb_dense_bwd(idx, row_offsets, d_out, grad_table, B, F, D, 0, stream);
}

}  // extern "C"
