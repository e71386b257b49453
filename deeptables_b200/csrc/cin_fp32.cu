// CIN (layers.py:638-734) -- exact-fp32 formulation for arbitrary shapes.
//
// This follows the reference's own decomposition (outer product per embedding dim, then a width-1
// conv == GEMM, layers.py:690-709) but keeps every tensor in a [B, D, *] layout so no transposes
// are needed, materialises the outer product Z only for a bounded chunk of batch rows, and runs the
// GEMMs as plain fp32 library GEMMs.  It is the any-shape path (odd D, odd layer sizes, direct=True
// with wide layers, ...) and the high-precision GPU cross-check for the tensor-core kernel in
// cin_wgmma.cu, which is the product path for the shapes it supports.
//
//   x0t[b,d,i]            = E[b,i,d]                       (gather fused into the transpose)
//   Z_k[(b,d), i*H_k + j] = x0t[b,d,i] * h_k[b,d,j]        (layers.py:690-695)
//   T_k[(b,d), l]         = act(Z_k @ W_k + bias_k)        (layers.py:705-709)
//   h_{k+1}               = T_k[..., :L/2] (or T_k when direct) ; pooled = sum_d of the rest (712-726)
#include "dtb_common.cuh"
#include "dense_tc.h"
#include "cin_shapes.h"
#include "cin_impl.h"

namespace dtb {

__global__ void cin_gather_t_kernel(const int32_t* __restrict__ idx, const float* __restrict__ table,
                                    const int64_t* __restrict__ row_offsets, float* __restrict__ x0t, int B,
                                    int F, int D, int* status) {
  // thread per (b, i, d) with d fastest for coalesced table reads; write transposed [b, d, i]
  const int64_t total = (int64_t)B * F * D;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(t / (F * D));
    const int r = (int)(t - (int64_t)b * F * D);
    const int i = r / D, d = r - i * D;
    const int64_t rb = table_row(row_offsets, i, __ldg(idx + (int64_t)b * F + i), D, status);
    x0t[((int64_t)b * D + d) * F + i] = rb >= 0 ? __ldg(table + rb + d) : 0.f;
  }
}

// Z[(r), i*H + j] = x0t[r, i] * h[r*ldh + j],  r = flattened (b,d) row of the chunk
__global__ void cin_build_z_kernel(const float* __restrict__ x0t, const float* __restrict__ h, int ldh,
                                   float* __restrict__ Z, int64_t n_rows, int F, int H) {
  const int K = F * H;
  const int64_t total = n_rows * K;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / K;
    const int c = (int)(t - r * K);
    const int i = c / H, j = c - i * H;
    Z[t] = x0t[r * F + i] * h[r * ldh + j];
  }
}

__global__ void cin_bias_act_kernel(float* __restrict__ T, const float* __restrict__ bias, int64_t total,
                                    int L, int act) {
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    float v = T[t];
    if (bias) v += bias[t % L];
    if (act == DTB_ACT_RELU) v = fmaxf(v, 0.f);
    T[t] = v;
  }
}

// pooled[b, pcol0 + l] = sum_d T[(b,d), lo + l]   for l in [0, n)
__global__ void cin_pool_kernel(const float* __restrict__ T, float* __restrict__ pooled, int B, int D, int L,
                                int lo, int n, int P, int pcol0) {
  const int64_t total = (int64_t)B * n;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(t / n), l = (int)(t - (int64_t)b * n);
    float s = 0.f;
    for (int d = 0; d < D; ++d) s += T[((int64_t)b * D + d) * L + lo + l];
    pooled[(int64_t)b * P + pcol0 + l] = s;
  }
}

// dC[(b,d), l] = (dpool part + dh part) * act'(T)
__global__ void cin_dc_kernel(const float* __restrict__ T, const float* __restrict__ d_pooled,
                              const float* __restrict__ dh_next, float* __restrict__ dC, int B, int D, int L,
                              int P, int pool_lo, int pool_n, int pcol0, int hid_n, int act) {
  const int64_t total = (int64_t)B * D * L;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / L;
    const int l = (int)(t - r * L);
    const int b = (int)(r / D);
    float g = 0.f;
    if (l >= pool_lo && l < pool_lo + pool_n) g += d_pooled[(int64_t)b * P + pcol0 + (l - pool_lo)];
    if (dh_next && l < hid_n) g += dh_next[r * hid_n + l];
    if (act == DTB_ACT_RELU && !(T[t] > 0.f)) g = 0.f;
    dC[t] = g;
  }
}

// warp per (b,d) row:  dx0t[r,i] += sum_j dZ[r,(i,j)] h[r,j] ;  dh[r,j] (=|+=) sum_i dZ[r,(i,j)] x0t[r,i]
__global__ void cin_dz_reduce_kernel(const float* __restrict__ dZ, const float* __restrict__ x0t,
                                     const float* __restrict__ h, int ldh, float* __restrict__ dx0t,
                                     float* __restrict__ dh, int64_t n_rows, int F, int H, int dh_into_dx0) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < n_rows; r += n_warps) {
    const float* z = dZ + r * (int64_t)F * H;
    for (int j0 = 0; j0 < H; j0 += 32) {
      const int j = j0 + lane;
      const float hj = j < H ? h[r * ldh + j] : 0.f;
      float dhj = 0.f;
      for (int i = 0; i < F; ++i) {
        const float zz = j < H ? z[i * H + j] : 0.f;
        dhj += zz * x0t[r * F + i];
        const float part = warp_sum(zz * hj);
        if (lane == 0) dx0t[r * F + i] += part;
      }
      __syncwarp();
      if (j < H) {
        if (dh_into_dx0) dx0t[r * F + j] += dhj;   // layer 0: h_0 is x0 itself (H == F)
        else dh[r * H + j] = dhj;
      }
      __syncwarp();
    }
  }
}

// grad_table[row(b,i)*D + d] += dx0t[b,d,i]
__global__ void cin_scatter_t_kernel(const int32_t* __restrict__ idx, const int64_t* __restrict__ row_offsets,
                                     const float* __restrict__ dx0t, float* __restrict__ grad_table, int B,
                                     int F, int D) {
  const int64_t total = (int64_t)B * F * D;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(t / (F * D));
    const int r = (int)(t - (int64_t)b * F * D);
    const int i = r / D, d = r - i * D;
    const int64_t rb = table_row(row_offsets, i, __ldg(idx + (int64_t)b * F + i), D, nullptr);
    if (rb >= 0) atomicAdd(grad_table + rb + d, dx0t[((int64_t)b * D + d) * F + i]);
  }
}

__global__ void cin_colsum_kernel(const float* __restrict__ A, float* __restrict__ out, int64_t rows, int cols) {
  // small helper for d_bias: one block per column strip, grid-stride over rows
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rl = threadIdx.x >> 5;
  __shared__ float s[8][32];
  float a = 0.f;
  if (c < cols)
    for (int64_t r = (int64_t)blockIdx.y * 8 + rl; r < rows; r += (int64_t)gridDim.y * 8) a += A[r * cols + c];
  s[rl][threadIdx.x & 31] = a;
  __syncthreads();
  if (rl == 0 && c < cols) {
    for (int k = 1; k < 8; ++k) a += s[k][threadIdx.x & 31];
    atomicAdd(out + c, a);
  }
}

static int ew_grid(int64_t total) {
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = (int64_t)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  return (int)(blocks < 1 ? 1 : blocks);
}

// chunk of batch rows whose Z fits the budget
static int fp32_chunk_rows(int B, int D, int kmax) {
  const int64_t budget = (int64_t)384 << 20;   // bytes per Z buffer
  int64_t rows = budget / ((int64_t)D * kmax * 4);
  if (rows < 1) rows = 1;
  if (rows > B) rows = B;
  return (int)rows;
}

// packed bf16 hi/lo images of one layer's filter for the tensor-core GEMMs (dense_tc.cu), either orientation
static size_t fp32_pack_bytes(const CinShape& s) {
  size_t m = 0;
  for (int k = 0; k < s.n_layers; ++k) {
    const int K = s.F * s.H[k], L = s.L[k];
    const size_t a = dense_tc_pack_bytes(K, L), b = dense_tc_pack_bytes(L, K);
    m = a > m ? a : m;
    m = b > m ? b : m;
  }
  return m;
}
static size_t fp32_pack_offset(const CinShape& s, int B, int training) {
  return cin_fp32_workspace_bytes(s, B, training) - fp32_pack_bytes(s) - 1024;
}

size_t cin_fp32_saved_bytes(const CinShape& s, int B) {
  return (size_t)B * s.D * (s.F + s.sumL) * sizeof(float);
}

size_t cin_fp32_workspace_bytes(const CinShape& s, int B, int training) {
  const int bc = fp32_chunk_rows(B, s.D, s.Kmax);
  size_t z = (size_t)bc * s.D * s.Kmax * sizeof(float);
  size_t bytes = z;                                                    // Z chunk
  if (!training) {
    bytes += (size_t)B * s.D * (s.F + s.sumL) * sizeof(float);          // x0t + T_k live in workspace
  } else {
    bytes += z;                                                         // dZ chunk
    bytes += (size_t)B * s.D * s.sumL * sizeof(float);                  // dC_k of every row: phase 2 reads it
    bytes += 2 * (size_t)bc * s.D * s.Hmax * sizeof(float);             // dh ping-pong
    bytes += (size_t)bc * s.D * s.F * sizeof(float);                    // dx0t
  }
  return (bytes + 255) / 256 * 256 + fp32_pack_bytes(s) + 1024;
}

int cin_fp32_fwd(const CinShape& s, const int32_t* idx, const float* table, const int64_t* row_offsets,
                 const float* weights, const float* bias, float* pooled, void* saved, void* workspace,
                 size_t workspace_bytes, int B, int act, int* status, cudaStream_t st) {
  if (workspace_bytes < cin_fp32_workspace_bytes(s, B, saved != nullptr)) {
    set_error("dtb_cin_fwd: workspace too small");
    return DTB_ERR_INVALID_ARG;
  }
  uint8_t* pack = reinterpret_cast<uint8_t*>(workspace) + fp32_pack_offset(s, B, saved != nullptr);
  const size_t pack_bytes = fp32_pack_bytes(s);
  const int D = s.D, F = s.F;
  const int bc = fp32_chunk_rows(B, D, s.Kmax);
  float* Z = reinterpret_cast<float*>(workspace);
  float* act_base = saved ? reinterpret_cast<float*>(saved) : Z + (size_t)bc * D * s.Kmax;
  float* x0t = act_base;                           // [B, D, F]
  float* Tk[kCinMaxLayers];
  {
    float* p = x0t + (size_t)B * D * F;
    for (int k = 0; k < s.n_layers; ++k) {
      Tk[k] = p;
      p += (size_t)B * D * s.L[k];
    }
  }
  const int64_t n_g = (int64_t)B * F * D;
  cin_gather_t_kernel<<<ew_grid(n_g), 256, 0, st>>>(idx, table, row_offsets, x0t, B, F, D, status);
  DTB_LAUNCH_OK();
  for (int k = 0; k < s.n_layers; ++k) {
    const int H = s.H[k], L = s.L[k], K = F * H;
    const float* hk = k == 0 ? x0t : Tk[k - 1];
    const int ldh = k == 0 ? F : s.L[k - 1];
    for (int b0 = 0; b0 < B; b0 += bc) {
      const int nb = B - b0 < bc ? B - b0 : bc;
      const int64_t rows = (int64_t)nb * D;
      cin_build_z_kernel<<<ew_grid(rows * K), 256, 0, st>>>(x0t + (size_t)b0 * D * F,
                                                             hk + (size_t)b0 * D * ldh, ldh, Z, rows, F, H);
      DTB_LAUNCH_OK();
      float* T = Tk[k] + (size_t)b0 * D * L;
      {
        const int rc = dense_tc_rows(Z, K, weights + s.w_off[k], L, 0, nullptr, T, L, (int)rows, K, L, DTB_ACT_NONE, pack,
                                     pack_bytes, st);
        if (rc != DTB_OK) return rc;
      }
      if (bias || act != DTB_ACT_NONE) {
        cin_bias_act_kernel<<<ew_grid(rows * L), 256, 0, st>>>(T, bias ? bias + s.b_off[k] : nullptr, rows * L,
                                                               L, act);
        DTB_LAUNCH_OK();
      }
    }
    if (s.pool_n[k] > 0) {
      cin_pool_kernel<<<ew_grid((int64_t)B * s.pool_n[k]), 256, 0, st>>>(Tk[k], pooled, B, D, L, s.pool_lo[k],
                                                                          s.pool_n[k], s.P, s.pcol0[k]);
      DTB_LAUNCH_OK();
    }
  }
  return DTB_OK;
}

// phase 1: dC_k (kept for every row), dZ = dC W^T and its reduction into grad_table -- after it the table gradient is
// final; phase 2: dW_k += Z_k^T dC_k (Z_k rebuilt from the saved activations) and d_bias; phase 0: both.
int cin_fp32_bwd(const CinShape& s, const int32_t* idx, const float* table, const int64_t* row_offsets,
                 const float* weights, const float* d_pooled, const void* saved, float* grad_table,
                 float* d_weights, float* d_bias, void* workspace, size_t workspace_bytes, int B, int act,
                 int phase, cudaStream_t st) {
  (void)table;
  if (workspace_bytes < cin_fp32_workspace_bytes(s, B, 1)) {
    set_error("dtb_cin_bwd: workspace too small");
    return DTB_ERR_INVALID_ARG;
  }
  uint8_t* pack = reinterpret_cast<uint8_t*>(workspace) + fp32_pack_offset(s, B, 1);
  const size_t pack_bytes = fp32_pack_bytes(s);
  const int D = s.D, F = s.F;
  const int bc = fp32_chunk_rows(B, D, s.Kmax);
  float* Z = reinterpret_cast<float*>(workspace);
  float* dZ = Z + (size_t)bc * D * s.Kmax;
  float* dC_all = dZ + (size_t)bc * D * s.Kmax;
  float* dh0 = dC_all + (size_t)B * D * s.sumL;
  float* dh1 = dh0 + (size_t)bc * D * s.Hmax;
  float* dx0t = dh1 + (size_t)bc * D * s.Hmax;
  const float* x0t_all = reinterpret_cast<const float*>(saved);
  const float* Tk[kCinMaxLayers];
  {
    const float* p = x0t_all + (size_t)B * D * F;
    for (int k = 0; k < s.n_layers; ++k) {
      Tk[k] = p;
      p += (size_t)B * D * s.L[k];
    }
  }
  float* dCk[kCinMaxLayers];
  {
    float* p = dC_all;
    for (int k = 0; k < s.n_layers; ++k) {
      dCk[k] = p;
      p += (size_t)B * D * s.L[k];
    }
  }
  for (int b0 = 0; b0 < B && phase != 2; b0 += bc) {
    const int nb = B - b0 < bc ? B - b0 : bc;
    const int64_t rows = (int64_t)nb * D;
    const float* x0t = x0t_all + (size_t)b0 * D * F;
    DTB_CUDA_OK(cudaMemsetAsync(dx0t, 0, rows * F * sizeof(float), st));
    float* dh_next = nullptr;   // gradient wrt h_{k+1} (compact [rows, H_{k+1}])
    float* dh_cur = dh0;
    for (int k = s.n_layers - 1; k >= 0; --k) {
      const int H = s.H[k], L = s.L[k], K = F * H;
      const float* T = Tk[k] + (size_t)b0 * D * L;
      float* dC = dCk[k] + (size_t)b0 * D * L;
      const int hid_n = (k + 1 < s.n_layers) ? s.H[k + 1] : 0;
      cin_dc_kernel<<<ew_grid(rows * L), 256, 0, st>>>(T, d_pooled + (size_t)b0 * s.P, dh_next, dC, nb, D, L,
                                                       s.P, s.pool_lo[k], s.pool_n[k], s.pcol0[k], hid_n, act);
      DTB_LAUNCH_OK();
      const float* hk = k == 0 ? x0t : Tk[k - 1] + (size_t)b0 * D * s.L[k - 1];
      const int ldh = k == 0 ? F : s.L[k - 1];
      // dZ[rows, K] = dC W_k^T
      {
        const int rc = dense_tc_rows(dC, L, weights + s.w_off[k], L, 1, nullptr, dZ, K, (int)rows, L, K, DTB_ACT_NONE,
                                     pack, pack_bytes, st);
        if (rc != DTB_OK) return rc;
      }
      int blocks = ceil_div(rows, 8);
      const int cap = sm_count() * 8;
      if (blocks > cap) blocks = cap;
      cin_dz_reduce_kernel<<<blocks, 256, 0, st>>>(dZ, x0t, hk, ldh, dx0t, dh_cur, rows, F, H, k == 0 ? 1 : 0);
      DTB_LAUNCH_OK();
      dh_next = dh_cur;
      dh_cur = (dh_cur == dh0) ? dh1 : dh0;
    }
    cin_scatter_t_kernel<<<ew_grid((int64_t)nb * F * D), 256, 0, st>>>(idx + (size_t)b0 * F, row_offsets, dx0t,
                                                                       grad_table, nb, F, D);
    DTB_LAUNCH_OK();
  }
  for (int b0 = 0; b0 < B && phase != 1; b0 += bc) {
    const int nb = B - b0 < bc ? B - b0 : bc;
    const int64_t rows = (int64_t)nb * D;
    const float* x0t = x0t_all + (size_t)b0 * D * F;
    for (int k = 0; k < s.n_layers; ++k) {
      const int H = s.H[k], L = s.L[k], K = F * H;
      const float* dC = dCk[k] + (size_t)b0 * D * L;
      if (d_bias) {
        dim3 grid(ceil_div(L, 32), 64);
        cin_colsum_kernel<<<grid, 256, 0, st>>>(dC, d_bias + s.b_off[k], rows, L);
        DTB_LAUNCH_OK();
      }
      const float* hk = k == 0 ? x0t : Tk[k - 1] + (size_t)b0 * D * s.L[k - 1];
      const int ldh = k == 0 ? F : s.L[k - 1];
      cin_build_z_kernel<<<ew_grid(rows * K), 256, 0, st>>>(x0t, hk, ldh, Z, rows, F, H);
      DTB_LAUNCH_OK();
      // dW_k[K, L] += Z^T dC
      const int rc = dense_tc_wgrad(Z, K, dC, L, d_weights + s.w_off[k], L, nullptr, (int)rows, K, L, st);
      if (rc != DTB_OK) return rc;
    }
  }
  return DTB_OK;
}

}  // namespace dtb
