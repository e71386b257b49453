// Dense-layer GEMMs on the Hopper tensor cores (wgmma, fp32 accumulators in registers): keras Dense forward / data gradient /
// weight gradient (dnn() tower, deepnets.py:401-427; per-net logit layers wider than 8, deepmodel.py:292; the AutoInt
// Q/K/V/residual projections, layers.py:106-127) and the GEMMs of the any-shape CIN formulation (cin_fp32.cu).
//
// fp32 in, fp32 out.  Operands are split on the fly into bf16 hi + lo and multiplied in three tensor passes
// (hi*hi + lo*hi + hi*lo, fp32 accumulation): each operand is represented to 2^-18, the dropped lo*lo term is
// 2^-18 of a product, i.e. fp32-grade results (the same scheme the CIN kernels use, cin_wgmma.cu).
//
//   rows kernel   out[M, Nout] = act(A[M, K] . W + bias)       W given as packed images (dense_tc_pack_kernel)
//                 forward:   A = X,  W = kernel          [K = in_dim,  Nout = out_dim]
//                 dgrad:     A = dZ, W = kernel^T        [K = out_dim, Nout = in_dim]
//   wgrad kernel  dW[K, N] += sum_m X[m, k] dZ[m, n]     both operands converted on the fly; reduction over batch rows
//
// These shapes are HBM-bound (126 kFLOP per 1.7 KB row for 429 -> 128 -> 64), so the structure is a streaming one:
// coalesced fp32 reads -> registers -> bf16 hi/lo core matrices in shared memory (canonical K-major, no swizzle)
// -> wgmma (both operands from shared memory), 4-stage mbarrier ring, weights by bulk async copy.  Two consumer
// warpgroups own 64 rows each of a 128-row tile; they release a stage as soon as their MMAs on it complete, so the
// producers and the weight loader run up to four stages ahead while the consumers apply bias / activation to their
// accumulator registers and store them.
#include "dtb_common.cuh"
#include "wgmma.cuh"
#include "dense_tc.h"
#include <cuda_bf16.h>
#include <cstdlib>

namespace dtb {

constexpr int kDtThreads = 544;        // rows kernel: warps 0-7 producers, 8-15 two MMA + epilogue warpgroups, 16 weight loader
constexpr int kDtWgThreads = 512;      // wgrad kernel: warps 0-3 X producers, 4-7 dZ producers, 8-15 two MMA + epilogue warpgroups
constexpr int kDtKc = 32;              // reduction elements per pipeline stage (two wgmma k-steps)
constexpr int kDtStages = 4;
constexpr int kDtAImg = 128 * kDtKc * 2;          // bytes of one bf16 [128 x 32] image
constexpr int kDtAStage = 2 * kDtAImg;            // hi + lo
constexpr int kDtMaxNT = 128;            // widest wgmma N used (64 accumulator registers per thread)

static inline int dt_round_up(int x, int m) { return (x + m - 1) / m * m; }

// ------------------------------------------------------------------------------------------
// weight pack: fp32 W (row-major, leading dimension ldw) -> per (n-tile, k-chunk) [hi image | lo image],
// image = canonical K-major no-swizzle tile of B[n][kk]:  core (kk/8, n/8) at ((kk/8)*(NT/8) + n/8)*128 B,
// row n%8 at 16 B, element kk%8 at 2 B.   transposed = 0: B[n][kk] = W[(k0+kk)*ldw + n0+n]   (forward)
//                                         transposed = 1: B[n][kk] = W[(n0+n)*ldw + k0+kk]   (data gradient)
// ------------------------------------------------------------------------------------------
__global__ void dense_tc_pack_kernel(const float* __restrict__ w, uint8_t* __restrict__ out, int K, int N, int ldw,
                                     int NT, int n_tiles, int n_chunks, int transposed) {
  const int64_t per_chunk = (int64_t)NT * kDtKc;
  const int64_t total = per_chunk * n_chunks * n_tiles;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t img = t / per_chunk;
    const int rem = (int)(t - img * per_chunk);
    const int nt = (int)(img / n_chunks), c = (int)(img - (int64_t)nt * n_chunks);
    int kk, n;
    if (transposed) { n = rem / kDtKc; kk = rem - n * kDtKc; }     // kk fastest: coalesced reads of W rows
    else            { kk = rem / NT;   n = rem - kk * NT; }        // n fastest
    const int k = c * kDtKc + kk, col = nt * NT + n;
    float v = 0.f;
    if (k < K && col < N) v = transposed ? w[(int64_t)col * ldw + k] : w[(int64_t)k * ldw + col];
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
    const int64_t off = ((int64_t)(kk >> 3) * (NT >> 3) + (n >> 3)) * 128 + (n & 7) * 16 + (kk & 7) * 2;
    uint8_t* base = out + img * per_chunk * 4;
    *reinterpret_cast<__nv_bfloat16*>(base + off) = hi;
    *reinterpret_cast<__nv_bfloat16*>(base + per_chunk * 2 + off) = lo;
  }
}

struct DenseTcRowsParams {
  const float* A;        // [M, K], leading dimension lda
  const uint8_t* wpack;  // images [n_tile][k_chunk][hi | lo]
  const float* bias;     // [Nout] or null
  float* out;            // [M, Nout], leading dimension ldo
  int M, K, Nout, lda, ldo, NT, n_tiles, n_chunks, act, vec2;
};

struct DtSmem {
  int a_off, b_off, bar_off, total, b_stage;
};
__host__ __device__ inline DtSmem dt_layout(int NT) {
  DtSmem l;
  l.b_stage = NT * kDtKc * 4;
  l.a_off = 0;
  l.b_off = kDtStages * kDtAStage;
  l.bar_off = l.b_off + kDtStages * l.b_stage;
  l.bar_off = (l.bar_off + 15) / 16 * 16;
  l.total = l.bar_off + 256;
  return l;
}

// [16 rows x 32 columns] fp32 block of a row-major matrix -> registers (one 128-byte request per row, all 16 in flight),
// and registers -> bf16 hi/lo words of a K-major image whose MMA rows are the matrix ROWS and whose reduction index is
// the matrix COLUMN (rows kernel: A = X tile).  A lane pair (k even, k+1) exchanges values so that the even lane stores
// the packed hi word and the odd lane the packed lo word.
__device__ __forceinline__ void dt_load_rows16(float (&v)[16], const float* __restrict__ src, int ld, int row0,
                                               int n_rows_valid, int col0, int n_cols_valid, int lane) {
#pragma unroll
  for (int j = 0; j < 16; ++j)
    v[j] = (j < n_rows_valid && lane < n_cols_valid) ? __ldg(src + (int64_t)(row0 + j) * ld + col0 + lane) : 0.f;
}
__device__ __forceinline__ void dt_store_rows16(const float (&v)[16], uint8_t* img_hi, uint8_t* img_lo, int img_row0,
                                                int lane) {
  const bool even = (lane & 1) == 0;
  const int kk = lane & ~1;
  uint8_t* img = even ? img_hi : img_lo;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const float other = __shfl_xor_sync(0xffffffffu, v[j], 1);
    const float a = even ? v[j] : other, b = even ? other : v[j];
    uint32_t hi, lo;
    tc::split_bf16x2(a, b, hi, lo);
    const int r_img = img_row0 + j;
    const int off = (kk >> 3) * 2048 + (r_img >> 3) * 128 + (r_img & 7) * 16 + (kk & 7) * 2;
    *reinterpret_cast<uint32_t*>(img + off) = even ? hi : lo;
  }
}

// One k-chunk (kDtKc = 32) of the three bf16 passes on this warpgroup's 64 rows: A image rows [64 wg, 64 wg + 64),
// B image NT rows; then wait for the MMAs, so that the caller may release the stage.
template <int NT>
__device__ __forceinline__ void dt_mma_chunk(float (&acc)[NT / 2], uint32_t a_addr, uint32_t b_addr, int wg, bool first) {
  constexpr uint32_t lbo_b = (NT >> 3) * 128;
  constexpr uint32_t img_b = NT * kDtKc * 2;
  tc::wgmma_fence();
#pragma unroll
  for (int pass = 0; pass < 3; ++pass) {
    // pass 0: A_hi*B_hi ; 1: A_lo*B_hi ; 2: A_hi*B_lo
    const uint32_t a_img = a_addr + (pass == 1 ? kDtAImg : 0) + wg * 1024;
    const uint32_t b_img = b_addr + (pass == 2 ? img_b : 0);
#pragma unroll
    for (int ks = 0; ks < kDtKc / 16; ++ks) {
      const uint64_t da = tc::make_smem_desc(a_img + ks * 4096, 2048, 128);
      const uint64_t db = tc::make_smem_desc(b_img + ks * 2 * lbo_b, lbo_b, 128);
      tc::Wgmma<NT>::ss(acc, da, db, (uint32_t)(!first || pass != 0 || ks != 0));
    }
  }
  tc::wgmma_commit();
  tc::wgmma_wait<0>();
  tc::wgmma_fence_acc(acc);
}

template <int NT>
__global__ void __launch_bounds__(kDtThreads, 1) dense_tc_rows_kernel(const __grid_constant__ DenseTcRowsParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const DtSmem lay = dt_layout(NT);
  uint8_t* smem_a = smem + lay.a_off;
  uint8_t* smem_b = smem + lay.b_off;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + lay.bar_off);
  uint64_t* full_a = bars;                 // [stage] 8 producer warps
  uint64_t* full_b = bars + 4;             // [stage] bulk copy (tx)
  uint64_t* empty = bars + 8;              // [stage] 8 consumer warps

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_mtiles = (p.M + 127) / 128;
  const int n_items = n_mtiles * p.n_tiles;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kDtStages; ++s) {
      tc::mbar_init(&full_a[s], 8);
      tc::mbar_init(&full_b[s], 1);
      tc::mbar_init(&empty[s], 8);
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp < 8) {
    // ============================ A producers: fp32 rows -> bf16 hi/lo images =============================
    // warp w converts rows [16w, 16w + 16) of the tile.  The loads of the NEXT (item, chunk) are issued before this
    // chunk's barrier wait and conversion: 8 warps x 16-32 requests of 128 bytes keep 16-32 KB in flight per SM.
    uint32_t it = 0;
    float cur[16], nxt[16];
    int item = blockIdx.x, c = 0;
    if (item < n_items) {
      const int row0 = (item / p.n_tiles) * 128 + warp * 16;
      dt_load_rows16(cur, p.A, p.lda, row0, p.M - row0, 0, p.K, lane);
    }
    while (item < n_items) {
      int n_item = item, n_c = c + 1;
      if (n_c == p.n_chunks) { n_c = 0; n_item = item + gridDim.x; }
      if (n_item < n_items) {
        const int row0 = (n_item / p.n_tiles) * 128 + warp * 16;
        dt_load_rows16(nxt, p.A, p.lda, row0, p.M - row0, n_c * kDtKc, p.K - n_c * kDtKc, lane);
      }
      const uint32_t s = it % kDtStages, ph = (it / kDtStages) & 1;
      ++it;
      tc::mbar_wait(&empty[s], ph ^ 1);
      uint8_t* a_stage = smem_a + s * kDtAStage;
      dt_store_rows16(cur, a_stage, a_stage + kDtAImg, warp * 16, lane);
      tc::fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&full_a[s]);
#pragma unroll
      for (int j = 0; j < 16; ++j) cur[j] = nxt[j];
      item = n_item;
      c = n_c;
    }
  } else if (warp < 16) {
    // ============================ MMA + epilogue: warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile ====
    const int wg = (warp >> 2) - 2;
    const int wq = warp & 3;
    const uint32_t a_u32 = tc::smem_u32(smem_a), b_u32 = tc::smem_u32(smem_b);
    uint32_t it = 0;
    float acc[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      const int mt = item / p.n_tiles, nt = item - mt * p.n_tiles;
      for (int c = 0; c < p.n_chunks; ++c, ++it) {
        const uint32_t s = it % kDtStages, ph = (it / kDtStages) & 1;
        tc::mbar_wait(&full_b[s], ph);
        tc::mbar_wait(&full_a[s], ph);
        dt_mma_chunk<NT>(acc, a_u32 + s * kDtAStage, b_u32 + s * (uint32_t)lay.b_stage, wg, c == 0);
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&empty[s]);
      }
      const int row_a = mt * 128 + wg * 64 + wq * 16 + (lane >> 2);
      const int n0 = nt * NT + 2 * (lane & 3);
#pragma unroll
      for (int i = 0; i < NT / 2; i += 2) {
        const int grow = row_a + (((i >> 1) & 1) << 3);
        const int col = n0 + 8 * (i >> 2);
        if (grow >= p.M || col >= p.Nout) continue;
        float o0 = acc[i], o1 = acc[i + 1];
        const bool two = col + 1 < p.Nout;
        if (p.bias) {
          o0 += __ldg(p.bias + col);
          if (two) o1 += __ldg(p.bias + col + 1);
        }
        if (p.act == DTB_ACT_RELU) {
          o0 = fmaxf(o0, 0.f); o1 = fmaxf(o1, 0.f);
        } else if (p.act == DTB_ACT_TANH) {
          o0 = tanhf(o0); o1 = tanhf(o1);
        }
        float* dst = p.out + (int64_t)grow * p.ldo + col;
        if (two && p.vec2) {
          *reinterpret_cast<float2*>(dst) = make_float2(o0, o1);
        } else {
          dst[0] = o0;
          if (two) dst[1] = o1;
        }
      }
    }
  } else {
    // ============================ weight loader ==============================================================
    if (lane == 0) {
      uint32_t it = 0;
      const uint32_t bytes = (uint32_t)lay.b_stage;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int mt = item / p.n_tiles, nt = item - mt * p.n_tiles;
        const uint8_t* src = p.wpack + (size_t)nt * p.n_chunks * bytes;
        for (int c = 0; c < p.n_chunks; ++c, ++it) {
          const uint32_t s = it % kDtStages, ph = (it / kDtStages) & 1;
          tc::mbar_wait(&empty[s], ph ^ 1);
          tc::mbar_arrive_expect_tx(&full_b[s], bytes);
          tc::bulk_g2s(smem_b + (size_t)s * bytes, src + (size_t)c * bytes, bytes, &full_b[s]);
        }
      }
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------
// weight gradient: dW[k, n] += sum_m X[m, k] dZ[m, n].   MMA M = 128 in-dim indices k (grid.x), N = NT out-dim indices
// (grid.z), reduction over batch rows in chunks of 32 (grid.y splits the batch).  Both operands are fp32 row-major
// matrices whose ROWS are the reduction index: a lane reads the same column of two consecutive rows (coalesced across
// the warp) and packs the pair into one K-major word.
// ------------------------------------------------------------------------------------------
struct DenseTcWgradParams {
  const float* X;     // [M, K]  ldx
  const float* dZ;    // [M, N]  ldz
  float* dW;          // [K, N]  ldw, accumulated
  float* dbias;       // [N] accumulated by the k-tile-0 CTAs (or null)
  int M, K, N, ldx, ldz, ldw, NT, chunks_per_split, n_chunks_total;
};

// rows [m0, m0+32) x 4 column groups of 32 of src -> K-major image with MMA row = column index, reduction index = row;
// this warp handles row pairs [pair0, pair0 + 4).  All 32 requests (4 groups x 4 pairs x 2 rows) are issued before the
// first conversion.  Adds the column sums of the values it touched to colsum[] (for the bias gradient).
__device__ __forceinline__ void dt_convert_cols4(const float* __restrict__ src, int ld, int m0, int m_valid, int col0,
                                                 int n_cols, uint8_t* img_hi, uint8_t* img_lo, int img_row0, int img_rows,
                                                 int pair0, int lane, float (&colsum)[4]) {
  float a[4][4], b[4][4];
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const bool cok = col0 + g * 32 + lane < n_cols;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int mm = (pair0 + j) * 2;
      a[g][j] = (cok && mm < m_valid) ? __ldg(src + (int64_t)(m0 + mm) * ld + col0 + g * 32 + lane) : 0.f;
      b[g][j] = (cok && mm + 1 < m_valid) ? __ldg(src + (int64_t)(m0 + mm + 1) * ld + col0 + g * 32 + lane) : 0.f;
    }
  }
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const int r_img = img_row0 + g * 32 + lane;
    const int base = (r_img >> 3) * 128 + (r_img & 7) * 16;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int mm = (pair0 + j) * 2;
      uint32_t hi, lo;
      tc::split_bf16x2(a[g][j], b[g][j], hi, lo);
      const int off = (mm >> 3) * (img_rows >> 3) * 128 + base + (mm & 7) * 2;
      if (r_img < img_rows) {                     // NT is a multiple of 16, the column groups of 32: the tail group is half used
        *reinterpret_cast<uint32_t*>(img_hi + off) = hi;
        *reinterpret_cast<uint32_t*>(img_lo + off) = lo;
      }
      colsum[g] += a[g][j] + b[g][j];
    }
  }
}

template <int NT>
__global__ void __launch_bounds__(kDtWgThreads, 1) dense_tc_wgrad_kernel(const __grid_constant__ DenseTcWgradParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const DtSmem lay = dt_layout(NT);
  uint8_t* smem_a = smem + lay.a_off;
  uint8_t* smem_b = smem + lay.b_off;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + lay.bar_off);
  uint64_t* full = bars;                   // [stage] 8 producer warps
  uint64_t* empty = bars + 4;              // [stage] 8 consumer warps

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = blockIdx.x * 128, n0 = blockIdx.z * NT;
  const int c_begin = blockIdx.y * p.chunks_per_split;
  int c_end = c_begin + p.chunks_per_split;
  if (c_end > p.n_chunks_total) c_end = p.n_chunks_total;
  const int n_ch = c_end > c_begin ? c_end - c_begin : 0;
  const int b_img_bytes = NT * kDtKc * 2;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kDtStages; ++s) {
      tc::mbar_init(&full[s], 8);
      tc::mbar_init(&empty[s], 8);
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp < 8) {
    // warps 0-3: X -> A images (MMA rows = k);  warps 4-7: dZ -> B images (MMA rows = n); each warp owns 4 row pairs
    const bool is_a = warp < 4;
    const int pair0 = (warp & 3) * 4;
    float bsum[kDtMaxNT / 32];
#pragma unroll
    for (int g = 0; g < kDtMaxNT / 32; ++g) bsum[g] = 0.f;
    for (int c = 0; c < n_ch; ++c) {
      const uint32_t s = c % kDtStages, ph = (c / kDtStages) & 1;
      tc::mbar_wait(&empty[s], ph ^ 1);
      const int m0 = (c_begin + c) * kDtKc;
      const int m_valid = p.M - m0;
      if (is_a) {
        uint8_t* st = smem_a + s * kDtAStage;
        float unused[4] = {0.f, 0.f, 0.f, 0.f};
        dt_convert_cols4(p.X, p.ldx, m0, m_valid, k0, p.K, st, st + kDtAImg, 0, 128, pair0, lane, unused);
      } else {
        uint8_t* st = smem_b + s * lay.b_stage;
        dt_convert_cols4(p.dZ, p.ldz, m0, m_valid, n0, p.N, st, st + b_img_bytes, 0, NT, pair0, lane, bsum);
      }
      tc::fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&full[s]);
    }
    if (!is_a && p.dbias && blockIdx.x == 0) {
#pragma unroll
      for (int g = 0; g < kDtMaxNT / 32; ++g) {
        const int n = n0 + g * 32 + lane;
        if (g * 32 < NT && n < p.N && bsum[g] != 0.f) atomicAdd(p.dbias + n, bsum[g]);
      }
    }
  } else if (n_ch > 0) {
    // ---- MMA + epilogue: warpgroup wg owns in-dim rows [k0 + 64 wg, k0 + 64 wg + 64) -> dW[k, n0 ...] -------------
    const int wg = (warp >> 2) - 2;
    const uint32_t a_u32 = tc::smem_u32(smem_a), b_u32 = tc::smem_u32(smem_b);
    float acc[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
    for (int c = 0; c < n_ch; ++c) {
      const uint32_t s = c % kDtStages, ph = (c / kDtStages) & 1;
      tc::mbar_wait(&full[s], ph);
      dt_mma_chunk<NT>(acc, a_u32 + s * kDtAStage, b_u32 + s * (uint32_t)lay.b_stage, wg, c == 0);
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&empty[s]);
    }
    const int k_a = k0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int n_a = n0 + 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) {
      const int k = k_a + (((i >> 1) & 1) << 3);
      const int n = n_a + 8 * (i >> 2) + (i & 1);
      if (k < p.K && n < p.N) atomicAdd(p.dW + (int64_t)k * p.ldw + n, acc[i]);
    }
  }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
// wgmma N of a [*, Nout] output: the smallest supported width that holds it, else kDtMaxNT-wide column tiles
static int dt_nt(int Nout) {
  const int np = dt_round_up(Nout, 16);
  return np <= 16 ? 16 : np <= 32 ? 32 : np <= 64 ? 64 : kDtMaxNT;
}

struct DtTiling {
  int NT, n_tiles, n_chunks;
};
static DtTiling dt_tiling(int K, int Nout) {
  DtTiling t;
  t.NT = dt_nt(Nout);
  t.n_tiles = (Nout + t.NT - 1) / t.NT;
  t.n_chunks = (K + kDtKc - 1) / kDtKc;
  return t;
}

size_t dense_tc_pack_bytes(int K, int Nout) {
  const DtTiling t = dt_tiling(K, Nout);
  return (size_t)t.n_tiles * t.n_chunks * t.NT * kDtKc * 4 + 256;
}

template <int NT>
static int dt_launch_rows(const DenseTcRowsParams& p, int n_items, cudaStream_t st) {
  const DtSmem lay = dt_layout(NT);
  DTB_CUDA_OK(cudaFuncSetAttribute(dense_tc_rows_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, lay.total));
  int grid = sm_count();
  if (grid > n_items) grid = n_items;
  dense_tc_rows_kernel<NT><<<grid, kDtThreads, lay.total, st>>>(p);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dense_tc_rows(const float* A, int lda, const float* W, int ldw, int transposed, const float* bias, float* out,
                  int ldo, int M, int K, int Nout, int act, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  if (M <= 0) return DTB_OK;
  if (!workspace || workspace_bytes < dense_tc_pack_bytes(K, Nout) || (reinterpret_cast<uintptr_t>(workspace) & 15)) {
    set_error("dense_tc_rows: workspace missing, misaligned or smaller than the packed weights (%zu bytes needed)",
              dense_tc_pack_bytes(K, Nout));
    return DTB_ERR_INVALID_ARG;
  }
  const DtTiling t = dt_tiling(K, Nout);
  const int64_t total = (int64_t)t.n_tiles * t.n_chunks * t.NT * kDtKc;
  int blocks = (int)((total + 255) / 256);
  if (blocks > sm_count() * 4) blocks = sm_count() * 4;
  dense_tc_pack_kernel<<<blocks, 256, 0, st>>>(W, reinterpret_cast<uint8_t*>(workspace), K, Nout, ldw, t.NT, t.n_tiles,
                                               t.n_chunks, transposed);
  DTB_LAUNCH_OK();
  DenseTcRowsParams p{};
  p.A = A; p.wpack = reinterpret_cast<const uint8_t*>(workspace); p.bias = bias; p.out = out;
  p.M = M; p.K = K; p.Nout = Nout; p.lda = lda; p.ldo = ldo; p.NT = t.NT; p.n_tiles = t.n_tiles; p.n_chunks = t.n_chunks;
  p.act = act;
  p.vec2 = (ldo % 2 == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0) ? 1 : 0;    // column pairs as one 8-byte store
  const int n_items = ((M + 127) / 128) * t.n_tiles;
  switch (t.NT) {
    case 16: return dt_launch_rows<16>(p, n_items, st);
    case 32: return dt_launch_rows<32>(p, n_items, st);
    case 64: return dt_launch_rows<64>(p, n_items, st);
    default: return dt_launch_rows<kDtMaxNT>(p, n_items, st);
  }
}

template <int NT>
static int dt_launch_wgrad(const DenseTcWgradParams& p, dim3 grid, cudaStream_t st) {
  const DtSmem lay = dt_layout(NT);
  DTB_CUDA_OK(cudaFuncSetAttribute(dense_tc_wgrad_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, lay.total));
  dense_tc_wgrad_kernel<NT><<<grid, kDtWgThreads, lay.total, st>>>(p);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

int dense_tc_wgrad(const float* X, int ldx, const float* dZ, int ldz, float* dW, int ldw, float* dbias, int M, int K,
                   int N, cudaStream_t st) {
  if (M <= 0) return DTB_OK;
  DenseTcWgradParams p{};
  p.NT = dt_nt(N);
  const int n_tiles = (N + p.NT - 1) / p.NT;
  p.X = X; p.dZ = dZ; p.dW = dW; p.dbias = dbias;
  p.M = M; p.K = K; p.N = N; p.ldx = ldx; p.ldz = ldz; p.ldw = ldw;
  p.n_chunks_total = (M + kDtKc - 1) / kDtKc;
  const int k_tiles = (K + 127) / 128;
  int splits = sm_count() / (k_tiles * n_tiles);
  if (splits < 1) splits = 1;
  if (splits > p.n_chunks_total) splits = p.n_chunks_total;
  p.chunks_per_split = (p.n_chunks_total + splits - 1) / splits;
  splits = (p.n_chunks_total + p.chunks_per_split - 1) / p.chunks_per_split;
  const dim3 grid(k_tiles, splits, n_tiles);
  switch (p.NT) {
    case 16: return dt_launch_wgrad<16>(p, grid, st);
    case 32: return dt_launch_wgrad<32>(p, grid, st);
    case 64: return dt_launch_wgrad<64>(p, grid, st);
    default: return dt_launch_wgrad<kDtMaxNT>(p, grid, st);
  }
}

// ------------------------------------------------------------------------------------------
// tensor-core self test: C[128, N] = bf16(A[128, K]) . bf16(B[K, N]), one warpgroup, two m64 row blocks.  Isolates
// descriptor / operand-layout mistakes from the GEMM pipelines above: B in the K-major image of the weight pack, A
// either in the same image form (shared memory) or as register fragments.
// ------------------------------------------------------------------------------------------
template <int N, bool kARegs>
__global__ void __launch_bounds__(128, 1) tc_selftest_kernel(const float* __restrict__ A, const float* __restrict__ Bm,
                                                             float* __restrict__ C, int K) {
  __shared__ __align__(128) uint8_t smem_b[N * 64 * 2];
  __shared__ __align__(128) uint8_t smem_a[128 * 64 * 2];
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  for (int e = t; e < K * N; e += 128) {
    const int k = e / N, n = e - k * N;
    const int off = ((k >> 3) * (N >> 3) + (n >> 3)) * 128 + (n & 7) * 16 + (k & 7) * 2;
    *reinterpret_cast<__nv_bfloat16*>(smem_b + off) = __float2bfloat16_rn(Bm[e]);
  }
  if (!kARegs) {
    for (int e = t; e < 128 * K; e += 128) {
      const int r = e / K, k = e - r * K;
      const int off = ((k >> 3) * 16 + (r >> 3)) * 128 + (r & 7) * 16 + (k & 7) * 2;
      *reinterpret_cast<__nv_bfloat16*>(smem_a + off) = __float2bfloat16_rn(A[e]);
    }
  }
  tc::fence_proxy_async_smem();
  __syncthreads();
  float acc[2][N / 2];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[h][i] = 0.f;
  const int r0 = warp * 16 + (lane >> 2), c0 = 2 * (lane & 3);
  constexpr uint32_t lbo_b = (N >> 3) * 128;
  tc::wgmma_fence();
  for (int ks = 0; ks < K / 16; ++ks) {
    const uint64_t db = tc::make_smem_desc(tc::smem_u32(smem_b) + ks * 2 * lbo_b, lbo_b, 128);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if constexpr (kARegs) {
        const float* a = A + (int64_t)(h * 64 + r0) * K + ks * 16 + c0;
        const uint32_t frag[4] = {tc::pack_bf16x2(a[0], a[1]), tc::pack_bf16x2(a[8 * K], a[8 * K + 1]),
                                  tc::pack_bf16x2(a[8], a[9]), tc::pack_bf16x2(a[8 * K + 8], a[8 * K + 9])};
        tc::Wgmma<N>::rs(acc[h], frag, db, ks != 0);
      } else {
        const uint64_t da = tc::make_smem_desc(tc::smem_u32(smem_a) + ks * 4096 + h * 1024, 2048, 128);
        tc::Wgmma<N>::ss(acc[h], da, db, ks != 0);
      }
    }
  }
  tc::wgmma_commit();
  tc::wgmma_wait<0>();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    tc::wgmma_fence_acc(acc[h]);
#pragma unroll
    for (int i = 0; i < N / 2; ++i)
      C[(h * 64 + r0 + (((i >> 1) & 1) << 3)) * N + 8 * (i >> 2) + c0 + (i & 1)] = acc[h][i];
  }
}

template <int N>
static int tc_selftest_launch(const float* A, const float* Bm, float* C, int K, int a_regs, cudaStream_t st) {
  if (a_regs) tc_selftest_kernel<N, true><<<1, 128, 0, st>>>(A, Bm, C, K);
  else tc_selftest_kernel<N, false><<<1, 128, 0, st>>>(A, Bm, C, K);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

}  // namespace dtb

extern "C" int dtb_tc_selftest(const float* A, const float* Bmat, float* C, void* workspace, int N, int K,
                               int a_operand_in_regs, void* stream) {
  DTB_CHECK_ARG(A && Bmat && C && workspace, "NULL argument");
  DTB_CHECK_ARG((N == 16 || N == 32 || N == 64 || N == 128) && K % 16 == 0 && K >= 16 && K <= 64,
                "N in {16, 32, 64, 128}, K <= 64 a multiple of 16");
  cudaStream_t st = (cudaStream_t)stream;
  switch (N) {
    case 16: return dtb::tc_selftest_launch<16>(A, Bmat, C, K, a_operand_in_regs, st);
    case 32: return dtb::tc_selftest_launch<32>(A, Bmat, C, K, a_operand_in_regs, st);
    case 64: return dtb::tc_selftest_launch<64>(A, Bmat, C, K, a_operand_in_regs, st);
    default: return dtb::tc_selftest_launch<128>(A, Bmat, C, K, a_operand_in_regs, st);
  }
}
