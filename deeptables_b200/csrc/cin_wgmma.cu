// CIN forward and backward fused on the Hopper tensor cores (precision codes 2-4).
//
// For batch row b, embedding dim d:  T_k[(b,d), l] = sum_{i,j} x0[b,i,d] h_k[b,j,d] W_k[i*H + j, l].  One warpgroup
// owns 64 GEMM rows m = (b, d).  The A operand Z_k[m, (i,j)] = x0[m,i] h_k[m,j] never exists in memory: each thread
// keeps h_k of its two accumulator rows in registers, in the accumulator's own fragment layout, which is also the
// register layout wgmma expects for an A operand -- so layer k's output feeds layer k+1 without leaving the registers.
// Per x0 field i the thread scales its h fragment by x0[m,i] and issues wgmma with A from registers; the weight chunk
// of field i (all hidden fields x all feature maps, pre-packed as K-major bf16/fp16 core matrices) arrives in shared
// memory by one bulk async copy.  A forward CTA (one per SM) runs two such warpgroups on a pair of adjacent tiles, so
// each chunk is copied once per 128 rows, into a ring of full/empty mbarrier stages; a third, producer warpgroup owns
// the copies, gathers the next pair's x0 rows, and stores each finished layer's saved rows and pooled sums from a
// shared-memory staging tile while the consumers go on to the next layer.
//
// Precision: 2 = bf16x3 split (Z_hi W_hi + Z_lo W_hi + Z_hi W_lo: fp32-grade), 3 = one bf16 pass, 4 = one fp16 pass on
// operands scaled by exact powers of two (per GEMM row for Z, per layer for W_k), undone on the fp32 accumulator.
// The saved activations have the layout of the any-shape formulation (x0t, then T_k).  The backward (below) runs the
// data and weight gradients as two fused wgmma kernels in bf16x3 for every precision code.  The data-gradient kernel
// (one warpgroup per CTA; one W_k^T chunk serves two x0 fields where 2 H_k <= NPJ) hands dC_k to the
// weight-gradient kernel already split into the bf16 hi/lo image wgmma reads; the weight-gradient CTA is two
// warpgroups that share each copied 64-row block among four m64 A tiles (one or two x0 fields each), fed by a
// multi-stage ring that a third, producer warpgroup refills.
#include "dtb_common.cuh"
#include "cin_impl.h"
#include "wgmma.cuh"
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cudaTypedefs.h>      // CUtensorMap, PFN_cuTensorMapEncodeTiled
#include <type_traits>

namespace dtb {

constexpr int kWgRows = 64;          // GEMM rows per CTA (one m64 wgmma block)
constexpr int kWgMaxHp = 64;         // padded hidden fields per layer (wgmma K per x0 field)
constexpr int kWgMaxNP = 128;        // feature maps per layer (wgmma N)

static inline int round_up16(int x) { return (x + 15) / 16 * 16; }

struct CinWgParams {
  const int32_t* idx;
  const float* table;
  const int64_t* row_offsets;
  const uint8_t* wpack;
  const float* bias;
  float* pooled;
  float* saved;          // training: x0t [B*D, F] then T_k [B*D, L_k]; null for inference
  int* status;
  const int* wmax;       // fp16: bit pattern of max|W_k| per layer
  int B, D, F, n_layers, act, P;
  int n_tiles;           // 64-row tiles: ceil(B * D / 64)
  int hp_max, stages;    // the widest layer's padded hidden fields; weight-chunk stages in shared memory
  int L[kCinMaxLayers], Hp[kCinMaxLayers], hid_n[kCinMaxLayers];
  int pool_lo[kCinMaxLayers], pool_n[kCinMaxLayers], pcol0[kCinMaxLayers];
  unsigned long long wpack_off[kCinMaxLayers], saved_off[kCinMaxLayers], bias_off[kCinMaxLayers];
};

// bytes of one x0 field's weight chunk of layer k: NP feature maps x Hp hidden fields, hi (+ lo) image
__host__ __device__ inline uint32_t cin_wg_chunk_bytes(int NP, int Hp, int mode) {
  return (uint32_t)NP * Hp * 2 * (mode == 0 ? 2 : 1);
}

// W_k [F*H, L] -> per field i: image of B[n][kk] = W_k[(i*H + kk), n] (zero outside H x L), core (kk/8, n/8) at
// ((kk/8)*(NP/8) + n/8)*128 B, row n%8 at 16 B, element kk%8 at 2 B.  mode 0: bf16 hi then lo image; 1: bf16 hi only;
// 2: fp16 of W scaled by the power of two that brings max|W_k| into [2^9, 2^10).
__global__ void cin_wg_pack_kernel(const float* __restrict__ w, uint8_t* __restrict__ out, int F, int H, int Hp, int L,
                                   int NP, int mode, const int* __restrict__ wmax) {
  float s = 1.f, inv;
  if (mode == 2) tc::pow2_scale_to_1024(__int_as_float(*wmax), s, inv);
  const int64_t per_chunk = (int64_t)NP * Hp;
  const int64_t total = per_chunk * F;
  const uint32_t chunk_bytes = cin_wg_chunk_bytes(NP, Hp, mode);
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(t / per_chunk);
    const int rem = (int)(t - (int64_t)i * per_chunk);
    const int kk = rem / NP, n = rem - kk * NP;
    const float v = (kk < H && n < L) ? w[((int64_t)i * H + kk) * L + n] : 0.f;
    const int64_t off = ((int64_t)(kk >> 3) * (NP >> 3) + (n >> 3)) * 128 + (n & 7) * 16 + (kk & 7) * 2;
    uint8_t* base = out + (int64_t)i * chunk_bytes;
    if (mode == 2) {
      *reinterpret_cast<__half*>(base + off) = __float2half_rn(v * s);
    } else {
      const __nv_bfloat16 hi = __float2bfloat16_rn(v);
      *reinterpret_cast<__nv_bfloat16*>(base + off) = hi;
      if (mode == 0) *reinterpret_cast<__nv_bfloat16*>(base + per_chunk * 2 + off) = __float2bfloat16_rn(v - __bfloat162float(hi));
    }
  }
}

__global__ void cin_wg_wmax_kernel(const float* __restrict__ w, int64_t n, int* __restrict__ out) {
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float a = fabsf(w[i]);
    if (a < __int_as_float(0x7f800000)) m = fmaxf(m, a);      // ignore inf / nan
  }
  for (int off = 16; off >= 1; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out, __float_as_int(m));    // non-negative floats order as ints
}

// Forward CTA: consumer warpgroups 0 and 1 each own one 64-row tile of a pair of adjacent tiles (128 GEMM rows) and
// share every weight chunk copied for the pair; producer warpgroup 2 brings the chunks into a ring of full/empty
// mbarrier stages (thread 0 of its first warp), gathers the x0 rows of the next pair into the other of two x0 slots
// and takes each finished layer's tile from the consumers' staging buffers to the saved T_k rows and the pooled sums
// (its other three warps).  One CTA per SM runs pairs blockIdx.x, blockIdx.x + gridDim.x, ...
constexpr int kFwdThreads = 384;
constexpr int kFwdMaxStages = 8;
constexpr int kFwdAux = 96;             // producer threads that gather x0 and store the epilogues (warps 1-3 of it)
// the registers the CTA gets at launch (384 x 168) are shared out again: 2 x 128 x 216 + 128 x 72 = 384 x 168
constexpr int kFwdConsumerRegs = 216, kFwdProducerRegs = 72;

struct CinWgSmem {
  int stage, x0_off, ot_off, bar_off, total;
};
// stages x weight chunks of the widest layer (hp_max), two x0 slots of 128 rows, one staging tile per consumer, and
// the mbarriers: full/empty per stage, x0 full per slot, staging full/empty per consumer
__host__ __device__ inline CinWgSmem cin_wg_layout(int NP, int F, int mode, int hp_max, int stages) {
  CinWgSmem l;
  l.stage = (int)cin_wg_chunk_bytes(NP, hp_max, mode);
  l.x0_off = stages * l.stage;
  l.ot_off = l.x0_off + (2 * 2 * kWgRows * F * 4 + 127) / 128 * 128;
  l.bar_off = l.ot_off + 2 * kWgRows * (NP + 1) * 4;
  l.total = l.bar_off + 8 * (2 * stages + 2 + 4);
  return l;
}
// as many stages as fit in shared memory, 2 to kFwdMaxStages (0: not even 2 fit)
static int cin_wg_fwd_stages(int NP, int F, int mode, int hp_max) {
  int s = kFwdMaxStages;
  while (s >= 2 && cin_wg_layout(NP, F, mode, hp_max, s).total > 227 * 1024) --s;
  return s >= 2 ? s : 0;
}

// weight chunk of layer k, x0 field i -> source and size
__device__ __forceinline__ void cin_wg_chunk_src(const CinWgParams& p, int NP, int mode, int k, int i, const uint8_t*& src,
                                                 uint32_t& bytes) {
  bytes = cin_wg_chunk_bytes(NP, p.Hp[k], mode);
  src = p.wpack + p.wpack_off[k] + (size_t)i * bytes;
}

template <int NP, int kMode>
__global__ void __launch_bounds__(kFwdThreads, 1) cin_wg_fwd_kernel(const __grid_constant__ CinWgParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int S = p.stages;
  const CinWgSmem lay = cin_wg_layout(NP, p.F, kMode, p.hp_max, S);
  float* x0buf = reinterpret_cast<float*>(smem + lay.x0_off);    // slot s: [128 rows][F]
  float* otbuf = reinterpret_cast<float*>(smem + lay.ot_off);    // consumer w: [64 rows][NP + 1]
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + lay.bar_off);
  uint64_t* empty = full + S;
  uint64_t* x0_full = empty + S;
  uint64_t* ot_full = x0_full + 2;
  uint64_t* ot_empty = ot_full + 2;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, wq = warp & 3;
  const int F = p.F, D = p.D;
  const int64_t BD = (int64_t)p.B * D;
  const int n_tiles = p.n_tiles, n_pairs = (p.n_tiles + 1) / 2;      // from the parameters: reloaded, not spilled

  if (tid == 0) {
    for (int s = 0; s < S; ++s) {
      tc::mbar_init(&full[s], 1);
      tc::mbar_init(&empty[s], 8);      // each warp of both consumers; a consumer alone in a pair arrives twice
    }
    for (int s = 0; s < 2; ++s) {
      tc::mbar_init(&x0_full[s], kFwdAux);
      tc::mbar_init(&ot_full[s], 128);
      tc::mbar_init(&ot_empty[s], kFwdAux);
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (wg == 2) {
    tc::setmaxnreg_dec<kFwdProducerRegs>();
    const int pt = tid - 2 * 128;
    if (pt == 0) {
      // weight chunks: pair x layer x field, chunk c into stage c % S once both consumers released chunk c - S
      int st = 0;
      uint32_t ph = 0, c = 0;
      for (int pr = blockIdx.x; pr < n_pairs; pr += gridDim.x)
        for (int k = 0; k < p.n_layers; ++k)
          for (int i = 0; i < F; ++i, ++c) {
            const uint8_t* src;
            uint32_t bytes;
            cin_wg_chunk_src(p, NP, kMode, k, i, src, bytes);
            if (c >= (uint32_t)S) tc::mbar_wait(&empty[st], ph ^ 1);
            tc::mbar_arrive_expect_tx(&full[st], bytes);
            tc::bulk_g2s(smem + st * lay.stage, src, bytes, &full[st]);
            if (++st == S) { st = 0; ph ^= 1; }
          }
    } else if (pt >= 32) {
      const int gt = pt - 32, gw = gt >> 5;
      const int lgD = __ffs(D) - 1;      // D is a power of two
      // x0 rows of pair pr into slot s (m fastest: consecutive threads read consecutive floats of one embedding row),
      // then the pair's x0t block, contiguous in saved, from shared memory
      auto gather = [&](int pr, int s) {
        float* xs = x0buf + s * 2 * kWgRows * F;
        const int64_t gm0 = (int64_t)pr * 2 * kWgRows;
        const int n = 2 * kWgRows * F;
        constexpr int U = 4;      // independent id -> row -> value chains in flight per thread
        for (int e0 = gt; e0 < n; e0 += kFwdAux * U) {
          int64_t rb[U];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int e = e0 + u * kFwdAux, i = e >> 7;
            const int64_t gm = gm0 + (e & 127), b = gm >> lgD;
            rb[u] = -1;
            if (e < n && gm < BD) {
              rb[u] = table_row(p.row_offsets, i, __ldg(p.idx + b * F + i), D, p.status);
              if (rb[u] >= 0) rb[u] += gm & (D - 1);
            }
          }
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int e = e0 + u * kFwdAux;
            if (e < n) xs[(e & 127) * F + (e >> 7)] = rb[u] >= 0 ? __ldg(p.table + rb[u]) : 0.f;
          }
        }
        tc::named_bar_sync(1, kFwdAux);
        tc::mbar_arrive(&x0_full[s]);
        if (p.saved) {
          const int rows = BD - gm0 < 2 * kWgRows ? (int)(BD - gm0) : 2 * kWgRows;
          for (int e = gt; e < rows * F; e += kFwdAux) p.saved[gm0 * F + e] = xs[e];
        }
      };
      uint32_t ot_ph = 0;      // bit w: phase of consumer w's staging-full barrier
      int jj = 0;
      if ((int)blockIdx.x < n_pairs) gather(blockIdx.x, 0);
      // the next pair's x0 goes in after this pair's layer-0 tiles are stored (before them with one layer): a
      // consumer waits for the store of layer k at the end of layer k + 1, and layers 1 and more are the long ones
      const int k_gather = p.n_layers > 1 ? 1 : 0;
      for (int pr = blockIdx.x; pr < n_pairs; pr += gridDim.x, ++jj) {
        const int nw = 2 * pr + 1 < n_tiles ? 2 : 1;
        for (int k = 0; k < p.n_layers; ++k) {
          // slot (jj + 1) & 1 held pair jj - 1, whose last layer both consumers have handed over: its x0 is read
          if (k == k_gather && pr + (int)gridDim.x < n_pairs) gather(pr + gridDim.x, (jj + 1) & 1);
          const int L = p.L[k], rows_b = kWgRows / D, pool_n = p.pool_n[k];
          for (int w = 0; w < nw; ++w) {
            const float* ot = otbuf + w * kWgRows * (NP + 1);
            const int64_t gm0 = (int64_t)(2 * pr + w) * kWgRows;
            tc::mbar_wait(&ot_full[w], (ot_ph >> w) & 1);
            ot_ph ^= 1u << w;
            if (p.saved) {
              float* T = p.saved + p.saved_off[k];
              for (int m = gw; m < kWgRows; m += kFwdAux / 32)
                if (gm0 + m < BD)
                  for (int col = lane; col < L; col += 32) T[(gm0 + m) * L + col] = ot[m * (NP + 1) + col];
            }
            for (int e = gt; e < rows_b * pool_n; e += kFwdAux) {
              const int bl = e / pool_n, q = e - bl * pool_n;
              const int64_t b = gm0 / D + bl;
              if (b < p.B) {
                float sum = 0.f;
                for (int d = 0; d < D; ++d) sum += ot[(bl * D + d) * (NP + 1) + p.pool_lo[k] + q];
                p.pooled[b * p.P + p.pcol0[k] + q] = sum;
              }
            }
            tc::mbar_arrive(&ot_empty[w]);
          }
        }
      }
    }
    return;
  }
  tc::setmaxnreg_inc<kFwdConsumerRegs>();

  // consumers
  const int r0 = wq * 16 + (lane >> 2), c2 = 2 * (lane & 3);    // accumulator rows r0, r0 + 8; column pair base
  constexpr uint32_t lbo_b = (NP >> 3) * 128;
  constexpr bool kTwoSets = kMode != 0;      // A-fragment sets: one wgmma group in flight while the next is built
  float* ot = otbuf + wg * kWgRows * (NP + 1);
  int st = 0, ep = 0;
  uint32_t ph = 0;
  int jj = 0;
  for (int pr = blockIdx.x; pr < n_pairs; pr += gridDim.x, ++jj) {
    if (2 * pr + wg >= n_tiles) break;      // the last pair of an odd tile count: warpgroup 1 has no tile
    const uint32_t rel = 2 * pr + 1 < n_tiles ? 1u : 2u;      // empty-barrier arrivals per warp
    const float* x0s = x0buf + ((jj & 1) * 2 + wg) * kWgRows * F;      // [m][i]
    tc::mbar_wait(&x0_full[jj & 1], (jj >> 1) & 1);
    // h_0 = x0, in accumulator fragment order: hh[q] = h[row r0 + 8*((q>>1)&1), col 8*(q>>2) + c2 + (q&1)]
    float hh[kWgMaxHp / 2];
#pragma unroll
    for (int q = 0; q < kWgMaxHp / 2; ++q) {
      const int row = r0 + (((q >> 1) & 1) << 3), col = 8 * (q >> 2) + c2 + (q & 1);
      hh[q] = col < F ? x0s[row * F + col] : 0.f;
    }
    for (int k = 0; k < p.n_layers; ++k) {
      const int Hp = p.Hp[k], L = p.L[k];
      // fp16: srow scales the thread's two Z rows into range, inv_acc undoes it and the weight scale on the
      // accumulator.  Both come from x0, h and max|W_k| alone, so inv_acc is worked out again for the epilogue
      // rather than held through the MMAs (hh does not change in between).
      [[maybe_unused]] float srow[2] = {1.f, 1.f}, inv_acc[2] = {1.f, 1.f};
      auto fp16_scales = [&]() {
        float xmax[2] = {0.f, 0.f};
        for (int i = 0; i < F; ++i) {
          xmax[0] = fmaxf(xmax[0], fabsf(x0s[r0 * F + i]));
          xmax[1] = fmaxf(xmax[1], fabsf(x0s[(r0 + 8) * F + i]));
        }
        float sw, inv_w;
        tc::pow2_scale_to_1024(__int_as_float(__ldg(p.wmax + k)), sw, inv_w);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float m = 0.f;
#pragma unroll
          for (int q = 0; q < kWgMaxHp / 2; ++q)
            if (((q >> 1) & 1) == h && q < Hp / 2) m = fmaxf(m, fabsf(hh[q]));      // stale entries beyond Hp
          m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
          m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
          float inv_row;
          tc::pow2_scale_to_1024(xmax[h] * m, srow[h], inv_row);
          inv_acc[h] = inv_row * inv_w;
        }
      };
      if constexpr (kMode == 2) fp16_scales();
      float acc[NP / 2];
#pragma unroll
      for (int q = 0; q < NP / 2; ++q) acc[q] = 0.f;
      // the layer's fields with KS = Hp / 16 k-steps known at compile time: a branch on Hp between wgmma groups in
      // flight would make ptxas serialize every wgmma
      auto run_layer = [&](auto ks_c) {
        constexpr int KS = decltype(ks_c)::value;
        // A fragments of field i: Z[m, kk] = x0[m, i] h[m, kk]
        auto build = [&](uint32_t (&ahi)[KS][4], uint32_t (&alo)[KS][4], int i) {
          float x[2] = {x0s[r0 * F + i], x0s[(r0 + 8) * F + i]};
          if constexpr (kMode == 2) { x[0] *= srow[0]; x[1] *= srow[1]; }
#pragma unroll
          for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
            for (int f = 0; f < 4; ++f) {
              const float xv = x[f & 1];
              const float z0 = xv * hh[8 * ks + 2 * f], z1 = xv * hh[8 * ks + 2 * f + 1];
              if constexpr (kMode == 0) tc::split_bf16x2(z0, z1, ahi[ks][f], alo[ks][f]);
              else if constexpr (kMode == 1) ahi[ks][f] = tc::pack_bf16x2(z0, z1);
              else ahi[ks][f] = tc::pack_f16x2(z0, z1);
            }
          }
        };
        // field i: its MMAs on the chunk in stage st go out; once field i - 1's are done, its stage is released and
        // the fragments of field i + 1 are built into the set field i - 1 used, while field i's MMAs run.  bf16x3
        // has no registers for a second hi + lo set next to the accumulator (ptxas serializes the wgmma): it waits
        // for field i's MMAs, releases their stage and builds into the same set, while the other consumer multiplies.
        auto field = [&](uint32_t (&ahi)[KS][4], uint32_t (&alo)[KS][4], uint32_t (&nhi)[KS][4],
                         uint32_t (&nlo)[KS][4], int i) {
          tc::mbar_wait(&full[st], ph);
          const uint32_t b_hi = tc::smem_u32(smem + st * lay.stage);
          const uint32_t b_lo = b_hi + (uint32_t)NP * KS * 16 * 2;
          tc::wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < KS; ++ks) {
            const uint32_t first = (i == 0 && ks == 0) ? 0u : 1u;
            const uint64_t dh = tc::make_smem_desc(b_hi + ks * 2 * lbo_b, lbo_b, 128);
            if constexpr (kMode == 2) {
              tc::WgmmaF16<NP>::rs(acc, ahi[ks], dh, first);
            } else {
              tc::Wgmma<NP>::rs(acc, ahi[ks], dh, first);
              if constexpr (kMode == 0) {
                tc::Wgmma<NP>::rs(acc, alo[ks], dh, 1u);
                tc::Wgmma<NP>::rs(acc, ahi[ks], tc::make_smem_desc(b_lo + ks * 2 * lbo_b, lbo_b, 128), 1u);
              }
            }
          }
          tc::wgmma_commit();
          if constexpr (kTwoSets) {
            tc::wgmma_wait<1>();
            tc::mbar_arrive_if(&empty[st == 0 ? S - 1 : st - 1], rel, i > 0 && lane == 0);
          } else {
            tc::wgmma_wait<0>();
            tc::mbar_arrive_if(&empty[st], rel, lane == 0);
          }
          if (++st == S) { st = 0; ph ^= 1; }
          if (i + 1 < F) build(nhi, nlo, i + 1);
        };
        uint32_t ahi0[KS][4], alo0[KS][4], ahi1[KS][4], alo1[KS][4];
        build(ahi0, alo0, 0);
        for (int i = 0; i < F; i += 2) {
          if constexpr (kTwoSets) {
            field(ahi0, alo0, ahi1, alo1, i);
            if (i + 1 < F) field(ahi1, alo1, ahi0, alo0, i + 1);
          } else {
            field(ahi0, alo0, ahi0, alo0, i);
            if (i + 1 < F) field(ahi0, alo0, ahi0, alo0, i + 1);
          }
        }
        tc::wgmma_wait<0>();
      };
      switch (Hp >> 4) {
        case 1: run_layer(std::integral_constant<int, 1>{}); break;
        case 2: run_layer(std::integral_constant<int, 2>{}); break;
        case 3: run_layer(std::integral_constant<int, 3>{}); break;
        default: run_layer(std::integral_constant<int, 4>{}); break;
      }
      tc::wgmma_fence_acc(acc);
      if constexpr (kTwoSets) tc::mbar_arrive_if(&empty[st == 0 ? S - 1 : st - 1], rel, lane == 0);
      if constexpr (kMode == 2) fp16_scales();
      // ---- epilogue of layer k: bias / act in registers, then the tile goes to the staging buffer once the producer
      //      has taken the previous one; the producer stores the saved rows and the pooled sums from it
      const float* bias = p.bias ? p.bias + p.bias_off[k] : nullptr;
      const int hid_next = k + 1 < p.n_layers ? p.hid_n[k] : 0;
      if (ep > 0) tc::mbar_wait(&ot_empty[wg], (ep - 1) & 1);
      ++ep;
#pragma unroll
      for (int q = 0; q < NP / 2; ++q) {
        const int h = (q >> 1) & 1;
        const int row = r0 + (h << 3), col = 8 * (q >> 2) + c2 + (q & 1);
        float v = acc[q];
        if constexpr (kMode == 2) v *= inv_acc[h];
        if (bias && col < L) v += __ldg(bias + col);
        if (p.act == DTB_ACT_RELU) v = fmaxf(v, 0.f);
        if (col < L) ot[row * (NP + 1) + col] = v;
        if (q < kWgMaxHp / 2) hh[q] = col < hid_next ? v : 0.f;
      }
      tc::mbar_arrive(&ot_full[wg]);
    }
  }
}

// ==========================================================================================
// Backward (bf16x3 split, every precision code), two kernels:
//   dgrad, per 64-row tile, layers last -> first (one warpgroup per CTA):
//     dC_k = (d_pooled part + dh_{k+1}) * act'(T_k)                 registers, accumulator fragment layout
//     dZ_{k,i}[m, j] = sum_l dC_k[m, l] W_k[i*H + j, l]             wgmma: A = dC_k from registers, B = W_k^T chunk
//     dx0[m, i] += sum_j dZ h_k[m, j] ;  dh_k[m, j] += dZ x0[m, i]   registers (dh_k feeds dC_{k-1})
//     N = NPJ, the padded largest H.  Where 2 H_k <= NPJ, one chunk holds fields 2t and 2t + 1 (columns [0, NPJ/2) and
//     [NPJ/2, NPJ)), so a narrow layer (layer 0 at the headline shape) runs half the MMAs and copies half the weights.
//     dC_k is stored as the bf16 hi/lo image the weight gradient multiplies (below), its column sums go to d_bias,
//     and dx0 is scattered into grad_table.
//   wgrad, per (layer k, group of x0 fields, row split):
//     dW_k[i*H + j, l] += sum_m x0[m, i] h_k[m, j] dC_k[m, l]       wgmma: A = x0 h from registers (rows j),
//                                                                   B = dC_k block as a K-major image (K = m)
//     Two consumer warpgroups x two m64 A tiles per CTA, plus a producer warpgroup: one copy of each 64-row block
//     (dC_k image and x0 rows by bulk copy; for k >= 1 the h_k rows by one 2-D tensor copy of their first hpitch
//     columns, or whole rows by bulk copy when ldh % 4 != 0) serves four tiles.  A tile holds one field (H > 32) or
//     two (rows 0-31 and 32-63).  The blocks pass through a ring of up to four stages (as many as fit in shared
//     memory) with a full and an empty mbarrier each.  One producer thread owns every empty-barrier wait and every
//     refill (setmaxnreg: 24 registers for it, 240 for the consumers); the consumers only wait on full barriers,
//     build A fragments (branch-free, each h value read once per block) and issue wgmma, releasing a stage once their
//     MMAs on it are done.  No CTA-wide barrier sits in the loop, so one warpgroup builds while the other multiplies.
//     A last field group with tiles for one warpgroup only runs them on both, on alternate blocks, and gets a longer
//     row split than the full groups, so that all SMs have work and finish together.
// ==========================================================================================

// dC_k of one 64-row block: K-major image (K = m, N = l < NP) of bf16 hi then lo, core (m/8, l/8) at
// ((m/8)*(NP/8) + l/8)*128 B, row l%8 at 16 B, element m%8 at 2 B.  Zero past L_k and past the last row.
__host__ __device__ inline uint32_t cin_wg_dc_block_bytes(int NP) { return (uint32_t)NP * kWgRows * 4; }

struct CinWgBwdParams {
  const int32_t* idx;
  const int64_t* row_offsets;
  const uint8_t* wpack;      // per layer, per chunk of fpc x0 fields: W_k^T image [NPJ x LP], hi then lo
  const float* d_pooled;
  const float* saved;        // x0t [B*D, F] then T_k [B*D, L_k]
  float* grad_table;
  uint8_t* dc;               // dC_k images, per layer, per 64-row block (cin_wg_dc_block_bytes(NPdc))
  float* dbias;              // null, or d_bias of all layers (offsets bias_off)
  int B, D, F, n_layers, act, P, NPdc;
  int L[kCinMaxLayers], LP[kCinMaxLayers], H[kCinMaxLayers], hid_n[kCinMaxLayers];
  int fpc[kCinMaxLayers];    // x0 fields per weight chunk: 2 when 2 H_k <= NPJ, else 1
  int nch[kCinMaxLayers];    // weight chunks of layer k: ceil(F / fpc)
  int pool_lo[kCinMaxLayers], pool_n[kCinMaxLayers], pcol0[kCinMaxLayers];
  unsigned long long wpack_off[kCinMaxLayers], saved_off[kCinMaxLayers], dc_off[kCinMaxLayers], bias_off[kCinMaxLayers];
};

// W_k [F*H, L] -> per chunk c of fpc x0 fields: K-major image of B[n][kk] = W_k[i*H + j, kk], N = NPJ, K = LP, where
// field i = c*fpc + n / (NPJ/fpc) and j = n % (NPJ/fpc); zero for j >= H, i >= F or kk >= L
__global__ void cin_wg_pack_t_kernel(const float* __restrict__ w, uint8_t* __restrict__ out, int F, int H, int L, int LP,
                                     int NPJ, int fpc) {
  const int64_t per_chunk = (int64_t)NPJ * LP;
  const int64_t total = per_chunk * ((F + fpc - 1) / fpc);
  const int half = NPJ / fpc;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(t / per_chunk);
    const int rem = (int)(t - (int64_t)c * per_chunk);
    const int n = rem / LP, kk = rem - n * LP;          // kk fastest: coalesced reads of W rows
    const int sub = n / half, j = n - sub * half, i = c * fpc + sub;
    const float v = (i < F && j < H && kk < L) ? w[((int64_t)i * H + j) * L + kk] : 0.f;
    const int64_t off = ((int64_t)(kk >> 3) * (NPJ >> 3) + (n >> 3)) * 128 + (n & 7) * 16 + (kk & 7) * 2;
    uint8_t* base = out + (int64_t)c * per_chunk * 4;
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    *reinterpret_cast<__nv_bfloat16*>(base + off) = hi;
    *reinterpret_cast<__nv_bfloat16*>(base + per_chunk * 2 + off) = __float2bfloat16_rn(v - __bfloat162float(hi));
  }
}

struct CinWgBwdSmem {
  int w_off, x0_off, dx_off, bsum_off, bar_off, total;
};
__host__ __device__ inline CinWgBwdSmem cin_wg_bwd_layout(int NPJ, int F) {
  CinWgBwdSmem l;
  l.w_off = 0;
  l.x0_off = 2 * NPJ * kWgMaxNP * 4;                 // two W^T chunk buffers (hi + lo)
  l.dx_off = l.x0_off + kWgRows * F * 4;
  l.bsum_off = l.dx_off + kWgRows * F * 4;           // this CTA's d_bias partial sums [layer][l]
  l.bar_off = (l.bsum_off + kCinMaxLayers * kWgMaxNP * 4 + 15) / 16 * 16;
  l.total = l.bar_off + 16;
  return l;
}

template <int NPJ>
__global__ void __launch_bounds__(128) cin_wg_dgrad_kernel(const __grid_constant__ CinWgBwdParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const CinWgBwdSmem lay = cin_wg_bwd_layout(NPJ, p.F);
  constexpr uint32_t wbuf_bytes = NPJ * kWgMaxNP * 4;
  uint8_t* wbuf = smem + lay.w_off;
  float* x0s = reinterpret_cast<float*>(smem + lay.x0_off);      // [m][i]
  float* dxs = reinterpret_cast<float*>(smem + lay.dx_off);      // [m][i]
  float* bsum = reinterpret_cast<float*>(smem + lay.bsum_off);   // [k][l]
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + lay.bar_off);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int F = p.F, D = p.D;
  const int64_t BD = (int64_t)p.B * D;
  const int n_tiles = (int)((BD + kWgRows - 1) / kWgRows);
  const int r0 = warp * 16 + (lane >> 2), c2 = 2 * (lane & 3);
  constexpr uint32_t lbo_b = (NPJ >> 3) * 128;
  const int K0 = p.n_layers - 1;
  const int NPdc = p.NPdc;
  const uint32_t dc_img = NPdc * kWgRows * 2;                     // bytes of the hi (and of the lo) image of a block
  const bool do_bias = p.dbias != nullptr;
  const bool odd_row = (lane >> 2) & 1;
  for (int e = tid; e < kCinMaxLayers * kWgMaxNP; e += 128) bsum[e] = 0.f;

  if (tid == 0) {
    tc::mbar_init(&full[0], 1);
    tc::mbar_init(&full[1], 1);
    tc::fence_barrier_init();
  }
  __syncthreads();
  auto issue = [&](uint32_t c, int k, int i) {
    const uint32_t bytes = (uint32_t)NPJ * p.LP[k] * 4;
    tc::mbar_arrive_expect_tx(&full[c & 1], bytes);
    tc::bulk_g2s(wbuf + (c & 1) * wbuf_bytes, p.wpack + p.wpack_off[k] + (size_t)i * bytes, bytes, &full[c & 1]);
  };
  if (tid == 0 && (int)blockIdx.x < n_tiles) issue(0, K0, 0);

  uint32_t chunk = 0;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t gm0 = (int64_t)tile * kWgRows;
    for (int e = tid; e < kWgRows * F; e += 128) {
      const int m = e / F;
      x0s[e] = gm0 + m < BD ? p.saved[gm0 * F + e] : 0.f;
      dxs[e] = 0.f;
    }
    __syncthreads();
    // the thread's two accumulator rows r0, r0 + 8: inside the batch?  which batch row?
    bool row_ok[2];
    int64_t row_b[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      row_ok[h] = gm0 + r0 + 8 * h < BD;
      row_b[h] = row_ok[h] ? (gm0 + r0 + 8 * h) / D : 0;
    }
    float dh[NPJ / 2];                   // gradient wrt h_{k+1}, accumulator fragment order (columns j)
#pragma unroll
    for (int q = 0; q < NPJ / 2; ++q) dh[q] = 0.f;
    for (int k = K0; k >= 0; --k) {
      const int L = p.L[k], LP = p.LP[k], H = p.H[k];
      // ---- dC_k in A-fragment order: dc element q <-> row r0 + 8*((q>>1)&1), column l = 8*(q>>2) + c2 + (q&1)
      uint32_t ahi[kWgMaxNP / 16][4], alo[kWgMaxNP / 16][4];
      {
        const float* T = p.saved + p.saved_off[k];
        uint8_t* img = p.dc + p.dc_off[k] + (size_t)tile * cin_wg_dc_block_bytes(NPdc);
        // All global reads of the layer come first, in a loop with no store and no branch around a load: a load
        // under a branch whose value a shuffle consumes at once, or one that a dC image store (which may alias T) must
        // precede, waits out its own memory round trip.  Rows past the batch end and columns l >= L read in-range
        // addresses and are zeroed by selects.
        const int pool_lo = p.pool_lo[k], pool_hi = pool_lo + p.pool_n[k], hid = p.hid_n[k];
        const bool relu = p.act == DTB_ACT_RELU;
        int64_t tb[2], pb[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          tb[h] = row_ok[h] ? (gm0 + r0 + 8 * h) * L : 0;
          pb[h] = row_b[h] * p.P + p.pcol0[k] - pool_lo;
        }
        float gq[kWgMaxNP / 2];
#pragma unroll
        for (int q = 0; q < kWgMaxNP / 2; ++q) {
          const int h = (q >> 1) & 1, l = 8 * (q >> 2) + c2 + (q & 1);
          const bool ok = row_ok[h] && l < L, pooled = ok && l >= pool_lo && l < pool_hi;
          const float tv = __ldg(T + (ok ? tb[h] + l : 0));
          const float dp = __ldg(p.d_pooled + (pooled ? pb[h] + l : 0));
          float v = pooled ? 0.f + dp : 0.f;
          if (q < NPJ / 2) v = ok && l < hid ? v + dh[q] : v;
          gq[q] = ok && !(relu && !(tv > 0.f)) ? v : 0.f;
        }
        float bs[2] = {0.f, 0.f};
#pragma unroll
        for (int q = 0; q < kWgMaxNP / 2; q += 2) {
          const int row = r0 + (((q >> 1) & 1) << 3), l = 8 * (q >> 2) + c2;
          const float g[2] = {gq[q], gq[q + 1]};
          tc::split_bf16x2(g[0], g[1], ahi[q >> 3][(q >> 1) & 3], alo[q >> 3][(q >> 1) & 3]);
          // dC image: the lane of the partner row (lane ^ 4) swaps one value, so each lane holds rows (2t, 2t + 1) of
          // one column and stores their hi and lo pairs as one word each.  Only the stores are conditional: a branch
          // around the register work would make ptxas serialize the wgmma that follow.
          {
            const float other = __shfl_xor_sync(0xffffffffu, odd_row ? g[0] : g[1], 4);
            const float z0 = odd_row ? other : g[0], z1 = odd_row ? g[1] : other;
            const int mr = odd_row ? row - 1 : row, lc = odd_row ? l + 1 : l;
            uint32_t hi, lo;
            tc::split_bf16x2(z0, z1, hi, lo);
            const uint32_t off = ((mr >> 3) * (NPdc >> 3) + (lc >> 3)) * 128 + (lc & 7) * 16 + (mr & 7) * 2;
            if (l < NPdc) {
              *reinterpret_cast<uint32_t*>(img + off) = hi;
              *reinterpret_cast<uint32_t*>(img + dc_img + off) = lo;
            }
          }
          // d_bias: q and q + 2 are rows r0 and r0 + 8 of the same columns; then the sum over the 8 row lanes
          if (do_bias) {
            if ((q & 2) == 0) {
              bs[0] = g[0];
              bs[1] = g[1];
            } else {
#pragma unroll
              for (int u = 0; u < 2; ++u) {
                float v = bs[u] + g[u];
                v += __shfl_xor_sync(0xffffffffu, v, 4);
                v += __shfl_xor_sync(0xffffffffu, v, 8);
                v += __shfl_xor_sync(0xffffffffu, v, 16);
                if (lane < 4 && l + u < L && v != 0.f) atomicAdd(&bsum[k * kWgMaxNP + l + u], v);
              }
            }
          }
        }
      }
      // h_k in fragment order (columns j), and the fresh dh_k accumulators
      float hh[NPJ / 2];
      {
        const float* hsrc = k == 0 ? nullptr : p.saved + p.saved_off[k - 1];
        const int ldh = k == 0 ? F : p.L[k - 1];
#pragma unroll
        for (int q = 0; q < NPJ / 2; ++q) {
          const int row = r0 + (((q >> 1) & 1) << 3), j = 8 * (q >> 2) + c2 + (q & 1);
          const int64_t gm = gm0 + row;
          hh[q] = (j < H && gm < BD) ? (k == 0 ? x0s[row * F + j] : hsrc[gm * ldh + j]) : 0.f;
          dh[q] = 0.f;
        }
      }
      const int fpc = p.fpc[k], nch = p.nch[k];
      for (int t = 0; t < nch; ++t, ++chunk) {
        if (tid == 0) {
          int nk = k, nt = t + 1;
          bool more = true;
          if (nt == nch) {
            nt = 0;
            if (--nk < 0) { nk = K0; more = tile + (int)gridDim.x < n_tiles; }
          }
          if (more) issue(chunk + 1, nk, nt);
        }
        float acc[NPJ / 2];
#pragma unroll
        for (int q = 0; q < NPJ / 2; ++q) acc[q] = 0.f;
        tc::mbar_wait(&full[chunk & 1], (chunk >> 1) & 1);
        const uint32_t b_hi = tc::smem_u32(wbuf + (chunk & 1) * wbuf_bytes);
        const uint32_t b_lo = b_hi + (uint32_t)NPJ * LP * 2;
        tc::wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < kWgMaxNP / 16; ++ks) {
          if (ks * 16 < LP) {
            const uint64_t dh_desc = tc::make_smem_desc(b_hi + ks * 2 * lbo_b, lbo_b, 128);
            tc::Wgmma<NPJ>::rs(acc, ahi[ks], dh_desc, ks == 0 ? 0u : 1u);
            tc::Wgmma<NPJ>::rs(acc, alo[ks], dh_desc, 1u);
            tc::Wgmma<NPJ>::rs(acc, ahi[ks], tc::make_smem_desc(b_lo + ks * 2 * lbo_b, lbo_b, 128), 1u);
          }
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::wgmma_fence_acc(acc);
        // dx0[m, i] += sum_j dZ h ; dh[m, j] += dZ x0[m, i]
        if (fpc == 2) {
          // field 2t in columns [0, NPJ/2), field 2t + 1 in [NPJ/2, NPJ): acc[q] and acc[q + Q] are the same j of the
          // two fields, and hh / dh past Q are zero (H <= NPJ/2).  A missing field 2t + 1 (odd F) has zero weights.
          constexpr int Q = NPJ / 4;
          const int i0 = 2 * t;
          const bool two = i0 + 1 < F;
          const int i1 = two ? i0 + 1 : i0;
          const float x_a0 = x0s[r0 * F + i0], x_b0 = x0s[(r0 + 8) * F + i0];
          const float x_a1 = two ? x0s[r0 * F + i1] : 0.f, x_b1 = two ? x0s[(r0 + 8) * F + i1] : 0.f;
          float s_a0 = 0.f, s_b0 = 0.f, s_a1 = 0.f, s_b1 = 0.f;
#pragma unroll
          for (int q = 0; q < Q; ++q) {
            if ((q >> 1) & 1) {
              s_b0 += acc[q] * hh[q];
              s_b1 += acc[q + Q] * hh[q];
              dh[q] += acc[q] * x_b0;
              dh[q] += acc[q + Q] * x_b1;
            } else {
              s_a0 += acc[q] * hh[q];
              s_a1 += acc[q + Q] * hh[q];
              dh[q] += acc[q] * x_a0;
              dh[q] += acc[q + Q] * x_a1;
            }
          }
#pragma unroll
          for (int o = 1; o <= 2; o <<= 1) {
            s_a0 += __shfl_xor_sync(0xffffffffu, s_a0, o);
            s_b0 += __shfl_xor_sync(0xffffffffu, s_b0, o);
            s_a1 += __shfl_xor_sync(0xffffffffu, s_a1, o);
            s_b1 += __shfl_xor_sync(0xffffffffu, s_b1, o);
          }
          if ((lane & 3) == 0) {
            dxs[r0 * F + i0] += s_a0;
            dxs[(r0 + 8) * F + i0] += s_b0;
            if (two) {
              dxs[r0 * F + i1] += s_a1;
              dxs[(r0 + 8) * F + i1] += s_b1;
            }
          }
        } else {
          const int i = t;
          const float x_a = x0s[r0 * F + i], x_b = x0s[(r0 + 8) * F + i];
          float s_a = 0.f, s_b = 0.f;
#pragma unroll
          for (int q = 0; q < NPJ / 2; ++q) {
            if ((q >> 1) & 1) { s_b += acc[q] * hh[q]; dh[q] += acc[q] * x_b; }
            else              { s_a += acc[q] * hh[q]; dh[q] += acc[q] * x_a; }
          }
          s_a += __shfl_xor_sync(0xffffffffu, s_a, 1);
          s_a += __shfl_xor_sync(0xffffffffu, s_a, 2);
          s_b += __shfl_xor_sync(0xffffffffu, s_b, 1);
          s_b += __shfl_xor_sync(0xffffffffu, s_b, 2);
          if ((lane & 3) == 0) {
            dxs[r0 * F + i] += s_a;
            dxs[(r0 + 8) * F + i] += s_b;
          }
        }
        __syncthreads();
      }
    }
    // layer 0: h_0 is x0 itself, so dh_0 adds to dx0; then scatter into the table gradient
#pragma unroll
    for (int q = 0; q < NPJ / 2; ++q) {
      const int row = r0 + (((q >> 1) & 1) << 3), j = 8 * (q >> 2) + c2 + (q & 1);
      if (j < F) dxs[row * F + j] += dh[q];
    }
    __syncthreads();
    for (int e = tid; e < kWgRows * F; e += 128) {
      const int i = e / kWgRows, m = e - i * kWgRows;
      const int64_t gm = gm0 + m;
      if (gm < BD) {
        const int64_t b = gm / D;
        const int64_t rb = table_row(p.row_offsets, i, __ldg(p.idx + b * F + i), D, nullptr);
        if (rb >= 0) atomicAdd(p.grad_table + rb + (gm - b * D), dxs[m * F + i]);
      }
    }
    __syncthreads();
  }
  if (do_bias) {
    for (int e = tid; e < p.n_layers * kWgMaxNP; e += 128) {
      const int k = e / kWgMaxNP, l = e - k * kWgMaxNP;
      if (l < p.L[k] && bsum[e] != 0.f) atomicAdd(p.dbias + p.bias_off[k] + l, bsum[e]);
    }
  }
}

struct CinWgWgradParams {
  CUtensorMap hmap;      // htensor: T_{k-1} as a [B*D, ldh] fp32 tensor, box hpitch columns x 64 rows
  const float* x0t;      // [B*D, F]
  const float* h;        // T_{k-1} [B*D, ldh] (its first H columns are h_k); null for k = 0, where h_0 = x0
  const uint8_t* dc;     // dC_k images, one per 64-row block
  float* dw;             // dW_k [F*H, L]
  int64_t BD;
  int F, H, L, ldh;
  int fields_per_tile;   // 2: rows 0-31 of an A tile are field 2t, rows 32-63 field 2t + 1 (H <= 32); else 1
  int hpitch;            // floats between h rows in shared memory
  int htensor;           // 1: an h block arrives as one tensor copy of its first hpitch columns; 0: whole rows (ldh)
  int stages;            // depth of the ring of row blocks in shared memory (2 .. kWgradMaxStages)
  int groups;            // field groups of kWgradTiles A tiles; CTAs [0, (groups-1) splits) run the full ones
  int splits, blocks_per_split;            // row splits of each of the first groups - 1 field groups
  int last_splits, last_blocks_per_split;  // and of the last one
  int last_pair;         // 1: the last group has tiles for one warpgroup only; both run them, on alternate blocks
};

constexpr int kWgradTiles = 4;          // A tiles per CTA: two warpgroups x two m64 accumulators
constexpr int kWgradMaxStages = 4;
constexpr int kWgradThreads = 384;      // consumer warpgroups 0 and 1, producer warpgroup 2
// the registers the CTA gets at launch (384 x 168) are shared out again: 2 x 128 x 240 + 128 x 24 = 384 x 168
constexpr int kWgradConsumerRegs = 240, kWgradProducerRegs = 24;

struct CinWgWgradSmem {
  int x0_off, h_off, stage, bar_off, total;
};
__host__ __device__ inline CinWgWgradSmem cin_wg_wgrad_layout(int NP, int F, int hpitch, int stages) {
  CinWgWgradSmem l;
  l.x0_off = (int)cin_wg_dc_block_bytes(NP);
  l.h_off = l.x0_off + (kWgRows * F * 4 + 127) / 128 * 128;
  l.stage = l.h_off + (kWgRows * hpitch * 4 + 127) / 128 * 128;
  l.bar_off = stages * l.stage;
  l.total = l.bar_off + 2 * stages * 8;       // a full and an empty mbarrier per stage
  return l;
}
// as many stages as fit in shared memory, 2 to kWgradMaxStages
static int cin_wg_wgrad_stages(int NP, int F, int hpitch) {
  int s = kWgradMaxStages;
  while (s > 2 && cin_wg_wgrad_layout(NP, F, hpitch, s).total > 227 * 1024) --s;
  return s;
}

template <int NP>
__global__ void __launch_bounds__(kWgradThreads, 1) cin_wg_wgrad_kernel(const __grid_constant__ CinWgWgradParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int S = p.stages;
  const CinWgWgradSmem lay = cin_wg_wgrad_layout(NP, p.F, p.h ? p.hpitch : 0, S);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + lay.bar_off);
  uint64_t* empty = full + S;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, wq = warp & 3;
  const int F = p.F, H = p.H;
  // CTA -> field group g and row split y.  The full groups come first, split-major, so that the CTAs reading the same
  // rows run side by side; the last group has its own split count.
  const int nfull = p.groups - 1;
  int g, y, bps;
  if ((int)blockIdx.x < nfull * p.splits) {
    g = (int)blockIdx.x % nfull; y = (int)blockIdx.x / nfull; bps = p.blocks_per_split;
  } else {
    g = nfull; y = (int)blockIdx.x - nfull * p.splits; bps = p.last_blocks_per_split;
  }
  // pair: both warpgroups run the group's first two tiles, warpgroup w on the blocks n = w mod 2
  const bool pair = g == nfull && p.last_pair;
  // otherwise the first warpgroup always has a tile; the second may have none (last field group) and then leaves
  const bool wg1_on = pair || (g * kWgradTiles + 2) * p.fields_per_tile < F;
  const int64_t n_blocks = (p.BD + kWgRows - 1) / kWgRows;
  const int64_t blk0 = (int64_t)y * bps;
  int64_t blk1 = blk0 + bps;
  if (blk1 > n_blocks) blk1 = n_blocks;
  const int nb = blk1 > blk0 ? (int)(blk1 - blk0) : 0;

  if (tid == 0) {
    for (int i = 0; i < S; ++i) {
      tc::mbar_init(&full[i], 1);
      tc::mbar_init(&empty[i], wg1_on && !pair ? 2 : 1);      // one release per warpgroup that reads the block
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (wg == 2) {
    // producer: one thread brings block b into stage b % S (its dC image, its x0 rows and, k >= 1, its h rows) once
    // the readers of block b - S have released the stage
    tc::setmaxnreg_dec<kWgradProducerRegs>();
    if (tid == 2 * 128) {
      for (int b = 0; b < nb; ++b) {
        const int st = b % S;
        const int64_t gm0 = (blk0 + b) * kWgRows;
        const int rows = p.BD - gm0 < kWgRows ? (int)(p.BD - gm0) : kWgRows;      // a multiple of 4: D divides 64
        uint8_t* sb = smem + st * lay.stage;
        uint32_t bytes = cin_wg_dc_block_bytes(NP) + rows * F * 4;
        if (p.h) bytes += p.htensor ? kWgRows * p.hpitch * 4 : rows * p.ldh * 4;    // a tensor box always lands whole
        if (b >= S) tc::mbar_wait(&empty[st], (b / S - 1) & 1);
        tc::mbar_arrive_expect_tx(&full[st], bytes);
        tc::bulk_g2s(sb, p.dc + (blk0 + b) * cin_wg_dc_block_bytes(NP), cin_wg_dc_block_bytes(NP), &full[st]);
        tc::bulk_g2s(sb + lay.x0_off, p.x0t + gm0 * F, rows * F * 4, &full[st]);
        if (p.h) {
          if (p.htensor) tc::tma_load_2d(sb + lay.h_off, &p.hmap, 0, (int)gm0, &full[st]);
          else tc::bulk_g2s(sb + lay.h_off, p.h + gm0 * p.ldh, rows * p.ldh * 4, &full[st]);
        }
      }
    }
    return;
  }
  tc::setmaxnreg_inc<kWgradConsumerRegs>();
  if (wg == 1 && !wg1_on) return;

  // consumers: wait for full stages, build A, issue wgmma, release stages
  const int c2 = 2 * (lane & 3);
  constexpr uint32_t lbo_b = (NP >> 3) * 128;
  constexpr uint32_t img = NP * kWgRows * 2;
  // this warp's 16 A rows belong to one field of each of its warpgroup's two tiles; the thread's rows are jw, jw + 8
  const int upper = p.fields_per_tile == 2 && wq >= 2;
  const int jw = (wq - 2 * upper) * 16 + (lane >> 2);
  // h columns actually read: clamped into the copied rows, so that every shared-memory read stays inside its stage
  const int jc[2] = {min(jw, H - 1), min(jw + 8, H - 1)};
  int field[2];
  bool tile_on[2], row_ok[2][2];
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const int t = g * kWgradTiles + (pair ? 0 : wg * 2) + s;
    tile_on[s] = t * p.fields_per_tile < F;                         // warpgroup-uniform
    field[s] = t * p.fields_per_tile + upper;
    row_ok[s][0] = field[s] < F && jw < H;
    row_ok[s][1] = field[s] < F && jw + 8 < H;
    if (field[s] >= F) field[s] = 0;                                 // keeps the x0 reads in range
  }
  const int n0 = pair ? wg : 0, step = pair ? 2 : 1;
  // rows of the CTA's blocks, counted from its first block.  It fits an int: the dC images alone take 64 B per row
  // (NP >= 16), so no device holds 2^31 rows.
  const int rows_end = (int)((blk1 * kWgRows < p.BD ? blk1 * kWgRows : p.BD) - blk0 * kWgRows);

  float acc[2][NP / 2];
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int q = 0; q < NP / 2; ++q) acc[s][q] = 0.f;
  // one A fragment set: a warpgroup builds a tile while the other warpgroup's MMAs run
  uint32_t ahi[kWgRows / 16][4], alo[kWgRows / 16][4];
  for (int n = n0; n < nb; n += step) {
    const int st = n % S;
    const int rows = min(rows_end - n * kWgRows, kWgRows);
    const uint8_t* sb = smem + st * lay.stage;
    const float* xs = reinterpret_cast<const float*>(sb + lay.x0_off);          // [m][i]
    const float* hs = p.h ? reinterpret_cast<const float*>(sb + lay.h_off) : xs; // [m][j], pitch hp
    int hp = p.h ? p.hpitch : F, xp = F;
    // opaque per block: the row offsets below are recomputed each block instead of held in registers across the loop
    asm volatile("" : "+r"(hp), "+r"(xp));
    const uint32_t b_hi = tc::smem_u32(sb), b_lo = b_hi + img;
    tc::mbar_wait(&full[st], (n / S) & 1);
    // the thread's A elements are rows j = jw + 8r and columns m = 16 ks + 8 hb + c2 + e.  Each h[m, j] is read once
    // per block, each x0[m, field] once per tile; rows past the batch end and rows j >= H are zeroed by a select on
    // the product (the shared memory behind them may hold anything), so the reads are unconditional and in range.
    float hv[kWgRows / 16][2][2][2];
#pragma unroll
    for (int ks = 0; ks < kWgRows / 16; ++ks)
#pragma unroll
      for (int hb = 0; hb < 2; ++hb)
#pragma unroll
        for (int e = 0; e < 2; ++e)
#pragma unroll
          for (int r = 0; r < 2; ++r) hv[ks][hb][e][r] = hs[(ks * 16 + hb * 8 + c2 + e) * hp + jc[r]];
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      // the MMAs that read the A registers are done; before tile 0 this includes all of the warpgroup's previous
      // block's, whose stage is released (the producer may refill it with block n - step + S: step < S)
      tc::wgmma_wait<0>();
      if (s == 0 && n > n0 && wq == 0 && lane == 0) tc::mbar_arrive(&empty[(n - step) % S]);
      float xv[kWgRows / 16][2][2];
#pragma unroll
      for (int ks = 0; ks < kWgRows / 16; ++ks)
#pragma unroll
        for (int hb = 0; hb < 2; ++hb)
#pragma unroll
          for (int e = 0; e < 2; ++e) xv[ks][hb][e] = xs[(ks * 16 + hb * 8 + c2 + e) * xp + field[s]];
#pragma unroll
      for (int ks = 0; ks < kWgRows / 16; ++ks) {
#pragma unroll
        for (int hb = 0; hb < 2; ++hb) {
          const int m = ks * 16 + hb * 8 + c2;
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const float z0 = row_ok[s][r] && m < rows ? xv[ks][hb][0] * hv[ks][hb][0][r] : 0.f;
            const float z1 = row_ok[s][r] && m + 1 < rows ? xv[ks][hb][1] * hv[ks][hb][1][r] : 0.f;
            tc::split_bf16x2(z0, z1, ahi[ks][2 * hb + r], alo[ks][2 * hb + r]);
          }
        }
      }
      // an absent tile (past the last field) runs too, on zero rows, so that no wgmma sits in a branch
      tc::wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < kWgRows / 16; ++ks) {
        const uint64_t dhi = tc::make_smem_desc(b_hi + ks * 2 * lbo_b, lbo_b, 128);
        tc::Wgmma<NP>::rs(acc[s], ahi[ks], dhi, 1u);
        tc::Wgmma<NP>::rs(acc[s], alo[ks], dhi, 1u);
        tc::Wgmma<NP>::rs(acc[s], ahi[ks], tc::make_smem_desc(b_lo + ks * 2 * lbo_b, lbo_b, 128), 1u);
      }
      tc::wgmma_commit();
    }
  }
  tc::wgmma_wait<0>();
  tc::wgmma_fence_acc(acc[0]);
  tc::wgmma_fence_acc(acc[1]);
  // the thread's rows again, from a fresh read of its index: kept live through the loop they would not fit the
  // register budget at NP = 128
  int lane_e;
  asm volatile("mov.u32 %0, %%tid.x;" : "=r"(lane_e));
  const int wq_e = (lane_e >> 5) & 3;
  lane_e &= 31;
  const int jw_e = (wq_e - 2 * (p.fields_per_tile == 2 && wq_e >= 2)) * 16 + (lane_e >> 2);
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    if (!tile_on[s]) continue;
#pragma unroll
    for (int q = 0; q < NP / 2; ++q) {
      const int r = (q >> 1) & 1, j = jw_e + 8 * r, l = 8 * (q >> 2) + 2 * (lane_e & 3) + (q & 1);
      if (row_ok[s][r] && l < p.L && acc[s][q] != 0.f)
        atomicAdd(p.dw + ((int64_t)field[s] * H + j) * p.L + l, acc[s][q]);
    }
  }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
static int cin_wg_np(const CinShape& s) {
  int np = 16;
  while (np < s.Lmax) np *= 2;
  return np;
}

static int cin_wg_hp_max(const CinShape& s) {
  int hp = 16;
  for (int k = 0; k < s.n_layers; ++k) hp = round_up16(s.H[k]) > hp ? round_up16(s.H[k]) : hp;
  return hp;
}

bool cin_wg_supported(const CinShape& s) {
  if (!(s.D == 4 || s.D == 8 || s.D == 16 || s.D == 32)) return false;      // D divides the 64-row tile
  if (s.F < 1 || s.F > kWgMaxHp || s.Lmax > kWgMaxNP) return false;
  for (int k = 0; k < s.n_layers; ++k)
    if (round_up16(s.H[k]) > kWgMaxHp) return false;
  return cin_wg_fwd_stages(cin_wg_np(s), s.F, 0, cin_wg_hp_max(s)) >= 2;      // bf16x3 needs the most
}

size_t cin_wg_workspace_bytes(const CinShape& s) {
  const int np = cin_wg_np(s);
  size_t b = 0;
  for (int k = 0; k < s.n_layers; ++k) b += (size_t)s.F * cin_wg_chunk_bytes(np, round_up16(s.H[k]), 0);
  return b + 256;      // + the max|W_k| words of the fp16 variant
}

template <int NP, int kMode>
static int cin_wg_launch(const CinWgParams& p, cudaStream_t st) {
  const int smem = cin_wg_layout(NP, p.F, kMode, p.hp_max, p.stages).total;
  DTB_CUDA_OK(cudaFuncSetAttribute(cin_wg_fwd_kernel<NP, kMode>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  // setmaxnreg only redistributes the registers the CTA got at launch: a smaller allocation would block the consumers
  cudaFuncAttributes fa;
  DTB_CUDA_OK(cudaFuncGetAttributes(&fa, cin_wg_fwd_kernel<NP, kMode>));
  if (fa.numRegs * kFwdThreads < 2 * 128 * kFwdConsumerRegs + 128 * kFwdProducerRegs) {
    set_error("dtb_cin_fwd: the CIN forward kernel was built with too few registers for its warpgroup split");
    return DTB_ERR_CUDA;
  }
  const int n_pairs = (p.n_tiles + 1) / 2;
  const int grid = n_pairs < sm_count() ? n_pairs : sm_count();
  cin_wg_fwd_kernel<NP, kMode><<<grid, kFwdThreads, smem, st>>>(p);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

template <int kMode>
static int cin_wg_dispatch(const CinWgParams& p, int np, cudaStream_t st) {
  switch (np) {
    case 16: return cin_wg_launch<16, kMode>(p, st);
    case 32: return cin_wg_launch<32, kMode>(p, st);
    case 64: return cin_wg_launch<64, kMode>(p, st);
    default: return cin_wg_launch<128, kMode>(p, st);
  }
}

int cin_wg_fwd(const CinShape& s, const int32_t* idx, const float* table, const int64_t* row_offsets,
               const float* weights, const float* bias, float* pooled, void* saved, void* workspace,
               size_t workspace_bytes, int B, int act, int mode, int* status, cudaStream_t st) {
  if (workspace_bytes < cin_wg_workspace_bytes(s) || (reinterpret_cast<uintptr_t>(workspace) & 127)) {
    set_error("dtb_cin_fwd: workspace too small or not 128-byte aligned for the packed weights");
    return DTB_ERR_INVALID_ARG;
  }
  const int np = cin_wg_np(s);
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  int* wmax = reinterpret_cast<int*>(ws + cin_wg_workspace_bytes(s) - 256);
  CinWgParams p{};
  p.idx = idx; p.table = table; p.row_offsets = row_offsets; p.wpack = ws; p.bias = bias; p.pooled = pooled;
  p.saved = reinterpret_cast<float*>(saved); p.status = status; p.wmax = wmax;
  p.B = B; p.D = s.D; p.F = s.F; p.n_layers = s.n_layers; p.act = act; p.P = s.P;
  p.n_tiles = (int)(((int64_t)B * s.D + kWgRows - 1) / kWgRows);
  p.hp_max = cin_wg_hp_max(s); p.stages = cin_wg_fwd_stages(np, s.F, mode, p.hp_max);
  if (mode == 2) DTB_CUDA_OK(cudaMemsetAsync(wmax, 0, sizeof(int) * kCinMaxLayers, st));
  size_t woff = 0, soff = (size_t)B * s.D * s.F;
  for (int k = 0; k < s.n_layers; ++k) {
    p.L[k] = s.L[k]; p.Hp[k] = round_up16(s.H[k]); p.hid_n[k] = k + 1 < s.n_layers ? s.H[k + 1] : 0;
    p.pool_lo[k] = s.pool_lo[k]; p.pool_n[k] = s.pool_n[k]; p.pcol0[k] = s.pcol0[k];
    p.wpack_off[k] = woff; p.saved_off[k] = soff; p.bias_off[k] = s.b_off[k];
    const int64_t n_w = (int64_t)s.F * s.H[k] * s.L[k];
    if (mode == 2) {
      cin_wg_wmax_kernel<<<(int)((n_w + 255) / 256 < 64 ? (n_w + 255) / 256 : 64), 256, 0, st>>>(weights + s.w_off[k], n_w,
                                                                                                 wmax + k);
      DTB_LAUNCH_OK();
    }
    const int64_t total = (int64_t)s.F * np * p.Hp[k];
    int blocks = (int)((total + 255) / 256);
    if (blocks > sm_count() * 8) blocks = sm_count() * 8;
    cin_wg_pack_kernel<<<blocks, 256, 0, st>>>(weights + s.w_off[k], ws + woff, s.F, s.H[k], p.Hp[k], s.L[k], np, mode,
                                               wmax + k);
    DTB_LAUNCH_OK();
    woff += (size_t)s.F * cin_wg_chunk_bytes(np, p.Hp[k], mode);
    soff += (size_t)B * s.D * s.L[k];
  }
  switch (mode) {
    case 0: return cin_wg_dispatch<0>(p, np, st);
    case 1: return cin_wg_dispatch<1>(p, np, st);
    default: return cin_wg_dispatch<2>(p, np, st);
  }
}

static int cin_wg_npj(const CinShape& s) {
  int hp = 16;
  for (int k = 0; k < s.n_layers; ++k) hp = round_up16(s.H[k]) > hp ? round_up16(s.H[k]) : hp;
  int np = 16;
  while (np < hp) np *= 2;
  return np;
}
// x0 fields per W_k^T chunk of the data gradient: two when both fit in the NPJ columns
static int cin_wg_dgrad_fpc(const CinShape& s, int k) { return 2 * s.H[k] <= cin_wg_npj(s) ? 2 : 1; }
static size_t cin_wg_pack_t_bytes(const CinShape& s) {
  size_t b = 0;
  for (int k = 0; k < s.n_layers; ++k) {
    const int fpc = cin_wg_dgrad_fpc(s, k);
    b += (size_t)((s.F + fpc - 1) / fpc) * cin_wg_npj(s) * round_up16(s.L[k]) * 4;
  }
  return (b + 255) / 256 * 256;
}
// dC_k images of every layer: whole 64-row blocks of cin_wg_np columns (4 bytes per element, hi + lo)
static size_t cin_wg_dc_layer_bytes(const CinShape& s, int B) {
  return (size_t)(((int64_t)B * s.D + kWgRows - 1) / kWgRows) * cin_wg_dc_block_bytes(cin_wg_np(s));
}
size_t cin_wg_bwd_workspace_bytes(const CinShape& s, int B) {
  return cin_wg_pack_t_bytes(s) + s.n_layers * cin_wg_dc_layer_bytes(s, B);
}

template <int NPJ>
static int cin_wg_dgrad_launch(const CinWgBwdParams& p, cudaStream_t st) {
  const CinWgBwdSmem lay = cin_wg_bwd_layout(NPJ, p.F);
  DTB_CUDA_OK(cudaFuncSetAttribute(cin_wg_dgrad_kernel<NPJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, lay.total));
  const int64_t n_tiles = ((int64_t)p.B * p.D + kWgRows - 1) / kWgRows;
  int per_sm = (227 * 1024) / (lay.total + 1024);
  per_sm = per_sm < 1 ? 1 : (per_sm > 4 ? 4 : per_sm);
  int64_t grid = (int64_t)sm_count() * per_sm;
  if (grid > n_tiles) grid = n_tiles;
  cin_wg_dgrad_kernel<NPJ><<<(int)grid, 128, lay.total, st>>>(p);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

template <int NP>
static int cin_wg_wgrad_launch(const CinWgWgradParams& p, int n_ctas, cudaStream_t st) {
  const int smem = cin_wg_wgrad_layout(NP, p.F, p.h ? p.hpitch : 0, p.stages).total;
  DTB_CUDA_OK(cudaFuncSetAttribute(cin_wg_wgrad_kernel<NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  // setmaxnreg only redistributes the registers the CTA got at launch: a smaller allocation would block the consumers
  cudaFuncAttributes fa;
  DTB_CUDA_OK(cudaFuncGetAttributes(&fa, cin_wg_wgrad_kernel<NP>));
  if (fa.numRegs * kWgradThreads < 2 * 128 * kWgradConsumerRegs + 128 * kWgradProducerRegs) {
    set_error("dtb_cin_bwd: the CIN weight-gradient kernel was built with too few registers for its warpgroup split");
    return DTB_ERR_CUDA;
  }
  cin_wg_wgrad_kernel<NP><<<n_ctas, kWgradThreads, smem, st>>>(p);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

// cuTensorMapEncodeTiled from the driver the runtime already loaded (no link against libcuda)
static PFN_cuTensorMapEncodeTiled_v12000 cin_wg_tmap_encoder() {
  static const PFN_cuTensorMapEncodeTiled_v12000 fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &f, 12000, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      f = nullptr;
    return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(f);
  }();
  return fn;
}

// row splits of the weight gradient's field groups.  A full group's CTA costs 1 per row block.  With last_pair the
// last group's CTA runs two blocks at a time, so it costs 1/2 per block and gets the SMs the full groups leave over.
static void cin_wg_wgrad_grid(CinWgWgradParams& w, int64_t n_blocks, int sms) {
  auto fit = [&](int64_t splits, int& s, int& bps) {      // at most n_blocks splits, none of them empty
    splits = splits < 1 ? 1 : (splits > n_blocks ? n_blocks : splits);
    bps = (int)((n_blocks + splits - 1) / splits);
    s = (int)((n_blocks + bps - 1) / bps);
  };
  const int nfull = w.groups - 1;
  if (!w.last_pair) {
    fit(sms / w.groups, w.splits, w.blocks_per_split);
    w.last_splits = w.splits; w.last_blocks_per_split = w.blocks_per_split;
    return;
  }
  if (nfull == 0) {
    w.splits = w.blocks_per_split = 0;
    fit(sms, w.last_splits, w.last_blocks_per_split);
    return;
  }
  int64_t best = -1;
  for (int sf = 1; sf * nfull < sms; ++sf) {
    int s, bps, sl, bpsl;
    fit(sf, s, bps);
    fit(sms - sf * nfull, sl, bpsl);
    const int64_t cost = bps > (bpsl + 1) / 2 ? bps : (bpsl + 1) / 2;
    if (best < 0 || cost < best) {
      best = cost;
      w.splits = s; w.blocks_per_split = bps; w.last_splits = sl; w.last_blocks_per_split = bpsl;
    }
  }
}

int cin_wg_bwd(const CinShape& s, const int32_t* idx, const int64_t* row_offsets, const float* weights,
               const float* d_pooled, const void* saved, float* grad_table, float* d_weights, float* d_bias,
               void* workspace, size_t workspace_bytes, int B, int act, int phase, cudaStream_t st) {
  if (workspace_bytes < cin_wg_bwd_workspace_bytes(s, B) || (reinterpret_cast<uintptr_t>(workspace) & 127)) {
    set_error("dtb_cin_bwd: workspace too small or not 128-byte aligned");
    return DTB_ERR_INVALID_ARG;
  }
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  uint8_t* dc = ws + cin_wg_pack_t_bytes(s);
  const float* sv = reinterpret_cast<const float*>(saved);
  const int npj = cin_wg_npj(s), np = cin_wg_np(s);
  size_t dc_off[kCinMaxLayers], saved_off[kCinMaxLayers];
  {
    size_t o = (size_t)B * s.D * s.F;
    for (int k = 0; k < s.n_layers; ++k) {
      dc_off[k] = k * cin_wg_dc_layer_bytes(s, B); saved_off[k] = o;
      o += (size_t)B * s.D * s.L[k];
    }
  }
  if (phase != 2) {
    CinWgBwdParams p{};
    p.idx = idx; p.row_offsets = row_offsets; p.wpack = ws; p.d_pooled = d_pooled; p.saved = sv;
    p.grad_table = grad_table; p.dc = dc; p.dbias = d_bias;
    p.B = B; p.D = s.D; p.F = s.F; p.n_layers = s.n_layers; p.act = act; p.P = s.P; p.NPdc = np;
    size_t woff = 0;
    for (int k = 0; k < s.n_layers; ++k) {
      p.L[k] = s.L[k]; p.LP[k] = round_up16(s.L[k]); p.H[k] = s.H[k]; p.hid_n[k] = k + 1 < s.n_layers ? s.H[k + 1] : 0;
      p.fpc[k] = cin_wg_dgrad_fpc(s, k); p.nch[k] = (s.F + p.fpc[k] - 1) / p.fpc[k];
      p.pool_lo[k] = s.pool_lo[k]; p.pool_n[k] = s.pool_n[k]; p.pcol0[k] = s.pcol0[k];
      p.wpack_off[k] = woff; p.saved_off[k] = saved_off[k]; p.dc_off[k] = dc_off[k]; p.bias_off[k] = s.b_off[k];
      const int64_t total = (int64_t)p.nch[k] * npj * p.LP[k];
      int blocks = (int)((total + 255) / 256);
      if (blocks > sm_count() * 8) blocks = sm_count() * 8;
      cin_wg_pack_t_kernel<<<blocks, 256, 0, st>>>(weights + s.w_off[k], ws + woff, s.F, s.H[k], s.L[k], p.LP[k], npj,
                                                   p.fpc[k]);
      DTB_LAUNCH_OK();
      woff += (size_t)p.nch[k] * npj * p.LP[k] * 4;
    }
    int rc;
    switch (npj) {
      case 16: rc = cin_wg_dgrad_launch<16>(p, st); break;
      case 32: rc = cin_wg_dgrad_launch<32>(p, st); break;
      default: rc = cin_wg_dgrad_launch<64>(p, st); break;
    }
    if (rc != DTB_OK) return rc;
  }
  if (phase != 1) {
    const int64_t BD = (int64_t)B * s.D;
    const int64_t n_blocks = (BD + kWgRows - 1) / kWgRows;
    for (int k = 0; k < s.n_layers; ++k) {
      CinWgWgradParams w{};
      w.x0t = sv; w.h = k == 0 ? nullptr : sv + saved_off[k - 1]; w.ldh = k == 0 ? s.F : s.L[k - 1];
      w.dc = dc + dc_off[k]; w.dw = d_weights + s.w_off[k];
      w.BD = BD; w.F = s.F; w.H = s.H[k]; w.L = s.L[k];
      w.fields_per_tile = s.H[k] <= 32 ? 2 : 1;
      // T_{k-1} is a tensor with 16-byte row strides when ldh % 4 == 0: one tensor copy per block brings the first
      // hpitch >= H columns of its 64 rows, landing at a pitch that makes the A-fragment reads free of bank conflicts
      // (pitch % 16 in {4, 12}); otherwise one bulk copy brings the whole rows
      w.htensor = k > 0 && w.ldh % 4 == 0 && BD <= INT32_MAX;
      if (w.htensor) {
        const int h4 = (s.H[k] + 3) / 4 * 4;
        w.hpitch = h4 + (20 - h4 % 16) % 16;
        PFN_cuTensorMapEncodeTiled_v12000 encode = cin_wg_tmap_encoder();
        const cuuint64_t dims[2] = {(cuuint64_t)w.ldh, (cuuint64_t)BD};
        const cuuint64_t strides[1] = {(cuuint64_t)w.ldh * sizeof(float)};
        const cuuint32_t box[2] = {(cuuint32_t)w.hpitch, (cuuint32_t)kWgRows}, estrides[2] = {1, 1};
        if (!encode || encode(&w.hmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(w.h), dims, strides, box,
                              estrides, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
          set_error("dtb_cin_bwd: cannot encode the tensor map of the CIN weight gradient's h rows");
          return DTB_ERR_CUDA;
        }
      } else {
        w.hpitch = w.ldh;
      }
      w.stages = cin_wg_wgrad_stages(np, s.F, w.h ? w.hpitch : 0);
      const int a_tiles = (s.F + w.fields_per_tile - 1) / w.fields_per_tile;
      w.groups = (a_tiles + kWgradTiles - 1) / kWgradTiles;
      // a last group with tiles for one warpgroup shares them between both; a warpgroup keeps up to two blocks of
      // the ring until it releases the older one, so the other needs at least one more stage
      w.last_pair = a_tiles - (w.groups - 1) * kWgradTiles <= 2 && w.stages >= 3;
      cin_wg_wgrad_grid(w, n_blocks, sm_count());
      const int ctas = (w.groups - 1) * w.splits + w.last_splits;
      int rc;
      switch (np) {
        case 16: rc = cin_wg_wgrad_launch<16>(w, ctas, st); break;
        case 32: rc = cin_wg_wgrad_launch<32>(w, ctas, st); break;
        case 64: rc = cin_wg_wgrad_launch<64>(w, ctas, st); break;
        default: rc = cin_wg_wgrad_launch<128>(w, ctas, st); break;
      }
      if (rc != DTB_OK) return rc;
    }
  }
  return DTB_OK;
}

}  // namespace dtb
