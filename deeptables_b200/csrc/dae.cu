// Training batches of the denoising auto-encoder (deeptables_b200/dae.py, fe/dae.py) with swap noise built on the device.
//
// Row i of a batch is the clean row X[p1[base + i]].  Its noisy copy takes k of its columns from the donor row
// X[p2[base + i]]: the k columns c with the smallest 64-bit keys (h(c) << 32) | c, where h is the counter hash of
// include/deeptables_b200.h (dtb_dae_swap_batch).  The keys are unique, so the choice is well defined and every k-subset
// is equally likely.  Nothing is stored per column: one warp per row finds the k-th smallest hash by a 4-pass radix
// select over the recomputed hashes (8 bits per pass, a 256-bin histogram per warp in shared memory), then writes the
// row, columns fastest, so the reads of X and the writes of both outputs are coalesced along the columns.  Columns whose
// hash equals the k-th smallest are taken in ascending column order, counted with ballots in the write loop, which is
// the order their keys give.  Any column count works; the work per row is 5 passes over its columns.
#include "dtb_common.cuh"

namespace dtb {

constexpr int kDaeWarps = 8;

__global__ void __launch_bounds__(kDaeWarps * 32) dae_swap_batch_kernel(
    const float* __restrict__ X, int cols, const int64_t* __restrict__ p1, const int64_t* __restrict__ p2,
    const int* __restrict__ step_dev, const int* __restrict__ epoch_first_step_dev, int batch_rows, int rows, int k,
    uint32_t seed, float* __restrict__ x_in, float* __restrict__ x_tgt) {
  __shared__ int hist[kDaeWarps][256];
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int step = *step_dev;
  const int64_t base = (int64_t)(step - *epoch_first_step_dev) * batch_rows;
  const uint64_t a = mix32(((uint64_t)seed << 32) | (uint32_t)(step + 1));
  for (int i = blockIdx.x * kDaeWarps + w; i < rows; i += gridDim.x * kDaeWarps) {   // warp-uniform
    const float* src = X + p1[base + i] * (int64_t)cols;
    float* tgt = x_tgt + (int64_t)i * cols;
    if (k == 0) {
      for (int c = lane; c < cols; c += 32) {
        const float t = src[c];
        tgt[c] = t;
        if (x_in) x_in[(int64_t)i * cols + c] = t;
      }
      continue;
    }
    const float* donor = X + p2[base + i] * (int64_t)cols;
    float* in = x_in + (int64_t)i * cols;
    const uint64_t b = (uint64_t)mix32((a << 32) | (uint32_t)i) << 32;    // h(c) = mix32(b | c)
    uint32_t prefix = 0;    // after the passes: the k-th smallest hash T
    int need = k;           // after the passes: how many columns with h == T are taken
    if (k < cols) {
      for (int shift = 24; shift >= 0; shift -= 8) {
        for (int d = lane; d < 256; d += 32) hist[w][d] = 0;
        __syncwarp();
        for (int c = lane; c < cols; c += 32) {
          const uint32_t h = mix32(b | (uint32_t)c);
          if (((uint64_t)(h ^ prefix) >> (shift + 8)) == 0) atomicAdd(&hist[w][(h >> shift) & 255u], 1);
        }
        __syncwarp();
        int cnt[8], tot = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          cnt[j] = hist[w][lane * 8 + j];
          tot += cnt[j];
        }
        int inc = tot;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int v = __shfl_up_sync(full, inc, o);
          if (lane >= o) inc += v;
        }
        const int exc = inc - tot;
        const int owner = __ffs(__ballot_sync(full, exc < need && inc >= need)) - 1;   // the lane holding the digit
        int digit = 0, below = exc;
        if (lane == owner) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            if (below + cnt[j] >= need) {
              digit = lane * 8 + j;
              break;
            }
            below += cnt[j];
          }
        }
        digit = __shfl_sync(full, digit, owner);
        below = __shfl_sync(full, below, owner);
        need -= below;
        prefix |= (uint32_t)digit << shift;
        __syncwarp();           // every lane has read the histogram before the next pass clears it
      }
    }
    int ties = 0;               // columns with h == T before this chunk
    for (int c0 = 0; c0 < cols; c0 += 32) {
      const int c = c0 + lane;
      bool swap = true;         // k == cols: the donor row whole
      if (k < cols) {
        const uint32_t h = c < cols ? mix32(b | (uint32_t)c) : 0u;
        const bool tie = c < cols && h == prefix;
        const unsigned tb = __ballot_sync(full, tie);
        swap = h < prefix || (tie && ties + __popc(tb & ((1u << lane) - 1u)) < need);
        ties += __popc(tb);
      }
      if (c < cols) {
        const float t = src[c];
        tgt[c] = t;
        in[c] = swap ? donor[c] : t;
      }
    }
  }
}

}  // namespace dtb

using namespace dtb;

extern "C" {

int dtb_dae_swap_batch(const float* X, int cols, const int64_t* p1, const int64_t* p2, const int* step_dev,
                       const int* epoch_first_step_dev, int batch_rows, int rows, int k, unsigned long long seed,
                       float* x_in, float* x_tgt, void* stream) {
  DTB_CHECK_ARG(X && p1 && step_dev && epoch_first_step_dev && x_tgt, "NULL argument");
  DTB_CHECK_ARG(cols > 0 && rows >= 0 && rows <= batch_rows && k >= 0 && k <= cols, "bad shape");
  DTB_CHECK_ARG((k == 0) == (p2 == nullptr) && (k == 0 || x_in), "p2 and x_in are needed exactly when k > 0");
  DTB_CHECK_ARG(seed < (1ull << 32), "seed must be below 2^32");
  if (rows == 0) return DTB_OK;
  const int64_t blocks = (rows + kDaeWarps - 1) / kDaeWarps;
  const int64_t cap = (int64_t)sm_count() * 16;
  dae_swap_batch_kernel<<<(unsigned)(blocks < cap ? blocks : cap), kDaeWarps * 32, 0, (cudaStream_t)stream>>>(
      X, cols, p1, p2, step_dev, epoch_first_step_dev, batch_rows, rows, k, (uint32_t)seed, x_in, x_tgt);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

}  // extern "C"
