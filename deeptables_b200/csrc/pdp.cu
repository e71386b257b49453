// Partial dependence and ICE (deeptables_b200/utils/partial_dependence.py): the weighted sums of the model outputs of
// each grid point over fixed blocks of X rows.
//
// Row k*rows_per_group + j of prob is X row j (of the chunk) with the feature columns taken from grid point k.  Each
// (grid point, block of block_rows rows, output column) gets one float64 sum of w[j] * p, in a fixed order: one warp per
// sum, lane l adding rows l, l+32, ... of the block in order, then a fixed butterfly.  A block's sum depends only on the
// rows in it, so the host, adding each grid point's blocks in index order, gets the same bits whichever way the rows
// were cut into chunks, as long as every chunk starts on a block boundary.
#include "dtb_common.cuh"

namespace dtb {

constexpr int kPdpThreads = 256;

__global__ void __launch_bounds__(kPdpThreads) pdp_block_sums_kernel(const float* __restrict__ prob,
                                                                     const double* __restrict__ weight,
                                                                     int64_t groups, int rows_per_group, int cols,
                                                                     int block_rows, double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int blocks = (rows_per_group + block_rows - 1) / block_rows;
  const int64_t items = groups * blocks * cols;
  const int64_t warps = (int64_t)gridDim.x * (kPdpThreads / 32);
  for (int64_t it = blockIdx.x * (int64_t)(kPdpThreads / 32) + (threadIdx.x >> 5); it < items; it += warps) {
    const int c = (int)(it % cols);
    const int64_t gb = it / cols;
    const int b = (int)(gb % blocks);
    const int64_t g = gb / blocks;
    const int lo = b * block_rows;
    const int hi = min(lo + block_rows, rows_per_group);
    const float* pg = prob + (g * rows_per_group) * cols + c;
    double acc = 0.0;
    if (weight) {
      // w * p rounded before the add (no fused multiply-add), so the host can restate the order
      for (int j = lo + lane; j < hi; j += 32) acc = __dadd_rn(acc, __dmul_rn(weight[j], (double)pg[(int64_t)j * cols]));
    } else {
      for (int j = lo + lane; j < hi; j += 32) acc += (double)pg[(int64_t)j * cols];
    }
    acc = warp_sum(acc);
    if (lane == 0) out[it] = acc;
  }
}

static inline int pdp_grid(int64_t threads) {
  const int64_t cap = (int64_t)sm_count() * 16;
  const int64_t blocks = (threads + kPdpThreads - 1) / kPdpThreads;
  return (int)(blocks < 1 ? 1 : blocks > cap ? cap : blocks);
}

}  // namespace dtb

using namespace dtb;

extern "C" {

int dtb_pdp_block_sums(const float* prob, const double* weight, int64_t groups, int rows_per_group, int cols,
                       int block_rows, double* out, void* stream) {
  DTB_CHECK_ARG(prob && out, "NULL prob or out");
  DTB_CHECK_ARG(groups > 0 && rows_per_group > 0 && cols > 0 && block_rows > 0, "bad shape");
  const int64_t blocks = (rows_per_group + (int64_t)block_rows - 1) / block_rows;
  DTB_CHECK_ARG(groups <= INT64_MAX / 32 / blocks / cols, "too many sums");
  pdp_block_sums_kernel<<<pdp_grid(groups * blocks * cols * 32), kPdpThreads, 0, (cudaStream_t)stream>>>(
      prob, weight, groups, rows_per_group, cols, block_rows, out);
  DTB_LAUNCH_OK();
  return DTB_OK;
}

}  // extern "C"
