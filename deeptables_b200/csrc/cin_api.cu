// C-ABI entry points for CIN: shape validation and dispatch between the fused tensor-core forward (cin_wgmma.cu) and the
// any-shape formulation (cin_fp32.cu: outer product in bounded chunks of batch rows, GEMMs on the wgmma kernels of
// dense_tc.cu), and likewise between the two backwards.  Both forwards save the same activations.
#include "dtb_common.cuh"
#include "cin_shapes.h"
#include "cin_impl.h"

using namespace dtb;

static bool is_fused_tc(int precision) {
  return precision == DTB_CIN_TC_BF16X3 || precision == DTB_CIN_TC_BF16X1 || precision == DTB_CIN_TC_F16X1;
}

// auto: the fp32-grade bf16x3 fused forward where the shape fits it, else the any-shape formulation
static int resolve_precision(const CinShape& s, int precision) {
  if (precision != DTB_CIN_AUTO) return precision;
  return cin_wg_supported(s) ? DTB_CIN_TC_BF16X3 : DTB_CIN_FP32;
}

extern "C" {

int dtb_cin_tc_supported(int F, int D, const int* layer_sizes_host, int n_layers, int direct) {
  CinShape s;
  if (!s.init(F, D, layer_sizes_host, n_layers, direct)) return 0;
  return cin_wg_supported(s) ? 1 : 0;
}

int dtb_cin_resolved_precision(int F, int D, const int* layer_sizes_host, int n_layers, int direct, int precision) {
  CinShape s;
  if (!s.init(F, D, layer_sizes_host, n_layers, direct)) return DTB_ERR_INVALID_ARG;
  return resolve_precision(s, precision);
}

size_t dtb_cin_saved_bytes(int B, int F, int D, const int* layer_sizes_host, int n_layers, int direct) {
  CinShape s;
  if (!s.init(F, D, layer_sizes_host, n_layers, direct) || B <= 0) return 0;
  return cin_fp32_saved_bytes(s, B);
}

size_t dtb_cin_workspace_bytes(int B, int F, int D, const int* layer_sizes_host, int n_layers, int direct,
                               int training) {
  CinShape s;
  if (!s.init(F, D, layer_sizes_host, n_layers, direct) || B <= 0) return 0;
  const size_t a = cin_fp32_workspace_bytes(s, B, training);
  size_t b = 0;
  if (cin_wg_supported(s)) {
    b = cin_wg_workspace_bytes(s);
    const size_t c = training ? cin_wg_bwd_workspace_bytes(s, B) : 0;
    b = b > c ? b : c;
  }
  return a > b ? a : b;
}

int dtb_cin_fwd(const int32_t* idx, const float* table, const int64_t* row_offsets, const float* weights,
                const float* bias, float* pooled, void* saved, void* workspace, size_t workspace_bytes, int B,
                int F, int D, const int* layer_sizes_host, int n_layers, int direct, int act, int precision,
                int* status, void* stream) {
  DTB_CHECK_ARG(idx && table && row_offsets && weights && pooled && workspace, "NULL argument");
  DTB_CHECK_ARG(act == DTB_ACT_NONE || act == DTB_ACT_RELU, "unsupported activation");
  DTB_CHECK_ARG(precision >= 0 && precision <= DTB_CIN_TC_F16X1, "bad precision code");
  CinShape s;
  if (!s.init(F, D, layer_sizes_host, n_layers, direct)) {
    set_error("dtb_cin_fwd: invalid CIN configuration (cross_layer_size must be even except for the last "
              "layer when direct=False; 1..%d layers)", kCinMaxLayers);
    return DTB_ERR_INVALID_ARG;
  }
  if (B <= 0) return DTB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  precision = resolve_precision(s, precision);
  if (is_fused_tc(precision)) {
    if (!cin_wg_supported(s)) {
      set_error("dtb_cin_fwd: tensor-core path requested but shape unsupported (F=%d D=%d)", F, D);
      return DTB_ERR_UNSUPPORTED;
    }
    return cin_wg_fwd(s, idx, table, row_offsets, weights, bias, pooled, saved, workspace, workspace_bytes, B, act,
                      precision - DTB_CIN_TC_BF16X3, status, st);
  }
  return cin_fp32_fwd(s, idx, table, row_offsets, weights, bias, pooled, saved, workspace, workspace_bytes, B,
                      act, status, st);
}

static int cin_bwd_impl(const int32_t* idx, const float* table, const int64_t* row_offsets, const float* weights,
                        const float* d_pooled, const void* saved, float* grad_table, float* d_weights, float* d_bias,
                        void* workspace, size_t workspace_bytes, int B, int F, int D, const int* layer_sizes_host,
                        int n_layers, int direct, int act, int precision, int phase, void* stream) {
  DTB_CHECK_ARG(idx && table && row_offsets && weights && d_pooled && saved && grad_table && d_weights &&
                    workspace,
                "NULL argument");
  DTB_CHECK_ARG(act == DTB_ACT_NONE || act == DTB_ACT_RELU, "unsupported activation");
  DTB_CHECK_ARG(precision >= 0 && precision <= DTB_CIN_TC_F16X1, "bad precision code");
  CinShape s;
  if (!s.init(F, D, layer_sizes_host, n_layers, direct)) {
    set_error("dtb_cin_bwd: invalid CIN configuration");
    return DTB_ERR_INVALID_ARG;
  }
  if (B <= 0) return DTB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  precision = resolve_precision(s, precision);
  if (is_fused_tc(precision)) {
    if (!cin_wg_supported(s)) {
      set_error("dtb_cin_bwd: tensor-core path requested but shape unsupported (F=%d D=%d)", F, D);
      return DTB_ERR_UNSUPPORTED;
    }
    return cin_wg_bwd(s, idx, row_offsets, weights, d_pooled, saved, grad_table, d_weights, d_bias, workspace,
                      workspace_bytes, B, act, phase, st);
  }
  return cin_fp32_bwd(s, idx, table, row_offsets, weights, d_pooled, saved, grad_table, d_weights, d_bias,
                      workspace, workspace_bytes, B, act, phase, st);
}

int dtb_cin_bwd(const int32_t* idx, const float* table, const int64_t* row_offsets, const float* weights,
                const float* d_pooled, const void* saved, float* grad_table, float* d_weights, float* d_bias,
                void* workspace, size_t workspace_bytes, int B, int F, int D, const int* layer_sizes_host,
                int n_layers, int direct, int act, int precision, void* stream) {
  return cin_bwd_impl(idx, table, row_offsets, weights, d_pooled, saved, grad_table, d_weights, d_bias, workspace,
                      workspace_bytes, B, F, D, layer_sizes_host, n_layers, direct, act, precision, 0, stream);
}

int dtb_cin_bwd_phase(const int32_t* idx, const float* table, const int64_t* row_offsets, const float* weights,
                      const float* d_pooled, const void* saved, float* grad_table, float* d_weights, float* d_bias,
                      void* workspace, size_t workspace_bytes, int B, int F, int D, const int* layer_sizes_host,
                      int n_layers, int direct, int act, int precision, int phase, void* stream) {
  DTB_CHECK_ARG(phase == 1 || phase == 2, "phase must be 1 (embedding gradient) or 2 (weight gradient)");
  return cin_bwd_impl(idx, table, row_offsets, weights, d_pooled, saved, grad_table, d_weights, d_bias, workspace,
                      workspace_bytes, B, F, D, layer_sizes_host, n_layers, direct, act, precision, phase, stream);
}

}  // extern "C"
