// Internal interface between cin_api.cu and the two CIN forward implementations (one backward serves both).
#pragma once
#include <cuda_runtime.h>
#include "cin_shapes.h"

namespace dtb {

size_t cin_fp32_saved_bytes(const CinShape& s, int B);
size_t cin_fp32_workspace_bytes(const CinShape& s, int B, int training);
int cin_fp32_fwd(const CinShape& s, const int32_t* idx, const float* table, const int64_t* row_offsets,
                 const float* weights, const float* bias, float* pooled, void* saved, void* workspace,
                 size_t workspace_bytes, int B, int act, int* status, cudaStream_t st);
int cin_fp32_bwd(const CinShape& s, const int32_t* idx, const float* table, const int64_t* row_offsets,
                 const float* weights, const float* d_pooled, const void* saved, float* grad_table,
                 float* d_weights, float* d_bias, void* workspace, size_t workspace_bytes, int B, int act,
                 int phase, cudaStream_t st);

// fused tensor-core forward (cin_wgmma.cu); mode 0 = bf16x3, 1 = one bf16 pass, 2 = one scaled fp16 pass.  Its saved
// activations have the layout of cin_fp32_fwd's, so either backward reads either forward's activations.
bool cin_wg_supported(const CinShape& s);
size_t cin_wg_workspace_bytes(const CinShape& s);
int cin_wg_fwd(const CinShape& s, const int32_t* idx, const float* table, const int64_t* row_offsets,
               const float* weights, const float* bias, float* pooled, void* saved, void* workspace,
               size_t workspace_bytes, int B, int act, int mode, int* status, cudaStream_t st);
// fused backward, bf16x3 (phase 1: embedding gradient + dC_k; 2: weight and bias gradients; 0: both)
size_t cin_wg_bwd_workspace_bytes(const CinShape& s, int B);
int cin_wg_bwd(const CinShape& s, const int32_t* idx, const int64_t* row_offsets, const float* weights,
               const float* d_pooled, const void* saved, float* grad_table, float* d_weights, float* d_bias,
               void* workspace, size_t workspace_bytes, int B, int act, int phase, cudaStream_t st);

}  // namespace dtb
