/*
 * deeptables_b200 -- C ABI of the H100-native (sm_90a) feature-interaction engine.
 *
 * The reference (DataCanvasIO/DeepTables) has no native boundary at all: every op below is, in
 * the reference, a chain of TensorFlow/Keras ops inside a Keras layer (file:line cited per
 * entry point, relative to /root/reference).  This header is therefore the boundary a
 * maintainer would bind (ctypes stub shown in INTEGRATION.md) to replace those layers' `call`
 * bodies.  Conventions:
 *
 *  - every pointer is a DEVICE pointer unless the name ends in `_host`; the caller owns every
 *    buffer (outputs and workspaces alike); the library never allocates device memory and links no GEMM library;
 *  - `stream` is a `cudaStream_t` passed as `void*`; all work is enqueued asynchronously on it;
 *  - return value: 0 = OK, negative = error (DTB_ERR_*); `dtb_last_error()` gives the text;
 *    no C++ exception crosses this boundary;
 *  - categorical ids: `idx` is int32 [B, F] row-major; the F tables live in ONE buffer
 *    `table` [sum_f V_f, D] (row-major, uniform D) with `row_offsets` int64 [F+1] the prefix sum
 *    of the vocabulary sizes (device memory).  Row r of field f is table[(row_offsets[f]+r)*D].
 *    An id outside [0, V_f) sets bit f&31 of *status (if status != NULL) and reads as zeros
 *    (TF-GPU behaviour; TF-CPU raises -- the host checks `status`, layers.py:893-898);
 *  - embedding gradients are scatter-ADDED into `grad_table` (same shape as `table`), which the
 *    caller keeps zeroed between steps (the row-wise Adam kernel re-zeroes rows it consumes);
 *  - fp32 everywhere unless stated; "rows" are batch rows.
 */
#ifndef DEEPTABLES_B200_H_
#define DEEPTABLES_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DTB_OK 0
#define DTB_ERR_INVALID_ARG (-1)
#define DTB_ERR_UNSUPPORTED (-2)
#define DTB_ERR_CUDA (-3)

/* activation codes (keras Activation names the hot path uses) */
#define DTB_ACT_NONE 0
#define DTB_ACT_RELU 1
#define DTB_ACT_TANH 2 /* Dense layers and the FGCNN convolution (layers.py:211,219) */

/* ---- library ---------------------------------------------------------------------------- */
int dtb_version(void);
const char* dtb_last_error(void);
int dtb_device_sm_count(int* out_host);
/* debug aid: 0 = `stream` is not capturing, 1 = capturing, 2 = its capture has been invalidated, < 0 = -cudaError */
int dtb_capture_status(void* stream);
/* number of kernels this library has launched so far (every kernel on the path is hand-written) */
long long dtb_launch_count(void);
/* kernels launched by replaying a CUDA graph captured through this library (counted once at capture): added per replay */
void dtb_launch_count_add(long long n);

/* ---- MultiColumnEmbedding (layers.py:889-904) ------------------------------------------- */
/* out[B,F,D] = table rows; the materialising form used by custom nets / tests. */
int dtb_embedding_gather(const int32_t* idx, const float* table, const int64_t* row_offsets,
                         float* out, int B, int F, int D, int* status, void* stream);
/* grad_table[row] += d_out[b,f,:]  (gradient of embedding_lookup). */
int dtb_embedding_scatter_add(const int32_t* idx, const int64_t* row_offsets, const float* d_out,
                              float* grad_table, int B, int F, int D, void* stream);

/* ---- linear (deepnets.py:43-66) + FM (layers.py:53-62), gather fused -------------------- */
/* out_lin[b] = sum_f w_lin[f]*sum_d e[b,f,d] + sum_c w_lin[F+c]*dense[b,c]   (NULL: skipped)
 * out_fm[b]  = 0.5*sum_d[(sum_f e)^2 - sum_f e^2]                             (NULL: skipped)
 * dense may be NULL iff C == 0; idx/table may be NULL iff F == 0. */
int dtb_fm_linear_fwd(const int32_t* idx, const float* table, const int64_t* row_offsets,
                      const float* dense, const float* w_lin, float* out_lin, float* out_fm,
                      int B, int F, int D, int C, int* status, void* stream);
/* g_lin/g_fm: dLoss/d out_lin, dLoss/d out_fm [B] (NULL: that branch absent).
 * grad_table += dE ; grad_wlin[F+C] += dW (both accumulate). */
int dtb_fm_linear_bwd(const int32_t* idx, const float* table, const int64_t* row_offsets,
                      const float* dense, const float* w_lin, const float* g_lin, const float* g_fm,
                      float* grad_table, float* grad_wlin, int B, int F, int D, int C, void* stream);
/* d_dense[B, C] = g_lin[b] * w_dense[c]: the gradient of the linear logit with respect to its continuous inputs
 * (w_dense = w_lin + F, the weights of the continuous columns). */
int dtb_linear_dense_grad(const float* g_lin, const float* w_dense, float* d_dense, int B, int C, void* stream);

/* ---- flatten_embeddings + concat_embedding_dense (deepmodel.py:269-278,348-357) --------- */
/* X[b, :] = [e[b,0,:], ..., e[b,F-1,:], dense[b,:]]   width W = F*D + C. */
int dtb_concat_emb_dense_fwd(const int32_t* idx, const float* table, const int64_t* row_offsets,
                             const float* dense, float* X, int B, int F, int D, int C, int* status,
                             void* stream);
/* grad_table += dX[:, :F*D] scattered by idx (the dense columns are inputs: no gradient). */
int dtb_concat_emb_dense_bwd(const int32_t* idx, const int64_t* row_offsets, const float* dX,
                             float* grad_table, int B, int F, int D, int C, void* stream);
/* The same pair for columns of different widths (fixed_embedding_dim=False, layers.py:862-877).  `table` is
 * [sum_f V_f, Dmax]; field f uses columns [0, dims_host[f]) of its rows and never touches the rest (padding).
 * X[b, :] = [e[b,0,0:D_0], ..., e[b,F-1,0:D_{F-1}], dense[b,:]], width W = sum_f D_f + C; C = 0 with dense NULL is
 * the plain flatten gather.  dims_host: F widths in [1, Dmax], host memory read at call time.  1 <= F <= 960.
 * The backward scatter-adds dX[:, :sum D_f] into grad_table ([sum_f V_f, Dmax]). */
int dtb_ragged_concat_emb_dense_fwd(const int32_t* idx, const float* table, const int64_t* row_offsets,
                                    const int* dims_host, const float* dense, float* X, int B, int F, int Dmax, int C,
                                    int* status, void* stream);
int dtb_ragged_concat_emb_dense_bwd(const int32_t* idx, const int64_t* row_offsets, const int* dims_host,
                                    const float* dX, float* grad_table, int B, int F, int Dmax, int C, void* stream);

/* ---- BatchNormalization(axis=-1) (deepmodel.py:359; layers.py:152; deepnets.py:422) ------ */
/* Training forward over X[rows, cols]: batch mean / biased variance (two-pass, fp64 accumulate),
 * Y = gamma*(X-mean)*rsqrt(var+eps)+beta, save_mean/save_var [cols] written for backward, and
 * moving = moving*momentum + batch*(1-momentum).  Y may alias X. */
int dtb_batchnorm_train_fwd(const float* X, float* Y, const float* gamma, const float* beta,
                            float* moving_mean, float* moving_var, float* save_mean, float* save_var,
                            double* workspace /* [2*cols] */, int rows, int cols, float eps,
                            float momentum, void* stream);
/* Inference forward with the moving statistics. */
int dtb_batchnorm_infer_fwd(const float* X, float* Y, const float* gamma, const float* beta,
                            const float* moving_mean, const float* moving_var, int rows, int cols,
                            float eps, void* stream);
/* Backward of the inference forward with respect to X only: dX = dY * gamma / sqrt(moving_var + eps), the scale
 * rounded as the forward rounds it.  dX may alias dY. */
int dtb_batchnorm_infer_bwd(const float* dY, float* dX, const float* gamma, const float* moving_var, int rows,
                            int cols, float eps, void* stream);
/* Backward of the training forward.  dX may alias dY.  dgamma/dbeta [cols] accumulate. */
int dtb_batchnorm_bwd(const float* X, const float* dY, float* dX, const float* gamma,
                      const float* save_mean, const float* save_var, float* dgamma, float* dbeta,
                      double* workspace /* [2*cols] */, int rows, int cols, float eps, void* stream);

/* ---- Dense (keras Dense used by deepnets.dnn 415-424, stacking 292, task_output 455; the four
 * projections of MultiheadAttention, layers.py:106-127) ----------------------------------------- */
/* Layers wider than 8 outputs run as hand-written wgmma GEMMs (csrc/dense_tc.cu: operands split on the fly into
 * bf16 hi + lo, three tensor passes, fp32 accumulation in registers => fp32-grade results; bias / activation fused into
 * the accumulator read-out); out_dim <= 8 (logit layers) as row-dot kernels.  The GEMM path packs the weights into
 * `workspace` (dtb_dense_workspace_bytes(in_dim, out_dim), 16-byte aligned; 0 for the narrow kernels). */
size_t dtb_dense_workspace_bytes(int in_dim, int out_dim);
/* Y[rows,out] = act(X[rows,in] @ W[in,out] + bias).  bias may be NULL. */
int dtb_dense_fwd(const float* X, const float* W, const float* bias, float* Y, void* workspace,
                  size_t workspace_bytes, int rows, int in_dim, int out_dim, int act, void* stream);
/* dY holds dLoss/dY on entry and is overwritten with dLoss/d(pre-activation).  dX may be NULL.
 * dW[in,out] and dbias[out] accumulate (dbias may be NULL).  dW NULL (then dbias must be NULL too, and dX set): no
 * weight-gradient kernel runs. */
int dtb_dense_bwd(const float* X, const float* W, const float* Y, float* dY, float* dX, float* dW,
                  float* dbias, void* workspace, size_t workspace_bytes, int rows, int in_dim, int out_dim,
                  int act, void* stream);

/* ---- Dropout (keras Dropout, deepmodel.py:430, deepnets.py:426; SpatialDropout1D on the (B,1,D)
 * field embeddings, layers.py:878-901, is element-wise too) -------------------------------------- */
/* Y[i] = keep(seed, i) ? X[i]/(1-rate) : 0 with a counter-based mask: calling it again on dLoss/dY with
 * the same seed IS the backward.  Y may alias X. */
int dtb_dropout(const float* X, float* Y, int64_t n, float rate, unsigned long long seed, void* stream);
/* CUDA-graph forms: the seed is read from DEVICE memory, so a captured train step replays with a fresh mask: same
 * bits as dtb_dropout for the same seed value.  dtb_seed_advance, once at the end of the captured step, moves each of
 * the step's n seeds (one per dropout call site) on by n, modulo 2^48. */
int dtb_dropout_dev(const float* X, float* Y, int64_t n, float rate, const unsigned long long* seed, void* stream);
int dtb_seed_advance(unsigned long long* seeds, int n, void* stream);

/* ---- losses on the task_output pre-activation (deepmodel.py:319-346, 436-457) ------------ */
/* task: 0 binary/multilabel (sigmoid + BCE, probabilities clipped to [1e-7,1-1e-7] as keras),
 *       1 regression (identity + MSE), 2 multiclass (softmax + CCE, y one-hot).
 * prob[rows,cols] always written; if dz != NULL: dz = dLoss/dz with Loss = mean over rows (and
 * over cols for task 0/1) of the per-sample loss times sample_weight (NULL = 1).
 * loss_sum (double, device, may be NULL) += sum of per-row losses (un-normalised). */
int dtb_loss_fwd_bwd(const float* z, const float* y_true, const float* sample_weight, float* prob,
                     float* dz, double* loss_sum, int rows, int cols, int task, void* stream);

/* Focal losses (layers.py:983-1083) passed as ModelConfig.loss: task 0 BinaryFocalLoss (sigmoid; the
 * loss is the mean over all rows x cols elements), task 2 CategoricalFocalLoss (softmax; mean over
 * rows of the per-sample sums).  Same outputs as dtb_loss_fwd_bwd; no sample weights. */
int dtb_focal_loss_fwd_bwd(const float* z, const float* y_true, float* prob, float* dz,
                           double* loss_sum, int rows, int cols, int task, float gamma, float alpha,
                           void* stream);

/* Keras 3 losses passed as ModelConfig.loss (deeptables_b200/losses.py), on the output of `task` (as above:
 * sigmoid / identity / softmax).  With p the output, y the label row, C = cols and eps = 1e-7, the per-row loss l is
 *   MEAN_SQUARED_ERROR       mean_c (p - y)^2
 *   MEAN_ABSOLUTE_ERROR      mean_c |y - p|
 *   MEAN_ABSOLUTE_PERCENTAGE_ERROR  100 mean_c |(y - p) / max(|y|, eps)|
 *   MEAN_SQUARED_LOGARITHMIC_ERROR  mean_c (log(max(p, eps) + 1) - log(max(y, eps) + 1))^2
 *   HUBER                    mean_c (|e| <= delta ? e^2 / 2 : delta |e| - delta^2 / 2),  e = p - y
 *   LOG_COSH                 mean_c (e + softplus(-2e) - log 2)
 *   POISSON                  mean_c (p - y log(p + eps))
 *   HINGE / SQUARED_HINGE    mean_c max(1 - y'p, 0) (squared); y' = 2y - 1 when every label of the batch is 0 or 1
 *   CATEGORICAL_HINGE        max(max_c((1 - y) p) - sum_c y p + 1, 0)
 *   KL_DIVERGENCE            sum_c Y log(Y / P),  Y = clip(y, eps, 1), P = clip(p, eps, 1)
 *   BINARY_CROSSENTROPY      dtb_loss_fwd_bwd's task-0 loss on y (1 - s) + s / 2
 *   CATEGORICAL_CROSSENTROPY -sum_c y_s log(clip(p / sum p, eps, 1 - eps)),  y_s = y (1 - s) + s / C
 * s = label_smoothing.  prob, dz, sample_weight and loss_sum as dtb_loss_fwd_bwd: loss_sum += sum_r w_r l_r (float64)
 * and dz = d(sum_r w_r l_r / rows)/dz under TensorFlow's gradient conventions (clip passes it on [lo, hi],
 * maximum(a, b) to a where a >= b, abs'(0) = 0, tied maxima share it, Huber at |e| = delta is quadratic);
 * dz may be NULL.  The hinge losses decide y' on the device (one more launch, into lp->scratch); nothing
 * synchronises with the host. */
#define DTB_LOSS_MEAN_SQUARED_ERROR 1
#define DTB_LOSS_MEAN_ABSOLUTE_ERROR 2
#define DTB_LOSS_MEAN_ABSOLUTE_PERCENTAGE_ERROR 3
#define DTB_LOSS_MEAN_SQUARED_LOGARITHMIC_ERROR 4
#define DTB_LOSS_HUBER 5
#define DTB_LOSS_LOG_COSH 6
#define DTB_LOSS_POISSON 7
#define DTB_LOSS_HINGE 8
#define DTB_LOSS_SQUARED_HINGE 9
#define DTB_LOSS_CATEGORICAL_HINGE 10
#define DTB_LOSS_KL_DIVERGENCE 11
#define DTB_LOSS_BINARY_CROSSENTROPY 12
#define DTB_LOSS_CATEGORICAL_CROSSENTROPY 13
typedef struct dtb_loss_params {  /* host memory, read at call time */
  int loss;                       /* DTB_LOSS_* */
  float delta;                    /* HUBER: > 0 and finite */
  float label_smoothing;          /* s of the two crossentropies, in [0, 1]; 0 for the others */
  int* scratch;                   /* device int the hinge losses use (NULL for the others) */
} dtb_loss_params;
int dtb_keras_loss_fwd_bwd(const float* z, const float* y_true, const float* sample_weight, float* prob, float* dz,
                           double* loss_sum, int rows, int cols, int task, const dtb_loss_params* lp, void* stream);

/* ---- keras Adam (deepmodel.py:321-322), dense semantics ---------------------------------- */
/* m += (g-m)(1-b1); v += (g^2-v)(1-b2); p -= m*alpha/(sqrt(v)+eps), alpha computed by caller
 * as lr*sqrt(1-b2^t)/(1-b1^t).  If zero_grad != 0, g is zeroed after use. */
int dtb_adam_dense(float* p, float* m, float* v, float* g, int64_t n, float alpha, double beta1,
                   double beta2, float eps, int zero_grad, void* stream);

/* Exact-lazy row-wise Adam for embedding tables (same arithmetic as dtb_adam_dense applied to
 * every row every step, but rows whose gradient is zero are caught up only when next touched).
 * last_step[row] = last optimiser step already applied to that row.  alpha_table[s] (device,
 * s = 1..) = alpha of step s (a learning-rate schedule is folded into it).  The replay of long
 * zero-gradient gaps stops early under a bound that holds while
 * fl(fl(7 * 2^-149 * max alpha) / eps) < 2^-108 (adam_rows.cu); the caller keeps tables past it dense.
 *   catchup: for every (b,f): apply the zero-gradient steps last_step+1 .. upto to that row once.
 *   apply  : for every (b,f): apply step `step` with the accumulated grad_table row once, zero
 *            the grad row, set last_step = step. */
int dtb_adam_rows_catchup(const int32_t* idx, const int64_t* row_offsets, float* table, float* m,
                          float* v, int32_t* last_step, const float* alpha_table, int upto,
                          double beta1, double beta2, float eps, int B, int F, int D, void* stream);
int dtb_adam_rows_apply(const int32_t* idx, const int64_t* row_offsets, float* table, float* m,
                        float* v, float* grad_table, int32_t* last_step, const float* alpha_table,
                        int step, double beta1, double beta2, float eps, int B, int F, int D,
                        void* stream);
/* Bring every row of the table up to date (before save / export / dense evaluation). */
int dtb_adam_rows_flush(float* table, float* m, float* v, int32_t* last_step,
                        const float* alpha_table, int upto, double beta1, double beta2, float eps,
                        int64_t n_rows, int D, void* stream);
/* CUDA-graph forms: the optimiser step counter lives in DEVICE memory (*step_dev = steps completed so far), so a
 * captured train step replays with the right bias correction: dense = step *step_dev + 1 with alpha_table[*step_dev + 1];
 * rows catch-up to *step_dev; rows apply = step *step_dev + 1; dtb_step_increment bumps the counter at the end. */
int dtb_adam_dense_dev(float* p, float* m, float* v, float* g, int64_t n, const float* alpha_table,
                       const int32_t* step_dev, double beta1, double beta2, float eps, int zero_grad, void* stream);
int dtb_adam_rows_catchup_dev(const int32_t* idx, const int64_t* row_offsets, float* table, float* m, float* v,
                              int32_t* last_step, const float* alpha_table, const int32_t* step_dev, double beta1,
                              double beta2, float eps, int B, int F, int D, void* stream);
int dtb_adam_rows_apply_dev(const int32_t* idx, const int64_t* row_offsets, float* table, float* m, float* v,
                            float* grad_table, int32_t* last_step, const float* alpha_table, const int32_t* step_dev,
                            double beta1, double beta2, float eps, int B, int F, int D, void* stream);
int dtb_step_increment(int32_t* step_dev, void* stream);

/* ---- keras SGD, RMSprop and Adagrad, dense semantics (optim.cu) ----------------------------------
 * Hyperparameters travel in a host-side struct read at call time (a captured graph keeps the values
 * of the call it captured).  The learning rate may instead come from a device table (the *_lr forms
 * below), which is how a schedule or a rate changed during training reaches a captured graph.  State slots s0..s2 are [n] floats
 * like p, NULL when the optimiser does not use them:
 *   SGD     s0 = momentum buffer (when momentum > 0)
 *   RMSprop s0 = velocity, s1 = average gradient (centered), s2 = momentum buffer (momentum > 0)
 *   Adagrad s0 = accumulator (the caller fills it with initial_accumulator_value)
 * The row forms follow dtb_adam_rows_*: last_step[row] = last step applied to the row, ownership per
 * launch by atomicMax on last_step, out-of-range ids skipped, D = 4*2^k (<= 128).  Skipped
 * zero-gradient steps are replayed in order with the same arithmetic; for SGD without momentum and
 * for Adagrad such a step is the identity, so catch-up and flush return at once.  The `_dev` forms
 * read the number of completed steps from device memory (CUDA-graph replay); the dense sweep does
 * not depend on the step number, so its one form serves both. */
#define DTB_OPTIM_SGD 1
#define DTB_OPTIM_RMSPROP 2
#define DTB_OPTIM_ADAGRAD 3
typedef struct dtb_optim_params {
  int kind;         /* DTB_OPTIM_* */
  int flag;         /* SGD: nesterov; RMSprop: centered */
  float lr;
  float momentum;   /* SGD and RMSprop; 0 = no momentum slot */
  double rho;       /* RMSprop; the kernels use rho and (float)(1.0 - rho) as Keras does */
  float eps;        /* RMSprop and Adagrad */
} dtb_optim_params;

int dtb_optim_dense(float* p, float* g, float* s0, float* s1, float* s2, int64_t n, const dtb_optim_params* hp,
                    int zero_grad, void* stream);
int dtb_optim_rows_catchup(const int32_t* idx, const int64_t* row_offsets, float* table, float* s0, float* s1,
                           float* s2, int32_t* last_step, int upto, const dtb_optim_params* hp, int B, int F, int D,
                           void* stream);
int dtb_optim_rows_apply(const int32_t* idx, const int64_t* row_offsets, float* table, float* s0, float* s1, float* s2,
                         float* grad_table, int32_t* last_step, int step, const dtb_optim_params* hp, int B, int F,
                         int D, void* stream);
int dtb_optim_rows_flush(float* table, float* s0, float* s1, float* s2, int32_t* last_step, int upto,
                         const dtb_optim_params* hp, int64_t n_rows, int D, void* stream);
int dtb_optim_rows_catchup_dev(const int32_t* idx, const int64_t* row_offsets, float* table, float* s0, float* s1,
                               float* s2, int32_t* last_step, const int32_t* step_dev, const dtb_optim_params* hp,
                               int B, int F, int D, void* stream);
int dtb_optim_rows_apply_dev(const int32_t* idx, const int64_t* row_offsets, float* table, float* s0, float* s1,
                             float* s2, float* grad_table, int32_t* last_step, const int32_t* step_dev,
                             const dtb_optim_params* hp, int B, int F, int D, void* stream);
int dtb_optim_rows_flush_dev(float* table, float* s0, float* s1, float* s2, int32_t* last_step,
                             const int32_t* step_dev, const dtb_optim_params* hp, int64_t n_rows, int D, void* stream);
/* Learning-rate table forms of the steps that apply a gradient: dtb_optim_dense, dtb_optim_rows_apply(_dev) and
 * dtb_optim_dense_reg with the rate of step s read from lr_table[s] (device, s = 1..) instead of hp->lr.  The step
 * is *step_dev + 1 when step_dev is not NULL (CUDA-graph replay), else the host's `step` (>= 1).  With a table
 * that holds hp->lr at that step they give the bits of the constant-rate symbols.  The zero-gradient catch-up and
 * flush need no table: a g = 0 step of SGD, RMSprop or Adagrad does not depend on the rate. */
int dtb_optim_dense_lr(float* p, float* g, float* s0, float* s1, float* s2, int64_t n, const dtb_optim_params* hp,
                       const float* lr_table, int step, const int32_t* step_dev, int zero_grad, void* stream);
int dtb_optim_rows_apply_lr(const int32_t* idx, const int64_t* row_offsets, float* table, float* s0, float* s1,
                            float* s2, float* grad_table, int32_t* last_step, const float* lr_table, int step,
                            const int32_t* step_dev, const dtb_optim_params* hp, int B, int F, int D, void* stream);

/* ---- keras.regularizers L1 / L2 / L1L2 on a weight (add_weight(regularizer=)) ------------------ */
/* Loss l1*sum|w| + l2*sum w^2, gradient l1*sign(w) + 2*l2*w with sign(0) = 0.  The total gradient is
 * g + (l1*sign(w) + (2*l2)*w), rounded the same way by every entry point below, so dtb_reg_grad
 * followed by dtb_adam_dense / dtb_optim_dense gives the bits of the fused *_reg sweep.
 * dtb_reg_grad: g += gradient (g may be NULL: loss only).  All four add loss_scale * loss, summed in
 * float64 from the weights before the step, into *loss_acc (may be NULL).  l1, l2 >= 0 and finite. */
int dtb_reg_grad(const float* p, float* g, int64_t n, float l1, float l2, double* loss_acc, double loss_scale,
                 void* stream);
/* dtb_adam_dense / dtb_adam_dense_dev / dtb_optim_dense with the regularization gradient added to g
 * in the same pass (no extra HBM traffic) */
int dtb_adam_dense_reg(float* p, float* m, float* v, float* g, int64_t n, float alpha, double beta1, double beta2,
                       float eps, int zero_grad, float l1, float l2, double* loss_acc, double loss_scale, void* stream);
int dtb_adam_dense_reg_dev(float* p, float* m, float* v, float* g, int64_t n, const float* alpha_table,
                           const int32_t* step_dev, double beta1, double beta2, float eps, int zero_grad, float l1,
                           float l2, double* loss_acc, double loss_scale, void* stream);
int dtb_optim_dense_reg(float* p, float* g, float* s0, float* s1, float* s2, int64_t n, const dtb_optim_params* hp,
                        int zero_grad, float l1, float l2, double* loss_acc, double loss_scale, void* stream);
/* dtb_optim_dense_reg with the rate from lr_table, as dtb_optim_dense_lr */
int dtb_optim_dense_reg_lr(float* p, float* g, float* s0, float* s1, float* s2, int64_t n, const dtb_optim_params* hp,
                           const float* lr_table, int step, const int32_t* step_dev, int zero_grad, float l1, float l2,
                           double* loss_acc, double loss_scale, void* stream);

/* ---- streaming metrics (keras.metrics accumulators; deepmodel.py:319-346 passes ModelConfig.metrics to compile) --- */
/* One device buffer `state` of 8-byte words holds every configured metric of a model; one dtb_metrics_update per
 * batch adds the batch to all of them.  Layout, with C = plan->cols:
 *   words [0, 8)              float64 sums over rows of the row means (over the C columns) of DTB_METRIC_SUM_* in bit
 *                             order: (p-y)^2, |p-y|, 100|p-y|/max(|y|,1e-7), (log(max(p,1e-7)+1)-log(max(y,1e-7)+1))^2,
 *                             log cosh(p-y), binary and categorical cross-entropy on probabilities; word 7 unused
 *   words [8, 8+3C)           float64 per column: sum y, sum y^2, sum (y-p)^2                 (DTB_METRIC_SUM_R2)
 *   counters from word 8+3C   uint64: [0] rows; [1] rows whose first arg-max of p is the first arg-max of y; [2] rows
 *                             whose p at the first arg-max of y is finite and exceeded by fewer than top_k others;
 *                             [3+kC+c], k = 0,1,2: TP, FP, FN of column c with the prediction "p_c is the row maximum
 *                             and |p_c| > 1e-9" (keras FBetaScore without a threshold); then for every threshold list
 *                             l in order a histogram [C][2][list_len[l]+1]: bucket j of (column c, label y_c != 0)
 *                             counts the elements with exactly j thresholds strictly below p (keras tests p > t), so
 *                             TP(t_i) is the sum of the label-1 buckets above i.  A NaN p is above no threshold.
 * Each list is ascending float32 at thresholds_dev[list_off[l] ..]; all lists together hold at most
 * DTB_METRIC_MAX_THRESHOLDS values.  The counters are integers added with atomics: the same batches give the same
 * bits whatever the block scheduling, eagerly or replayed from a CUDA graph.  The float64 sums are warp-reduced and
 * added with atomicAdd(double), as the loss sum of dtb_loss_fwd_bwd is: their last bits depend on the order.
 * Arg-max counters are kept only when plan->argmax is set, sums only for the bits of plan->sums.  The update reads
 * device memory and the plan only (no per-step host scalar): it can be captured in a CUDA graph. */
#define DTB_METRIC_MAX_LISTS 8
#define DTB_METRIC_MAX_THRESHOLDS 2048
#define DTB_METRIC_SUM_SE 1
#define DTB_METRIC_SUM_AE 2
#define DTB_METRIC_SUM_APE 4
#define DTB_METRIC_SUM_SLE 8
#define DTB_METRIC_SUM_LOGCOSH 16
#define DTB_METRIC_SUM_BCE 32
#define DTB_METRIC_SUM_CCE 64
#define DTB_METRIC_SUM_R2 128
typedef struct dtb_metric_plan {
  int cols;                            /* columns of prob / y_true */
  int n_lists;                         /* threshold lists, <= DTB_METRIC_MAX_LISTS */
  int list_len[DTB_METRIC_MAX_LISTS];  /* thresholds per list, >= 1 */
  int list_off[DTB_METRIC_MAX_LISTS];  /* first threshold of the list in thresholds_dev */
  int sums;                            /* DTB_METRIC_SUM_* bits */
  int argmax;                          /* keep the arg-max counters [1], [2] and the per-column TP / FP / FN */
  int top_k;                           /* k of counter [2], >= 1 when argmax is set */
} dtb_metric_plan;
size_t dtb_metrics_state_bytes(const dtb_metric_plan* plan);
int dtb_metrics_reset(void* state, const dtb_metric_plan* plan, void* stream);
int dtb_metrics_update(const float* prob, const float* y_true, void* state, const float* thresholds_dev, int rows,
                       const dtb_metric_plan* plan, void* stream);

/* ---- permutation feature importance (deeptables_b200/importance.py, utils/feature_importance.py) ---------------- */
/* keys[r] = ((hash(seed, iter, column, r) ^ 2^31) << 32) | r for r < rows < 2^32; sorted as signed 64-bit integers,
 * their low halves are the permutation of one pass.  seed < 2^32; iter, column >= 0. */
int dtb_perm_keys(long long* keys, int64_t rows, unsigned long long seed, int iter, int column, void* stream);
/* dst[b*width + column] = src[perm[b]*width + column] for 4-byte elements, perm[b] the low half of sorted_keys[b];
 * sorted_keys NULL copies the column back (perm[b] = b).  Other columns of dst are not touched. */
int dtb_shuffle_column(const void* src, void* dst, const long long* sorted_keys, int64_t rows, int width, int column,
                       void* stream);
/* Each scoring call writes one float64 to *out (device memory) and never synchronises with the host.  `scratch` is
 * device memory of dtb_importance_scratch_bytes(cols) bytes; `prob` is the model output [rows, cols]. */
#define DTB_IMPORTANCE_AUC 1
#define DTB_IMPORTANCE_LOG_LOSS 2
#define DTB_IMPORTANCE_ACCURACY 3
#define DTB_IMPORTANCE_F1 4          /* binary F1 of class `pos` */
#define DTB_IMPORTANCE_F1_MACRO 5
#define DTB_IMPORTANCE_MSE 6
#define DTB_IMPORTANCE_RMSE 7
#define DTB_IMPORTANCE_MAE 8
#define DTB_IMPORTANCE_R2 9
size_t dtb_importance_scratch_bytes(int cols);
/* binary ROC AUC from ascending predictions sorted_prob[i] = prob[order[i]] and positive[r] in {0, 1} */
int dtb_importance_auc(const float* sorted_prob, const long long* order, const int* positive, int64_t rows,
                       void* scratch, double* out, void* stream);
/* accuracy / F1 / macro F1 of the predicted class against label[r] (class codes; one column: 0 or 1) */
int dtb_importance_labels(int metric, const float* prob, const int* label, int64_t rows, int cols, int pos,
                          void* scratch, double* out, void* stream);
/* log loss (label[r]: the true column) or, on one column against target[r], MSE / RMSE / MAE / R2 (aux: the sum of
 * squared deviations of target from its mean) */
int dtb_importance_sums(int metric, const float* prob, const int* label, const double* target, int64_t rows, int cols,
                        double aux, void* scratch, double* out, void* stream);

/* ---- Kernel SHAP (deeptables_b200/explain.py, utils/shap.py) ----------------------------------------------------- */
/* The synthetic rows of `coalitions` coalitions over `bg_rows` background rows: row k*bg_rows + j is background row j
 * (bg_cat [bg_rows, fields], bg_cont [bg_rows, conts]) with every column whose bit is set in mask k replaced by the
 * value of explained row x_index[k] (x_cat [*, fields], x_cont [*, conts]).  masks: [coalitions, mask_words] bit sets;
 * cat_bit[f] / cont_bit[c]: the column's bit, or -1 for a column that always keeps the background's value.  Writes
 * out_cat [coalitions*bg_rows, fields] and out_cont [coalitions*bg_rows, conts]; fields or conts may be 0 (then their
 * pointers may be NULL). */
int dtb_shap_compose(const int32_t* x_cat, const float* x_cont, const int32_t* bg_cat, const float* bg_cont,
                     const uint32_t* masks, int mask_words, const int32_t* x_index, const int32_t* cat_bit,
                     const int32_t* cont_bit, int64_t coalitions, int bg_rows, int fields, int conts,
                     int32_t* out_cat, float* out_cont, void* stream);
/* out[g] (float64) = the mean, over rows g*rows_per_group .. +rows_per_group-1 of the model output prob [*, cols], of
 * the model function: the output itself (DTB_SHAP_VALUE, one column) or DeepTable.predict's class code
 * (DTB_SHAP_CLASS: p > 1 - p in float32 on one column, the first arg-max on several).  Fixed summation order. */
#define DTB_SHAP_VALUE 0
#define DTB_SHAP_CLASS 1
int dtb_shap_means(const float* prob, int64_t groups, int rows_per_group, int cols, int kind, double* out,
                   void* stream);

/* ---- expected gradients (deeptables_b200/explain.py, utils/shap.py DeepTablesGradientExplainer) -------------------- */
/* Pair p interpolates between explained row x_index[p] (x_cat [*, fields], x_cont [*, conts]) and background row
 * bg_index[p] (bg_cat, bg_cont) at alpha[p]: every value is v = b + alpha * (x - b), each operation rounded on its own
 * (no fused multiply-add).  Categorical field f interpolates its embedding rows (table [*, table_dim], row_offsets
 * [fields+1]; an id out of range reads as zeros) over its first col_offsets[f+1] - col_offsets[f] coordinates.
 * out_emb is [fields, pairs, table_dim] when field_major (every field of width table_dim: the layout of a tensor-backed
 * field block) and [pairs, col_offsets[fields]] otherwise; out_cont is [pairs, conts].  fields or conts may be 0 (then
 * their pointers may be NULL). */
int dtb_gradshap_compose(const int32_t* x_cat, const float* x_cont, const int32_t* bg_cat, const float* bg_cont,
                         const float* table, const int64_t* row_offsets, const int32_t* col_offsets, int table_dim,
                         const int32_t* x_index, const int32_t* bg_index, const float* alpha, int64_t pairs,
                         int fields, int conts, int field_major, float* out_emb, float* out_cont, void* stream);
/* out [pairs, fields + conts] (float64): for field f, sum over d in order of g_emb[p, col_offsets[f] + d] times the
 * float32 difference of the two embedding coordinates (g_emb [pairs, col_offsets[fields]]); for continuous column c,
 * g_cont[p, c] times x - b.  A zero difference contributes exactly 0.  Arguments as dtb_gradshap_compose. */
int dtb_gradshap_reduce(const int32_t* x_cat, const float* x_cont, const int32_t* bg_cat, const float* bg_cont,
                        const float* table, const int64_t* row_offsets, const int32_t* col_offsets, int table_dim,
                        const int32_t* x_index, const int32_t* bg_index, int64_t pairs, int fields, int conts,
                        const float* g_emb, const float* g_cont, double* out, void* stream);
/* out [rows, cols] (float64) = the mean of values [rows * samples, cols] over each row's samples, added in sample
 * order. */
int dtb_gradshap_means(const double* values, int64_t rows, int samples, int cols, double* out, void* stream);
/* dz [rows, cols] = the derivative of output column k with respect to the pre-activation z [rows, cols]: the identity
 * (regression), the sigmoid of each column (binary, multilabel) or the softmax over the columns (multiclass). */
#define DTB_GRADSHAP_IDENTITY 0
#define DTB_GRADSHAP_SIGMOID 1
#define DTB_GRADSHAP_SOFTMAX 2
int dtb_gradshap_output_grad(const float* z, int64_t rows, int cols, int k, int kind, float* dz, void* stream);

/* ---- partial dependence (deeptables_b200/utils/partial_dependence.py) --------------------------------------------- */
/* prob [groups*rows_per_group, cols]: row k*rows_per_group + j is row j of group k.  The rows of each group are cut into
 * blocks of block_rows (the last may be short); out [groups, blocks, cols] (float64) receives, for each block and
 * column, the sum over its rows of weight[j] * prob (weight [rows_per_group] float64, or NULL for weight 1).  Each sum
 * has one fixed order (lane stride 32 within the block, then a fixed butterfly), so a block's sum is the same bits
 * wherever the block sits in a launch. */
int dtb_pdp_block_sums(const float* prob, const double* weight, int64_t groups, int rows_per_group, int cols,
                       int block_rows, double* out, void* stream);

/* ---- linear probes (deeptables_b200/probe.py; reference deeptable.py probe_evaluate) ------------------------------ */
/* The objective of scikit-learn's lbfgs LogisticRegression over the float32 features X [n, d] (row stride ldx floats)
 * with class codes y [n] and float64 weights W [K, d + 1] (column d: the intercept, read only when fit_intercept):
 * z_k = sum_j x_j W[k, j] (+ W[k, d]).  Binary (K = 1, y in {0, 1}): loss log(1 + e^z) - y z, residual sigma(z) - y.
 * Multinomial (K = classes, y in [0, K)): loss logsumexp(z) - z_y, residual softmax(z)_k - [k = y].
 * partials [ceil(n / DTB_PROBE_BLOCK_ROWS), 1 + K (d + 1)] (float64) receives, per block of DTB_PROBE_BLOCK_ROWS rows,
 * the sum of the losses, then sum r_k x_j at 1 + k (d + 1) + j (x_d = 1; 0 without an intercept).  Every sum runs over
 * the block's rows in order, so a block's partial is the same bits for every tile_rows in [1, dtb_probe_tile_rows]
 * (0: that most).  X is read once; every product and sum is float64. */
#define DTB_PROBE_BLOCK_ROWS 1024
#define DTB_PROBE_MAX_CLASSES 64
int dtb_probe_loss_grad(const float* X, int64_t ldx, const int32_t* y, const double* W, int64_t n, int d, int K,
                        int fit_intercept, int tile_rows, double* partials, void* stream);
/* The most rows of d columns a loss_grad tile stages for K classes; 0 when a row does not fit in shared memory. */
int dtb_probe_tile_rows(int d, int K);
/* out[c] = partials[0, c] + partials[1, c] + ... in block order (out [width] float64). */
int dtb_probe_join(const double* partials, int64_t blocks, int width, double* out, void* stream);
/* The fitted probe on X [n, d]: proba [n, max(K, 2)] float64 (binary: [1 - sigma(z), sigma(z)]; multinomial: softmax)
 * and codes [n]: binary z > 0, multinomial the first arg-max of z. */
int dtb_probe_predict(const float* X, int64_t ldx, const double* W, int64_t n, int d, int K, int fit_intercept,
                      double* proba, int32_t* codes, void* stream);
/* *count += the number of rows i with pred[i] == truth[i] (an integer count; the caller zeroes *count). */
int dtb_probe_correct(const int32_t* pred, const int32_t* truth, int64_t n, unsigned long long* count, void* stream);

/* ---- target encoding (deeptables_b200/target_encoding.py; reference preprocessing/utils.py) ---------------------- */
/* A column's rows carry a category code (-1: unknown), a fold id in [0, folds) and, for class targets, a class index
 * in [0, classes).  A continuous target has classes = 0.  Group g of a column's statistics is every fold (g = 0) or,
 * when folds > 1, every fold but f (g = 1 + f): the fitting rows of the rows held out in fold f. */
#define DTB_TE_CHUNK 1024
#define DTB_TE_SMOOTH 0   /* scikit-learn, float smooth: (smooth mu + S) / (smooth + n); mu when smooth + n = 0 */
#define DTB_TE_AUTO 1     /* scikit-learn, smooth='auto': l = var n / (var n + SSD / n); l (S / n) + (1 - l) mu, mu
                             when l is NaN.  var is the group's target variance, SSD the category's sum of squared
                             differences from S / n */
#define DTB_TE_RECALLED 2 /* category_encoders' TargetEncoder as recalled, min_samples_leaf = 20:
                             s = 1 / (1 + exp(-(n - 20) / smooth)); mu (1 - s) + (S / n) s; mu when n = 0 */
/* out[i] = map[in[i]] when 0 <= in[i] < map_len, else -1 (the host's factorised codes into sorted category order). */
int dtb_te_remap(const int64_t* in, const int32_t* map, int64_t n, int map_len, int32_t* out, void* stream);
/* keys[i] = (code * folds + fold) * max(classes, 1) + class, where a code -1 counts as unknown_code; -1 when that is
 * -1 too (the row joins no category).  codes NULL: every code is 0; fold NULL: every fold is 0; cls is read only when
 * classes > 0.  scikit-learn counts the rows outside given categories toward the first one: unknown_code 0. */
int dtb_te_keys(const int32_t* codes, const uint8_t* fold, const int32_t* cls, int64_t n, int folds, int classes,
                int unknown_code, int64_t* keys, void* stream);
/* keys [n] sorted ascending, each -1 or in [0, slots): starts[s] (s in [0, slots]) = the first position whose key is
 * >= s (n for s = slots), so slot s holds starts[s+1] - starts[s] rows. */
int dtb_te_segment_starts(const int64_t* keys, int64_t n, int64_t slots, int64_t* starts, void* stream);
/* For each chunk of a slot's sorted rows (DTB_TE_CHUNK rows counted from the slot's start, the last may be short)
 * beginning at position q: partial[q] = the sum over its rows r of y[perm[r]] (seg_sum NULL), or of (y[perm[r]] - c)^2
 * with c = seg_sum[slot] / (the slot's rows).  Lane l of a warp adds rows q+l, q+l+32, ... in order, then a fixed
 * butterfly; tile_rows (a multiple of 32) only splits the work between CTAs.  Other entries of partial are untouched. */
int dtb_te_segment_stats(const int64_t* keys, const int64_t* perm, const double* y, const int64_t* starts,
                         const double* seg_sum, int64_t n, int tile_rows, double* partial, void* stream);
/* out[s] = the chunk partials of slot s added in chunk order (0 for an empty slot). */
int dtb_te_segment_join(const int64_t* starts, const double* partial, int64_t slots, double* out, void* stream);
/* table [groups, cats, n_out] and, when prior is not NULL, prior [groups, n_out] (float64), groups = folds + 1 when
 * folds > 1, else 1; n_out = classes when classes > 2, else 1.  starts (and, for a continuous target, sums and m2: the
 * joined chunk sums and sums of squares around each slot's mean) are one column's statistics keyed as dtb_te_keys; the
 * p_ arrays are those of the whole target, keyed with every code 0.  For group g and output j, n, S are the rows and the
 * target sum (class targets: the rows of class j, or of class 1 when classes = 2) over the group's folds, each added in
 * increasing fold order, and mu the same ratio for the whole target.  Class targets take SSD and var in closed form from
 * the counts; continuous ones add, in fold order, each fold's sum of squares plus n_k (mean_k - mean)^2.  The encoding
 * is the formula DTB_TE_*. */
int dtb_te_encodings(const int64_t* starts, const double* sums, const double* m2, const int64_t* p_starts,
                     const double* p_sums, const double* p_m2, int64_t cats, int folds, int classes, int formula,
                     double smooth, double* table, double* prior, void* stream);
/* out[r * out_stride + c * n_out + j] (float64) = the encoding of codes[c * n + r] in group g (fold NULL: 0, else
 * 1 + fold[r]) of column c, whose table [groups, cats[c], n_out] starts at table + table_off[c]; for code -1
 * prior[g, j], or prior[unknown_group, j] when unknown_group >= 0 (scikit-learn's fit_transform gives every unknown
 * row the last fold's mean); NaN for a code >= cats[c]. */
int dtb_te_gather(const int32_t* codes, const uint8_t* fold, const double* table, const int64_t* table_off,
                  const int32_t* cats, const double* prior, int64_t n, int cols, int n_out, int unknown_group,
                  int out_stride, double* out, void* stream);

/* ---- gradient-boosted leaf features (deeptables_b200/gbm.py; reference preprocessor.py:431-452) ------------------- */
/* Feature i of a booster is read from the model's own inputs: feat_col[i] = c >= 0 is column c of cat [rows, cat_stride]
 * (int32 codes, compared as their float32 values), feat_col[i] = -1 - c is column c of cont [rows, cont_stride].
 * edges (float32) holds each feature's increasing bin edges at edge_off[i] .. edge_off[i+1]-1; the bin of x is the
 * number of edges < x, NaN the last bin (the number of edges).  bins [rows, nf] uint8, row-major. */
int dtb_gbdt_bin(const int32_t* cat, int cat_stride, const float* cont, int cont_stride, const int32_t* feat_col,
                 const float* edges, const int32_t* edge_off, int64_t rows, int nf, uint8_t* bins, void* stream);
/* Gradient and hessian of class k of the float64 scores [rows, K] (LightGBM's objectives): DTB_GBDT_BINARY p - y,
 * p(1-p) with p = sigmoid(s); DTB_GBDT_L2 s - y, 1; DTB_GBDT_SOFTMAX p_k - [y = k], K/(K-1) p_k(1-p_k).  Computed in
 * float64, rounded to float32 into g, h; label is float32 (binary, L2) or the class code as float32 (softmax).
 * max_gh[0..1] (device, caller zeroes) receive max |g| and max h by integer atomics on their bit patterns. */
#define DTB_GBDT_BINARY 0
#define DTB_GBDT_L2 1
#define DTB_GBDT_SOFTMAX 2
int dtb_gbdt_grad(const double* scores, const float* label, int64_t rows, int K, int k, int objective, float* g,
                  float* h, float* max_gh, void* stream);
/* Fixed point: gq = rint(g * 2^shift_g), hq = rint(h * 2^shift_h) as int64 (the caller picks the shifts so that no
 * sum over rows reaches 2^62). */
int dtb_gbdt_fixed(const float* g, const float* h, int64_t rows, int shift_g, int shift_h, int64_t* gq, int64_t* hq,
                   void* stream);
/* Histogram of one leaf: the rows index[begin .. begin+count) of bins.  hist_g / hist_h (int64) and hist_n (int32),
 * each [nf, nb] (nb >= every feature's bin count, <= 256), are overwritten with the sums of gq, hq and the row count
 * per (feature, bin).  Integer sums: the result does not depend on the order of the rows. */
int dtb_gbdt_hist(const uint8_t* bins, const int32_t* index, int64_t begin, int64_t count, const int64_t* gq,
                  const int64_t* hq, int nf, int nb, int64_t* hist_g, int64_t* hist_h, int32_t* hist_n, void* stream);
/* The subtraction trick on [elements] of the three arrays, leaving the left child in parent_* and the right one in
 * small_*: small_is_left = 0 (small holds the right child): parent -= small; small_is_left = 1: (parent, small) =
 * (small, parent - small). */
int dtb_gbdt_hist_sub(int64_t* parent_g, int64_t* parent_h, int32_t* parent_n, int64_t* small_g, int64_t* small_h,
                      int32_t* small_n, int64_t elements, int small_is_left, void* stream);
/* Best split of each leaf in leaves[0 .. n_leaves): the histogram of leaf l is hist_* + l * nf * nb.  Candidate
 * (feature f, bin t < n_bins[f] - 1) sends bins <= t left.  Valid when both sides have >= min_child_samples rows and a
 * hessian >= min_child_weight; gain in float64 from the integer sums (G = gq_sum * scale_g, H = hq_sum * scale_h),
 * T(G)^2/(H+lambda) left + right - parent - min_split_gain, T the L1 soft threshold at alpha; ties to the lowest
 * feature, then the lowest t.  out[i] gets the leaf's sums and its best split (feature -1, gain 0 when none has
 * gain > 0). */
typedef struct {
  double gain;
  int64_t g, h, left_g, left_h;
  int32_t count, left_count, feature, bin;
} dtb_gbdt_split_rec;
typedef struct {
  double lambda_l2, lambda_l1, min_split_gain, min_child_weight, scale_g, scale_h;
  int32_t min_child_samples;
} dtb_gbdt_split_params;
int dtb_gbdt_split(const int64_t* hist_g, const int64_t* hist_h, const int32_t* hist_n, const int32_t* leaves,
                   int n_leaves, const int32_t* n_bins, int nf, int nb, const dtb_gbdt_split_params* params_host,
                   dtb_gbdt_split_rec* out, void* stream);
/* Split the segment index[begin .. begin+count) in place: rows whose bin of `feature` is <= bin first (left_count of
 * them, from the split record), the rest after; the order inside each half is unspecified.  scratch: int32 [count + 2]. */
int dtb_gbdt_partition(const uint8_t* bins, int nf, int32_t* index, int64_t begin, int64_t count, int feature,
                       int bin, int64_t left_count, int32_t* scratch, void* stream);
/* After a tree: for every leaf l, each row r of index[seg_begin[l] .. + seg_count[l]) gets
 * scores[r * K + k] += (double)leaf_value[l] and, when leaf_out is not NULL, leaf_out[r * leaf_stride] = l. */
int dtb_gbdt_update(const int32_t* index, const int64_t* seg_begin, const int64_t* seg_count, int n_leaves,
                    int64_t max_count, const float* leaf_value, double* scores, int K, int k, int32_t* leaf_out,
                    int64_t leaf_stride, void* stream);
/* Leaf index of every row in each of n_trees trees, walked on the raw values (x <= threshold goes left, NaN right).
 * Tree t's internal nodes are node_* [node_off[t] .. node_off[t+1]); a child >= 0 is a node of the same tree, a child
 * < 0 the leaf ~child; a tree without nodes is the single leaf 0.  Trees are staged in shared memory in chunks of at
 * most DTB_GBDT_STAGE_NODES nodes (a larger tree is refused).  Leaf j of tree t goes to out_cat[r * out_stride +
 * out_col + t] (int32) when out_cat is not NULL, else to out_cont[...] as float32. */
#define DTB_GBDT_STAGE_NODES 2048
int dtb_gbdt_leaves(const int32_t* cat, int cat_stride, const float* cont, int cont_stride, const int32_t* feat_col,
                    const int32_t* node_feature, const float* node_threshold, const int32_t* node_left,
                    const int32_t* node_right, const int32_t* node_off, int n_trees, int max_tree_nodes,
                    int64_t rows, int32_t* out_cat, float* out_cont, int out_stride, int out_col, void* stream);

/* ---- quantile-bin discretisation (deeptables_b200/discrete.py; reference preprocessor.py:406-415) ------------------ */
/* out_cat[r * out_stride + out_col + j] (int32) = the number of inner edges e of column j with e <= (double)x, where
 * x = cont[r * cont_stride + src_col[j]] (numpy's searchsorted side='right': ties go to the upper bin, -0.0 == 0.0).
 * Column j's increasing float64 inner edges are edges[edge_off[j] .. edge_off[j+1]); a column without edges gets
 * code 0.  src_col[j] < cont_stride is the caller's to guarantee (device memory).  One launch covers every row and
 * column, with 64-bit indexing; the edges are searched in global memory, so a column may have any number of them. */
int dtb_discretize(const float* cont, int cont_stride, int64_t rows, const int32_t* src_col, const double* edges,
                   const int64_t* edge_off, int n_cols, int32_t* out_cat, int out_stride, int out_col, void* stream);

/* ---- denoising auto-encoder batches (deeptables_b200/dae.py; reference fe/dae.py) ---------------------------------- */
/* One training batch of rows <= batch_rows rows from X [*, cols] (float32, row-major), with
 * base = (*step_dev - *epoch_first_step_dev) * batch_rows and s = *step_dev + 1 read from device memory, so that one
 * captured CUDA graph serves every full batch of every epoch:
 *   x_tgt[i, :] = X[p1[base + i], :]
 *   x_in[i, c]  = X[p2[base + i], c] when c is one of row i's k swapped columns at step s, else x_tgt[i, c].
 * The swapped columns of row i are the k columns c with the smallest keys (h << 32) | c, compared as unsigned 64-bit
 * integers, where h is the 32-bit counter hash (mix32 of dtb_common.cuh, seed < 2^32, every operand taken mod 2^32)
 *   a = mix32((seed << 32) | s),  b = mix32((a << 32) | i),  h = mix32((b << 32) | c).
 * k == cols takes the donor row whole.  p2 and x_in are NULL exactly when k == 0 (x_in may also be given then: it gets
 * x_tgt).  p1 / p2 entries are the caller's to keep inside X.  No host synchronisation. */
int dtb_dae_swap_batch(const float* X, int cols, const int64_t* p1, const int64_t* p2, const int* step_dev,
                       const int* epoch_first_step_dev, int batch_rows, int rows, int k, unsigned long long seed,
                       float* x_in, float* x_tgt, void* stream);

/* Data-parallel exchange of the embedding gradient by rows (deepmodel.py:88-103: MirroredStrategy
 * exchanges embedding gradients as IndexedSlices too).  pack: every (b,f) reference claims its row once
 * per step (claim[row] = step); the owner MOVES the accumulated gradient row into packed[b,f,:] and zeroes
 * the table row, other references of that row write zeros.  unpack: adds one rank's packed rows into the
 * local gradient table; at most one reference per row carries data, so no atomics are needed and
 * calling it for rank 0..W-1 in order yields identical bits on every replica. */
int dtb_grad_rows_pack(const int32_t* idx, const int64_t* row_offsets, float* grad_table, int32_t* claim,
                       float* packed /* [B,F,D] */, int step, int B, int F, int D, void* stream);
int dtb_grad_rows_unpack(const int32_t* idx, const int64_t* row_offsets, const float* packed,
                         float* grad_table, int B, int F, int D, void* stream);

/* ---- CIN (layers.py:638-734), gather fused ------------------------------------------------ */
/* Shapes: F0 = F fields, D, n_layers layer sizes L[k] (host array), direct flag; H[0]=F,
 * H[k+1] = direct ? L[k] : L[k]/2 (all L[k]); K[k] = F*H[k].
 * weights: concatenation of the n_layers filters, filter k is [K[k], L[k]] row-major (the
 * reference's f_k[0]); bias: concatenation of [L[k]] or NULL.  act in {NONE, RELU}.
 * pooled[B, P] with P = direct ? sum L : sum_{k<last} L[k]/2 + L[last]  (layers.py:725-726; the
 * final Dense(1) / residual MLP is a dtb_dense_* call).
 * saved (training only, may be NULL for inference): workspace of dtb_cin_saved_bytes() holding
 * the activations backward needs. */
size_t dtb_cin_saved_bytes(int B, int F, int D, const int* layer_sizes_host, int n_layers, int direct);
size_t dtb_cin_workspace_bytes(int B, int F, int D, const int* layer_sizes_host, int n_layers,
                               int direct, int training);
int dtb_cin_fwd(const int32_t* idx, const float* table, const int64_t* row_offsets,
                const float* weights, const float* bias, float* pooled, void* saved,
                void* workspace, size_t workspace_bytes, int B, int F, int D,
                const int* layer_sizes_host, int n_layers, int direct, int act, int precision,
                int* status, void* stream);
/* d_pooled[B,P] -> grad_table += dE, d_weights/d_bias accumulate. */
int dtb_cin_bwd(const int32_t* idx, const float* table, const int64_t* row_offsets,
                const float* weights, const float* d_pooled, const void* saved, float* grad_table,
                float* d_weights, float* d_bias, void* workspace, size_t workspace_bytes, int B, int F,
                int D, const int* layer_sizes_host, int n_layers, int direct, int act, int precision,
                void* stream);
/* The same backward in two launches: phase 1 = everything that contributes to grad_table (after it the
 * embedding gradient of this op is final), phase 2 = d_weights / d_bias.  The host starts the data-parallel
 * exchange of the table gradient between the two so that it overlaps the weight-gradient kernels. */
int dtb_cin_bwd_phase(const int32_t* idx, const float* table, const int64_t* row_offsets,
                      const float* weights, const float* d_pooled, const void* saved, float* grad_table,
                      float* d_weights, float* d_bias, void* workspace, size_t workspace_bytes, int B, int F,
                      int D, const int* layer_sizes_host, int n_layers, int direct, int act, int precision,
                      int phase, void* stream);
/* precision (forward; codes 2-4 share the fused bf16x3 backward of csrc/cin_wgmma.cu, code 1 the any-shape backward):
 *   0 = auto: 2 where dtb_cin_tc_supported(), else 1;
 *   1 = the any-shape materialising formulation (outer product in HBM chunks + the bf16x3 GEMMs of csrc/dense_tc.cu);
 *   2 = fused wgmma forward (csrc/cin_wgmma.cu: embedding dim 4/8/16/32, <= 64 fields, <= 64 hidden fields and <= 128
 *       feature maps per layer), bf16x3 split: fp32-grade; 3 = the same with one bf16 pass; 4 = one pass on fp16
 *       operands scaled by exact powers of two.  Codes 2-4 return DTB_ERR_UNSUPPORTED outside the fused shapes.
 * The backward takes its own precision: code 1 after a fused forward runs the any-shape backward on that forward's
 * saved activations (both forwards save the same layout), which tests use as the reference for the fused backward. */
#define DTB_CIN_AUTO 0
#define DTB_CIN_FP32 1
#define DTB_CIN_TC_BF16X3 2
#define DTB_CIN_TC_BF16X1 3
#define DTB_CIN_TC_F16X1 4
int dtb_cin_tc_supported(int F, int D, const int* layer_sizes_host, int n_layers, int direct);
/* which of the codes 1-4 a forward + backward with `precision` runs for this shape (0 = auto is resolved) */
int dtb_cin_resolved_precision(int F, int D, const int* layer_sizes_host, int n_layers, int direct, int precision);
/* Test hook for the tensor-core path: C[128,N] = bf16(A[128,K]) @ bf16(Bmat[K,N]) on one warpgroup
 * (two m64 wgmma row blocks; N in {16, 32, 64, 128}, K <= 64 a multiple of 16), the A operand from registers
 * (a_operand_in_regs = 1) or from shared memory (0); workspace is not used and may be any non-NULL pointer. */
int dtb_tc_selftest(const float* A, const float* Bmat, float* C, void* workspace, int N, int K,
                    int a_operand_in_regs, void* stream);

/* ---- Cross (layers.py:417-436) on a dense [B,W] input ------------------------------------- */
/* x_{l+1} = x0*(x_l . w_l) + x_l + b_l ; kernels/biases [n_layers, W]; Y [B,W].
 * xw_saved [B, n_layers] keeps the per-layer scalars x_l.w_l for backward. */
int dtb_cross_fwd(const float* X, const float* kernels, const float* biases, float* Y,
                  float* xw_saved, int B, int W, int n_layers, void* stream);
size_t dtb_cross_bwd_workspace_bytes(int B, int W, int n_layers);
int dtb_cross_bwd(const float* X, const float* kernels, const float* biases, const float* xw_saved,
                  const float* dY, float* dX, float* d_kernels, float* d_biases, void* workspace,
                  size_t workspace_bytes, int B, int W, int n_layers, void* stream);

/* ---- InnerProduct / OuterProduct (layers.py:473-487, 541-581), gather fused --------------- */
/* ip[B,P] (NULL: skipped), op[B,P] (NULL: skipped); P = F(F-1)/2 pairs (i<j) row-major.
 * kernel_type 0 mat [D,P,D], 1 vec [P,D], 2 num [P,1].  Both refuse P > 1024 (F >= 46) with
 * DTB_ERR_UNSUPPORTED. */
int dtb_pnn_fwd(const int32_t* idx, const float* table, const int64_t* row_offsets,
                const float* op_kernel, float* ip, float* op, int B, int F, int D, int kernel_type,
                int* status, void* stream);
int dtb_pnn_bwd(const int32_t* idx, const float* table, const int64_t* row_offsets,
                const float* op_kernel, const float* d_ip, const float* d_op, float* grad_table,
                float* d_op_kernel, int B, int F, int D, int kernel_type, void* stream);

/* ---- AFM (layers.py:742-812; afm_nets deepnets.py:99-107), gather fused ---------------------- */
/* pooled[B,D] = sum_p softmax_p(act((e_i*e_j) att_kernel + att_bias) . projection_h) (e_i*e_j) over
 * the F(F-1)/2 field pairs in itertools.combinations order (what AFM.call hands to its Dropout and
 * Dense(1, use_bias=False)).  att_kernel [D,H] row-major, att_bias [H], projection_h [H];
 * act = DTB_ACT_NONE | DTB_ACT_RELU.  D in {4,8,16,32}, H <= 32, else DTB_ERR_UNSUPPORTED.
 * Backward: adds into grad_table (same layout as the table) and into d_att_kernel / d_att_bias /
 * d_projection_h (caller zero-fills); workspace of dtb_afm_workspace_bytes(B,F,D,H) bytes. */
size_t dtb_afm_workspace_bytes(int B, int F, int D, int H);
int dtb_afm_fwd(const int32_t* idx, const float* table, const int64_t* row_offsets,
                const float* att_kernel, const float* att_bias, const float* projection_h,
                float* pooled, int B, int F, int D, int H, int act, int* status, void* stream);
int dtb_afm_bwd(const int32_t* idx, const float* table, const int64_t* row_offsets,
                const float* att_kernel, const float* att_bias, const float* projection_h,
                const float* d_pooled, float* grad_table, float* d_att_kernel, float* d_att_bias,
                float* d_projection_h, void* workspace, size_t workspace_bytes, int B, int F, int D,
                int H, int act, void* stream);

/* ---- FiBiNet: SENET + BilinearInteraction (layers.py:245-382; fibi_nets deepnets.py:344-371) -- */
/* On a dense block X [B,F,D] (the concatenated embeddings or their SENET re-weighting).
 * Bilinear: out[b,p,:] = (x_i W_s) * x_j over the F(F-1)/2 pairs in itertools.combinations order;
 * W [n_w,D,D] row-major, bilinear_type 0 field_all (n_w = 1, s = 0) | 1 field_each (n_w = F-1, s = i)
 * | 2 field_interaction (n_w = pairs, s = p).  Backward: dX [B,F,D] overwritten (may be NULL), dW
 * accumulated (caller zero-fills).  D in {4,8,16,32}, else DTB_ERR_UNSUPPORTED.
 * SENET: Z[b,f] = mean (pooling_op 0) or max (1) over d; V = X * A[:,:,None]; the two Dense layers
 * between Z and A are dtb_dense_* calls.  Max-pool gradient: ties share it (tf.reduce_max). */
int dtb_bilinear_fwd(const float* X, const float* W, float* out, int B, int F, int D,
                     int bilinear_type, void* stream);
int dtb_bilinear_bwd(const float* X, const float* W, const float* d_out, float* dX, float* dW, int B,
                     int F, int D, int bilinear_type, void* stream);
int dtb_senet_pool_fwd(const float* X, float* Z, int B, int F, int D, int pooling_op, void* stream);
int dtb_senet_pool_bwd(const float* X, const float* Z, const float* dZ, float* dX, int B, int F,
                       int D, int pooling_op, void* stream);
int dtb_senet_scale_fwd(const float* X, const float* A, float* V, int B, int F, int D, void* stream);
int dtb_senet_scale_bwd(const float* X, const float* A, const float* dV, float* dX, float* dA, int B,
                        int F, int D, void* stream);

/* ---- FGCNN (layers.py:161-242; fg_nets deepnets.py:227-261) -------------------------------- */
/* Channels-last block X [B,H,W,Cin] (H = fields, W = embedding width).  Convolution along H only:
 * Y[b,h,w,co] = act(bias[co] + sum_{t,ci} X[b,h+t-pad,w,ci] kernel[t,ci,co]), kernel [kh,1,Cin,Cout]
 * as Keras stores it, TensorFlow 'same' padding (pad = (kh-1)/2 in front), act = NONE | RELU | TANH.
 * Cin, Cout <= 32, kh <= 8, else DTB_ERR_UNSUPPORTED.  Backward: dX overwritten (may be NULL),
 * d_kernel / d_bias accumulated (caller zero-fills; d_bias may be NULL).
 * Max pooling along H: windows of `pool` rows, stride `pool`, 'same' padding; Y [B,ceil(H/pool),WC];
 * the gradient goes to the first maximum of a window; dX [B,H,WC] overwritten.
 * The recombination layer is dtb_dense_fwd/bwd with DTB_ACT_TANH. */
int dtb_conv_fields_fwd(const float* X, const float* kernel, const float* bias, float* Y, int B,
                        int H, int W, int Cin, int Cout, int kh, int act, void* stream);
int dtb_conv_fields_bwd(const float* X, const float* kernel, const float* Y, const float* dY,
                        float* dX, float* d_kernel, float* d_bias, int B, int H, int W, int Cin,
                        int Cout, int kh, int act, void* stream);
int dtb_maxpool_fields_fwd(const float* X, float* Y, int B, int H, int WC, int pool, void* stream);
int dtb_maxpool_fields_bwd(const float* X, const float* dY, float* dX, int B, int H, int WC, int pool,
                           void* stream);

/* ---- MultiheadAttention core (layers.py:129-150), between the projections and the BN ------- */
/* qkvr [B, F, 4*D]: the four relu(Dense) projections of each field row, concatenated [Q|K|V|R]
 * (one dtb_dense_fwd with the four kernels side by side).  Y[B,F,D] = relu(concat_h softmax(Q_h
 * K_h^T / sqrt(D/heads)) V_h + R).  Backward: d_qkvr [B,F,4*D] (overwritten); with mask_relu_inputs
 * the result is zeroed where qkvr is zero, i.e. it is the gradient of the PRE-relu projections (the
 * caller then runs dtb_dense_bwd with act = linear and skips the activation-gradient pass). */
int dtb_attention_core_fwd(const float* qkvr, float* Y, int B, int F, int D, int heads,
                           int use_residual, void* stream);
int dtb_attention_core_bwd(const float* qkvr, const float* Y, const float* dY, float* d_qkvr, int B,
                           int F, int D, int heads, int use_residual, int mask_relu_inputs,
                           void* stream);
/* The same with dropout on the softmax weights (layers.py:111,141; training only): weight (b, h, q, k) -- batch row,
 * head, query field, key field -- is kept with probability 1 - rate and scaled by 1 / (1 - rate).  The mask is that of
 * dtb_dropout at element index ((b * heads + h) * F + q) * F + k, with b counted from row_offset (a slice of a batch
 * that starts at row r and passes row_offset = r draws the bits of the whole batch).  The backward regenerates it:
 * nothing is stored.  The seed is *seed_dev when seed_dev is not NULL (CUDA-graph form), else `seed`.  rate = 0 runs
 * the kernels of dtb_attention_core_fwd/bwd. */
int dtb_attention_core_dropout_fwd(const float* qkvr, float* Y, int B, int F, int D, int heads, int use_residual,
                                   float rate, unsigned long long seed, const unsigned long long* seed_dev,
                                   long long row_offset, void* stream);
int dtb_attention_core_dropout_bwd(const float* qkvr, const float* Y, const float* dY, float* d_qkvr, int B, int F,
                                   int D, int heads, int use_residual, int mask_relu_inputs, float rate,
                                   unsigned long long seed, const unsigned long long* seed_dev, long long row_offset,
                                   void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DEEPTABLES_B200_H_ */
