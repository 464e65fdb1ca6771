/*
 * rnnt.h — C-ABI of the H100-native (sm_90a) RNN-Transducer loss (libwarprnnt.so).
 *
 * Binary drop-in for the reference library's interface: the same five exported symbols, the
 * same enum values and the same 32-byte by-value options struct, so anything that links the
 * reference (its PyTorch / TensorFlow bindings, tests/*.cu) links this instead.  Each
 * declaration names the reference interface it replaces (paths relative to the reference
 * checkout).  Only the CUDA device path exists here: there is no CPU implementation behind
 * this ABI (see `loc` below).
 *
 * All tensors are dense, row-major, no padding between dimensions:
 *   activations / gradients  [minibatch, maxT, maxU, alphabet_size]
 *   flat_labels              [minibatch, maxU - 1]   (padded to maxU-1 per utterance)
 *   label_lengths, input_lengths, costs  [minibatch]
 */
#ifndef B200_RNNT_H_
#define B200_RNNT_H_

#ifdef __cplusplus
#include <cstddef>
extern "C" {
#else
#include <stdbool.h>
#include <stddef.h>
#endif

/* Opaque CUDA stream handle (same forward declaration trick as reference include/rnnt.h:14). */
typedef struct CUstream_st* CUstream;

/* Return codes — values fixed by reference include/rnnt.h:16-22. */
typedef enum {
    RNNT_STATUS_SUCCESS = 0,
    RNNT_STATUS_MEMOPS_FAILED = 1,    /* a cudaMemcpy/cudaMemset-class call failed            */
    RNNT_STATUS_INVALID_VALUE = 2,    /* null pointer, non-positive dimension, unknown loc    */
    RNNT_STATUS_EXECUTION_FAILED = 3, /* kernel launch/execution error, or loc == RNNT_CPU    */
    RNNT_STATUS_UNKNOWN_ERROR = 4
} rnntStatus_t;

/* Replaces reference include/rnnt.h:25 (src/rnnt_entrypoint.cpp:14-16).  Returns 1: the
 * reference's tests refuse to run against any other value (tests/test_cpu.cpp:382-385). */
int get_warprnnt_version(void);

/* Replaces reference include/rnnt.h:31 (src/rnnt_entrypoint.cpp:18-35).  Static strings. */
const char* rnntGetStatusString(rnntStatus_t status);

/* Reference include/rnnt.h:33-36. */
typedef enum {
    RNNT_CPU = 0, /* not available in this library: compute calls return EXECUTION_FAILED */
    RNNT_GPU = 1
} rnntComputeLocation;

/*
 * Options, passed BY VALUE.  Layout fixed by reference include/rnnt.h:43-64
 * (x86-64: 32 bytes, offsets 0/4/8/16/20/24/28).  Zero-initialise before filling.
 */
struct rnntOptions {
    rnntComputeLocation loc;  /* must be RNNT_GPU                                              */
    unsigned int num_threads; /* accepted and ignored (no host threading on the device path)  */
    CUstream stream;          /* all device work is enqueued here                              */
    int blank_label;          /* index of the blank symbol                                     */
    int maxT;                 /* time extent of the activation tensor                          */
    int maxU;                 /* label extent of the activation tensor (max label length + 1) */
    bool batch_first;         /* ignored, as the reference's GPU path ignores it
                                 (include/detail/gpu_rnnt_kernel.h:7 always indexes [N,T,U,V]; the
                                 reference's tests/test_gpu.cu:42-50 leave it false with [N,T,U,V]
                                 data).  For [T,U,N,V] tensors use rnnt_b200_loss_async_layout. */
};
#ifndef __cplusplus
typedef struct rnntOptions rnntOptions;
#endif

/*
 * RNN-T negative log-likelihood per utterance and, optionally, its gradient with respect to
 * the raw logits.  Replaces reference include/rnnt.h:104-113 (src/rnnt_entrypoint.cpp:38-93)
 * for loc == RNNT_GPU, with the GPU path's conventions (include/detail/gpu_rnnt.h:82-215):
 *
 *   activations   DEVICE, raw (un-normalised) logits; log-softmax over the last axis is
 *                 computed inside.
 *   gradients     DEVICE, same shape, or NULL for loss only.  When non-NULL every element is
 *                 defined on return: d cost[b] / d logit for valid cells, 0 for padded cells
 *                 (t >= input_lengths[b] or u > label_lengths[b]).  Not scaled or reduced.
 *   flat_labels, label_lengths, input_lengths
 *                 DEVICE pointers, as every caller of the reference's GPU path passes them
 *                 (tests/test_gpu.cu:54-59); HOST pointers are also accepted (detected with
 *                 cudaPointerGetAttributes and staged through the workspace).
 *   costs         HOST pointer (as the reference: D2H copy inside the call,
 *                 include/detail/gpu_rnnt.h:209-213); a DEVICE pointer is accepted too.
 *   workspace     DEVICE scratch of get_workspace_size(..., gpu=true, ...) bytes.
 *
 * The call returns after the stream has finished (costs are readable on return), like the
 * reference.  Errors are reported by return code only; nothing is thrown across the ABI.
 * Limits: minibatch*maxT*maxU < 2^31 cells (elements are indexed with 64 bits).
 */
rnntStatus_t compute_rnnt_loss(const float* const activations, float* gradients,
                               const int* const flat_labels, const int* const label_lengths,
                               const int* const input_lengths, int alphabet_size, int minibatch,
                               float* costs, void* workspace, struct rnntOptions options);

/* Double-precision twin.  Replaces reference include/rnnt.h:115-124
 * (src/rnnt_entrypoint.cpp:130-185). */
rnntStatus_t compute_rnnt_loss_fp64(const double* const activations, double* gradients,
                                    const int* const flat_labels,
                                    const int* const label_lengths,
                                    const int* const input_lengths, int alphabet_size,
                                    int minibatch, double* costs, void* workspace,
                                    struct rnntOptions options);

/*
 * Scratch size in bytes.  Replaces reference include/rnnt.h:139-143
 * (src/rnnt_entrypoint.cpp:96-128): same signature, same INVALID_VALUE rule for non-positive
 * extents.  The byte count differs from the reference's (this library keeps a different
 * lattice: see DESIGN.md "HBM layout"); callers always size through this function.
 * gpu == false returns the reference's CPU formula for source compatibility only.
 */
#ifdef __cplusplus
rnntStatus_t get_workspace_size(int maxT, int maxU, int minibatch, bool gpu, size_t* size_bytes,
                                size_t dtype_size = sizeof(float));
#else
rnntStatus_t get_workspace_size(int maxT, int maxU, int minibatch, bool gpu, size_t* size_bytes,
                                size_t dtype_size);
#endif

/* Same function under the name BASELINE.json's north_star uses (the reference has no such
 * symbol; exported so either spelling links). */
rnntStatus_t get_rnnt_workspace_size(int maxT, int maxU, int minibatch, bool gpu,
                                     size_t* size_bytes, size_t dtype_size);

/* ---------------------------------------------------------------------------------------
 * Extensions (no reference counterpart).  Used by the warprnnt_pytorch operator to drop
 * the framework-side passes SURVEY.md §8(f).1 lists, and by bench.py for device timing.
 * ------------------------------------------------------------------------------------- */

/*
 * Asynchronous variant: identical computation, but
 *   - costs_device [minibatch] is written on the DEVICE and the call does NOT synchronise;
 *   - gradients are multiplied by grad_scale (pass 1.0f for the plain gradient): folds the
 *     'mean' 1/N of warprnnt_pytorch/__init__.py:38-40 into the write-back.
 * flat_labels/label_lengths/input_lengths must be DEVICE pointers here.
 */
rnntStatus_t compute_rnnt_loss_async(const float* const activations, float* gradients,
                                     const int* const flat_labels,
                                     const int* const label_lengths,
                                     const int* const input_lengths, int alphabet_size,
                                     int minibatch, float* costs_device, float grad_scale,
                                     void* workspace, struct rnntOptions options);

rnntStatus_t compute_rnnt_loss_async_fp64(const double* const activations, double* gradients,
                                          const int* const flat_labels,
                                          const int* const label_lengths,
                                          const int* const input_lengths, int alphabet_size,
                                          int minibatch, double* costs_device, double grad_scale,
                                          void* workspace, struct rnntOptions options);

/*
 * Training-step split used by warprnnt_pytorch (SURVEY.md §8(f).1): the gradient pass runs in
 * autograd's backward with the upstream gradient folded in, so the framework never makes a
 * separate pass over the [N,T,U,V] tensor (the reference multiplies it in place afterwards,
 * pytorch_binding/warprnnt_pytorch/__init__.py:47-50).  All pointers DEVICE, no synchronisation.
 *
 *   rnnt_b200_forward   log-softmax statistics + alpha (+ beta when prepare_backward != 0) lattices
 *                       into `workspace`, costs_device[minibatch] = -log-likelihood.
 *   rnnt_b200_backward  gradient pass only, from the SAME workspace and the same activations:
 *                       gradients[b,...] = grad_scale * grad_costs_device[b] * d cost[b]/d logits
 *                       (grad_costs_device may be NULL = all ones).  Zeros on padding.
 */
rnntStatus_t rnnt_b200_forward(const float* const activations, const int* const flat_labels,
                               const int* const label_lengths, const int* const input_lengths,
                               int alphabet_size, int minibatch, float* costs_device,
                               int prepare_backward, void* workspace, struct rnntOptions options);
rnntStatus_t rnnt_b200_forward_fp64(const double* const activations, const int* const flat_labels,
                                    const int* const label_lengths, const int* const input_lengths,
                                    int alphabet_size, int minibatch, double* costs_device,
                                    int prepare_backward, void* workspace, struct rnntOptions options);
rnntStatus_t rnnt_b200_backward(const float* const activations, float* gradients,
                                const int* const flat_labels, const int* const label_lengths,
                                const int* const input_lengths, int alphabet_size, int minibatch,
                                const float* grad_costs_device, float grad_scale, void* workspace,
                                struct rnntOptions options);
rnntStatus_t rnnt_b200_backward_fp64(const double* const activations, double* gradients,
                                     const int* const flat_labels, const int* const label_lengths,
                                     const int* const input_lengths, int alphabet_size,
                                     int minibatch, const double* grad_costs_device,
                                     double grad_scale, void* workspace, struct rnntOptions options);

/*
 * Explicit activation layout (SURVEY.md §8(f).4).  RNNT_B200_LAYOUT_TUNV takes activations and
 * gradients as [maxT, maxU, minibatch, alphabet_size] - the layout the reference's CPU path indexes
 * when batch_first == false (include/detail/cpu_rnnt.h:139-144) and that its GPU path never
 * implemented.  Labels, lengths and costs stay [minibatch, ...].  Otherwise identical to
 * compute_rnnt_loss_async (all pointers DEVICE, no synchronisation).
 */
enum { RNNT_B200_LAYOUT_NTUV = 0, RNNT_B200_LAYOUT_TUNV = 1 };
rnntStatus_t rnnt_b200_loss_async_layout(int layout, const float* activations, float* gradients,
                                         const int* flat_labels, const int* label_lengths,
                                         const int* input_lengths, int alphabet_size, int minibatch,
                                         float* costs_device, float grad_scale, void* workspace,
                                         struct rnntOptions options);
rnntStatus_t rnnt_b200_loss_async_layout_fp64(int layout, const double* activations, double* gradients,
                                              const int* flat_labels, const int* label_lengths,
                                              const int* input_lengths, int alphabet_size, int minibatch,
                                              double* costs_device, double grad_scale, void* workspace,
                                              struct rnntOptions options);

/*
 * 16-bit storage variants (SURVEY.md §8(f).3): logits and gradients in bf16 or fp16, arithmetic,
 * lattice and costs in fp32; 6 B per logit instead of 12.  Same semantics as the async / split
 * entries above; workspace sized with dtype_size = sizeof(float).  dtype: RNNT_B200_BF16 / _FP16.
 * The 16-B fast path needs alphabet_size % 8 == 0 and 16-B aligned tensors (else element-wise).
 */
enum { RNNT_B200_BF16 = 1, RNNT_B200_FP16 = 2 };
rnntStatus_t rnnt_b200_loss_async_16(int dtype, const void* activations, void* gradients,
                                     const int* flat_labels, const int* label_lengths,
                                     const int* input_lengths, int alphabet_size, int minibatch,
                                     float* costs_device, float grad_scale, void* workspace,
                                     struct rnntOptions options);
rnntStatus_t rnnt_b200_forward_16(int dtype, const void* activations, const int* flat_labels,
                                  const int* label_lengths, const int* input_lengths,
                                  int alphabet_size, int minibatch, float* costs_device,
                                  int prepare_backward, void* workspace, struct rnntOptions options);
rnntStatus_t rnnt_b200_backward_16(int dtype, const void* activations, void* gradients,
                                   const int* flat_labels, const int* label_lengths,
                                   const int* input_lengths, int alphabet_size, int minibatch,
                                   const float* grad_costs_device, float grad_scale, void* workspace,
                                   struct rnntOptions options);

/*
 * Gradient regularisers, passed BY VALUE to the *_ex entries below.  Zero-initialised = both off, and the
 * *_ex entries then launch exactly the kernels of their plain counterparts.  Both act on the gradient
 * only: costs are the plain negative log-likelihood for every setting, bitwise identical to the costs
 * without options (other implementations differ on what they report here).
 *
 *   fastemit_lambda  FastEmit (Yu et al., ICASSP 2021): the gradient with respect to the label
 *                    log-probabilities is scaled by (1 + lambda).  Per valid cell, with p = softmax(logits),
 *                    e_b / e_y the blank / label transition occupancies and occ = e_b + e_y:
 *                      g_k = p_k (occ + lambda e_y) - [k = blank] e_b - [k = y_u] (1 + lambda) e_y
 *                    This is the gradient of -ll - lambda sum_{t,u} sg[e_y] log p_y (sg = stop-gradient),
 *                    NOT the gradient of the returned cost.  Must be finite and >= 0; 0 = off.
 *   clamp            c > 0: every element of the per-utterance gradient is clipped to [-c, c] after the
 *                    blank / label terms and before grad_scale * grad_costs[b]; c <= 0 = off.  Not NaN.
 * Invalid values return RNNT_STATUS_INVALID_VALUE before any device access.
 */
struct rnntGradOptions {
    float fastemit_lambda;   /* float for every storage type: fp64 calls see the options rounded to float */
    float clamp;
};
#ifndef __cplusplus
typedef struct rnntGradOptions rnntGradOptions;
#endif

/* Storage type codes of the *_ex entries (RNNT_B200_BF16 / _FP16 above are the same codes). */
enum { RNNT_B200_FP32 = 0, RNNT_B200_FP64 = 3 };

/*
 * Full call with gradient options: dtype RNNT_B200_FP32 / _FP64 / _BF16 / _FP16, layout RNNT_B200_LAYOUT_NTUV
 * or (fp32 / fp64 only) _TUNV.  Otherwise compute_rnnt_loss_async(_fp64), rnnt_b200_loss_async_layout(_fp64)
 * and rnnt_b200_loss_async_16: costs_device is double* for fp64 and float* otherwise, grad_scale is rounded
 * to the arithmetic type.  Unsupported (dtype, layout) pairs return RNNT_STATUS_INVALID_VALUE.
 */
rnntStatus_t rnnt_b200_loss_async_ex(int dtype, int layout, const void* activations, void* gradients,
                                     const int* flat_labels, const int* label_lengths,
                                     const int* input_lengths, int alphabet_size, int minibatch,
                                     void* costs_device, double grad_scale, struct rnntGradOptions grad_options,
                                     void* workspace, struct rnntOptions options);
/* Backward half of the training-step split with gradient options, for all four storage types
 * (rnnt_b200_backward / _fp64 / _16; grad_costs_device is double* for fp64, float* otherwise). */
rnntStatus_t rnnt_b200_backward_ex(int dtype, const void* activations, void* gradients,
                                   const int* flat_labels, const int* label_lengths,
                                   const int* input_lengths, int alphabet_size, int minibatch,
                                   const void* grad_costs_device, double grad_scale,
                                   struct rnntGradOptions grad_options, void* workspace,
                                   struct rnntOptions options);

/*
 * Additive joint network, logits never materialised (SURVEY.md §8(f).2): for models whose logits
 * are  h[b,t,u,k] = trans[b,t,k] + pred[b,u,k]  (how the reference's own timing script builds them,
 * pytorch_binding/test/test_time.py:73).  trans [minibatch,maxT,V], pred [minibatch,maxU,V];
 * outputs costs_device [minibatch] and, when both gradient pointers are non-NULL,
 * grad_trans = grad_scale * d cost/d trans, grad_pred likewise (docs/rnnt_notes.tex:147-153).
 * All pointers DEVICE, fp32, no synchronisation.  Workspace from rnnt_b200_add_joint_workspace_size.
 * HBM traffic is O(N (T+U) V) instead of O(N T U V).
 * Padded rows (trans frames t >= input_lengths[b], pred rows u > label_lengths[b]) are not read, so they may hold
 * anything, NaN and inf included, and get a zero gradient.
 */
rnntStatus_t rnnt_b200_add_joint_loss(const float* trans, const float* pred, float* grad_trans,
                                      float* grad_pred, const int* flat_labels,
                                      const int* label_lengths, const int* input_lengths,
                                      int alphabet_size, int minibatch, float* costs_device,
                                      float grad_scale, void* workspace, struct rnntOptions options);
rnntStatus_t rnnt_b200_add_joint_workspace_size(int maxT, int maxU, int minibatch, int alphabet_size,
                                                size_t* size_bytes);
/* Training-step split of the same (see rnnt_b200_forward / rnnt_b200_backward): the backward half
 * folds grad_costs_device[b] * grad_scale into the factor gradients. */
rnntStatus_t rnnt_b200_add_joint_forward(const float* trans, const float* pred, const int* flat_labels,
                                         const int* label_lengths, const int* input_lengths,
                                         int alphabet_size, int minibatch, float* costs_device,
                                         int prepare_backward, void* workspace, struct rnntOptions options);
rnntStatus_t rnnt_b200_add_joint_backward(const float* trans, const float* pred, float* grad_trans,
                                          float* grad_pred, const int* flat_labels,
                                          const int* label_lengths, const int* input_lengths,
                                          int alphabet_size, int minibatch, const float* grad_costs_device,
                                          float grad_scale, void* workspace, struct rnntOptions options);
/* The same with gradient options.  FastEmit only: the factor gradients never pass through per-logit values,
 * so any nonzero clamp returns RNNT_STATUS_INVALID_VALUE. */
rnntStatus_t rnnt_b200_add_joint_backward_ex(const float* trans, const float* pred, float* grad_trans,
                                             float* grad_pred, const int* flat_labels,
                                             const int* label_lengths, const int* input_lengths,
                                             int alphabet_size, int minibatch, const float* grad_costs_device,
                                             float grad_scale, struct rnntGradOptions grad_options,
                                             void* workspace, struct rnntOptions options);

/*
 * Smoothed additive joint (DESIGN.md §9; k2's rnnt_loss_smoothed): the lattice of rnnt_b200_add_joint_forward, with
 * each blank / label factor of a valid cell (t, u), k in {blank, y_u}, replaced by
 *     lp(t,u,k) = c (f[t,k] + g[u,k] - lse(t,u)) + lm_only_scale (g[u,k] - Lg(u)) + am_only_scale (f[t,k] + log ug[k] - La(t))
 * with c = 1 - lm_only_scale - am_only_scale; a term whose scale is exactly 0 is left out.
 *   Lg(u) = log sum_v exp(g[u,v])                          the lm-only (per label position) normaliser
 *   ug[v] = (1/M) sum_{b, u < U_b} softmax(g[b,u])[v] + FLT_MIN,  M = sum_b U_b   (valid rows of the whole batch)
 *   La(t) = log sum_v exp(f[t,v]) ug[v]                    the am-only normaliser
 * The gradients are the exact gradients of the returned cost in trans and pred, including the path through ug: with
 * am_only_scale > 0 one utterance's grad_pred depends on the whole batch.  FastEmit scales the gradient of each
 * (interpolated) label factor by 1 + fastemit_lambda.  Padded rows of trans and pred are not read (they may hold NaN
 * or inf) and get a zero gradient, as in the plain joint.
 * Valid scales are finite, >= 0, with lm_only_scale + am_only_scale <= 1 + 2^-23 (one float32 ulp of slack, so
 * that pairs meant to sum to 1, such as (0.6f, 0.4f), are accepted; c is then 0); anything else returns
 * RNNT_STATUS_INVALID_VALUE before any device access.  Both scales 0 is the plain joint, bitwise.
 * The smoothed workspace is the plain joint's followed by the smoothing sections, so rnnt_b200_add_joint_prune_ranges
 * works on it as is (the windows of the smoothed lattice).  The backward half must get the scales its forward got.
 */
struct rnntSmoothOptions {
    float lm_only_scale;
    float am_only_scale;
};
#ifndef __cplusplus
typedef struct rnntSmoothOptions rnntSmoothOptions;
#endif
rnntStatus_t rnnt_b200_add_joint_smoothed_workspace_size(int maxT, int maxU, int minibatch, int alphabet_size,
                                                         size_t* size_bytes);
rnntStatus_t rnnt_b200_add_joint_smoothed_forward(const float* trans, const float* pred, const int* flat_labels,
                                                  const int* label_lengths, const int* input_lengths,
                                                  int alphabet_size, int minibatch, float* costs_device,
                                                  int prepare_backward, struct rnntSmoothOptions smooth,
                                                  void* workspace, struct rnntOptions options);
/* Gradient options as rnnt_b200_add_joint_backward_ex (FastEmit only; a nonzero clamp is INVALID_VALUE). */
rnntStatus_t rnnt_b200_add_joint_smoothed_backward(const float* trans, const float* pred, float* grad_trans,
                                                   float* grad_pred, const int* flat_labels,
                                                   const int* label_lengths, const int* input_lengths,
                                                   int alphabet_size, int minibatch, const float* grad_costs_device,
                                                   float grad_scale, struct rnntGradOptions grad_options,
                                                   struct rnntSmoothOptions smooth, void* workspace,
                                                   struct rnntOptions options);

/*
 * Pruned RNN-T loss (Kuang et al., "Pruned RNN-T for fast, memory-efficient ASR training", Interspeech 2022).
 * activations [minibatch, maxT, s_range, alphabet_size]: row (b, t, s) holds the logits of lattice cell
 * (t, u = ranges[b*maxT + t] + s); ranges [minibatch, maxT] int32 window starts (any values); labels, lengths and
 * costs as rnnt_b200_loss_async_ex; options.maxU is the full lattice width (max label length + 1).
 * The loss is the RNN-T loss over the paths that only visit cells covered by a row of their frame, on the dense
 * [T_b, U_b] lattice: a cell with no row has log-zero blank and label factors, a covered cell takes its blank logit
 * and, for u < U_b - 1, the logit of y_u from its own row.  A row with t >= T_b, u < 0 or u >= U_b is padding: not
 * read by the forward, zero gradient.  The gradient of a valid row is the dense formula at (b, t, u).  An utterance
 * with no surviving path costs +inf and gets an all-zero gradient.  With s_range = maxU and ranges == 0 this is
 * exactly rnnt_b200_loss_async_ex, bitwise.
 * dtype: RNNT_B200_FP32 / _FP64 / _BF16 / _FP16 (costs double* for fp64, float* otherwise); layout must be
 * RNNT_B200_LAYOUT_NTUV; s_range >= 1; minibatch * maxT * s_range < 2^31; ranges a DEVICE pointer.  The gradient
 * options are those of rnnt_b200_loss_async_ex.  Workspace from rnnt_b200_pruned_workspace_size.
 */
rnntStatus_t rnnt_b200_pruned_workspace_size(int maxT, int maxU, int s_range, int minibatch, size_t dtype_size,
                                             size_t* size_bytes);
rnntStatus_t rnnt_b200_pruned_loss_async_ex(int dtype, int layout, const void* activations, void* gradients,
                                            const int* ranges, int s_range, const int* flat_labels,
                                            const int* label_lengths, const int* input_lengths, int alphabet_size,
                                            int minibatch, void* costs_device, double grad_scale,
                                            struct rnntGradOptions grad_options, void* workspace,
                                            struct rnntOptions options);
/* Training-step split of the same (rnnt_b200_forward / rnnt_b200_backward_ex); the backward half reads the
 * lattices the forward left in `workspace` and must get the same ranges. */
rnntStatus_t rnnt_b200_pruned_forward(int dtype, const void* activations, const int* ranges, int s_range,
                                      const int* flat_labels, const int* label_lengths, const int* input_lengths,
                                      int alphabet_size, int minibatch, void* costs_device, int prepare_backward,
                                      void* workspace, struct rnntOptions options);
rnntStatus_t rnnt_b200_pruned_backward_ex(int dtype, const void* activations, void* gradients, const int* ranges,
                                          int s_range, const int* flat_labels, const int* label_lengths,
                                          const int* input_lengths, int alphabet_size, int minibatch,
                                          const void* grad_costs_device, double grad_scale,
                                          struct rnntGradOptions grad_options, void* workspace,
                                          struct rnntOptions options);

/*
 * Pruning ranges from the additive joint's lattice: call after rnnt_b200_add_joint_forward with
 * prepare_backward = 1 (or a full rnnt_b200_add_joint_loss with gradients) on the same workspace, stream and
 * options.  Writes ranges [minibatch, options.maxT] (DEVICE int32).  Per utterance, with R = s_range >= 2 and
 * E = max(U_b - R, 0), for cell (t,u)
 *   e_b(t,u) = exp(alpha(t,u) + lp_blank(t,u) + beta(t+1,u) - ll)      (blank occupancy)
 *   e_y(t,u) = exp(alpha(t,u) + lp_y(t,u) + beta(t,u+1) - ll)          (label occupancy)
 *   1. For 0 < t < T_b - 1, s[t] is the smallest a in [0, E] maximising
 *      sum_{u=a}^{min(a+R,U_b)-1} e_b(t,u) - [a>0] e_y(t,a-1).  This is k2's criterion.
 *   2. Set s[0] = 0.  If T_b > 1, set s[T_b-1] = E.  For t >= T_b, set s[t] = E.
 *   3. Sweep once, for t = T_b-2 down to 0: s[t] = min(max(s[t], s[t+1] - (R-1)), s[t+1]).
 * After the sweep the windows are non-decreasing, consecutive windows overlap (no label is skipped), the last frame
 * covers U_b - 1 when T_b > 1, and, for T_b > 1, s[0] == 0 leaves a path while an utterance without one
 * (E > (T_b-1)(R-1)) ends with s[0] > 0.  A path can still be lost when frame 1's best window starts beyond R - 1
 * (DESIGN.md §8); the pruned loss then reports +inf for that utterance.
 * Returns RNNT_STATUS_INVALID_VALUE for s_range < 2, NULL pointers, or extents the joint does not accept.
 */
rnntStatus_t rnnt_b200_add_joint_prune_ranges(const int* label_lengths, const int* input_lengths, int minibatch,
                                              int s_range, int* ranges, const void* workspace,
                                              struct rnntOptions options);

/*
 * Lattice options, passed BY VALUE to the *_lat entries below.  Unlike rnntGradOptions they change the lattice, so
 * they change the cost as well as the gradient.  Zero-initialised = off, and the *_lat entries then launch exactly
 * the kernels of the entries without them and compute the same results, bitwise.
 *
 *   delay_penalty  lambda of the delay-penalised transducer (Kang et al., "Delay-penalized transducer for
 *                  low-latency streaming ASR", ICASSP 2023; k2's delay_penalty).  With T_b the frame count of
 *                  utterance b after the usual clamp into [1, maxT], every valid cell (t, u) with a label
 *                  transition (u < U_b - 1) gets
 *                      lp_y(t,u) <- lp_y(t,u) + lambda ((T_b - 1)/2 - t)
 *                  and nothing else changes: blank factors are unchanged, the cost is -log of the sum over all paths
 *                  of the penalised factors (so it includes the penalty and can be negative), and the gradient is the
 *                  exact gradient of that cost.  A path's log-score gains lambda sum_labels ((T_b - 1)/2 - t_emit),
 *                  which favours emitting labels early.  Pruned loss: the same rule on the covered cells; uncovered
 *                  cells stay log zero.  Additive joint: the penalty is added after the smoothing interpolation.
 *                  With FastEmit, the surrogate stays -fastemit_lambda sum sg[e_y] log p_y, with e_y the label
 *                  occupancy of the penalised lattice and p_y the unpenalised softmax probability; clamp is unchanged.
 *                  Must be finite and >= 0 (a negative value is rejected, where k2 ignores it); 0 = off.
 * Invalid values return RNNT_STATUS_INVALID_VALUE before any device access.  Workspace sizes do not change.
 */
struct rnntLatticeOptions {
    float delay_penalty;   /* float for every storage type, as rnntGradOptions */
};
#ifndef __cplusplus
typedef struct rnntLatticeOptions rnntLatticeOptions;
#endif

/* rnnt_b200_loss_async_ex with lattice options (dtype, layout, costs, grad_scale and gradient options as there). */
rnntStatus_t rnnt_b200_loss_async_lat(int dtype, int layout, const void* activations, void* gradients,
                                      const int* flat_labels, const int* label_lengths,
                                      const int* input_lengths, int alphabet_size, int minibatch,
                                      void* costs_device, double grad_scale, struct rnntGradOptions grad_options,
                                      struct rnntLatticeOptions lattice_options, void* workspace,
                                      struct rnntOptions options);
/* Training-step split of the same for all four storage types (costs_device / grad_costs_device are double* for
 * fp64, float* otherwise).  The backward half's pass over the logits needs the penalty again: it must get the
 * lattice options its forward got, as it must get the same workspace. */
rnntStatus_t rnnt_b200_forward_lat(int dtype, const void* activations, const int* flat_labels,
                                   const int* label_lengths, const int* input_lengths, int alphabet_size,
                                   int minibatch, void* costs_device, int prepare_backward,
                                   struct rnntLatticeOptions lattice_options, void* workspace,
                                   struct rnntOptions options);
rnntStatus_t rnnt_b200_backward_lat(int dtype, const void* activations, void* gradients,
                                    const int* flat_labels, const int* label_lengths,
                                    const int* input_lengths, int alphabet_size, int minibatch,
                                    const void* grad_costs_device, double grad_scale,
                                    struct rnntGradOptions grad_options, struct rnntLatticeOptions lattice_options,
                                    void* workspace, struct rnntOptions options);
/* The pruned loss with lattice options: rnnt_b200_pruned_loss_async_ex, _forward and _backward_ex plus
 * lattice_options; the backward half must get the options (and the ranges) its forward got. */
rnntStatus_t rnnt_b200_pruned_loss_async_lat(int dtype, int layout, const void* activations, void* gradients,
                                             const int* ranges, int s_range, const int* flat_labels,
                                             const int* label_lengths, const int* input_lengths, int alphabet_size,
                                             int minibatch, void* costs_device, double grad_scale,
                                             struct rnntGradOptions grad_options,
                                             struct rnntLatticeOptions lattice_options, void* workspace,
                                             struct rnntOptions options);
rnntStatus_t rnnt_b200_pruned_forward_lat(int dtype, const void* activations, const int* ranges, int s_range,
                                          const int* flat_labels, const int* label_lengths, const int* input_lengths,
                                          int alphabet_size, int minibatch, void* costs_device, int prepare_backward,
                                          struct rnntLatticeOptions lattice_options, void* workspace,
                                          struct rnntOptions options);
rnntStatus_t rnnt_b200_pruned_backward_lat(int dtype, const void* activations, void* gradients, const int* ranges,
                                           int s_range, const int* flat_labels, const int* label_lengths,
                                           const int* input_lengths, int alphabet_size, int minibatch,
                                           const void* grad_costs_device, double grad_scale,
                                           struct rnntGradOptions grad_options,
                                           struct rnntLatticeOptions lattice_options, void* workspace,
                                           struct rnntOptions options);
/* The additive joint's forward half with smoothing (rnntSmoothOptions, both 0 = the plain joint, which then wants
 * rnnt_b200_add_joint_workspace_size; else rnnt_b200_add_joint_smoothed_workspace_size) and lattice options.  The
 * penalty lives in the factors this forward leaves in the workspace, so the backward halves
 * (rnnt_b200_add_joint_backward, _backward_ex, _smoothed_backward, with the smoothing scales of the forward) take no
 * lattice options, and rnnt_b200_add_joint_prune_ranges gives the windows of the penalised lattice. */
rnntStatus_t rnnt_b200_add_joint_forward_lat(const float* trans, const float* pred, const int* flat_labels,
                                             const int* label_lengths, const int* input_lengths, int alphabet_size,
                                             int minibatch, float* costs_device, int prepare_backward,
                                             struct rnntSmoothOptions smooth,
                                             struct rnntLatticeOptions lattice_options, void* workspace,
                                             struct rnntOptions options);

/*
 * Lattice topology, the `rnnt_type` argument of the *_topo entries below (k2's rnnt_type; DESIGN.md §11).
 *   RNNT_B200_RNNT_REGULAR   the transducer of every other entry: a blank moves to the next frame, a label stays on
 *                            the frame, so a frame may emit any number of labels.
 *   RNNT_B200_RNNT_MODIFIED  one symbol per frame (optimized_transducer's one_sym_per_frame): every frame takes
 *                            exactly one transition, a blank (u stays) or the label y_u (u + 1), both to the next
 *                            frame.  With T_b, U_b = label_len + 1 after the usual clamps:
 *                              alpha(0,0) = 0, alpha(t,u) = lse(alpha(t-1,u) + lp_blank(t-1,u),
 *                                                               alpha(t-1,u-1) + lp_label(t-1,u-1)),
 *                              cost = -lse(alpha(T_b-1,U_b-1) + lp_blank(T_b-1,U_b-1),
 *                                          alpha(T_b-1,U_b-2) + lp_label(T_b-1,U_b-2)).
 *                            An utterance with U_b - 1 > T_b has no path: its cost is +inf and its gradient is zero.
 *                            The delay penalty, FastEmit and clamp apply as for the regular topology.
 * Any other value returns RNNT_STATUS_INVALID_VALUE before any device access.  rnnt_type = RNNT_B200_RNNT_REGULAR
 * runs exactly the kernels of the *_lat entry of the same name and computes the same results, bitwise.  Workspace
 * sizes do not change.  A backward half must get the rnnt_type its forward got.
 */
enum { RNNT_B200_RNNT_REGULAR = 0, RNNT_B200_RNNT_MODIFIED = 1 };

/* rnnt_b200_loss_async_lat, _forward_lat and _backward_lat with a topology. */
rnntStatus_t rnnt_b200_loss_async_topo(int dtype, int layout, const void* activations, void* gradients,
                                       const int* flat_labels, const int* label_lengths,
                                       const int* input_lengths, int alphabet_size, int minibatch,
                                       void* costs_device, double grad_scale, struct rnntGradOptions grad_options,
                                       struct rnntLatticeOptions lattice_options, int rnnt_type, void* workspace,
                                       struct rnntOptions options);
rnntStatus_t rnnt_b200_forward_topo(int dtype, const void* activations, const int* flat_labels,
                                    const int* label_lengths, const int* input_lengths, int alphabet_size,
                                    int minibatch, void* costs_device, int prepare_backward,
                                    struct rnntLatticeOptions lattice_options, int rnnt_type, void* workspace,
                                    struct rnntOptions options);
rnntStatus_t rnnt_b200_backward_topo(int dtype, const void* activations, void* gradients,
                                     const int* flat_labels, const int* label_lengths,
                                     const int* input_lengths, int alphabet_size, int minibatch,
                                     const void* grad_costs_device, double grad_scale,
                                     struct rnntGradOptions grad_options, struct rnntLatticeOptions lattice_options,
                                     int rnnt_type, void* workspace, struct rnntOptions options);
/* rnnt_b200_pruned_loss_async_lat, _forward_lat and _backward_lat with a topology.  A modified utterance whose
 * windows leave it no path costs +inf with a zero gradient. */
rnntStatus_t rnnt_b200_pruned_loss_async_topo(int dtype, int layout, const void* activations, void* gradients,
                                              const int* ranges, int s_range, const int* flat_labels,
                                              const int* label_lengths, const int* input_lengths, int alphabet_size,
                                              int minibatch, void* costs_device, double grad_scale,
                                              struct rnntGradOptions grad_options,
                                              struct rnntLatticeOptions lattice_options, int rnnt_type,
                                              void* workspace, struct rnntOptions options);
rnntStatus_t rnnt_b200_pruned_forward_topo(int dtype, const void* activations, const int* ranges, int s_range,
                                           const int* flat_labels, const int* label_lengths, const int* input_lengths,
                                           int alphabet_size, int minibatch, void* costs_device, int prepare_backward,
                                           struct rnntLatticeOptions lattice_options, int rnnt_type, void* workspace,
                                           struct rnntOptions options);
rnntStatus_t rnnt_b200_pruned_backward_topo(int dtype, const void* activations, void* gradients, const int* ranges,
                                            int s_range, const int* flat_labels, const int* label_lengths,
                                            const int* input_lengths, int alphabet_size, int minibatch,
                                            const void* grad_costs_device, double grad_scale,
                                            struct rnntGradOptions grad_options,
                                            struct rnntLatticeOptions lattice_options, int rnnt_type,
                                            void* workspace, struct rnntOptions options);

/* The additive joint with a topology: rnnt_b200_add_joint_forward_lat plus rnnt_type; one backward half for the
 * plain and the smoothed joint (rnntSmoothOptions both 0 = plain) with gradient options as
 * rnnt_b200_add_joint_backward_ex; and the pruning ranges of a modified (or regular) joint workspace.  With
 * RNNT_B200_RNNT_MODIFIED the ranges are steps 1-3 of rnnt_b200_add_joint_prune_ranges with
 * e_y(t,u) = exp(alpha(t,u) + lp_y(t,u) + beta(t+1,u+1) - ll).  They do not guarantee a path: a window may advance
 * R-1 labels in one frame and a modified path one, so the pruned modified loss of an utterance may be +inf with a
 * zero gradient (DESIGN.md §11). */
rnntStatus_t rnnt_b200_add_joint_forward_topo(const float* trans, const float* pred, const int* flat_labels,
                                              const int* label_lengths, const int* input_lengths, int alphabet_size,
                                              int minibatch, float* costs_device, int prepare_backward,
                                              struct rnntSmoothOptions smooth,
                                              struct rnntLatticeOptions lattice_options, int rnnt_type,
                                              void* workspace, struct rnntOptions options);
rnntStatus_t rnnt_b200_add_joint_backward_topo(const float* trans, const float* pred, float* grad_trans,
                                               float* grad_pred, const int* flat_labels, const int* label_lengths,
                                               const int* input_lengths, int alphabet_size, int minibatch,
                                               const float* grad_costs_device, float grad_scale,
                                               struct rnntGradOptions grad_options, struct rnntSmoothOptions smooth,
                                               int rnnt_type, void* workspace, struct rnntOptions options);
rnntStatus_t rnnt_b200_add_joint_prune_ranges_topo(const int* label_lengths, const int* input_lengths, int minibatch,
                                                   int s_range, int* ranges, const void* workspace, int rnnt_type,
                                                   struct rnntOptions options);

/* Forced alignment (DESIGN.md §12): the highest-scoring path through the lattice of each utterance, and the frame
 * at which it emits each label.  The lattice is the loss's: T_b, U_b = label_length + 1 after the loss's clamps,
 * and the natural-log blank / label log-probabilities lp_0(t,u), lp_y(t,u) of the dense (or pruned, uncovered cells
 * at log zero) logits.  No delay penalty is applied.
 *   RNNT_B200_RNNT_REGULAR   an alignment is one frame per label, t_0 <= t_1 <= ... <= t_{U_b-2} in [0, T_b-1]:
 *                            label j is emitted from cell (t_j, j), the blank of frame t from (t, #{j : t_j <= t});
 *                            T_b + U_b - 1 factors.
 *   RNNT_B200_RNNT_MODIFIED  frames strictly increase, t_0 < t_1 < ...: frame t_j emits label j from (t_j, j), every
 *                            other frame t a blank from (t, #{j : t_j < t}); T_b factors.
 * Outputs, every element written:
 *   frames [N, maxU-1] int32: t_j of the best alignment; -1 for j >= label_length.
 *   scores [N]: that alignment's log-probability (natural log, <= 0; the sign is opposite to the costs), float for
 *          RNNT_B200_FP32 / _BF16 / _FP16, double for RNNT_B200_FP64.
 * Ties: where the two predecessors of a cell score exactly equal, the blank predecessor (t-1, u) wins, so among equal
 * partial paths labels are emitted as early as possible (uniform logits: regular - every label at frame 0,
 * modified - label j at frame j).
 * No path (best score log zero: a modified utterance with U_b - 1 > T_b, windows without a path, -inf logits):
 * scores[b] = -inf and frames[b, :] = -1.  A NaN factor: scores[b] = NaN and frames[b, :] = -1.  Other utterances
 * are unaffected.
 * dtype is RNNT_B200_FP32, _FP64, _BF16 or _FP16; layout NTUV or TUNV (TUNV: FP32 / FP64 only); the pruned entry
 * takes [N, maxT, s_range, V] logits and `ranges` as rnnt_b200_pruned_loss_async_topo.  All pointers are device
 * pointers; the call is stream-ordered on options.stream and does not synchronise.  The workspace is that of the
 * loss: get_workspace_size / rnnt_b200_pruned_workspace_size.  Arguments the loss entries reject, an unknown dtype,
 * layout or rnnt_type, s_range < 1 and NULL pointers (frames may be NULL when maxU == 1) are
 * RNNT_STATUS_INVALID_VALUE before any device access. */
rnntStatus_t rnnt_b200_align(int dtype, int layout, const void* activations, const int* flat_labels,
                             const int* label_lengths, const int* input_lengths, int alphabet_size, int minibatch,
                             int rnnt_type, int* frames, void* scores_device, void* workspace,
                             struct rnntOptions options);
rnntStatus_t rnnt_b200_pruned_align(int dtype, const void* activations, const int* ranges, int s_range,
                                    const int* flat_labels, const int* label_lengths, const int* input_lengths,
                                    int alphabet_size, int minibatch, int rnnt_type, int* frames,
                                    void* scores_device, void* workspace, struct rnntOptions options);

/* The loss, its gradient and forced alignment on caller-supplied factors (DESIGN.md §13; k2's
 * mutual_information_recursion).  The lattice machinery above without the log-softmax: the caller forms the
 * natural-log transition factors, by any joiner, prior, fusion or penalty.  Inputs, label-major with t contiguous:
 *   px [N, S, T]    px[b, s, t] = lp_y(t, s), the label factor out of cell (t, s) (emitting label s at frame t)
 *   py [N, S+1, T]  py[b, s, t] = lp_0(t, s), the blank factor out of cell (t, s)
 * with T = options.maxT and S + 1 = options.maxU; label_lengths / input_lengths give S_b and T_b (clamped as the loss
 * clamps them: U_b = S_b + 1).  There are no labels, no blank index and no alphabet; options.blank_label is ignored.
 * Factors need not be normalised: any finite value or -inf is valid, and positive factors give negative costs.  The
 * fp32 arithmetic (RNNT_B200_FP32 / _BF16 / _FP16) represents factors of magnitude below 2^22 ln 2 (about 2.9e6).
 *   RNNT_B200_RNNT_REGULAR   k2's -mutual_information_recursion(px with a -inf column T appended, py,
 *                            boundary = [0, 0, S_b, T_b]): the recursion of the dense loss.
 *   RNNT_B200_RNNT_MODIFIED  the same with k2's px of width T: one transition per frame (DESIGN.md §11).
 * forward: costs[b] = -log-likelihood (float, double for RNNT_B200_FP64); +inf without a path; NaN when a factor of
 *   the utterance is NaN or +inf.  prepare_backward: also the beta lattice, for a backward on the same workspace.
 * backward: py_grad[b,s,t] = -g[b] e_0(t,s) and px_grad[b,s,t] = -g[b] e_y(t,s), the blank and label transition
 *   occupancies (the exact gradient of the cost), g[b] = grad_scale * grad_costs_device[b] (arithmetic type; NULL:
 *   ones); zero on padding (t >= T_b, s > S_b for py, s >= S_b for px) and for an utterance without a path.  It reads
 *   only the workspace of a forward with prepare_backward and must get that forward's rnnt_type.
 * align: frames [N, S] and scores [N] as rnnt_b200_align, on these factors.
 * Other utterances' results do not depend on a NaN, +inf or -inf factor of one utterance.  dtype: RNNT_B200_FP32,
 * _FP64, _BF16 or _FP16, for px, py and the gradients alike.  All pointers are device pointers; the calls are
 * stream-ordered on options.stream and do not synchronise.  The workspace is rnnt_b200_lattice_workspace_size's.  An
 * unknown dtype or rnnt_type, NULL pointers (px, px_grad and frames may be NULL when maxU == 1), minibatch, maxT or
 * maxU < 1, maxU > 1024 and minibatch * maxT * maxU >= 2^31 are RNNT_STATUS_INVALID_VALUE before any device access. */
rnntStatus_t rnnt_b200_lattice_workspace_size(int maxT, int maxU, int minibatch, size_t dtype_size,
                                              size_t* size_bytes);
rnntStatus_t rnnt_b200_lattice_forward(int dtype, const void* px, const void* py, const int* label_lengths,
                                       const int* input_lengths, int minibatch, int rnnt_type, void* costs_device,
                                       int prepare_backward, void* workspace, struct rnntOptions options);
rnntStatus_t rnnt_b200_lattice_backward(int dtype, void* px_grad, void* py_grad, const int* label_lengths,
                                        const int* input_lengths, int minibatch, int rnnt_type,
                                        const void* grad_costs_device, double grad_scale, void* workspace,
                                        struct rnntOptions options);
rnntStatus_t rnnt_b200_lattice_align(int dtype, const void* px, const void* py, const int* label_lengths,
                                     const int* input_lengths, int minibatch, int rnnt_type, int* frames,
                                     void* scores_device, void* workspace, struct rnntOptions options);

/* Fused joiner (DESIGN.md §14): the lattice factors of icefall's / torchaudio's / NeMo's joiner
 *   logits[b,t,u,:] = weight act(enc[b,t] + pred[b,u]) + bias
 * without forming the [N, T, U, V] logits, and the gradients of the four inputs back from the factors' gradients.
 * Inputs, all bf16 device pointers, row-major and 16-byte aligned (bias: 2-byte):
 *   enc [N, maxT, hidden], pred [N, maxU, hidden], weight [alphabet_size, hidden] (nn.Linear's layout),
 *   bias [alphabet_size] or NULL (zero).
 * flat_labels [N, maxU-1], label_lengths and input_lengths are int32 device pointers, as the loss takes them (S_b and
 * T_b clamped into [0, maxU-1] and [1, maxT], as the lattice clamps them); options.blank_label is the blank column.
 * forward: with h = round_bf16(act(fp32(enc[b,t]) + fp32(pred[b,u]))) (act: tanhf or relu), logit_v = sum_k h_k
 *   weight[v,k] in fp32 plus fp32(bias[v]) and lse the fp32 logsumexp over all alphabet_size columns,
 *   py [N, maxU, maxT]    py[b,u,t] = logit_blank - lse
 *   px [N, maxU-1, maxT]  px[b,u,t] = logit_{labels[b,u]} - lse          (float; rnnt_b200_lattice_forward's layout)
 *   -inf on padding (t >= T_b; u > S_b for py, u >= S_b for px).  Labels are compared with column indices, never used
 *   as addresses: a label outside [0, alphabet_size) gives px = NaN on its row.  Padded rows of enc and pred are not
 *   read.  The workspace keeps one fp32 lse per cell for the backward.
 * backward: from dpx, dpy (float, the factors' gradients) and the workspace of a forward with the same arguments,
 *   dlogit_v = dpy [v = blank] + dpx [v = label] - (dpx + dpy) softmax_v, rounded to bf16 in a chunk scratch;
 *   grad_weight = sum dlogit (x) h, grad_bias = sum dlogit, ds = (dlogit weight) act'(s) (tanh: 1 - h^2 from the
 *   rounded h; relu: [s > 0]), grad_enc[b,t] = sum_u ds, grad_pred[b,u] = sum_t ds.  dpx / dpy on padding are not
 *   read; padding rows of grad_enc and grad_pred are zero.  The four gradients are accumulated in fp32 and written
 *   once in bf16 (shapes of enc, pred, weight, bias); grad_bias may be NULL.  Bitwise deterministic for a given
 *   chunk_cells: no float atomics.
 * chunk_cells: cells (b, u, t) per pass through the scratch (h, dlogits and ds rows); 0 picks the largest multiple of
 *   64 whose scratch fits in 256 MiB.  The workspace never grows with N T U V: per-cell lse, fp32 accumulators of
 *   the four gradients, and the scratch.  The backward must get the forward's chunk_cells.
 * Launches: the forward 2 per chunk; the backward 5 per chunk, 1 more, and one memset of the accumulators.  The
 * calls are stream-ordered on options.stream without host synchronisation (graph-capturable).
 * activation other than RNNT_B200_ACT_TANH / _RELU, hidden not a multiple of 16 in [16, 1024], alphabet_size < 2,
 * blank_label outside [0, alphabet_size), chunk_cells < 0, minibatch, maxT or maxU < 1, maxU > 1024,
 * minibatch * maxT * maxU >= 2^31, NULL pointers (flat_labels, px and dpx may be NULL when maxU == 1; bias and
 * grad_bias may be NULL) and misaligned pointers are RNNT_STATUS_INVALID_VALUE before any device access; RNNT_CPU
 * then returns RNNT_STATUS_EXECUTION_FAILED. */
enum { RNNT_B200_ACT_TANH = 0, RNNT_B200_ACT_RELU = 1 };
rnntStatus_t rnnt_b200_joiner_workspace_size(int maxT, int maxU, int minibatch, int hidden, int alphabet_size,
                                             int chunk_cells, size_t* size_bytes);
rnntStatus_t rnnt_b200_joiner_forward(int activation, const void* enc, const void* pred, const void* weight,
                                      const void* bias, const int* flat_labels, const int* label_lengths,
                                      const int* input_lengths, int hidden, int alphabet_size, int minibatch,
                                      int chunk_cells, float* px, float* py, void* workspace,
                                      struct rnntOptions options);
rnntStatus_t rnnt_b200_joiner_backward(int activation, const void* enc, const void* pred, const void* weight,
                                       const void* bias, const int* flat_labels, const int* label_lengths,
                                       const int* input_lengths, int hidden, int alphabet_size, int minibatch,
                                       int chunk_cells, const float* dpx, const float* dpy, void* grad_enc,
                                       void* grad_pred, void* grad_weight, void* grad_bias, void* workspace,
                                       struct rnntOptions options);

/* Pruned fused joiner (DESIGN.md §15): the fused joiner's factors on the pruned lattice of rnnt_b200_pruned_*, without
 * the [N, T, s_range, V] logits.  Arguments as the fused joiner's, plus ranges [N, maxT] (int32 device pointer) and
 * s_range = R >= 1.  Row (b, t, r), r < R, stands for lattice cell (t, u = ranges[b,t] + r), u formed without
 * overflow for any int32 window start; the row is valid when t < T_b and 0 <= u <= S_b (R > maxU is allowed).
 * forward: px [N, maxU-1, maxT] and py [N, maxU, maxT] in rnnt_b200_joiner_forward's layout; on a valid row's cell
 *   the fused joiner's values, every other element -inf (every element is written).  Padded rows of enc and pred,
 *   and pred rows no valid row selects, are not read.  The workspace keeps one fp32 lse per row.
 * backward: the fused joiner's gradients over the valid rows only: dpx / dpy are read only at the cells valid rows
 *   cover.  grad_enc[b,t] sums its rows in r order, grad_pred[b,u] the rows selecting u in t order; bf16, fp32
 *   accumulation, bitwise deterministic for a given chunk_cells.  With s_range = maxU and ranges = 0 both halves are
 *   bitwise the fused joiner's.
 * chunk_cells counts rows (b, t, r).  The workspace holds the per-row lse (4 N maxT R bytes), the same fp32
 * accumulators (grad_pred's stays N maxU hidden) and scratch as the fused joiner's.
 * Launches: the forward 1 (the -inf fill) + 2 per chunk; the backward 5 per chunk, 1 more, and one memset.
 * The fused joiner's rules, NULL ranges, s_range < 1 and minibatch * maxT * s_range >= 2^31 are
 * RNNT_STATUS_INVALID_VALUE before any device access. */
rnntStatus_t rnnt_b200_pruned_joiner_workspace_size(int maxT, int maxU, int s_range, int minibatch, int hidden,
                                                    int alphabet_size, int chunk_cells, size_t* size_bytes);
rnntStatus_t rnnt_b200_pruned_joiner_forward(int activation, const void* enc, const void* pred, const void* weight,
                                             const void* bias, const int* flat_labels, const int* label_lengths,
                                             const int* input_lengths, const int* ranges, int s_range, int hidden,
                                             int alphabet_size, int minibatch, int chunk_cells, float* px, float* py,
                                             void* workspace, struct rnntOptions options);
rnntStatus_t rnnt_b200_pruned_joiner_backward(int activation, const void* enc, const void* pred, const void* weight,
                                              const void* bias, const int* flat_labels, const int* label_lengths,
                                              const int* input_lengths, const int* ranges, int s_range, int hidden,
                                              int alphabet_size, int minibatch, int chunk_cells, const float* dpx,
                                              const float* dpy, void* grad_enc, void* grad_pred, void* grad_weight,
                                              void* grad_bias, void* workspace, struct rnntOptions options);

/* Dropout on the joiner's hidden activation (DESIGN.md §16): NeMo's RNNTJoint, Sequential(act, Dropout(p), Linear),
 * for the fused and pruned fused joiners.  Passed BY VALUE to the *_drop entries below, which take the arguments of
 * the entry of the same name and this before the workspace.
 *   p      dropout probability, 0 <= p < 1.
 *   seed   device pointer to a 64-bit seed, 8-byte aligned, read on the device (no host synchronisation; graph
 *          capture records the pointer, so a replay uses whatever seed it then holds).  May be NULL when p == 0.
 * Mask: element k of cell (b, t, u) is dropped iff x < thr, with x = word (k & 3) of
 *   curand_Philox4x32_10(ctr = (k >> 2, (b maxU + u) maxT + t, 0, 0), key = (lo32(seed), hi32(seed)))
 * and thr = floor((double) p 2^32).  It is a pure function of the seed and the element: the same for any chunk_cells,
 * dense or pruned, forward or backward, so nothing is stored.  It depends on the padded extents maxT and maxU, as
 * eager dropout on an [N, maxT, maxU, hidden] tensor does.  A pruned row uses the mask of the cell it stands for.
 * forward: the logits GEMM operand is h~ = keep ? round_bf16(h scale) : 0, scale = (float)(1 / (1 - (double) p)),
 *   with h the fused joiner's rounded h; px, py follow from h~.  The bias column is never dropped.
 * backward: dlogit as without dropout; grad_weight = sum dlogit (x) h~; ds = (dlogit weight) keep scale act'(s), act'
 *   as without dropout (tanh: 1 - h^2 from the undropped rounded h).  The backward must get the forward's p and seed.
 * Workspace sizes, launches and every other rule are those of the entry of the same name; p == 0 runs its kernels
 * and gives its results bitwise.  NaN p, p < 0, p >= 1, a NULL seed with p > 0 and a misaligned seed are
 * RNNT_STATUS_INVALID_VALUE before any device access. */
struct rnntJoinerDropout {
    float p;
    const unsigned long long* seed;
};
rnntStatus_t rnnt_b200_joiner_forward_drop(int activation, const void* enc, const void* pred, const void* weight,
                                           const void* bias, const int* flat_labels, const int* label_lengths,
                                           const int* input_lengths, int hidden, int alphabet_size, int minibatch,
                                           int chunk_cells, float* px, float* py, struct rnntJoinerDropout dropout,
                                           void* workspace, struct rnntOptions options);
rnntStatus_t rnnt_b200_joiner_backward_drop(int activation, const void* enc, const void* pred, const void* weight,
                                            const void* bias, const int* flat_labels, const int* label_lengths,
                                            const int* input_lengths, int hidden, int alphabet_size, int minibatch,
                                            int chunk_cells, const float* dpx, const float* dpy, void* grad_enc,
                                            void* grad_pred, void* grad_weight, void* grad_bias,
                                            struct rnntJoinerDropout dropout, void* workspace,
                                            struct rnntOptions options);
rnntStatus_t rnnt_b200_pruned_joiner_forward_drop(int activation, const void* enc, const void* pred,
                                                  const void* weight, const void* bias, const int* flat_labels,
                                                  const int* label_lengths, const int* input_lengths,
                                                  const int* ranges, int s_range, int hidden, int alphabet_size,
                                                  int minibatch, int chunk_cells, float* px, float* py,
                                                  struct rnntJoinerDropout dropout, void* workspace,
                                                  struct rnntOptions options);
rnntStatus_t rnnt_b200_pruned_joiner_backward_drop(int activation, const void* enc, const void* pred,
                                                   const void* weight, const void* bias, const int* flat_labels,
                                                   const int* label_lengths, const int* input_lengths,
                                                   const int* ranges, int s_range, int hidden, int alphabet_size,
                                                   int minibatch, int chunk_cells, const float* dpx,
                                                   const float* dpy, void* grad_enc, void* grad_pred,
                                                   void* grad_weight, void* grad_bias,
                                                   struct rnntJoinerDropout dropout, void* workspace,
                                                   struct rnntOptions options);
/* Kernels (memsets not counted) the last fused or pruned joiner call on this thread launched. */
int rnnt_b200_joiner_last_launch_count(void);

/* Debug / test hook: forward and backward log-likelihoods (natural log, as doubles on the host) that
 * the last loss+gradient call left in `workspace`.  The reference checks their agreement in debug
 * builds (include/detail/cpu_rnnt.h:167-170); tests/test_gpu_round2.py does the same.  Synchronises. */
rnntStatus_t rnnt_b200_debug_log_likelihoods(const void* workspace, int maxT, int maxU, int minibatch,
                                             size_t dtype_size, double* llf_host, double* llb_host);

/* Number of kernels the last compute call on this thread launched (bench.py's gpu_launches). */
int rnnt_b200_last_launch_count(void);

/* Per-kernel device timing for bench.py's roofline leg.  With profiling enabled on the calling
 * thread, each compute call records CUDA events on options.stream around its three kernels;
 * rnnt_b200_last_kernel_ms() waits for them and writes {rowstats, lattice, grad} milliseconds
 * (-1 where not run) and returns how many were measured. */
void rnnt_b200_set_profiling(int enabled);
int rnnt_b200_last_kernel_ms(float* ms3);
/* Mean {rowstats, lattice, grad} milliseconds over every call recorded on this thread since the
 * previous collect (waits for their events), returns the number of calls and resets the record.
 * Lets a timed loop run without any host synchronisation between steps. */
int rnnt_b200_profile_collect(float* ms3_mean);

/* Host-side dispatch policy, for tests and tuning notes (no device access).  `what`:
 *   0  lanes sharing one short row in the chunk kernels for alphabet size a and element size b bytes (0: row too long
 *      for the chunk kernels);  1  1 if those lanes are `32 / lanes` apart in the warp (bank-aware mapping), 0 if adjacent;
 *   2  label columns per lane of the fp32 wavefront for maxU = a;  3  its threads per utterance and direction;
 *   4  diagonals of its factor ring (b != 0: next to the streaming passes of other batch groups);
 *   5  split-K slabs of the additive joint's S product for alphabet size a;
 *   6  as 1, but with the RNNT_B200_CHUNK_MAP tuning hook applied (the mapping the chunk kernels are given);
 *   7  1 if the RNNT_B200_PDL tuning hook asks for programmatic dependent launch, else 0.
 * 4, 5 and 6 honour the tuning hooks (README), 0 and 1 do not.   Returns -1 for an unknown `what`. */
int rnnt_b200_debug_policy(int what, int a, int b);

/* Build identification string, e.g. "b200-rnnt sm_90a <date>". */
const char* rnnt_b200_build_info(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_RNNT_H_ */
