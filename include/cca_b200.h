/*
 * cca_b200.h -- C ABI of the Hopper-native (sm_90a) criss-cross attention operator.
 *
 * This is the drop-in boundary for CCNet's hot path.  The reference exposes the path
 * only as a Python nn.Module (cc_attention/functions.py:15-49; the mounted branch has
 * no native FFI -- SURVEY.md F1), so the entry points below are what a binding for that
 * module binds: one call per recurrence step for forward (replaces functions.py:30-47:
 * the six layout copies, INF mask, two QK^T bmm, cat+softmax, two A.V bmm) and one for
 * its backward (replaces the autograd graph of those lines, SURVEY.md 8a row a11).
 * The 1x1 Q/K/V projections (functions.py:29,32,35) and the gamma*o+x residual
 * (functions.py:49) stay with the caller, exactly where the reference has them.
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types.
 *   - tensors are NCHW-contiguous (default) or channels-last (CCA_FLAG_NHWC), same dtype
 *     for q,k,v,out (CCA_F32 or CCA_BF16); lse / stats / delta are always fp32 [B,H,W].
 *   - q,k: [B,Cq,H,W]   v,out,dout,dv: [B,C,H,W]   lse: [B,H,W].
 *   - "device" entry points take device pointers valid on the current CUDA device and a
 *     cudaStream_t (as void*); they enqueue work and return without synchronising.
 *   - "host" entry points take host pointers, do H2D, compute, D2H and synchronise.
 *   - every function returns CCA_OK (0) or a negative cca_status; the message of the
 *     last failure on the calling thread is available from cca_b200_last_error().
 *   - inputs are never written; outputs need no initialisation.
 *   - re-entrant: no global scratch; the caller supplies the (small) workspace.  Process-wide state is limited to
 *     read-mostly caches (tensor maps, device attributes) and launch knobs read once from the environment.
 *   - every compute entry point returns CCA_ERR_DEVICE unless the current device is compute capability 10.x.
 */
#ifndef CCA_B200_H_
#define CCA_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CCA_B200_VERSION 200 /* 0.2.0 */

#if defined(__GNUC__)
#define CCA_API __attribute__((visibility("default")))
#else
#define CCA_API
#endif

typedef enum cca_dtype {
    CCA_F32 = 0,  /* float32 I/O, fp32 accumulate                                       */
    CCA_BF16 = 1  /* bfloat16 I/O, fp32 accumulate, fp32 lse.  Lines longer than 112 pixels: an */
                  /* output element is the sum of up to 2*ceil(L/112) bf16-rounded partial      */
                  /* results (TMA reduce-add, no fixed order): gradients at the 1e-2 budget --  */
                  /* call CCA_F32 on upcast tensors for fp32-grade accumulation (INTEGRATION.md) */
} cca_dtype;

typedef enum cca_status {
    CCA_OK = 0,
    CCA_ERR_INVALID = -1,      /* bad pointer / shape / dtype / flags                    */
    CCA_ERR_UNSUPPORTED = -2,  /* shape outside what the kernels cover (see limits)      */
    CCA_ERR_WORKSPACE = -3,    /* workspace too small                                    */
    CCA_ERR_CUDA = -4,         /* CUDA runtime error (message in cca_b200_last_error)    */
    CCA_ERR_DEVICE = -5        /* current device is not sm_90                            */
} cca_status;

/* flags (bit mask) */
#define CCA_FLAG_AUTO 0u        /* pick the fastest kernel family that covers the shape  */
#define CCA_FLAG_FORCE_SIMT 1u  /* generic CUDA-core kernels (any shape within limits)   */
#define CCA_FLAG_FORCE_TC 2u    /* wgmma tensor-core kernels; error if not applicable    */
#define CCA_FLAG_NHWC 4u        /* tensors are channels-last: q,k [B,H,W,Cq]; v,out,dout,dq.. [B,H,W,C]
                                 * (torch.channels_last of the same logical NCHW shape).  This is the
                                 * layout of the tensor-core kernels: rows and columns of the image are
                                 * both "L pixels with contiguous channels", so TMA boxes and UMMA operand
                                 * tiles serve the two branches symmetrically.  Without the flag tensors
                                 * are NCHW-contiguous and the generic kernels run.                      */

/* which workspace */
#define CCA_WS_FORWARD 0
#define CCA_WS_BACKWARD 1

CCA_API int cca_b200_version(void);
CCA_API const char *cca_b200_last_error(void);
CCA_API const char *cca_b200_strerror(int status);

/* 1 if the current CUDA device can run this library (compute capability 10.x), else 0;
 * negative cca_status on CUDA failure. */
CCA_API int cca_b200_device_ok(void);

/* Number of kernels this library has launched in this process so far (for audits). */
CCA_API unsigned long long cca_b200_launch_count(void);

/* 1 if the tensor-core (wgmma) kernels cover this problem in NHWC layout on the current device, else 0.
 * which = CCA_WS_FORWARD or CCA_WS_BACKWARD (the two directions have separate predicates).
 * Covered: Cq in {16,32,48,64}, C % 64 == 0, H and W up to 896 (lines longer than 112 pixels are tiled). */
CCA_API int cca_b200_tc_supported(int which, int B, int Cq, int C, int H, int W, int dtype);

/* Introspection of the tensor-core kernels' work decomposition (host-only, no CUDA call; see csrc/cca_items.cuh):
 * item_space: out8 = {total items, items per sample, column/first-key-block items, other column items, row items,
 *                     tiles per column line, tiles per row line, padded tile length (80 or 112; 0 = not covered)}
 * decode_item: out10 = {is_column, sample, line, query tile, key block, q0, lq, k0, lk, index inside the sample};
 *   lagged = 0: samples one after the other; 1: the consumers of a sample trail its producers by one block. */
CCA_API void cca_b200_item_space(int B, int H, int W, int *out8);
CCA_API void cca_b200_decode_item(int B, int H, int W, int index, int lagged, int *out10);

/* Bytes of device workspace the forward / backward call needs for this problem. */
CCA_API size_t cca_b200_workspace_bytes(int which, int B, int Cq, int C, int H, int W, int dtype);

/*
 * One criss-cross attention step, forward (replaces functions.py:30-47):
 *   e_col[b,h,w,g] = <q[b,:,h,w], k[b,:,g,w]>   (-inf at g == h)
 *   e_row[b,h,w,g] = <q[b,:,h,w], k[b,:,h,g]>
 *   a = softmax over the H+W entries;  out = a_col . v(column) + a_row . v(row)
 *   lse[b,h,w] = logsumexp of the H+W logits (saved for backward).
 */
CCA_API int cca_b200_forward(const void *q, const void *k, const void *v, void *out, float *lse,
                     void *workspace, size_t workspace_bytes,
                     int B, int Cq, int C, int H, int W, int dtype, unsigned flags,
                     void *cuda_stream);

/*
 * Backward of the step above: given dout = dL/dout, and the forward's q,k,v,out,lse,
 * writes dq, dk, dv (closed form; the attention matrix is recomputed, never stored).
 */
CCA_API int cca_b200_backward(const void *dout, const void *q, const void *k, const void *v,
                      const void *out, const float *lse, void *dq, void *dk, void *dv,
                      void *workspace, size_t workspace_bytes,
                      int B, int Cq, int C, int H, int W, int dtype, unsigned flags,
                      void *cuda_stream);

/*
 * The three 1x1 projections in front of the step (replace functions.py:29,32,35 -- query_conv, key_conv, value_conv -- and
 * their input gradient) as hand-written wgmma GEMMs on the channels-last view: x, v, dx are [pixels, C], q, k, dq, dk are
 * [pixels, Cq] row-major fp32 (a channels-last [B,C,H,W] tensor IS that matrix with pixels = B*H*W); weights are the conv
 * weights [out, in] row-major ([out,in,1,1] contiguous).  fp32 accuracy via the bf16 hi/lo split (3 MMAs per product).
 *   qkv_project       : q = x Wq^T + bq,  k = x Wk^T + bk,  v = x Wv^T + bv
 *   qkv_project_dgrad : dx (+)= s (dq Wq + dk Wk + dv Wv)    (accumulate != 0 adds onto dx)
 *   qkv_project_wgrad : dWq = s dq^T x, dWk = s dk^T x, dWv = s dv^T x  and  db = s [sum_p dq | sum_p dk | sum_p dv]
 *                       (db: 2 Cq + C floats in that order, may be NULL; outputs are cleared by the call)
 * `scale` (s) is a DEVICE pointer to one float or NULL (= 1): the gamma of functions.py:49, applied to the small matrices
 * instead of to the [pixels, C] gradient.  Covered: C % 64 == 0, Cq % 64 == 0, 2 Cq + C <= 1024 (wgrad: C % 256 == 0).
 */
CCA_API int cca_b200_qkv_supported(int C, int Cq);
CCA_API size_t cca_b200_qkv_workspace_bytes(int C, int Cq);
CCA_API int cca_b200_qkv_project(const float *x, const float *wq, const float *bq, const float *wk, const float *bk,
                                 const float *wv, const float *bv, float *q, float *k, float *v,
                                 void *workspace, size_t workspace_bytes, long long pixels, int C, int Cq, void *cuda_stream);
CCA_API int cca_b200_qkv_project_dgrad(const float *dq, const float *dk, const float *dv, const float *wq, const float *wk,
                                       const float *wv, const float *scale, float *dx, void *workspace, size_t workspace_bytes,
                                       long long pixels, int C, int Cq, int accumulate, void *cuda_stream);
CCA_API int cca_b200_qkv_wgrad_supported(int C, int Cq);
CCA_API int cca_b200_qkv_project_wgrad(const float *x, const float *dq, const float *dk, const float *dv, const float *scale,
                                       float *dwq, float *dwk, float *dwv, float *db,
                                       long long pixels, int C, int Cq, void *cuda_stream);

/*
 * Host-buffer variants: same maths, pointers are HOST memory (pinned or pageable).
 * They allocate device memory, copy in, run on an internal stream, copy out, free and
 * synchronise.  These are the calls a non-CUDA host language binds directly.
 */
CCA_API int cca_b200_forward_host(const void *q, const void *k, const void *v, void *out, float *lse,
                          int B, int Cq, int C, int H, int W, int dtype, unsigned flags);
CCA_API int cca_b200_backward_host(const void *dout, const void *q, const void *k, const void *v,
                           const void *out, const float *lse, void *dq, void *dk, void *dv,
                           int B, int Cq, int C, int H, int W, int dtype, unsigned flags);

#ifdef __cplusplus
}
#endif
#endif /* CCA_B200_H_ */
