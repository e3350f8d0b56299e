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
 *     for q,k,v,out (CCA_F32, CCA_BF16 or CCA_F16); lse / stats / delta are always fp32 [B,H,W].
 *   - q,k: [B,Cq,H,W]   v,out,dout,dv: [B,C,H,W]   lse: [B,H,W].
 *   - "device" entry points take device pointers valid on the current CUDA device and a
 *     cudaStream_t (as void*); they enqueue work and return without synchronising.
 *   - "host" entry points take host pointers, do H2D, compute, D2H and synchronise.
 *   - every function returns CCA_OK (0) or a negative cca_status; the message of the
 *     last failure on the calling thread is available from cca_b200_last_error().
 *   - inputs are never written; outputs need no initialisation.
 *   - re-entrant: no global scratch; the caller supplies the (small) workspace.  Process-wide state is limited to
 *     read-mostly caches (tensor maps, device attributes) and launch knobs read once from the environment.
 *   - every compute entry point returns CCA_ERR_DEVICE unless the current device is compute capability 9.x (sm_90).
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
    CCA_BF16 = 1, /* bfloat16 I/O, fp32 accumulate, fp32 lse.  Lines longer than 112 pixels: an */
                  /* output element is the sum of up to 2*ceil(L/112) bf16-rounded partial      */
                  /* results (TMA reduce-add, no fixed order): gradients at the 1e-2 budget --  */
                  /* call CCA_F32 on upcast tensors for fp32-grade accumulation (INTEGRATION.md) */
    CCA_F16 = 2   /* float16 I/O (what torch.autocast uses by default), fp32 accumulate, fp32    */
                  /* lse / delta; P and dS enter the f16 MMAs rounded to f16.  Both kernel      */
                  /* families, the same shapes as CCA_BF16 (cca_b200_tc_supported(.., CCA_F16)  */
                  /* says whether the tensor-core kernels cover a problem); long lines as for   */
                  /* CCA_BF16 (partial results rounded to f16).  Values beyond the f16 range    */
                  /* overflow to inf, as in any f16 computation.                                */
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
#define CCA_FLAG_DETERMINISTIC 8u /* bit-reproducible results (what torch.use_deterministic_algorithms asks
                                 * for).  One-tile shapes and the generic kernels are deterministic anyway:
                                 * the flag changes nothing there.  Lines longer than 112 pixels on the
                                 * tensor-core kernels: every item stores its share into partial planes of
                                 * the workspace (cca_b200_workspace_bytes_ex) instead of reduce-adding it
                                 * onto the output in no fixed order, and one more kernel adds the planes
                                 * in a fixed order.  fp32 only there: 16-bit I/O on such lines returns
                                 * CCA_ERR_UNSUPPORTED (call CCA_F32 on upcast tensors).                   */
#define CCA_FLAG_CAUSAL 16u     /* causal criss-cross attention over clips: honoured by cca_b200_forward3d, _backward3d,
                                 * _attention_forward3d and _attention_backward3d (the 2D entry points handle flag bits as
                                 * before).  The time keys of frame t are the frames s < t.  Workspace sizes are those
                                 * without the flag.  The bit was added without a version change: a library without it
                                 * ignores the bit and computes the bidirectional op.  A caller detects causal support by
                                 * the presence of the cca_b200_forward3d_step symbol (dlsym / GetProcAddress).           */

/* which workspace */
#define CCA_WS_FORWARD 0
#define CCA_WS_BACKWARD 1

CCA_API int cca_b200_version(void);
CCA_API const char *cca_b200_last_error(void);
CCA_API const char *cca_b200_strerror(int status);

/* 1 if the current CUDA device can run this library (compute capability 9.x, sm_90), else 0;
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
/* item_planes: out2 = {partial plane of the item's out / dQ tile, partial plane of its dK / dV tile} in the deterministic
 *   mode (CCA_FLAG_DETERMINISTIC) on tiled lines; same index / lagged as decode_item. */
CCA_API void cca_b200_item_planes(int B, int H, int W, int index, int lagged, int *out2);

/* Bytes of device workspace the forward / backward call needs for this problem.  _ex: for these flags (with
 * CCA_FLAG_DETERMINISTIC | CCA_FLAG_NHWC on tiled lines it adds the partial planes: nparts * B*H*W * C floats forward,
 * nparts * B*H*W * (2 Cq + C) backward, nparts = ceil(H/112) + ceil(W/112)); the plain call assumes flags without
 * CCA_FLAG_DETERMINISTIC. */
CCA_API size_t cca_b200_workspace_bytes(int which, int B, int Cq, int C, int H, int W, int dtype);
CCA_API size_t cca_b200_workspace_bytes_ex(int which, int B, int Cq, int C, int H, int W, int dtype, unsigned flags);

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
/* qkv_project_wgrad with flags.  CCA_FLAG_DETERMINISTIC: every split-K CTA stores its partial dW and db into the device
 * workspace (cca_b200_qkv_wgrad_workspace_bytes, which depends on the current device's SM count) and a second kernel adds
 * them in split order -- bit-reproducible on one card model (the split count follows the SM count).  Without the flag it
 * is cca_b200_qkv_project_wgrad (the workspace may be NULL). */
CCA_API size_t cca_b200_qkv_wgrad_workspace_bytes(int C, int Cq);
CCA_API int cca_b200_qkv_project_wgrad_ex(const float *x, const float *dq, const float *dk, const float *dv, const float *scale,
                                          float *dwq, float *dwk, float *dwv, float *db, long long pixels, int C, int Cq,
                                          void *workspace, size_t workspace_bytes, unsigned flags, void *cuda_stream);

/*
 * The attention map of one step (functions.py:40, the softmax output `concate`) and its gradient:
 *   attn[b,h,w,g] = a of the forward above: g < H the weight of column key (g, w) (0 at g == h), g >= H the weight of row
 *                   key (h, g - H).  Always fp32, contiguous [B,H,W,H+W], for every dtype of q, k.
 *   backward: rho[p] = sum_j attn[p,j] dattn[p,j],  dS = attn * (dattn - rho),  dq[p] = sum_j dS[p,j] k[key j],
 *             dk[key] = sum_p dS[p,key] q[p]   (attn and dattn are read, S and lse are not recomputed).
 * q, k (and dq, dk) are [B,Cq,H,W] NCHW (generic kernels, any Cq and line length) or channels-last with CCA_FLAG_NHWC
 * (tensor-core kernels: Cq in {16,32,48,64}, H and W up to 896, any C).  Flags as for cca_b200_forward; the forward is
 * deterministic in every mode, the backward with one tile per line and with CCA_FLAG_DETERMINISTIC (fp32 on tiled lines;
 * 16-bit I/O there returns CCA_ERR_UNSUPPORTED).  The map holds B*H*W*(H+W) floats: indices into it are 64-bit.  attn and
 * dattn need only the alignment of a float (views at any element offset are fine).
 */
CCA_API int cca_b200_attention_tc_supported(int B, int Cq, int H, int W, int dtype);
CCA_API size_t cca_b200_attention_workspace_bytes(int backward, int B, int Cq, int H, int W, int dtype, unsigned flags);
CCA_API int cca_b200_attention_forward(const void *q, const void *k, float *attn, void *workspace, size_t workspace_bytes,
                                       int B, int Cq, int H, int W, int dtype, unsigned flags, void *cuda_stream);
CCA_API int cca_b200_attention_backward(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk,
                                        void *workspace, size_t workspace_bytes, int B, int Cq, int H, int W, int dtype,
                                        unsigned flags, void *cuda_stream);

/*
 * Criss-cross attention over clips (the 3D op of CCNet's video extension): q, k [B,Cq,T,H,W], v, out [B,C,T,H,W].  Pixel
 * (b,t,h,w) attends to its column {(b,t,g,w)} (self masked), its row {(b,t,h,g)} and its time line {(b,s,h,w)} (self masked):
 * one softmax over the H+W+T logits <q_u, k_j>, out_u = sum_j a_uj v_j, lse[B,T,H,W] fp32 as for the 2D step.  At T = 1 it
 * is the 2D step on every frame.
 * NDHWC tensors (torch.channels_last_3d, CCA_FLAG_NHWC): the tensor-core path.  The column and row branches run on the 2D
 * tensor-core kernels over the [B*T,H,W,C] frames view, the time branch on kernels of its own.  It covers
 * (cca_b200_tc3d_supported) the shapes cca_b200_tc_supported covers for B*T frames, and 1 <= T <= 32.
 * NCDHW-contiguous tensors (no CCA_FLAG_NHWC): generic kernels, any Cq and C, H + W + T - 2 <= 2048; beyond that
 * CCA_ERR_UNSUPPORTED.  Flags, alignment and the deterministic mode as for cca_b200_forward / cca_b200_backward (the time
 * pass adds each output element once, in a fixed order; the generic kernels are deterministic).  Workspace:
 * cca_b200_workspace_bytes3d for the same flags (one size that covers whichever family runs).
 */
CCA_API int cca_b200_tc3d_supported(int which, int B, int Cq, int C, int T, int H, int W, int dtype);
CCA_API size_t cca_b200_workspace_bytes3d(int which, int B, int Cq, int C, int T, int H, int W, int dtype, unsigned flags);
CCA_API int cca_b200_forward3d(const void *q, const void *k, const void *v, void *out, float *lse,
                               void *workspace, size_t workspace_bytes,
                               int B, int Cq, int C, int T, int H, int W, int dtype, unsigned flags, void *cuda_stream);
CCA_API int cca_b200_backward3d(const void *dout, const void *q, const void *k, const void *v,
                                const void *out, const float *lse, void *dq, void *dk, void *dv,
                                void *workspace, size_t workspace_bytes,
                                int B, int Cq, int C, int T, int H, int W, int dtype, unsigned flags, void *cuda_stream);

/*
 * Causal mode (CCA_FLAG_CAUSAL) of the 3D op and its map: pixel (b,t,h,w) attends to its column (self masked), its row and
 * the time keys (b,s,h,w) with s < t only, one softmax over them.  Frame 0 has no time key: its row is the 2D step's.  The
 * map keeps its layout [B,T,H,W,H+W+T]; entries H+W+s with s >= t are exactly 0.  Same coverage, workspace, deterministic
 * mode and limits as without the flag.
 *
 * Time windows of causal mode and the ring-buffer step: the *_window and *_step_ring entry points below.
 *
 * Streaming step: frame S of the causal forward, from the new frame and caches of the S previous frames' keys and values
 * (the queries of past frames do not enter).  q, k [B,Cq,H,W] and v, out [B,C,H,W] of the new frame, k_cache [B,Cq,S,H,W],
 * v_cache [B,C,S,H,W] in time order, lse [B,H,W] fp32.  out and lse equal frame S of cca_b200_forward3d with CCA_FLAG_CAUSAL
 * on the clip whose frames 0..S-1 have keys and values k_cache, v_cache and whose frame S has k, v: bit for bit in fp32 on the
 * tensor-core path on lines of at most 112 pixels and with CCA_FLAG_DETERMINISTIC (longer lines without it: the 2D passes
 * add their partial results in no fixed order, in the clip forward as in the step).  S = 0 (the caches may then be NULL) is the 2D step on the frame.
 * CCA_FLAG_NHWC: q, k, v, out channels-last, the caches NDHWC (torch.channels_last_3d); the tensor-core path, covering what
 * cca_b200_tc3d_supported(CCA_WS_FORWARD, B, Cq, C, S + 1, H, W, dtype) covers (S <= 31).  Without it: NCHW / NCDHW tensors
 * and the generic kernel, any Cq and C, H + W + S - 1 <= 2048.  Flags, alignment and the deterministic mode as for
 * cca_b200_forward3d (16-bit I/O with CCA_FLAG_DETERMINISTIC on tiled lines: CCA_ERR_UNSUPPORTED).  Every argument is checked
 * before any CUDA call (S < 0 and NULL caches with S > 0 are CCA_ERR_INVALID); nothing is written on an error.  No backward:
 * causal training uses cca_b200_forward3d / _backward3d with CCA_FLAG_CAUSAL.
 */
CCA_API size_t cca_b200_workspace_bytes3d_step(int B, int Cq, int C, int S, int H, int W, int dtype, unsigned flags);
CCA_API int cca_b200_forward3d_step(const void *q, const void *k, const void *v, const void *k_cache, const void *v_cache,
                                    void *out, float *lse, void *workspace, size_t workspace_bytes,
                                    int B, int Cq, int C, int S, int H, int W, int dtype, unsigned flags, void *cuda_stream);

/*
 * Time windows of causal mode: the *_window entry points are the ones above with an `int window` before dtype.  window = W
 * >= 1 (with CCA_FLAG_CAUSAL only) limits the time keys of frame t to the frames t - W <= s < t; window = 0 is every past
 * frame (the entry points without the suffix are these with window 0).  The map keeps its layout; a time entry outside
 * [t - W, t) is exactly 0.  With W >= T - 1 the results are bit for bit those of window 0.  The tensor-core coverage is
 * unchanged (1 <= T <= 32); the generic kernels take H + W_img - 1 + min(W, T - 1) <= 2048 (the time keys of a pixel), so a
 * windowed clip may be as long as memory allows.  Workspace: cca_b200_workspace_bytes3d / _attention_workspace_bytes3d.
 * window < 0, or window > 0 without CCA_FLAG_CAUSAL, is CCA_ERR_INVALID, returned before any CUDA call.
 *
 * Ring-buffer step: cca_b200_forward3d_step on rings of N slots, k_ring [B,Cq,N,H,W], v_ring [B,C,N,H,W] (NDHWC with
 * CCA_FLAG_NHWC), holding S <= N past frames, frame j (time order) in slot (head + j) % N.  cca_b200_forward3d_step is this
 * call with N = S, head = 0.  A stream over a window of W frames keeps N = W slots and writes each new frame's k and v into
 * the slot of the oldest one: frame t of the stream, stepped with the min(t, W) frames before it, is frame t of the windowed
 * clip forward (bit for bit where cca_b200_forward3d_step is).  S > N, head outside [0, N) when N > 0 and NULL rings with
 * S > 0 are CCA_ERR_INVALID.  Callers detect these entry points by the presence of their symbols.
 */
CCA_API int cca_b200_forward3d_window(const void *q, const void *k, const void *v, void *out, float *lse,
                                      void *workspace, size_t workspace_bytes,
                                      int B, int Cq, int C, int T, int H, int W, int window, int dtype, unsigned flags,
                                      void *cuda_stream);
CCA_API int cca_b200_backward3d_window(const void *dout, const void *q, const void *k, const void *v,
                                       const void *out, const float *lse, void *dq, void *dk, void *dv,
                                       void *workspace, size_t workspace_bytes,
                                       int B, int Cq, int C, int T, int H, int W, int window, int dtype, unsigned flags,
                                       void *cuda_stream);
CCA_API int cca_b200_attention_forward3d_window(const void *q, const void *k, float *attn, void *workspace, size_t workspace_bytes,
                                                int B, int Cq, int T, int H, int W, int window, int dtype, unsigned flags,
                                                void *cuda_stream);
CCA_API int cca_b200_attention_backward3d_window(const float *dattn, const float *attn, const void *q, const void *k, void *dq,
                                                 void *dk, void *workspace, size_t workspace_bytes,
                                                 int B, int Cq, int T, int H, int W, int window, int dtype, unsigned flags,
                                                 void *cuda_stream);
CCA_API int cca_b200_forward3d_step_ring(const void *q, const void *k, const void *v, const void *k_ring, const void *v_ring,
                                         void *out, float *lse, void *workspace, size_t workspace_bytes,
                                         int B, int Cq, int C, int N, int S, int head, int H, int W, int dtype, unsigned flags,
                                         void *cuda_stream);

/*
 * The attention map of the 3D op above and its gradient:
 *   attn[b,t,h,w,g], fp32 contiguous [B,T,H,W,H+W+T]: g < H the weight of column key (t,g,w) (0 at g == h), H <= g < H+W
 *                   that of row key (t,h,g-H), g >= H+W that of time key (g-H-W,h,w) (0 at g-H-W == t); normalised by the
 *                   lse of cca_b200_forward3d.  At T = 1, attn[...,:H+W] is the 2D map of every frame and attn[...,H+W] is 0.
 *   backward: as for cca_b200_attention_backward, over the H+W+T entries of a row.
 * NDHWC q, k (and dq, dk) with CCA_FLAG_NHWC: the tensor-core path (cca_b200_attention_tc3d_supported: the shapes
 * cca_b200_attention_tc_supported covers for B*T frames, and 1 <= T <= 32).  NCDHW-contiguous q, k: generic kernels of any
 * Cq and shape.  Flags, the deterministic mode and alignment as for cca_b200_attention_forward / _backward: attn and dattn
 * need only the alignment of a float; indices into the map are 64-bit.  Workspace: cca_b200_attention_workspace_bytes3d for
 * the same flags (one size that covers whichever family runs).
 */
CCA_API int cca_b200_attention_tc3d_supported(int B, int Cq, int T, int H, int W, int dtype);
CCA_API size_t cca_b200_attention_workspace_bytes3d(int backward, int B, int Cq, int T, int H, int W, int dtype, unsigned flags);
CCA_API int cca_b200_attention_forward3d(const void *q, const void *k, float *attn, void *workspace, size_t workspace_bytes,
                                         int B, int Cq, int T, int H, int W, int dtype, unsigned flags, void *cuda_stream);
CCA_API int cca_b200_attention_backward3d(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk,
                                          void *workspace, size_t workspace_bytes,
                                          int B, int Cq, int T, int H, int W, int dtype, unsigned flags, void *cuda_stream);

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
