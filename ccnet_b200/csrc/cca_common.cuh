// Shared declarations for the criss-cross attention kernels (sm_90a).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/cca_b200.h"

namespace cca {

struct Dims {
    int B, Cq, C, H, W;
};
// a batch of clips [B, C, T, H, W] (the 3D op, cca_tc_time.cu); frames(): the [B*T, C, H, W] view of its frames.  window:
// causal mode's time window (frame t sees the frames t - window .. t - 1; 0: every past frame)
struct Dims3 {
    int B, Cq, C, T, H, W;
    int window;
    Dims frames() const { return Dims{B * T, Cq, C, H, W}; }
    // the most time keys a query frame has: T - 1, or a shorter window
    __host__ __device__ int time_keys() const { return window > 0 && window < T - 1 ? window : T - 1; }
};

// A "line" is one image row (row branch) or one image column (column branch) of a sample.
// Element (channel c, position j) of the line lives at  c*cs + base + j*sj  inside the sample.
struct Line {
    int L;     // positions on the line (W for a row, H for a column)
    long sj;   // stride between positions (1 for a row, W for a column)
    long base; // offset of position 0, channel 0
    long cs;   // channel stride (H*W)
};

template <typename T> __device__ __forceinline__ float to_f(T x);
template <> __device__ __forceinline__ float to_f<float>(float x) { return x; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 x) { return __bfloat162float(x); }
template <> __device__ __forceinline__ float to_f<__half>(__half x) { return __half2float(x); }
template <typename T> __device__ __forceinline__ T from_f(float x);
template <> __device__ __forceinline__ float from_f<float>(float x) { return x; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }
template <> __device__ __forceinline__ __half from_f<__half>(float x) { return __float2half_rn(x); }

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

// f(E{}) with E the element type of a cca_dtype: float, __nv_bfloat16 or __half
template <typename F> decltype(auto) with_elem(int dtype, F &&f)
{
    if (dtype == CCA_F16) return f(__half{});
    if (dtype == CCA_BF16) return f(__nv_bfloat16{});
    return f(float{});
}

// device helpers of the generic kernels
template <typename T> __device__ __forceinline__ float ldg_f(const T *p) { return to_f<T>(__ldg(p)); }
__device__ __forceinline__ float warp_max(float x)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, o));
    return x;
}
__device__ __forceinline__ float warp_sum(float x)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}
// grid of a grid-stride kernel with one warp per pixel and `warps` warps per block
inline int warp_grid(long npix, int warps)
{
    const long want = (npix + warps - 1) / warps;
    return (int)(want < (1L << 20) ? (want > 0 ? want : 1) : (1L << 20));
}

// host-side launchers (defined in the .cu files, called from cca_capi.cu)
//   generic kernels, NCHW tensors (cca_simt.cu); the workspace is the column pass's (m, l) per pixel (forward) or delta
//   (backward)
cudaError_t simt_forward(const void *q, const void *k, const void *v, void *out, float *lse, void *ws,
                         Dims d, int dtype, cudaStream_t st);
cudaError_t simt_backward(const void *dout, const void *q, const void *k, const void *v, const void *out,
                          const float *lse, void *dq, void *dk, void *dv, void *ws, Dims d, int dtype,
                          cudaStream_t st);
bool simt_supported(Dims d, bool backward);
size_t simt_workspace(int which, Dims d);

bool tc_forward_supported(Dims d, int dtype);
size_t tc_forward_workspace(Dims d);
// det: planes mode on tiled lines (fp32 only; the workspace then has tc_planes_bytes more at its end)
cudaError_t tc_forward(const void *q, const void *k, const void *v, void *out, float *lse, void *ws,
                       Dims d, int dtype, cudaStream_t st, const char **why, bool det = false);
// values pass alone (tc_forward = tc_stats + tc_values): the final lse combines the statistics pass's planes and extra_parts
// more planes of `parts`; `planes` is the planes-mode buffer (det on tiled lines)
cudaError_t tc_values(const void *q, const void *k, const void *v, void *out, float *lse, const float *parts, unsigned int *cdone,
                      void *planes, Dims d, int dtype, cudaStream_t st, const char **why, bool det, int extra_parts);
// statistics pre-pass of the tensor-core forward (cca_tc_stats.cu): partial lse planes; also clears n_counters counters
cudaError_t tc_stats(const void *q, const void *k, float *parts, unsigned int *counters, int n_counters, Dims d, int dtype,
                     cudaStream_t st, const char **why);

// deterministic mode on tiled lines (cca_tc_det.cu): fp32 planes-mode item kernels + the plane sum
bool tc_tiled(Dims d);                          // a line longer than one tile in either direction
size_t tc_planes_bytes(int which, Dims d);      // plane workspace (0 on one-tile shapes)
cudaError_t tc_forward_planes(const void *q, const void *k, const void *v, float *out, float *lse, const float *parts,
                              unsigned int *cdone, void *planes, Dims d, cudaStream_t st, const char **why, int extra_parts = 0);
cudaError_t tc_backward_planes(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                               float *delta, unsigned int *counters, float *dq, float *dk, float *dv, void *planes, Dims d,
                               int delta_mode, cudaStream_t st, const char **why);

bool tc_backward_supported(Dims d, int dtype);
size_t tc_backward_workspace(Dims d);
cudaError_t tc_backward(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                        void *dq, void *dk, void *dv, void *ws, Dims d, int dtype, cudaStream_t st, const char **why,
                        bool det = false);

// the 3D op over clips (criss-cross attention along H, W and T; cca_tc_time.cu): the H and W branches are the 2D kernels on
// the frames view of NDHWC tensors, the time branch has kernels of its own.  T up to kTimeMaxT.
constexpr int kTimeMaxT = 32;
bool tc3d_supported(Dims3 d, int dtype);
size_t tc_forward3d_workspace(Dims3 d);
size_t tc_backward3d_workspace(Dims3 d);
cudaError_t tc_forward3d(const void *q, const void *k, const void *v, void *out, float *lse, void *ws, Dims3 d, int dtype,
                         cudaStream_t st, const char **why, bool det);
//   generic kernels, NCDHW tensors of any Cq and C (cca_simt_3d.cu): one warp per pixel, its H + W - 1 + d.time_keys() keys
//   (H + W + T - 2 without a window) in shared memory, so that many <= kMaxKeys3d; the backward's workspace is delta [B*T*H*W]
constexpr int kMaxKeys3d = 2048;
bool simt3d_supported(Dims3 d);
size_t simt3d_workspace(int which, Dims3 d);
cudaError_t simt_forward3d(const void *q, const void *k, const void *v, void *out, float *lse, Dims3 d, int dtype, cudaStream_t st);
cudaError_t simt_backward3d(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                            void *dq, void *dk, void *dv, void *ws, Dims3 d, int dtype, cudaStream_t st);
cudaError_t tc_backward3d(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                          void *dq, void *dk, void *dv, void *ws, Dims3 d, int dtype, cudaStream_t st, const char **why, bool det);
//   causal mode (CCA_FLAG_CAUSAL: the time keys of frame t are the frames t - d.window <= s < t, every s < t at window 0;
//   cca_tc_causal.cu): the same passes and workspaces with the causal time kernels, and the streaming step: frame S of the
//   causal forward from the new frame's q, k, v [B,H,W,c] and rings kc [B,N,H,W,Cq], vc [B,N,H,W,C] holding the S past
//   frames, frame j in slot (head + j) % N (S <= kTimeMaxT - 1; workspace: tc_forward3d_workspace of Dims3{B, Cq, C, 1, H, W})
cudaError_t tc_forward3d_causal(const void *q, const void *k, const void *v, void *out, float *lse, void *ws, Dims3 d, int dtype,
                                cudaStream_t st, const char **why, bool det);
cudaError_t tc_backward3d_causal(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                                 void *dq, void *dk, void *dv, void *ws, Dims3 d, int dtype, cudaStream_t st, const char **why,
                                 bool det);
cudaError_t tc_forward3d_step(const void *q, const void *k, const void *v, const void *kc, const void *vc, void *out, float *lse,
                              void *ws, Dims d, int N, int S, int head, int dtype, cudaStream_t st, const char **why, bool det);
//   generic kernels of causal mode (cca_simt_causal.cu), NCDHW tensors: the forward and backward (same limits and workspace as
//   simt_forward3d / simt_backward3d) and the step on NCHW q, k, v and NCDHW rings (H + W + S - 1 <= kMaxKeys3d)
cudaError_t simt_forward3d_causal(const void *q, const void *k, const void *v, void *out, float *lse, Dims3 d, int dtype,
                                  cudaStream_t st);
cudaError_t simt_backward3d_causal(const void *dout, const void *q, const void *k, const void *v, const void *out,
                                   const float *lse, void *dq, void *dk, void *dv, void *ws, Dims3 d, int dtype, cudaStream_t st);
cudaError_t simt_forward3d_step(const void *q, const void *k, const void *v, const void *kc, const void *vc, void *out, float *lse,
                                Dims d, int N, int S, int head, int dtype, cudaStream_t st);

// the attention map attn[B,H,W,H+W] (fp32) and its gradient w.r.t. q, k (Dims.C is not used)
//   generic kernels, NCHW q, k (cca_simt_attn.cu); the backward's workspace is rho [B*H*W]
size_t simt_attention_workspace(int backward, Dims d);
cudaError_t simt_attention_forward(const void *q, const void *k, float *attn, Dims d, int dtype, cudaStream_t st);
cudaError_t simt_attention_backward(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk,
                                    void *ws, Dims d, int dtype, cudaStream_t st);
//   rho[p] = sum_j attn[p,j] dattn[p,j] over the hw2 entries (H+W; H+W+T for the 3D map) of each of the npix pixels (one warp per pixel, fixed
//   order); also clears clear_bytes at each of c0 and c1 (may be 0)
cudaError_t attn_rho(const float *dattn, const float *attn, float *rho, long npix, int hw2, void *c0, void *c1, long clear_bytes,
                     cudaStream_t st);
//   tensor-core kernels, channels-last q, k (cca_tc_attn.cu); det: planes mode on tiled lines (fp32 only)
bool tc_attention_supported(Dims d, int dtype);
size_t tc_attention_workspace(int backward, Dims d, bool det);
cudaError_t tc_attention_forward(const void *q, const void *k, float *attn, void *ws, Dims d, int dtype, cudaStream_t st,
                                 const char **why);
cudaError_t tc_attention_backward(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk, void *ws,
                                  Dims d, int dtype, cudaStream_t st, const char **why, bool det);

// the attention map of the 3D op, attn[B,T,H,W,H+W+T] (fp32: column, row, time keys) and its gradient w.r.t. q, k
//   generic kernels, NCDHW q, k of any Cq and shape (cca_simt_attn3d.cu); the backward's workspace is rho [B*T*H*W]
size_t simt_attention3d_workspace(int backward, Dims3 d);
cudaError_t simt_attention_forward3d(const void *q, const void *k, float *attn, Dims3 d, int dtype, cudaStream_t st);
cudaError_t simt_attention_backward3d(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk,
                                      void *ws, Dims3 d, int dtype, cudaStream_t st);
//   tensor-core path, NDHWC q, k (cca_tc_attn3d.cu): the 2D map kernels on the frames view + time kernels; T <= kTimeMaxT
bool tc3d_attention_supported(Dims3 d, int dtype);
size_t tc_attention3d_workspace(int backward, Dims3 d, bool det);
cudaError_t tc_attention_forward3d(const void *q, const void *k, float *attn, void *ws, Dims3 d, int dtype, cudaStream_t st,
                                   const char **why);
cudaError_t tc_attention_backward3d(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk, void *ws,
                                    Dims3 d, int dtype, cudaStream_t st, const char **why, bool det);
//   causal mode: the same passes with the causal time map kernels (cca_tc_causal.cu) and the causal generic kernels
//   (cca_simt_causal.cu); the map keeps its layout, time entries s >= t are 0
cudaError_t tc_attention_forward3d_causal(const void *q, const void *k, float *attn, void *ws, Dims3 d, int dtype, cudaStream_t st,
                                          const char **why);
cudaError_t tc_attention_backward3d_causal(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk,
                                           void *ws, Dims3 d, int dtype, cudaStream_t st, const char **why, bool det);
cudaError_t simt_attention_forward3d_causal(const void *q, const void *k, float *attn, Dims3 d, int dtype, cudaStream_t st);
cudaError_t simt_attention_backward3d_causal(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk,
                                             void *ws, Dims3 d, int dtype, cudaStream_t st);

// wgmma GEMMs of the 1x1 Q/K/V projections (cca_gemm.cu), fp32 channels-last tensors as [pixels, channels] matrices
bool qkv_gemm_supported(int C, int Cq);
size_t qkv_gemm_workspace(int C, int Cq);
cudaError_t qkv_project(const float *x, const float *wq, const float *bq, const float *wk, const float *bk, const float *wv, const float *bv,
                        float *q, float *k, float *v, void *ws, long P, int C, int Cq, cudaStream_t st, const char **why);
cudaError_t qkv_project_dgrad(const float *dq, const float *dk, const float *dv, const float *wq, const float *wk, const float *wv,
                              const float *scale, float *dx, void *ws, long P, int C, int Cq, int accumulate, cudaStream_t st,
                              const char **why);
bool qkv_wgrad_supported(int C, int Cq);
// ws != nullptr: deterministic variant (per-split partials in ws, qkv_wgrad_workspace bytes, summed in split order)
cudaError_t qkv_project_wgrad(const float *x, const float *dq, const float *dk, const float *dv, const float *scale, float *dwq,
                              float *dwk, float *dwv, float *db, long P, int C, int Cq, cudaStream_t st, const char **why,
                              void *ws = nullptr);
size_t qkv_wgrad_workspace(int C, int Cq);

void count_launch(int n = 1);
// Launch knobs of the tensor-core kernels, read once from the environment (std::atomic, safe under DataParallel threads):
//   CCA_B200_PDL = 0/1        programmatic dependent launch between the launches of one op (default 1)
//   CCA_B200_DELTA = -1/0/1   backward: -1 automatic, 0 every item computes delta, 1 column items produce it for the sample
//   CCA_B200_LAG = 0/1        item order: consumers of a sample trail its producers by one block (default: 1 in the
//                             backward; picked from the shape in the forward values kernel, cca_tc_fwd.cuh)
//   CCA_B200_L2HINT = 0/1     L2 eviction hints on the bulk copies (default 1)
int tc_pdl();
int tc_delta_mode();
int tc_lag();          // -1 = per-kernel default
int tc_l2_hints();
#ifdef CCA_DEBUG_HOOKS
void set_tc_pdl(int on);
void set_tc_delta_mode(int m);
void set_tc_lag(int v);
void set_tc_l2_hints(int v);
#endif

}  // namespace cca
