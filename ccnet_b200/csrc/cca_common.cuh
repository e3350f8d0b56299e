// Shared declarations for the criss-cross attention kernels (sm_90a).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/cca_b200.h"

namespace cca {

struct Dims {
    int B, Cq, C, H, W;
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
template <typename T> __device__ __forceinline__ T from_f(float x);
template <> __device__ __forceinline__ float from_f<float>(float x) { return x; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

// host-side launchers (defined in the .cu files, called from cca_capi.cu)
cudaError_t simt_forward(const void *q, const void *k, const void *v, void *out, float *lse, void *ws,
                         Dims d, int dtype, cudaStream_t st, const char **why);
cudaError_t simt_backward(const void *dout, const void *q, const void *k, const void *v, const void *out,
                          const float *lse, void *dq, void *dk, void *dv, void *ws, Dims d, int dtype,
                          cudaStream_t st, const char **why);
bool simt_supported(Dims d, bool backward);

bool tc_forward_supported(Dims d, int dtype);
size_t tc_forward_workspace(Dims d);
cudaError_t tc_forward(const void *q, const void *k, const void *v, void *out, float *lse, void *ws,
                       Dims d, int dtype, cudaStream_t st, const char **why);
// statistics pre-pass of the tensor-core forward (cca_tc_stats.cu): partial lse planes; also clears a byte range and counters
cudaError_t tc_stats(const void *q, const void *k, float *parts, void *zero_ptr, long zero_bytes, unsigned int *counters,
                     int n_counters, Dims d, int dtype, cudaStream_t st, const char **why);

bool tc_backward_supported(Dims d, int dtype);
size_t tc_backward_workspace(Dims d);
cudaError_t tc_backward(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                        void *dq, void *dk, void *dv, void *ws, Dims d, int dtype, cudaStream_t st, const char **why);

// wgmma GEMMs of the 1x1 Q/K/V projections (cca_gemm.cu), fp32 channels-last tensors as [pixels, channels] matrices
bool qkv_gemm_supported(int C, int Cq);
size_t qkv_gemm_workspace(int C, int Cq);
cudaError_t qkv_project(const float *x, const float *wq, const float *bq, const float *wk, const float *bk, const float *wv, const float *bv,
                        float *q, float *k, float *v, void *ws, long P, int C, int Cq, cudaStream_t st, const char **why);
cudaError_t qkv_project_dgrad(const float *dq, const float *dk, const float *dv, const float *wq, const float *wk, const float *wv,
                              const float *scale, float *dx, void *ws, long P, int C, int Cq, int accumulate, cudaStream_t st,
                              const char **why);
bool qkv_wgrad_supported(int C, int Cq);
cudaError_t qkv_project_wgrad(const float *x, const float *dq, const float *dk, const float *dv, const float *scale, float *dwq,
                              float *dwk, float *dwv, float *db, long P, int C, int Cq, cudaStream_t st, const char **why);

void count_launch(int n = 1);
// Launch knobs of the tensor-core kernels, read once from the environment (std::atomic, safe under DataParallel threads):
//   CCA_B200_PDL = 0/1        programmatic dependent launch between the launches of one op (default 1)
//   CCA_B200_ZERO_AHEAD = n   the items of sample b clear the outputs of sample b+n (default 1)
//   CCA_B200_DELTA = -1/0/1   backward: -1 automatic, 0 every item computes delta, 1 column items produce it for the sample
//   CCA_B200_LAG = 0/1        item order: consumers of a sample trail its producers by one block (default 1)
//   CCA_B200_L2HINT = 0/1     L2 eviction hints on the bulk copies (default 1)
int tc_pdl();
int tc_zero_ahead();
int tc_delta_mode();
int tc_lag();          // -1 = per-kernel default
int tc_l2_hints();
#ifdef CCA_DEBUG_HOOKS
void set_tc_pdl(int on);
void set_tc_zero_ahead(int n);
void set_tc_delta_mode(int m);
void set_tc_lag(int v);
void set_tc_l2_hints(int v);
#endif

}  // namespace cca
