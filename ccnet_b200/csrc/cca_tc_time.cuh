// Pieces of the time branch of the 3D op shared by its kernels (cca_tc_time.cu) and the time kernels of the 3D attention map
// (cca_tc_attn3d.cu): one warp per T-line (the T pixels at a fixed (b, h, w) of an NDHWC clip batch), q and k of the line
// staged in shared memory as fp32.
#pragma once
#include "cca_tc_common.cuh"

namespace cca {
namespace tc {
namespace {

constexpr int kWarps = 4;   // T-lines per CTA

struct TimeParams {
    const void *q, *k, *v, *dout;
    void *out, *dq, *dk, *dv;
    float *part;              // stats: the time plane [B*T*H*W] (log2-sum-exp2 of the T-line logits, self excluded)
    const float *lse;         // final natural-log lse [B*T*H*W]
    const float *delta;       // backward: <dout, out> per pixel (the 2D backward's workspace)
    long lines;               // B*H*W
    long hw;                  // H*W
    int T, Cq, C;
};

// pixel of frame 0 of a T-line (b, hw); frame t is t * hw pixels further
__device__ __forceinline__ long line_pix0(long line, const TimeParams &p)
{
    const long b = line / p.hw;
    return b * p.T * p.hw + (line - b * p.hw);
}

template <typename E>
__device__ __forceinline__ void stage_qk(const TimeParams &p, long pix0, float *qs, float *ks, int lane)
{
    const E *q = static_cast<const E *>(p.q), *k = static_cast<const E *>(p.k);
    const int ld = p.Cq + 1;
    for (int t = 0; t < p.T; ++t) {
        const long base = (pix0 + t * p.hw) * p.Cq;
        for (int c = lane; c < p.Cq; c += 32) {
            qs[t * ld + c] = to_f(q[base + c]);
            ks[t * ld + c] = to_f(k[base + c]);
        }
    }
    __syncwarp();
}

// s[j] = log2e * (q_t . k_j), j < T, of query frame t
template <int TM>
__device__ __forceinline__ void row_logits(const TimeParams &p, const float *qs, const float *ks, int t, float (&s)[TM])
{
    const int ld = p.Cq + 1;
#pragma unroll
    for (int j = 0; j < TM; ++j) s[j] = 0.f;
    for (int c = 0; c < p.Cq; ++c) {
        const float a = qs[t * ld + c];
#pragma unroll
        for (int j = 0; j < TM; ++j)
            if (j < p.T) s[j] = fmaf(a, ks[j * ld + c], s[j]);
    }
#pragma unroll
    for (int j = 0; j < TM; ++j) s[j] *= kLog2e;
}

template <typename E> __device__ __forceinline__ void add_to(E *dst, float x) { *dst = from_f<E>(to_f(*dst) + x); }

// f(std::integral_constant<int, TM>{}): TM, the frames the kernels' register arrays hold, for lines of T frames
template <typename F> decltype(auto) with_time_tier(int T, F &&f)
{
    if (T <= 8) return f(std::integral_constant<int, 8>{});
    if (T <= 16) return f(std::integral_constant<int, 16>{});
    return f(std::integral_constant<int, kTimeMaxT>{});
}

inline TimeParams time_params(Dims3 d)
{
    TimeParams p = {};
    p.lines = (long)d.B * d.H * d.W;
    p.hw = (long)d.H * d.W;
    p.T = d.T; p.Cq = d.Cq; p.C = d.C;
    return p;
}

}  // namespace

// the time statistics pass alone: part[B*T*H*W] = log2-sum-exp2 of each pixel's time logits (self excluded; -inf at T = 1),
// written once the previous launch on the stream has completed (programmatic dependent launch)
cudaError_t tc_time_stats(const void *q, const void *k, float *part, Dims3 d, int dtype, cudaStream_t st);

}  // namespace tc
}  // namespace cca
