// Pieces of the time branch of the 3D op shared by its kernels (cca_tc_time.cu; causal: cca_tc_causal.cu) and the time kernels
// of the 3D attention map (cca_tc_attn3d.cu): one warp per T-line (the T pixels at a fixed (b, h, w) of an NDHWC clip batch),
// q and k of the line staged in shared memory as fp32.
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
    int window;               // causal kernels: query frame t sees key frames t - window <= j < t (T: every j < t).  In the
                              // tail padding, so that the bidirectional kernels' parameter layout (and TimeMapParams) is unchanged
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
    p.window = d.window > 0 ? d.window : d.T;
    return p;
}

// Key frame j of query frame t on a line of T frames: every other frame, or with Causal (CCA_FLAG_CAUSAL) the frames before t
// inside the window.  The kernel bodies below take Causal as a template parameter; the kernels of cca_tc_time.cu instantiate
// them with false, those of cca_tc_causal.cu with true.
template <bool Causal> __device__ __forceinline__ bool time_key(int j, int t, const TimeParams &p)
{
    return Causal ? j < t && j >= t - p.window : j < p.T && j != t;
}

enum TimeKind { kStats = 0, kValues = 1, kBackward = 2 };

// floats of shared memory per warp: Q, K [T][Cq+1]; values: + P [T][T+1]; backward: + P, dS [T][T+1], dO, V chunks [T][33]
__host__ __device__ inline long warp_floats(int kind, int T, int Cq)
{
    const long qk = 2L * T * (Cq + 1), pp = (long)T * (T + 1), ch = 32L + 1;
    return kind == kStats ? qk : kind == kValues ? qk + pp : qk + 2 * pp + 2 * T * ch;
}

// lane t < T: P[t][j] = exp2(s_j - lse2_t), 0 where j is not a key of t, into pr and row t of ps
template <int TM, bool Causal>
__device__ __forceinline__ void row_probs(const TimeParams &p, const float *qs, const float *ks, long pix0, int t, float (&pr)[TM],
                                          float *ps)
{
    float s[TM];
    row_logits<TM>(p, qs, ks, t, s);
    const float nl2 = -__ldcg(p.lse + pix0 + t * p.hw) * kLog2e;
#pragma unroll
    for (int j = 0; j < TM; ++j) {
        pr[j] = time_key<Causal>(j, t, p) ? exp2f(s[j] + nl2) : 0.f;
        if (j < p.T) ps[t * (p.T + 1) + j] = pr[j];
    }
}

// the time statistics pass: the time plane (log2-sum-exp2 of every pixel's time logits)
template <int TM, typename E, bool Causal> __device__ __forceinline__ void time_stats(const TimeParams &p)
{
    extern __shared__ float sm[];
    pdl_launch_dependents();                  // the 2D values kernel may start its prologue; it waits for this grid
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long line = (long)blockIdx.x * kWarps + warp;
    const bool ok = line < p.lines;
    float *qs = sm + warp * warp_floats(kStats, p.T, p.Cq), *ks = qs + (long)p.T * (p.Cq + 1);
    const long pix0 = ok ? line_pix0(line, p) : 0;
    float l2 = -INFINITY;                     // (T = 1, and frame 0 when causal: no time key)
    if (ok) {
        stage_qk<E>(p, pix0, qs, ks, lane);
        if (lane < p.T) {
            float s[TM];
            row_logits<TM>(p, qs, ks, lane, s);
            float m = -INFINITY;
#pragma unroll
            for (int j = 0; j < TM; ++j)
                if (time_key<Causal>(j, lane, p)) m = fmaxf(m, s[j]);
            if (m > -INFINITY) {
                float sum = 0.f;
#pragma unroll
                for (int j = 0; j < TM; ++j)
                    if (time_key<Causal>(j, lane, p)) sum += exp2f(s[j] - m);
                l2 = m + log2f(sum);
            }
        }
    }
    pdl_wait();                               // the 2D statistics grid has completed: the values kernel waits for this one only
    if (ok && lane < p.T) p.part[pix0 + lane * p.hw] = l2;
}

// the time values pass: out += P_T V_T with the final lse
template <int TM, typename E, bool Causal> __device__ __forceinline__ void time_values(const TimeParams &p)
{
    extern __shared__ float sm[];
    pdl_wait();                               // out (stored / added by the 2D values kernel) and the final lse
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long line = (long)blockIdx.x * kWarps + warp;
    if (line >= p.lines) return;
    float *qs = sm + warp * warp_floats(kValues, p.T, p.Cq), *ks = qs + (long)p.T * (p.Cq + 1), *ps = ks + (long)p.T * (p.Cq + 1);
    const long pix0 = line_pix0(line, p);
    stage_qk<E>(p, pix0, qs, ks, lane);
    if (lane < p.T) {
        float pr[TM];
        row_probs<TM, Causal>(p, qs, ks, pix0, lane, pr, ps);
    }
    __syncwarp();
    const E *v = static_cast<const E *>(p.v);
    E *out = static_cast<E *>(p.out);
    const int lt = p.T + 1;
    const long fs = p.hw * p.C;               // elements from one frame to the next
    v += pix0 * p.C;
    out += pix0 * p.C;
    for (int c = lane; c < p.C; c += 32) {
        float vr[TM];
#pragma unroll
        for (int j = 0; j < TM; ++j) vr[j] = j < p.T ? to_f(v[j * fs + c]) : 0.f;
        for (int t = 0; t < p.T; ++t) {
            float a = 0.f;
#pragma unroll
            for (int j = 0; j < TM; ++j)
                if (j < p.T) a = fmaf(ps[t * lt + j], vr[j], a);
            add_to(out + t * fs + c, a);
        }
    }
}

// the time backward: the whole T-line in one warp, so dk and dv of key frame s collect dS[t][s] from exactly the query frames
// t that see s (P and dS are 0 elsewhere)
template <int TM, typename E, bool Causal> __device__ __forceinline__ void time_bwd(const TimeParams &p)
{
    extern __shared__ float sm[];
    pdl_wait();                               // dq, dk, dv (written by the 2D backward) and its delta
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long line = (long)blockIdx.x * kWarps + warp;
    if (line >= p.lines) return;
    const int T = p.T, ld = p.Cq + 1, lt = T + 1;
    float *qs = sm + warp * warp_floats(kBackward, T, p.Cq), *ks = qs + (long)T * ld, *ps = ks + (long)T * ld, *ds = ps + T * lt;
    float *gs = ds + T * lt, *vs = gs + T * 33;
    const long pix0 = line_pix0(line, p), hw = p.hw;
    stage_qk<E>(p, pix0, qs, ks, lane);
    float pr[TM], dp[TM];
#pragma unroll
    for (int j = 0; j < TM; ++j) dp[j] = 0.f;
    if (lane < T) row_probs<TM, Causal>(p, qs, ks, pix0, lane, pr, ps);
    __syncwarp();
    // 32 channels at a time: dv[s] += sum_t P[t][s] dO[t] (lane = channel), dP[t][s] += dO[t] . v[s] (lane = frame t)
    const E *dO = static_cast<const E *>(p.dout), *v = static_cast<const E *>(p.v);
    E *dv = static_cast<E *>(p.dv);
    for (int c0 = 0; c0 < p.C; c0 += 32) {
        const int c = c0 + lane;              // (C % 64 == 0 on this path)
        for (int t = 0; t < T; ++t) {
            const long e = (pix0 + t * hw) * p.C + c;
            gs[t * 33 + lane] = to_f(dO[e]);
            vs[t * 33 + lane] = to_f(v[e]);
        }
        __syncwarp();
        for (int s = 0; s < T; ++s) {
            float a = 0.f;
            for (int t = 0; t < T; ++t) a = fmaf(ps[t * lt + s], gs[t * 33 + lane], a);
            add_to(dv + (pix0 + s * hw) * p.C + c, a);
        }
        if (lane < T)
            for (int cc = 0; cc < 32; ++cc) {
                const float g = gs[lane * 33 + cc];
#pragma unroll
                for (int j = 0; j < TM; ++j)
                    if (j < T) dp[j] = fmaf(g, vs[j * 33 + cc], dp[j]);
            }
        __syncwarp();
    }
    // dS = P (dP - delta)
    if (lane < T) {
        const float dl = __ldcg(p.delta + pix0 + lane * hw);
#pragma unroll
        for (int j = 0; j < TM; ++j)
            if (j < T) ds[lane * lt + j] = pr[j] * (dp[j] - dl);
    }
    __syncwarp();
    // dq[t] += sum_s dS[t][s] k[s],  dk[s] += sum_t dS[t][s] q[t]   (lane = channel)
    E *dq = static_cast<E *>(p.dq), *dk = static_cast<E *>(p.dk);
    for (int c = lane; c < p.Cq; c += 32)
        for (int t = 0; t < T; ++t) {
            float a = 0.f, b = 0.f;
            for (int j = 0; j < T; ++j) {
                a = fmaf(ds[t * lt + j], ks[j * ld + c], a);
                b = fmaf(ds[j * lt + t], qs[j * ld + c], b);
            }
            add_to(dq + (pix0 + t * hw) * p.Cq + c, a);
            add_to(dk + (pix0 + t * hw) * p.Cq + c, b);
        }
}

// one launch of a time kernel: kWarps lines per CTA, `floats` of shared memory per warp
template <typename P> cudaError_t launch_lines(void (*kern)(P), long lines, long floats, const P &p, cudaStream_t st)
{
    const unsigned grid = (unsigned)((lines + kWarps - 1) / kWarps);
    return launch_kernel(kern, grid, 32 * kWarps, (size_t)kWarps * floats * sizeof(float), true, st, p);
}

// The passes of the 3D forward and backward on the tensor-core path.  launch(kind, p) runs the time kernel of `kind`; the
// caller picks the causal or the bidirectional kernels.
template <typename Launch>
cudaError_t forward3d_passes(Launch &&launch, const void *q, const void *k, const void *v, void *out, float *lse, void *ws, Dims3 d,
                             int dtype, cudaStream_t st, const char **why, bool det)
{
    const Dims f = d.frames();
    const FwdWs w = fwd_ws(f, 1, ws);
    cudaError_t e = tc_stats(q, k, w.parts, w.cdone, f.B, f, dtype, st, why);
    if (e != cudaSuccess) return e;
    TimeParams p = time_params(d);
    p.q = q; p.k = k; p.v = v; p.out = out; p.lse = lse;
    p.part = w.parts + (long)make_space(f.B, f.H, f.W).nparts * f.B * f.H * f.W;
    if ((e = launch(kStats, p)) != cudaSuccess) return e;
    e = tc_values(q, k, v, out, lse, w.parts, w.cdone, w.planes, f, dtype, st, why, det, 1);
    if (e != cudaSuccess) return e;
    return launch(kValues, p);
}

template <typename Launch>
cudaError_t backward3d_passes(Launch &&launch, const void *dout, const void *q, const void *k, const void *v, const void *out,
                              const float *lse, void *dq, void *dk, void *dv, void *ws, Dims3 d, int dtype, cudaStream_t st,
                              const char **why, bool det)
{
    cudaError_t e = tc_backward(dout, q, k, v, out, lse, dq, dk, dv, ws, d.frames(), dtype, st, why, det);
    if (e != cudaSuccess) return e;
    TimeParams p = time_params(d);
    p.q = q; p.k = k; p.v = v; p.dout = dout; p.lse = lse;
    p.dq = dq; p.dk = dk; p.dv = dv;
    p.delta = bwd_ws(d.frames(), ws).delta;             // (left there by tc_backward)
    return launch(kBackward, p);
}

}  // namespace

// the time statistics pass alone: part[B*T*H*W] = log2-sum-exp2 of each pixel's time logits (self excluded; -inf at T = 1),
// written once the previous launch on the stream has completed (programmatic dependent launch)
cudaError_t tc_time_stats(const void *q, const void *k, float *part, Dims3 d, int dtype, cudaStream_t st);

}  // namespace tc
}  // namespace cca
