// Causal criss-cross attention over clips on the tensor-core path (CCA_FLAG_CAUSAL): pixel (b, t, h, w) attends to its column
// (self masked), its row and the time keys (b, s, h, w) with t - window <= s < t only, one softmax over them.  Only the time
// kernels change: they are the bodies of cca_tc_time.cuh and cca_tc_attn3d.cuh instantiated with Causal = true (logits of key
// frames t - window <= j < t where the bidirectional kernels take j != t; the window is a run-time field, T when unbounded,
// so a window needs no kernels of its own), run in the same passes.  Frame 0 has no time key: its time plane is -inf, so
// its row is the 2D op's row, as at T = 1.  The time backward owns a whole T-line in one warp, so dk and dv of key frame s
// collect dS[t][s] from the query frames t > s only (P and dS are 0 elsewhere), with no other change.
//
// The streaming step (tc_forward3d_step): frame S of the causal clip forward, computed from the new frame's q, k, v and rings
// of capacity N holding the S previous frames' k and v (frame j in slot (head + j) % N), without the past queries.  It composes the forward's passes on the new frame:
//   2D statistics on the frame's NHWC view (B frames) -> time step statistics (query: the new frame; keys: the S cached frames
//   at the same (h, w); no self entry) into one more lse plane -> 2D values with that plane (extra_parts = 1) -> time step
//   values (out += P_T V_cache with the final lse)
// chained with programmatic dependent launch.  The step kernels give each cached frame j < S one lane (S <= 31) and compute
// every value with the operations, in the order, of the clip kernels for the last frame of a clip of S + 1 frames: the logit
// sum_c fmaf(q_c, k_jc) over c ascending, times log2e, the max, the sum of exp2(s_j - m) over j ascending, m + log2(sum),
// P_j = exp2(fma(logit, log2e, -lse log2e)) (the contraction the clip's values kernel compiles to), and
// out += sum_j fmaf(P_j, v_jc) over j ascending.  The fp32 step is therefore bit-identical to frame S of the causal clip
// forward (the 2D passes compute a frame alike whatever the batch around it).
#include "cca_tc_attn3d.cuh"

namespace cca {
namespace tc {
namespace {

template <int TM, typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_causal_stats_kernel(const __grid_constant__ TimeParams p)
{
    time_stats<TM, E, true>(p);
}

template <int TM, typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_causal_values_kernel(const __grid_constant__ TimeParams p)
{
    time_values<TM, E, true>(p);
}

template <int TM, typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_causal_bwd_kernel(const __grid_constant__ TimeParams p)
{
    time_bwd<TM, E, true>(p);
}

template <int TM, typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_causal_map_fwd_kernel(const __grid_constant__ TimeMapParams p)
{
    time_map_fwd<TM, E, true>(p);
}

template <int TM, typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_causal_map_bwd_kernel(const __grid_constant__ TimeMapParams p)
{
    time_map_bwd<TM, E, true>(p);
}

cudaError_t launch_time(int kind, const TimeParams &p, int dtype, cudaStream_t st)
{
    return with_elem(dtype, [&](auto e) {
        using E = decltype(e);
        return with_time_tier(p.T, [&](auto tm) {
            constexpr int TM = decltype(tm)::value;
            void (*kern)(TimeParams) = kind == kStats    ? cca_time_causal_stats_kernel<TM, E>
                                       : kind == kValues ? cca_time_causal_values_kernel<TM, E>
                                                         : cca_time_causal_bwd_kernel<TM, E>;
            return launch_lines(kern, p.lines, warp_floats(kind, p.T, p.Cq), p, st);
        });
    });
}

cudaError_t launch_time_map(bool backward, const TimeMapParams &p, int dtype, cudaStream_t st)
{
    return with_elem(dtype, [&](auto e) {
        using E = decltype(e);
        return with_time_tier(p.t.T, [&](auto tm) {
            constexpr int TM = decltype(tm)::value;
            return launch_lines(backward ? cca_time_causal_map_bwd_kernel<TM, E> : cca_time_causal_map_fwd_kernel<TM, E>, p.t.lines,
                                map_warp_floats(backward, p.t.T, p.t.Cq), p, st);
        });
    });
}

// ---- the streaming step
struct StepParams {
    const void *q;            // the new frame's q [B*H*W, Cq]
    const void *kc, *vc;      // the rings [B, N, H, W, Cq], [B, N, H, W, C]: past frame j < S in slot (head + j) % N
    void *out;                // the new frame's out [B*H*W, C]
    float *part;              // stats: the time plane [B*H*W]
    const float *lse;         // values: the final natural-log lse [B*H*W]
    long lines;               // B*H*W: one warp per pixel of the new frame
    long hw;                  // H*W
    int S, Cq, C;
    int N, head;
};

// slot of past frame j in the rings
__device__ __forceinline__ long step_slot(const StepParams &p, int j)
{
    const int s = p.head + j;
    return s < p.N ? s : s - p.N;
}

// floats of shared memory per warp: q [Cq+1], the cached keys K [S][Cq+1], one float per lane
__host__ __device__ inline long step_floats(int S, int Cq) { return (long)(S + 1) * (Cq + 1) + 32; }

// q and the S cached keys of pixel `line` staged as fp32; lane j < S returns q . k_j, the c-ascending FMA chain of row_logits.
// The callers scale it by log2e the way the clip kernels' code compiles: a separate multiply in the statistics (the scaled
// logit also feeds the max), fused into the exponent's FMA in the values (exp2(fma(s, log2e, -lse log2e))).
template <typename E> __device__ __forceinline__ float step_logit(const StepParams &p, long line, float *qs, float *ks, int lane)
{
    const long b = line / p.hw, x = line - b * p.hw;
    const E *q = static_cast<const E *>(p.q) + line * p.Cq, *k = static_cast<const E *>(p.kc) + (b * p.N * p.hw + x) * p.Cq;
    const int ld = p.Cq + 1;
    for (int c = lane; c < p.Cq; c += 32) qs[c] = to_f(q[c]);
    for (int j = 0; j < p.S; ++j) {
        const E *kj = k + step_slot(p, j) * p.hw * p.Cq;
        for (int c = lane; c < p.Cq; c += 32) ks[j * ld + c] = to_f(kj[c]);
    }
    __syncwarp();
    float s = 0.f;
    if (lane < p.S)
        for (int c = 0; c < p.Cq; ++c) s = fmaf(qs[c], ks[lane * ld + c], s);
    return s;
}

template <typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_step_stats_kernel(const __grid_constant__ StepParams p)
{
    extern __shared__ float sm[];
    pdl_launch_dependents();                  // the 2D values kernel may start its prologue; it waits for this grid
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long line = (long)blockIdx.x * kWarps + warp;
    const bool ok = line < p.lines;
    float *qs = sm + warp * step_floats(p.S, p.Cq), *ks = qs + p.Cq + 1, *es = ks + (long)p.S * (p.Cq + 1);
    float l2 = -INFINITY;                     // (S = 0: no time key)
    if (ok) {
        const float s = __fmul_rn(step_logit<E>(p, line, qs, ks, lane), kLog2e);
        const float m = warp_max(lane < p.S ? s : -INFINITY);
        if (m > -INFINITY) {
            es[lane] = lane < p.S ? exp2f(s - m) : 0.f;
            __syncwarp();
            float sum = 0.f;
            for (int j = 0; j < p.S; ++j) sum += es[j];
            l2 = m + log2f(sum);
        }
    }
    pdl_wait();                               // the 2D statistics grid has completed: the values kernel waits for this one only
    if (ok && lane == 0) p.part[line] = l2;
}

template <typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_step_values_kernel(const __grid_constant__ StepParams p)
{
    extern __shared__ float sm[];
    pdl_wait();                               // out (stored / added by the 2D values kernel) and the final lse
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long line = (long)blockIdx.x * kWarps + warp;
    if (line >= p.lines) return;
    float *qs = sm + warp * step_floats(p.S, p.Cq), *ks = qs + p.Cq + 1, *ps = ks + (long)p.S * (p.Cq + 1);
    const float s = step_logit<E>(p, line, qs, ks, lane);
    const float nl2 = -__ldcg(p.lse + line) * kLog2e;
    if (lane < p.S) ps[lane] = exp2f(fmaf(s, kLog2e, nl2));
    __syncwarp();
    const long b = line / p.hw, x = line - b * p.hw, fs = p.hw * p.C;
    const E *v = static_cast<const E *>(p.vc) + (b * p.N * p.hw + x) * p.C;
    E *out = static_cast<E *>(p.out) + line * p.C;
    for (int c = lane; c < p.C; c += 32) {
        float a = 0.f;
        for (int j = 0; j < p.S; ++j) a = fmaf(ps[j], to_f(v[step_slot(p, j) * fs + c]), a);
        add_to(out + c, a);
    }
}

cudaError_t launch_step(bool stats, const StepParams &p, int dtype, cudaStream_t st)
{
    return with_elem(dtype, [&](auto e) {
        using E = decltype(e);
        return launch_lines(stats ? cca_time_step_stats_kernel<E> : cca_time_step_values_kernel<E>, p.lines, step_floats(p.S, p.Cq), p,
                            st);
    });
}

}  // namespace
}  // namespace tc

using namespace tc;

cudaError_t tc_forward3d_causal(const void *q, const void *k, const void *v, void *out, float *lse, void *ws, Dims3 d, int dtype,
                                cudaStream_t st, const char **why, bool det)
{
    return forward3d_passes([&](int kind, const TimeParams &p) { return launch_time(kind, p, dtype, st); }, q, k, v, out, lse, ws,
                            d, dtype, st, why, det);
}

cudaError_t tc_backward3d_causal(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                                 void *dq, void *dk, void *dv, void *ws, Dims3 d, int dtype, cudaStream_t st, const char **why,
                                 bool det)
{
    return backward3d_passes([&](int kind, const TimeParams &p) { return launch_time(kind, p, dtype, st); }, dout, q, k, v, out,
                             lse, dq, dk, dv, ws, d, dtype, st, why, det);
}

cudaError_t tc_attention_forward3d_causal(const void *q, const void *k, float *attn, void *ws, Dims3 d, int dtype, cudaStream_t st,
                                          const char **why)
{
    auto stats = [&](float *part) {
        TimeParams p = time_params(d);
        p.q = q; p.k = k; p.part = part;
        return launch_time(kStats, p, dtype, st);
    };
    return attention_forward3d_passes(stats, [&](bool backward, const TimeMapParams &p) { return launch_time_map(backward, p, dtype, st); },
                                      q, k, attn, ws, d, dtype, st, why);
}

cudaError_t tc_attention_backward3d_causal(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk,
                                           void *ws, Dims3 d, int dtype, cudaStream_t st, const char **why, bool det)
{
    return attention_backward3d_passes([&](bool backward, const TimeMapParams &p) { return launch_time_map(backward, p, dtype, st); },
                                       dattn, attn, q, k, dq, dk, ws, d, dtype, st, why, det);
}

// the step's workspace is the forward workspace of one frame (fwd_ws with the time plane; planes mode: tc_planes_bytes follow)
cudaError_t tc_forward3d_step(const void *q, const void *k, const void *v, const void *kc, const void *vc, void *out, float *lse,
                              void *ws, Dims d, int N, int S, int head, int dtype, cudaStream_t st, const char **why, bool det)
{
    const FwdWs w = fwd_ws(d, 1, ws);
    cudaError_t e = tc_stats(q, k, w.parts, w.cdone, d.B, d, dtype, st, why);
    if (e != cudaSuccess) return e;
    StepParams p = {};
    p.q = q; p.kc = kc; p.vc = vc; p.out = out; p.lse = lse;
    p.lines = (long)d.B * d.H * d.W;
    p.hw = (long)d.H * d.W;
    p.part = w.parts + (long)make_space(d.B, d.H, d.W).nparts * p.lines;
    p.S = S; p.Cq = d.Cq; p.C = d.C;
    p.N = N; p.head = head;
    if ((e = launch_step(true, p, dtype, st)) != cudaSuccess) return e;
    e = tc_values(q, k, v, out, lse, w.parts, w.cdone, w.planes, d, dtype, st, why, det, 1);
    if (e != cudaSuccess) return e;
    return launch_step(false, p, dtype, st);
}

}  // namespace cca
