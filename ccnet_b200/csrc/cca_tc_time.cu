// Criss-cross attention over clips (the 3D op): q, k [B, Cq, T, H, W], v [B, C, T, H, W] in NDHWC memory
// (torch.channels_last_3d).  Every pixel (b, t, h, w) attends to its column (b, t, *, w; self masked), its row (b, t, h, *)
// and its time line (b, *, h, w; self masked), one softmax over all H + W + T logits.
//
// In NDHWC memory the frames view [B*T, H, W, C] of a clip batch is an ordinary NHWC tensor whose pixel index is the clip's
// pixel index, so the column and row branches are the 2D tensor-core kernels run unchanged on that view:
//   forward : 2D statistics -> time statistics (one more partial lse plane) -> 2D values with that plane folded into the
//             final lse (launch_fwd's extra_parts) -> time values (out += P_T V_T with the final lse)
//   backward: 2D backward with the 3D lse and out (its P is the 3D P restricted to a row / column, its delta = <dO, out> is
//             the 3D delta, left in its workspace) -> time backward
// The passes are chained with programmatic dependent launch; each time kernel waits (griddepcontrol.wait) before it writes
// or reads what an earlier pass wrote.
//
// Time kernels: one warp owns one T-line (the T pixels at a fixed (b, h, w)).  Lane t < T is query frame t for the T x T
// logits, P and dS (staged in shared memory); for the products with V, dO, Q and K the lanes walk the channels.  A T-line
// lives in one warp, so each output element gets exactly one add from the time pass: no atomics, and the result is as
// reproducible as the 2D passes before it (CCA_FLAG_DETERMINISTIC needs no planes here).  The pass moves ~(2Cq + 3C)
// elements per pixel for 2T(Cq + C) FLOPs, bandwidth-bound on CUDA cores, so it uses no tensor cores.  The shared memory
// per warp grows with T * Cq; kTimeMaxT = 32 keeps the backward's four warps under 140 KB.
#include "cca_items.cuh"
#include "cca_tc_time.cuh"

namespace cca {
namespace tc {
namespace {

enum TimeKind { kStats = 0, kValues = 1, kBackward = 2 };

// floats of shared memory per warp: Q, K [T][Cq+1]; values: + P [T][T+1]; backward: + P, dS [T][T+1], dO, V chunks [T][33]
__host__ __device__ inline long warp_floats(int kind, int T, int Cq)
{
    const long qk = 2L * T * (Cq + 1), pp = (long)T * (T + 1), ch = 32L + 1;
    return kind == kStats ? qk : kind == kValues ? qk + pp : qk + 2 * pp + 2 * T * ch;
}

// lane t < T: P[t][j] = exp2(s_j - lse2_t), 0 at j == t, into pr and row t of ps
template <int TM>
__device__ __forceinline__ void row_probs(const TimeParams &p, const float *qs, const float *ks, long pix0, int t, float (&pr)[TM],
                                          float *ps)
{
    float s[TM];
    row_logits<TM>(p, qs, ks, t, s);
    const float nl2 = -__ldcg(p.lse + pix0 + t * p.hw) * kLog2e;
#pragma unroll
    for (int j = 0; j < TM; ++j) {
        pr[j] = j < p.T && j != t ? exp2f(s[j] + nl2) : 0.f;
        if (j < p.T) ps[t * (p.T + 1) + j] = pr[j];
    }
}

template <int TM, typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_stats_kernel(const __grid_constant__ TimeParams p)
{
    extern __shared__ float sm[];
    pdl_launch_dependents();                  // the 2D values kernel may start its prologue; it waits for this grid
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long line = (long)blockIdx.x * kWarps + warp;
    const bool ok = line < p.lines;
    float *qs = sm + warp * warp_floats(kStats, p.T, p.Cq), *ks = qs + (long)p.T * (p.Cq + 1);
    const long pix0 = ok ? line_pix0(line, p) : 0;
    float l2 = -INFINITY;                     // (T = 1: no time key)
    if (ok) {
        stage_qk<E>(p, pix0, qs, ks, lane);
        if (lane < p.T) {
            float s[TM];
            row_logits<TM>(p, qs, ks, lane, s);
            float m = -INFINITY;
#pragma unroll
            for (int j = 0; j < TM; ++j)
                if (j < p.T && j != lane) m = fmaxf(m, s[j]);
            if (m > -INFINITY) {
                float sum = 0.f;
#pragma unroll
                for (int j = 0; j < TM; ++j)
                    if (j < p.T && j != lane) sum += exp2f(s[j] - m);
                l2 = m + log2f(sum);
            }
        }
    }
    pdl_wait();                               // the 2D statistics grid has completed: the values kernel waits for this one only
    if (ok && lane < p.T) p.part[pix0 + lane * p.hw] = l2;
}

template <int TM, typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_values_kernel(const __grid_constant__ TimeParams p)
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
        row_probs<TM>(p, qs, ks, pix0, lane, pr, ps);
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

template <int TM, typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_bwd_kernel(const __grid_constant__ TimeParams p)
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
    if (lane < T) row_probs<TM>(p, qs, ks, pix0, lane, pr, ps);
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

cudaError_t launch_time(int kind, const TimeParams &p, int dtype, cudaStream_t st)
{
    const unsigned grid = (unsigned)((p.lines + kWarps - 1) / kWarps);
    const size_t smem = (size_t)kWarps * warp_floats(kind, p.T, p.Cq) * sizeof(float);
    return with_elem(dtype, [&](auto e) {
        using E = decltype(e);
        auto tier = [&](auto tm) {
            constexpr int TM = decltype(tm)::value;
            void (*kern)(TimeParams) = kind == kStats    ? cca_time_stats_kernel<TM, E>
                                       : kind == kValues ? cca_time_values_kernel<TM, E>
                                                         : cca_time_bwd_kernel<TM, E>;
            return launch_kernel(kern, grid, 32 * kWarps, smem, true, st, p);
        };
        return with_time_tier(p.T, tier);
    });
}

}  // namespace

cudaError_t tc_time_stats(const void *q, const void *k, float *part, Dims3 d, int dtype, cudaStream_t st)
{
    TimeParams p = time_params(d);
    p.q = q; p.k = k; p.part = part;
    return launch_time(kStats, p, dtype, st);
}

}  // namespace tc

using namespace tc;

bool tc3d_supported(Dims3 d, int dtype)
{
    return d.T >= 1 && d.T <= kTimeMaxT && (long)d.B * d.T < (1L << 31) && shape_supported(d.frames(), dtype);
}

// Workspace of the 3D forward: that of the 2D forward on the frames view with one more partial lse plane, the time plane
// (planes mode: tc_planes_bytes of the frames view follow).
size_t tc_forward3d_workspace(Dims3 d) { return fwd_ws(d.frames(), 1, nullptr).bytes; }

// Workspace of the 3D backward: that of the 2D backward on the frames view (delta first)
size_t tc_backward3d_workspace(Dims3 d) { return tc_backward_workspace(d.frames()); }

cudaError_t tc_forward3d(const void *q, const void *k, const void *v, void *out, float *lse, void *ws, Dims3 d, int dtype,
                         cudaStream_t st, const char **why, bool det)
{
    const Dims f = d.frames();
    const FwdWs w = fwd_ws(f, 1, ws);
    cudaError_t e = tc_stats(q, k, w.parts, w.cdone, f.B, f, dtype, st, why);
    if (e != cudaSuccess) return e;
    TimeParams p = time_params(d);
    p.q = q; p.k = k; p.v = v; p.out = out; p.lse = lse;
    p.part = w.parts + (long)make_space(f.B, f.H, f.W).nparts * f.B * f.H * f.W;
    if ((e = launch_time(kStats, p, dtype, st)) != cudaSuccess) return e;
    e = tc_values(q, k, v, out, lse, w.parts, w.cdone, w.planes, f, dtype, st, why, det, 1);
    if (e != cudaSuccess) return e;
    return launch_time(kValues, p, dtype, st);
}

cudaError_t tc_backward3d(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                          void *dq, void *dk, void *dv, void *ws, Dims3 d, int dtype, cudaStream_t st, const char **why, bool det)
{
    cudaError_t e = tc_backward(dout, q, k, v, out, lse, dq, dk, dv, ws, d.frames(), dtype, st, why, det);
    if (e != cudaSuccess) return e;
    TimeParams p = time_params(d);
    p.q = q; p.k = k; p.v = v; p.dout = dout; p.lse = lse;
    p.dq = dq; p.dk = dk; p.dv = dv;
    p.delta = bwd_ws(d.frames(), ws).delta;             // (left there by tc_backward)
    return launch_time(kBackward, p, dtype, st);
}

}  // namespace cca
