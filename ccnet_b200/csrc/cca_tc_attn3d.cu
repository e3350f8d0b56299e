// The attention map of criss-cross attention over clips (the 3D op) on the tensor-core path: q, k [B, Cq, T, H, W] in NDHWC
// memory (torch.channels_last_3d), attn [B, T, H, W, H+W+T] fp32 with each row ordered column keys (g < H; self entry 0),
// row keys (H <= g < H+W), time keys (g = H+W+s; self entry s = t is 0).
//
// In NDHWC memory the frames view [B*T, H, W, Cq] is an ordinary NHWC tensor, so the column and row entries are the 2D map
// kernels (cca_tc_attn.cuh) run on that view with rows of H + W + T entries:
//   forward : 2D statistics -> time statistics (cca_tc_time.cu, one more partial lse plane) -> 2D map kernel with that plane
//             folded into its lse combine -> time map kernel (the T time entries of every row, from the same planes and the
//             same combine, so the whole row is normalised by one lse, bit for bit)
//   backward: rho over the whole row (also clears dq, dk) -> 2D map item kernel (planes mode: + planes_sum) -> time map
//             backward: dS_t = attn_t (dattn_t - rho), dq += dS_t K_T, dk += dS_t^T Q_T
// The passes are chained with programmatic dependent launch.  The time kernels are those of the 3D op's time branch: one
// warp per T-line, q and k of the line in shared memory, plain fp32 FMA; each dq / dk element gets one read-add-write from
// the time pass, so the backward is as reproducible as the 2D passes before it.
#include "cca_tc_attn.cuh"
#include "cca_tc_time.cuh"

namespace cca {
namespace tc {
namespace {

struct TimeMapParams {
    TimeParams t;              // q, k and the shape of the lines (T, Cq, hw, lines)
    const float *parts;        // forward: [nparts][npix] partial log2-sum-exp2 planes, the time plane last
    int nparts;
    long npix;                 // B*T*H*W
    long row;                  // H + W + T: the map's row length
    int off;                   // H + W: the first time entry of a row
    float *attn;               // forward: the map
    const float *map, *dattn, *rho;   // backward: the forward's map, its gradient, rho
};

// floats of shared memory per warp: Q, K [T][Cq+1]; backward: + dS [T][T+1]
__host__ __device__ inline long map_warp_floats(bool backward, int T, int Cq)
{
    return 2L * T * (Cq + 1) + (backward ? (long)T * (T + 1) : 0);
}

template <int TM, typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_map_fwd_kernel(const __grid_constant__ TimeMapParams p)
{
    extern __shared__ float sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long line = (long)blockIdx.x * kWarps + warp;
    if (line >= p.t.lines) return;
    float *qs = sm + warp * map_warp_floats(false, p.t.T, p.t.Cq), *ks = qs + (long)p.t.T * (p.t.Cq + 1);
    const long pix0 = line_pix0(line, p.t);
    stage_qk<E>(p.t, pix0, qs, ks, lane);
    pdl_wait();                                // the lse planes (complete with the map kernel launched before this one)
    if (lane < p.t.T) {
        float s[TM];
        row_logits<TM>(p.t, qs, ks, lane, s);
        const long pix = pix0 + lane * p.t.hw;
        const float nl2 = -combine_lse2<0>(nullptr, p.parts, p.npix, p.nparts, pix);
        float *row = p.attn + pix * p.row + p.off;
#pragma unroll
        for (int j = 0; j < TM; ++j)
            if (j < p.t.T) row[j] = j == lane ? 0.f : exp2f(s[j] + nl2);
    }
}

template <int TM, typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_map_bwd_kernel(const __grid_constant__ TimeMapParams p)
{
    extern __shared__ float sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long line = (long)blockIdx.x * kWarps + warp;
    if (line >= p.t.lines) return;
    const int T = p.t.T, ld = p.t.Cq + 1, lt = T + 1;
    float *qs = sm + warp * map_warp_floats(true, T, p.t.Cq), *ks = qs + (long)T * ld, *ds = ks + (long)T * ld;
    const long pix0 = line_pix0(line, p.t), hw = p.t.hw;
    stage_qk<E>(p.t, pix0, qs, ks, lane);
    pdl_wait();                                // rho, and dq, dk complete (the 2D map backward or its plane sum)
    if (lane < T) {
        const long pix = pix0 + lane * hw;
        const float rho = __ldcg(p.rho + pix);
        const float *a = p.map + pix * p.row + p.off, *d = p.dattn + pix * p.row + p.off;
        for (int j = 0; j < T; ++j) ds[lane * lt + j] = j == lane ? 0.f : __ldg(a + j) * (__ldg(d + j) - rho);
    }
    __syncwarp();
    // dq[t] += sum_s dS[t][s] k[s],  dk[s] += sum_t dS[t][s] q[t]   (lane = channel)
    E *dq = static_cast<E *>(p.t.dq), *dk = static_cast<E *>(p.t.dk);
    for (int c = lane; c < p.t.Cq; c += 32)
        for (int t = 0; t < T; ++t) {
            float a = 0.f, b = 0.f;
            for (int j = 0; j < T; ++j) {
                a = fmaf(ds[t * lt + j], ks[j * ld + c], a);
                b = fmaf(ds[j * lt + t], qs[j * ld + c], b);
            }
            add_to(dq + (pix0 + t * hw) * p.t.Cq + c, a);
            add_to(dk + (pix0 + t * hw) * p.t.Cq + c, b);
        }
}

cudaError_t launch_time_map(bool backward, const TimeMapParams &p, int dtype, cudaStream_t st)
{
    const unsigned grid = (unsigned)((p.t.lines + kWarps - 1) / kWarps);
    const size_t smem = (size_t)kWarps * map_warp_floats(backward, p.t.T, p.t.Cq) * sizeof(float);
    return with_elem(dtype, [&](auto e) {
        return with_time_tier(p.t.T, [&](auto tm) {
            constexpr int TM = decltype(tm)::value;
            using E = decltype(e);
            return launch_kernel(backward ? cca_time_map_bwd_kernel<TM, E> : cca_time_map_fwd_kernel<TM, E>, grid, 32 * kWarps, smem,
                                 true, st, p);
        });
    });
}

TimeMapParams map_params(Dims3 d)
{
    TimeMapParams p = {};
    p.t = time_params(d);
    p.npix = (long)d.B * d.T * d.H * d.W;
    p.row = (long)d.H + d.W + d.T;
    p.off = d.H + d.W;
    return p;
}

}  // namespace
}  // namespace tc

using namespace tc;

bool tc3d_attention_supported(Dims3 d, int dtype)
{
    return d.T >= 1 && d.T <= kTimeMaxT && (long)d.B * d.T < (1L << 31) && tc_attention_supported(d.frames(), dtype);
}

// forward: the 3D forward's statistics workspace (the frames view's planes, the time plane, counters); backward: that of
// the 2D map backward on the frames view (rho, then the planes-mode dQ, dK planes)
size_t tc_attention3d_workspace(int backward, Dims3 d, bool det)
{
    Dims f = d.frames();
    f.C = kNC;
    return backward ? attn_bwd_ws(f, det, nullptr).bytes : fwd_ws(f, 1, nullptr).bytes;
}

cudaError_t tc_attention_forward3d(const void *q, const void *k, float *attn, void *ws, Dims3 d, int dtype, cudaStream_t st,
                                   const char **why)
{
    const Dims f = d.frames();
    float *parts = fwd_ws(f, 1, ws).parts;
    cudaError_t e = tc_stats(q, k, parts, nullptr, 0, f, dtype, st, why);
    if (e != cudaSuccess) return e;
    TimeMapParams p = map_params(d);
    p.t.q = q; p.t.k = k;
    p.parts = parts;
    p.nparts = make_space(f.B, f.H, f.W).nparts + 1;
    p.attn = attn;
    if ((e = tc_time_stats(q, k, parts + (p.nparts - 1) * p.npix, d, dtype, st)) != cudaSuccess) return e;
    e = with_elem_tile(dtype, f, [&](auto el, auto lk) {
        return launch_attn_fwd<lk(), decltype(el), true>(q, k, attn, parts, f, d.T, st, why);
    });
    if (e != cudaSuccess) return e;
    return launch_time_map(false, p, dtype, st);
}

cudaError_t tc_attention_backward3d(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk, void *ws,
                                    Dims3 d, int dtype, cudaStream_t st, const char **why, bool det)
{
    cudaError_t e = map_backward<true>(dattn, attn, q, k, dq, dk, ws, d.frames(), d.T, dtype, st, why, det);
    // T = 1: no time key; the 2D passes' results stand (a +0 added to a -0 would change their bits)
    if (e != cudaSuccess || d.T == 1) return e;
    TimeMapParams p = map_params(d);
    p.t.q = q; p.t.k = k; p.t.dq = dq; p.t.dk = dk;
    p.map = attn;
    p.dattn = dattn;
    p.rho = attn_bwd_ws(d.frames(), false, ws).rho;
    return launch_time_map(true, p, dtype, st);
}

}  // namespace cca
