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
// the time pass, so the backward is as reproducible as the 2D passes before it.  The time kernels' bodies and the passes live
// in cca_tc_attn3d.cuh, shared with the causal map (cca_tc_causal.cu).
#include "cca_tc_attn3d.cuh"

namespace cca {
namespace tc {
namespace {

template <int TM, typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_map_fwd_kernel(const __grid_constant__ TimeMapParams p)
{
    time_map_fwd<TM, E, false>(p);
}

template <int TM, typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_map_bwd_kernel(const __grid_constant__ TimeMapParams p)
{
    time_map_bwd<TM, E, false>(p);
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

}  // namespace

cudaError_t tc_attention3d_rows(const void *q, const void *k, float *attn, const float *parts, Dims3 d, int dtype, cudaStream_t st,
                                const char **why)
{
    const Dims f = d.frames();
    return with_elem_tile(dtype, f, [&](auto el, auto lk) {
        return launch_attn_fwd<lk(), decltype(el), true>(q, k, attn, parts, f, d.T, st, why);
    });
}

cudaError_t tc_attention3d_rows_backward(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk,
                                         void *ws, Dims3 d, int dtype, cudaStream_t st, const char **why, bool det)
{
    return map_backward<true>(dattn, attn, q, k, dq, dk, ws, d.frames(), d.T, dtype, st, why, det);
}

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
    return attention_forward3d_passes([&](float *part) { return tc_time_stats(q, k, part, d, dtype, st); },
                                      [&](bool backward, const TimeMapParams &p) { return launch_time_map(backward, p, dtype, st); },
                                      q, k, attn, ws, d, dtype, st, why);
}

cudaError_t tc_attention_backward3d(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk, void *ws,
                                    Dims3 d, int dtype, cudaStream_t st, const char **why, bool det)
{
    return attention_backward3d_passes([&](bool backward, const TimeMapParams &p) { return launch_time_map(backward, p, dtype, st); },
                                       dattn, attn, q, k, dq, dk, ws, d, dtype, st, why, det);
}

}  // namespace cca
