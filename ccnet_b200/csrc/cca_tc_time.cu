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

template <int TM, typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_stats_kernel(const __grid_constant__ TimeParams p)
{
    time_stats<TM, E, false>(p);
}

template <int TM, typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_values_kernel(const __grid_constant__ TimeParams p)
{
    time_values<TM, E, false>(p);
}

template <int TM, typename E>
__global__ void __launch_bounds__(32 * kWarps) cca_time_bwd_kernel(const __grid_constant__ TimeParams p)
{
    time_bwd<TM, E, false>(p);
}

cudaError_t launch_time(int kind, const TimeParams &p, int dtype, cudaStream_t st)
{
    return with_elem(dtype, [&](auto e) {
        using E = decltype(e);
        auto tier = [&](auto tm) {
            constexpr int TM = decltype(tm)::value;
            void (*kern)(TimeParams) = kind == kStats    ? cca_time_stats_kernel<TM, E>
                                       : kind == kValues ? cca_time_values_kernel<TM, E>
                                                         : cca_time_bwd_kernel<TM, E>;
            return launch_lines(kern, p.lines, warp_floats(kind, p.T, p.Cq), p, st);
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
    return forward3d_passes([&](int kind, const TimeParams &p) { return launch_time(kind, p, dtype, st); }, q, k, v, out, lse, ws,
                            d, dtype, st, why, det);
}

cudaError_t tc_backward3d(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                          void *dq, void *dk, void *dv, void *ws, Dims3 d, int dtype, cudaStream_t st, const char **why, bool det)
{
    return backward3d_passes([&](int kind, const TimeParams &p) { return launch_time(kind, p, dtype, st); }, dout, q, k, v, out,
                             lse, dq, dk, dv, ws, d, dtype, st, why, det);
}

}  // namespace cca
