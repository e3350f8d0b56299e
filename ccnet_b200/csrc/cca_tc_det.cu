// Deterministic mode of the tensor-core kernels on tiled lines (CCA_FLAG_DETERMINISTIC): the fp32 planes-mode instantiations
// of the forward values and backward kernels (cca_tc_fwd.cuh, cca_tc_bwd.cuh), and the kernel that adds their partial planes.
// Every element of a plane is written once by one item; the sum runs over the planes in ascending order, in fp32, so the
// result does not depend on which CTA ran which item or when.
#include "cca_tc_bwd.cuh"
#include "cca_tc_fwd.cuh"

namespace cca {
namespace tc {

template cudaError_t launch_fwd<80, float, true>(const FwdArgs &);
template cudaError_t launch_fwd<112, float, true>(const FwdArgs &);
template cudaError_t launch_bwd<80, float, true>(const BwdArgs &);
template cudaError_t launch_bwd<112, float, true>(const BwdArgs &);

namespace {
struct PlaneSums {
    const float4 *src[3];   // [nparts][n4] float4 each
    float4 *dst[3];
    long n4[3];
    int count, nparts;
};

// dst[i] = src[0][i] + src[1][i] + ... + src[nparts - 1][i], for up to three tensors
__global__ void __launch_bounds__(256) cca_planes_sum_kernel(const __grid_constant__ PlaneSums p)
{
    pdl_wait();                                            // the item kernel has written every plane
    const long nth = (long)gridDim.x * blockDim.x;
    for (int t = 0; t < p.count; ++t) {
        const long n4 = p.n4[t];
        for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += nth) {
            float4 s = __ldcs(p.src[t] + i);
            for (int k = 1; k < p.nparts; ++k) {
                const float4 x = __ldcs(p.src[t] + (long)k * n4 + i);
                s.x += x.x; s.y += x.y; s.z += x.z; s.w += x.w;
            }
            p.dst[t][i] = s;
        }
    }
}

}  // namespace

cudaError_t planes_sum(const float *const *src, float *const *dst, const long *n, int count, int nparts, cudaStream_t st)
{
    PlaneSums p = {};
    long total = 0;
    for (int t = 0; t < count; ++t) {
        p.src[t] = reinterpret_cast<const float4 *>(src[t]);
        p.dst[t] = reinterpret_cast<float4 *>(dst[t]);
        p.n4[t] = n[t] / 4;
        total += p.n4[t];
    }
    p.count = count; p.nparts = nparts;
    const long want = (total + 255) / 256;
    const int grid = (int)(want < 8L * sm_count() ? (want > 0 ? want : 1) : 8L * sm_count());
    return launch_kernel(cca_planes_sum_kernel, grid, 256, 0, true, st, p);
}

}  // namespace tc

using namespace tc;

bool tc_tiled(Dims d)
{
    const ItemSpace sp = make_space(d.B, d.H, d.W);
    return sp.col.nt > 1 || sp.row.nt > 1;
}

size_t tc_planes_bytes(int which, Dims d)
{
    if (!tc_tiled(d)) return 0;
    return which == CCA_WS_FORWARD ? planes_ws(d, {d.C}, nullptr).bytes : planes_ws(d, {d.Cq, d.Cq, d.C}, nullptr).bytes;
}

cudaError_t tc_forward_planes(const void *q, const void *k, const void *v, float *out, float *lse, const float *parts,
                              unsigned int *cdone, void *planes, Dims d, cudaStream_t st, const char **why, int extra_parts)
{
    float *po = planes_ws(d, {d.C}, planes).p[0];
    const FwdArgs a{q, k, v, po, lse, parts, cdone, d, st, why, extra_parts};
    cudaError_t e = with_tile(d, [&](auto lk) { return launch_fwd<lk(), float, true>(a); });
    if (e != cudaSuccess) return e;
    const float *src[1] = {po};
    float *dst[1] = {out};
    const long n[1] = {(long)d.B * d.H * d.W * d.C};
    return planes_sum(src, dst, n, 1, make_space(d.B, d.H, d.W).nparts, st);
}

cudaError_t tc_backward_planes(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                               float *delta, unsigned int *counters, float *dq, float *dk, float *dv, void *planes, Dims d,
                               int delta_mode, cudaStream_t st, const char **why)
{
    const PlanesWs w = planes_ws(d, {d.Cq, d.Cq, d.C}, planes);
    const BwdArgs a{dout, q, k, v, out, lse, delta, counters, w.p[0], w.p[1], w.p[2], d, delta_mode, st, why};
    cudaError_t e = with_tile(d, [&](auto lk) { return launch_bwd<lk(), float, true>(a); });
    if (e != cudaSuccess) return e;
    const long npix = (long)d.B * d.H * d.W;
    const float *src[3] = {w.p[0], w.p[1], w.p[2]};
    float *dst[3] = {dq, dk, dv};
    const long n[3] = {npix * d.Cq, npix * d.Cq, npix * d.C};
    return planes_sum(src, dst, n, 3, make_space(d.B, d.H, d.W).nparts, st);
}

}  // namespace cca
