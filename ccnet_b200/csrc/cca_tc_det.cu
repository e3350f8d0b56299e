// Deterministic mode of the tensor-core kernels on tiled lines (CCA_FLAG_DETERMINISTIC): the fp32 planes-mode instantiations
// of the forward values and backward kernels (cca_tc_fwd.cuh, cca_tc_bwd.cuh), and the kernel that adds their partial planes.
// Every element of a plane is written once by one item; the sum runs over the planes in ascending order, in fp32, so the
// result does not depend on which CTA ran which item or when.
#include "cca_tc_bwd.cuh"
#include "cca_tc_fwd.cuh"

namespace cca {
namespace tc {

template cudaError_t launch_fwd<80, float, true>(const void *, const void *, const void *, void *, float *, const float *,
                                                 unsigned int *, Dims, cudaStream_t, const char **, int);
template cudaError_t launch_fwd<112, float, true>(const void *, const void *, const void *, void *, float *, const float *,
                                                  unsigned int *, Dims, cudaStream_t, const char **, int);
template cudaError_t launch_bwd<80, float, true>(const void *, const void *, const void *, const void *, const void *, const float *,
                                                 float *, unsigned int *, void *, void *, void *, Dims, int, cudaStream_t,
                                                 const char **);
template cudaError_t launch_bwd<112, float, true>(const void *, const void *, const void *, const void *, const void *, const float *,
                                                  float *, unsigned int *, void *, void *, void *, Dims, int, cudaStream_t,
                                                  const char **);

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
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(256); cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = tc_pdl() ? 1 : 0;
    cudaError_t e = cudaLaunchKernelEx(&cfg, cca_planes_sum_kernel, p);
    count_launch();
    return e != cudaSuccess ? e : cudaGetLastError();
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
    const size_t per = (size_t)make_space(d.B, d.H, d.W).nparts * d.B * d.H * d.W * sizeof(float);
    return (which == CCA_WS_FORWARD ? align256(per * d.C) : 2 * align256(per * d.Cq) + align256(per * d.C)) + 256;
}

cudaError_t tc_forward_planes(const void *q, const void *k, const void *v, float *out, float *lse, const float *parts,
                              unsigned int *cdone, void *planes, Dims d, cudaStream_t st, const char **why, int extra_parts)
{
    const ItemSpace sp = make_space(d.B, d.H, d.W);
    const int lk = lk_for(max_tile(sp));
    float *po = reinterpret_cast<float *>((reinterpret_cast<uintptr_t>(planes) + 255) & ~(uintptr_t)255);
    cudaError_t e = lk == 80 ? launch_fwd<80, float, true>(q, k, v, po, lse, parts, cdone, d, st, why, extra_parts)
                             : launch_fwd<112, float, true>(q, k, v, po, lse, parts, cdone, d, st, why, extra_parts);
    if (e != cudaSuccess) return e;
    const float *src[1] = {po};
    float *dst[1] = {out};
    const long n[1] = {(long)d.B * d.H * d.W * d.C};
    return planes_sum(src, dst, n, 1, sp.nparts, st);
}

cudaError_t tc_backward_planes(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                               float *delta, unsigned int *counters, float *dq, float *dk, float *dv, void *planes, Dims d,
                               int delta_mode, cudaStream_t st, const char **why)
{
    const ItemSpace sp = make_space(d.B, d.H, d.W);
    const size_t per = (size_t)sp.nparts * d.B * d.H * d.W * sizeof(float);
    // 256-byte aligned plane buffers inside the workspace (TMA needs 16)
    uint8_t *base = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(planes) + 255) & ~(uintptr_t)255);
    float *pq = reinterpret_cast<float *>(base), *pk = reinterpret_cast<float *>(base + align256(per * d.Cq));
    float *pv = reinterpret_cast<float *>(base + 2 * align256(per * d.Cq));
    const int lk = lk_for(max_tile(sp));
    cudaError_t e = lk == 80 ? launch_bwd<80, float, true>(dout, q, k, v, out, lse, delta, counters, pq, pk, pv, d, delta_mode, st, why)
                             : launch_bwd<112, float, true>(dout, q, k, v, out, lse, delta, counters, pq, pk, pv, d, delta_mode, st, why);
    if (e != cudaSuccess) return e;
    const long npix = (long)d.B * d.H * d.W;
    const float *src[3] = {pq, pk, pv};
    float *dst[3] = {dq, dk, dv};
    const long n[3] = {npix * d.Cq, npix * d.Cq, npix * d.C};
    return planes_sum(src, dst, n, 3, sp.nparts, st);
}

}  // namespace cca
