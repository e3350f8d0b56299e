// Host dispatch of the wgmma forward values kernel (kernel: cca_tc_fwd.cuh) and its fp32 / bf16 instantiations.
#include "cca_tc_fwd.cuh"

namespace cca {
using namespace tc;

bool tc_forward_supported(Dims d, int dtype) { return tc::shape_supported(d, dtype); }

// Workspace of the forward: [nparts][B*H*W] fp32 partial lse planes, then [B] unsigned per-sample counters.
size_t tc_forward_workspace(Dims d)
{
    const ItemSpace sp = make_space(d.B, d.H, d.W);
    const size_t parts = (size_t)sp.nparts * d.B * d.H * d.W * sizeof(float);
    return ((parts + 15) & ~(size_t)15) + (((size_t)d.B * sizeof(unsigned int) + 15) & ~(size_t)15);
}

// q,k,v,out are channels-last (NHWC), fp32, bf16 or f16.  Two launches: statistics pre-pass (q,k only), values.
cudaError_t tc_forward(const void *q, const void *k, const void *v, void *out, float *lse, void *ws, Dims d, int dtype,
                       cudaStream_t st, const char **why, bool det)
{
    const ItemSpace sp = make_space(d.B, d.H, d.W);
    const long npix = (long)d.B * d.H * d.W;
    float *parts = reinterpret_cast<float *>(ws);
    const size_t parts_bytes = ((size_t)sp.nparts * npix * sizeof(float) + 15) & ~(size_t)15;
    unsigned int *cdone = reinterpret_cast<unsigned int *>(reinterpret_cast<uint8_t *>(ws) + parts_bytes);
    // statistics; it also clears the per-sample counters of the values kernel
    cudaError_t e = tc_stats(q, k, parts, nullptr, 0, cdone, d.B, d, dtype, st, why);
    if (e != cudaSuccess) return e;
    return tc_values(q, k, v, out, lse, parts, cdone, reinterpret_cast<uint8_t *>(ws) + tc_forward_workspace(d), d, dtype, st,
                     why, det, 0);
}

cudaError_t tc_values(const void *q, const void *k, const void *v, void *out, float *lse, const float *parts, unsigned int *cdone,
                      void *planes, Dims d, int dtype, cudaStream_t st, const char **why, bool det, int extra_parts)
{
    if (det && tc_tiled(d))       // (fp32: cca_capi.cu refuses 16-bit I/O here)
        return tc_forward_planes(q, k, v, reinterpret_cast<float *>(out), lse, parts, cdone, planes, d, st, why, extra_parts);
    const int lk = lk_for(max_tile(make_space(d.B, d.H, d.W)));
    if (dtype == CCA_F16)
        return lk == 80 ? launch_fwd<80, __half>(q, k, v, out, lse, parts, cdone, d, st, why, extra_parts)
                        : launch_fwd<112, __half>(q, k, v, out, lse, parts, cdone, d, st, why, extra_parts);
    if (dtype == CCA_BF16)
        return lk == 80 ? launch_fwd<80, __nv_bfloat16>(q, k, v, out, lse, parts, cdone, d, st, why, extra_parts)
                        : launch_fwd<112, __nv_bfloat16>(q, k, v, out, lse, parts, cdone, d, st, why, extra_parts);
    return lk == 80 ? launch_fwd<80, float>(q, k, v, out, lse, parts, cdone, d, st, why, extra_parts)
                    : launch_fwd<112, float>(q, k, v, out, lse, parts, cdone, d, st, why, extra_parts);
}

}  // namespace cca
