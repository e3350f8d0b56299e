// Host dispatch of the wgmma forward values kernel (kernel: cca_tc_fwd.cuh) and its fp32 / bf16 instantiations.
#include "cca_tc_fwd.cuh"

namespace cca {
using namespace tc;

bool tc_forward_supported(Dims d, int dtype) { return tc::shape_supported(d, dtype); }

size_t tc_forward_workspace(Dims d) { return fwd_ws(d, 0, nullptr).bytes; }

// q,k,v,out are channels-last (NHWC), fp32, bf16 or f16.  Two launches: statistics pre-pass (q,k only), values.
cudaError_t tc_forward(const void *q, const void *k, const void *v, void *out, float *lse, void *ws, Dims d, int dtype,
                       cudaStream_t st, const char **why, bool det)
{
    const FwdWs w = fwd_ws(d, 0, ws);
    // statistics; it also clears the per-sample counters of the values kernel
    cudaError_t e = tc_stats(q, k, w.parts, w.cdone, d.B, d, dtype, st, why);
    if (e != cudaSuccess) return e;
    return tc_values(q, k, v, out, lse, w.parts, w.cdone, w.planes, d, dtype, st, why, det, 0);
}

cudaError_t tc_values(const void *q, const void *k, const void *v, void *out, float *lse, const float *parts, unsigned int *cdone,
                      void *planes, Dims d, int dtype, cudaStream_t st, const char **why, bool det, int extra_parts)
{
    if (det && tc_tiled(d))       // (fp32: cca_capi.cu refuses 16-bit I/O here)
        return tc_forward_planes(q, k, v, reinterpret_cast<float *>(out), lse, parts, cdone, planes, d, st, why, extra_parts);
    const FwdArgs a{q, k, v, out, lse, parts, cdone, d, st, why, extra_parts};
    return with_elem_tile(dtype, d, [&](auto e, auto lk) { return launch_fwd<lk(), decltype(e)>(a); });
}

}  // namespace cca
