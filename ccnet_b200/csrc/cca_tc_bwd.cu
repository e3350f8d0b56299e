// Host dispatch of the wgmma backward kernel (kernel: cca_tc_bwd.cuh) and its fp32 / bf16 instantiations.
#include "cca_tc_bwd.cuh"

namespace cca {
using namespace tc;

bool tc_backward_supported(Dims d, int dtype) { return tc::shape_supported(d, dtype); }

size_t tc_backward_workspace(Dims d) { return bwd_ws(d, nullptr).bytes; }

// all tensors channels-last (NHWC), fp32, bf16 or f16
cudaError_t tc_backward(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                        void *dq, void *dk, void *dv, void *ws, Dims d, int dtype, cudaStream_t st, const char **why, bool det)
{
    const BwdWs w = bwd_ws(d, ws);
    int mode = tc_delta_mode();                       // -1: automatic = producers compute delta for their sample (the consumers
    if (mode < 0) mode = 1;                           // only ever wait for lower-indexed items, tiled or not)
    if (det && tc_tiled(d))                           // (fp32: cca_capi.cu refuses 16-bit I/O here)
        return tc_backward_planes(dout, q, k, v, out, lse, w.delta, w.counters, reinterpret_cast<float *>(dq),
                                  reinterpret_cast<float *>(dk), reinterpret_cast<float *>(dv), w.planes, d, mode, st, why);
    const BwdArgs a{dout, q, k, v, out, lse, w.delta, w.counters, dq, dk, dv, d, mode, st, why};
    return with_elem_tile(dtype, d, [&](auto e, auto lk) { return launch_bwd<lk(), decltype(e)>(a); });
}

}  // namespace cca
