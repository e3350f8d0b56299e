// Host dispatch of the wgmma backward kernel (kernel: cca_tc_bwd.cuh) and its fp32 / bf16 instantiations.
#include "cca_tc_bwd.cuh"

namespace cca {
using namespace tc;

bool tc_backward_supported(Dims d, int dtype) { return tc::shape_supported(d, dtype); }

// Workspace of the backward: delta [B,H,W] fp32, then 3*B unsigned counters.
size_t tc_backward_workspace(Dims d)
{
    const size_t delta = ((size_t)d.B * d.H * d.W * sizeof(float) + 15) & ~(size_t)15;
    return delta + (((size_t)3 * d.B * sizeof(unsigned int) + 15) & ~(size_t)15);
}

// all tensors channels-last (NHWC), fp32, bf16 or f16
cudaError_t tc_backward(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                        void *dq, void *dk, void *dv, void *ws, Dims d, int dtype, cudaStream_t st, const char **why, bool det)
{
    float *delta = reinterpret_cast<float *>(ws);
    const size_t delta_bytes = ((size_t)d.B * d.H * d.W * sizeof(float) + 15) & ~(size_t)15;
    unsigned int *counters = reinterpret_cast<unsigned int *>(reinterpret_cast<uint8_t *>(ws) + delta_bytes);
    const ItemSpace sp = make_space(d.B, d.H, d.W);
    const int lk = lk_for(max_tile(sp));
    int mode = tc_delta_mode();                       // -1: automatic = producers compute delta for their sample (the consumers
    if (mode < 0) mode = 1;                           // only ever wait for lower-indexed items, tiled or not)
    if (det && tc_tiled(d))                           // (fp32: cca_capi.cu refuses 16-bit I/O here)
        return tc_backward_planes(dout, q, k, v, out, lse, delta, counters, reinterpret_cast<float *>(dq),
                                  reinterpret_cast<float *>(dk), reinterpret_cast<float *>(dv),
                                  reinterpret_cast<uint8_t *>(ws) + tc_backward_workspace(d), d, mode, st, why);
    if (dtype == CCA_F16)
        return lk == 80 ? launch_bwd<80, __half>(dout, q, k, v, out, lse, delta, counters, dq, dk, dv, d, mode, st, why)
                        : launch_bwd<112, __half>(dout, q, k, v, out, lse, delta, counters, dq, dk, dv, d, mode, st, why);
    if (dtype == CCA_BF16)
        return lk == 80 ? launch_bwd<80, __nv_bfloat16>(dout, q, k, v, out, lse, delta, counters, dq, dk, dv, d, mode, st, why)
                        : launch_bwd<112, __nv_bfloat16>(dout, q, k, v, out, lse, delta, counters, dq, dk, dv, d, mode, st, why);
    return lk == 80 ? launch_bwd<80, float>(dout, q, k, v, out, lse, delta, counters, dq, dk, dv, d, mode, st, why)
                    : launch_bwd<112, float>(dout, q, k, v, out, lse, delta, counters, dq, dk, dv, d, mode, st, why);
}

}  // namespace cca
