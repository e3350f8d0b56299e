// Host dispatch of the attention-map kernels (cca_tc_attn.cuh) and their fp32 / bf16 / f16 instantiations.
#include "cca_tc_attn.cuh"

namespace cca {
using namespace tc;

// the map kernels have no condition on C: shape_fits is asked with one 64-channel chunk
bool tc_attention_supported(Dims d, int dtype) { d.C = kNC; return shape_supported(d, dtype); }

// forward: the statistics workspace (partial planes + counters); backward: rho [B*H*W], then (planes mode) the dQ, dK planes
size_t tc_attention_workspace(int backward, Dims d, bool det)
{
    d.C = kNC;
    return backward ? attn_bwd_ws(d, det, nullptr).bytes : fwd_ws(d, 0, nullptr).bytes;
}

cudaError_t tc_attention_forward(const void *q, const void *k, float *attn, void *ws, Dims d, int dtype, cudaStream_t st,
                                 const char **why)
{
    // the statistics pre-pass, unchanged: no counters
    float *parts = fwd_ws(d, 0, ws).parts;
    cudaError_t e = tc_stats(q, k, parts, nullptr, 0, d, dtype, st, why);
    if (e != cudaSuccess) return e;
    return with_elem_tile(dtype, d, [&](auto el, auto lk) {
        return launch_attn_fwd<lk(), decltype(el), false>(q, k, attn, parts, d, 0, st, why);
    });
}

cudaError_t tc_attention_backward(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk, void *ws,
                                  Dims d, int dtype, cudaStream_t st, const char **why, bool det)
{
    return map_backward<false>(dattn, attn, q, k, dq, dk, ws, d, 0, dtype, st, why, det);
}

}  // namespace cca
