// Host dispatch of the attention-map kernels (cca_tc_attn.cuh) and their fp32 / bf16 / f16 instantiations.
#include "cca_tc_attn.cuh"

namespace cca {
namespace tc {
namespace {

bool qk_maps(CUtensorMap *m, const void *q, const void *k, Dims d, int LK, int dtype)
{
    const void *base[2] = {q, k};
    for (int t = 0; t < 2; ++t)
        for (int r = 0; r < 2; ++r)
            if (!get_map(&m[2 * t + r], base[t], d.B, d.H, d.W, d.Cq, LK, r == 0, dtype)) return false;
    return true;
}

template <typename K, typename... Args>
cudaError_t launch_pdl(K kern, int smem, const ItemSpace &sp, cudaStream_t st, Args... args)
{
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    const int sms = sm_count();
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(sp.total < sms ? sp.total : sms); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = tc_pdl() ? 1 : 0;
    e = cudaLaunchKernelEx(&cfg, kern, args...);
    count_launch();
    return e != cudaSuccess ? e : cudaGetLastError();
}

template <int LK, typename E>
cudaError_t launch_attn_fwd(const void *q, const void *k, float *attn, const float *parts, Dims d, cudaStream_t st, const char **why)
{
    CUtensorMap m[4];
    if (!qk_maps(m, q, k, d, LK, kDtype<E>)) {
        if (why) *why = "cuTensorMapEncodeTiled failed";
        return cudaErrorInvalidValue;
    }
    AttnFwdParams p;
    p.sp = make_space(d.B, d.H, d.W);
    p.Cq = d.Cq;
    p.npix = (long)d.B * d.H * d.W;
    p.parts = parts;
    p.attn = attn;
    return launch_pdl(cca_tc_attn_fwd_kernel<LK, E>, StatsSmem<LK, E>::kBytes, p.sp, st, m[0], m[1], m[2], m[3], p);
}

// PL: dq, dk are the [nparts*B, H, W, Cq] fp32 plane buffers
template <int LK, typename E, bool PL>
cudaError_t launch_attn_bwd(const float *dattn, const float *attn, const float *rho, const void *q, const void *k, void *dq, void *dk,
                            Dims d, cudaStream_t st, const char **why)
{
    CUtensorMap m[8];
    AttnBwdParams p;
    p.sp = make_space(d.B, d.H, d.W);
    const void *base[2] = {dq, dk};
    bool ok = qk_maps(m, q, k, d, LK, kDtype<E>);
    for (int t = 0; t < 2 && ok; ++t)
        for (int r = 0; r < 2 && ok; ++r)       // output boxes: one tile of the direction (a store never reaches the next tile)
            ok = get_map(&m[4 + 2 * t + r], base[t], PL ? p.sp.nparts * d.B : d.B, d.H, d.W, d.Cq,
                         r == 0 ? p.sp.col.tl : p.sp.row.tl, r == 0, kDtype<E>);
    if (!ok) {
        if (why) *why = "cuTensorMapEncodeTiled failed";
        return cudaErrorInvalidValue;
    }
    p.Cq = d.Cq;
    p.attn = attn; p.dattn = dattn; p.rho = rho;
    return launch_pdl(cca_tc_attn_bwd_kernel<LK, E, PL>, AttnBwdSmem<LK, E>::kBytes, p.sp, st, m[0], m[1], m[2], m[3], m[4], m[5],
                      m[6], m[7], p);
}

template <typename E>
cudaError_t attn_fwd_typed(const void *q, const void *k, float *attn, const float *parts, Dims d, cudaStream_t st, const char **why)
{
    return lk_for(max_tile(make_space(d.B, d.H, d.W))) == 80 ? launch_attn_fwd<80, E>(q, k, attn, parts, d, st, why)
                                                           : launch_attn_fwd<112, E>(q, k, attn, parts, d, st, why);
}
template <typename E, bool PL>
cudaError_t attn_bwd_typed(const float *dattn, const float *attn, const float *rho, const void *q, const void *k, void *dq, void *dk,
                           Dims d, cudaStream_t st, const char **why)
{
    return lk_for(max_tile(make_space(d.B, d.H, d.W))) == 80
               ? launch_attn_bwd<80, E, PL>(dattn, attn, rho, q, k, dq, dk, d, st, why)
               : launch_attn_bwd<112, E, PL>(dattn, attn, rho, q, k, dq, dk, d, st, why);
}
}  // namespace
}  // namespace tc

using namespace tc;

// the map kernels have no condition on C: shape_fits is asked with one 64-channel chunk
bool tc_attention_supported(Dims d, int dtype) { d.C = kNC; return shape_supported(d, dtype); }

// forward: the statistics workspace (partial planes + counters); backward: rho [B*H*W], then (planes mode) the dQ, dK planes
size_t tc_attention_workspace(int backward, Dims d, bool det)
{
    d.C = kNC;
    if (!backward) return tc_forward_workspace(d);
    const size_t npix = (size_t)d.B * d.H * d.W;
    size_t n = align256(npix * sizeof(float));
    if (det && tc_tiled(d)) n += 2 * align256((size_t)make_space(d.B, d.H, d.W).nparts * npix * d.Cq * sizeof(float)) + 256;
    return n;
}

cudaError_t tc_attention_forward(const void *q, const void *k, float *attn, void *ws, Dims d, int dtype, cudaStream_t st,
                                 const char **why)
{
    // the statistics pre-pass, unchanged: nothing to clear, no counters
    cudaError_t e = tc_stats(q, k, reinterpret_cast<float *>(ws), nullptr, 0, nullptr, 0, d, dtype, st, why);
    if (e != cudaSuccess) return e;
    const float *parts = reinterpret_cast<const float *>(ws);
    if (dtype == CCA_F16) return attn_fwd_typed<__half>(q, k, attn, parts, d, st, why);
    if (dtype == CCA_BF16) return attn_fwd_typed<__nv_bfloat16>(q, k, attn, parts, d, st, why);
    return attn_fwd_typed<float>(q, k, attn, parts, d, st, why);
}

cudaError_t tc_attention_backward(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk, void *ws,
                                  Dims d, int dtype, cudaStream_t st, const char **why, bool det)
{
    const long npix = (long)d.B * d.H * d.W;
    float *rho = reinterpret_cast<float *>(ws);
    const bool planes = det && tc_tiled(d);      // (fp32: cca_capi.cu refuses 16-bit I/O here)
    // rho, and (unless the planes are summed into them) dq and dk cleared for the reduce-adds
    const long clear = planes ? 0 : npix * d.Cq * (dtype == CCA_F32 ? 4 : 2);
    cudaError_t e = attn_rho(dattn, attn, rho, npix, d.H + d.W, planes ? nullptr : dq, planes ? nullptr : dk, clear, st);
    if (e != cudaSuccess) return e;
    if (planes) {
        const ItemSpace sp = make_space(d.B, d.H, d.W);
        uint8_t *base = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(ws) + align256(npix * sizeof(float)) + 255) &
                                                    ~(uintptr_t)255);
        float *pq = reinterpret_cast<float *>(base), *pk = reinterpret_cast<float *>(base + align256(sp.nparts * npix * d.Cq * sizeof(float)));
        e = attn_bwd_typed<float, true>(dattn, attn, rho, q, k, pq, pk, d, st, why);
        if (e != cudaSuccess) return e;
        const float *src[2] = {pq, pk};
        float *dst[2] = {reinterpret_cast<float *>(dq), reinterpret_cast<float *>(dk)};
        const long n[2] = {npix * d.Cq, npix * d.Cq};
        return planes_sum(src, dst, n, 2, sp.nparts, st);
    }
    if (dtype == CCA_F16) return attn_bwd_typed<__half, false>(dattn, attn, rho, q, k, dq, dk, d, st, why);
    if (dtype == CCA_BF16) return attn_bwd_typed<__nv_bfloat16, false>(dattn, attn, rho, q, k, dq, dk, d, st, why);
    return attn_bwd_typed<float, false>(dattn, attn, rho, q, k, dq, dk, d, st, why);
}

}  // namespace cca
