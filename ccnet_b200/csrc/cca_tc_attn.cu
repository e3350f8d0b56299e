// Host dispatch of the attention-map kernels (cca_tc_attn.cuh) and their fp32 / bf16 / f16 instantiations.
#include "cca_tc_attn.cuh"

namespace cca {
namespace tc {
namespace {

template <int LK, typename E>
cudaError_t launch_attn_fwd(const void *q, const void *k, float *attn, const float *parts, Dims d, cudaStream_t st, const char **why)
{
    CUtensorMap m[4];
    if (cudaError_t e = get_maps(m, {{q, d.B, d.Cq, LK, LK}, {k, d.B, d.Cq, LK, LK}}, d, kDtype<E>, why)) return e;
    AttnFwdParams p;
    p.sp = make_space(d.B, d.H, d.W);
    p.Cq = d.Cq;
    p.npix = (long)d.B * d.H * d.W;
    p.parts = parts;
    p.attn = attn;
    return launch_kernel(cca_tc_attn_fwd_kernel<LK, E>, item_grid(p.sp), kThreads, StatsSmem<LK, E>::kBytes, true, st, m[0], m[1], m[2],
                         m[3], p);
}

// PL: dq, dk are the [nparts*B, H, W, Cq] fp32 plane buffers
template <int LK, typename E, bool PL>
cudaError_t launch_attn_bwd(const float *dattn, const float *attn, const float *rho, const void *q, const void *k, void *dq, void *dk,
                            Dims d, cudaStream_t st, const char **why)
{
    CUtensorMap m[8];
    AttnBwdParams p;
    p.sp = make_space(d.B, d.H, d.W);
    // output boxes: one tile of the direction (a store never reaches the next tile)
    const int nb = PL ? p.sp.nparts * d.B : d.B;
    if (cudaError_t e = get_maps(m, {{q, d.B, d.Cq, LK, LK}, {k, d.B, d.Cq, LK, LK}, {dq, nb, d.Cq, p.sp.col.tl, p.sp.row.tl},
                                     {dk, nb, d.Cq, p.sp.col.tl, p.sp.row.tl}},
                                 d, kDtype<E>, why))
        return e;
    p.Cq = d.Cq;
    p.attn = attn; p.dattn = dattn; p.rho = rho;
    return launch_kernel(cca_tc_attn_bwd_kernel<LK, E, PL>, item_grid(p.sp), kThreads, AttnBwdSmem<LK, E>::kBytes, true, st, m[0], m[1],
                         m[2], m[3], m[4], m[5], m[6], m[7], p);
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
        return launch_attn_fwd<lk(), decltype(el)>(q, k, attn, parts, d, st, why);
    });
}

cudaError_t tc_attention_backward(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk, void *ws,
                                  Dims d, int dtype, cudaStream_t st, const char **why, bool det)
{
    const long npix = (long)d.B * d.H * d.W;
    const bool planes = det && tc_tiled(d);      // (fp32: cca_capi.cu refuses 16-bit I/O here)
    const AttnBwdWs w = attn_bwd_ws(d, planes, ws);
    // rho, and (unless the planes are summed into them) dq and dk cleared for the reduce-adds
    const long clear = planes ? 0 : npix * d.Cq * (dtype == CCA_F32 ? 4 : 2);
    cudaError_t e = attn_rho(dattn, attn, w.rho, npix, d.H + d.W, planes ? nullptr : dq, planes ? nullptr : dk, clear, st);
    if (e != cudaSuccess) return e;
    if (planes) {
        float *pq = w.planes.p[0], *pk = w.planes.p[1];
        e = with_tile(d, [&](auto lk) { return launch_attn_bwd<lk(), float, true>(dattn, attn, w.rho, q, k, pq, pk, d, st, why); });
        if (e != cudaSuccess) return e;
        const float *src[2] = {pq, pk};
        float *dst[2] = {reinterpret_cast<float *>(dq), reinterpret_cast<float *>(dk)};
        const long n[2] = {npix * d.Cq, npix * d.Cq};
        return planes_sum(src, dst, n, 2, make_space(d.B, d.H, d.W).nparts, st);
    }
    return with_elem_tile(dtype, d, [&](auto el, auto lk) {
        return launch_attn_bwd<lk(), decltype(el), false>(dattn, attn, w.rho, q, k, dq, dk, d, st, why);
    });
}

}  // namespace cca
