// Generic CUDA-core kernels of the attention map of criss-cross attention over clips, attn[B,T,H,W,H+W+T] (fp32), and of its
// gradient w.r.t. q, k, for NCDHW-contiguous q, k [B,Cq,T,H,W] of any Cq and shape: the shapes the tensor-core kernels of
// cca_tc_attn3d.cu do not cover, and impl="simt".  Row g of pixel (b,t,h,w): column key (t,g,w) for g < H (self entry g = h
// is 0), row key (t,h,g-H) for g < H+W, time key (g-H-W,h,w) after that (self entry g-H-W = t is 0).
// The rows live in the map itself (no shared memory), so any row length is taken; every map index is 64-bit.  One warp per
// pixel, sums in a fixed order, no atomics: the key set is symmetric, so dk is GATHERED per key pixel from the rows of the
// queries that see it.  The backward's rho is attn_rho (cca_simt_attn.cu) over rows of H + W + T entries.
#include "cca_common.cuh"

namespace cca {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

struct Px {
    long b, off;   // sample, offset inside the sample's [T,H,W] volume
    int t, h, w;
};
__device__ __forceinline__ Px px_of(long p, const Dims3 &d, long vol, long hw)
{
    Px x;
    x.b = p / vol; x.off = p - x.b * vol;
    x.t = (int)(x.off / hw);
    const long r = x.off - x.t * hw;
    x.h = (int)(r / d.W); x.w = (int)(r - (long)x.h * d.W);
    return x;
}
// volume offset of key g of pixel x, -1 for the two masked self entries
__device__ __forceinline__ long key_of(int g, const Px &x, const Dims3 &d, long hw)
{
    if (g < d.H) return g == x.h ? -1 : x.t * hw + (long)g * d.W + x.w;
    g -= d.H;
    if (g < d.W) return x.t * hw + (long)x.h * d.W + g;
    g -= d.W;
    return g == x.t ? -1 : g * hw + (long)x.h * d.W + x.w;
}

// logits into the row, then max, log-sum-exp2 and the normalised row in place (each lane rereads only what it wrote)
template <typename E>
__global__ void __launch_bounds__(kThreads) cca_attn3d_map_kernel(const E *__restrict__ q, const E *__restrict__ k, float *__restrict__ attn,
                                                                 Dims3 d)
{
    const long hw = (long)d.H * d.W, vol = hw * d.T, npix = vol * d.B, rl = (long)d.H + d.W + d.T;
    const int lane = threadIdx.x & 31;
    for (long p = (long)blockIdx.x * kWarps + (threadIdx.x >> 5); p < npix; p += (long)gridDim.x * kWarps) {
        const Px x = px_of(p, d, vol, hw);
        const E *qp = q + x.b * d.Cq * vol + x.off, *kb = k + x.b * d.Cq * vol;
        float *row = attn + p * rl;
        float m = -INFINITY;
        for (int g = lane; g < rl; g += 32) {
            const long o = key_of(g, x, d, hw);
            float e = -INFINITY;
            if (o >= 0) {
                e = 0.f;
                for (int c = 0; c < d.Cq; ++c) e = fmaf(ldg_f(qp + c * vol), ldg_f(kb + c * vol + o), e);
            }
            row[g] = e;
            m = fmaxf(m, e);
        }
        m = warp_max(m) * kLog2e;
        float l = 0.f;
        for (int g = lane; g < rl; g += 32) l += exp2f(fmaf(row[g], kLog2e, -m));
        const float lse2 = m + log2f(warp_sum(l));
        for (int g = lane; g < rl; g += 32) row[g] = exp2f(fmaf(row[g], kLog2e, -lse2));
    }
}

// dq[b,c,t,h,w] = sum_g dS[p,g] k[b,c,key g]; lanes own channels, the keys are walked in order
template <typename E>
__global__ void __launch_bounds__(kThreads) cca_attn3d_dq_kernel(const float *__restrict__ dattn, const float *__restrict__ attn,
                                                                const float *__restrict__ rho, const E *__restrict__ k,
                                                                E *__restrict__ dq, Dims3 d)
{
    const long hw = (long)d.H * d.W, vol = hw * d.T, npix = vol * d.B, rl = (long)d.H + d.W + d.T;
    const int lane = threadIdx.x & 31;
    for (long p = (long)blockIdx.x * kWarps + (threadIdx.x >> 5); p < npix; p += (long)gridDim.x * kWarps) {
        const Px x = px_of(p, d, vol, hw);
        const float *a = attn + p * rl, *da = dattn + p * rl;
        const float r = rho[p];
        for (int c0 = 0; c0 < d.Cq; c0 += 32) {
            const int c = c0 + lane;
            const E *kc = k + (x.b * d.Cq + (c < d.Cq ? c : 0)) * vol;
            float acc = 0.f;
            for (int g = 0; g < rl; ++g) {
                const long o = key_of(g, x, d, hw);
                if (o < 0) continue;                                   // the self entries do not depend on q, k
                acc = fmaf(__ldg(a + g) * (__ldg(da + g) - r), ldg_f(kc + o), acc);
            }
            if (c < d.Cq) dq[(x.b * d.Cq + c) * vol + x.off] = from_f<E>(acc);
        }
    }
}

// dk of key pixel (t,y,x) = sum over the queries whose row holds it -- column queries (t,i,x), i != y (entry y), row queries
// (t,y,j) (entry H + x), time queries (s,y,x), s != t (entry H + W + t) -- of dS * q, in that order
template <typename E>
__global__ void __launch_bounds__(kThreads) cca_attn3d_dk_kernel(const float *__restrict__ dattn, const float *__restrict__ attn,
                                                                const float *__restrict__ rho, const E *__restrict__ q,
                                                                E *__restrict__ dk, Dims3 d)
{
    const long hw = (long)d.H * d.W, vol = hw * d.T, npix = vol * d.B, rl = (long)d.H + d.W + d.T;
    const int lane = threadIdx.x & 31;
    for (long p = (long)blockIdx.x * kWarps + (threadIdx.x >> 5); p < npix; p += (long)gridDim.x * kWarps) {
        const Px x = px_of(p, d, vol, hw);
        const long s0 = x.b * vol;
        for (int c0 = 0; c0 < d.Cq; c0 += 32) {
            const int c = c0 + lane;
            const E *qc = q + (x.b * d.Cq + (c < d.Cq ? c : 0)) * vol;
            float acc = 0.f;
            for (int i = 0; i < rl; ++i) {
                long qo, g;                                            // query pixel (volume offset), its entry of this key
                if (i < d.H) {
                    if (i == x.h) continue;
                    qo = x.t * hw + (long)i * d.W + x.w; g = x.h;
                } else if (i < d.H + d.W) {
                    qo = x.t * hw + (long)x.h * d.W + (i - d.H); g = d.H + x.w;
                } else {
                    const int s = i - d.H - d.W;
                    if (s == x.t) continue;
                    qo = s * hw + (long)x.h * d.W + x.w; g = d.H + d.W + x.t;
                }
                const long e = (s0 + qo) * rl + g;
                acc = fmaf(__ldg(attn + e) * (__ldg(dattn + e) - rho[s0 + qo]), ldg_f(qc + qo), acc);
            }
            if (c < d.Cq) dk[(x.b * d.Cq + c) * vol + x.off] = from_f<E>(acc);
        }
    }
}

template <typename E>
cudaError_t fwd_typed(const void *q, const void *k, float *attn, Dims3 d, cudaStream_t st)
{
    const long npix = (long)d.B * d.T * d.H * d.W;
    cca_attn3d_map_kernel<E><<<warp_grid(npix, kWarps), kThreads, 0, st>>>((const E *)q, (const E *)k, attn, d);
    count_launch();
    return cudaGetLastError();
}

template <typename E>
cudaError_t bwd_typed(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk, float *rho, Dims3 d,
                      cudaStream_t st)
{
    const long npix = (long)d.B * d.T * d.H * d.W;
    cudaError_t e = attn_rho(dattn, attn, rho, npix, d.H + d.W + d.T, nullptr, nullptr, 0, st);
    if (e != cudaSuccess) return e;
    cca_attn3d_dq_kernel<E><<<warp_grid(npix, kWarps), kThreads, 0, st>>>(dattn, attn, rho, (const E *)k, (E *)dq, d);
    count_launch();
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    cca_attn3d_dk_kernel<E><<<warp_grid(npix, kWarps), kThreads, 0, st>>>(dattn, attn, rho, (const E *)q, (E *)dk, d);
    count_launch();
    return cudaGetLastError();
}

}  // namespace

size_t simt_attention3d_workspace(int backward, Dims3 d)
{
    return backward ? (size_t)d.B * d.T * d.H * d.W * sizeof(float) + 16 : 16;
}

cudaError_t simt_attention_forward3d(const void *q, const void *k, float *attn, Dims3 d, int dtype, cudaStream_t st)
{
    return with_elem(dtype, [&](auto e) { return fwd_typed<decltype(e)>(q, k, attn, d, st); });
}

cudaError_t simt_attention_backward3d(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk,
                                      void *ws, Dims3 d, int dtype, cudaStream_t st)
{
    float *rho = reinterpret_cast<float *>(ws);
    return with_elem(dtype, [&](auto e) { return bwd_typed<decltype(e)>(dattn, attn, q, k, dq, dk, rho, d, st); });
}

}  // namespace cca
