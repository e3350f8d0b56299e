// Generic CUDA-core kernels of the attention map attn[B,H,W,H+W] (cc_attention/functions.py:40, the softmax output
// `concate`) and of its gradient w.r.t. q, k, for NCHW q, k of any Cq and line length (the shapes the tensor-core kernels of
// cca_tc_attn.cuh do not cover, and impl="simt").  Kept plain: one warp per pixel, sums in a fixed order, no atomics.  (A
// translation unit of their own, so that cca_simt.cu and its line kernels stay as they are.)
#include "cca_common.cuh"

namespace cca {
namespace {

constexpr int kThreads = 256;

// attn[b,h,w,g]: g < H column key (g, w), g >= H row key (h, g - H)
constexpr int kMapWarps = kThreads / 32;

// offset (inside a sample's [H,W] plane) of key g of pixel (h, w)
__device__ __forceinline__ long map_key(int g, int h, int w, Dims d) { return g < d.H ? (long)g * d.W + w : (long)h * d.W + (g - d.H); }

// logits into the row, then max, log-sum-exp2 and the normalised row in place (each lane rereads only what it wrote)
template <typename T>
__global__ void __launch_bounds__(kThreads) cca_attn_map_kernel(const T *__restrict__ q, const T *__restrict__ k, float *__restrict__ attn, Dims d)
{
    const long hw = (long)d.H * d.W, npix = hw * d.B;
    const int hw2 = d.H + d.W, lane = threadIdx.x & 31;
    for (long p = (long)blockIdx.x * kMapWarps + (threadIdx.x >> 5); p < npix; p += (long)gridDim.x * kMapWarps) {
        const long b = p / hw, s = p - b * hw;
        const int h = (int)(s / d.W), w = (int)(s - (long)h * d.W);
        const T *qb = q + b * d.Cq * hw + s, *kb = k + b * d.Cq * hw;
        float *row = attn + p * hw2;
        float m = -INFINITY;
        for (int g = lane; g < hw2; g += 32) {
            float e = -INFINITY;                                   // the self entry (functions.py:38, INF)
            if (g != h) {
                const long ko = map_key(g, h, w, d);
                e = 0.f;
                for (int c = 0; c < d.Cq; ++c) e = fmaf(ldg_f(qb + c * hw), ldg_f(kb + c * hw + ko), e);
            }
            row[g] = e;
            m = fmaxf(m, e);
        }
        m = warp_max(m) * kLog2e;
        float l = 0.f;
        for (int g = lane; g < hw2; g += 32) l += exp2f(fmaf(row[g], kLog2e, -m));
        const float lse2 = m + log2f(warp_sum(l));
        for (int g = lane; g < hw2; g += 32) row[g] = exp2f(fmaf(row[g], kLog2e, -lse2));
    }
}

__global__ void __launch_bounds__(kThreads) cca_attn_rho_kernel(const float *__restrict__ dattn, const float *__restrict__ attn,
                                                                float *__restrict__ rho, long npix, int hw2, uint4 *c0, uint4 *c1,
                                                                long n16)
{
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // the item kernel waits for this grid before it reads rho
    const long tid = (long)blockIdx.x * blockDim.x + threadIdx.x, nth = (long)gridDim.x * blockDim.x;
    for (long i = tid; i < n16; i += nth) { c0[i] = make_uint4(0, 0, 0, 0); c1[i] = make_uint4(0, 0, 0, 0); }
    const int lane = threadIdx.x & 31;
    for (long p = (long)blockIdx.x * kMapWarps + (threadIdx.x >> 5); p < npix; p += (long)gridDim.x * kMapWarps) {
        const float *a = attn + p * hw2, *da = dattn + p * hw2;
        float s = 0.f;
        for (int g = lane; g < hw2; g += 32) s = fmaf(__ldg(a + g), __ldg(da + g), s);
        s = warp_sum(s);
        if (lane == 0) rho[p] = s;
    }
}

// dq[b,c,h,w] = sum_g dS[p,g] k[b,c,key g]; lanes own channels, the keys are walked in order
template <typename T>
__global__ void __launch_bounds__(kThreads) cca_attn_dq_kernel(const float *__restrict__ dattn, const float *__restrict__ attn,
                                                               const float *__restrict__ rho, const T *__restrict__ k,
                                                               T *__restrict__ dq, Dims d)
{
    const long hw = (long)d.H * d.W, npix = hw * d.B;
    const int hw2 = d.H + d.W, lane = threadIdx.x & 31;
    for (long p = (long)blockIdx.x * kMapWarps + (threadIdx.x >> 5); p < npix; p += (long)gridDim.x * kMapWarps) {
        const long b = p / hw, s = p - b * hw;
        const int h = (int)(s / d.W), w = (int)(s - (long)h * d.W);
        const float *a = attn + p * hw2, *da = dattn + p * hw2;
        const float r = rho[p];
        for (int c0 = 0; c0 < d.Cq; c0 += 32) {
            const int c = c0 + lane;
            const T *kc = k + (b * d.Cq + (c < d.Cq ? c : 0)) * hw;
            float acc = 0.f;
            for (int g = 0; g < hw2; ++g) {
                if (g == h) continue;                                  // the self entry does not depend on q, k
                const float ds = __ldg(a + g) * (__ldg(da + g) - r);
                acc = fmaf(ds, ldg_f(kc + map_key(g, h, w, d)), acc);
            }
            if (c < d.Cq) dq[(b * d.Cq + c) * hw + s] = from_f<T>(acc);
        }
    }
}

// dk[b,c,y,x] = sum over the queries whose map holds key (y, x) -- column queries (h, x), h != y (entry y) and row queries
// (y, w) (entry H + x) -- of dS * q; a gather in a fixed order, no atomics
template <typename T>
__global__ void __launch_bounds__(kThreads) cca_attn_dk_kernel(const float *__restrict__ dattn, const float *__restrict__ attn,
                                                               const float *__restrict__ rho, const T *__restrict__ q,
                                                               T *__restrict__ dk, Dims d)
{
    const long hw = (long)d.H * d.W, npix = hw * d.B;
    const int hw2 = d.H + d.W, lane = threadIdx.x & 31;
    for (long p = (long)blockIdx.x * kMapWarps + (threadIdx.x >> 5); p < npix; p += (long)gridDim.x * kMapWarps) {
        const long b = p / hw, s = p - b * hw;
        const int y = (int)(s / d.W), x = (int)(s - (long)y * d.W);
        for (int c0 = 0; c0 < d.Cq; c0 += 32) {
            const int c = c0 + lane;
            const T *qc = q + (b * d.Cq + (c < d.Cq ? c : 0)) * hw;
            float acc = 0.f;
            for (int i = 0; i < hw2; ++i) {
                const bool col = i < d.H;
                if (col && i == y) continue;
                const long qs = col ? (long)i * d.W + x : (long)y * d.W + (i - d.H);   // query pixel inside the sample
                const long e = (b * hw + qs) * hw2 + (col ? y : d.H + x);
                const float ds = __ldg(attn + e) * (__ldg(dattn + e) - rho[b * hw + qs]);
                acc = fmaf(ds, ldg_f(qc + qs), acc);
            }
            if (c < d.Cq) dk[(b * d.Cq + c) * hw + s] = from_f<T>(acc);
        }
    }
}

template <typename T>
cudaError_t attn_fwd_typed(const void *q, const void *k, float *attn, Dims d, cudaStream_t st)
{
    const long npix = (long)d.B * d.H * d.W;
    cca_attn_map_kernel<T><<<warp_grid(npix, kMapWarps), kThreads, 0, st>>>((const T *)q, (const T *)k, attn, d);
    count_launch();
    return cudaGetLastError();
}

template <typename T>
cudaError_t attn_bwd_typed(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk, void *ws, Dims d,
                           cudaStream_t st)
{
    const long npix = (long)d.B * d.H * d.W;
    float *rho = reinterpret_cast<float *>(ws);
    cudaError_t e = attn_rho(dattn, attn, rho, npix, d.H + d.W, nullptr, nullptr, 0, st);
    if (e != cudaSuccess) return e;
    cca_attn_dq_kernel<T><<<warp_grid(npix, kMapWarps), kThreads, 0, st>>>(dattn, attn, rho, (const T *)k, (T *)dq, d);
    count_launch();
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    cca_attn_dk_kernel<T><<<warp_grid(npix, kMapWarps), kThreads, 0, st>>>(dattn, attn, rho, (const T *)q, (T *)dk, d);
    count_launch();
    return cudaGetLastError();
}

}  // namespace

cudaError_t attn_rho(const float *dattn, const float *attn, float *rho, long npix, int hw2, void *c0, void *c1, long clear_bytes,
                     cudaStream_t st)
{
    cca_attn_rho_kernel<<<warp_grid(npix, kMapWarps), kThreads, 0, st>>>(dattn, attn, rho, npix, hw2, reinterpret_cast<uint4 *>(c0),
                                                           reinterpret_cast<uint4 *>(c1), clear_bytes / 16);
    count_launch();
    return cudaGetLastError();
}

size_t simt_attention_workspace(int backward, Dims d) { return backward ? (size_t)d.B * d.H * d.W * sizeof(float) + 16 : 16; }

cudaError_t simt_attention_forward(const void *q, const void *k, float *attn, Dims d, int dtype, cudaStream_t st)
{
    return with_elem(dtype, [&](auto e) { return attn_fwd_typed<decltype(e)>(q, k, attn, d, st); });
}

cudaError_t simt_attention_backward(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk,
                                    void *ws, Dims d, int dtype, cudaStream_t st)
{
    return with_elem(dtype, [&](auto e) { return attn_bwd_typed<decltype(e)>(dattn, attn, q, k, dq, dk, ws, d, st); });
}

}  // namespace cca
