// Generic CUDA-core kernels of criss-cross attention over clips (the 3D op), for NCDHW-contiguous q, k [B,Cq,T,H,W] and
// v, out [B,C,T,H,W] of any Cq and C: the shapes the tensor-core path of cca_tc_time.cu does not cover (other channel
// counts, T > kTimeMaxT, lines over 896 pixels), impl="simt", and the independent GPU cross-check of that path.
//
// Key set of pixel (b,t,h,w), in this order (the masked self entries of the column and time branches are skipped, the row
// branch keeps its self entry): column (b,t,g,w) g != h, row (b,t,h,g), time (b,s,h,w) s != t -- Le = H + W + T - 2 keys.
// The set is symmetric: the queries that see key pixel j are exactly j's own key set, which lets the backward GATHER dk
// and dv per key pixel instead of scattering them.  One warp per pixel; the per-key values live in shared memory, so the
// kernels take Le <= kMaxKeys3d (H + W + T - 2 <= 2048).  Sums run in a fixed order and nothing is added atomically: the
// results are deterministic.  Plain fp32 FMA, outputs rounded to the I/O type once.
#include "cca_common.cuh"

namespace cca {
namespace {

constexpr int kWarps3 = 4;
constexpr int kThreads3 = 32 * kWarps3;


struct Pix {
    long b, off;   // sample, offset inside the sample's [T,H,W] volume
    int t, h, w;
};
__device__ __forceinline__ Pix pix_of(long p, const Dims3 &d, long vol, long hw)
{
    Pix x;
    x.b = p / vol; x.off = p - x.b * vol;
    x.t = (int)(x.off / hw);
    const long r = x.off - x.t * hw;
    x.h = (int)(r / d.W); x.w = (int)(r - (long)x.h * d.W);
    return x;
}
// volume offset of key i of pixel x
__device__ __forceinline__ int key_off(int i, const Pix &x, const Dims3 &d)
{
    if (i < d.H - 1) return (x.t * d.H + (i < x.h ? i : i + 1)) * d.W + x.w;
    i -= d.H - 1;
    if (i < d.W) return (x.t * d.H + x.h) * d.W + i;
    i -= d.W;
    return ((i < x.t ? i : i + 1) * d.H + x.h) * d.W + x.w;
}

// out = sum_j P_j v_j, lse = log sum_j exp(q . k_j)
template <typename E>
__global__ void __launch_bounds__(kThreads3) cca_simt3d_fwd_kernel(const E *__restrict__ q, const E *__restrict__ k,
                                                                    const E *__restrict__ v, E *__restrict__ out,
                                                                    float *__restrict__ lse, Dims3 d)
{
    extern __shared__ float sm3[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, Le = d.H + d.W + d.T - 2;
    float *row = sm3 + (long)warp * 2 * Le;
    int *offs = reinterpret_cast<int *>(row + Le);
    const long hw = (long)d.H * d.W, vol = hw * d.T, npix = vol * d.B;
    for (long p = (long)blockIdx.x * kWarps3 + warp; p < npix; p += (long)gridDim.x * kWarps3) {
        const Pix x = pix_of(p, d, vol, hw);
        const E *qp = q + x.b * d.Cq * vol + x.off, *kb = k + x.b * d.Cq * vol;
        float m = -INFINITY;
        for (int i = lane; i < Le; i += 32) {
            const int o = key_off(i, x, d);
            float e = 0.f;
            for (int c = 0; c < d.Cq; ++c) e = fmaf(ldg_f(qp + c * vol), ldg_f(kb + c * vol + o), e);
            row[i] = e; offs[i] = o;
            m = fmaxf(m, e);
        }
        m = warp_max(m);
        float l = 0.f;
        for (int i = lane; i < Le; i += 32) {
            const float pe = expf(row[i] - m);
            row[i] = pe;
            l += pe;
        }
        l = warp_sum(l);
        const float inv = 1.f / l;
        for (int i = lane; i < Le; i += 32) row[i] *= inv;
        if (lane == 0) lse[p] = m + logf(l);
        __syncwarp();
        const E *vb = v + x.b * d.C * vol;
        E *op = out + x.b * d.C * vol + x.off;
        for (int c = lane; c < d.C; c += 32) {
            const E *vc = vb + c * vol;
            float acc = 0.f;
            for (int i = 0; i < Le; ++i) acc = fmaf(row[i], ldg_f(vc + offs[i]), acc);
            op[c * vol] = from_f<E>(acc);
        }
        __syncwarp();
    }
}

// delta[p] = <dout_p, out_p>
template <typename E>
__global__ void __launch_bounds__(kThreads3) cca_simt3d_delta_kernel(const E *__restrict__ dout, const E *__restrict__ out,
                                                                      float *__restrict__ delta, Dims3 d)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long hw = (long)d.H * d.W, vol = hw * d.T, npix = vol * d.B;
    for (long p = (long)blockIdx.x * kWarps3 + warp; p < npix; p += (long)gridDim.x * kWarps3) {
        const long b = p / vol, off = p - b * vol;
        const E *g = dout + b * d.C * vol + off, *o = out + b * d.C * vol + off;
        float s = 0.f;
        for (int c = lane; c < d.C; c += 32) s = fmaf(ldg_f(g + c * vol), ldg_f(o + c * vol), s);
        s = warp_sum(s);
        if (lane == 0) delta[p] = s;
    }
}

// Pixel p as a query: dq_p = sum_n dS_pn k_n.  As a key (its queries are its own key set): dk_p = sum_n dS_np q_n,
// dv_p = sum_n P_np dout_n.  dS_uj = P_uj (dout_u . v_j - delta_u), P_uj = exp(q_u . k_j - lse_u).
template <typename E>
__global__ void __launch_bounds__(kThreads3) cca_simt3d_bwd_kernel(const E *__restrict__ dout, const E *__restrict__ q,
                                                                    const E *__restrict__ k, const E *__restrict__ v,
                                                                    const float *__restrict__ lse,
                                                                    const float *__restrict__ delta, E *__restrict__ dq,
                                                                    E *__restrict__ dk, E *__restrict__ dv, Dims3 d)
{
    extern __shared__ float sm3[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, Le = d.H + d.W + d.T - 2;
    float *sq = sm3 + (long)warp * 4 * Le, *pk = sq + Le, *sk = pk + Le;
    int *offs = reinterpret_cast<int *>(sk + Le);
    const long hw = (long)d.H * d.W, vol = hw * d.T, npix = vol * d.B;
    for (long p = (long)blockIdx.x * kWarps3 + warp; p < npix; p += (long)gridDim.x * kWarps3) {
        const Pix x = pix_of(p, d, vol, hw);
        const long sq0 = x.b * d.Cq * vol, sv0 = x.b * d.C * vol, s0 = x.b * vol;
        const E *qb = q + sq0, *kb = k + sq0, *vb = v + sv0, *gb = dout + sv0;
        const float lse_p = lse[p], delta_p = delta[p];
        for (int i = lane; i < Le; i += 32) {
            const int o = key_off(i, x, d);
            float e1 = 0.f, e2 = 0.f, g1 = 0.f, g2 = 0.f;
            for (int c = 0; c < d.Cq; ++c) {
                e1 = fmaf(ldg_f(qb + c * vol + x.off), ldg_f(kb + c * vol + o), e1);
                e2 = fmaf(ldg_f(qb + c * vol + o), ldg_f(kb + c * vol + x.off), e2);
            }
            for (int c = 0; c < d.C; ++c) {
                g1 = fmaf(ldg_f(gb + c * vol + x.off), ldg_f(vb + c * vol + o), g1);
                g2 = fmaf(ldg_f(gb + c * vol + o), ldg_f(vb + c * vol + x.off), g2);
            }
            const float p1 = expf(e1 - lse_p), p2 = expf(e2 - lse[s0 + o]);
            sq[i] = p1 * (g1 - delta_p);
            pk[i] = p2;
            sk[i] = p2 * (g2 - delta[s0 + o]);
            offs[i] = o;
        }
        __syncwarp();
        for (int c = lane; c < d.Cq; c += 32) {
            const E *kc = kb + c * vol, *qc = qb + c * vol;
            float a = 0.f, b = 0.f;
            for (int i = 0; i < Le; ++i) {
                a = fmaf(sq[i], ldg_f(kc + offs[i]), a);
                b = fmaf(sk[i], ldg_f(qc + offs[i]), b);
            }
            dq[sq0 + c * vol + x.off] = from_f<E>(a);
            dk[sq0 + c * vol + x.off] = from_f<E>(b);
        }
        for (int c = lane; c < d.C; c += 32) {
            const E *gc = gb + c * vol;
            float a = 0.f;
            for (int i = 0; i < Le; ++i) a = fmaf(pk[i], ldg_f(gc + offs[i]), a);
            dv[sv0 + c * vol + x.off] = from_f<E>(a);
        }
        __syncwarp();
    }
}

template <typename E>
cudaError_t fwd3(const void *q, const void *k, const void *v, void *out, float *lse, Dims3 d, cudaStream_t st)
{
    const long npix = (long)d.B * d.T * d.H * d.W;
    const size_t smem = (size_t)kWarps3 * 2 * (d.H + d.W + d.T - 2) * sizeof(float);
    cudaError_t e = cudaFuncSetAttribute(cca_simt3d_fwd_kernel<E>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    cca_simt3d_fwd_kernel<E><<<warp_grid(npix, kWarps3), kThreads3, smem, st>>>(static_cast<const E *>(q), static_cast<const E *>(k),
                                                                       static_cast<const E *>(v), static_cast<E *>(out), lse, d);
    count_launch();
    return cudaGetLastError();
}

template <typename E>
cudaError_t bwd3(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse, void *dq,
                 void *dk, void *dv, float *delta, Dims3 d, cudaStream_t st)
{
    const long npix = (long)d.B * d.T * d.H * d.W;
    cca_simt3d_delta_kernel<E><<<warp_grid(npix, kWarps3), kThreads3, 0, st>>>(static_cast<const E *>(dout),
                                                                                  static_cast<const E *>(out), delta, d);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const size_t smem = (size_t)kWarps3 * 4 * (d.H + d.W + d.T - 2) * sizeof(float);
    if ((e = cudaFuncSetAttribute(cca_simt3d_bwd_kernel<E>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess)
        return e;
    cca_simt3d_bwd_kernel<E><<<warp_grid(npix, kWarps3), kThreads3, smem, st>>>(
        static_cast<const E *>(dout), static_cast<const E *>(q), static_cast<const E *>(k), static_cast<const E *>(v), lse,
        delta, static_cast<E *>(dq), static_cast<E *>(dk), static_cast<E *>(dv), d);
    count_launch();
    return cudaGetLastError();
}

}  // namespace

bool simt3d_supported(Dims3 d)
{
    const long le = (long)d.H + d.W - 1 + d.time_keys();      // (H + W + T - 2 without a window)
    return le >= 1 && le <= kMaxKeys3d && (long)d.T * d.H * d.W < (1L << 31);
}

size_t simt3d_workspace(int which, Dims3 d)
{
    return (which == CCA_WS_BACKWARD ? (size_t)d.B * d.T * d.H * d.W * sizeof(float) : 0) + 16;
}

cudaError_t simt_forward3d(const void *q, const void *k, const void *v, void *out, float *lse, Dims3 d, int dtype, cudaStream_t st)
{
    return with_elem(dtype, [&](auto e) { return fwd3<decltype(e)>(q, k, v, out, lse, d, st); });
}

cudaError_t simt_backward3d(const void *dout, const void *q, const void *k, const void *v, const void *out, const float *lse,
                            void *dq, void *dk, void *dv, void *ws, Dims3 d, int dtype, cudaStream_t st)
{
    float *delta = reinterpret_cast<float *>(ws);
    return with_elem(dtype, [&](auto e) { return bwd3<decltype(e)>(dout, q, k, v, out, lse, dq, dk, dv, delta, d, st); });
}

}  // namespace cca
