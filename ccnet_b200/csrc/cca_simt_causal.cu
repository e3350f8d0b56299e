// Generic CUDA-core kernels of causal criss-cross attention over clips (CCA_FLAG_CAUSAL), NCDHW tensors of any Cq and C: the
// key set of pixel (b,t,h,w) is its column (self masked), its row and the time keys (b,s,h,w) with lo(t) <= s < t, where
// lo(t) = max(0, t - window) (0 without a window), so Le = H + W - 1 + t - lo(t) varies per pixel.  The kernels follow the bidirectional ones of cca_simt_3d.cu and cca_simt_attn3d.cu
// (same warp layout, sums in the same order), which keep their own code.  The key set is no longer symmetric: the backward
// and the map backward gather dk and dv of a key pixel of frame t from the time queries u > t (the transposed time set) and,
// as before, from the column and row queries.  Nothing is added atomically: the results are deterministic.
//
// The streaming step (simt_forward3d_step): one warp per pixel of the new frame over its column (self masked), its row and
// the S past frames of the rings (frame j in slot (head + j) % N), in that order, with the arithmetic of the causal forward's
// last frame.
#include "cca_common.cuh"

namespace cca {
namespace {

// ---- the op
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
// first time key of frame t: max(0, t - window)
__device__ __forceinline__ int time_lo(int t, const Dims3 &d) { return t - min(t, d.time_keys()); }
// the longest walk of the backward: column and row, and up to d.time_keys() frames on each side of t
__host__ __device__ inline int bwd_walk(const Dims3 &d) { return d.H + d.W - 1 + min(d.T - 1, 2 * d.time_keys()); }

// volume offset of entry i of pixel x's walk: column (g != h), row, then the time entries from frame lo on -- with `causal`
// the frames lo <= s < t (the forward's key set), else the frames s != t from lo on (the backward's walk)
__device__ __forceinline__ int key_off(int i, const Pix &x, const Dims3 &d, int lo, bool causal)
{
    if (i < d.H - 1) return (x.t * d.H + (i < x.h ? i : i + 1)) * d.W + x.w;
    i -= d.H - 1;
    if (i < d.W) return (x.t * d.H + x.h) * d.W + i;
    i += lo - d.W;
    return ((causal || i < x.t ? i : i + 1) * d.H + x.h) * d.W + x.w;
}

// out = sum_j P_j v_j, lse = log sum_j exp(q . k_j) over the H + W - 1 + t - lo(t) keys of frame t (shared memory laid out
// for the longest set, H + W - 1 + d.time_keys())
template <typename E>
__global__ void __launch_bounds__(kThreads3) cca_simt3d_causal_fwd_kernel(const E *__restrict__ q, const E *__restrict__ k,
                                                                           const E *__restrict__ v, E *__restrict__ out,
                                                                           float *__restrict__ lse, Dims3 d)
{
    extern __shared__ float sm3[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, Lmax = d.H + d.W - 1 + d.time_keys();
    float *row = sm3 + (long)warp * 2 * Lmax;
    int *offs = reinterpret_cast<int *>(row + Lmax);
    const long hw = (long)d.H * d.W, vol = hw * d.T, npix = vol * d.B;
    for (long p = (long)blockIdx.x * kWarps3 + warp; p < npix; p += (long)gridDim.x * kWarps3) {
        const Pix x = pix_of(p, d, vol, hw);
        const int lo = time_lo(x.t, d), Le = d.H + d.W - 1 + x.t - lo;
        const E *qp = q + x.b * d.Cq * vol + x.off, *kb = k + x.b * d.Cq * vol;
        float m = -INFINITY;
        for (int i = lane; i < Le; i += 32) {
            const int o = key_off(i, x, d, lo, true);
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

// Pixel p as a query: dq_p = sum_n dS_pn k_n.  As a key: dk_p = sum_n dS_np q_n, dv_p = sum_n P_np dout_n over the queries n
// that see p.  dS_uj = P_uj (dout_u . v_j - delta_u), P_uj = exp(q_u . k_j - lse_u).  The column and row parts are symmetric,
// as in the bidirectional kernel, but the time queries of p (frame t) are the frames t < u <= t + window while its time keys
// are the frames t - window <= s < t: the walk covers those frames of the line once, in ascending order, entry s < t weighing
// as a key of p (sq) and entry u > t as a query (pk, sk), the other weights 0 -- the transposed set, gathered, not
// scattered.  The walk has up to H + W - 1 + 2 window entries: the time entries' offsets are recomputed instead of staged,
// so that shared memory holds 3 floats per entry and an int per column and row entry.
template <typename E>
__global__ void __launch_bounds__(kThreads3) cca_simt3d_causal_bwd_kernel(const E *__restrict__ dout, const E *__restrict__ q,
                                                                           const E *__restrict__ k, const E *__restrict__ v,
                                                                           const float *__restrict__ lse,
                                                                           const float *__restrict__ delta, E *__restrict__ dq,
                                                                           E *__restrict__ dk, E *__restrict__ dv, Dims3 d)
{
    extern __shared__ float sm3[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n2 = d.H + d.W - 1, Lmax = bwd_walk(d);
    float *sq = sm3 + (long)warp * (3 * Lmax + n2), *pk = sq + Lmax, *sk = pk + Lmax;
    int *offs = reinterpret_cast<int *>(sk + Lmax);
    const long hw = (long)d.H * d.W, vol = hw * d.T, npix = vol * d.B;
    for (long p = (long)blockIdx.x * kWarps3 + warp; p < npix; p += (long)gridDim.x * kWarps3) {
        const Pix x = pix_of(p, d, vol, hw);
        const int lo = time_lo(x.t, d), nk = x.t - lo, Le = n2 + nk + min(d.T - 1 - x.t, d.time_keys());
        const long sq0 = x.b * d.Cq * vol, sv0 = x.b * d.C * vol, s0 = x.b * vol;
        const E *qb = q + sq0, *kb = k + sq0, *vb = v + sv0, *gb = dout + sv0;
        const float lse_p = lse[p], delta_p = delta[p];
        for (int i = lane; i < Le; i += 32) {
            const int o = key_off(i, x, d, lo, false);
            const bool key = i < n2 + nk;                                 // o is a key of p
            const bool query = i < n2 || !key;                            // p is a key of o
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
            sq[i] = key ? p1 * (g1 - delta_p) : 0.f;
            pk[i] = query ? p2 : 0.f;
            sk[i] = query ? p2 * (g2 - delta[s0 + o]) : 0.f;
            if (i < n2) offs[i] = o;
        }
        __syncwarp();
        // the time entries from n2 on: frames lo, lo + 1, ... skipping t, at offset s * hw + (the pixel's offset in its frame)
        const int t0 = (int)(x.off - x.t * hw), tskip = n2 + nk;
        for (int c = lane; c < d.Cq; c += 32) {
            const E *kc = kb + c * vol, *qc = qb + c * vol;
            float a = 0.f, b = 0.f;
            for (int i = 0; i < n2; ++i) {
                a = fmaf(sq[i], ldg_f(kc + offs[i]), a);
                b = fmaf(sk[i], ldg_f(qc + offs[i]), b);
            }
            for (int i = n2, o = lo * (int)hw + t0; i < Le; ++i, o += (int)hw) {
                if (i == tskip) o += (int)hw;
                a = fmaf(sq[i], ldg_f(kc + o), a);
                b = fmaf(sk[i], ldg_f(qc + o), b);
            }
            dq[sq0 + c * vol + x.off] = from_f<E>(a);
            dk[sq0 + c * vol + x.off] = from_f<E>(b);
        }
        for (int c = lane; c < d.C; c += 32) {
            const E *gc = gb + c * vol;
            float a = 0.f;
            for (int i = 0; i < n2; ++i) a = fmaf(pk[i], ldg_f(gc + offs[i]), a);
            for (int i = n2, o = lo * (int)hw + t0; i < Le; ++i, o += (int)hw) {
                if (i == tskip) o += (int)hw;
                a = fmaf(pk[i], ldg_f(gc + o), a);
            }
            dv[sv0 + c * vol + x.off] = from_f<E>(a);
        }
        __syncwarp();
    }
}

// ---- the attention map
constexpr int kMapThreads = 256;
constexpr int kMapWarps = kMapThreads / 32;

// volume offset of key g of pixel x, -1 for the masked entries (the column's self entry; time entries outside [lo, t))
__device__ __forceinline__ long key_of(int g, const Pix &x, const Dims3 &d, long hw, int lo)
{
    if (g < d.H) return g == x.h ? -1 : x.t * hw + (long)g * d.W + x.w;
    g -= d.H;
    if (g < d.W) return x.t * hw + (long)x.h * d.W + g;
    g -= d.W;
    return g >= x.t || g < lo ? -1 : g * hw + (long)x.h * d.W + x.w;
}

// logits into the row, then max, log-sum-exp2 and the normalised row in place (each lane rereads only what it wrote)
template <typename E>
__global__ void __launch_bounds__(kMapThreads) cca_attn3d_causal_map_kernel(const E *__restrict__ q, const E *__restrict__ k,
                                                                           float *__restrict__ attn, Dims3 d)
{
    const long hw = (long)d.H * d.W, vol = hw * d.T, npix = vol * d.B, rl = (long)d.H + d.W + d.T;
    const int lane = threadIdx.x & 31;
    for (long p = (long)blockIdx.x * kMapWarps + (threadIdx.x >> 5); p < npix; p += (long)gridDim.x * kMapWarps) {
        const Pix x = pix_of(p, d, vol, hw);
        const int lo = time_lo(x.t, d);
        const E *qp = q + x.b * d.Cq * vol + x.off, *kb = k + x.b * d.Cq * vol;
        float *row = attn + p * rl;
        float m = -INFINITY;
        for (int g = lane; g < rl; g += 32) {
            const long o = key_of(g, x, d, hw, lo);
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

// dq[b,c,t,h,w] = sum_g dS[p,g] k[b,c,key g]; lanes own channels, the keys are walked in order (the time entries from lo(t)
// to t - 1 only: the others are masked)
template <typename E>
__global__ void __launch_bounds__(kMapThreads) cca_attn3d_causal_dq_kernel(const float *__restrict__ dattn, const float *__restrict__ attn,
                                                                          const float *__restrict__ rho, const E *__restrict__ k,
                                                                          E *__restrict__ dq, Dims3 d)
{
    const long hw = (long)d.H * d.W, vol = hw * d.T, npix = vol * d.B, rl = (long)d.H + d.W + d.T;
    const int lane = threadIdx.x & 31;
    for (long p = (long)blockIdx.x * kMapWarps + (threadIdx.x >> 5); p < npix; p += (long)gridDim.x * kMapWarps) {
        const Pix x = pix_of(p, d, vol, hw);
        const int lo = time_lo(x.t, d), n2 = d.H + d.W, gend = n2 + x.t;
        const float *a = attn + p * rl, *da = dattn + p * rl;
        const float r = rho[p];
        for (int c0 = 0; c0 < d.Cq; c0 += 32) {
            const int c = c0 + lane;
            const E *kc = k + (x.b * d.Cq + (c < d.Cq ? c : 0)) * vol;
            float acc = 0.f;
            for (int g = 0; g < gend; g = g == n2 - 1 ? n2 + lo : g + 1) {
                const long o = key_of(g, x, d, hw, lo);
                if (o < 0) continue;                                   // the masked entries do not depend on q, k
                acc = fmaf(__ldg(a + g) * (__ldg(da + g) - r), ldg_f(kc + o), acc);
            }
            if (c < d.Cq) dq[(x.b * d.Cq + c) * vol + x.off] = from_f<E>(acc);
        }
    }
}

// dk of key pixel (t,y,x) = sum over the queries whose row holds it -- column queries (t,i,x), i != y (entry y), row queries
// (t,y,j) (entry H + x), time queries (s,y,x), t < s <= t + window (the transposed time set) (entry H + W + t) -- of dS * q,
// in that order
template <typename E>
__global__ void __launch_bounds__(kMapThreads) cca_attn3d_causal_dk_kernel(const float *__restrict__ dattn, const float *__restrict__ attn,
                                                                          const float *__restrict__ rho, const E *__restrict__ q,
                                                                          E *__restrict__ dk, Dims3 d)
{
    const long hw = (long)d.H * d.W, vol = hw * d.T, npix = vol * d.B, rl = (long)d.H + d.W + d.T;
    const int lane = threadIdx.x & 31;
    for (long p = (long)blockIdx.x * kMapWarps + (threadIdx.x >> 5); p < npix; p += (long)gridDim.x * kMapWarps) {
        const Pix x = pix_of(p, d, vol, hw);
        const long s0 = x.b * vol;
        for (int c0 = 0; c0 < d.Cq; c0 += 32) {
            const int c = c0 + lane;
            const E *qc = q + (x.b * d.Cq + (c < d.Cq ? c : 0)) * vol;
            float acc = 0.f;
            const int n2 = d.H + d.W, iend = n2 + min(d.T - 1, x.t + d.time_keys()) + 1;
            for (int i = 0; i < iend; i = i == n2 - 1 ? n2 + x.t + 1 : i + 1) {
                long qo, g;                                            // query pixel (volume offset), its entry of this key
                if (i < d.H) {
                    if (i == x.h) continue;
                    qo = x.t * hw + (long)i * d.W + x.w; g = x.h;
                } else if (i < d.H + d.W) {
                    qo = x.t * hw + (long)x.h * d.W + (i - d.H); g = d.H + x.w;
                } else {
                    const int s = i - d.H - d.W;
                    if (s <= x.t) continue;
                    qo = s * hw + (long)x.h * d.W + x.w; g = d.H + d.W + x.t;
                }
                const long e = (s0 + qo) * rl + g;
                acc = fmaf(__ldg(attn + e) * (__ldg(dattn + e) - rho[s0 + qo]), ldg_f(qc + qo), acc);
            }
            if (c < d.Cq) dk[(x.b * d.Cq + c) * vol + x.off] = from_f<E>(acc);
        }
    }
}

// ---- the streaming step
// q, k, v [B,c,H,W] of the new frame, rings kc [B,Cq,N,H,W], vc [B,C,N,H,W] with past frame j < S in slot (head + j) % N:
// out [B,C,H,W], lse [B,H,W]
template <typename E>
__global__ void __launch_bounds__(kThreads3) cca_simt3d_step_kernel(const E *__restrict__ q, const E *__restrict__ k,
                                                                     const E *__restrict__ v, const E *__restrict__ kc,
                                                                     const E *__restrict__ vc, E *__restrict__ out,
                                                                     float *__restrict__ lse, Dims d, int N, int S, int head)
{
    extern __shared__ float sm3[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n2 = d.H + d.W - 1, Le = n2 + S;
    float *row = sm3 + (long)warp * 2 * Le;
    int *offs = reinterpret_cast<int *>(row + Le);
    const long hw = (long)d.H * d.W, cvol = hw * N, npix = hw * d.B;
    for (long p = (long)blockIdx.x * kWarps3 + warp; p < npix; p += (long)gridDim.x * kWarps3) {
        const long b = p / hw, off = p - b * hw;
        const int h = (int)(off / d.W), w = (int)(off - (long)h * d.W);
        const E *qp = q + b * d.Cq * hw + off, *kb = k + b * d.Cq * hw, *kcb = kc + b * d.Cq * cvol;
        float m = -INFINITY;
        for (int i = lane; i < n2; i += 32) {          // column keys (g != h) and row keys of the frame
            const int o = i < d.H - 1 ? (i < h ? i : i + 1) * d.W + w : h * d.W + (i - d.H + 1);
            float e = 0.f;
            for (int c = 0; c < d.Cq; ++c) e = fmaf(ldg_f(qp + c * hw), ldg_f(kb + c * hw + o), e);
            row[i] = e; offs[i] = o;
            m = fmaxf(m, e);
        }
        for (int j = lane; j < S; j += 32) {           // past frame j at (h, w), in its ring slot
            const long ot = (j + head) * hw + off;
            const int o = (int)(ot < cvol ? ot : ot - cvol);
            float e = 0.f;
            for (int c = 0; c < d.Cq; ++c) e = fmaf(ldg_f(qp + c * hw), ldg_f(kcb + c * cvol + o), e);
            row[n2 + j] = e; offs[n2 + j] = o;
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
        const E *vb = v + b * d.C * hw, *vcb = vc + b * d.C * cvol;
        E *op = out + b * d.C * hw + off;
        for (int c = lane; c < d.C; c += 32) {
            const E *vf = vb + c * hw, *vt = vcb + c * cvol;
            float acc = 0.f;
            for (int i = 0; i < n2; ++i) acc = fmaf(row[i], ldg_f(vf + offs[i]), acc);
            for (int i = n2; i < Le; ++i) acc = fmaf(row[i], ldg_f(vt + offs[i]), acc);
            op[c * hw] = from_f<E>(acc);
        }
        __syncwarp();
    }
}

template <typename K, typename... Args> cudaError_t launch(K kern, long npix, int warps, size_t smem, cudaStream_t st, Args... args)
{
    if (smem > 0) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    kern<<<warp_grid(npix, warps), 32 * warps, smem, st>>>(args...);
    count_launch();
    return cudaGetLastError();
}

}  // namespace

cudaError_t simt_forward3d_causal(const void *q, const void *k, const void *v, void *out, float *lse, Dims3 d, int dtype,
                                  cudaStream_t st)
{
    const long npix = (long)d.B * d.T * d.H * d.W;
    const size_t smem = (size_t)kWarps3 * 2 * (d.H + d.W - 1 + d.time_keys()) * sizeof(float);
    return with_elem(dtype, [&](auto e) {
        using E = decltype(e);
        return launch(cca_simt3d_causal_fwd_kernel<E>, npix, kWarps3, smem, st, (const E *)q, (const E *)k, (const E *)v, (E *)out,
                      lse, d);
    });
}

cudaError_t simt_backward3d_causal(const void *dout, const void *q, const void *k, const void *v, const void *out,
                                   const float *lse, void *dq, void *dk, void *dv, void *ws, Dims3 d, int dtype, cudaStream_t st)
{
    const long npix = (long)d.B * d.T * d.H * d.W;
    const size_t smem = (size_t)kWarps3 * (3 * bwd_walk(d) + d.H + d.W - 1) * sizeof(float);
    float *delta = reinterpret_cast<float *>(ws);
    return with_elem(dtype, [&](auto e) {
        using E = decltype(e);
        cudaError_t r = launch(cca_simt3d_delta_kernel<E>, npix, kWarps3, 0, st, (const E *)dout, (const E *)out, delta, d);
        if (r != cudaSuccess) return r;
        return launch(cca_simt3d_causal_bwd_kernel<E>, npix, kWarps3, smem, st, (const E *)dout, (const E *)q, (const E *)k,
                      (const E *)v, lse, (const float *)delta, (E *)dq, (E *)dk, (E *)dv, d);
    });
}

cudaError_t simt_attention_forward3d_causal(const void *q, const void *k, float *attn, Dims3 d, int dtype, cudaStream_t st)
{
    const long npix = (long)d.B * d.T * d.H * d.W;
    return with_elem(dtype, [&](auto e) {
        using E = decltype(e);
        return launch(cca_attn3d_causal_map_kernel<E>, npix, kMapWarps, 0, st, (const E *)q, (const E *)k, attn, d);
    });
}

cudaError_t simt_attention_backward3d_causal(const float *dattn, const float *attn, const void *q, const void *k, void *dq, void *dk,
                                             void *ws, Dims3 d, int dtype, cudaStream_t st)
{
    const long npix = (long)d.B * d.T * d.H * d.W;
    float *rho = reinterpret_cast<float *>(ws);
    cudaError_t r = attn_rho(dattn, attn, rho, npix, d.H + d.W + d.T, nullptr, nullptr, 0, st);
    if (r != cudaSuccess) return r;
    return with_elem(dtype, [&](auto e) {
        using E = decltype(e);
        cudaError_t r2 = launch(cca_attn3d_causal_dq_kernel<E>, npix, kMapWarps, 0, st, dattn, attn, (const float *)rho, (const E *)k,
                                (E *)dq, d);
        if (r2 != cudaSuccess) return r2;
        return launch(cca_attn3d_causal_dk_kernel<E>, npix, kMapWarps, 0, st, dattn, attn, (const float *)rho, (const E *)q, (E *)dk, d);
    });
}

cudaError_t simt_forward3d_step(const void *q, const void *k, const void *v, const void *kc, const void *vc, void *out, float *lse,
                                Dims d, int N, int S, int head, int dtype, cudaStream_t st)
{
    const long npix = (long)d.B * d.H * d.W;
    const size_t smem = (size_t)kWarps3 * 2 * (d.H + d.W - 1 + S) * sizeof(float);
    return with_elem(dtype, [&](auto e) {
        using E = decltype(e);
        return launch(cca_simt3d_step_kernel<E>, npix, kWarps3, smem, st, (const E *)q, (const E *)k, (const E *)v, (const E *)kc,
                      (const E *)vc, (E *)out, lse, d, N, S, head);
    });
}

}  // namespace cca
